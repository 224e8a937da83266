"""numpy dtypes byte-compatible with the reference PODs (and with include/etx_b200.h).

Each dtype cites the reference struct it mirrors; sizes are asserted at import time and checked
against the compiled reference headers by tests/test_layout.py (oracle_sizeof).
"""
import numpy as np

INVALID = 0xFFFFFFFF

f4, u4, u2, u8 = np.float32, np.uint32, np.uint16, np.uint64

# etx::ArrayView<T>  (render/shared/base.hxx:52-56)
ARRAY_VIEW = np.dtype([("a", u8), ("count", u8)])

# etx::Vertex (render/shared/math.hxx:599) 56 B
VERTEX = np.dtype([("pos", f4, 3), ("nrm", f4, 3), ("tan", f4, 3), ("btn", f4, 3), ("tex", f4, 2)])
# etx::Triangle (math.hxx:607) 32 B
TRIANGLE = np.dtype([("i", u4, 3), ("material_index", u4), ("geo_n", f4, 3), ("pad", f4)])

SPECTRAL_IMAGE = np.dtype([("spectrum_index", u4), ("image_index", u4)])
SAMPLED_IMAGE = np.dtype([("value", f4, 4), ("image_index", u4), ("channel", u4)])
REFRACTIVE_INDEX = np.dtype([("cls", u4), ("eta_index", u4), ("k_index", u4)])
THINFILM = np.dtype([("ior", REFRACTIVE_INDEX), ("thickness_image", u4), ("min_thickness", f4), ("max_thickness", f4), ("pad", f4)])
SUBSURFACE = np.dtype([("spectrum_index", u4), ("image_index", u4), ("cls", u4), ("path", u4)])

# etx::Material (render/shared/material.hxx:52-97) 200 B
MATERIAL = np.dtype([
    ("reflectance", SPECTRAL_IMAGE), ("scattering", SPECTRAL_IMAGE), ("emission", SPECTRAL_IMAGE),
    ("roughness", SAMPLED_IMAGE), ("metalness", SAMPLED_IMAGE), ("transmission", SAMPLED_IMAGE),
    ("subsurface", SUBSURFACE), ("thinfilm", THINFILM),
    ("ext_ior", REFRACTIVE_INDEX), ("int_ior", REFRACTIVE_INDEX),
    ("cls", u4), ("int_medium", u4), ("ext_medium", u4), ("normal_image_index", u4),
    ("diffuse_variation", u4), ("two_sided", u4),
    ("normal_scale", f4), ("opacity", f4), ("emission_collimation", f4),
])

# etx::EmitterProfile (render/shared/emitter.hxx:7-42) 48 B
EMITTER_PROFILE = np.dtype([
    ("emission", SPECTRAL_IMAGE), ("direction", f4, 3), ("cls", u4),
    ("angular_size", f4), ("equivalent_disk_size", f4), ("angular_size_cosine", f4), ("pad", f4, 3),
])
# etx::Emitter (emitter.hxx:44-71) 32 B
EMITTER = np.dtype([
    ("cls", u4), ("profile", u4), ("triangle_index", u4),
    ("spectrum_weight", f4), ("additional_weight", f4), ("triangle_area", f4), ("pad", f4, 2),
])

# etx::SpectralDistribution (render/shared/spectrum.hxx:449-) 3552 B
SPECTRUM = np.dtype([
    ("entries", [("wavelength", f4), ("power", f4)], 441), ("entry_count", u4), ("integrated", f4, 3), ("pad", u4, 2),
])

DIST_ENTRY = np.dtype([("value", f4), ("pdf", f4), ("cdf", f4)])
DISTRIBUTION = np.dtype([("values", ARRAY_VIEW), ("total_weight", f4), ("pad", u4, 3)])

# etx::Image (render/shared/image.hxx:8-50) 112 B
IMAGE = np.dtype([
    ("pixels", ARRAY_VIEW), ("x_distributions", ARRAY_VIEW), ("y_distribution", DISTRIBUTION),
    ("fsize", f4, 2), ("offset", f4, 2), ("scale", f4, 2), ("isize", u4, 2),
    ("normalization", f4), ("options", u4), ("format", u4), ("data_size", u4),
])

# etx::Medium (render/shared/medium.hxx:8-47) 80 B
MEDIUM = np.dtype([
    ("density", ARRAY_VIEW), ("bounds_min", f4, 3), ("bounds_pad0", f4), ("bounds_max", f4, 3), ("bounds_pad1", f4),
    ("cls", u2), ("enable_explicit_connections", u2), ("absorption_index", u4), ("scattering_index", u4),
    ("phase_function_g", f4), ("max_sigma", f4), ("dimensions", u4, 3),
])

# etx::Camera (render/shared/camera.hxx:8-39) 176 B
CAMERA = np.dtype([
    ("view_proj", f4, 16), ("position", f4, 3), ("cls", u4), ("target", f4, 3), ("tan_half_fov", f4),
    ("side", f4, 3), ("aspect", f4), ("up", f4, 3), ("area", f4), ("direction", f4, 3), ("image_plane", f4),
    ("film_size", u4, 2), ("lens_radius", f4), ("focal_distance", f4),
    ("clip_near", f4), ("clip_far", f4), ("lens_image", u4), ("medium_index", u4),
])

# etx::Scene (render/shared/scene.hxx:22-65) 528 B
SCENE = np.dtype([
    ("vertices", ARRAY_VIEW), ("triangles", ARRAY_VIEW), ("triangle_to_emitter", ARRAY_VIEW), ("materials", ARRAY_VIEW),
    ("emitter_profiles", ARRAY_VIEW), ("emitter_instances", ARRAY_VIEW), ("images", ARRAY_VIEW), ("mediums", ARRAY_VIEW),
    ("spectrums", ARRAY_VIEW), ("emitters_distribution", DISTRIBUTION),
    ("environment_emitters", u4, 63), ("environment_emitter_count", u4),
    ("bounding_sphere_center", f4, 3), ("bounding_sphere_radius", f4),
    ("pixel_sampler_image", u4), ("pixel_sampler_radius", f4),
    ("min_path_length", u4), ("max_path_length", u4), ("samples", u4), ("random_path_termination", u4),
    ("noise_threshold", f4), ("radiance_clamp", f4),
    ("black_spectrum", u4), ("white_spectrum", u4), ("rayleigh_spectrum", u4), ("mie_spectrum", u4), ("ozone_spectrum", u4),
    ("subsurface_scatter_material", u4), ("subsurface_exit_material", u4),
    ("default_dielectric_eta", u4), ("default_conductor_eta", u4), ("default_conductor_k", u4),
    ("flags", u4), ("pad", u4),
])

# include/etx_b200.h
VCM_OPTIONS = np.dtype([("options", u4), ("radius_decay", u4), ("kernel", u4), ("initial_radius", f4), ("blue_noise", u4)])
STATUS = np.dtype([
    ("last_iteration_time", np.float64), ("total_time", np.float64), ("completed_iterations", u4), ("current_iteration", u4),
    ("iteration_in_flight", u4), ("light_vertices", u4), ("overflow", u4), ("pad", u4),
])
COUNTERS = np.dtype([(n, u8) for n in (
    "rays_closest", "rays_shadow", "nodes_visited", "tris_tested", "bounces_light", "bounces_camera", "light_vertices",
    "connections", "merge_queries", "merge_candidates", "merge_accepts", "splats", "kernel_launches", "nodes_closest", "tris_closest")])
DEVICE_CONFIG = np.dtype([("device_index", np.int32), ("max_light_vertices", u4), ("flags", u4), ("pad", u4)])
# etxb_update_info (etxb_update_scene / etxb_group_update_scene), 56 B with the C padding before the doubles
UPDATE_INFO = np.dtype({"names": ["kept", "images_kept", "images_uploaded", "grids_kept", "grids_uploaded", "fingerprint_seconds", "bvh_seconds", "total_seconds",
                                  "bytes_hashed"],
                        "formats": [u4, u4, u4, u4, u4, np.float64, np.float64, np.float64, u8], "offsets": [0, 4, 8, 12, 16, 24, 32, 40, 48], "itemsize": 56})
KEPT_GEOMETRY, KEPT_WIDE_TREE, KEPT_PATH_STATE = 1, 2, 4
# etxb_closure_query (96 B) and the per-query statistics etxb_debug_closure_eval / oracle_bsdf_eval return (include/etx_b200.h)
CLOSURE_QUERY = np.dtype([
    ("nrm", f4, 3), ("tan", f4, 3), ("btn", f4, 3), ("w_i", f4, 3), ("w_o", f4, 3), ("uv", f4, 2), ("wavelength", f4),
    ("material", u4), ("path_source", u4), ("seed", u4), ("reserved", u4, 3),
])
CLOSURE_STATS = 32
# etxb_sample_query (96 B) and the per-sample record etxb_debug_bsdf_sample / oracle_bsdf_sample return (include/etx_b200.h)
SAMPLE_QUERY = np.dtype([
    ("nrm", f4, 3), ("tan", f4, 3), ("btn", f4, 3), ("w_i", f4, 3), ("uv", f4, 2), ("wavelength", f4),
    ("material", u4), ("path_source", u4), ("seed", u4), ("medium", u4), ("mode", u4), ("fixed", f4, 3), ("reserved", u4),
])
SAMPLE_RESULT = np.dtype([("w_o", f4, 3), ("pdf", f4), ("weight", f4, 3), ("eta", f4), ("properties", u4), ("medium_index", u4),
                          ("seed_start", u4), ("seed_end", u4)])
SAMPLE_BOUNCE, SAMPLE_GIVEN = 0, 1
# etxb_emitter_query (80 B) and the per-sample record etxb_debug_emitter / oracle_emitter return (include/etx_b200.h)
EMITTER_QUERY = np.dtype([("op", u4), ("emitter", u4), ("seed", u4), ("directly_visible", u4), ("rnd", f4, 2), ("wavelength", f4),
                          ("source", f4, 3), ("target", f4, 3), ("direction", f4, 3), ("uv", f4, 2), ("reserved", u4, 2)])
EMITTER_RESULT = np.dtype([("value", f4, 3), ("origin", f4, 3), ("normal", f4, 3), ("direction", f4, 3), ("barycentric", f4, 3),
                           ("pdf_sample", f4), ("pdf_area", f4), ("pdf_dir", f4), ("pdf_dir_out", f4), ("emitter_index", u4), ("triangle_index", u4),
                           ("medium_index", u4), ("flags", u4), ("seed_start", u4), ("seed_end", u4), ("reserved", u4)])
EMITTER_SELECT, EMITTER_SAMPLE_IN, EMITTER_EMISSION, EMITTER_RADIANCE = 0, 1, 2, 3
EMITTER_FLAG_DELTA, EMITTER_FLAG_DISTANT = 1, 2
# etxb_medium_query (96 B) and the per-sample record etxb_debug_medium / oracle_medium return (include/etx_b200.h)
MEDIUM_QUERY = np.dtype([("op", u4), ("medium", u4), ("seed", u4), ("reserved0", u4), ("wavelength", f4), ("origin", f4, 3), ("direction", f4, 3),
                         ("max_t", f4), ("end", f4, 3), ("throughput", f4, 3), ("g", f4), ("rnd", f4, 2), ("w_o", f4, 3)])
MEDIUM_RESULT = np.dtype([("value", f4, 3), ("pos", f4, 3), ("dir", f4, 3), ("t_min", f4), ("t_max", f4), ("t", f4), ("flag", u4),
                          ("seed_start", u4), ("seed_end", u4), ("reserved", u4)])
MEDIUM_BOUNDS, MEDIUM_DENSITY, MEDIUM_TRANSMITTANCE, MEDIUM_SAMPLE, MEDIUM_PHASE, MEDIUM_SEGMENT = 0, 1, 2, 3, 4, 5
# etxb_subsurface_query (128 B) and the per-sample record etxb_debug_subsurface / oracle_subsurface return (include/etx_b200.h)
SUBSURFACE_QUERY = np.dtype([("op", u4), ("seed", u4), ("material", u4), ("triangle", u4), ("max_count", u4), ("direction", u4), ("wavelength", f4),
                             ("u", f4), ("v", f4), ("origin", f4, 3), ("dir", f4, 3), ("t_min", f4), ("t_max", f4), ("color", f4, 3),
                             ("distances", f4, 3), ("rnd", f4), ("radius", f4), ("normal", f4, 3), ("reserved", u4, 4)])
SUBSURFACE_PROBE = np.dtype([("o", f4, 3), ("d", f4, 3), ("min_t", f4), ("max_t", f4), ("u", f4, 3), ("v", f4, 3), ("w", f4, 3), ("basis_prob", f4, 3),
                             ("sampled_radius", f4), ("reserved", u4, 3)])
SUBSURFACE_HIT = np.dtype([("u", f4), ("v", f4), ("t", f4), ("tri", u4), ("w_i", f4, 3), ("weight", f4, 3), ("pos", f4, 3), ("nrm", f4, 3)])
SUBSURFACE_RESULT = np.dtype([("flag", u4), ("count", u4), ("selected", u4), ("rays", u4), ("seed_start", u4), ("seed_end", u4),
                              ("selected_sample_weight", f4), ("total_weight", f4), ("albedo", f4, 3), ("extinction", f4, 3), ("scattering", f4, 3),
                              ("s_r", f4), ("eval", f4, 3), ("geometric_weight", f4), ("reserved", u4, 2), ("probes", SUBSURFACE_PROBE, 3),
                              ("hits", SUBSURFACE_HIT, 24)])
SUBSURFACE_TRACE_MATERIAL, SUBSURFACE_CONTINUOUS_TRACE, SUBSURFACE_REMAP, SUBSURFACE_PROFILE, SUBSURFACE_GATHER = 0, 1, 2, 3, 4
BSDF_DIFFUSE, BSDF_REFLECTION, BSDF_TRANSMISSION, BSDF_MEDIUM_CHANGED, BSDF_DELTA = 1, 2, 4, 8, 16
# etxb_debug_thresholds / etxb_debug_branch_counts (include/etx_b200.h): a threshold of 0 always takes the large-queue branch, NEVER never does
DEBUG_THRESHOLDS = np.dtype([("merge_sort_min_queries", u4), ("merge_min_warps_per_sm", u4), ("tail_queue", u4), ("sort_queue_min", u4), ("merge_qpw", u4)])
DEFAULT_THRESHOLDS = {"merge_sort_min_queries": 16384, "merge_min_warps_per_sm": 32, "tail_queue": 8192, "sort_queue_min": 1024, "merge_qpw": 0}
NEVER = INVALID
MERGE_QPW = (1, 2, 4, 8, 16, 32)
DEBUG_BRANCH_COUNTS = np.dtype([("merge_sorts", u8), ("merge_launches", u8, 6), ("connect_launches", u8), ("pair_sorts", u8), ("queue_sorts", u8)])
# the device's light-vertex record (dvcm.cuh LightVertexRec, BUF_PHOTON_RECORDS), etxb_merge_query / etxb_merge_result / etxb_merge_grid (etxb_debug_merge)
LIGHT_VERTEX_REC = np.dtype([("throughput", f4, 3), ("d_vcm", f4), ("w_i", f4, 3), ("d_vc", f4), ("bc", f4, 3), ("d_vm", f4), ("pos", f4, 3), ("tri", u4),
                             ("nrm", f4, 3), ("material", u4), ("medium", u4), ("path_length", u4), ("path_index", u4), ("ordinal", u4)])
MERGE_QUERY = np.dtype([("tri", u4), ("u", f4), ("v", f4), ("w_i", f4, 3), ("throughput", f4, 3), ("wavelength", f4), ("d_vcm", f4), ("d_vm", f4),
                        ("total_path_depth", u4), ("seed", u4), ("medium", u4), ("reserved", u4)])
MERGE_RESULT = np.dtype([("merged", f4, 3), ("seed", u4), ("pos", f4, 3), ("nrm", f4, 3), ("reserved", u4, 2)])
MERGE_GRID = np.dtype([("bbox_min", f4, 3), ("bbox_max", f4, 3), ("cell_size", f4), ("radius_squared", f4), ("hash_table_mask", u4), ("photon_count", u4),
                       ("merge_queries", u8), ("merge_candidates", u8), ("merge_accepts", u8)])
CLOSURE_OUTPUTS = ("func_r", "func_g", "func_b", "bsdf_r", "bsdf_g", "bsdf_b", "pdf", "rev_pdf")
PATH_CAMERA, PATH_LIGHT = 1, 2

EXPECTED_SIZES = {
    "VERTEX": (VERTEX, 56), "TRIANGLE": (TRIANGLE, 32), "MATERIAL": (MATERIAL, 200), "EMITTER_PROFILE": (EMITTER_PROFILE, 48),
    "EMITTER": (EMITTER, 32), "SPECTRUM": (SPECTRUM, 3552), "DISTRIBUTION": (DISTRIBUTION, 32), "IMAGE": (IMAGE, 112),
    "MEDIUM": (MEDIUM, 80), "CAMERA": (CAMERA, 176), "SCENE": (SCENE, 528), "CLOSURE_QUERY": (CLOSURE_QUERY, 96),
    "SAMPLE_QUERY": (SAMPLE_QUERY, 96), "SAMPLE_RESULT": (SAMPLE_RESULT, 48),
    "EMITTER_QUERY": (EMITTER_QUERY, 80), "EMITTER_RESULT": (EMITTER_RESULT, 104),
    "MEDIUM_QUERY": (MEDIUM_QUERY, 96), "MEDIUM_RESULT": (MEDIUM_RESULT, 64),
    "SUBSURFACE_QUERY": (SUBSURFACE_QUERY, 128), "SUBSURFACE_PROBE": (SUBSURFACE_PROBE, 96), "SUBSURFACE_HIT": (SUBSURFACE_HIT, 64),
    "SUBSURFACE_RESULT": (SUBSURFACE_RESULT, 1920),
    "LIGHT_VERTEX_REC": (LIGHT_VERTEX_REC, 96), "MERGE_QUERY": (MERGE_QUERY, 64), "MERGE_RESULT": (MERGE_RESULT, 48), "MERGE_GRID": (MERGE_GRID, 64),
}
for _name, (_dt, _size) in EXPECTED_SIZES.items():
    assert _dt.itemsize == _size, f"{_name}: {_dt.itemsize} != {_size}"

# Material::Class (material.hxx:53-68)
MAT_DIFFUSE, MAT_TRANSLUCENT, MAT_PLASTIC, MAT_CONDUCTOR, MAT_DIELECTRIC, MAT_THINFILM, MAT_MIRROR, MAT_BOUNDARY, MAT_VELVET, MAT_PRINCIPLED, MAT_VOID = range(11)
# EmitterProfile::Class (emitter.hxx:8-13)
EMITTER_AREA, EMITTER_ENVIRONMENT, EMITTER_DIRECTIONAL = range(3)
# SpectralDistribution::Class (spectrum.hxx:452-458)
SPD_INVALID, SPD_REFLECTANCE, SPD_CONDUCTOR, SPD_DIELECTRIC, SPD_ILLUMINANT = range(5)
SCENE_COMMITTED, SCENE_SPECTRAL = 1, 2

# VCMOptions bits (rt/shared/vcm_shared.hxx:24-37)
VCM_CONNECT_TO_CAMERA, VCM_DIRECT_HIT, VCM_CONNECT_TO_LIGHT, VCM_CONNECT_VERTICES = 1, 2, 4, 8
VCM_MERGE_VERTICES, VCM_ENABLE_MIS, VCM_ENABLE_MERGING = 16, 32, 64
VCM_CONNECT_ONLY = VCM_DIRECT_HIT | VCM_CONNECT_TO_LIGHT | VCM_CONNECT_TO_CAMERA | VCM_CONNECT_VERTICES | VCM_ENABLE_MIS
VCM_FULL = VCM_CONNECT_ONLY | VCM_ENABLE_MERGING | VCM_MERGE_VERTICES

# film layers / buffer ids (include/etx_b200.h)
FILM_RESULT, FILM_CAMERA, FILM_LIGHT, FILM_LIGHT_ITERATION, FILM_NORMALS, FILM_ALBEDO, FILM_CAMERA_ADAPTIVE, FILM_DENOISED = range(8)
(BUF_LIGHT_PATH_COUNT, BUF_LIGHT_PATH_OFFSET, BUF_LIGHT_PATH_WAVELENGTH, BUF_LIGHT_SAMPLER, BUF_CAMERA_SAMPLER, BUF_LV_POS,
 BUF_LV_THROUGHPUT, BUF_LV_MIS, BUF_FILM_LIGHT_ITERATION, BUF_FILM_CAMERA, BUF_FILM_LIGHT, BUF_PHOTON_RECORDS,
 BUF_CAMERA_GATHERED, BUF_PIXEL_INFO, BUF_PIXEL_ERROR, BUF_BVH_NODES, BUF_BVH_TRIS, BUF_WIDE_NODES) = range(18)
# the trees' 64-byte nodes (csrc/bvh.h BvhNode, WideNode)
BVH_NODE = np.dtype([("lo0", "<f4", 3), ("hi0", "<f4", 3), ("lo1", "<f4", 3), ("hi1", "<f4", 3), ("child0", "<i4"), ("child1", "<i4"), ("pad", "<u4", 2)])
WIDE_NODE = np.dtype([("origin", "<f4", 3), ("exp", "u1", 3), ("count", "u1"), ("qlo", "u1", (4, 3)), ("qhi", "u1", (4, 3)), ("child", "<i4", 4),
                      ("pad", "<u4", 2)])
INTEGRATOR_VCM, INTEGRATOR_PT = 0, 1
PIXEL_COUNT_MASK, PIXEL_CONVERGED, PIXEL_TMP = (1 << 30) - 1, 1 << 30, 1 << 31
PT_OPTIONS = np.dtype([("nee", np.uint32), ("direct", np.uint32), ("mis", np.uint32), ("blue_noise", np.uint32)])
PT_STATUS = np.dtype([("pixels_processed", np.uint32), ("active_pixels", np.uint32), ("noise_level", np.float32), ("max_sample_count", np.uint32)])


def default_pt_options():
    """PTOptions (path_tracing_shared.hxx:8-14): everything on."""
    o = np.zeros(1, dtype=PT_OPTIONS)
    o["nee"] = o["direct"] = o["mis"] = o["blue_noise"] = 1
    return o


def default_vcm_options():
    """VCMOptions::default_values (rt/integrators/vcm_shared.cxx:6-13)."""
    o = np.zeros(1, dtype=VCM_OPTIONS)
    o["options"] = VCM_FULL
    o["radius_decay"] = 256
    o["kernel"] = 1
    o["initial_radius"] = 0.0
    o["blue_noise"] = 1
    return o
