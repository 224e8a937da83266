/* etx_b200.h — C ABI of the H100-native wavefront VCM module (libetx_b200.so).
 *
 * This is the drop-in boundary for ONE path of serhii-rieznik/etx-tracer: everything the reference's
 * CPU VCM integrator does between `CPUVCM::run()` and the film (sources/etx/rt/integrators/vcm_cpu.cxx:81-241,
 * vcm_shared.cxx:49-152, sources/etx/rt/shared/vcm_shared.hxx, sources/etx/rt/rt.cxx:327-579).
 * A host adapter `GPUVCM : Integrator` (etx_tracer_b200/host/gpu_vcm.hpp) forwards the reference's
 * Integrator vtable (sources/etx/rt/integrators/integrator.hxx:12-98) to these calls; INTEGRATION.md shows
 * the binding a maintainer of the reference would add.
 *
 * Conventions: plain C, no C++/torch types; all functions return 0 on success or a negative etxb_error;
 * the caller owns every host buffer it passes, the module owns all device memory; one context drives one
 * CUDA device (one process per GPU; for multi-GPU runs the module issues the NCCL collectives itself, the
 * host only distributes the communicator ids: see etxb_comm_init and etxb_group_comm_init below).
 *
 * The scene is passed in the reference's OWN in-memory layout (struct etx::Scene, 528 B, and
 * struct etx::Camera, 176 B — sources/etx/render/shared/scene.hxx:22-65, camera.hxx:8-39), so the
 * reference-side call is `etxb_upload_scene(ctx, &rt.scene(), sizeof(Scene), &rt.camera(), sizeof(Camera))`.
 * The etxb_* structs below are byte-compatible C mirrors of those PODs for callers that are not the
 * reference (tests, bench); oracle/layout_check.cxx static_asserts every offset against the real headers.
 */
#ifndef ETX_B200_H
#define ETX_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ETXB_INVALID_INDEX 0xffffffffu

typedef enum etxb_error {
  ETXB_OK = 0,
  ETXB_ERR_INVALID_ARGUMENT = -1,
  ETXB_ERR_NO_DEVICE = -2,
  ETXB_ERR_CUDA = -3,
  ETXB_ERR_UNSUPPORTED = -4,
  ETXB_ERR_NOT_READY = -5,
  ETXB_ERR_OUT_OF_MEMORY = -6,
  ETXB_ERR_OVERFLOW = -7
} etxb_error;

/* ---- byte-compatible mirrors of the reference PODs ------------------------------------------------ */

/* etx::ArrayView<T> (base.hxx:52-56) */
typedef struct etxb_array_view {
  const void* a;
  uint64_t count;
} etxb_array_view;

/* etx::Vertex (math.hxx:599), 56 B */
typedef struct etxb_vertex {
  float pos[3], nrm[3], tan[3], btn[3], tex[2];
} etxb_vertex;

/* etx::Triangle (math.hxx:607), 32 B */
typedef struct etxb_triangle {
  uint32_t i[3];
  uint32_t material_index;
  float geo_n[3];
  float pad;
} etxb_triangle;

/* etx::SpectralImage / SampledImage / RefractiveIndex / Thinfilm / SubsurfaceMaterial (material.hxx:8-50) */
typedef struct etxb_spectral_image {
  uint32_t spectrum_index, image_index;
} etxb_spectral_image;
typedef struct etxb_sampled_image {
  float value[4];
  uint32_t image_index, channel;
} etxb_sampled_image;
typedef struct etxb_refractive_index {
  uint32_t cls, eta_index, k_index;
} etxb_refractive_index;
typedef struct etxb_thinfilm {
  etxb_refractive_index ior;
  uint32_t thickness_image;
  float min_thickness, max_thickness, pad;
} etxb_thinfilm;
typedef struct etxb_subsurface {
  uint32_t spectrum_index, image_index, cls, path;
} etxb_subsurface;

/* etx::Material::Class (material.hxx:53-68) */
enum {
  ETXB_MAT_DIFFUSE = 0,
  ETXB_MAT_TRANSLUCENT = 1,
  ETXB_MAT_PLASTIC = 2,
  ETXB_MAT_CONDUCTOR = 3,
  ETXB_MAT_DIELECTRIC = 4,
  ETXB_MAT_THINFILM = 5,
  ETXB_MAT_MIRROR = 6,
  ETXB_MAT_BOUNDARY = 7,
  ETXB_MAT_VELVET = 8,
  ETXB_MAT_PRINCIPLED = 9,
  ETXB_MAT_VOID = 10
};

/* etx::Material (material.hxx:52-97), 200 B */
typedef struct etxb_material {
  etxb_spectral_image reflectance, scattering, emission;
  etxb_sampled_image roughness, metalness, transmission;
  etxb_subsurface subsurface;
  etxb_thinfilm thinfilm;
  etxb_refractive_index ext_ior, int_ior;
  uint32_t cls, int_medium, ext_medium, normal_image_index, diffuse_variation, two_sided;
  float normal_scale, opacity, emission_collimation;
} etxb_material;

/* etx::EmitterProfile (emitter.hxx:7-42), 48 B; Class: 0 Area, 1 Environment, 2 Directional */
typedef struct etxb_emitter_profile {
  etxb_spectral_image emission;
  float direction[3];
  uint32_t cls;
  float angular_size, equivalent_disk_size, angular_size_cosine, pad0, pad1, pad2;
} etxb_emitter_profile;

/* etx::Emitter (emitter.hxx:44-71), 32 B */
typedef struct etxb_emitter {
  uint32_t cls, profile, triangle_index;
  float spectrum_weight, additional_weight, triangle_area, pad0, pad1;
} etxb_emitter;

/* etx::SpectralDistribution (spectrum.hxx:449-), 3552 B */
typedef struct etxb_spectrum {
  struct {
    float wavelength, power;
  } entries[441];
  uint32_t entry_count;
  float integrated[3];
  uint32_t pad[2];
} etxb_spectrum;

/* etx::Distribution::Entry / Distribution (distribution.hxx:7-15) */
typedef struct etxb_distribution_entry {
  float value, pdf, cdf;
} etxb_distribution_entry;
typedef struct etxb_distribution {
  etxb_array_view values; /* etxb_distribution_entry[count] */
  float total_weight;
  uint32_t pad[3];
} etxb_distribution;

/* etx::Image (image.hxx:8-50), 112 B; format 1 = RGBA32F, 2 = RGBA8 */
typedef struct etxb_image {
  etxb_array_view pixels;
  etxb_array_view x_distributions; /* etxb_distribution[isize.y] */
  etxb_distribution y_distribution;
  float fsize[2], offset[2], scale[2];
  uint32_t isize[2];
  float normalization;
  uint32_t options, format, data_size;
} etxb_image;

/* etx::Medium (medium.hxx:8-47), 80 B */
typedef struct etxb_medium {
  etxb_array_view density; /* float[dx*dy*dz], normalised to max 1 */
  float bounds_min[3], bounds_pad0, bounds_max[3], bounds_pad1;
  uint16_t cls, enable_explicit_connections;
  uint32_t absorption_index, scattering_index;
  float phase_function_g, max_sigma;
  uint32_t dimensions[3];
} etxb_medium;

/* etx::Camera (camera.hxx:8-39), 176 B; cls 0 = Perspective, 1 = Equirectangular */
typedef struct etxb_camera {
  float view_proj[16]; /* column-major float4 col[4] */
  float position[3];
  uint32_t cls;
  float target[3], tan_half_fov;
  float side[3], aspect;
  float up[3], area;
  float direction[3], image_plane;
  uint32_t film_size[2];
  float lens_radius, focal_distance;
  float clip_near, clip_far;
  uint32_t lens_image, medium_index;
} etxb_camera;

/* etx::Scene (scene.hxx:22-65), 528 B */
#define ETXB_SCENE_COMMITTED 1u
#define ETXB_SCENE_SPECTRAL 2u
typedef struct etxb_scene {
  etxb_array_view vertices, triangles, triangle_to_emitter, materials, emitter_profiles, emitter_instances, images, mediums, spectrums;
  etxb_distribution emitters_distribution;
  uint32_t environment_emitters[63];
  uint32_t environment_emitter_count;
  float bounding_sphere_center[3], bounding_sphere_radius;
  uint32_t pixel_sampler_image;
  float pixel_sampler_radius;
  uint32_t min_path_length, max_path_length, samples, random_path_termination;
  float noise_threshold, radiance_clamp;
  uint32_t black_spectrum, white_spectrum, rayleigh_spectrum, mie_spectrum, ozone_spectrum;
  uint32_t subsurface_scatter_material, subsurface_exit_material;
  uint32_t default_dielectric_eta, default_conductor_eta, default_conductor_k;
  uint32_t flags;
  uint32_t pad;
} etxb_scene;

/* ---- options / status -------------------------------------------------------------------------- */

/* VCMOptions bit flags (vcm_shared.hxx:24-37) */
#define ETXB_VCM_CONNECT_TO_CAMERA (1u << 0)
#define ETXB_VCM_DIRECT_HIT (1u << 1)
#define ETXB_VCM_CONNECT_TO_LIGHT (1u << 2)
#define ETXB_VCM_CONNECT_VERTICES (1u << 3)
#define ETXB_VCM_MERGE_VERTICES (1u << 4)
#define ETXB_VCM_ENABLE_MIS (1u << 5)
#define ETXB_VCM_ENABLE_MERGING (1u << 6)
#define ETXB_VCM_CONNECT_ONLY (ETXB_VCM_DIRECT_HIT | ETXB_VCM_CONNECT_TO_LIGHT | ETXB_VCM_CONNECT_TO_CAMERA | ETXB_VCM_CONNECT_VERTICES | ETXB_VCM_ENABLE_MIS)
#define ETXB_VCM_FULL (ETXB_VCM_CONNECT_ONLY | ETXB_VCM_ENABLE_MERGING | ETXB_VCM_MERGE_VERTICES)

/* Mirrors VCMOptions (vcm_shared.hxx:12-72); defaults = VCMOptions::default_values (vcm_shared.cxx:6-13).
 * The option keys the reference UI uses ("vcm-initial_radius", "vcm-radius_decay", "vcm-blue_noise", "vcm-kernel",
 * "vcm-direct_hit", ... vcm_shared.cxx:15-28) map 1:1 onto these fields; see etxb_options_set_key. */
typedef struct etxb_vcm_options {
  uint32_t options;      /* ETXB_VCM_* bits, default ETXB_VCM_FULL */
  uint32_t radius_decay; /* default 256 */
  uint32_t kernel;       /* 0 Tophat, 1 Epanechnikov (default) */
  float initial_radius;  /* 0 => 5 * R_scene / max(W,H) (vcm_cpu.cxx:102-106) */
  uint32_t blue_noise;   /* default 1 */
} etxb_vcm_options;

/* Mirrors Integrator::Status (integrator.hxx:24-37) + device counters. */
typedef struct etxb_status {
  double last_iteration_time; /* seconds, device time of the last finished iteration */
  double total_time;          /* seconds, sum over finished iterations */
  uint32_t completed_iterations;
  uint32_t current_iteration;
  uint32_t iteration_in_flight; /* 1 while an enqueued iteration has not finished */
  uint32_t light_vertices;      /* vertices stored by the last light pass */
  uint32_t overflow;            /* non-zero if a fixed-capacity pool overflowed (results invalid) */
  uint32_t pad;
} etxb_status;

/* Per-iteration event counters (feed the algorithmic-bytes formula, SURVEY.md §8(d)). */
typedef struct etxb_counters {
  uint64_t rays_closest;    /* closest-hit queries */
  uint64_t rays_shadow;     /* transmittance (any-hit) queries */
  uint64_t nodes_visited;   /* only counted when built with ETXB_COUNT_TRAVERSAL */
  uint64_t tris_tested;     /* idem */
  uint64_t bounces_light;   /* light-subpath surface events */
  uint64_t bounces_camera;  /* camera-subpath surface events */
  uint64_t light_vertices;  /* stored light vertices */
  uint64_t connections;     /* camera-vertex x light-vertex connection attempts */
  uint64_t merge_queries;   /* hash-grid gathers */
  uint64_t merge_candidates;
  uint64_t merge_accepts;
  uint64_t splats;
  uint64_t kernel_launches; /* kernels of this module launched */
  uint64_t nodes_closest;   /* the part of nodes_visited / tris_tested spent by the closest-hit kernel (k_trace_closest) */
  uint64_t tris_closest;
} etxb_counters;

typedef struct etxb_device_config {
  int32_t device_index;        /* CUDA device ordinal */
  uint32_t max_light_vertices; /* pool capacity; 0 => 16 per pixel */
  uint32_t flags;              /* reserved */
  uint32_t pad;
} etxb_device_config;

/* Film layers readable with etxb_read_film: values follow Film::layer (film.cxx:381-418). */
enum {
  ETXB_FILM_RESULT = 0,      /* max(0, camera + light) as float4 */
  ETXB_FILM_CAMERA = 1,      /* camera image (running mean over iterations) */
  ETXB_FILM_LIGHT = 2,       /* light image (running mean over iterations) */
  ETXB_FILM_LIGHT_ITERATION = 3,
  /* layers the path tracer fills (Film::Normals shown as n * 0.5 + 0.5, Film::Albedo, Film::CameraAdaptive; film.cxx:406-414) */
  ETXB_FILM_NORMALS = 4,
  ETXB_FILM_ALBEDO = 5,
  /* the mean of the even-indexed samples, kept by both integrators: the second half buffer of etxb_denoise's variance estimate */
  ETXB_FILM_CAMERA_ADAPTIVE = 6,
  /* Film::Denoised: the last etxb_denoise; zeros before it, kept until the next etxb_denoise or a film resize */
  ETXB_FILM_DENOISED = 7
};

/* Named device buffers for etxb_read_buffer (parity tests). */
enum {
  ETXB_BUF_LIGHT_PATH_COUNT = 0,   /* uint32[N]  vertices stored per light path (VCMLightPath::count) */
  ETXB_BUF_LIGHT_PATH_OFFSET = 1,  /* uint32[N]  first vertex of the path in the pool (VCMLightPath::index) */
  ETXB_BUF_LIGHT_PATH_WAVELENGTH = 2, /* float[N] */
  ETXB_BUF_LIGHT_SAMPLER = 3,      /* uint32[N]  sampler seed at the end of the light subpath */
  ETXB_BUF_CAMERA_SAMPLER = 4,     /* uint32[N]  sampler seed at the end of the camera subpath */
  ETXB_BUF_LV_POS = 5,             /* float[3*P] light vertex positions, path-major order */
  ETXB_BUF_LV_THROUGHPUT = 6,      /* float[3*P] */
  ETXB_BUF_LV_MIS = 7,             /* float[3*P] d_vcm, d_vc, d_vm */
  ETXB_BUF_FILM_LIGHT_ITERATION = 8, /* float4[N] per-iteration light splats (summed over the ranks of a pixel-tile run) */
  ETXB_BUF_FILM_CAMERA = 9,        /* float4[N] */
  ETXB_BUF_FILM_LIGHT = 10,        /* float4[N] */
  ETXB_BUF_PHOTON_RECORDS = 11,    /* packed photon records of this context's last light pass, path-major, 96 B each */
  ETXB_BUF_CAMERA_GATHERED = 12,   /* float[3*N] last iteration's camera contribution per path */
  ETXB_BUF_PIXEL_INFO = 13,        /* uint32[N]  Film's InternalData in film storage order (film.cxx:27-32): sample_count bits 0-29, converged bit 30, tmp bit 31 */
  ETXB_BUF_PIXEL_ERROR = 14,       /* float[N]   InternalData::error_level */
  ETXB_BUF_BVH_NODES = 15,         /* the committed BVH2: 64-byte nodes (csrc/bvh.h BvhNode), root first */
  ETXB_BUF_BVH_TRIS = 16,          /* float4[3*S] leaf-ordered triangle corners; .w of the first corner holds the triangle index */
  ETXB_BUF_WIDE_NODES = 17,        /* the committed 4-wide tree: 64-byte nodes (csrc/bvh.h WideNode); empty where the scene walks the BVH2 */
  ETXB_BUF_COUNT
};

typedef struct etxb_ctx etxb_ctx;

/* ---- entry points -------------------------------------------------------------------------------- */

/* Library identity: "fast" (product build) or "parity" (strict-IEEE build used by the bit-exact tests). */
const char* etxb_build_flavor(void);
/* Number of CUDA devices visible, or a negative etxb_error. */
int etxb_device_count(void);

/* Replaces Raytracing/Integrator construction (rt.cxx:27-36, vcm_cpu.cxx:62-66). */
int etxb_create(etxb_ctx** out_ctx, const etxb_device_config* cfg);
void etxb_destroy(etxb_ctx* ctx);
const char* etxb_last_error(const etxb_ctx* ctx);

/* Replaces Raytracing::commit_changes (rt.cxx:58-64,323): copies the scene to HBM, builds the BVH,
 * allocates film + queues for camera->film_size.  `scene`/`camera` use the reference layouts. */
int etxb_upload_scene(etxb_ctx* ctx, const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes);

/* The restart after an edit of the committed Scene / Camera (the application restarts its integrator after every camera move and every
 * material, medium, emitter or scene-settings edit, app.cxx:131-141, 368-403).  The context then renders exactly what a fresh context
 * renders after etxb_upload_scene with the same PODs: the film is cleared and etxb_begin(ctx, 0) applied; options and the selected
 * integrator stay.  What is reused is decided by content, never by pointer (the application edits the PODs in place and
 * rebuild_area_emitters reallocates its arrays): upload and update record a 128-bit hash of the vertex + triangle arrays, of each image
 * (pixels, sampling tables, scalar fields) and of each density grid (values, dimensions).
 *  - same geometry hash: the device vertices, triangles and BVH2 stay (no BVH build), and the 4-wide tree of a product-build scene with
 *    stochastic BSDFs stays; an edit that newly needs that tree collapses it from the device's BVH2;
 *  - images and density grids: each kept or copied on its own hash;
 *  - per-path / per-vertex / shadow / connection-record / sort / film buffers: kept where the upload would allocate the same size;
 *  - everything else (materials, spectra, emitters, their distribution, media records, scene scalars, camera, scene-class flags) is
 *    derived again as the upload derives it.
 * Every check of the upload runs before any device buffer changes: a refused update returns the error and the previous scene stays
 * committed and renderable.  A CUDA failure part-way leaves the scene not ready, like a failed upload.  Iterations in flight are drained
 * first.  Without a committed scene it is an upload.  ETXB_ERR_UNSUPPORTED on a context with a communicator (etxb_comm_init).
 * `info` (may be NULL) reports what was kept, the bytes hashed, the host time spent hashing, the time spent building trees (BVH2 and
 * 4-wide, both on the device: wall time including the new geometry's upload) and in the whole call. */
typedef struct etxb_update_info {
  uint32_t kept; /* ETXB_KEPT_* bits */
  uint32_t images_kept, images_uploaded;
  uint32_t grids_kept, grids_uploaded;
  double fingerprint_seconds, bvh_seconds, total_seconds;
  uint64_t bytes_hashed; /* what the content hashes read: geometry, images with their sampling tables, density grids */
} etxb_update_info;
#define ETXB_KEPT_GEOMETRY (1u << 0)   /* device vertices + triangles + BVH2 */
#define ETXB_KEPT_WIDE_TREE (1u << 1)  /* the 4-wide tree (product build, scenes with stochastic BSDFs; set only where one exists) */
#define ETXB_KEPT_PATH_STATE (1u << 2) /* per-path / per-vertex / film buffers not re-allocated */
int etxb_update_scene(etxb_ctx* ctx, const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes, etxb_update_info* info);

/* Blue-noise tables (thirdparty/bluenoise): sobol[256*256], and for the variant selected by
 * next_power(min(scene.samples,256)) (bluenoise.cxx:73-95) scrambling[128*128*8], ranking[128*128*8], as uint8. */
int etxb_upload_blue_noise(etxb_ctx* ctx, const uint8_t* sobol_256x256, const uint8_t* scrambling, const uint8_t* ranking);
/* CIE 2006 XYZ table, 441 x float3, 390..830 nm (spectrum.hxx:28 spectral_xyz) and the RGB response table
 * 391 x float3 (spectrum.cxx:399 rgb_response). */
int etxb_upload_color_tables(etxb_ctx* ctx, const float* xyz_441x3, const float* rgb_response_391x3);

/* VCMOptions::default_values / load (vcm_shared.cxx:6-28). */
void etxb_options_default(etxb_vcm_options* opt);
int etxb_options_set_key(etxb_vcm_options* opt, const char* key, double value);
int etxb_set_options(etxb_ctx* ctx, const etxb_vcm_options* opt);

/* The pixel-tile rule without a communicator: this context renders only the 32x32 tiles with (tile % world) == rank, on one GPU.
 * world == 1 (default) renders the full frame. */
int etxb_set_partition(etxb_ctx* ctx, uint32_t rank, uint32_t world);

/* Externally driven iteration index: the next enqueued iteration renders VCMIteration::iteration = `iteration`; the index no
 * longer advances by itself (used by etxb_group below). */
int etxb_set_next_iteration(etxb_ctx* ctx, uint32_t iteration);

/* CPUVCMImpl::start (vcm_cpu.cxx:81-93): clears film, sets iteration = first_iteration. */
int etxb_begin(etxb_ctx* ctx, uint32_t first_iteration);

/* ---- coarse preview: Film pixel size (film.cxx:147-230, 345-461) ------------------------------------------------------------------
 * Film::set_pixel_size: the size is clamped to [1, 1024] and takes effect at the next etxb_begin (or etxb_update_scene, which ends in
 * it), like Film::clear.  At pixel size s both integrators trace Film::pixel_count() = ceil(W / s) x ceil(H / s) paths per iteration,
 * path i in the s x s block (i % ceil(W / s), i / ceil(W / s)); the block's pixels each take the path's value with their own sample count.
 * The film and every layer stay W x H; the path-indexed buffers (ETXB_BUF_*_SAMPLER, _LIGHT_PATH_*, _CAMERA_GATHERED) keep W x H
 * entries, of which the first Film::pixel_count() belong to the iteration.  The application previews with 8 while the camera moves and
 * goes back to 1 when it stops (app.cxx:131-141).  Refused (ETXB_ERR_UNSUPPORTED) above 1 on a context with a communicator or a pixel
 * partition, and on a group with communicators: tiles and replica splits index film pixels.  Which pixel of its block a path
 * samples is the one departure from the reference: Film::active_pixel offsets the block origin by rand() % s in x and then in y, and rand()
 * is process-global state called from worker threads in timing-dependent order, so no run of the reference can be repeated.  Here the
 * offset is a hash of (path index, iteration) — x from a first 32-bit value, y from a second, each % s (pm::preview_offset in
 * etx_tracer_b200/csrc/portable_math.h, the one definition the device and the oracle call).  It does not draw from the path's sampler,
 * so every iteration stays a function of the scene, the options and its index. */
int etxb_set_film_pixel_size(etxb_ctx* ctx, uint32_t size);

/* ---- film export (SURVEY 8(f) N4): RTApplication::on_save_image_selected (sources/raytracer/app.cxx:261-295) -------------------------
 * The reference saves the selected Film layer either as float OpenEXR (tinyexr SaveEXR) or tone-mapped to 8-bit PNG (1 - exp(-exposure c),
 * sRGB curve, stb_image_write).  etxb_read_film_ldr tone-maps on the device (4 bytes per pixel leave the GPU); the two writers and the host
 * tone map are plain host code (usable on any float4 / RGBA8 buffer, e.g. a multi-GPU frame from etxb_group_comm_reduce_film). */
#define ETXB_SAVE_EXR 0u
#define ETXB_SAVE_PNG_TONEMAPPED 1u
int etxb_read_film_ldr(etxb_ctx* ctx, uint32_t layer, float exposure, uint8_t* dst_rgba8, uint64_t dst_bytes);
int etxb_save_film(etxb_ctx* ctx, uint32_t layer, const char* file_name, uint32_t mode, float exposure);
int etxb_write_exr(const char* file_name, const float* rgba, uint32_t width, uint32_t height);
int etxb_write_png(const char* file_name, const uint8_t* rgba8, uint32_t width, uint32_t height);
int etxb_tonemap_rgba8(const float* rgba, uint64_t pixel_count, float exposure, uint8_t* out_rgba8);

/* ---- the viewer (DESIGN §14): RenderContext's fragment shader (sources/raytracer/render.cxx:252-388) and its reference image ------------
 * etxb_read_film_view computes one of the six OutputViews of a film layer on the device: float4 as the shader returns it (unclamped), or the
 * RGBA8 an 8-bit UNORM window stores (clamp to [0, 1], floor(255 x + 0.5), NaN -> 0).  Like etxb_read_film_ldr it does not wait for
 * iterations in flight.  The reference views (Reference, Relative / Absolute Difference) and etxb_film_error need a reference:
 * ETXB_ERR_NOT_READY without one.  All the calls below are ETXB_ERR_UNSUPPORTED on a context with a communicator or a pixel partition (its
 * film holds only its own tiles). */
#define ETXB_VIEW_TONEMAPPED 0u /* OutputView::TonemappedImage */
#define ETXB_VIEW_ALPHA 1u      /* AlphaChannel */
#define ETXB_VIEW_HDR 2u        /* HDRImage */
#define ETXB_VIEW_REFERENCE 3u  /* ReferenceImage */
#define ETXB_VIEW_RELATIVE 4u   /* RelativeDifference */
#define ETXB_VIEW_ABSOLUTE 5u   /* AbsoluteDifference */
#define ETXB_VIEW_OPT_TONEMAPPING 1u /* ViewOptions (raytracer/options.hxx:40-45) */
#define ETXB_VIEW_OPT_SRGB 2u
#define ETXB_VIEW_OPT_SKIP_COLOR_CONVERSION 4u
typedef struct etxb_view {
  uint32_t view;    /* ETXB_VIEW_*; ETXB_ERR_INVALID_ARGUMENT past 5 */
  uint32_t options; /* ETXB_VIEW_OPT_* bits; ETXB_ERR_INVALID_ARGUMENT for any other bit */
  float exposure;   /* finite */
  uint32_t rgba8;   /* 0: float4 per pixel (16 bytes), 1: RGBA8 (4 bytes) */
} etxb_view;
/* The film's error against the reference (float64 sums in a reduction whose shape depends on the pixel count alone: the same bits on every
 * call).  Pixels whose RGB has a NaN or inf are counted in `nonfinite` and left out of every sum and every other count. */
typedef struct etxb_film_error_info {
  uint64_t pixels;          /* W * H */
  uint64_t nonfinite;       /* pixels with a NaN / inf in RGB */
  uint64_t negative;        /* finite pixels with a negative RGB channel */
  uint64_t lum_above;       /* finite pixels where the reference's float32 luminance exceeds the layer's by more than 1/8192 (the Absolute
                               Difference view's red) */
  uint64_t lum_below;       /* ... the layer's exceeds the reference's (its green) */
  double mse;               /* mean over finite pixels and RGB of (c - r)^2 */
  double rel_mse;           /* mean of (c - r)^2 / (r^2 + eps), eps = (0.01 mean_rgb(reference))^2; not finite when eps is 0 (an all-zero
                               reference) or not finite (a reference with a NaN / inf pixel).  Every mean is NaN when no pixel is finite. */
  double mean_abs_lum;      /* means over finite pixels of |c_lum - r_lum|, c_lum, r_lum (float64, the view's weights) */
  double mean_lum;
  double reference_mean_lum;
  uint32_t iterations;      /* completed iterations the film held */
  uint32_t pad;
} etxb_film_error_info;
/* ImagePool::add_from_data: host float4 pixels (film storage order, W x H of the film) into the reference slot.  ETXB_ERR_INVALID_ARGUMENT for
 * another size.  The slot is kept across etxb_begin / etxb_update_scene / etxb_upload_scene at the same film size and dropped at another. */
int etxb_set_reference_image(etxb_ctx* ctx, const float* rgba, uint32_t width, uint32_t height);
/* Use as Reference (app.cxx:252-259): the layer, copied on the device into the reference slot. */
int etxb_use_film_as_reference(etxb_ctx* ctx, uint32_t layer);
int etxb_clear_reference(etxb_ctx* ctx);
int etxb_read_film_view(etxb_ctx* ctx, uint32_t layer, const etxb_view* view, void* dst, uint64_t dst_bytes);
/* Waits for the iterations in flight first, so that the numbers belong to a whole number of iterations. */
int etxb_film_error(etxb_ctx* ctx, uint32_t layer, etxb_film_error_info* out);
/* Open Reference Image (app.cxx:243-250): the float4 pixels ImagePool::add_from_file(file, 0, {}, {1, 1}) holds, host code.  Rows in file
 * order; 8-bit files through sRGB -> linear, 8-bit truncation and back to [0, 1]; OpenEXR with inf -> 65504 and NaN / negatives -> 0; HDR
 * and PFM as read.  A file that cannot be read gives the 1 x 1 white placeholder and a warning in `err` (ETXB_OK).  rgba = NULL: the size. */
int etxb_reference_image_file_read(const char* file_name, uint32_t* width, uint32_t* height, float* rgba, uint64_t capacity, char* err, uint64_t err_bytes);

/* ---- scene files (SURVEY 8(f) N2): SceneRepresentation::load_from_file (render/host/scene_representation.cxx:679-838) ------------------
 * Reads the reference's `.json` + `.obj` + `.mtl` scene dialect (et::camera / et::medium / et::dir / et::env / et::spectrum blocks, the material
 * directives of parse_material :1682-2079, PNG / JPEG / TGA / BMP / EXR / HDR / PFM textures) into the Scene / Camera PODs etxb_create takes: host C++, no CUDA, no
 * third-party reader.  The object owns every array the PODs point into; keep it alive until etxb_create has returned (the module copies).
 * A file without an et::dir / et::env block gets the reference's default atmosphere (sun + sky images, generated here on the host threads).
 * `et::medium ... volume file.nvdb` becomes a heterogeneous medium with a dense grid (own NanoVDB 32.x reader, codecs none / ZIP; medium_pool.cxx:102-159).
 * Failure: ETXB_ERR_UNSUPPORTED with the reason in `err` (missing or corrupt file, BLOSC-compressed volume, glTF).
 * `data_folder` = where tables.bin lives; NULL = the `data/` folder beside the shared library. */
typedef struct etxb_scene_file etxb_scene_file;
int etxb_scene_file_load(const char* file_name, const char* data_folder, etxb_scene_file** out, char* err, uint64_t err_bytes);
const etxb_scene* etxb_scene_file_scene(const etxb_scene_file* sf);
const etxb_camera* etxb_scene_file_camera(const etxb_scene_file* sf);
uint32_t etxb_scene_file_warning_count(const etxb_scene_file* sf);
const char* etxb_scene_file_warning(const etxb_scene_file* sf, uint32_t index);
uint32_t etxb_scene_file_material_count(const etxb_scene_file* sf);
const char* etxb_scene_file_material_name(const etxb_scene_file* sf, uint32_t index);
void etxb_scene_file_free(etxb_scene_file* sf);
/* Scene::samples (the iteration count the integrators stop at, and what selects the blue-noise variant) — the application's "samples" setting */
void etxb_scene_file_set_samples(etxb_scene_file* sf, uint32_t samples);
/* One call from file to device: etxb_upload_color_tables + etxb_upload_blue_noise (the variant BNSampler picks for scene.samples,
 * thirdparty/bluenoise/bluenoise.cxx:73-95) + etxb_upload_scene, all from tables.bin and the loaded PODs. */
int etxb_scene_file_commit(etxb_ctx* ctx, const etxb_scene_file* sf);
/* A string value of the application's options file (util/options.cxx; ids "integrator" and "scene" are what RTApplication::init reads,
 * raytracer/app.cxx:88-105): copies it to `out` (NUL-terminated, truncated to out_bytes) and returns its length; 0 = id absent; < 0 = error. */
int etxb_options_file_string(const char* file_name, const char* id, char* out, uint64_t out_bytes);
/* The loader's image readers on their own — every PNG form stb_image decodes (bit depths 1-16, palette, colour keys, Adam7), baseline / progressive JPEG
 * (same bytes as stb_image's decoder), TGA, BMP, OpenEXR scan lines (none /
 * RLE / ZIPS / ZIP / PIZ; half and float), Radiance HDR, the reference's PFM variant — as ImagePool::load_data uses them (image_pool.cxx:271-383): rows in file order,
 * RGBA8 (*eight_bit = 1; the file's values, no sRGB step) or RGBA32F.  pixels = NULL queries the size. */
int etxb_image_file_read(const char* file_name, uint32_t* width, uint32_t* height, uint32_t* eight_bit, void* pixels, uint64_t capacity, char* err, uint64_t err_bytes);
/* Two parts of the loader on their own.  etxb_mesh_tangents: the tangent-space generator the reference calls for meshes with texture coordinates
 * (build_tangents, scene_representation.cxx:337-398) over etx::Vertex / etx::Triangle arrays, writing tan / btn of the vertices whose tangent is not valid
 * yet.  etxb_nvdb_density: the dense grid MediumPool::load_nvdb (medium_pool.cxx:102-159) builds from the first float grid of a NanoVDB file — call with
 * values = NULL for the dimensions (x, y, z; all 0 = the medium stays homogeneous), then with a buffer of x*y*z floats (x fastest; not yet normalised). */
int etxb_mesh_tangents(etxb_vertex* vertices, uint64_t vertex_count, const etxb_triangle* triangles, uint64_t triangle_count);
int etxb_nvdb_density(const char* file_name, uint32_t dimensions[3], float* values, uint64_t value_capacity, char* err, uint64_t err_bytes);
/* The procedural sun disk (128 x 128) and sky dome (sky_width x sky_height) images of an atmosphere block — what the loader generates for a
 * `newmtl et::atmosphere` block and for every scene file that declares no distant emitter (scene_representation.cxx:805-820, :1376-1495;
 * render/host/scattering.cxx) — for callers that assemble the emitters themselves.  parameters = altitude, anisotropy, rayleigh, mie, ozone
 * (scattering::Parameters); direction normalised; angular_size in radians; either output may be NULL. */
int etxb_atmosphere_images(const char* data_folder, const float direction[3], float angular_size, const float parameters[5], uint32_t sky_width, uint32_t sky_height,
                           float* sun_rgba_128x128, float* sky_rgba);
/* A table of tables.bin by name ("color_tables/xyz_441x3", "bluenoise/sobol", "spectra/gold.eta_power", ...); NULL when absent. */
const void* etxb_scene_file_table(const etxb_scene_file* sf, const char* name, uint64_t* bytes);

/* ---- the unidirectional path tracer on the same context (SURVEY 8(f) N3) -----------------------------------------
 * Replaces CPUPathTracing (rt/integrators/path_tracing.cxx:12-170) + run_path_iteration (rt/shared/path_tracing_shared.hxx:485-510)
 * + Film::accumulate_camera_image with the normal / albedo layers and Film::estimate_noise_levels (render/host/film.cxx:173-330).
 * etxb_set_integrator selects which algorithm etxb_begin / etxb_enqueue_iteration / etxb_poll / etxb_read_film drive: with
 * ETXB_INTEGRATOR_PT one iteration = one path per active pixel (CPUPathTracingImpl::execute_range) followed by update()'s
 * film.estimate_noise_levels(current_iteration, samples, noise_threshold); a pixel the estimate marks converged is skipped from
 * then on (Film::active_pixel).  The coarse preview (etxb_set_film_pixel_size) applies to it as to the VCM: a path whose chosen pixel has
 * converged is skipped with its whole block.
 * Pixel tiles: on a context with a communicator (etxb_comm_init, either order) each rank traces its own tiles and the noise estimate is
 * exchanged inside etxb_enqueue_iteration (see the pixel-tile section below); the ranks then render the one-GPU frame and history.
 * etxb_set_integrator(ETXB_INTEGRATOR_PT) is refused (ETXB_ERR_UNSUPPORTED, before any collective) on a context with a pixel partition but no
 * communicator and on the lanes of a group in pixel-tile mode (etxb_group_comm_init with world >= 2), whose lanes would each keep their own
 * per-pixel history. */
#define ETXB_INTEGRATOR_VCM 0u
#define ETXB_INTEGRATOR_PT 1u
/* PTOptions (path_tracing_shared.hxx:8-14); the reference's option ids are "nee", "direct", "mis", "bn" (path_tracing.cxx:36-39) */
typedef struct etxb_pt_options {
  uint32_t nee, direct, mis, blue_noise; /* all default 1 */
} etxb_pt_options;
/* On a context with a communicator the status is global: pixels_processed is summed over the ranks at the end of every iteration,
 * active_pixels and noise_level at every estimate — so every rank's update loop ends at the same iteration. */
typedef struct etxb_pt_status {
  uint32_t pixels_processed; /* CPUPathTracingImpl::pixels_processed of the last finished iteration; 0 => the reference stops the run (:90-92) */
  uint32_t active_pixels;    /* Film::active_pixel_count (film.cxx:430): pixel count after a clear, pixels converged in the last estimate after one */
  float noise_level;         /* Film::noise_level (film.cxx:461) */
  uint32_t max_sample_count; /* Scene::samples */
} etxb_pt_status;
void etxb_pt_options_default(etxb_pt_options* opt);
int etxb_pt_options_set_key(etxb_pt_options* opt, const char* key, double value);
int etxb_pt_set_options(etxb_ctx* ctx, const etxb_pt_options* opt);
int etxb_set_integrator(etxb_ctx* ctx, uint32_t integrator);
int etxb_pt_get_status(etxb_ctx* ctx, etxb_pt_status* out);
/* Scene::noise_threshold / Scene::radiance_clamp (scene.hxx:45-46) changed without a new upload */
int etxb_set_scene_settings(etxb_ctx* ctx, float noise_threshold, float radiance_clamp);

/* One VCM iteration = start_next_iteration + gather_light_vertices + complete_light_vertices +
 * gather_camera_vertices + complete_camera_vertices (vcm_cpu.cxx:95-241).  Asynchronous: returns after
 * the work is queued on the context's stream. */
int etxb_enqueue_iteration(etxb_ctx* ctx);

/* CPUVCM::update (vcm_cpu.cxx:264-276): non-blocking; fills status. */
int etxb_poll(etxb_ctx* ctx, etxb_status* status);
/* Blocks until all queued work is done. */
int etxb_wait(etxb_ctx* ctx);
/* CPUVCM::stop (vcm_cpu.cxx:278-288). */
int etxb_stop(etxb_ctx* ctx, int wait_for_iteration);

/* Film::layer (film.cxx:381-418): row-major float4, y already flipped in storage like the reference. */
int etxb_read_film(etxb_ctx* ctx, uint32_t layer, float* dst_rgba, uint64_t dst_bytes);
int etxb_film_size(const etxb_ctx* ctx, uint32_t* width, uint32_t* height);
/* Film::denoise(layer) (film.cxx:420-423): filters ETXB_FILM_RESULT or ETXB_FILM_CAMERA into ETXB_FILM_DENOISED on the device.  The filter is
 * non-local means with a two-half-buffer variance estimate and, for the path tracer, normal and albedo feature weights (DESIGN §13) — not
 * OpenImageDenoise, whose trained weights this module does not have.  Drains the context first, like etxb_read_film.  ETXB_ERR_INVALID_ARGUMENT
 * for other layers; ETXB_ERR_NOT_READY without a scene or where a pixel has fewer than two samples; ETXB_ERR_UNSUPPORTED on a context with a
 * communicator or a pixel partition (its film holds only its own tiles).  The same output for the same film on the same build. */
int etxb_denoise(etxb_ctx* ctx, uint32_t layer);

int etxb_get_counters(etxb_ctx* ctx, etxb_counters* out);
/* Per-kernel device time of the last iteration (CUDA events): names[i] -> ms[i]; returns count. */
int etxb_get_kernel_times(etxb_ctx* ctx, const char** names, float* ms, uint32_t* launches, uint32_t capacity);

/* Introspection for parity tests. */
int etxb_read_buffer(etxb_ctx* ctx, uint32_t buffer_id, void* dst, uint64_t dst_bytes, uint64_t* out_bytes);
void* etxb_stream(etxb_ctx* ctx); /* cudaStream_t the module launches on */

/* Unit entry points used by the parity tests (same kernels the iteration uses). */
/* Closest-hit query for `count` rays (rt.cxx:428 Raytracing::trace): rays = float[8]*count {o,min_t,d,max_t},
 * seeds in/out = sampler state per ray; hits out = {u, v, tri, t} (IntersectionBase, math.hxx:666). */
int etxb_debug_trace(etxb_ctx* ctx, const float* rays, uint32_t* seeds, uint32_t count, float* hits_uv_t, uint32_t* hits_tri);
/* Occlusion query for `count` segments (rt.cxx:468 Raytracing::trace_transmittance in an opaque scene): segments = float[6]*count {p0,p1};
 * occluded out = 1 where a non-Void surface lies between p0 and p1, else 0. */
int etxb_debug_occluded(etxb_ctx* ctx, const float* segments, uint32_t count, uint32_t* occluded);
/* Which tree etxb_debug_trace and etxb_debug_occluded walk: 0 = the BVH2 shared with the oracle, 1 = the product build's 4-wide quantised tree
 * (returns 1 if it exists). */
int etxb_debug_select_tree(etxb_ctx* ctx, int wide);
/* Both trees of a triangle soup, built without committing a scene: with the host builder (device = 0: csrc/bvh_build.cpp, the specification)
 * or on the device (device = 1: what etxb_upload_scene runs).  positions = float[3*vertex_count], indices = uint32[3*triangle_count] (each
 * index below vertex_count).  The caller sizes every array for max(1, triangle_count) entries (nodes of 64 bytes, tri_pos of 3 float4, tri_index
 * of one uint32, wide nodes of 64 bytes); the counts, max_depth and max_stack come back, and `seconds` is the wall time of the two builds. */
typedef struct etxb_debug_trees {
  void* bvh_nodes;
  float* tri_pos;
  uint32_t* tri_index;
  void* wide_nodes;
  uint32_t bvh_node_count, slot_count, wide_node_count, max_depth, max_stack, pad;
  double seconds;
} etxb_debug_trees;
int etxb_debug_build_trees(etxb_ctx* ctx, const float* positions, uint32_t vertex_count, const uint32_t* indices, uint32_t triangle_count, uint32_t device,
                           etxb_debug_trees* out);
/* etxb_denoise's kernels on host arrays: color / camera / half / normals / albedo / out / out_variance are float[4 * width * height] (RGBA,
 * one layout for every array); counts = uint32[width * height] samples per pixel; normals and albedo may be null (no feature weight) and
 * out_variance may be null.  out_variance receives the smoothed per-pixel variance of the mean.  ETXB_ERR_NOT_READY where a count is below 2. */
int etxb_debug_denoise(etxb_ctx* ctx, const float* color, const float* camera, const float* half, const uint32_t* counts, const float* normals,
                       const float* albedo, uint32_t width, uint32_t height, float* out, float* out_variance);
/* etxb_read_film_view's kernel on host arrays: layer / reference = float[4 * count] (reference may be null for views 0-2); out = float[4 * count]
 * or uint8[4 * count] as view->rgba8 says. */
int etxb_debug_film_view(etxb_ctx* ctx, const float* layer, const float* reference, uint32_t count, const etxb_view* view, void* out);
/* etxb_film_error's kernels on host arrays (float[4 * width * height] each); `iterations` comes back 0. */
int etxb_debug_film_error(etxb_ctx* ctx, const float* layer, const float* reference, uint32_t width, uint32_t height, etxb_film_error_info* out);
/* The path tracer's noise estimate (etxb_enqueue_iteration's Film::estimate_noise_levels) on host arrays, as `world` pixel-tile ranks run it:
 * each rank's view holds its own pixels and zeros elsewhere, the level pass runs per rank, the masks are summed (the all-reduce), the dilation
 * runs per rank and the owned pixels are composed.  world = 1 is the one-GPU estimate.  camera / adaptive = float[4 * width * height] and
 * info_in / info_out = uint32[width * height] (ETXB_BUF_PIXEL_INFO words), in storage order; error_out = float[width * height]
 * (ETXB_BUF_PIXEL_ERROR, zero where a pixel was not evaluated); stats_out = uint32[2]: the converged count and the bits of the float error sum. */
int etxb_debug_noise_estimate(etxb_ctx* ctx, uint32_t width, uint32_t height, uint32_t world, float threshold, const float* camera, const float* adaptive,
                              const uint32_t* info_in, uint32_t* info_out, float* error_out, uint32_t* stats_out);
/* Sampler / spectral KATs evaluated on the device (sampler.hxx:54,66; spectrum.hxx:219,234). */
int etxb_debug_sampler(etxb_ctx* ctx, const uint32_t* a, const uint32_t* b, uint32_t count, uint32_t draws, uint32_t* out_seed, float* out_values);
int etxb_debug_math(etxb_ctx* ctx, uint32_t fn, const float* x, const float* y, uint32_t count, float* out);
/* Vertex-closure query (dclosure.cuh: make_closure + closure_evaluate, as the photon gather and the vertex connections run them) on the
 * uploaded scene.  One query is 96 bytes: the shading frame as interpolated, w_i pointing AT the surface (BSDFData::w_i), w_o pointing away,
 * uv, the wavelength (ignored in RGB scenes, which use the undefined wavelength -1), the material index, the path source (1 = camera,
 * 2 = light) and a sampler seed. */
typedef struct etxb_closure_query {
  float nrm[3], tan[3], btn[3];
  float w_i[3], w_o[3];
  float uv[2];
  float wavelength;
  uint32_t material, path_source, seed;
  uint32_t reserved[3];
} etxb_closure_query;
/* Per query, `repetitions` evaluations; repetition r starts from the sampler Smp::init(seed, r) (= the reference's Sampler(seed, r)).
 * out = double[ETXB_CLOSURE_STATS] per query: the outputs are ordered {func.rgb, bsdf.rgb, pdf, rev_pdf} (a spectral value fills all three
 * components); [0..8) their means, [8..16) their variances (population, over the finite repetitions), [16..24) repetition 0's raw values,
 * [24] the number of repetitions with a non-finite output, [25] with pdf < 0 or rev_pdf < 0, [26] with pdf == 0 but a non-zero func or bsdf. */
#define ETXB_CLOSURE_STATS 32
int etxb_debug_closure_eval(etxb_ctx* ctx, const etxb_closure_query* queries, uint32_t count, uint32_t repetitions, double* out);
/* BSDF sampling query (dbsdf.cuh bsdf_sample, as every bounce of the light pass, the camera pass and the path tracer calls it) on the
 * uploaded scene.  One query is 96 bytes: the shading frame as interpolated, w_i pointing AT the surface, uv, the wavelength (ignored in
 * RGB scenes), the material index, the path source (1 = camera, 2 = light), a sampler seed, the current medium (what Boundary and Void
 * return), the mode and three fixed values.  Repetition r starts from the sampler Smp::init(seed, r) (= the reference's Sampler(seed, r)):
 *   mode 0 ("bounce")  draws rnd_bsdf, rnd_connection, rnd_support with next_2d() and pushes (rnd_bsdf.x, rnd_bsdf.y, rnd_support.x)
 *                      as the fixed values, as a bounce does (vcm_shared.hxx:1013-1025)
 *   mode 1 ("given")   pushes fixed[0..3) as they are
 * then bsdf_sample and pop_fixed. */
typedef struct etxb_sample_query {
  float nrm[3], tan[3], btn[3];
  float w_i[3];
  float uv[2];
  float wavelength;
  uint32_t material, path_source, seed, medium, mode;
  float fixed[3];
  uint32_t reserved;
} etxb_sample_query;
/* One 48-byte record per (query, repetition), repetition-minor: w_o, pdf, weight (rgb; a spectral value fills all three), eta, properties
 * (BSDFSample::Properties), medium_index, the sampler state Smp::init(seed, r) left and the state after pop_fixed (their distance in the
 * stream is the number of draws the sample made). */
typedef struct etxb_sample_result {
  float w_o[3];
  float pdf;
  float weight[3];
  float eta;
  uint32_t properties, medium_index, seed_start, seed_end;
} etxb_sample_result;
int etxb_debug_bsdf_sample(etxb_ctx* ctx, const etxb_sample_query* queries, uint32_t count, uint32_t repetitions, etxb_sample_result* out);
/* Emitter query (dvcm.cuh: the emitter selection, sample_emitter, sample_emission and emitter_get_radiance, as the light pass, the camera
 * pass and the path tracer call them) on the uploaded scene.  One query is 80 bytes: the op, an emitter index, a sampler seed,
 * directly_visible (0 / 1), a 2-D random number, the wavelength (ignored in RGB scenes), a source and a target position, a direction and a
 * uv.  The ops:
 *   0 select     distribution_sample(emitter_dist, emitter_count + 1, rnd[0]): emitter_index and emitter_discrete_pdf as pdf_sample
 *   1 sample_in  sample_emitter(emitter, rnd, from_point = source): next-event estimation
 *   2 emission   sample_emission on the sampler Smp::init(seed, r) of repetition r: the start of a light path
 *   3 radiance   emitter_get_radiance(emitter, source, target, direction, uv, directly_visible): value and pdf_area, pdf_dir, pdf_dir_out
 * Ops 0, 1 and 3 ignore the seed and return the same record for every repetition; op 0 ignores the emitter index. */
typedef struct etxb_emitter_query {
  uint32_t op, emitter, seed, directly_visible;
  float rnd[2];
  float wavelength;
  float source[3], target[3], direction[3];
  float uv[2];
  uint32_t reserved[2];
} etxb_emitter_query;
#define ETXB_EMITTER_SELECT 0u
#define ETXB_EMITTER_SAMPLE_IN 1u
#define ETXB_EMITTER_EMISSION 2u
#define ETXB_EMITTER_RADIANCE 3u
/* One 104-byte record per (query, repetition), repetition-minor: every field of the device EmitterSample (the value, rgb; a spectral value
 * fills all three), flags (bit 0 is_delta, bit 1 is_distant), and for op 2 the sampler state Smp::init(seed, r) left and the state after
 * sample_emission (0 for the other ops).  Op 0 fills emitter_index and pdf_sample, op 3 value, the three pdfs and emitter_index; in
 * both, triangle_index and medium_index are 0xffffffff (kInvalidIndex) and the other fields 0. */
typedef struct etxb_emitter_result {
  float value[3];
  float origin[3], normal[3], direction[3], barycentric[3];
  float pdf_sample, pdf_area, pdf_dir, pdf_dir_out;
  uint32_t emitter_index, triangle_index, medium_index, flags, seed_start, seed_end, reserved;
} etxb_emitter_result;
int etxb_debug_emitter(etxb_ctx* ctx, const etxb_emitter_query* queries, uint32_t count, uint32_t repetitions, etxb_emitter_result* out);
/* Medium query (dmedium.cuh and trace_transmittance of dtrace.cuh, as the bounces and shadow rays call them) on the uploaded scene.  One
 * query is 96 bytes: the op, a medium index, a sampler seed, the wavelength (ignored in RGB scenes), an origin, a direction, a distance
 * max_t, an end point, a throughput (rgb; a spectral throughput is throughput[0]), a phase g, a 2-D random number and a second direction
 * w_o.  The ops:
 *   0 bounds         medium_intersects_bounds(medium, origin, direction, max_t): flag, pos / dir (the medium's local frame), t_min, t_max
 *   1 density        medium_sample_density(medium, origin as a local coordinate): value[0]; the medium must be heterogeneous
 *   2 transmittance  medium_transmittance(medium, origin, direction, max_t): value
 *   3 sample         sample_medium(medium, throughput, origin, direction, max_t): value = weight, pos, t = sampled_medium_t;
 *                    max_t must be at least kRayEpsilon (the homogeneous free-flight loop runs while t < kRayEpsilon)
 *   4 phase          phase_function(direction, w_o, g): value[0]; sample_phase_function(direction, g, rnd): dir.  Ignores the medium.
 *   5 segment        trace_transmittance<SP, false>(origin, end, medium) on the scene's BVH: value; medium 0xffffffff = no medium
 * Every op runs on the sampler Smp::init(seed, r) of repetition r; ops 0, 1 and 4 draw nothing.  The hook refuses, before any launch, an
 * op past 5, a medium index past the scene's count (except 0xffffffff for op 5; op 4 ignores it), a zero or non-finite direction
 * (ops 0 to 4), a non-finite origin, end point, max_t, throughput or wavelength, coordinates past 1e15, heterogeneous tracking whose
 * local segment would overflow or whose max_sigma x (|local origin| + 2) passes 2^16 (op 5: in every heterogeneous medium), a
 * homogeneous sample whose extinction x kRayEpsilon passes 8, and count x repetitions past 2^31. */
typedef struct etxb_medium_query {
  uint32_t op, medium, seed, reserved0;
  float wavelength;
  float origin[3], direction[3];
  float max_t;
  float end[3];
  float throughput[3];
  float g;
  float rnd[2];
  float w_o[3];
} etxb_medium_query;
#define ETXB_MEDIUM_BOUNDS 0u
#define ETXB_MEDIUM_DENSITY 1u
#define ETXB_MEDIUM_TRANSMITTANCE 2u
#define ETXB_MEDIUM_SAMPLE 3u
#define ETXB_MEDIUM_PHASE 4u
#define ETXB_MEDIUM_SEGMENT 5u
/* One 64-byte record per (query, repetition), repetition-minor: value (rgb; a spectral value fills all three), pos, dir, t_min, t_max, t
 * (sampled_medium_t), flag (op 0: 1 when the segment meets the bounds), and the sampler state Smp::init(seed, r) left and the state after
 * the op, for every op.  Fields an op does not name are 0. */
typedef struct etxb_medium_result {
  float value[3], pos[3], dir[3];
  float t_min, t_max, t;
  uint32_t flag, seed_start, seed_end, reserved;
} etxb_medium_result;
int etxb_debug_medium(etxb_ctx* ctx, const etxb_medium_query* queries, uint32_t count, uint32_t repetitions, etxb_medium_result* out);
/* Subsurface query (dsss.cuh, as the bounces call it) on the uploaded scene.  One query is 128 bytes: the op, a sampler seed, a material
 * index, a triangle index, a hit-buffer size max_count, a probe direction (0 to 2), the wavelength (ignored in RGB scenes), barycentric
 * coordinates u, v on the triangle, a ray (origin, direction, t_min, t_max), a color and scattering distances, a random number rnd, a
 * radius and a normal.  The ops:
 *   0 trace_material    trace_material(origin, direction, t_min, t_max, material; 0xffffffff = any material): hits[0], count 0 or 1
 *   1 continuous_trace  continuous_trace(the same, max_count): count and hits[0, count) in buffer order
 *   2 remap             remap_channel(color[k], distances[k]) for k = 0, 1, 2: albedo, extinction, scattering
 *   3 profile           at the entry make_intersection(direction, triangle, u, v): s_r = sample_s_r(rnd), eval = ss_evaluate(radius)
 *                       at the entry's texture coordinates, probes[0] = ss_sample(probe direction) on the sampler (three draws, one when
 *                       its channel's distance is 0), geometric_weight = ss_geometric_weight(normal, probes[0])
 *   4 gather            ss_gather at the entry make_intersection(direction, triangle, u, v) (its material is the triangle's): flag (the
 *                       return), count, selected, selected_sample_weight, total_weight, rays, per exit hits[i] with the w_i, weight, pos
 *                       and nrm of ss_exit_intersection; for a Christensen-Burley material, probes[0..2] are the gather's three samples
 * Every op runs on the sampler Smp::init(seed, r) of repetition r.  The hook refuses, before any launch, an op past 4, a material index
 * past the scene's count (ops 0 and 1; 0xffffffff is any material), a triangle index past the scene's count (ops 3 and 4), a gather on a
 * triangle whose material has no subsurface class, a max_count of 0 or above 8 (op 1), a non-finite input the op reads, a zero
 * direction (ops 0, 1, 3 and 4), and count x repetitions past 2^31. */
typedef struct etxb_subsurface_query {
  uint32_t op, seed, material, triangle, max_count, direction;
  float wavelength, u, v;
  float origin[3], dir[3];
  float t_min, t_max;
  float color[3], distances[3];
  float rnd, radius;
  float normal[3];
  uint32_t reserved[4];
} etxb_subsurface_query;
#define ETXB_SUBSURFACE_TRACE_MATERIAL 0u
#define ETXB_SUBSURFACE_CONTINUOUS_TRACE 1u
#define ETXB_SUBSURFACE_REMAP 2u
#define ETXB_SUBSURFACE_PROFILE 3u
#define ETXB_SUBSURFACE_GATHER 4u
/* One probe of a Christensen-Burley gather (96 bytes): the ray (origin, direction, t_min, t_max), the basis u, v, w, basis_prob and
 * sampled_radius; an empty probe is origin 0, direction 0, [kRayEpsilon, kMaxFloat] with everything else 0. */
typedef struct etxb_subsurface_probe {
  float o[3], d[3], min_t, max_t, u[3], v[3], w[3], basis_prob[3], sampled_radius;
  uint32_t reserved[3];
} etxb_subsurface_probe;
/* One hit (64 bytes): barycentric u, v, t and triangle (0xffffffff = none); for a gather exit also w_i, weight (rgb; a spectral value
 * fills all three), and the pos and nrm of ss_exit_intersection. */
typedef struct etxb_subsurface_hit {
  float u, v, t;
  uint32_t tri;
  float w_i[3], weight[3], pos[3], nrm[3];
} etxb_subsurface_hit;
/* One 1920-byte record per (query, repetition), repetition-minor: the fields each op names above, and the sampler state Smp::init(seed,
 * r) left and the state after the op, for every op.  Fields an op does not name are 0. */
typedef struct etxb_subsurface_result {
  uint32_t flag, count, selected, rays, seed_start, seed_end;
  float selected_sample_weight, total_weight;
  float albedo[3], extinction[3], scattering[3];
  float s_r, eval[3], geometric_weight;
  uint32_t reserved[2];
  etxb_subsurface_probe probes[3];
  etxb_subsurface_hit hits[24];
} etxb_subsurface_result;
int etxb_debug_subsurface(etxb_ctx* ctx, const etxb_subsurface_query* queries, uint32_t count, uint32_t repetitions, etxb_subsurface_result* out);
/* Queue sizes from which the light and camera passes take their large-queue branches.  A pass of a long queue runs the same paths as
 * one of a short queue, in another order; these let a small film take either branch.  Each field is a queue size: 0 = always the
 * large-queue branch, 0xffffffff = never.
 *   merge_sort_min_queries  the gather queue is sorted by its merge keys (default 16384); must not be below tail_queue
 *   merge_min_warps_per_sm  the gather gives a warp 32 queries, halved while the queue fills fewer than this many warps per SM (default 32)
 *   tail_queue              from this size the vertex connections run over the host-sized pair list and the queue size is read back every
 *                           bounce; below it, every 4 bounces (default 8192)
 *   sort_queue_min          scenes with stochastic BSDFs: path queues and connection pair lists are sorted by material (default 1024)
 *   merge_qpw               queries per warp of the gather, 1, 2, 4, ..., 32; 0 = chosen from merge_min_warps_per_sm (default 0)
 * NULL restores the defaults; the setting stays until the next call. */
typedef struct etxb_debug_thresholds {
  uint32_t merge_sort_min_queries, merge_min_warps_per_sm, tail_queue, sort_queue_min, merge_qpw;
} etxb_debug_thresholds;
int etxb_debug_set_thresholds(etxb_ctx* ctx, const etxb_debug_thresholds* thresholds);
/* Host-side counts since the last etxb_begin of the branches above: gather-queue sorts, gather launches by queries per warp
 * (index k = 2^k queries; the parity build's serial gather counts as 1), vertex-connection launches over the host-sized pair list,
 * pair-list sorts and path-queue sorts. */
typedef struct etxb_debug_branch_counts {
  uint64_t merge_sorts;
  uint64_t merge_launches[6];
  uint64_t connect_launches, pair_sorts, queue_sorts;
} etxb_debug_branch_counts;
int etxb_debug_get_branch_counts(etxb_ctx* ctx, etxb_debug_branch_counts* out);
/* The photon gather (VCMSpatialGridData::gather, vcm_shared.hxx:805-925), query by query, through the launch code of the camera pass.
 * `records` = `record_count` light-vertex records of the device layout (96 B each: {throughput.xyz, d_vcm}, {w_i, d_vc}, {barycentric, d_vm},
 * {pos, triangle}, {nrm, material}, {medium, path_length, path_index, ordinal}); `light_wavelengths` = one wavelength per light path index
 * (path_count of them; ignored in RGB scenes).  The photon grid is built from them at the context's current iteration and options, then
 * each query becomes one camera vertex of a one-bounce queue (at most path_count queries) with the merge key the camera pass gives it, and the
 * gather runs under the current etxb_debug_set_thresholds: the parity build's serial gather; the product build's Lambert and closure gathers.
 * The context's path state, photon grid and light image change; call etxb_begin before rendering again. */
typedef struct etxb_merge_query {
  uint32_t tri;                       /* the hit: triangle and the barycentrics (u, v) etxb_debug_trace returns */
  float u, v;
  float w_i[3];                       /* the direction the camera path arrived along (pointing AT the surface) */
  float throughput[3];
  float wavelength;                   /* ignored in RGB scenes */
  float d_vcm, d_vm;
  uint32_t total_path_depth, seed, medium;
  uint32_t reserved;
} etxb_merge_query;
typedef struct etxb_merge_result {
  float merged[3];                    /* what the gather added to VCMPathState::merged */
  uint32_t seed;                      /* the path's sampler state afterwards */
  float pos[3], nrm[3];               /* the staged camera vertex */
  uint32_t reserved[2];
} etxb_merge_result;
typedef struct etxb_merge_grid {
  float bbox_min[3], bbox_max[3];     /* the photon grid the queries were gathered on */
  float cell_size, radius_squared;
  uint32_t hash_table_mask, photon_count;
  uint64_t merge_queries, merge_candidates, merge_accepts;  /* the gather's counters for this call */
} etxb_merge_grid;
int etxb_debug_merge(etxb_ctx* ctx, const void* records, uint32_t record_count, const float* light_wavelengths, const etxb_merge_query* queries, uint32_t count,
                     etxb_merge_result* out, etxb_merge_grid* grid);

/* ---- several iterations in flight on one device -----------------------------------------------------------------------
 * The reference runs ONE iteration at a time and spreads its paths over the CPU's threads (vcm_cpu.cxx:115-171, TaskScheduler).
 * A GPU wavefront iteration ends in a long, latency-bound tail (few paths, ~50 more bounces); an etxb_group keeps `lanes`
 * independent contexts on one device, one host thread each, pulling iteration indices from per-lane queues that etxb_group_enqueue
 * fills, so that tail overlaps other iterations.  Uploads/options go to every lane (etxb_group_lane); the film is the mean of the lanes' films weighted by the
 * iterations each finished — the same set of iterations as a single context running them in order.
 * Replaces the run()/update() pump of CPUVCM (vcm_cpu.cxx:247-276) for throughput rendering. */
typedef struct etxb_group etxb_group;
int etxb_group_create(etxb_group** out_group, const etxb_device_config* config, uint32_t lanes); /* 1..8 lanes */
void etxb_group_destroy(etxb_group* group);
uint32_t etxb_group_lanes(const etxb_group* group);
etxb_ctx* etxb_group_lane(etxb_group* group, uint32_t lane);
const char* etxb_group_last_error(const etxb_group* group);
int etxb_group_begin(etxb_group* group, uint32_t first_iteration);   /* Integrator::run: clears every lane's film */
/* etxb_set_film_pixel_size for every lane (waits for the group to go idle); ETXB_ERR_UNSUPPORTED above 1 on a group with communicators */
int etxb_group_set_film_pixel_size(etxb_group* group, uint32_t size);
/* etxb_update_scene for every lane: waits for the group to go idle, validates and hashes once (and builds a new geometry's BVH once),
 * updates each lane, then etxb_group_begin(group, 0).  `info` is lane 0's, with `kept` the bits every lane kept.  ETXB_ERR_UNSUPPORTED on
 * a group with communicators (etxb_group_comm_init, etxb_group_comm_init_replicas). */
int etxb_group_update_scene(etxb_group* group, const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes, etxb_update_info* info);
int etxb_group_enqueue(etxb_group* group, uint32_t iterations);      /* asynchronous: queues `iterations` more iterations */
int etxb_group_wait(etxb_group* group);                              /* blocks until the queue has drained; returns the first error */
int etxb_group_poll(etxb_group* group, etxb_status* status);         /* completed = sum over lanes; total_time = wall time with work in flight */
int etxb_group_read_film(etxb_group* group, uint32_t layer, float* dst_rgba, uint64_t dst_bytes);

/* ---- pixel-tile sharding over several GPUs (one process per GPU, NCCL over NVLink) ----------------------------------------
 * The reference renders one frame with one thread pool (vcm_cpu.cxx:115-241).  Here rank r owns the 32x32 pixel tiles with tile % world == r
 * (etxb_set_partition's rule) and runs the light and camera subpaths of its pixels; what is global is exchanged INSIDE etxb_enqueue_iteration:
 * all-reduce of the per-iteration light image (light-tracing splats land on any pixel, vcm_cpu.cxx:147-154 -> film.cxx:332-343) and an
 * all-gather of the photon records (merging queries every light path's vertices, vcm_cpu.cxx:219-221).  The host only distributes the NCCL id
 * (any transport: MPI, a file, torch.distributed) — rank 0 calls etxb_comm_unique_id, every rank calls etxb_comm_init with those bytes.
 * The path tracer (ETXB_INTEGRATOR_PT) runs over the same tiles.  Its noise estimate (Film::estimate_noise_levels) is the one global step: each
 * rank packs a mask of its pixels that have not converged (one bit per pixel, ceil(W / 32) words per row), the ranks all-reduce the masks
 * with the converged count, the error sum and pixels_processed, and each rank dilates the whole mask onto its own pixels.  Every other
 * iteration only pixels_processed is all-reduced (4 bytes).  The collectives of an iteration follow from its index, the noise threshold and
 * Scene::samples, so these, and the options, must be equal on every rank; a rank whose tiles have all converged traces no path but keeps
 * joining the collectives until etxb_pt_status says the frame is done. */
#define ETXB_COMM_ID_BYTES 128
int etxb_comm_unique_id(void* out_id, uint64_t bytes);
int etxb_comm_init(etxb_ctx* ctx, uint32_t world, uint32_t rank, const void* id, uint64_t bytes); /* collective */
int etxb_comm_world(const etxb_ctx* ctx, uint32_t* world, uint32_t* rank);
/* Collective: sums the disjoint tiles of `layer` on rank 0 (ncclReduce of the float4 layer); dst_rgba is written on rank 0 only, with
 * etxb_read_film's read-out.  Layers: Result, Camera, Light (complete on every rank), and the path tracer's Normals, Albedo and CameraAdaptive.
 * ETXB_ERR_INVALID_ARGUMENT for LightIteration and Denoised. */
int etxb_comm_reduce_film(etxb_ctx* ctx, uint32_t layer, float* dst_rgba, uint64_t dst_bytes);
/* The same with several iterations in flight per GPU: ids = (lanes + 1) x ETXB_COMM_ID_BYTES (one communicator per lane + one for the frame
 * reduce); lane l renders the iteration ordinals l, l + lanes, ... on every rank.  ETXB_ERR_INVALID_ARGUMENT, before any collective, on a group
 * that already has a communicator (from either init) or, for world >= 2, a split lane. */
int etxb_group_comm_init(etxb_group* group, uint32_t world, uint32_t rank, const void* ids, uint32_t id_count); /* collective */
/* Whole-frame iterations dealt to the ranks instead (the job's j-th iteration on rank j % world; etxb_group_enqueue then counts iterations of the
 * JOB): no collective inside an iteration, one count-weighted ncclReduce of the films per frame.  id = one ETXB_COMM_ID_BYTES id.
 * ETXB_ERR_INVALID_ARGUMENT, before any collective, on a group that already has a communicator. */
int etxb_group_comm_init_replicas(etxb_group* group, uint32_t world, uint32_t rank, const void* id, uint64_t bytes); /* collective */
/* Optional, before etxb_group_comm_init_replicas: reserves the group's LAST lane for camera-split iterations.  When an etxb_group_enqueue(n >= world)
 * is not a multiple of the ranks, its last n % world iterations are then split over world / (n % world) ranks each: every part traces the whole
 * light pass itself (same photon map, no exchange) and the camera pass of its pixel tiles, and the parts meet in etxb_group_comm_reduce_film —
 * instead of leaving some ranks one whole iteration behind the others.  ETXB_ERR_INVALID_ARGUMENT on a group in pixel-tile mode. */
int etxb_group_reserve_split_lane(etxb_group* group);
/* Test hook (needs no device): the queues a `lanes`-lane group on rank `rank` of `world` holds after etxb_group_begin and one
 * etxb_group_enqueue(enqueues[i]) per entry, in `mode` 0 (one GPU), 1 (pixel tiles) or 2 (replicas), with its last lane reserved for camera-split
 * iterations if `split_lane`: (queue, ordinal, part, parts) quads, queue by queue in the order the lanes pop them; returns their number. */
int etxb_debug_group_plan(uint32_t mode, uint32_t lanes, uint32_t world, uint32_t rank, int split_lane, const uint32_t* enqueues, uint32_t count,
                          uint32_t* out_quads, uint32_t capacity);
int etxb_group_comm_reduce_film(etxb_group* group, uint32_t layer, float* dst_rgba, uint64_t dst_bytes);        /* collective, both modes */

#ifdef __cplusplus
}
#endif
#endif /* ETX_B200_H */
