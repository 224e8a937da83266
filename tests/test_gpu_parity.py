"""Parity tests proper: the CUDA path (through the C ABI) against the oracle / its committed golden vectors.  Run with -m gpu.

parity flavor (libetx_b200_parity.so: -fmad=false + portable transcendentals): BIT-EXACT sampler states, light-vertex pool and camera
film; the light image is float-atomic accumulated, so it is compared with a 1e-6 relative-L2 tolerance.
fast flavor (libetx_b200.so, the product build): FMA contraction + CUDA libm change roundings, a few paths per thousand take a
different branch (RR / hit order), and camera-side connections / stochastic merges draw from per-item derived streams; it is held to a
per-image relative-L2 tolerance (2e-2 at 3 spp for the Lambert/delta configs) and >= 97 % identical light-path sampler end states.
"""
import numpy as np
import pytest

from conftest import bit_equal, golden, rel_l2
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


C1 = dict(samples=16, spectral=False)
C2 = dict(samples=256, spectral=True, sphere=True)


def test_native_library_is_the_one_loaded(api):
    g = api.GPUVCM(scenes.cornell_box(16, 16, **C1), flavor="fast")
    assert g.lib.etxb_build_flavor().decode() == "fast"
    g.render(1)
    c = g.counters()
    assert c["kernel_launches"] > 0 and c["rays_closest"] > 0
    g.close()


def test_device_kats_are_bit_exact(api):
    k = golden("kat.npz")
    g = api.GPUVCM(scenes.cornell_box(16, 16, **C2), flavor="parity")
    seeds, vals = g.debug_sampler(k["sampler_a"], k["sampler_b"], 16)
    assert bit_equal(seeds, k["sampler_seeds"]) and bit_equal(vals, k["sampler_values"])
    assert bit_equal(g.debug_math(7, k["x"]), k["spectral_sample"])
    assert bit_equal(g.debug_math(8, k["wl"]), k["sampling_pdf"])
    for fn, key in ((9, "to_rgb_x"), (10, "to_rgb_y"), (11, "to_rgb_z")):
        assert bit_equal(g.debug_math(fn, k["wl"]), k[key])
    assert bit_equal(g.debug_math(14, k["bn_pixel"], k["bn_sample"]), k["bn_dim0_x"])
    assert bit_equal(g.debug_math(15, k["bn_pixel"], k["bn_sample"]), k["bn_dim4_y"])
    for nm, fn in (("sin", 0), ("cos", 1), ("exp", 2), ("log", 3), ("acos", 5), ("atan", 12), ("asin", 13)):
        assert bit_equal(g.debug_math(fn, k[f"pm_{nm}_x"]), k[f"pm_{nm}"]), nm
    assert bit_equal(g.debug_math(4, k["pm_pow_x"], k["pm_pow_y"]), k["pm_pow"])
    assert bit_equal(g.debug_math(6, k["pm_atan2_x"], k["pm_atan2_y"]), k["pm_atan2"])
    g.close()


def test_sampler_is_bit_exact_in_the_product_build_too(api):
    k = golden("kat.npz")
    g = api.GPUVCM(scenes.cornell_box(16, 16, **C1), flavor="fast")
    seeds, vals = g.debug_sampler(k["sampler_a"], k["sampler_b"], 16)
    assert bit_equal(seeds, k["sampler_seeds"]) and bit_equal(vals, k["sampler_values"])
    g.close()


def test_closest_hit_matches_golden_rays(api):
    t = golden("trace_c2.npz")
    sd = scenes.cornell_box(32, 32, **C2)
    g = api.GPUVCM(sd, flavor="parity")
    uvt, tri, seeds = g.debug_trace(t["rays"], t["seeds"])
    assert bit_equal(tri, t["tri"]) and bit_equal(uvt, t["uvt"]) and bit_equal(seeds, t["seeds_out"])
    assert (tri != S.INVALID).mean() > 0.99  # closed box: (almost) every ray hits
    g.close()
    f = api.GPUVCM(sd, flavor="fast")
    uvt, tri, seeds = f.debug_trace(t["rays"], t["seeds"])
    same = tri == t["tri"]
    assert same.mean() > 0.995
    np.testing.assert_allclose(uvt[same][:, 2], t["uvt"][same][:, 2], rtol=1e-4, atol=1e-5)
    f.close()


@pytest.mark.parametrize("name,kwargs", [("oracle_c1_32.npz", C1), ("oracle_c2_32.npz", C2)])
def test_iteration_is_bit_exact_against_golden_render(api, name, kwargs):
    ref = golden(name)
    g = api.GPUVCM(scenes.cornell_box(32, 32, **kwargs), flavor="parity")
    st = g.render(int(ref["iterations"][0]))
    assert st["overflow"] == 0 and st["completed_iterations"] == int(ref["iterations"][0])
    assert bit_equal(g.buffer(S.BUF_LIGHT_SAMPLER, np.uint32), ref["light_sampler"])
    assert bit_equal(g.buffer(S.BUF_LIGHT_PATH_COUNT, np.uint32), ref["light_path_count"])
    assert bit_equal(g.buffer(S.BUF_LV_POS, np.float32), ref["lv_pos"])
    assert bit_equal(g.buffer(S.BUF_CAMERA_SAMPLER, np.uint32), ref["camera_sampler"])
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], ref["film_camera"][..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], ref["film_light"][..., :3]) < 1e-6
    assert rel_l2(g.film(S.FILM_RESULT)[..., :3], ref["film_result"][..., :3]) < 1e-6
    g.close()


@pytest.mark.parametrize("name", ["oracle_c3_24.npz", "oracle_c4_24.npz", "oracle_c5_24.npz", "oracle_vmf_24.npz"])
def test_configs_3_to_5_are_bit_exact_against_golden_renders(api, name):
    """Committed oracle renders of BASELINE configs 3-5 (full geometry, small film) and of the vMF diffuse box: the fixtures travel to the
    GPU box, the reference does not."""
    import golden_scenes
    factory, iters, opts = golden_scenes.SCENES[name]
    ref = golden(name)
    g = api.GPUVCM(factory(), flavor="parity")
    if opts:
        g.options[:] = opts()
    st = g.render(iters)
    assert st["overflow"] == 0 and st["completed_iterations"] == int(ref["iterations"][0]) == iters
    assert bit_equal(g.buffer(S.BUF_LIGHT_SAMPLER, np.uint32), ref["light_sampler"])
    assert bit_equal(g.buffer(S.BUF_LIGHT_PATH_COUNT, np.uint32), ref["light_path_count"])
    assert bit_equal(g.buffer(S.BUF_LV_POS, np.float32), ref["lv_pos"])
    assert bit_equal(g.buffer(S.BUF_CAMERA_SAMPLER, np.uint32), ref["camera_sampler"])
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], ref["film_camera"][..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], ref["film_light"][..., :3]) < 1e-6
    g.close()


@pytest.mark.parametrize("kwargs,options", [
    (C1, None), (C2, None),
    (C1, dict(options=S.VCM_CONNECT_ONLY)),                                  # "volumetric BDPT" = VCM without merging (BASELINE config 5)
    (C2, dict(options=S.VCM_FULL & ~S.VCM_ENABLE_MIS, kernel=0, blue_noise=0)),  # no MIS, top-hat kernel, no blue noise
    (C1, dict(initial_radius=0.05, radius_decay=4)),
])
def test_iteration_is_bit_exact_against_live_oracle(api, oracle_mod, kwargs, options):
    sd = scenes.cornell_box(48, 40, **kwargs)  # non-square film exercises the y-flip and aspect handling
    opts = S.default_vcm_options()
    for k, v in (options or {}).items():
        opts[k] = v
    o = oracle_mod.Oracle(sd)
    o.set_options(opts)
    o.begin(0)
    o.run(3, threads=1)
    g = api.GPUVCM(sd, flavor="parity")
    g.options[:] = opts
    g.render(3)
    for bid, dt in ((S.BUF_LIGHT_PATH_COUNT, np.uint32), (S.BUF_LIGHT_PATH_OFFSET, np.uint32), (S.BUF_LIGHT_PATH_WAVELENGTH, np.float32),
                    (S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_LV_POS, np.float32), (S.BUF_LV_THROUGHPUT, np.float32), (S.BUF_LV_MIS, np.float32),
                    (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_CAMERA_GATHERED, np.float32)):
        assert bit_equal(g.buffer(bid, dt), o.buffer(bid, dt)), f"buffer {bid}"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], o.film(S.FILM_LIGHT)[..., :3]) < 1e-6
    gc, oc = g.counters(), o.counters()
    for key in ("rays_closest", "rays_shadow", "bounces_light", "bounces_camera", "splats"):
        assert gc[key] == int(oc[key][0]), key
    g.close()


@pytest.mark.parametrize("name,kwargs", [("oracle_c1_32.npz", C1), ("oracle_c2_32.npz", C2)])
def test_product_build_is_within_tolerance(api, name, kwargs):
    ref = golden(name)
    g = api.GPUVCM(scenes.cornell_box(32, 32, **kwargs), flavor="fast")
    g.render(int(ref["iterations"][0]))
    assert (g.buffer(S.BUF_LIGHT_SAMPLER, np.uint32) == ref["light_sampler"]).mean() >= 0.97
    # (scenes with stochastic BSDFs run connections / merges as parallel stages with derived streams in the product build; these two
    # configs are Lambert + delta only, so the camera streams stay in the reference's order as well)
    assert (g.buffer(S.BUF_CAMERA_SAMPLER, np.uint32) == ref["camera_sampler"]).mean() >= 0.97
    img = g.film(S.FILM_RESULT)[..., :3]
    assert np.isfinite(img).all()
    assert rel_l2(img, ref["film_result"][..., :3]) < 2e-2  # per-image relative L2 tolerance of the product build
    assert abs(img.mean() - ref["film_result"][..., :3].mean()) / ref["film_result"][..., :3].mean() < 5e-3
    g.close()


def test_full_size_properties_config2(api):
    """BASELINE config 2 at its real size (1024x1024, spectral, dielectric sphere): size-independent properties."""
    sd = scenes.config("C2")
    g = api.GPUVCM(sd, flavor="fast")
    st = g.render(1)
    assert st["overflow"] == 0
    a0 = g.film(S.FILM_CAMERA).copy()
    l0 = g.film(S.FILM_LIGHT).copy()
    assert np.isfinite(a0).all() and np.isfinite(l0).all()  # spectral to_rgb may give slightly negative channels
    # determinism: the camera image of an iteration depends only on (pixel, iteration)
    g.render(1)
    assert bit_equal(g.film(S.FILM_CAMERA), a0)
    # iteration 1 alone, then 0+1 together: Film running mean (film.cxx:199-207) => result == lerp(img1, img0, 1/2) exactly
    g.render(1, first_iteration=1)
    a1 = g.film(S.FILM_CAMERA).copy()
    g.render(2)
    both = g.film(S.FILM_CAMERA)[..., :3]
    want = (a1[..., :3] * np.float32(0.5) + a0[..., :3] * np.float32(0.5)).astype(np.float32)
    assert bit_equal(both, want)
    # Result layer = max(0, camera + light) (film.cxx:398-405)
    res = g.film(S.FILM_RESULT)[..., :3]
    cam, lig = g.film(S.FILM_CAMERA)[..., :3], g.film(S.FILM_LIGHT)[..., :3]
    assert bit_equal(res, np.maximum(np.float32(0), cam + lig))
    assert 0.05 < res.mean() < 1.0
    g.close()


def test_pixel_tile_partition_is_exact_without_merging(api):
    """Two ranks' tiles = the full frame: camera subpaths only touch their paired light path (vcm_shared.hxx:771)."""
    W, H = 96, 80
    sd = scenes.cornell_box(W, H, **C1)
    imgs = []
    for rank, world in ((0, 1), (0, 2), (1, 2)):
        g = api.GPUVCM(sd, flavor="parity")
        g.options["options"] = S.VCM_CONNECT_ONLY
        g.set_partition(rank, world)
        g.render(2)
        imgs.append((g.film(S.FILM_CAMERA)[..., :3].copy(), g.film(S.FILM_LIGHT)[..., :3].copy()))
        g.close()
    full, r0, r1 = imgs
    assert bit_equal(r0[0] + r1[0], full[0])  # disjoint pixels: one of the two is exactly zero everywhere
    assert rel_l2(r0[1] + r1[1], full[1]) < 1e-6  # light splats land anywhere: summed like the NCCL all-reduce does
    # path (x, y) lies in tile (y // 32) * ceil(W / 32) + x // 32 and rank r renders the tiles with tile % 2 == r; the Camera layer is
    # stored y-flipped (film.cxx:189), so film row H - 1 - y holds path row y
    ys, xs = np.mgrid[0:H, 0:W]
    owner = (((H - 1 - ys) // 32) * ((W + 31) // 32) + xs // 32) % 2
    for rank, (camera, _) in enumerate((r0, r1)):
        assert (camera.view(np.uint32)[owner != rank] == 0).all(), f"rank {rank} wrote camera pixels outside its tiles"


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("kind", sorted(scenes.MATERIAL_KINDS))
def test_every_material_class_is_bit_exact(api, oracle_mod, kind, spectral):
    """One scene per Material::Class (material.hxx:53-68): stochastic microfacet walks, thin-film Fresnel, delta lobes, mixtures.
    Their evaluate()/pdf() consume the path's sampler, so a single out-of-order draw shows up in the end-of-path sampler states."""
    sd = scenes.material_box(kind, 32, 32, spectral=spectral)
    o = oracle_mod.Oracle(sd)
    o.begin(0)
    o.run(2, threads=1)
    g = api.GPUVCM(sd, flavor="parity")
    g.render(2)
    for bid, dt in ((S.BUF_LIGHT_PATH_COUNT, np.uint32), (S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_LV_POS, np.float32), (S.BUF_LV_THROUGHPUT, np.float32),
                    (S.BUF_LV_MIS, np.float32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_CAMERA_GATHERED, np.float32)):
        a, b = g.buffer(bid, dt), o.buffer(bid, dt)
        assert a.shape == b.shape, f"{kind} buffer {bid}: {a.shape} vs {b.shape}"
        same = (a.view(np.uint32) == b.view(np.uint32))
        assert same.all(), f"{kind} buffer {bid}: {100.0 * same.mean():.3f}% identical, first mismatch at {int(np.argmin(same))}"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], o.film(S.FILM_LIGHT)[..., :3]) < 1e-6
    g.close()
    # product build: same scene within tolerance
    f = api.GPUVCM(sd, flavor="fast")
    f.render(2)
    img, ref = f.film(S.FILM_RESULT)[..., :3], o.film(S.FILM_RESULT)[..., :3]
    assert np.isfinite(img).all()
    assert rel_l2(img, ref) < 0.15 and abs(img.mean() - ref.mean()) / ref.mean() < 0.03
    f.close()


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("variant", [dict(), dict(sun=False, area_light=False), dict(env=False, area_light=False, textures=False), dict(textures=False, sun=False)])
def test_distant_emitters_and_textures_are_bit_exact(api, oracle_mod, variant, spectral):
    """Environment map (importance-sampled lat-long image), finite-size directional emitter, camera misses, scattering / alpha /
    normal / roughness textures (scene_emitters.hxx, image.hxx, scene.hxx:202-226,291-305, scene_bsdf.hxx:128-144)."""
    sd = scenes.sky_room(40, 32, spectral=spectral, **variant)
    o = oracle_mod.Oracle(sd)
    o.begin(0)
    o.run(2, threads=1)
    g = api.GPUVCM(sd, flavor="parity")
    g.render(2)
    for bid, dt in ((S.BUF_LIGHT_PATH_COUNT, np.uint32), (S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_LV_POS, np.float32), (S.BUF_LV_THROUGHPUT, np.float32),
                    (S.BUF_LV_MIS, np.float32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_CAMERA_GATHERED, np.float32)):
        a, b = g.buffer(bid, dt), o.buffer(bid, dt)
        assert a.shape == b.shape, f"buffer {bid}: {a.shape} vs {b.shape}"
        same = (a.view(np.uint32) == b.view(np.uint32))
        assert same.all(), f"buffer {bid}: {100.0 * same.mean():.3f}% identical, first mismatch at {int(np.argmin(same))}"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], o.film(S.FILM_LIGHT)[..., :3]) < 1e-6
    g.close()
    f = api.GPUVCM(sd, flavor="fast")
    f.render(2)
    img, ref = f.film(S.FILM_RESULT)[..., :3], o.film(S.FILM_RESULT)[..., :3]
    assert np.isfinite(img).all() and rel_l2(img, ref) < 0.15
    f.close()


def test_million_triangle_room_is_bit_exact(api, oracle_mod):
    """BASELINE config 3's geometry (998 562 triangles, BVH depth > 30, plastic / conductor / thin-film props, env map) at a small film."""
    sd = scenes.procedural_room(64, 36, env_size=(256, 128))
    assert sd.triangle_count > 990_000
    o = oracle_mod.Oracle(sd)
    o.begin(0)
    o.run(1, threads=1)
    g = api.GPUVCM(sd, flavor="parity")
    g.render(1)
    for bid, dt in ((S.BUF_LIGHT_PATH_COUNT, np.uint32), (S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_LV_POS, np.float32), (S.BUF_CAMERA_SAMPLER, np.uint32),
                    (S.BUF_CAMERA_GATHERED, np.float32)):
        assert bit_equal(g.buffer(bid, dt), o.buffer(bid, dt)), f"buffer {bid}"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    g.close()


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("kind", ["fog", "cloud", "tinted", "camera"])
def test_participating_media_are_bit_exact(api, oracle_mod, kind, spectral):
    """Boundary materials + homogeneous / heterogeneous media (scene_medium.hxx, vcm_shared.hxx:379-449, 934-995, 1097-1170,
    rt.cxx:468-579): free-flight sampling, medium light vertices, explicit connections from medium points, transmittance through
    sorted boundary crossings, ratio tracking."""
    sd = scenes.media_box(kind, 32, 32, spectral=spectral)
    o = oracle_mod.Oracle(sd)
    o.begin(0)
    o.run(2, threads=1)
    g = api.GPUVCM(sd, flavor="parity")
    g.render(2)
    for bid, dt in ((S.BUF_LIGHT_PATH_COUNT, np.uint32), (S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_LV_POS, np.float32), (S.BUF_LV_THROUGHPUT, np.float32),
                    (S.BUF_LV_MIS, np.float32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_CAMERA_GATHERED, np.float32)):
        a, b = g.buffer(bid, dt), o.buffer(bid, dt)
        assert a.shape == b.shape, f"buffer {bid}: {a.shape} vs {b.shape}"
        same = (a.view(np.uint32) == b.view(np.uint32))
        assert same.all(), f"buffer {bid}: {100.0 * same.mean():.3f}% identical, first mismatch at {int(np.argmin(same))}"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], o.film(S.FILM_LIGHT)[..., :3]) < 1e-6
    g.close()
    f = api.GPUVCM(sd, flavor="fast")
    f.render(2)
    img, ref = f.film(S.FILM_RESULT)[..., :3], o.film(S.FILM_RESULT)[..., :3]
    assert np.isfinite(img).all() and rel_l2(img, ref) < 0.2
    f.close()


def _compare_with_oracle(api, oracle_mod, sd, iterations, opts=None, fast_tolerance=None):
    o = oracle_mod.Oracle(sd)
    if opts is not None:
        o.set_options(opts)
    o.begin(0)
    o.run(iterations, threads=1)
    g = api.GPUVCM(sd, flavor="parity")
    if opts is not None:
        g.options[:] = opts
    g.render(iterations)
    for bid, dt in ((S.BUF_LIGHT_PATH_COUNT, np.uint32), (S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_LV_POS, np.float32), (S.BUF_LV_THROUGHPUT, np.float32),
                    (S.BUF_LV_MIS, np.float32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_CAMERA_GATHERED, np.float32)):
        a, b = g.buffer(bid, dt), o.buffer(bid, dt)
        assert a.shape == b.shape, f"buffer {bid}: {a.shape} vs {b.shape}"
        same = (a.view(np.uint32) == b.view(np.uint32))
        assert same.all(), f"buffer {bid}: {100.0 * same.mean():.3f}% identical, first mismatch at {int(np.argmin(same))}"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], o.film(S.FILM_LIGHT)[..., :3]) < 1e-6
    g.close()
    if fast_tolerance is not None:
        f = api.GPUVCM(sd, flavor="fast")
        if opts is not None:
            f.options[:] = opts
        f.render(iterations)
        img, ref = f.film(S.FILM_RESULT)[..., :3], o.film(S.FILM_RESULT)[..., :3]
        assert np.isfinite(img).all() and rel_l2(img, ref) < fast_tolerance
        f.close()


def test_config4_sss_dragon_is_bit_exact(api, oracle_mod):
    """BASELINE config 4's scene (displaced ~871 k-triangle mesh, plastic + random-walk subsurface, three area emitters) at a small film:
    trace_material / continuous_trace inside a deep BVH, subsurface exits as light and camera vertices."""
    sd = scenes.sss_dragon(40, 40)
    assert sd.triangle_count > 860_000
    _compare_with_oracle(api, oracle_mod, sd, 1, fast_tolerance=0.3)


def test_config5_cloud_is_bit_exact_connect_only(api, oracle_mod):
    """BASELINE config 5: heterogeneous cloud in a Boundary cube under sun + sky, VCM with merging off (= volumetric BDPT),
    delta tracking through a 64^3 grid here (256^3 in the bench workload; the tracker is the same)."""
    sd = scenes.cloud_box(40, 40, grid=64)
    opts = S.default_vcm_options()
    opts["options"] = S.VCM_CONNECT_ONLY
    _compare_with_oracle(api, oracle_mod, sd, 2, opts=opts, fast_tolerance=0.3)


def test_reference_loaded_cornell_asset_is_bit_exact(api, oracle_mod):
    """The Scene / Camera PODs built by the reference's OWN loader from its shipped Cornell asset (fog volume behind a 137k-triangle
    Boundary mesh, sun + sky, conductor box), committed as a byte dump (tests/golden/ref_cornell_40.npz, tools/dump_reference_scene.py;
    tests/test_reference_loader.py checks the dump against the live loader where the reference tree exists), go unchanged into
    etxb_upload_scene and into the oracle."""
    import os
    from conftest import GOLDEN
    from etx_tracer_b200 import pod_io
    sd = pod_io.load(os.path.join(GOLDEN, "ref_cornell_40.npz"))
    assert sd.triangle_count == 138318 and (sd.width, sd.height) == (40, 40)
    # bit-exact for the parity build; the product build of this asset is held to the converged statistical test
    # (test_gpu_statistical.py::test_reference_cornell_asset_product_build), not to a 2-spp image distance
    _compare_with_oracle(api, oracle_mod, sd, 2)


@pytest.mark.parametrize("lanes", [2, 3])
def test_iterations_in_flight_render_the_same_frame(api, lanes):
    """etxb_group: `lanes` contexts render the iteration indices 0..n-1 between them (each index exactly once, whichever lane takes it);
    the combined film is the mean over those iterations, i.e. the single-context frame up to float summation order."""
    sd = scenes.cornell_box(64, 64, samples=16, spectral=True, sphere=True)
    n = 7
    ref = api.GPUVCM(sd, flavor="fast")
    ref.render(n)
    grp = api.GPUVCMGroup(sd, lanes=lanes, flavor="fast")
    st = grp.render(n)
    assert st["completed_iterations"] == n and st["iteration_in_flight"] == 0 and st["overflow"] == 0 and st["total_time"] > 0.0
    assert sum(g.status()["completed_iterations"] for g in grp.lanes) == n
    for layer in (S.FILM_RESULT, S.FILM_CAMERA, S.FILM_LIGHT):
        a, b = grp.film(layer)[..., :3], ref.film(layer)[..., :3]
        assert np.isfinite(a).all() and rel_l2(a, b) < 1e-5, f"layer {layer}: {rel_l2(a, b):.3e}"
    # a second batch continues the same sequence (indices n .. 2n-1)
    grp.enqueue(n)
    grp.wait()
    ref.run(0)
    for _ in range(2 * n):
        ref.iterate()
    ref.wait()
    assert grp.status()["completed_iterations"] == 2 * n
    assert rel_l2(grp.film(S.FILM_RESULT)[..., :3], ref.film(S.FILM_RESULT)[..., :3]) < 1e-5
    grp.close()
    ref.close()


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("kind", scenes.CAMERA_KINDS)
def test_camera_variants_are_bit_exact(api, oracle_mod, kind, spectral):
    """scene_camera.hxx: thin lens with a disk aperture, aperture image sampled through its table, equirectangular camera (which the
    reference's light paths cannot connect to: its sample_film returns nothing)."""
    sd = scenes.camera_box(kind, 32, 32, spectral=spectral)
    # a small merge radius: with the default one the lens' MIS weights push every light-image splat below the driver's
    # dot(val, val) > eps cut (vcm_cpu.cxx:160-166) and the light image would be empty
    opts = S.default_vcm_options()
    opts["initial_radius"] = 0.02
    o = oracle_mod.Oracle(sd)
    o.set_options(opts)
    o.begin(0)
    o.run(2, threads=1)
    g = api.GPUVCM(sd, flavor="parity")
    g.options[:] = opts
    g.render(2)
    if kind != "equirectangular":
        assert o.film(S.FILM_LIGHT)[..., :3].any()
    for bid, dt in ((S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_LV_POS, np.float32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_CAMERA_GATHERED, np.float32)):
        a, b = g.buffer(bid, dt), o.buffer(bid, dt)
        same = (a.view(np.uint32) == b.view(np.uint32))
        assert a.shape == b.shape and same.all(), f"{kind} buffer {bid}: {100.0 * same.mean():.3f}% identical"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    assert rel_l2(g.film(S.FILM_LIGHT)[..., :3], o.film(S.FILM_LIGHT)[..., :3]) < 1e-6
    if kind == "equirectangular":
        assert not g.film(S.FILM_LIGHT)[..., :3].any()
    g.close()
    f = api.GPUVCM(sd, flavor="fast")
    f.options[:] = opts
    f.render(2)
    img, ref = f.film(S.FILM_RESULT)[..., :3], o.film(S.FILM_RESULT)[..., :3]
    assert np.isfinite(img).all() and rel_l2(img, ref) < 0.05
    f.close()


def test_device_closest_hits_against_float64_brute_force_on_the_million_triangle_room(api):
    """The device ray casters against an independent answer: every ray against EVERY triangle of BASELINE config 3's geometry in float64 (no BVH,
    no shared code) — the BVH2 walk the oracle shares, and the 4-wide quantised tree of the product build (dwide.cuh)."""
    sd = scenes.procedural_room(32, 18, env_size=(64, 32))
    import ctypes as C
    sc = sd.scene
    nv, nt = int(sc["vertices"]["count"][0]), int(sc["triangles"]["count"][0])
    verts = np.frombuffer((C.c_char * (nv * S.VERTEX.itemsize)).from_address(int(sc["vertices"]["a"][0])), dtype=S.VERTEX)
    tris = np.frombuffer((C.c_char * (nt * S.TRIANGLE.itemsize)).from_address(int(sc["triangles"]["a"][0])), dtype=S.TRIANGLE)
    pos = verts["pos"].astype(np.float64)
    a, b, c = pos[tris["i"][:, 0]], pos[tris["i"][:, 1]], pos[tris["i"][:, 2]]
    rng = np.random.default_rng(7)
    n = 256
    lo, hi = pos.min(axis=0), pos.max(axis=0)
    origin = lo + (hi - lo) * (0.3 + 0.4 * rng.random((n, 3)))
    direction = rng.normal(size=(n, 3))
    direction /= np.linalg.norm(direction, axis=1, keepdims=True)
    rays = np.zeros((n, 8), dtype=np.float32)
    rays[:, 0:3], rays[:, 3], rays[:, 4:7], rays[:, 7] = origin, 1e-4, direction, 3.0e38
    o64, d64 = rays[:, 0:3].astype(np.float64), rays[:, 4:7].astype(np.float64)
    e1, e2 = b - a, c - a
    best_t = np.full(n, np.inf)
    best_tri = np.full(n, -1, dtype=np.int64)
    for k in range(n):  # Moeller-Trumbore over all triangles, one ray at a time (vectorised over the million triangles)
        pv = np.cross(d64[k], e2)
        det = (e1 * pv).sum(axis=1)
        ok = np.abs(det) > 0
        inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
        tv = o64[k] - a
        u = (tv * pv).sum(axis=1) * inv
        qv = np.cross(tv, e1)
        v = (qv * d64[k]).sum(axis=1) * inv
        t = (qv * e2).sum(axis=1) * inv
        hit = ok & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > 1e-4)
        if hit.any():
            j = np.where(hit, t, np.inf).argmin()
            best_t[k], best_tri[k] = t[j], j
    seeds = np.arange(n, dtype=np.uint32) + 1
    assert (best_tri >= 0).mean() > 0.5  # the room is open to the sky: a quarter of the random rays leave through the windows
    for flavor, wide in (("parity", False), ("fast", False), ("fast", True)):
        g = api.GPUVCM(sd, flavor=flavor)
        assert g.debug_select_tree(wide) or not wide, "the room has stochastic BSDFs: the product build must have built the wide tree"
        uvt, tri, _ = g.debug_trace(rays, seeds)
        g.close()
        found = tri != S.INVALID
        assert np.array_equal(found, best_tri >= 0), (flavor, wide)
        # the same triangle, or (edge / coplanar ties) another one at the same distance
        same = tri[found].astype(np.int64) == best_tri[found]
        np.testing.assert_allclose(uvt[found, 2], best_t[found], rtol=2e-4, atol=1e-5, err_msg=f"{flavor} wide={wide}")
        assert same.mean() > 0.97, (flavor, wide, same.mean())
