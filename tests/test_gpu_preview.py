"""The coarse preview (etxb_set_film_pixel_size): at pixel size s both integrators trace one path per s x s block and the film repeats its value
over the block.  Parity build bit-exact against the oracle's restated Film (sampler end states, light paths, vertex pool, camera film, the path
tracer's layers and per-pixel history; the light image within 1e-6 relative L2: float-atomic order); the application's flow (move at 8, release
at 1) through etxb_update_scene; no state left behind by a size change; groups; refusals; the product build against the oracle.  Run with -m gpu.
"""
import numpy as np
import pytest

from conftest import bit_equal, rel_l2
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

PATH_BUFFERS = ((S.BUF_LIGHT_SAMPLER, np.uint32), (S.BUF_CAMERA_SAMPLER, np.uint32), (S.BUF_LIGHT_PATH_COUNT, np.uint32),
                (S.BUF_LIGHT_PATH_OFFSET, np.uint32), (S.BUF_CAMERA_GATHERED, np.float32))
POOL_BUFFERS = ((S.BUF_LV_POS, np.float32), (S.BUF_LV_THROUGHPUT, np.float32), (S.BUF_LV_MIS, np.float32))
PT_LAYERS = (S.FILM_CAMERA, S.FILM_NORMALS, S.FILM_ALBEDO, S.FILM_CAMERA_ADAPTIVE)


@pytest.fixture(scope="module")
def preview_oracle():
    """the parity oracle with the Film pixel size (oracle/oracle_preview.cxx)"""
    from oracle import oracle_preview_py
    if not oracle_preview_py.available():
        pytest.skip("oracle/_ref/liboracle_preview_parity.so not built (run build() where /root/reference exists)")
    return oracle_preview_py


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


def _folds(w, h, s):
    """per film pixel (storage order), how many clamped positions of its block's light splat land on it"""
    rows, cols = np.mgrid[0:h, 0:w]
    y = h - 1 - rows
    mx = np.where(cols == w - 1, (cols // s) * s + s - cols, 1)
    my = np.where(y == h - 1, (y // s) * s + s - y, 1)
    return mx * my


def _paths(w, h, s):
    return ((w + s - 1) // s) * ((h + s - 1) // s)


def _cornell(w, h, spectral):
    return scenes.cornell_box(w, h, samples=64, spectral=spectral, sphere=spectral)


def _oracle(preview_oracle, sd, size, iterations, pt=False, opts=None, noise_threshold=None):
    o = preview_oracle.Oracle(sd)
    if pt:
        o.set_integrator(S.INTEGRATOR_PT)
        o.pt_set_options(S.default_pt_options())
        if noise_threshold is not None:
            o.set_scene_settings(noise_threshold)
    elif opts is not None:
        o.set_options(opts)
    o.set_film_pixel_size(size)
    o.begin(0)
    o.run(iterations, threads=1)
    return o


def _device(api, sd, size, iterations, flavor="parity", pt=False, opts=None, noise_threshold=None):
    g = api.GPUPathTracing(sd, flavor=flavor) if pt else api.GPUVCM(sd, flavor=flavor)
    if noise_threshold is not None:
        g.set_scene_settings(noise_threshold)
    if opts is not None:
        g.options[:] = opts
    g.set_film_pixel_size(size)
    g.size = size
    g.render(iterations)
    return g


def _assert_vcm_equal(g, o, n_paths):
    for bid, dt in PATH_BUFFERS:
        a, b = g.buffer(bid, dt), o.buffer(bid, dt)
        k = n_paths * (3 if bid == S.BUF_CAMERA_GATHERED else 1)
        assert b.size == k and bit_equal(a[:k], b), f"buffer {bid}"
    for bid, dt in POOL_BUFFERS:
        assert bit_equal(g.buffer(bid, dt), o.buffer(bid, dt)), f"buffer {bid}"
    assert bit_equal(g.film(S.FILM_CAMERA)[..., :3], o.film(S.FILM_CAMERA)[..., :3])
    ref, img = o.film(S.FILM_LIGHT)[..., :3], g.film(S.FILM_LIGHT)[..., :3]
    if not ref.any():
        assert not img.any()
        return
    # float-atomic order; where the last column / row of a partial block folds k clamped positions onto one pixel the reference adds each
    # splat k times and the device multiplies the cell's sum by k once: rounding that grows with k
    fold = _folds(g.width, g.height, g.size)
    assert rel_l2(img[fold == 1], ref[fold == 1]) < 1e-6
    if (fold > 1).any():
        assert rel_l2(img[fold > 1], ref[fold > 1]) < 1e-6 * float(fold.max())


def _assert_pt_equal(g, o, n_paths):
    for bid in (S.BUF_CAMERA_SAMPLER,):
        a, b = g.buffer(bid, np.uint32), o.buffer(bid, np.uint32)
        assert b.size == n_paths and bit_equal(a[:n_paths], b)
    for layer in PT_LAYERS:
        assert bit_equal(g.film(layer)[..., :3], o.film(layer)[..., :3]), f"layer {layer}"
    assert bit_equal(g.buffer(S.BUF_PIXEL_INFO, np.uint32), o.buffer(S.BUF_PIXEL_INFO, np.uint32))


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("size", [2, 3, 8, 1024])
def test_parity_vcm_preview_is_bit_exact(api, preview_oracle, size, spectral):
    sd = _cornell(26, 19, spectral)
    o = _oracle(preview_oracle, sd, size, 3)
    g = _device(api, sd, size, 3)
    _assert_vcm_equal(g, o, _paths(26, 19, size))
    g.close()


@pytest.mark.parametrize("spectral", [False, True])
@pytest.mark.parametrize("size", [2, 3, 8, 1024])
def test_parity_path_tracer_preview_is_bit_exact(api, preview_oracle, size, spectral):
    sd = _cornell(26, 19, spectral)
    o = _oracle(preview_oracle, sd, size, 3, pt=True)
    g = _device(api, sd, size, 3, pt=True)
    _assert_pt_equal(g, o, _paths(26, 19, size))
    g.close()


@pytest.mark.parametrize("kind", scenes.CAMERA_KINDS)
def test_parity_preview_camera_variants(api, preview_oracle, kind):
    sd = scenes.camera_box(kind, 30, 22, spectral=True)
    opts = S.default_vcm_options()
    opts["initial_radius"] = 0.02
    o = _oracle(preview_oracle, sd, 3, 2, opts=opts)
    g = _device(api, sd, 3, 2, opts=opts)
    _assert_vcm_equal(g, o, _paths(30, 22, 3))
    g.close()
    o = _oracle(preview_oracle, sd, 3, 2, pt=True)
    g = _device(api, sd, 3, 2, pt=True)
    _assert_pt_equal(g, o, _paths(30, 22, 3))
    g.close()


def test_parity_preview_environment_with_blue_noise(api, preview_oracle):
    """blue noise reads the pixel a path chose (its first bounce), not the path index"""
    sd = scenes.sky_room(30, 22)
    o = _oracle(preview_oracle, sd, 4, 2)
    g = _device(api, sd, 4, 2)
    _assert_vcm_equal(g, o, _paths(30, 22, 4))
    g.close()
    o = _oracle(preview_oracle, sd, 4, 2, pt=True)
    g = _device(api, sd, 4, 2, pt=True)
    _assert_pt_equal(g, o, _paths(30, 22, 4))
    g.close()


def test_parity_path_tracer_preview_with_adaptive_sampling(api, preview_oracle):
    """44 iterations at s = 2 with a noise threshold: converged pixels skip their blocks' paths, the per-pixel counts diverge"""
    sd = _cornell(26, 19, False)
    o = _oracle(preview_oracle, sd, 2, 44, pt=True, noise_threshold=0.2)
    g = _device(api, sd, 2, 44, pt=True, noise_threshold=0.2)
    info = o.buffer(S.BUF_PIXEL_INFO, np.uint32)
    counts = info & 0x3fffffff
    assert (info & (1 << 30)).any() and counts.min() < counts.max(), "the threshold should converge some pixels"
    _assert_pt_equal(g, o, _paths(26, 19, 2))
    assert bit_equal(g.buffer(S.BUF_PIXEL_ERROR, np.float32), o.buffer(S.BUF_PIXEL_ERROR, np.float32))
    g.close()


def _state(g, pt):
    layers = PT_LAYERS if pt else (S.FILM_CAMERA, S.FILM_LIGHT)
    out = {f"layer{k}": g.film(k)[..., :3] for k in layers}
    out["sampler"] = g.buffer(S.BUF_CAMERA_SAMPLER, np.uint32)
    if pt:
        out["info"] = g.buffer(S.BUF_PIXEL_INFO, np.uint32)
    return out


def _assert_same_state(a, b, pt):
    sa, sb = _state(a, pt), _state(b, pt)
    for key in sa:
        if key == f"layer{S.FILM_LIGHT}":
            assert rel_l2(sa[key], sb[key]) < 1e-6, key
        else:
            assert bit_equal(sa[key], sb[key]), key


@pytest.mark.parametrize("pt", [False, True])
def test_no_state_left_behind_by_a_size_change(api, pt):
    sd = _cornell(26, 19, True)
    a = _device(api, sd, 8, 2, pt=pt)
    a.set_film_pixel_size(1)
    a.render(2)
    b = _device(api, sd, 1, 2, pt=pt)
    _assert_same_state(a, b, pt)
    a.close()
    b.close()


def _moved(sd0):
    sd = scenes.cornell_box(26, 19, samples=64, spectral=True, sphere=True, finalize=False)
    sd.set_camera([0.2, 1.1, 3.6], [0.0, 0.9, -6.18], [0.0, 1.0, 0.0], sd.width, sd.height, 39.597755335771296, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=64, spectral=True)


@pytest.mark.parametrize("flavor", ["parity", "fast"])
@pytest.mark.parametrize("pt", [False, True])
def test_application_flow_move_at_8_release_at_1(api, pt, flavor):
    """RTApplication::frame: set_pixel_size(8) + restart while the camera moves, set_pixel_size(1) + restart when it stops"""
    s1 = _cornell(26, 19, True)
    s2 = _moved(s1)
    a = _device(api, s1, 1, 2, flavor=flavor, pt=pt)
    a.set_film_pixel_size(8)
    a.update_scene(s2)
    for _ in range(2):
        a.iterate()
    a.wait()
    b = _device(api, s2, 8, 2, flavor=flavor, pt=pt)
    _assert_same_state(a, b, pt)
    a.set_film_pixel_size(1)
    a.update_scene(s2)
    for _ in range(2):
        a.iterate()
    a.wait()
    b.close()
    b = _device(api, s2, 1, 2, flavor=flavor, pt=pt)
    _assert_same_state(a, b, pt)
    a.close()
    b.close()


def test_group_of_two_lanes_at_8_matches_one_context(api):
    sd = _cornell(26, 19, True)
    grp = api.GPUVCMGroup(sd, lanes=2, flavor="parity")
    grp.set_film_pixel_size(8)
    grp.render(4)
    one = _device(api, sd, 8, 4)
    for layer in (S.FILM_CAMERA, S.FILM_LIGHT):
        assert rel_l2(grp.film(layer)[..., :3], one.film(layer)[..., :3]) < 1e-5, layer
    grp.close()
    one.close()


def test_refusals(api):
    from etx_tracer_b200.api import EtxbError
    sd = _cornell(16, 16, False)
    g = api.GPUVCM(sd, flavor="parity")
    lib, h = g.lib, g.h
    assert lib.etxb_set_partition(h, 0, 2) == 0
    assert lib.etxb_set_film_pixel_size(h, 8) == -4
    assert lib.etxb_set_film_pixel_size(h, 1) == 0
    assert lib.etxb_set_partition(h, 0, 1) == 0
    assert lib.etxb_set_film_pixel_size(h, 8) == 0
    assert lib.etxb_set_partition(h, 0, 2) == -4
    with pytest.raises(EtxbError) as e:
        g.comm_init(1, 0, api.comm_unique_ids(1, flavor="parity"))
    assert e.value.code == -4
    g.close()
    grp = api.GPUVCMGroup(sd, lanes=2, flavor="parity")
    grp.set_film_pixel_size(4)
    with pytest.raises(EtxbError) as e:
        grp.comm_init_replicas(1, 0, api.comm_unique_ids(1, flavor="parity"))
    assert e.value.code == -4
    grp.close()


def _tier_c(img, ref_a, ref_b):
    """DESIGN §3 Tier C: the render's relative MSE against an oracle render within 2x the oracle's own run-to-run relative MSE"""
    def rel_mse(x, y):
        return float(((x.astype(np.float64) - y) ** 2).sum() / max((y.astype(np.float64) ** 2).sum(), 1e-30))
    spread = rel_mse(ref_a, ref_b)
    return rel_mse(img, ref_a), spread


def test_product_build_is_deterministic_and_meets_tier_c(api, preview_oracle):
    for sd, size in ((_cornell(32, 24, True), 2), (_cornell(32, 24, True), 8), (scenes.procedural_room(32, 18, env_size=(64, 32)), 2),
                     (scenes.procedural_room(32, 18, env_size=(64, 32)), 8)):
        opts = S.default_vcm_options()
        opts["initial_radius"] = 0.05
        opts["radius_decay"] = 1 << 30  # a constant radius: the two oracle windows estimate the same image
        n = 64
        a = _device(api, sd, size, n, flavor="fast", opts=opts)
        b = _device(api, sd, size, n, flavor="fast", opts=opts)
        # what does not depend on float-atomic order is bit-exact (the product build adds unoccluded shadow-ray contributions atomically)
        for bid in (S.BUF_LIGHT_SAMPLER, S.BUF_CAMERA_SAMPLER, S.BUF_LIGHT_PATH_COUNT):
            assert bit_equal(a.buffer(bid, np.uint32), b.buffer(bid, np.uint32)), bid
        assert rel_l2(a.film(S.FILM_CAMERA)[..., :3], b.film(S.FILM_CAMERA)[..., :3]) < 1e-5
        # the camera layer: its running mean counts each pixel's own samples, so a window that starts at iteration n is a plain mean too
        img = a.film(S.FILM_CAMERA)[..., :3]
        o1 = _oracle(preview_oracle, sd, size, n, opts=opts)
        r1 = o1.film(S.FILM_CAMERA)[..., :3]
        o2 = preview_oracle.Oracle(sd)
        o2.set_options(opts)
        o2.set_film_pixel_size(size)
        o2.begin(n)
        o2.run(n, threads=8)
        r2 = o2.film(S.FILM_CAMERA)[..., :3]
        err, spread = _tier_c(img, r1, r2)
        assert err < 2.0 * spread, (size, err, spread)
        a.close()
        b.close()
