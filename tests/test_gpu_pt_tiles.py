"""The path tracer's noise estimate over pixel tiles on one GPU: the test hook etxb_debug_noise_estimate runs it as `world` ranks do (each rank's
view zero outside its tiles, the masks summed as the all-reduce sums them) and must give the one-GPU history; a context with a one-rank
communicator runs the exchange and renders the frame a context without one renders.  Run with -m gpu.  The two-GPU cases are in
test_gpu_multi_pt.py."""
import time

import numpy as np
import pytest

from conftest import bit_equal
import pt_tiles_model as M
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED = -1, -4
EARLY_THRESHOLD = 0.01  # M.left_lit_scene: the lit wall does not converge by iteration 40 at this threshold


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


def _case(w, h, seed):
    """a reachable history (one earlier estimate) and a film for the next one"""
    rng = np.random.default_rng(seed)
    info = rng.integers(32, 64, (h, w)).astype(np.uint32)
    cam, ada = M.random_film(rng, h, w)
    info = M.reference_estimate(cam, ada, info, 0.3)[0]
    cam, ada = M.random_film(rng, h, w)
    return cam, ada, info


FILMS = [(1, 1), (33, 31), (95, 70), (200, 1), (64, 64)]  # W x H


@pytest.mark.parametrize("flavor", ["parity", "fast"])
def test_every_world_gives_the_one_gpu_estimate(api, flavor):
    """For world 2, 3, 5, 8 the composed info words and error levels are bit-equal to world 1, the converged counts equal and the error sums
    within 1e-5 (float atomics in another order).  In the parity build world 1 is the numpy model of the reference's passes, bit for bit."""
    g = api.GPUVCM(flavor=flavor)
    try:
        for k, (w, h) in enumerate(FILMS):
            cam, ada, info = _case(w, h, 100 + k)
            thr = 0.3
            i1, e1, n1, s1 = g.debug_noise_estimate(cam, ada, info, thr, world=1)
            if flavor == "parity":
                want, err_want, n_want, s_want = M.reference_estimate(cam, ada, info, thr)
                assert np.array_equal(i1, want), (w, h)
                assert bit_equal(e1, err_want) and n1 == n_want and s1 == pytest.approx(s_want, rel=1e-5, abs=1e-6)
            if w * h >= 64 * 64:
                conv = (i1 & M.CONVERGED) != 0
                assert 0 < conv.sum() < conv.size, "the case must leave converged and active pixels"
            for world in (2, 3, 5, 8):
                iw, ew, nw, sw = g.debug_noise_estimate(cam, ada, info, thr, world=world)
                assert np.array_equal(iw, i1), (w, h, world)
                assert bit_equal(ew, e1) and nw == n1, (w, h, world)
                assert sw == pytest.approx(s1, rel=1e-5, abs=1e-6), (w, h, world)
    finally:
        g.close()


def _pump(g, timeout=300.0):
    g.run()
    t0 = time.time()
    while g.update():
        assert time.time() - t0 < timeout
        time.sleep(0.001)
    g.wait()
    return g.status()["completed_iterations"]


def _comm_ids(api):
    import torch  # noqa: F401  (loads torch's bundled libnccl, which the module shares)
    try:
        return api.comm_unique_ids(1)
    except api.EtxbError:
        pytest.skip("libnccl cannot be loaded")


TILED_LAYERS = (S.FILM_CAMERA, S.FILM_NORMALS, S.FILM_ALBEDO, S.FILM_CAMERA_ADAPTIVE, S.FILM_RESULT)


def test_one_rank_communicator_renders_the_frame_of_a_plain_context(api):
    """A context with a one-rank communicator runs the exchange after every iteration (the 4-byte pixels_processed, and the mask with the stats
    at every estimate) and must render what a context without one renders: the update loop ends at the same iteration, the history, the error
    levels, every layer etxb_comm_reduce_film reads out and the status are the same."""
    ids = _comm_ids(api)
    sd = scenes.cornell_box(96, 80, samples=48, spectral=False)
    ref = api.GPUPathTracing(sd, flavor="parity")
    g = api.GPUPathTracing(sd, flavor="parity")
    try:
        g.comm_init(1, 0, ids)
        for c in (ref, g):
            c.set_scene_settings(0.25, 0.0)
        n_ref, n = _pump(ref), _pump(g)
        assert n == n_ref
        info = ref.buffer(S.BUF_PIXEL_INFO, np.uint32)
        conv = (info & S.PIXEL_CONVERGED) != 0
        assert 0 < conv.sum() < conv.size, "the case must leave converged and active pixels"
        assert bit_equal(g.buffer(S.BUF_PIXEL_INFO, np.uint32), info)
        assert bit_equal(g.buffer(S.BUF_PIXEL_ERROR, np.float32), ref.buffer(S.BUF_PIXEL_ERROR, np.float32))
        for layer in TILED_LAYERS:
            assert bit_equal(g.comm_reduce_film(layer)[..., :3], ref.film(layer)[..., :3]), layer
        a, b = g.pt_status(), ref.pt_status()
        assert a["pixels_processed"] == b["pixels_processed"] and a["active_pixels"] == b["active_pixels"]
        assert abs(a["noise_level"] - b["noise_level"]) <= 1e-4 * abs(b["noise_level"])
        for layer in (S.FILM_LIGHT_ITERATION, S.FILM_DENOISED, 99):
            with pytest.raises(api.EtxbError) as e:
                g.comm_reduce_film(layer)
            assert e.value.code == ERR_INVALID_ARGUMENT
    finally:
        g.close()
        ref.close()


def test_one_rank_communicator_stops_when_every_pixel_converged(api):
    """The stop rule reads the all-reduced pixels_processed: everything converges at the first estimate (iteration 32) and iteration 33 processes
    nothing, as on a plain context (test_gpu_pt.py)."""
    ids = _comm_ids(api)
    g = api.GPUPathTracing(scenes.cornell_box(24, 24, samples=48, spectral=False), flavor="fast")
    try:
        g.comm_init(1, 0, ids)
        g.set_scene_settings(1e9, 0.0)
        assert _pump(g) == 34
        assert g.pt_status()["pixels_processed"] == 0
    finally:
        g.close()


def test_early_converging_tiles(api):
    """The scene of the two-GPU early-stop case: the pixels of rank 1 of two (no communicator here, so its status counts its own pixels) have
    all converged after the estimate of iteration 32, and its loop ends at 34, while the whole frame goes on."""
    sd = M.left_lit_scene()
    whole = api.GPUPathTracing(sd, flavor="fast")
    part = api.GPUPathTracing(sd, flavor="fast")
    try:
        part.set_partition(1, 2)
        for c in (whole, part):
            c.set_scene_settings(EARLY_THRESHOLD, 0.0)
        assert _pump(part) == 34
        assert _pump(whole) > 40
        own = M.owner_map(96, 32, 2) == 1
        info = part.buffer(S.BUF_PIXEL_INFO, np.uint32).reshape(32, 96)
        assert ((info[own] & S.PIXEL_CONVERGED) != 0).all() and ((info[own] & S.PIXEL_COUNT_MASK) == 33).all()
        assert (info[~own] == 0).all()  # another rank's pixels are left alone
    finally:
        whole.close()
        part.close()


def test_pixel_tiles_without_a_communicator_refuse_the_path_tracer(api):
    g = api.GPUVCM(scenes.cornell_box(32, 32, samples=4), flavor="fast")
    try:
        g.set_partition(0, 2)
        assert g.lib.etxb_set_integrator(g.h, S.INTEGRATOR_PT) == ERR_UNSUPPORTED
        g.set_partition(0, 1)
        assert g.lib.etxb_set_integrator(g.h, S.INTEGRATOR_PT) == 0
    finally:
        g.close()
