"""The path tracer over pixel tiles on two GPUs, one process each, with adaptive sampling on: the noise estimate's mask exchanged inside the
module (etxb_comm_init), against one GPU rendering the whole frame.  Run with -m gpu on a box with at least two devices; skipped on one."""
import os
import socket
import sys
import time

import numpy as np
import pytest

import pt_tiles_model as M
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

LAYERS = {"camera": S.FILM_CAMERA, "normals": S.FILM_NORMALS, "albedo": S.FILM_ALBEDO, "adaptive": S.FILM_CAMERA_ADAPTIVE}
PARITY_THRESHOLD = 0.25  # Cornell 96 x 80 (RGB): part of the film converges at the estimates from iteration 32 on, part does not by 48
EARLY_THRESHOLD = 0.01   # M.left_lit_scene: rank 1's tiles converge at iteration 32, the lit wall on rank 0 does not by iteration 40


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _case(name):
    if name == "early":
        return M.left_lit_scene(), EARLY_THRESHOLD, "fast"
    return scenes.cornell_box(96, 80, samples=48, spectral=False), PARITY_THRESHOLD, name


def _pump(g, timeout=600.0):
    g.run()
    t0 = time.time()
    while g.update():
        assert time.time() - t0 < timeout
        time.sleep(0.001)
    g.wait()
    return g.status()["completed_iterations"]


def _worker(rank, world, port, out_dir, name):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch
    import torch.distributed as dist
    from etx_tracer_b200 import api
    from etx_tracer_b200.multigpu import distribute_comm_ids
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        ids = lambda c: distribute_comm_ids(dist, rank, c, lambda k: api.comm_unique_ids(k), device=torch.device("cuda", rank))  # noqa: E731
        if name == "group":
            # a group in pixel-tile mode keeps one history per lane: refused alike on both ranks, before any collective
            g = api.GPUVCMGroup(scenes.cornell_box(32, 32, samples=4), lanes=2, flavor="fast", device=rank)
            g.comm_init(world, rank, ids(3))
            with pytest.raises(api.EtxbError) as e:
                g.set_integrator(S.INTEGRATOR_PT)
            np.savez(os.path.join(out_dir, f"rank{rank}.npz"), code=np.int32(e.value.code))
            g.close()
            return
        sd, thr, flavor = _case(name)
        g = api.GPUPathTracing(sd, flavor=flavor, device=rank)
        g.comm_init(world, rank, ids(1))
        g.set_scene_settings(thr, 0.0)
        n = _pump(g)
        st = g.pt_status()
        out = dict(iterations=np.int32(n), pixels_processed=np.uint32(st["pixels_processed"]), active_pixels=np.uint32(st["active_pixels"]),
                   noise_level=np.float32(st["noise_level"]), info=g.buffer(S.BUF_PIXEL_INFO, np.uint32), error=g.buffer(S.BUF_PIXEL_ERROR, np.float32))
        for key, layer in LAYERS.items():
            film = g.comm_reduce_film(layer)
            if rank == 0:
                out[key] = film
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
        g.close()
    finally:
        dist.destroy_process_group()


def _spawn(tmp_path, name):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path), name), nprocs=2, join=True)
    return [dict(np.load(tmp_path / f"rank{r}.npz")) for r in range(2)]


def _one_gpu(name):
    from etx_tracer_b200 import api
    sd, thr, flavor = _case(name)
    g = api.GPUPathTracing(sd, flavor=flavor)
    g.set_scene_settings(thr, 0.0)
    n = _pump(g)
    out = dict(iterations=n, status=g.pt_status(), info=g.buffer(S.BUF_PIXEL_INFO, np.uint32), error=g.buffer(S.BUF_PIXEL_ERROR, np.float32),
               width=g.width, height=g.height)
    for key, layer in LAYERS.items():
        out[key] = g.film(layer)
    g.close()
    return out


@pytest.mark.parametrize("name", ["parity", "fast", "early"])
def test_two_gpu_path_tracer_tiles_render_the_single_gpu_frame(tmp_path, name):
    """parity / fast: Cornell 96 x 80 (partial tiles in y) with adaptive sampling; early: a frame whose rank-1 tiles all converge at the first
    estimate, so rank 1 traces no path from iteration 33 on and still joins every collective.  In each, both ranks end their update loops at the
    one-GPU iteration and report its status; rank 0's reduced layers, and each rank's own pixels' history and error levels, are the one-GPU ones.
    The product build is held to the same equality: a path's arithmetic does not depend on which other paths run, and a path-tracer iteration
    has no stage that couples pixels."""
    ranks = _spawn(tmp_path, name)
    ref = _one_gpu(name)
    w, h = ref["width"], ref["height"]
    conv = (ref["info"] & S.PIXEL_CONVERGED) != 0
    assert 0 < conv.sum() < conv.size, "the case must leave converged and active pixels"
    if name == "early":
        assert ref["iterations"] > 40
    own = M.owner_map(w, h, 2).ravel()
    info, error = np.zeros_like(ref["info"]), np.zeros_like(ref["error"])
    for r, got in enumerate(ranks):
        assert int(got["iterations"]) == ref["iterations"], (r, int(got["iterations"]), ref["iterations"])
        assert int(got["pixels_processed"]) == ref["status"]["pixels_processed"]
        assert int(got["active_pixels"]) == ref["status"]["active_pixels"]
        assert abs(float(got["noise_level"]) - ref["status"]["noise_level"]) <= 1e-4 * abs(ref["status"]["noise_level"])
        info[own == r], error[own == r] = got["info"][own == r], got["error"][own == r]
    assert np.array_equal(info, ref["info"])
    assert np.array_equal(error.view(np.uint32), ref["error"].view(np.uint32))
    if name == "early":
        mine = own == 1
        assert ((info[mine] & S.PIXEL_COUNT_MASK) == 33).all()
    for key in LAYERS:
        # the ranks' tiles are disjoint and zero elsewhere, so the sum is exact (equal as floats: a -0 component may come back as +0)
        a, b = ranks[0][key][..., :3], ref[key][..., :3]
        assert np.array_equal(a, b), (key, float(np.abs(a - b).max()))


def test_two_gpu_tile_group_refuses_the_path_tracer(tmp_path):
    ranks = _spawn(tmp_path, "group")
    assert [int(r["code"]) for r in ranks] == [-4, -4]


@pytest.mark.parametrize("integrator", ["pt", "vcm"])
def test_render_on_two_gpus_writes_the_one_gpu_exr(tmp_path, integrator):
    """python -m etx_tracer_b200.render --gpus 2 (one process per GPU, rank 0 writes) against --gpus 1 on the same scene file: the path tracer with
    adaptive sampling writes the same EXR; the VCM's photon records arrive rank-major and are merged in another order (test_gpu_multi.py)."""
    import torch
    from etx_tracer_b200 import loader, render
    from test_host_cpp import _tiny_scene
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    scene = _tiny_scene(tmp_path)
    args = ["--integrator", integrator, "--spp", "40"] + (["--noise-threshold", "0.2"] if integrator == "pt" else [])
    one, two = str(tmp_path / "one.exr"), str(tmp_path / "two.exr")
    assert render.main([scene, "-o", one] + args) == 0
    assert render.main([scene, "-o", two, "--gpus", "2"] + args) == 0
    a, b = loader.read_image(two)[0][..., :3], loader.read_image(one)[0][..., :3]
    assert a.shape == b.shape and b.mean() > 1e-3
    if integrator == "pt":
        assert np.array_equal(a, b)
    else:
        assert float(np.sqrt(((a - b) ** 2).sum()) / np.sqrt((b ** 2).sum())) < 2e-3
