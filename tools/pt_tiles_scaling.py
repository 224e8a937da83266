#!/usr/bin/env python
"""The path tracer over pixel tiles on 1 and N GPUs with adaptive sampling on (DESIGN §7): C3 at 1920x1080, spectral, noise threshold 0.1, 256
samples.  Per GPU count: wall time to the end of the run, iterations run, pixel-samples traced (the sum of pixels_processed) per second,
each rank's active pixels over the run, and the device time per estimate of the noise kernels and of the mask exchange.  One JSON line.

usage: pt_tiles_scaling.py [--gpus 1 2 ...] [--scale S] [--samples K] [--compare-root DIR --rounds R]
  --compare-root DIR  also time the noise kernels (film_noise_levels, ms per estimate, one GPU) of the package under DIR (another build of
                      this project, e.g. the parent commit's), alternating R rounds with this one's.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if "--package-root" not in sys.argv:
    sys.path.insert(0, ROOT)
THRESHOLD = 0.1


def _estimates(iterations):
    """iterations that ran Film::estimate_noise_levels (even, from 32 on)"""
    return sum(1 for k in range(iterations) if k >= 32 and k % 2 == 0)


def _render(rank, world, comm_id, args, out_dir):
    import numpy as np
    from etx_tracer_b200 import scenes, structs as S
    from etx_tracer_b200.api import GPUPathTracing
    sd = scenes.config("C3", args.scale)
    sd.scene["samples"] = args.samples
    g = GPUPathTracing(sd, flavor="fast", device=rank, profile=True)
    if comm_id is not None:
        g.comm_init(world, rank, comm_id)
    g.set_scene_settings(THRESHOLD, 0.0)
    g.render(2)  # warm-up: module load, allocations, clocks
    h, w = g.height, g.width
    r, x = np.mgrid[0:h, 0:w]
    own = ((((h - 1 - r) // 32) * ((w + 31) // 32) + x // 32) % world) == rank
    g.run()
    iterations, traced, paused, active = 0, 0, 0.0, []
    t0 = time.perf_counter()
    while True:  # GPUPathTracing.update's stop rule, one iteration at a time
        g.iterate()
        g.wait()
        iterations += 1
        p = g.pt_status()["pixels_processed"]
        traced += p
        if iterations % args.sample_every == 0 or iterations == 1:
            t1 = time.perf_counter()
            info = g.buffer(S.BUF_PIXEL_INFO, np.uint32).reshape(h, w)
            active.append([iterations, int((own & ((info & S.PIXEL_CONVERGED) == 0)).sum())])
            paused += time.perf_counter() - t1
        if p == 0 or iterations >= args.samples:
            break
    wall = time.perf_counter() - t0 - paused
    kt = g.kernel_times()
    est = max(_estimates(iterations), 1)
    res = {"rank": rank, "iterations": iterations, "wall_s": wall, "pixel_samples": traced, "device_s": g.status()["total_time"],
           "active_pixels_of_rank": active,
           "film_noise_levels_ms_per_estimate": kt["film_noise_levels"][0] / est,
           "exchange_ms_per_estimate": kt.get("nccl_allreduce_pt_mask", (0.0, 0))[0] / est,
           "count_exchange_ms_per_iteration": kt.get("nccl_allreduce_pt_count", (0.0, 0))[0] / max(iterations - est, 1)}
    g.close()
    with open(os.path.join(out_dir, f"rank{rank}.json"), "w") as f:
        json.dump(res, f)


def _rank(rank, world, port, args, out_dir):
    import torch
    import torch.distributed as dist
    from etx_tracer_b200.api import comm_unique_ids
    from etx_tracer_b200.multigpu import distribute_comm_ids
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        _render(rank, world, distribute_comm_ids(dist, rank, 1, comm_unique_ids, device=torch.device("cuda", rank)), args, out_dir)
    finally:
        dist.destroy_process_group()


def run_world(world, args):
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as out_dir:
        if world == 1:
            _render(0, 1, None, args, out_dir)
        else:
            with socket.socket() as s:
                s.bind(("127.0.0.1", 0))
                port = s.getsockname()[1]
            mp.spawn(_rank, args=(world, port, args, out_dir), nprocs=world, join=True)
        ranks = [json.load(open(os.path.join(out_dir, f"rank{r}.json"))) for r in range(world)]
    wall = max(r["wall_s"] for r in ranks)
    return {"gpus": world, "iterations": ranks[0]["iterations"], "wall_s": round(wall, 3), "pixel_samples": ranks[0]["pixel_samples"],
            "Mpixel_samples_per_s": round(ranks[0]["pixel_samples"] / wall / 1e6, 2),
            "film_noise_levels_ms_per_estimate": [round(r["film_noise_levels_ms_per_estimate"], 4) for r in ranks],
            "exchange_ms_per_estimate": [round(r["exchange_ms_per_estimate"], 4) for r in ranks],
            "count_exchange_ms_per_iteration": [round(r["count_exchange_ms_per_iteration"], 4) for r in ranks],
            "active_pixels_of_rank": [r["active_pixels_of_rank"] for r in ranks]}


def noise_only(args):
    """film_noise_levels per estimate on one GPU, for the alternation with another build"""
    from etx_tracer_b200 import scenes
    from etx_tracer_b200.api import GPUPathTracing
    sd = scenes.config("C3", args.scale)
    sd.scene["samples"] = args.samples
    g = GPUPathTracing(sd, flavor="fast", profile=True)
    g.set_scene_settings(THRESHOLD, 0.0)
    n = 48
    g.render(n)
    ms = g.kernel_times()["film_noise_levels"][0] / _estimates(n)
    g.close()
    print(json.dumps({"film_noise_levels_ms_per_estimate": ms}))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        return [line.strip() for line in out.splitlines() if line.strip()]
    except (OSError, subprocess.SubprocessError):
        return ["unknown"]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--gpus", type=int, nargs="*", default=None, help="GPU counts to run (default: 1 and every visible device)")
    ap.add_argument("--scale", type=float, default=1.0, help="film scale of C3 (1 = 1920x1080)")
    ap.add_argument("--samples", type=int, default=256)
    ap.add_argument("--sample-every", type=int, default=16, help="iterations between two reads of the ranks' active pixels")
    ap.add_argument("--compare-root", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--package-root", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--noise-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.package_root:
        sys.path.insert(0, args.package_root)
    if args.noise_only:
        return noise_only(args)
    import torch
    visible = torch.cuda.device_count()
    counts = args.gpus or sorted({1, visible})
    out = {"workload": "C3 path tracer, pixel tiles", "threshold": THRESHOLD, "samples": args.samples, "scale": args.scale, "cards": _card(),
           "runs": []}
    for world in counts:
        if world > visible:
            out["runs"].append({"gpus": world, "skipped": f"{visible} device(s) visible"})
            continue
        out["runs"].append(run_world(world, args))
    if args.compare_root:
        me = [sys.executable, os.path.abspath(__file__), "--noise-only", "--scale", str(args.scale), "--samples", str(args.samples)]
        times = {"this": [], "compare": []}
        for _ in range(args.rounds):
            for key, root in (("this", ROOT), ("compare", os.path.abspath(args.compare_root))):
                r = subprocess.run(me + ["--package-root", root], capture_output=True, text=True, check=True)
                times[key].append(round(json.loads(r.stdout.strip().splitlines()[-1])["film_noise_levels_ms_per_estimate"], 4))
        out["film_noise_levels_alternated"] = times
    print(json.dumps(out))


if __name__ == "__main__":
    main()
