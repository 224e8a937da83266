"""What the coarse preview buys while the camera moves: C3 (procedural_room, 1920x1080, spectral), VCM and the path tracer, film pixel size
1, 2, 4 and 8.

For each (integrator, size) it reports
  * the median iteration time with one iteration in flight, each enqueue ended by the module's device synchronise (etxb_wait);
  * the median time from an etxb_update_scene camera move (the camera alternates between two poses) to the end of the first completed
    preview iteration after it.
Prints the card and its power limit next to the numbers, and one JSON line.

    python tools/preview_latency.py [--reps 7] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from etx_tracer_b200 import api, scenes  # noqa: E402

SIZES = (1, 2, 4, 8)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi found no GPU: this measurement runs on the device only")
    return q.stdout.strip().splitlines()[0]


def poses():
    """C3 and its camera in two poses (the camera array is edited in place, as the application edits its Camera POD)"""
    sd = scenes.config("C3")
    cam = sd.camera.copy()
    sd.set_camera([0.3, 1.65, 3.7], [0.0, 1.0, 0.0], [0.0, 1.0, 0.0], sd.width, sd.height, 55.0, clip_near=0.1, clip_far=100.0)
    moved = sd.camera.copy()
    sd.camera[:] = cam
    return sd, (cam, moved)


def measure(cls, sd, cams, size, reps):
    sd.camera[:] = cams[0]
    g = cls(sd, flavor="fast")
    g.set_film_pixel_size(size)
    g.run(0)
    for _ in range(2):  # warm-up: module load, first launches, allocations
        g.iterate()
        g.wait()
    iteration = []
    for _ in range(reps):
        t0 = time.perf_counter()
        g.iterate()
        g.wait()
        iteration.append(time.perf_counter() - t0)
    move = []
    for k in range(reps):
        t0 = time.perf_counter()
        sd.camera[:] = cams[(k + 1) % 2]
        g.update_scene(sd)
        g.iterate()
        g.wait()
        move.append(time.perf_counter() - t0)
    g.close()
    return statistics.median(iteration) * 1e3, statistics.median(move) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card_line = card()
    sd, cams = poses()
    print(f"card: {card_line}  (name, power limit, max SM clock)", flush=True)
    rows = []
    for name, cls in (("vcm", api.GPUVCM), ("pt", api.GPUPathTracing)):
        for size in SIZES:
            it_ms, move_ms = measure(cls, sd, cams, size, args.reps)
            rows.append({"integrator": name, "pixel_size": size, "paths": ((1920 + size - 1) // size) * ((1080 + size - 1) // size),
                         "iteration_ms": round(it_ms, 2), "move_to_first_iteration_ms": round(move_ms, 2)})
            print(f"{name:4s} s={size}: iteration {it_ms:8.2f} ms   camera move -> first iteration {move_ms:8.2f} ms", flush=True)
    result = {"card": card_line, "workload": "C3 1920x1080 spectral", "rows": rows}
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
