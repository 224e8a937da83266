"""Time to a committed tree: the host builder (csrc/bvh_build.cpp) against the device builder (csrc/bvh_build_device.cu), on C3, C4 and
procedural_room(target_triangles=8_000_000).

Per scene: both trees built by each builder through etxb_debug_build_trees (host: build_bvh + build_wide_bvh on one thread; device: the same
trees on the GPU, inputs already resident), the etxb_upload_scene call (ending with the module's device synchronise), and etxb_update_scene
after one moved vertex (two states alternate, so every call rebuilds).  Medians of --reps runs after one warm-up.  The device trees are
checked equal to the host trees byte for byte on every scene.  C3 and C4 render at a quarter of their film size (their geometry is
the config's).  Prints the card, its power limit and one JSON line.

    python tools/bvh_build_latency.py [--reps 5] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from etx_tracer_b200 import api, scenes  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi found no GPU: this measurement runs on the device only")
    return q.stdout.strip().splitlines()[0]


def median_ms(values):
    return round(statistics.median(values) * 1e3, 2)


def measure(name, sd, reps):
    pos = sd.a_vertices["pos"].astype(np.float32)
    idx = sd.a_triangles["i"].astype(np.uint32)
    g = api.GPUVCM(None, flavor="fast")
    host = g.debug_build_trees(pos, idx, device=False)
    dev = g.debug_build_trees(pos, idx, device=True)
    same = all(host[k].tobytes() == dev[k].tobytes() for k in ("bvh_nodes", "tri_pos", "tri_index", "wide_nodes")) and \
        host["max_depth"] == dev["max_depth"] and host["max_stack"] == dev["max_stack"]
    host_s = [g.debug_build_trees(pos, idx, device=False)["seconds"] for _ in range(reps)]
    dev_s = [g.debug_build_trees(pos, idx, device=True)["seconds"] for _ in range(reps)]
    g.close()

    g = api.GPUVCM(None, flavor="fast")
    g.set_scene(sd)  # warm-up
    upload_s = []
    for _ in range(reps):
        t0 = time.perf_counter()
        g.set_scene(sd)
        upload_s.append(time.perf_counter() - t0)
    v0 = sd.a_vertices["pos"][0].copy()
    update_s, bvh_s = [], []
    for k in range(reps + 1):
        sd.a_vertices["pos"][0] = v0 + np.float32(1e-3 * ((k % 2) + 1))
        t0 = time.perf_counter()
        info = g.update_scene(sd)
        if k:
            update_s.append(time.perf_counter() - t0)
            bvh_s.append(info["bvh_seconds"])
    sd.a_vertices["pos"][0] = v0
    g.close()
    r = {"scene": name, "triangles": int(idx.shape[0]), "trees_equal": bool(same), "bvh_nodes": int(host["bvh_nodes"].shape[0]),
         "wide_nodes": int(host["wide_nodes"].shape[0]), "host_build_ms": median_ms(host_s), "device_build_ms": median_ms(dev_s),
         "upload_ms": median_ms(upload_s), "update_after_vertex_move_ms": median_ms(update_s), "update_bvh_ms": median_ms(bvh_s)}
    print(r, flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card_line = card()
    results = []
    for name, make in (("C3", lambda: scenes.config("C3", scale=0.25)), ("C4", lambda: scenes.config("C4", scale=0.25)),
                       ("room_8M", lambda: scenes.procedural_room(480, 270, samples=16, target_triangles=8_000_000))):
        t0 = time.perf_counter()
        sd = make()
        print(f"{name} generated in {time.perf_counter() - t0:.1f} s", flush=True)
        results.append(measure(name, sd, args.reps))
    out = {"card": card_line, "reps": args.reps, "results": results}
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
