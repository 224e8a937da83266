"""Host latency of a restart after a scene edit on C3 (procedural_room, 1920x1080, spectral): etxb_upload_scene against etxb_update_scene.

For the upload and for each edit kind (camera only; a material parameter within its class; every non-Lambert material flipped to Lambert
and back, each direction on its own; film 1920x1080 <-> 1280x720) it times five calls, each ending with the module's device synchronise, and the time from the call
to the end of the first iteration rendered after it.  The edits alternate between two states, so every call sees a real change, the way
the application edits its Scene / Camera PODs in place.  Prints the card, its power limit, the medians, the bytes the module
hashed (etxb_update_info) and one JSON line.

    python tools/scene_update_latency.py [--reps 5] [--out result.json]
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
from etx_tracer_b200 import api, scenes, structs as S  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi found no GPU: this measurement runs on the device only")
    return q.stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card_line = card()
    t0 = time.perf_counter()
    sd = scenes.config("C3")
    print(f"C3 generated in {time.perf_counter() - t0:.1f} s: {sd.triangle_count} triangles, {sd.width}x{sd.height}", flush=True)
    g = api.GPUVCM(sd, flavor="fast")
    g.render(1)  # warm: module load, first launches

    def first_iteration():
        g.iterate()
        g.wait()

    results = {}

    def measure(name, call, prepare=None):
        calls, firsts, infos = [], [], []
        for r in range(args.reps):
            if prepare:
                prepare(r)  # untimed: back to the state the timed call changes
                first_iteration()
            t = time.perf_counter()
            info = call(r)
            t_call = time.perf_counter() - t
            first_iteration()
            firsts.append(time.perf_counter() - t)
            calls.append(t_call)
            if info:
                infos.append(info)
        row = {"call_s": statistics.median(calls), "to_first_iteration_s": statistics.median(firsts)}
        if infos:
            row["fingerprint_s"] = statistics.median(i["fingerprint_seconds"] for i in infos)
            row["bvh_s"] = statistics.median(i["bvh_seconds"] for i in infos)
            row["kept"] = sorted({i["kept"] for i in infos})
            row["bytes_hashed"] = infos[0]["bytes_hashed"]
        results[name] = row
        print(f"{name:24s} call {row['call_s'] * 1e3:9.1f} ms   to first iteration {row['to_first_iteration_s'] * 1e3:9.1f} ms"
              + (f"   hashing {row['fingerprint_s'] * 1e3:7.1f} ms   trees {row['bvh_s'] * 1e3:7.1f} ms   kept {row['kept']}" if infos else ""), flush=True)

    measure("upload", lambda r: g.set_scene(sd))

    cam = sd.camera.copy()
    moved = sd.camera.copy()
    sd.set_camera([0.3, 1.65, 3.7], [0.0, 1.0, 0.0], [0.0, 1.0, 0.0], sd.width, sd.height, 55.0, clip_near=0.1, clip_far=100.0)
    moved[:] = sd.camera
    sd.camera[:] = cam

    def camera(r):
        sd.camera[:] = moved if r % 2 == 0 else cam
        return g.update_scene(sd)
    measure("update: camera", camera)
    sd.camera[:] = cam

    plastic = sd.material_names["plastic"]
    rough = sd.a_materials[plastic]["roughness"]["value"].copy()

    def material(r):
        sd.a_materials[plastic]["roughness"]["value"][:2] = np.float32(0.35 if r % 2 == 0 else rough[0])
        return g.update_scene(sd)
    measure("update: material", material)
    sd.a_materials[plastic]["roughness"]["value"] = rough

    original = sd.a_materials.copy()
    lambert = sd.a_materials.copy()
    diffuse = sd.material_names["diffuse"]
    for name in ("plastic", "gold", "plastic_film"):
        lambert[sd.material_names[name]] = original[diffuse]

    def flip_to(target, before):
        def prepare(r):
            sd.a_materials[:] = before
            g.update_scene(sd)

        def call(r):
            sd.a_materials[:] = target
            return g.update_scene(sd)
        return call, prepare
    measure("update: flip to Lambert", *flip_to(lambert, original))
    measure("update: flip to plastic", *flip_to(original, lambert))  # the 4-wide tree is collapsed again from the device's BVH2

    def film(r):
        w, h = (1280, 720) if r % 2 == 0 else (1920, 1080)
        sd.set_camera([0.0, 1.6, 3.8], [0.0, 1.0, 0.0], [0.0, 1.0, 0.0], w, h, 55.0, clip_near=0.1, clip_far=100.0)
        return g.update_scene(sd)
    measure("update: film size", film)
    g.close()

    out = {"card": card_line, "scene": "C3", "triangles": sd.triangle_count, "reps": args.reps, "medians": results}
    print(f"card: {card_line}   bytes hashed per call (etxb_update_info): {results['update: camera']['bytes_hashed'] / 2**20:.1f} MiB")
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
