"""Error against device time for the VCM and the path tracer (product build) on one workload: how far each render is from a converged image
after every k iterations.

The reference is a file (--reference) or a long path-tracer render over a disjoint iteration range (first_iteration = 2^24): samples seed
from (pixel, iteration), so that range shares no sample with the measured runs, which start at iteration 0.  Each measured run renders
--iterations iterations one at a time and, every --every of them, reads etxb_film_error (it waits for the iteration in flight) and prints one
JSON line: integrator, iteration, device seconds, and the error fields.  A last line gives the card, its power limit and the CUDA-event medians
of etxb_read_film_view (8-bit tone-mapped view) and etxb_film_error at the workload's size, read in the same run.

    python tools/convergence.py [--workload C3] [--iterations 64] [--every 4] [--reference-iterations 1024] [--reference ref.exr] [--out f.jsonl]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from etx_tracer_b200 import api, scenes, structs as S  # noqa: E402

REFERENCE_FIRST_ITERATION = 1 << 24


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi found no GPU: this measurement runs on the device only")
    return q.stdout.strip().splitlines()[0]


def curve(cls, name, sd, reference, iterations, every, emit):
    g = cls(sd, flavor="fast")
    try:
        g.set_reference(reference)
        g.run()
        for i in range(1, iterations + 1):
            g.iterate()
            if i % every == 0 or i == iterations:
                e = g.film_error()
                emit({"integrator": name, "iteration": e["iterations"], "seconds": g.status()["total_time"], **e})
    finally:
        g.close()


def call_times(sd, reference, reps):
    """CUDA-event medians of one etxb_read_film_view and one etxb_film_error on the module's stream, after warm-up calls."""
    import torch
    g = api.GPUPathTracing(sd, flavor="fast")
    try:
        g.render(2)
        g.set_reference(reference)
        stream = torch.cuda.ExternalStream(g.stream())
        calls = {"read_film_view_ms": lambda: g.view(S.FILM_RESULT, S.VIEW_TONEMAPPED, S.VIEW_OPT_TONEMAPPING | S.VIEW_OPT_SRGB, 1.0, rgba8=True),
                 "film_error_ms": lambda: g.film_error()}
        out = {}
        for key, call in calls.items():
            for _ in range(3):
                call()
            ms = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                call()
                b.record(stream)
                b.synchronize()
                ms.append(a.elapsed_time(b))
            out[key] = round(statistics.median(ms), 3)
        return out
    finally:
        g.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workload", default="C3")
    ap.add_argument("--iterations", type=int, default=64)
    ap.add_argument("--every", type=int, default=4)
    ap.add_argument("--reference", default=None, help="reference image file (the film's size); default: a long path-tracer render")
    ap.add_argument("--reference-iterations", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.iterations < 1 or args.every < 1:
        ap.error("--iterations and --every must be at least 1")
    import torch
    torch.cuda.init()
    gpu = card()
    sd = scenes.config(args.workload)
    lines = []

    def emit(d):
        lines.append(json.dumps(d))
        print(lines[-1], flush=True)

    if args.reference:
        reference = api.read_reference_image(args.reference)
    else:
        g = api.GPUPathTracing(sd, flavor="fast")
        try:
            g.render(args.reference_iterations, first_iteration=REFERENCE_FIRST_ITERATION)
            reference = g.film(S.FILM_RESULT)
        finally:
            g.close()
    for name, cls in (("vcm", api.GPUVCM), ("pt", api.GPUPathTracing)):
        curve(cls, name, sd, reference, args.iterations, args.every, emit)
    emit({"card": gpu, "workload": args.workload, "film": [sd.width, sd.height],
          "reference": args.reference or f"pt, {args.reference_iterations} iterations from {REFERENCE_FIRST_ITERATION}", **call_times(sd, reference, args.reps)})
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
