"""How long Film::denoise takes on the device: etxb_denoise on C3 (procedural_room, 1920x1080, spectral) after a few iterations, under the path
tracer (normal and albedo guides) and the VCM (colour only).

For each integrator it reports, after warm-up calls,
  * the median time of one etxb_denoise between CUDA events recorded on the module's stream (the call is synchronous: it drains the context,
    runs its three kernels and synchronises);
  * the median host time of the call;
  * the device time of each of its kernels (the module's per-kernel CUDA events, a context created with profiling on).
Prints the card, its power limit and maximum SM clock, read in the same run, next to the numbers, and one JSON line.

    python tools/denoise_latency.py [--reps 20] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from etx_tracer_b200 import api, scenes, structs as S  # noqa: E402

KERNELS = ("denoise_variance", "denoise_smooth", "denoise_nlm")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("nvidia-smi found no GPU: this measurement runs on the device only")
    return q.stdout.strip().splitlines()[0]


def measure(cls, sd, reps):
    import torch
    g = cls(sd, flavor="fast", profile=True)
    try:
        g.render(4)
        stream = torch.cuda.ExternalStream(g.stream())
        for _ in range(3):  # warm-up: module load, scratch allocation, first launches
            g.denoise(S.FILM_RESULT)
        k0 = g.kernel_times()
        events, host = [], []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            t0 = time.perf_counter()
            g.denoise(S.FILM_RESULT)
            host.append(time.perf_counter() - t0)
            b.record(stream)
            b.synchronize()
            events.append(a.elapsed_time(b))
        k1 = g.kernel_times()
        kernels = {k: round((k1[k][0] - k0[k][0]) / reps, 3) for k in KERNELS}
        return {"event_ms_median": round(statistics.median(events), 3), "event_ms_min": round(min(events), 3),
                "host_ms_median": round(1e3 * statistics.median(host), 3), "kernel_ms": kernels}
    finally:
        g.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    gpu = card()
    sd = scenes.config("C3")
    result = {"card": gpu, "film": [sd.width, sd.height], "reps": args.reps}
    for name, cls in (("pt", api.GPUPathTracing), ("vcm", api.GPUVCM)):
        result[name] = measure(cls, sd, args.reps)
        print(f"{gpu}: {name} {sd.width}x{sd.height} etxb_denoise {result[name]['event_ms_median']} ms (events, median), kernels {result[name]['kernel_ms']}",
              file=sys.stderr)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
