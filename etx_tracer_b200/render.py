"""Headless render of a reference scene file on the GPU:  python -m etx_tracer_b200.render scene.json [-o out.exr]

What the reference application does between File > Open and File > Save (sources/raytracer/app.cxx: load_scene_file :318-352, the integrator
selected by options.json "integrator" :88-99, on_save_image_selected :261-295) without its window: the scene loader (the module's C++ one by default; host/render_main.cpp is this program in C++), one of the two
device integrators — "vcm" (CPUVCM's algorithm, the default) or "pt" (CPUPathTracing's) — pumped like IntegratorThread pumps Integrator::update,
and the film export (OpenEXR float layer, or the tone-mapped PNG).  There is no CPU fallback: without a CUDA device this fails.  With --gpus N
the frame is split into pixel tiles over N GPUs, one process each (both integrators; the exchange runs inside the module over NCCL).
"""
import argparse
import json
import sys
import time

from . import loader, structs as S
from .api import GPUPathTracing, GPUVCM, SceneFile, read_reference_image, tonemap, write_exr, write_png

LAYERS = {"result": S.FILM_RESULT, "camera": S.FILM_CAMERA, "light": S.FILM_LIGHT, "normals": S.FILM_NORMALS, "albedo": S.FILM_ALBEDO,
          "denoised": S.FILM_DENOISED}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("scene", help=".json scene description or .obj file in the reference's format")
    ap.add_argument("-o", "--output", default="render.exr", help=".exr (float layer) or .png (tone-mapped)")
    ap.add_argument("--integrator", choices=("vcm", "pt"), default="vcm")
    ap.add_argument("--spp", type=int, default=0, help="iterations; 0 = the scene's `samples`")
    ap.add_argument("--layer", choices=sorted(LAYERS), default=None, help="film layer to export (default: result, or denoised with --denoise)")
    ap.add_argument("--exposure", type=float, default=1.0, help="tone map exposure of a .png output")
    ap.add_argument("--option", action="append", default=[], metavar="KEY=VALUE", help="integrator option in the reference's ids, e.g. vcm-merging=0 or nee=0")
    ap.add_argument("--loader", choices=("cpp", "python"), default="cpp", help="the module's C++ scene loader (etxb_scene_file_load) or its Python twin (loader.py)")
    ap.add_argument("--denoise", action="store_true", help="denoise the Result layer before the export (the application's Denoise button); "
                    "--layer defaults to denoised")
    ap.add_argument("--noise-threshold", type=float, default=None, help="pt: Scene::noise_threshold of the adaptive sampling (default: the scene's)")
    ap.add_argument("--gpus", type=int, default=1, help="render pixel tiles on this many GPUs, one process each, exchanging over NCCL inside the "
                    "module; rank 0 writes the output")
    ap.add_argument("--reference", default=None, metavar="FILE", help="the viewer's reference image (EXR / HDR / PFM / PNG / JPEG, the film's size): "
                    "prints the final error against it as one JSON line")
    ap.add_argument("--view", choices=S.VIEW_NAMES, default=None, help="write this output view of the layer instead of the layer itself: 8-bit to a .png, "
                    "float to an .exr (tone mapping and sRGB on, --exposure)")
    ap.add_argument("--error-every", type=int, default=0, metavar="N", help="with --reference: one JSON error line per N completed iterations")
    args = ap.parse_args(argv)
    if args.gpus < 1:
        ap.error("--gpus must be at least 1")
    if args.error_every < 0 or (args.error_every and not args.reference):
        ap.error("--error-every needs --reference and N >= 1")
    if args.gpus > 1 and (args.reference or args.view):
        ap.error("--reference and --view need the whole film on one GPU: render with --gpus 1")
    if args.gpus == 1:
        return _render(args)
    if args.denoise:
        ap.error("--denoise needs the whole film and its sample counts on one GPU: render with --gpus 1 to denoise")
    import socket
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < args.gpus:
        ap.error(f"--gpus {args.gpus}: this machine has {torch.cuda.device_count()} CUDA devices")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_rank, args=(args, port), nprocs=args.gpus, join=True)
    return 0


def _rank(rank, args, port):
    """One process of a --gpus N render: a localhost process group hands the module's NCCL id to every rank, then each renders its tiles."""
    import os
    import torch
    import torch.distributed as dist
    from .api import comm_unique_ids
    from .multigpu import distribute_comm_ids
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=args.gpus, device_id=torch.device("cuda", rank))
    try:
        comm_id = distribute_comm_ids(dist, rank, 1, comm_unique_ids, device=torch.device("cuda", rank))
        _render(args, rank, comm_id)
    finally:
        dist.destroy_process_group()


def _render(args, rank=0, comm_id=None):
    world = args.gpus
    log = (lambda *a: print(*a, file=sys.stderr)) if rank == 0 else (lambda *a: None)
    t0 = time.time()
    sd = SceneFile(args.scene) if args.loader == "cpp" else loader.load_scene(args.scene)
    for w in (sd.warnings if args.loader == "cpp" else sd.loader_warnings):
        log("warning:", w)
    log(f"loaded {sd.triangle_count} triangles, {sd.width}x{sd.height}, in {time.time() - t0:.2f} s")
    if args.spp > 0:
        sd.scene["samples"] = args.spp
    g = (GPUPathTracing if args.integrator == "pt" else GPUVCM)(sd, flavor="fast", device=rank)
    if comm_id is not None:
        g.comm_init(world, rank, comm_id)
    for kv in args.option:
        key, _, value = kv.partition("=")
        g.set_option(key, float(value))
    if args.integrator == "pt" and args.noise_threshold is not None:
        g.set_scene_settings(args.noise_threshold, float(sd.scene["radiance_clamp"][0]))
    if args.reference:
        g.set_reference(read_reference_image(args.reference))
    g.run()
    reported = 0
    while g.update():  # non-blocking like Integrator::update; a UI would draw a preview here (g.film_ldr or g.view)
        if args.error_every and g.status()["completed_iterations"] >= reported + args.error_every:
            reported = _print_error(g)
        time.sleep(0.002)
    g.wait()
    if args.reference:
        _print_error(g)
    st = g.status()
    n = sd.width * sd.height * st["completed_iterations"]
    log(f"{st['completed_iterations']} iterations in {st['total_time']:.3f} s of device time{f' on rank 0 of {world}' if world > 1 else ''}: "
        f"{n / max(st['total_time'], 1e-9) / 1e6:.2f} Msamples/s")
    if args.denoise:
        g.denoise(S.FILM_RESULT)
    layer = args.layer or ("denoised" if args.denoise else "result")
    tonemapped = args.output.lower().endswith(".png")
    if args.view:
        out = g.view(LAYERS[layer], S.VIEW_NAMES.index(args.view), S.VIEW_OPT_TONEMAPPING | S.VIEW_OPT_SRGB, args.exposure, rgba8=tonemapped)
        (write_png if tonemapped else write_exr)(args.output, out)
    elif comm_id is None:
        g.save_image(args.output, LAYERS[layer], tonemapped=tonemapped, exposure=args.exposure)
    else:
        film = g.comm_reduce_film(LAYERS[layer])  # collective; the frame arrives on rank 0
        if rank == 0:
            if tonemapped:
                write_png(args.output, tonemap(film, args.exposure))
            else:
                write_exr(args.output, film)
    if rank == 0:
        print(args.output)
    g.close()
    return 0


def _print_error(g):
    """One JSON line: the Result layer's error against the reference after the iterations in flight, with the device time they took."""
    e = g.film_error(S.FILM_RESULT)
    print(json.dumps({"iteration": e["iterations"], "seconds": g.status()["total_time"], **e}), flush=True)
    return e["iterations"]


if __name__ == "__main__":
    sys.exit(main())
