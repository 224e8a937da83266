"""Headless render of a reference scene file on the GPU:  python -m etx_tracer_b200.render scene.json [-o out.exr]

What the reference application does between File > Open and File > Save (sources/raytracer/app.cxx: load_scene_file :318-352, the integrator
selected by options.json "integrator" :88-99, on_save_image_selected :261-295) without its window: the scene loader (the module's C++ one by default; host/render_main.cpp is this program in C++), one of the two
device integrators — "vcm" (CPUVCM's algorithm, the default) or "pt" (CPUPathTracing's) — pumped like IntegratorThread pumps Integrator::update,
and the film export (OpenEXR float layer, or the tone-mapped PNG).  There is no CPU fallback: without a CUDA device this fails.
"""
import argparse
import sys
import time

from . import loader, structs as S
from .api import GPUPathTracing, GPUVCM, SceneFile

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
    args = ap.parse_args(argv)

    t0 = time.time()
    sd = SceneFile(args.scene) if args.loader == "cpp" else loader.load_scene(args.scene)
    for w in (sd.warnings if args.loader == "cpp" else sd.loader_warnings):
        print("warning:", w, file=sys.stderr)
    print(f"loaded {sd.triangle_count} triangles, {sd.width}x{sd.height}, in {time.time() - t0:.2f} s", file=sys.stderr)
    if args.spp > 0:
        sd.scene["samples"] = args.spp
    g = (GPUPathTracing if args.integrator == "pt" else GPUVCM)(sd, flavor="fast")
    for kv in args.option:
        key, _, value = kv.partition("=")
        g.set_option(key, float(value))
    if args.integrator == "pt" and args.noise_threshold is not None:
        g.set_scene_settings(args.noise_threshold, float(sd.scene["radiance_clamp"][0]))
    g.run()
    while g.update():  # non-blocking like Integrator::update; a UI would draw a preview here (g.film_ldr)
        time.sleep(0.002)
    g.wait()
    st = g.status()
    n = sd.width * sd.height * st["completed_iterations"]
    print(f"{st['completed_iterations']} iterations in {st['total_time']:.3f} s of device time: {n / max(st['total_time'], 1e-9) / 1e6:.2f} Msamples/s", file=sys.stderr)
    if args.denoise:
        g.denoise(S.FILM_RESULT)
    layer = args.layer or ("denoised" if args.denoise else "result")
    g.save_image(args.output, LAYERS[layer], tonemapped=args.output.lower().endswith(".png"), exposure=args.exposure)
    print(args.output)
    g.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
