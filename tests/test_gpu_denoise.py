"""Film::denoise on the device (etxb_denoise, DESIGN §13): the kernels against the float64 model (tests/denoise_model.py) on seeded images in both
builds, bit-reproducible output, the VCM's CameraAdaptive layer, quality gates on renders of both integrators, the Denoised layer through every
film read-out and the C++ adapter, and the refusals.  Run with -m gpu.
"""
import subprocess

import numpy as np
import pytest

import denoise_model as M
from conftest import bit_equal
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, ERR_NOT_READY = -1, -4, -5

# Worst |device - model| / (|model| + 1e-3) over every case below, measured on an H100 80GB HBM3 (700 W): parity 1.74e-6, product 1.99e-6
# (both on "edges"; the float32 sums of the distances and of the weighted colours against float64).  The product build adds approximate
# division and __expf, whose error is about 2 ulp plus |x| 2^-22 relative: over the distances that still carry weight (|x| < ~20) that is
# below 1e-5 relative per weight, and averaged over a window of weights it stays under the float32 sums' own error, as measured.
# Bounds: about twice the measured values.
BOUND = {"parity": 3.5e-6, "fast": 4e-6}
VAR_BOUND = {"parity": 1.8e-6, "fast": 1.2e-6}  # the smoothed variance (no exp): measured 8.7e-7 (parity) and 5.5e-7 (product), on "mixed"


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


@pytest.fixture(scope="module")
def ctx(api):
    """one context per build for the host-array hook (it needs no scene)"""
    made = {f: api.GPUVCM(flavor=f) for f in ("parity", "fast")}
    yield made
    for g in made.values():
        g.close()


def _case(name, seed):
    """(color, camera, half, counts, normals, albedo) of one seeded case"""
    rng = np.random.default_rng(seed)
    shapes = {"odd": (23, 37), "one": (1, 1), "narrow": (40, 5), "flat": (9, 3), "edges": (40, 48), "nonfinite": (31, 29), "mixed": (33, 35)}
    h, w = shapes[name]
    y, x = np.mgrid[0:h, 0:w]
    clean = np.stack([0.5 + 0.3 * np.sin(x / 4.0), 0.4 + 0.2 * np.cos(y / 5.0), 0.2 + 0.01 * (x + y)], -1)
    normals = albedo = None
    if name == "edges":
        clean = np.where((x > w // 2)[..., None] | (y < h // 3)[..., None], 1.5 * clean, 0.05 * clean)
        normals = np.stack([np.where(x > w // 2, 1.0, 0.0), np.where(x > w // 2, 0.0, 1.0), np.zeros_like(x, float)], -1)
        albedo = np.stack([np.where(y < h // 3, 0.8, 0.2), np.full((h, w), 0.5), 0.01 * x], -1)
    elif name in ("odd", "mixed", "nonfinite"):
        normals = np.stack([np.cos(x / 9.0), np.sin(x / 9.0), np.zeros((h, w))], -1)
        albedo = np.stack([np.full((h, w), 0.6), 0.5 + 0.2 * (x > w // 3), np.full((h, w), 0.3)], -1)
    counts = np.full((h, w), 16, np.uint32) if name in ("odd", "edges", "narrow") else rng.integers(2, 70, (h, w)).astype(np.uint32)
    n = counts[..., None].astype(np.float64)
    sigma = 0.15
    camera = clean + sigma * rng.standard_normal((h, w, 3)) / np.sqrt(n)
    half = camera + sigma * rng.standard_normal((h, w, 3)) / np.sqrt(n)
    color = camera.copy()
    if name == "nonfinite":
        color[2, 3] = [np.nan, 0.1, 0.1]
        color[10, 20, 1] = np.inf
        color[30, 0] = -np.inf
        half[15, 15, 2] = np.nan  # a variance that is not finite: copied through like a non-finite colour
        albedo[5, 5, 0] = np.nan
    return tuple(a if a is None else np.asarray(a, np.float32) for a in (color, camera, half)) + (counts,) + \
        tuple(a if a is None else np.asarray(a, np.float32) for a in (normals, albedo))


CASES = ["odd", "one", "narrow", "flat", "edges", "nonfinite", "mixed"]


def _rel(a, b):
    return np.abs(a - b) / (np.abs(b) + 1e-3)


@pytest.mark.parametrize("flavor", ["parity", "fast"])
@pytest.mark.parametrize("case", CASES)
def test_kernels_match_the_model(ctx, flavor, case):
    color, camera, half, counts, normals, albedo = _case(case, CASES.index(case) + 11)
    out, var = ctx[flavor].debug_denoise(color, camera, half, counts, normals, albedo)
    ref, ref_var = M.denoise(color, camera, half, counts, normals, albedo)
    ok = np.isfinite(ref).all(-1)
    # copied through: the input, bit for bit (NaN payloads included)
    assert bit_equal(out[~ok][:, :3], color[~ok][:, :3])
    err = float(_rel(out[ok][:, :3], ref[ok]).max())
    verr = float(_rel(var[..., :3], ref_var).max())
    print(f"MEASURED denoise {flavor} {case} {err:.3e} var {verr:.3e}")
    assert err < BOUND[flavor], err
    assert verr < VAR_BOUND[flavor], verr
    if case in ("flat", "narrow", "one"):  # films narrower than the window: most candidates are skipped, the output stays finite
        assert np.isfinite(out).all()


def test_zero_guides_equal_no_guides_on_the_device(ctx):
    color, camera, half, counts, _, _ = _case("mixed", 3)
    zero = np.zeros_like(color)
    for g in ctx.values():
        a, _ = g.debug_denoise(color, camera, half, counts)
        b, _ = g.debug_denoise(color, camera, half, counts, zero, zero)
        assert bit_equal(a, b)


def test_repeated_calls_are_bit_identical(ctx):
    color, camera, half, counts, normals, albedo = _case("edges", 5)
    for g in ctx.values():
        runs = [g.debug_denoise(color, camera, half, counts, normals, albedo)[0] for _ in range(3)]
        assert bit_equal(runs[0], runs[1]) and bit_equal(runs[0], runs[2])


def test_a_pixel_with_one_sample_is_not_ready(api, ctx):
    color, camera, half, counts, _, _ = _case("odd", 7)
    counts = counts.copy()
    counts[4, 5] = 1
    with pytest.raises(api.EtxbError) as e:
        ctx["fast"].debug_denoise(color, camera, half, counts)
    assert e.value.code == ERR_NOT_READY


# ---- the VCM's CameraAdaptive layer -------------------------------------------------------------------------------------------------------------
def _lerp32(a, b, t):
    """lerpf (math.hxx:691) in float32 without contraction, as the parity build computes it"""
    t = np.float32(t)
    return a * (np.float32(1.0) - t) + b * t


@pytest.mark.parametrize("scene", ["C1", "C2"])
@pytest.mark.parametrize("size", [1, 2, 8])
def test_vcm_camera_adaptive_is_the_even_sample_mean(api, scene, size):
    """Parity build.  VCM iterations are independent (the index sets the seeds and the radius), so one iteration begun at index k gives that
    iteration's camera value; the layer after K iterations is then the reference's running lerp over the even ones (film.cxx:173-230),
    bit for bit, at pixel sizes 1, 2 and 8."""
    sd = scenes.cornell_box(40, 36, samples=64, spectral=scene == "C2", sphere=scene == "C2", sphere_segments=32, sphere_rings=17)
    g = api.GPUVCM(sd, flavor="parity")
    try:
        g.set_film_pixel_size(size)
        K = 6
        values = []
        for k in range(K):
            g.render(1, first_iteration=k)
            values.append(g.film(S.FILM_CAMERA)[..., :3].copy())
            if k == 0:
                assert bit_equal(g.film(S.FILM_CAMERA_ADAPTIVE)[..., :3], values[0])
        g.render(K)
        adaptive = g.film(S.FILM_CAMERA_ADAPTIVE)[..., :3]
        want = values[0]
        for k in range(2, K, 2):
            want = _lerp32(values[k], want, np.float64(k) / (k + 2.0))
        assert bit_equal(adaptive, want)
        assert not bit_equal(adaptive, g.film(S.FILM_CAMERA)[..., :3])
    finally:
        g.close()


@pytest.fixture(scope="module")
def adaptive_oracle():
    from oracle import oracle_vcm_adaptive_py
    if not oracle_vcm_adaptive_py.available():
        pytest.skip("oracle/_ref/liboracle_vcm_adaptive_parity.so not built (run build() where /root/reference exists)")
    return oracle_vcm_adaptive_py


@pytest.mark.parametrize("scene", ["C1", "C2"])
@pytest.mark.parametrize("size", [1, 2, 8])
def test_vcm_camera_adaptive_against_the_oracle(api, adaptive_oracle, scene, size):
    """Parity build: the VCM's CameraAdaptive layer, bit for bit the oracle's restated Film (oracle_vcm_adaptive.cxx), with the camera layer,
    after one iteration and after six"""
    sd = scenes.cornell_box(40, 36, samples=64, spectral=scene == "C2", sphere=scene == "C2", sphere_segments=32, sphere_rings=17)
    g = api.GPUVCM(sd, flavor="parity")
    o = adaptive_oracle.Oracle(sd)
    try:
        g.set_film_pixel_size(size)
        o.set_film_pixel_size(size)
        for iterations in (1, 6):
            g.render(iterations)
            o.begin(0)
            o.run(iterations, threads=1)
            for layer in (S.FILM_CAMERA, S.FILM_CAMERA_ADAPTIVE):
                assert bit_equal(g.film(layer)[..., :3], o.film(layer)[..., :3]), (iterations, layer)
    finally:
        g.close()
        o.close()


# ---- quality on renders -----------------------------------------------------------------------------------------------------------------------------
def _relmse(x, ref):
    x, ref = x[..., :3].astype(np.float64), ref[..., :3].astype(np.float64)
    return float(((x - ref) ** 2 / (ref ** 2 + 1e-2)).mean())


# relMSE = mean((x - ref)^2 / (ref^2 + 0.01)) against the product build's own render of `ref_spp` iterations begun at iteration 16, measured on
# an H100 80GB HBM3 (700 W):
#            noisy (16 spp)   denoised (16 spp)   the reference, denoised (bias check)
#   pt C2    0.3284           0.0960 (0.29x)      0.00297
#   pt C3    0.5435           0.2265 (0.42x)      0.00288
#   vcm C1   0.00416          0.00184 (0.44x)     0.000048
#   vcm C2   0.1173           0.0168 (0.14x)      0.00123
# Gates: the denoised relMSE is at most half the noisy one; denoising the reference moves it by less than about twice what was measured (an
# upper bound on the filter's bias: it includes the reference's own remaining noise, which the filter removes).
QUALITY = {
    "pt-C2": (2048, 6e-3),
    "pt-C3": (1024, 6e-3),
    "vcm-C1": (1024, 1e-4),
    "vcm-C2": (1024, 2.5e-3),
}


def _quality_scene(name):
    if name.endswith("C3"):
        return scenes.procedural_room(160, 96, samples=4096, spectral=True)
    if name.endswith("C2"):
        return scenes.cornell_box(96, 96, samples=4096, spectral=True, sphere=True, sphere_segments=64, sphere_rings=33)
    return scenes.cornell_box(96, 96, samples=4096, spectral=False, sphere=False)


@pytest.mark.parametrize("name", sorted(QUALITY))
def test_quality_gate_on_renders(api, name):
    ref_spp, bias_bound = QUALITY[name]
    sd = _quality_scene(name)
    pt = name.startswith("pt")
    g = (api.GPUPathTracing if pt else api.GPUVCM)(sd, flavor="fast")
    try:
        if pt:
            g.set_scene_settings(0.0)  # no adaptive sampling: every pixel takes every sample (the reference has no converged-early pixels)
        g.render(ref_spp, first_iteration=16)  # iterations 16 onwards: none of the noisy image's samples is in the reference
        ref = g.film(S.FILM_RESULT).copy()
        g.denoise(S.FILM_RESULT)
        bias = _relmse(g.film(S.FILM_DENOISED), ref)
        g.render(16)
        noisy = g.film(S.FILM_RESULT).copy()
        g.denoise(S.FILM_RESULT)
        den = g.film(S.FILM_DENOISED).copy()
    finally:
        g.close()
    e_noisy, e_den = _relmse(noisy, ref), _relmse(den, ref)
    print(f"MEASURED quality {name} noisy {e_noisy:.4g} denoised {e_den:.4g} bias {bias:.4g}")
    assert np.isfinite(den).all()
    assert e_den <= 0.5 * e_noisy, (e_noisy, e_den)
    assert bias < bias_bound, bias


# ---- the Denoised layer through the film read-outs, the C++ adapter ---------------------------------------------------------------------------------
def test_denoised_layer_through_every_read_out(api, tmp_path):
    sd = scenes.cornell_box(48, 40, samples=64, spectral=True, sphere=True, sphere_segments=32, sphere_rings=17)
    g = api.GPUPathTracing(sd, flavor="fast")
    try:
        assert not g.film(S.FILM_DENOISED).any()  # zeros before the first etxb_denoise, like StorageDenoised
        g.render(8)
        g.denoise(S.FILM_CAMERA)
        den = g.film(S.FILM_DENOISED).copy()
        assert np.isfinite(den).all() and den[..., :3].sum() > 0 and (den[..., 3] == 1.0).all()
        ldr = g.film_ldr(S.FILM_DENOISED, 1.5)
        assert np.abs(ldr.astype(int) - api.tonemap(den, 1.5).astype(int)).max() <= 1
        g.save_image(str(tmp_path / "d.exr"), S.FILM_DENOISED)
        back = api.read_image(str(tmp_path / "d.exr"))
        assert back.dtype == np.float32 and bit_equal(back, den)
        # the layer keeps its value through later iterations; the next etxb_denoise replaces it
        g.render(4)
        assert bit_equal(g.film(S.FILM_DENOISED), den)
        g.denoise(S.FILM_RESULT)
        assert not bit_equal(g.film(S.FILM_DENOISED), den)
        # a film resize starts it over
        g.update_scene(scenes.cornell_box(32, 24, samples=64, spectral=True, sphere=True, sphere_segments=32, sphere_rings=17))
        assert g.film(S.FILM_DENOISED).shape == (24, 32, 4) and not g.film(S.FILM_DENOISED).any()
    finally:
        g.close()


def test_native_renderer_denoises_what_the_python_front_end_denoises(tmp_path):
    """host/render_main.cpp --denoise (IntegratorAdapter::denoise) and `python -m etx_tracer_b200.render --denoise` on the same scene file, both
    integrators: the same Denoised layer (the VCM's light image is a float-atomic sum, so equal to rounding)."""
    from etx_tracer_b200 import loader, render
    from test_host_cpp import _build_native_renderer, _tiny_scene
    exe = _build_native_renderer(tmp_path)
    scene = _tiny_scene(tmp_path)
    for integrator, opts in (("pt", ["--option", "bn=0"]), ("vcm", ["--option", "vcm-merging=0"])):
        a, b = str(tmp_path / f"native_{integrator}.exr"), str(tmp_path / f"python_{integrator}.exr")
        args = ["--integrator", integrator, "--spp", "6", "--denoise"] + opts
        out = subprocess.run([exe, scene, "-o", a] + args, capture_output=True, text=True)
        assert out.returncode == 0, (out.returncode, out.stdout[-500:], out.stderr[-500:])
        assert render.main([scene, "-o", b] + args) == 0
        fa, fb = loader.read_image(a)[0].astype(np.float64), loader.read_image(b)[0].astype(np.float64)
        assert fa.shape == fb.shape == (30, 40, 4) and fb[..., :3].mean() > 1e-3
        err = float(np.sqrt(((fa - fb)[..., :3] ** 2).sum()) / np.sqrt((fb[..., :3] ** 2).sum()))
        assert err < 1e-5, (integrator, err)


# ---- refusals ---------------------------------------------------------------------------------------------------------------------------------------
def _denoises(g):
    g.render(3)
    g.denoise(S.FILM_RESULT)
    assert np.isfinite(g.film(S.FILM_DENOISED)).all()


@pytest.mark.parametrize("integrator", ["vcm", "pt"])
def test_refusals_leave_the_context_rendering(api, integrator):
    sd = scenes.cornell_box(40, 32, samples=64)
    g = (api.GPUPathTracing if integrator == "pt" else api.GPUVCM)(sd, flavor="fast")
    try:
        for layer in (S.FILM_LIGHT, S.FILM_NORMALS, S.FILM_DENOISED, 99):
            with pytest.raises(api.EtxbError) as e:
                g.denoise(layer)
            assert e.value.code == ERR_INVALID_ARGUMENT
        _denoises(g)
        g.render(1)  # one sample: the two half buffers are not both there yet
        with pytest.raises(api.EtxbError) as e:
            g.denoise(S.FILM_RESULT)
        assert e.value.code == ERR_NOT_READY
        _denoises(g)
        g.set_partition(0, 2)
        g.render(2)
        with pytest.raises(api.EtxbError) as e:
            g.denoise(S.FILM_RESULT)
        assert e.value.code == ERR_UNSUPPORTED
        g.set_partition(0, 1)
        _denoises(g)
    finally:
        g.close()


def test_a_context_with_a_communicator_is_refused(api):
    import torch  # noqa: F401  (loads torch's bundled libnccl, which the module shares)
    try:
        ids = api.comm_unique_ids(1)
    except api.EtxbError:
        pytest.skip("libnccl cannot be loaded")
    g = api.GPUVCM(scenes.cornell_box(40, 32, samples=64), flavor="fast")
    try:
        g.comm_init(1, 0, ids)
        g.render(2)
        with pytest.raises(api.EtxbError) as e:
            g.denoise(S.FILM_RESULT)
        assert e.value.code == ERR_UNSUPPORTED
        g.render(2)
        assert np.isfinite(g.film()).all()
    finally:
        g.close()


def test_no_scene_is_not_ready(api):
    g = api.GPUVCM(flavor="fast")
    try:
        with pytest.raises(api.EtxbError) as e:
            g.denoise(S.FILM_RESULT)
        assert e.value.code == ERR_NOT_READY
    finally:
        g.close()
