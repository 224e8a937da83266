"""The viewer on the device (DESIGN §14): k_film_view against the float32 model (tests/view_model.py) for every view, option set and exposure in
both builds; etxb_read_film_view against the same kernel on the read-back layers; the export's bytes from the same tone curve; etxb_film_error
against float64 numpy; the reference slot's round trips, lifetime and refusals.  Run with -m gpu.
"""
import numpy as np
import pytest

import view_model as M
from conftest import bit_equal
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED, ERR_NOT_READY = -1, -4, -5
FLAVORS = ("parity", "fast")
EXPOSURES = (1.0 / 1024.0, 1.0, 3.7, 1024.0)
OPTIONS = range(8)
# The tone curve is CUDA's expf / powf in both builds (it is the export's curve, whose bytes stay as they were), not the oracle's portable
# functions: on the views that go through it the device is held to the model within a few ulp of exp near 1 carried through the sRGB curve
# (slope up to ~12), i.e. 4e-6 absolute plus 1e-5 relative.
CURVE_ATOL, CURVE_RTOL = 4e-6, 1e-5


@pytest.fixture(scope="module")
def api():
    from etx_tracer_b200 import api as m
    return m


@pytest.fixture(scope="module")
def fns():
    try:
        return M.oracle_functions() or (M.numpy_exp, M.numpy_pow)
    except OSError:
        return M.numpy_exp, M.numpy_pow


@pytest.fixture(scope="module")
def ctx(api):
    made = {f: api.GPUVCM(flavor=f) for f in FLAVORS}
    yield made
    for g in made.values():
        g.close()


def _crafted(rng, n):
    """Pixels of every class the shader tells apart: valid across magnitudes, NaN / inf / negative in each channel, zeros, and luminance
    differences on both sides of 1/8192 against the reference."""
    c = (rng.uniform(0, 4, (n, 4)) * 10.0 ** rng.integers(-3, 3, (n, 1))).astype(np.float32)
    r = (rng.uniform(0, 4, (n, 4)) * 10.0 ** rng.integers(-3, 3, (n, 1))).astype(np.float32)
    k = n // 16
    for j, v in enumerate((np.nan, np.inf, -np.inf, -0.5)):
        c[j * k:(j + 1) * k, j % 4] = v
    c[4 * k:5 * k] = 0.0
    near = slice(5 * k, 7 * k)
    r[near] = c[near]
    step = (np.float32(1.0 / 8192.0) / np.float32(0.6780)) * rng.choice([0.5, 0.999, 1.0, 1.001, 2.0], (2 * k,)).astype(np.float32)
    r[near, 1] = c[near, 1] + step * rng.choice([-1, 1], (2 * k,))
    return c, r


def _same(a, b):
    """Bit-equal except in the NaN encodings: the device writes its canonical NaN where numpy keeps the input's."""
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and bit_equal(np.where(nan, 0, a), np.where(nan, 0, b))


def _curve_views(view, options):
    return view in (M.RESULT, M.REFERENCE) and not (options & M.SKIP_COLOR_CONVERSION) and (options & (M.TONEMAPPING | M.SRGB))


@pytest.mark.parametrize("flavor", FLAVORS)
def test_views_match_the_model(ctx, fns, flavor):
    g = ctx[flavor]
    c, r = _crafted(np.random.default_rng(7), 4096)
    for view in range(6):
        for options in OPTIONS:
            for exposure in EXPOSURES:
                want = M.film_view(c, r, view, options, exposure, *fns)
                got = g.debug_film_view(c, r, view, options, exposure)
                got8 = g.debug_film_view(c, r, view, options, exposure, rgba8=True)
                case = f"{flavor} view {view} options {options} exposure {exposure}"
                if _curve_views(view, options):
                    assert np.array_equal(np.isnan(got), np.isnan(want)), case
                    ok = np.isclose(got, want, rtol=CURVE_RTOL, atol=CURVE_ATOL, equal_nan=True)
                    assert ok.all(), (case, got[~ok][:4], want[~ok][:4])
                    assert np.abs(got8.astype(int) - M.unorm8(want).astype(int)).max() <= 1, case
                    assert np.array_equal(got8, M.unorm8(got)), case  # the 8-bit form is the float form stored
                else:
                    # lum is never contracted and the products are single roundings: these views are exact in both builds
                    assert _same(got, want), case
                    assert np.array_equal(got8, M.unorm8(want)), case


@pytest.mark.parametrize("flavor", FLAVORS)
def test_views_refuse_bad_arguments(ctx, api, flavor):
    g = ctx[flavor]
    c = np.ones((4, 4), np.float32)
    for view, options, exposure in ((6, 0, 1.0), (0, 8, 1.0), (0, 0, float("nan")), (0, 0, float("inf"))):
        with pytest.raises(api.EtxbError) as e:
            g.debug_film_view(c, c, view, options, exposure)
        assert e.value.code == ERR_INVALID_ARGUMENT
    for view in (M.REFERENCE, M.RELATIVE, M.ABSOLUTE):
        with pytest.raises(api.EtxbError) as e:
            g.debug_film_view(c, None, view, 0, 1.0)
        assert e.value.code == ERR_NOT_READY


@pytest.mark.parametrize("flavor", FLAVORS)
def test_error_matches_float64_numpy_at_1080p(ctx, flavor):
    g = ctx[flavor]
    rng = np.random.default_rng(11)
    c, r = _crafted(rng, 1920 * 1080)
    c, r = c.reshape(1080, 1920, 4), np.abs(r).reshape(1080, 1920, 4)
    want = M.film_error(c, r)
    got = g.debug_film_error(c, r)
    again = g.debug_film_error(c, r)
    assert got == again  # the same bits on every call
    assert got["iterations"] == 0
    for k, v in want.items():
        if isinstance(v, int):
            assert got[k] == v, k
        else:
            assert got[k] == pytest.approx(v, rel=1e-12, abs=0), k


@pytest.mark.parametrize("kind", ["vcm", "pt"])
def test_error_on_production_films_at_1080p(api, kind):
    """C1's Cornell box at 1920x1080, product build: the error of a render against another over a disjoint iteration range, against float64
    numpy on the two read-back films, and the same bits on a second call."""
    g = _integrator(api, kind, "fast", scenes.cornell_box(1920, 1080, samples=16))
    g.render(2, first_iteration=1000)
    g.use_as_reference(S.FILM_RESULT)
    ref = g.film(S.FILM_RESULT)
    g.render(2)
    film = g.film(S.FILM_RESULT)
    got = g.film_error()
    assert got == g.film_error() and got["iterations"] == 2 and got["pixels"] == 1920 * 1080 and got["mse"] > 0
    for k, v in M.film_error(film, ref).items():
        assert got[k] == (v if isinstance(v, int) else pytest.approx(v, rel=1e-12, abs=0)), k
    g.close()


def _scene(width=48, height=32):
    return scenes.cornell_box(width, height, samples=64, spectral=True, sphere=True)


def _integrator(api, kind, flavor, sd):
    return (api.GPUVCM if kind == "vcm" else api.GPUPathTracing)(sd, flavor=flavor)


@pytest.mark.parametrize("kind", ["vcm", "pt"])
@pytest.mark.parametrize("flavor", FLAVORS)
def test_read_path_equals_the_kernel_on_read_back_layers(api, flavor, kind):
    g = _integrator(api, kind, flavor, scenes.config("C1"))
    g.render(3)
    g.use_as_reference(S.FILM_RESULT)
    ref = g.film(S.FILM_RESULT)
    g.render(2, first_iteration=100)
    layers = range(S.FILM_DENOISED + 1)
    for layer in layers:
        film = g.film(layer)
        for view in range(6):
            for options in (M.TONEMAPPING | M.SRGB, M.SRGB, M.SKIP_COLOR_CONVERSION):
                for rgba8 in (False, True):
                    got = g.view(layer, view, options, 1.5, rgba8)
                    want = g.debug_film_view(film, ref, view, options, 1.5, rgba8)
                    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (layer, view, options, rgba8)
    # the export's bytes come from the same curve: trunc(255 clamp(Tonemapped view)), alpha 255, wherever the view tone-maps (validate() returns
    # the Camera layer's pixels with a negative channel, which the spectral-to-RGB step produces, as they are)
    for layer in (S.FILM_RESULT, S.FILM_CAMERA):
        film = g.film(layer)
        valid = (film >= 0).all(-1)
        assert valid.all() or layer != S.FILM_RESULT
        for exposure in (1.0, 3.0):
            v = g.view(layer, M.RESULT, M.TONEMAPPING | M.SRGB, exposure)
            ldr = g.film_ldr(layer, exposure)
            want = (np.float32(255.0) * np.clip(v[..., :3], 0, 1)).astype(np.uint8)
            assert np.array_equal(ldr[valid][:, :3], want[valid]) and (ldr[..., 3] == 255).all(), (layer, exposure)
    g.close()


@pytest.mark.parametrize("flavor", FLAVORS)
def test_round_trips_through_exr_and_use_as_reference(api, flavor, tmp_path):
    g = api.GPUVCM(_scene(), flavor=flavor)
    g.render(4)
    g.save_image(str(tmp_path / "ref.exr"), S.FILM_RESULT)
    ref = api.read_reference_image(str(tmp_path / "ref.exr"))
    assert bit_equal(ref, g.film(S.FILM_RESULT))
    g.set_reference(ref)
    e = g.film_error()
    assert e["mse"] == 0.0 and e["rel_mse"] == 0.0 and e["lum_above"] == 0 and e["lum_below"] == 0 and e["iterations"] == 4
    g.use_as_reference(S.FILM_RESULT)
    first = g.film(S.FILM_RESULT)
    g.render(4, first_iteration=1000)
    second = g.film(S.FILM_RESULT)
    got = g.film_error()
    again = g.film_error()
    assert got == again and got["iterations"] == 4 and got["mse"] > 0
    want = M.film_error(second, first)
    for k, v in want.items():
        assert got[k] == (v if isinstance(v, int) else pytest.approx(v, rel=1e-12, abs=0)), k
    assert got == g.debug_film_error(second, first) | {"iterations": 4}
    g.close()


@pytest.mark.parametrize("kind", ["vcm", "pt"])
def test_views_do_not_disturb_the_render(api, kind):
    """Parity build: views taken after every enqueued iteration, while it is in flight, leave the film as a render without them.  (The VCM's
    light image is a float-atomic sum, equal only to rounding from run to run: its camera layer is compared.)"""
    sd = _scene()
    plain = _integrator(api, kind, "parity", sd)
    plain.render(4)
    watched = _integrator(api, kind, "parity", sd)
    watched.run(0)
    watched.use_as_reference(S.FILM_RESULT)
    for _ in range(4):
        watched.iterate()
        for view in range(6):
            watched.view(S.FILM_RESULT, view, M.TONEMAPPING | M.SRGB, 1.0, rgba8=(view % 2 == 0))
    watched.wait()
    for layer in ((S.FILM_CAMERA,) if kind == "vcm" else (S.FILM_RESULT, S.FILM_CAMERA, S.FILM_CAMERA_ADAPTIVE)):
        assert bit_equal(watched.film(layer), plain.film(layer)), layer
    plain.close()
    watched.close()


def test_reference_slot_lifetime_and_refusals(api):
    sd = _scene()
    g = api.GPUVCM(sd, flavor="fast")
    g.render(2)
    with pytest.raises(api.EtxbError) as e:
        g.view(S.FILM_RESULT, M.REFERENCE)
    assert e.value.code == ERR_NOT_READY
    with pytest.raises(api.EtxbError) as e:
        g.film_error()
    assert e.value.code == ERR_NOT_READY
    with pytest.raises(api.EtxbError) as e:
        g.set_reference(np.zeros((sd.height + 1, sd.width, 4), np.float32))
    assert e.value.code == ERR_INVALID_ARGUMENT
    for view, options, exposure in ((6, 0, 1.0), (0, 8, 1.0), (0, 0, float("nan"))):
        with pytest.raises(api.EtxbError) as e:
            g.view(S.FILM_RESULT, view, options, exposure)
        assert e.value.code == ERR_INVALID_ARGUMENT
    ref = np.full((sd.height, sd.width, 4), 0.25, np.float32)
    g.set_reference(ref)
    assert bit_equal(g.view(S.FILM_RESULT, M.REFERENCE, 0), ref)
    g.render(2)  # etxb_begin keeps it
    assert bit_equal(g.view(S.FILM_RESULT, M.REFERENCE, 0), ref)
    g.update_scene(_scene())  # so does an update at the same film size
    assert bit_equal(g.view(S.FILM_RESULT, M.REFERENCE, 0), ref)
    g.set_scene(_scene())  # and a new upload (etxb_upload_scene) at the same film size
    assert bit_equal(g.view(S.FILM_RESULT, M.REFERENCE, 0), ref)
    g.clear_reference()
    with pytest.raises(api.EtxbError) as e:
        g.view(S.FILM_RESULT, M.ABSOLUTE)
    assert e.value.code == ERR_NOT_READY
    g.set_reference(ref)
    g.update_scene(_scene(40, 32))  # another film size drops it
    with pytest.raises(api.EtxbError) as e:
        g.view(S.FILM_RESULT, M.RELATIVE)
    assert e.value.code == ERR_NOT_READY
    g.set_reference(np.full((32, 40, 4), 0.5, np.float32))
    g.set_scene(_scene())  # so does an upload at another film size
    with pytest.raises(api.EtxbError) as e:
        g.film_error()
    assert e.value.code == ERR_NOT_READY
    g.close()
    p = api.GPUVCM(sd, flavor="fast")
    p.set_partition(0, 2)
    for call in (lambda: p.set_reference(ref), lambda: p.use_as_reference(), lambda: p.clear_reference(), lambda: p.view(),
                 lambda: p.film_error()):
        with pytest.raises(api.EtxbError) as e:
            call()
        assert e.value.code == ERR_UNSUPPORTED
    p.close()


def test_front_ends_write_the_same_view_and_error(tmp_path, capsys):
    """host/render_main.cpp and `python -m etx_tracer_b200.render` with --reference --view relative --error-every 4 on the same scene file: the
    same PNG and the same final error line (the device time aside)."""
    import json
    import subprocess
    from etx_tracer_b200 import render
    from test_host_cpp import _build_native_renderer, _tiny_scene
    exe = _build_native_renderer(tmp_path)
    scene = _tiny_scene(tmp_path)
    common = ["--integrator", "pt", "--option", "bn=0"]
    assert render.main([scene, "-o", str(tmp_path / "ref.exr"), "--spp", "16"] + common) == 0
    capsys.readouterr()
    args = ["--spp", "8", "--reference", str(tmp_path / "ref.exr"), "--view", "relative", "--error-every", "4"] + common
    out = subprocess.run([exe, scene, "-o", str(tmp_path / "native.png")] + args, capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout[-500:], out.stderr[-500:])
    assert render.main([scene, "-o", str(tmp_path / "python.png")] + args) == 0
    lines = {"native": [json.loads(s) for s in out.stdout.splitlines() if s.startswith("{")],
             "python": [json.loads(s) for s in capsys.readouterr().out.splitlines() if s.startswith("{")]}
    for name, got in lines.items():
        assert len(got) >= 2 and got[-1]["iterations"] == 8 and got[-1]["mse"] > 0, (name, got)
    a, b = lines["native"][-1], lines["python"][-1]
    a.pop("seconds"), b.pop("seconds")
    assert a == b
    assert open(tmp_path / "native.png", "rb").read() == open(tmp_path / "python.png", "rb").read()
