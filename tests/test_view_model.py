"""The viewer's model (tests/view_model.py) on hand-computed pixels: CPU only."""
import numpy as np
import pytest

import view_model as M

f32 = np.float32


@pytest.fixture(scope="module")
def fns():
    """The oracle's exp / pow where it is built, numpy's elsewhere: the hand-computed values hold for both."""
    try:
        return M.oracle_functions() or (M.numpy_exp, M.numpy_pow)
    except OSError:
        return M.numpy_exp, M.numpy_pow


def _px(*rows):
    return np.array(rows, f32)


def test_validate_markers_come_before_every_view(fns):
    c = _px([np.nan, 1, 1, 1], [1, np.inf, 1, 1], [1, 1, 1, np.nan], [np.inf, np.nan, 0, 1])
    r = np.ones_like(c)
    for view in (M.RESULT, M.ORIGINAL, M.REFERENCE, M.RELATIVE, M.ABSOLUTE):
        out = M.film_view(c, r, view, M.TONEMAPPING | M.SRGB, 2.0, *fns)
        assert np.array_equal(out[0], M.NAN_MARKER) and np.array_equal(out[2], M.NAN_MARKER) and np.array_equal(out[3], M.NAN_MARKER)
        assert np.array_equal(out[1], M.INF_MARKER)


def test_negative_pixel_is_returned_clamped_and_not_tonemapped(fns):
    c = _px([-1, 0.5, 2, 1], [0.25, 0.5, 1, -0.5])
    out = M.film_view(c, None, M.RESULT, M.TONEMAPPING | M.SRGB, 3.0, *fns)
    assert np.array_equal(out, _px([0, 0.5, 2, 1], [0.25, 0.5, 1, 0]))


def test_alpha_view_broadcasts_exposure_times_w(fns):
    c = _px([1, 2, 3, 0.5], [np.nan, 0, 0, 2])
    out = M.film_view(c, None, M.ALPHA, M.TONEMAPPING | M.SRGB, 4.0, *fns)
    assert np.array_equal(out, _px([2, 2, 2, 2], [8, 8, 8, 8]))  # the alpha view does not validate


def test_skip_color_conversion_scales_the_raw_value(fns):
    c = _px([np.nan, -1, 2, 1])
    out = M.film_view(c, None, M.RESULT, M.SKIP_COLOR_CONVERSION | M.TONEMAPPING, 0.5, *fns)
    assert np.isnan(out[0, 0]) and np.array_equal(out[0, 1:], _px([-0.5, 1, 0.5])[0])


def test_tonemap_reaches_w_and_srgb_does_not(fns):
    c = _px([1, 1, 1, 1])
    tm = M.film_view(c, None, M.RESULT, M.TONEMAPPING, 1.0, *fns)[0]
    assert np.allclose(tm, 1 - np.exp(-1.0), rtol=0, atol=2e-7)
    both = M.film_view(c, None, M.RESULT, M.TONEMAPPING | M.SRGB, 1.0, *fns)[0]
    assert both[3] == tm[3]
    assert abs(both[0] - (1.055 * (1 - np.exp(-1.0)) ** (1 / 2.4) - 0.055)) < 1e-6
    lin = M.film_view(_px([0.002, 0.5, 0, 0.25]), None, M.RESULT, M.SRGB, 1.0, *fns)[0]
    assert lin[0] == f32(12.92) * f32(0.002) and lin[2] == 0 and lin[3] == f32(0.25)


def test_hdr_view_is_exposure_times_c(fns):
    out = M.film_view(_px([1, 2, 4, 8]), None, M.ORIGINAL, M.TONEMAPPING | M.SRGB, 0.25, *fns)
    assert np.array_equal(out[0], _px([0.25, 0.5, 1, 2])[0])


@pytest.mark.parametrize("sign", [1, -1])
def test_difference_views_either_side_of_the_threshold(fns, sign):
    # luminance differences of 1/8192 exactly (not above the threshold) and of 2/8192 (above); sign = +1: the reference is brighter (red)
    base = _px([0, 0, 0, 1])
    g = f32(0.6780)
    d1 = _px([0, f32(1 / 8192) / g, 0, 1])
    assert M.lum(d1)[0] <= M.THRESHOLD
    d2 = _px([0, f32(4 / 8192) / g, 0, 1])
    assert M.lum(d2)[0] > M.THRESHOLD
    for d, flagged in ((d1, False), (d2, True)):
        c, r = (base, d) if sign > 0 else (d, base)
        rel = M.film_view(c, r, M.RELATIVE, 0, 2.0, *fns)[0]
        ab = M.film_view(c, r, M.ABSOLUTE, 0, 2.0, *fns)[0]
        k, other = (0, 1) if sign > 0 else (1, 0)
        assert rel[k] == f32(2.0) * M.lum(d)[0] and rel[other] == 0 and rel[2] == 0 and rel[3] == 0
        assert ab[k] == (1.0 if flagged else 0.0) and ab[other] == 0 and ab[2] == 0 and ab[3] == 0


def test_unorm8_rounds_to_nearest_and_maps_nan_to_zero():
    v = _px([0.5 / 255, 1.49 / 255, np.nan, 2.0], [-1, 254.5 / 255, np.inf, 1.0])
    assert np.array_equal(M.unorm8(v), np.array([[1, 1, 0, 255], [0, 255, 255, 255]], np.uint8))


def test_error_model_skips_non_finite_pixels():
    c = _px([1, 1, 1, 1], [np.nan, 0, 0, 1], [2, -1, 1, 1])
    r = _px([1, 1, 1, 1], [1, 1, 1, 1], [1, 1, 1, 1])
    e = M.film_error(c, r)
    assert e["pixels"] == 3 and e["nonfinite"] == 1 and e["negative"] == 1
    assert e["mse"] == pytest.approx((1 + 4) / 6) and e["lum_below"] == 0 and e["lum_above"] == 1
