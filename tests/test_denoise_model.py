"""Properties of the float64 denoiser model (tests/denoise_model.py, DESIGN §13) that the device kernels are held to in test_gpu_denoise.py."""
import numpy as np

import denoise_model as M


def _noisy(rng, h, w, n, sigma=0.1):
    """a smooth image, n i.i.d. samples per pixel around it; returns (F, H, counts, clean)"""
    y, x = np.mgrid[0:h, 0:w]
    clean = np.stack([0.5 + 0.3 * np.sin(x / 5.0), 0.4 + 0.2 * np.cos(y / 7.0), 0.3 + 0.001 * x * y], -1)
    s = clean[None] + sigma * rng.standard_normal((n, h, w, 3))
    return s.mean(0), s[0::2].mean(0), np.full((h, w), n, np.uint32), clean


def test_constant_image_is_unchanged():
    c = np.full((19, 23, 3), 0.37)
    out, var = M.denoise(c, c, c, np.full((19, 23), 8))
    assert np.array_equal(var, np.zeros_like(var))
    np.testing.assert_allclose(out, c, rtol=1e-12)


def test_zero_variance_leaves_the_image_unchanged():
    rng = np.random.default_rng(1)
    u = rng.uniform(0.0, 1.0, (21, 17, 3))
    out, _ = M.denoise(u, u, u, np.full((21, 17), 5))
    np.testing.assert_allclose(out, u, rtol=0, atol=1e-12)


def test_dual_buffer_variance_is_unbiased():
    """E[(H - O)^2 h (n - h) / n^2] = sigma^2 / n for i.i.d. samples, odd and even n; each estimate is sigma^2 / n times a chi-square with one
    degree of freedom, so the mean over N pixels has a standard error of sqrt(2 / N) sigma^2 / n"""
    rng = np.random.default_rng(2)
    sigma = 0.3
    for n in (2, 3, 7, 16):
        s = sigma * rng.standard_normal((n, 200, 200, 3))
        est = M.variance_of_mean(s.mean(0), s[0::2].mean(0), np.full((200, 200), n)).mean()
        truth = sigma * sigma / n
        se = np.sqrt(2.0 / (200 * 200 * 3)) * truth
        assert abs(est - truth) < 4.0 * se, (n, est, truth, se)


def test_zero_guides_equal_colour_only_nl_means():
    rng = np.random.default_rng(3)
    f, hh, n, _ = _noisy(rng, 24, 20, 6)
    zero = np.zeros_like(f)
    a, _ = M.denoise(f, f, hh, n)
    b, _ = M.denoise(f, f, hh, n, normals=zero, albedo=zero)
    assert np.array_equal(a, b)


def test_filter_reduces_the_error_and_respects_a_guide_edge():
    """the noise of a smooth image goes down; an albedo edge keeps the two sides of a colour step apart"""
    rng = np.random.default_rng(4)
    f, hh, n, clean = _noisy(rng, 32, 32, 8, sigma=0.2)
    out, _ = M.denoise(f, f, hh, n)
    assert ((out - clean) ** 2).mean() < 0.3 * ((f - clean) ** 2).mean()
    step = np.zeros((32, 32, 3))
    step[:, 16:] = 1.0
    s = step[None] + 0.05 * rng.standard_normal((8, 32, 32, 3))
    f, hh = s.mean(0), s[0::2].mean(0)
    guided, _ = M.denoise(f, f, hh, n, albedo=step)
    assert np.abs(guided[:, :15] - step[:, :15]).max() < 0.1 and np.abs(guided[:, 17:] - step[:, 17:]).max() < 0.1


def test_non_finite_pixels_pass_through_and_weigh_nothing():
    rng = np.random.default_rng(5)
    f, hh, n, _ = _noisy(rng, 18, 22, 4)
    bad = f.copy()
    bad[3, 4] = [np.nan, 0.5, 0.5]
    bad[10, 11, 2] = np.inf
    out, _ = M.denoise(bad, f, hh, n)
    assert np.isnan(out[3, 4, 0]) and np.array_equal(out[3, 4, 1:], bad[3, 4, 1:])
    assert np.array_equal(out[10, 11], bad[10, 11])
    mask = np.ones((18, 22), bool)
    mask[3, 4] = mask[10, 11] = False
    assert np.isfinite(out[mask]).all()
    # what the copied-through pixels hold does not reach their neighbours
    other = bad.copy()
    other[3, 4] = [-np.inf, 1e30, 7.0]
    other[10, 11] = np.nan
    out2, _ = M.denoise(other, f, hh, n)
    assert np.array_equal(out[mask], out2[mask])
