"""The coarse preview in the oracle's restated Film (no GPU): the pixel offset's distribution, a numpy model of what the film does with each
path at pixel size s (camera blocks, per-pixel counts, the clamped repeated light splat of partial blocks), and the normalisation: a preview's
block means estimate the same image as the full-resolution render's."""
import numpy as np
import pytest
from scipy import stats

from etx_tracer_b200 import scenes, structs as S


@pytest.fixture(scope="module")
def preview_oracle():
    """the parity oracle with the Film pixel size (oracle/oracle_preview.cxx)"""
    from oracle import oracle_preview_py
    if not oracle_preview_py.available():
        pytest.skip("oracle/_ref/liboracle_preview_parity.so not built (run build() where /root/reference exists)")
    return oracle_preview_py


@pytest.mark.parametrize("size", [3, 8])
def test_offset_is_uniform_over_the_block(preview_oracle, size):
    iterations = np.arange(4096, dtype=np.uint32)
    for index in (0, 1, 77, 123457):
        dx, dy = preview_oracle.preview_offset(np.full(iterations.size, index, np.uint32), iterations, size)
        assert dx.max() < size and dy.max() < size
        counts = np.bincount(dx * size + dy, minlength=size * size)
        assert stats.chisquare(counts).pvalue > 1e-4, (index, counts)
        for v in (dx, dy):
            assert stats.chisquare(np.bincount(v, minlength=size)).pvalue > 1e-4
    # across the paths of one iteration as well
    dx, dy = preview_oracle.preview_offset(np.arange(4096, dtype=np.uint32), 5, size)
    assert stats.chisquare(np.bincount(dx * size + dy, minlength=size * size)).pvalue > 1e-4


def _coarse(W, H, s):
    return (W + s - 1) // s, (H + s - 1) // s


def _block_of_pixel(W, H, s):
    """path index of every film pixel (storage order: row 0 is the top, film y = H - 1 - row)"""
    dx, _ = _coarse(W, H, s)
    rows, cols = np.mgrid[0:H, 0:W]
    y = H - 1 - rows
    return (cols // s) + (y // s) * dx


@pytest.mark.parametrize("size", [3, 4, 8, 1024])
def test_numpy_model_against_the_oracle(preview_oracle, size):
    W, H = 13, 7
    sd = scenes.cornell_box(W, H, samples=16, spectral=False)
    dims = _coarse(W, H, size)
    paths = dims[0] * dims[1]
    block = _block_of_pixel(W, H, size)

    o = preview_oracle.Oracle(sd)
    o.set_film_pixel_size(size)
    o.begin(0)
    o.run(1)
    # one path per block; camera blocks are the tapped per-path values after the first iteration
    assert o.buffer(S.BUF_LIGHT_SAMPLER, np.uint32).size == paths
    value = o.buffer(S.BUF_CAMERA_GATHERED, np.float32).reshape(-1, 3)
    assert value.shape[0] == paths
    assert np.array_equal(o.film(S.FILM_CAMERA)[..., :3], value[block])
    # the light image: each splat lands on its block's pixels with clamped coordinates, so a pixel of the last column / row of a partial block
    # holds its block's value times the number of clamped positions that fold onto it
    light = o.film(S.FILM_LIGHT)[..., :3].astype(np.float64)
    rows, cols = np.mgrid[0:H, 0:W]
    y = H - 1 - rows
    mx = np.where(cols == W - 1, (cols // size) * size + size - cols, 1)
    my = np.where(y == H - 1, (y // size) * size + size - y, 1)
    origin = np.zeros((paths, 3))
    for b in range(paths):
        sel = (block == b) & (mx == 1) & (my == 1)
        if sel.any():
            origin[b] = light[sel][0]
            assert np.array_equal(light[sel], np.broadcast_to(light[sel][0], light[sel].shape))
    single = (mx * my == 1)
    full = origin[block] * (mx * my)[..., None]
    has_origin = np.array([((block == b) & single).any() for b in range(paths)])[block]
    assert light.any()
    # k repeated float adds against one product: the rounding grows with k (up to 1024 x 1024 folds at s = 1024)
    np.testing.assert_allclose(light[has_origin], full[has_origin], rtol=1e-5 if size <= 8 else 1e-2, atol=0)
    assert (mx * my > 1).any() == ((W % size != 0) or (H % size != 0))

    # the path tracer: per-pixel counts — every pixel one sample per iteration without a noise threshold
    o.set_integrator(S.INTEGRATOR_PT)
    o.pt_set_options(S.default_pt_options())
    o.begin(0)
    o.run(3)
    info = o.buffer(S.BUF_PIXEL_INFO, np.uint32)
    assert info.size == W * H and np.all((info & 0x3fffffff) == 3)
    assert o.buffer(S.BUF_CAMERA_SAMPLER, np.uint32).size == paths


def _block_mean(img, s):
    H, W = img.shape[:2]
    return img.reshape(H // s, s, W // s, s, -1).mean(axis=(1, 3))


def _rel_mse(a, b):
    return float(((a - b) ** 2).sum() / max((b ** 2).sum(), 1e-30))


def _windows(preview_oracle, sd, size, n, pt, layer):
    """the film after iterations [0, n) and the mean over [n, 2n) (= 2 F(2n) - F(n)), block-averaged"""
    o = preview_oracle.Oracle(sd)
    if pt:
        o.set_integrator(S.INTEGRATOR_PT)
        o.pt_set_options(S.default_pt_options())
    else:
        opts = S.default_vcm_options()
        opts["radius_decay"] = 1 << 30  # a constant radius: both windows estimate the same image
        o.set_options(opts)
    o.set_film_pixel_size(size)
    o.begin(0)
    o.run(n, threads=4)
    first = o.film(layer)[..., :3].astype(np.float64)
    o.run(n, threads=4)
    second = 2.0 * o.film(layer)[..., :3].astype(np.float64) - first
    return first, second


@pytest.mark.parametrize("pt", [False, True])
@pytest.mark.parametrize("size", [2, 4])
def test_preview_block_means_estimate_the_full_resolution_image(preview_oracle, size, pt):
    """The camera layer, which both integrators estimate per block.  (The VCM's light-tracing layer is not compared: in the reference's
    preview its mean is about s^2 times the full-resolution one — see DESIGN §12.)"""
    sd = scenes.cornell_box(16, 16, samples=256, spectral=False)
    layer = S.FILM_CAMERA
    n = 192
    full, _ = _windows(preview_oracle, sd, 1, n, pt, layer)
    p1, p2 = _windows(preview_oracle, sd, size, n, pt, layer)
    full_b, p1_b, p2_b = _block_mean(full, size), _block_mean(p1, size), _block_mean(p2, size)
    spread = _rel_mse(p1_b, p2_b)  # the preview's own run-to-run spread (its variance dominates: one path per block)
    err = _rel_mse(p1_b, full_b)
    # the path tracer's preview is unbiased; the VCM's, as the reference computes it, is not quite: its MIS weights take eta_vcm from the
    # reduced path count while the camera's importance counts W x H pixels (a few per cent darker at s = 2, DESIGN §12), so it is held to
    # DESIGN §3's Tier C factor of 2
    assert err < (1.0 if pt else 2.0) * spread, (err, spread)
    assert abs(p1_b.mean() / full_b.mean() - 1.0) < 0.1
    assert abs(p2_b.mean() / full_b.mean() - 1.0) < 0.1
