"""The denoiser of DESIGN §13 in float64 numpy: the statement csrc/kernels_denoise.cuh is held to.

Non-local means on the colour with a dual-buffer variance estimate (Rousselle, Knaus, Zwicker 2012), combined with feature weights on the
normal and albedo guides by the minimum of the weights (Rousselle, Manzi, Zwicker 2013).  Arrays are (H, W, C) in one row order (the filter is
symmetric under a mirror, so the film's y-flipped storage order does not change it).
"""
import numpy as np

R = 10       # window radius
F = 3        # patch radius
KC = 0.45    # colour: k_c
ALPHA = 1.0
EPS = 1e-10
KF = 0.6     # features: k_f
TAU = 1e-3


def variance_of_mean(camera, half, counts):
    """Var(F) per channel from F (the mean of n samples) and H (the mean of the h = ceil(n / 2) even-indexed samples): the odd mean is
    O = (n F - h H) / (n - h) and Var = (H - O)^2 h (n - h) / n^2."""
    n = np.asarray(counts, np.float64)[..., None]
    h = np.ceil(n / 2.0)
    m = n - h
    f = np.asarray(camera, np.float64)[..., :3]
    hh = np.asarray(half, np.float64)[..., :3]
    odd = (n * f - h * hh) / m
    return (hh - odd) ** 2 * h * m / (n * n)


def box3(v):
    """3 x 3 box mean, clamped at the edge"""
    h, w = v.shape[:2]
    p = np.pad(v, ((1, 1), (1, 1), (0, 0)), mode="edge")
    return sum(p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w] for dy in (-1, 0, 1) for dx in (-1, 0, 1)) / 9.0


def _finite_or_zero(g):
    g = np.asarray(g, np.float64)[..., :3]
    return np.where(np.isfinite(g), g, 0.0)


def guide_inv_scale(g):
    """1 / (k_f^2 max(tau, |grad g|^2)), central differences clamped at the edge"""
    h, w = g.shape[:2]
    p = np.pad(g, ((1, 1), (1, 1), (0, 0)), mode="edge")
    gx = 0.5 * (p[1:1 + h, 2:2 + w] - p[1:1 + h, 0:w])
    gy = 0.5 * (p[2:2 + h, 1:1 + w] - p[0:h, 1:1 + w])
    g2 = (gx ** 2).sum(-1) + (gy ** 2).sum(-1)
    return 1.0 / (KF * KF * np.maximum(TAU, g2))


def _box_sum(a, k):
    """sums over every k x k window of a 2-D array (valid part); direct sums, no running sum whose cancellation would mix far-off terms in"""
    h, w = a.shape[0] - k + 1, a.shape[1] - k + 1
    rows = sum(a[:, j:j + w] for j in range(k))
    return sum(rows[i:i + h] for i in range(k))


def denoise(color, camera, half, counts, normals=None, albedo=None):
    """Returns (the filtered colour (H, W, 3), the smoothed variance of the mean (H, W, 3)).  A pixel whose colour or variance is not finite is
    copied through and weighs 0 as a neighbour; None guides (or zero guides) leave colour-only NL-means."""
    color = np.asarray(color, np.float64)[..., :3]
    counts = np.asarray(counts)
    assert counts.min() >= 2, "the variance estimate needs two samples per pixel"
    h, w = color.shape[:2]
    raw = variance_of_mean(camera, half, counts)
    ok = np.isfinite(color).all(-1) & np.isfinite(raw).all(-1)
    u = np.where(ok[..., None], color, 0.0)
    var = box3(np.where(ok[..., None], raw, 0.0))
    guides = []
    for g in (normals, albedo):
        if g is not None:
            g = _finite_or_zero(g)
            guides.append((g, guide_inv_scale(g)))
    P = R + F
    up = np.pad(u, ((P, P), (P, P), (0, 0)), mode="edge")
    vp = np.pad(var, ((P, P), (P, P), (0, 0)), mode="edge")
    ua, va = up[R:R + h + 2 * F, R:R + w + 2 * F], vp[R:R + h + 2 * F, R:R + w + 2 * F]
    # neighbour q = p + (dx, dy): zero-padded arrays with a validity mask (outside the film or not finite: skipped)
    qu = np.pad(u, ((R, R), (R, R), (0, 0)))
    qok = np.pad(ok, ((R, R), (R, R)))
    qg = [(np.pad(g, ((R, R), (R, R), (0, 0))), inv) for g, inv in guides]
    sw = np.zeros((h, w))
    su = np.zeros((h, w, 3))
    for dy in range(-R, R + 1):
        for dx in range(-R, R + 1):
            ub = up[R + dy:R + dy + h + 2 * F, R + dx:R + dx + w + 2 * F]
            vb = vp[R + dy:R + dy + h + 2 * F, R + dx:R + dx + w + 2 * F]
            term = (((ua - ub) ** 2 - ALPHA * (va + np.minimum(va, vb))) / (EPS + KC * KC * (va + vb))).mean(-1)
            dc = _box_sum(term, 2 * F + 1) / float((2 * F + 1) ** 2)
            wgt = np.exp(-np.maximum(0.0, dc))
            for (gq, inv), (g, _) in zip(qg, guides):
                d = ((g - gq[R + dy:R + dy + h, R + dx:R + dx + w]) ** 2).sum(-1) * inv
                wgt = np.minimum(wgt, np.exp(-d))
            wgt = wgt * qok[R + dy:R + dy + h, R + dx:R + dx + w]
            sw += wgt
            su += wgt[..., None] * qu[R + dy:R + dy + h, R + dx:R + dx + w]
    with np.errstate(invalid="ignore", divide="ignore"):
        out = su / sw[..., None]
    out = np.where(ok[..., None], out, color)
    return out, var
