"""float32 statement of the viewer's fragment shader (sources/raytracer/render.cxx:252-388) as k_film_view computes it (DESIGN §14), and the
float64 statement of etxb_film_error.  Test infrastructure: tests/test_view_model.py pins it on hand-computed pixels, tests/test_gpu_view.py
holds the device to it.

Every float32 operation is one numpy float32 operation, in the kernel's order, so each rounds as the device's does under -fmad=false.  exp and
pow are parameters: the oracle's portable functions (oracle_math) where the oracle is built, else float64 numpy rounded to float32.
"""
import numpy as np

f32 = np.float32
RESULT, ALPHA, ORIGINAL, REFERENCE, RELATIVE, ABSOLUTE = range(6)
TONEMAPPING, SRGB, SKIP_COLOR_CONVERSION = 1, 2, 4
LUM = (f32(0.2627), f32(0.6780), f32(0.0593))
THRESHOLD = f32(1.0) / f32(8192.0)
NAN_MARKER = np.array([123456.0, 0.0, 123456.0, 1.0], f32)
INF_MARKER = np.array([0.0, 123456.0, 123456.0, 1.0], f32)


def numpy_exp(x):
    return np.exp(np.asarray(x, np.float64)).astype(f32)


def numpy_pow(x, y):
    return np.power(np.asarray(x, np.float64), np.asarray(y, np.float64)).astype(f32)


def oracle_functions():
    """(exp, pow) of the oracle's parity build (oracle_math 2 and 4), or None where it is not built."""
    from oracle import oracle_py
    if not oracle_py.available("parity"):
        return None

    def exp(x):
        x = np.asarray(x, f32)
        return oracle_py.math_kat(2, x.ravel()).reshape(x.shape)

    def pow_(x, y):
        x = np.asarray(x, f32)
        y = np.broadcast_to(np.asarray(y, f32), x.shape)
        return oracle_py.math_kat(4, x.ravel(), y.ravel()).reshape(x.shape)

    return exp, pow_


def lum(v):
    """dot(v.xyz, lum) in float32, summed left to right."""
    return (v[..., 0] * LUM[0] + v[..., 1] * LUM[1]) + v[..., 2] * LUM[2]


def tone_curve(v, exposure, exp=numpy_exp):
    return f32(1.0) - exp(-f32(exposure) * v)


def linear_to_gamma(v, pow_=numpy_pow):
    return np.where(v <= f32(0.0031308), f32(12.92) * v, f32(1.055) * pow_(np.abs(v), f32(1.0) / f32(2.4)) - f32(0.055)).astype(f32)


def tonemap(v, options, exposure, exp=numpy_exp, pow_=numpy_pow):
    v = v.copy()
    if options & TONEMAPPING:
        v = tone_curve(v, exposure, exp)
    if options & SRGB:
        v[..., :3] = linear_to_gamma(v[..., :3], pow_)
    return v


def film_view(layer, reference, view, options, exposure, exp=numpy_exp, pow_=numpy_pow):
    """(N, 4) float32 -> (N, 4) float32: what the shader returns at each pixel."""
    c = np.asarray(layer, f32).reshape(-1, 4)
    e = f32(exposure)
    with np.errstate(all="ignore"):
        if view == ALPHA:
            return np.repeat(e * c[:, 3:4], 4, axis=1)
        if options & SKIP_COLOR_CONVERSION:
            return e * c
        r = None if reference is None else np.asarray(reference, f32).reshape(-1, 4)
        if view == RESULT:
            out = tonemap(c, options, exposure, exp, pow_)
        elif view == ORIGINAL:
            out = e * c
        elif view == REFERENCE:
            out = tonemap(r, options, exposure, exp, pow_)
        else:
            r_lum, c_lum = lum(r), lum(c)
            above, below = np.maximum(f32(0), r_lum - c_lum), np.maximum(f32(0), c_lum - r_lum)
            out = np.zeros_like(c)
            if view == RELATIVE:
                out[:, 0], out[:, 1] = e * above, e * below
            else:
                out[:, 0], out[:, 1] = (above > THRESHOLD).astype(f32), (below > THRESHOLD).astype(f32)
        # validate(): markers first, then the clamped value, returned without the view
        nan = np.isnan(c).any(1)
        inf = np.isinf(c).any(1) & ~nan
        neg = (c < 0).any(1) & ~nan & ~inf
        out[neg] = np.maximum(f32(0), c[neg])
        out[inf] = INF_MARKER
        out[nan] = NAN_MARKER
    return out.astype(f32)


def unorm8(v):
    """What an 8-bit UNORM target stores: clamp to [0, 1] (NaN -> 0), floor(255 x + 0.5)."""
    with np.errstate(invalid="ignore"):
        x = np.where(np.isnan(v), f32(0), np.clip(v, f32(0), f32(1))).astype(f32)
    return np.floor(x * f32(255) + f32(0.5)).astype(np.uint8)


def film_error(layer, reference):
    """etxb_film_error's fields (not `iterations`) in float64 numpy."""
    c = np.asarray(layer, f32).reshape(-1, 4)
    r = np.asarray(reference, f32).reshape(-1, 4)
    mean_rgb = r[:, :3].astype(np.float64).mean()
    eps = (0.01 * mean_rgb) ** 2
    finite = np.isfinite(c[:, :3]).all(1)
    cf, rf = c[finite], r[finite]
    c64, r64 = cf[:, :3].astype(np.float64), rf[:, :3].astype(np.float64)
    d2 = (c64 - r64) ** 2
    weights = np.array([0.2627, 0.6780, 0.0593])
    cl, rl = c64 @ weights, r64 @ weights
    with np.errstate(all="ignore"):
        r_lum, c_lum = lum(rf), lum(cf)
        above = np.maximum(f32(0), r_lum - c_lum) > THRESHOLD
        below = np.maximum(f32(0), c_lum - r_lum) > THRESHOLD
    return {
        "pixels": c.shape[0], "nonfinite": int((~finite).sum()), "negative": int((cf[:, :3] < 0).any(1).sum()),
        "lum_above": int(above.sum()), "lum_below": int(below.sum()),
        "mse": float(d2.mean()), "rel_mse": float((d2 / (r64 ** 2 + eps)).mean()),
        "mean_abs_lum": float(np.abs(cl - rl).mean()), "mean_lum": float(cl.mean()), "reference_mean_lum": float(rl.mean()),
    }
