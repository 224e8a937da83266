"""The oracle's media export (oracle_medium: the reference's scene_medium.hxx compiled in place, and the oracle's restatement of
Raytracing::trace_transmittance over the shared BVH) against plain float64 models, on the scene and queries of medium_queries.py.  This
pins the side the GPU media test compares against.  Runs without a GPU.

It also pins what the reference does on purpose (kept, not fixed):
  - a heterogeneous sample reports its position and sampled_medium_t in the medium's local [0,1]^3 frame;
  - a heterogeneous sample_medium with max_t = kMaxFloat returns weight 0 (medium_intersects_bounds refuses that max_t);
  - heterogeneous transmittance ignores the absorption and scattering spectra (it tracks max_sigma x density only);
  - sample_phase_function draws the mirror image of the lobe phase_function evaluates.  The integrators call both with the ray's own
    direction first (dpt.cuh:166-172, kernels.cuh:420-422 and 867-869: phase_function(ray_d, w_o, g) after
    sample_phase_function(ray_d, g, rnd)); the sampled cos(ray_d, w_o) then follows 2 pi phase_function(ray_d, -w_o, g), that is the
    Henyey-Greenstein lobe of -g, while phase_function(ray_d, w_o, g) is the lobe of g.
"""
import numpy as np
import pytest

import medium_queries as mq
from etx_tracer_b200 import structs as S

K_SIGMA = 5.5
K_EPSILON = 1.192092896e-07
G3 = 1.0 + 2.0 * (3 * K_EPSILON * 0.5) / (1.0 - 3 * K_EPSILON * 0.5)
EPS = float(mq.K_RAY_EPSILON)
N_MC = 1 << 14

_cache = {}


@pytest.fixture(scope="module")
def medium_oracle(oracle_mod):
    if not oracle_mod.has_medium():
        pytest.skip("oracle/_ref predates oracle_medium (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


def _run(oracle_mod, q, reps=1, spectral=False):
    if spectral not in _cache:
        _cache[spectral] = mq.scene(spectral)
    o = oracle_mod.Oracle(_cache[spectral])
    r = o.medium(q, reps)
    o.close()
    return r


def _grid(name):
    return mq._HET[name][0]().astype(np.float64)


def _density(name, c):
    """trilinear interpolation of the grid (x fastest) at local coordinates c, 0 outside [0, 1)^3"""
    g = _grid(name)
    g = g / g.max()
    dz, dy, dx = g.shape
    c = np.asarray(c, np.float64)
    out = np.zeros(c.shape[0])
    inside = ((c >= 0) & (c < 1)).all(-1)
    p = np.stack([np.clip(c[:, a] * d - 0.5, 0, d - 1) for a, d in enumerate((dx, dy, dz))], -1)
    i0 = np.minimum(p.astype(np.int64), np.array([dx, dy, dz]) - 1)
    i1 = np.minimum(i0 + 1, np.array([dx, dy, dz]) - 1)
    f = p - np.floor(p)
    for corner in range(8):
        sel = [(corner >> a) & 1 for a in range(3)]
        idx = [np.where(sel[a], i1[:, a], i0[:, a]) for a in range(3)]
        w = np.prod([np.where(sel[a], f[:, a], 1.0 - f[:, a]) for a in range(3)], axis=0)
        out += w * g[idx[2], idx[1], idx[0]]
    return np.where(inside, out, 0.0)


def _local(name, o, d, max_t):
    lo, hi = mq.bounds(name)
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    p0, p1 = (o - lo) / (hi - lo), (o + d * max_t - lo) / (hi - lo)
    seg = np.linalg.norm(p1 - p0)
    return p0, (p1 - p0) / seg, seg


def _slab(p, d, max_t, inflate=True):
    """medium_bounds in float64, with its comparisons (a NaN slab leaves t_min / t_max as they were)"""
    t_min, t_max = 0.0, max_t
    with np.errstate(divide="ignore", invalid="ignore"):
        for a in range(3):
            t_near, t_far = (0.0 - p[a]) / d[a], (1.0 - p[a]) / d[a]
            if t_near > t_far:
                t_near, t_far = t_far, t_near
            if inflate:
                t_far *= G3
            t_min = t_near if t_near > t_min else t_min
            t_max = t_far if t_far < t_max else t_max
            if t_min > t_max:
                return False, t_min, t_max
    return True, t_min, t_max


def _optical_depth(name, p, d, t0, t1, n=20000):
    t = t0 + (np.arange(n) + 0.5) / n * (t1 - t0)
    return float(_density(name, p[None, :] + t[:, None] * d[None, :]).sum() * (t1 - t0) / n)


@pytest.mark.parametrize("name", mq.HETEROGENEOUS)
def test_bounds_follow_the_slab_model(medium_oracle, name):
    q, band = mq.make(None, name, False, seed=21)
    s = q["op"] == S.MEDIUM_BOUNDS
    q, band = q[s], band[s]
    r = _run(medium_oracle, q)[:, 0]
    fails = []
    for i in range(q.shape[0]):
        if q["max_t"][i] >= mq.K_MAX_FLOAT:
            if r["flag"][i] != 0:
                fails.append(f"{i}: max_t = kMaxFloat must not meet the bounds")
            continue
        p, d, seg = _local(name, q["origin"][i], q["direction"][i], float(q["max_t"][i]))
        hit, t_min, t_max = _slab(p, d, seg)
        if abs(t_max - t_min) < 1e-5 * max(1.0, abs(t_max)):
            continue  # a tangent or corner ray: float32 rounding decides
        if bool(r["flag"][i]) != hit:
            fails.append(f"{i} ({band[i]}): flag {r['flag'][i]} model {hit} t {t_min:.7g} {t_max:.7g}")
        elif hit and not (np.isclose(r["t_min"][i], t_min, rtol=1e-5, atol=1e-6) and np.isclose(r["t_max"][i], t_max, rtol=1e-5, atol=1e-6)):
            fails.append(f"{i} ({band[i]}): t {r['t_min'][i]:.7g} {r['t_max'][i]:.7g} model {t_min:.7g} {t_max:.7g}")
        # the local direction is a float32 difference of two local points over their distance: an ulp of each over the distance
        dir_atol = 2e-6 + 4.0 * 6e-8 * max(1.0, float(np.abs(p).max())) / seg
        if not np.allclose(r["pos"][i], p, atol=2e-6) or not np.allclose(r["dir"][i], d, atol=dir_atol):
            fails.append(f"{i} ({band[i]}): local ray {r['pos'][i]} {r['dir'][i]} model {p} {d}")
    assert not fails, "\n".join(fails[:12])


@pytest.mark.parametrize("name", mq.HETEROGENEOUS)
def test_density_is_trilinear(medium_oracle, name):
    q, band = mq.make(None, name, False, seed=22)
    s = q["op"] == S.MEDIUM_DENSITY
    q, band = q[s], band[s]
    r = _run(medium_oracle, q)[:, 0]
    model = _density(name, q["origin"].astype(np.float64))
    err = np.abs(r["value"][:, 0] - model)
    bad = np.flatnonzero(err > 1e-6)
    assert bad.size == 0, [(band[i], q["origin"][i], r["value"][i, 0], model[i]) for i in bad[:8]]
    top = (band == "top") & (q["origin"] == 1.0).any(-1)
    assert (r["value"][top, 0] == 0).all(), "a coordinate of exactly 1 lies outside the grid"


@pytest.mark.parametrize("name", ("fog", "absorber", "scatterer", "dense", "vacuum", "invalid"))
def test_homogeneous_transmittance_is_exponential(medium_oracle, name):
    q, band = mq.make(None, name, False, seed=23)
    s = (q["op"] == S.MEDIUM_TRANSMITTANCE) & (q["max_t"] < 1e30)
    q = q[s]
    r = _run(medium_oracle, q)[:, 0]
    sig = _sigma(name)[0] + _sigma(name)[1]
    model = np.exp(-sig[None, :] * q["max_t"].astype(np.float64)[:, None])
    assert np.allclose(r["value"], model, rtol=1e-5, atol=1e-30), (r["value"][:4], model[:4])
    assert (r["seed_start"] == r["seed_end"]).all(), "homogeneous transmittance draws nothing"


def _sigma(name):
    """(absorption, scattering) rgb of a medium of medium_queries.scene"""
    table = {"fog": ((0.1,) * 3, (0.9,) * 3), "absorber": ((0.5, 2.0, 0.0), (0.0,) * 3), "scatterer": ((0.0,) * 3, (1.5, 1.0, 0.5)),
             "dense": ((2000.0,) * 3, (8000.0,) * 3), "vacuum": ((0.0,) * 3, (0.0,) * 3), "invalid": ((0.0,) * 3, (0.0,) * 3)}
    if name in table:
        return tuple(np.array(v, np.float64) for v in table[name])
    return tuple(np.array(v, np.float64) for v in (mq._HET[name][3], mq._HET[name][2]))


@pytest.mark.parametrize("name", ("cloud", "grid1", "grid235", "ones"))
def test_ratio_tracking_is_unbiased(medium_oracle, name):
    q = mq.distribution_queries(name, False, seed=24)
    q = q[q["op"] == S.MEDIUM_TRANSMITTANCE]
    r = _run(medium_oracle, q, N_MC)[0]
    p, d, seg = _local(name, q["origin"][0], q["direction"][0], float(q["max_t"][0]))
    _, t0, t1 = _slab(p, d, seg, inflate=False)
    expected = np.exp(-mq._HET[name][4] * _optical_depth(name, p, d, t0, t1))
    v = r["value"][:, 0].astype(np.float64)
    assert (r["value"][:, 0] == r["value"][:, 1]).all(), "heterogeneous transmittance is grey whatever the spectra"
    sigma = v.std() / np.sqrt(v.size)
    assert abs(v.mean() - expected) <= K_SIGMA * sigma + 1e-4, (v.mean(), expected, sigma)
    if name == "ones":
        assert (v == 0).any(), "Russian roulette never fired on the all-ones grid"


@pytest.mark.parametrize("name", ("cloud", "grid1", "grid235", "ones"))
def test_delta_tracking_scatters_with_the_optical_depth(medium_oracle, name):
    q = mq.distribution_queries(name, False, seed=25)
    q = q[q["op"] == S.MEDIUM_SAMPLE]
    r = _run(medium_oracle, q, N_MC)[0]
    p, d, seg = _local(name, q["origin"][0], q["direction"][0], float(q["max_t"][0]))
    _, t0, t1 = _slab(p, d, seg, inflate=False)
    p_scatter = 1.0 - np.exp(-mq._HET[name][4] * _optical_depth(name, p, d, t0, t1))
    scattered = r["t"] > 0
    f = scattered.mean()
    assert abs(f - p_scatter) <= K_SIGMA * np.sqrt(p_scatter * (1 - p_scatter) / scattered.size) + 1e-4, (f, p_scatter)
    # the reference's own frame: the position and t of a scattering event are local, t counted from where the ray enters the bounds
    pos = r["pos"][scattered].astype(np.float64)
    local = p[None, :] + (r["t"][scattered].astype(np.float64) + t0)[:, None] * d[None, :]
    assert np.allclose(pos, local, atol=1e-5), "a heterogeneous sample reports its position in the medium's local frame"


def test_heterogeneous_reference_behaviour(medium_oracle):
    q, band = mq.make(None, "cloud", False, seed=26)
    r = _run(medium_oracle, q)[:, 0]
    far = (q["op"] == S.MEDIUM_SAMPLE) & (band == "max_float")
    assert far.any() and (r["value"][far] == 0).all() and (r["t"][far] == 0).all(), "max_t = kMaxFloat gives weight 0"
    zero = mq.make(None, "zero_sigma", False, seed=26)[0]
    rz = _run(medium_oracle, zero)[:, 0]
    tr = zero["op"] == S.MEDIUM_TRANSMITTANCE
    assert (rz["value"][tr] == 1).all() and (rz["seed_start"] == rz["seed_end"]).all(), "max_sigma = 0: transmittance 1, no draws"


def free_flight_fails(name, throughput, max_t, rec, weight_rtol=2e-5):
    """sample_medium records `rec` of one homogeneous query (RGB) against the float64 model: the share that passes max_t, the distance
    distribution (KS against the channel mixture of exponentials, with the kRayEpsilon redraw) and each weight's closed form at its t
    (the pdf of the last channel draw: pc tr sigma_t, or pc tr past max_t).  Returns the failures."""
    a, s = _sigma(name)
    ext = a + s
    albedo = np.where(ext > 0, s / np.where(ext > 0, ext, 1.0), 0.0)
    pc = albedo * np.array(throughput, np.float64)
    pc = np.full(3, 1.0 / 3.0) if (pc <= K_EPSILON).all() else pc / pc.sum()  # sample_spectrum_component's is_zero branch
    norm = (pc * np.exp(-ext * EPS)).sum()  # the loop redraws t < kRayEpsilon
    t = rec["t"].astype(np.float64)
    sampled = t > 0
    p_pass = (pc * np.exp(-ext * max_t)).sum() / norm
    fails = []
    if abs((~sampled).mean() - p_pass) > K_SIGMA * np.sqrt(p_pass * (1 - p_pass) / t.size) + 1e-12:
        fails.append(f"{name}: share past max_t {(~sampled).mean():.5f}, model {p_pass:.5f}")
    ts = np.sort(t[sampled])
    if ts.size > 100:
        cdf = ((pc[None, :] * (np.exp(-ext * EPS)[None, :] - np.exp(-ext[None, :] * ts[:, None]))).sum(-1) / norm) / (1.0 - p_pass)
        ks = np.max(np.maximum(np.arange(1, ts.size + 1) / ts.size - cdf, cdf - np.arange(ts.size) / ts.size))
        if ks > 1.63 / np.sqrt(ts.size) * 1.2:  # KS at alpha 1e-2, with margin
            fails.append(f"{name}: KS distance {ks:.4g} of {ts.size} free-flight distances")
    tt = np.where(sampled, t, max_t)
    tr = np.exp(-ext[None, :] * tt[:, None])
    pdf = np.where(sampled[:, None], pc[None, :] * tr * ext[None, :], pc[None, :] * tr).sum(-1)
    w = np.where(sampled[:, None], tr * s[None, :], tr) / pdf[:, None]
    if not np.allclose(rec["value"], w, rtol=weight_rtol, atol=1e-30):
        fails.append(f"{name}: weights off the closed form by {np.nanmax(np.abs(rec['value'] / w - 1)):.3g} relative")
    return fails


@pytest.mark.parametrize("name,throughput", [("fog", (1.0, 1.0, 1.0)), ("scatterer", (1.0, 1.0, 1.0)), ("scatterer", (0.3, 1.0, 0.6)),
                                             ("absorber", (1.0, 1.0, 1.0)), ("dense", (0.3, 1.0, 0.6))])
def test_homogeneous_free_flight(medium_oracle, name, throughput):
    max_t = 2.0 if name != "dense" else 1e-3
    q = np.zeros(1, S.MEDIUM_QUERY)
    q["op"], q["medium"], q["seed"], q["max_t"] = S.MEDIUM_SAMPLE, mq.medium_index(name), 77, max_t
    q["direction"], q["throughput"] = (0.0, 0.0, 1.0), throughput
    r = _run(medium_oracle, q, N_MC * 4)[0]
    fails = free_flight_fails(name, throughput, max_t, r)
    assert not fails, fails


def _hg(mu, g):
    return (1.0 - g * g) / (4.0 * np.pi * (1.0 + g * g - 2.0 * g * mu) ** 1.5)


@pytest.mark.parametrize("g", mq.PHASE_G)
def test_phase_function_integrates_to_one(medium_oracle, g):
    # cos between w_i and w_o on a grid dense at both poles
    x = np.concatenate([-1.0 + np.geomspace(1e-9, 1.0, 6000), 1.0 - np.geomspace(1e-9, 1.0, 6000)[::-1]])
    mu = np.unique(x)
    q = np.zeros(mu.size, S.MEDIUM_QUERY)
    q["op"], q["g"], q["direction"] = S.MEDIUM_PHASE, g, (0.0, 0.0, 1.0)
    q["w_o"] = np.stack([np.sqrt(np.maximum(0.0, 1 - mu * mu)), np.zeros_like(mu), mu], -1)
    r = _run(medium_oracle, q)[:, 0]
    v = r["value"][:, 0].astype(np.float64)
    mu = q["w_o"][:, 2].astype(np.float64)
    integral = 2.0 * np.pi * np.trapezoid(v, mu)
    # the reference forms d = 1 + g^2 - 2 g cos in float32: at the peak of |g| = 0.999, d = (1 - |g|)^2 = 1e-6 carries an absolute
    # rounding of a few ulps of 2 (2.4e-7 each), and the value goes as d^-1.5.  Measured: the integral is 0.9654 at g = +-0.999 (the
    # oracle, on this grid); 4e-6 from 1 for |g| <= 0.9.  The bounds are about twice that.
    assert abs(integral - 1.0) < (0.07 if abs(g) > 0.99 else 2e-3), integral
    g32 = float(np.float32(g))
    d = 1.0 + g32 * g32 - 2.0 * g32 * mu
    # and 1 - g^2 a few ulps of 1 over its value
    assert (np.abs(v / _hg(mu, g32) - 1.0) <= 1e-5 + 4 * 6e-8 / (1.0 - g32 * g32) + 1.5 * 3 * 2.4e-7 / d).all()


@pytest.mark.parametrize("g", (0.0, 5e-4, 1e-3, 0.3, -0.7, 0.9, 0.999))
def test_phase_sampling_follows_the_mirrored_lobe(medium_oracle, g):
    """module docstring: the sampled cos(w_i, w_o) follows 2 pi phase_function(w_i, -w_o, g) under the integrators' convention"""
    n = 1 << 17
    rng = np.random.default_rng(31)
    q = np.zeros(n, S.MEDIUM_QUERY)
    q["op"], q["g"] = S.MEDIUM_PHASE, g
    w = rng.normal(size=(n, 3))
    q["direction"] = w / np.linalg.norm(w, axis=1, keepdims=True)
    q["rnd"] = rng.random((n, 2))
    r = _run(medium_oracle, q)[:, 0]
    d = r["dir"].astype(np.float64)
    assert np.allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-5)
    # a float32 cos_theta may round past 1 (sin_theta is then clamped to 0 and |w_o| = cos_theta): clip to the histogram's range
    mu = np.clip((d * q["direction"]).sum(-1), -1.0, 1.0)
    edges = np.linspace(-1.0, 1.0, 33)
    counts = np.histogram(mu, edges)[0].astype(np.float64)

    def cdf(m, gg):  # of 2 pi HG(m, gg) on [-1, 1]
        if abs(gg) < 1e-3:
            return (m + 1.0) / 2.0
        return (1.0 - gg * gg) / (2.0 * gg) * (1.0 / np.sqrt(1.0 + gg * gg - 2.0 * gg * m) - 1.0 / (1.0 + gg))

    p_mirror = np.diff(cdf(edges, -g))
    sigma = np.sqrt(n * p_mirror * (1 - p_mirror))
    assert (np.abs(counts - n * p_mirror) <= K_SIGMA * sigma + 2).all(), (counts[:4], n * p_mirror[:4])
    if abs(g) >= 0.3:
        p_same = np.diff(cdf(edges, g))
        assert (np.abs(counts - n * p_same) > K_SIGMA * sigma + 2).any(), "the sampled lobe is the evaluated one"


def _tri_hits(sd, o, d, t_max):
    """every triangle the segment o + t d, t in (kRayEpsilon, t_max), crosses: float64 Moller-Trumbore over all triangles"""
    v = np.concatenate([a["pos"] for a in sd.vertices]).astype(np.float64)
    tris = np.concatenate(sd.triangles)
    p0, p1, p2 = v[tris["i"][:, 0]], v[tris["i"][:, 1]], v[tris["i"][:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    h = np.cross(d[None, :], e2)
    a = (e1 * h).sum(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        f = 1.0 / a
        s = o[None, :] - p0
        u = f * (s * h).sum(-1)
        qv = np.cross(s, e1)
        vv = f * (qv * d[None, :]).sum(-1)
        t = f * (e2 * qv).sum(-1)
    hit = (np.abs(a) > 1e-12) & (u >= 0) & (vv >= 0) & (u + vv <= 1) & (t > EPS) & (t < t_max)
    idx = np.flatnonzero(hit)
    return idx[np.argsort(t[idx])], t, tris


def test_segment_crossings_follow_brute_force(medium_oracle):
    """the restated trace_transmittance: occluded by an opaque surface or by a 63rd Boundary crossing; otherwise (RGB, homogeneous media
    only) the product of exp(-sigma dt) over the media the crossings switch between"""
    sd = mq.scene(False)
    q, band = mq.make(sd, "segment", False, seed=27)
    r = _run(medium_oracle, q, 4)
    mats = sd.materials
    fails = []
    for i in range(q.shape[0]):
        o, e = q["origin"][i].astype(np.float64), q["end"][i].astype(np.float64)
        length = np.linalg.norm(e - o)
        if length * length <= EPS:
            if not (r["value"][i] == 1).all() or (r["seed_start"][i] != r["seed_end"][i]).any():
                fails.append(f"{i} degenerate: {r['value'][i, 0]}")
            continue
        d = (e - o) / length
        t_max = length - max(EPS, length * EPS)
        hits, t, tris = _tri_hits(sd, o, d, t_max)
        cls = np.array([int(mats[tris["material_index"][k]]["cls"][0]) for k in hits], dtype=np.int64)
        keep = cls != S.MAT_VOID
        hits, cls = hits[keep], cls[keep]
        occluded = (cls != S.MAT_BOUNDARY).any() or (cls.size >= 63)
        v = r["value"][i]
        if occluded:
            if not (v == 0).all():
                fails.append(f"{i} ({band[i]}): {cls.size} crossings, occluded, value {v[0]}")
            continue
        if (v == 0).all() and band[i] != "nested":
            fails.append(f"{i} ({band[i]}): {cls.size} crossings, not occluded, value 0")
        media, cur, last = [], int(q["medium"][i]), 0.0
        for k in hits:
            media.append((cur, t[k] - last))
            m = mats[tris["material_index"][k]]
            entering = float(np.dot(tris["geo_n"][k], d)) < 0
            cur, last = int(m["int_medium"][0] if entering else m["ext_medium"][0]), t[k]
        media.append((cur, t_max - last))
        if any(m != S.INVALID and mq.MEDIA[m] in mq.HETEROGENEOUS for m, _ in media):
            continue
        model = np.ones(3)
        for m, dt in media:
            if m != S.INVALID:
                model *= np.exp(-(sum(_sigma(mq.MEDIA[m]))) * dt)
        if not np.allclose(v, model[None, :], rtol=2e-4, atol=1e-30):
            fails.append(f"{i} ({band[i]}): {cls.size} crossings, value {v[0]} model {model}")
    assert not fails, "\n".join(fails[:12])
    expected = {"crossings_62": 1, "crossings_63": 0}
    for b, nonzero in expected.items():
        assert ((r["value"][band == b] != 0).any(-1).all(-1) == bool(nonzero)).all(), b
