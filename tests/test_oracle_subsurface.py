"""The oracle's subsurface export (oracle_subsurface: the reference's scene_bssrdf_subsurface.hxx and subsurface::gather compiled in place,
and the oracle's restatement of Raytracing::trace_material / continuous_trace over the shared BVH) against plain float64 models, on the
scenes and queries of subsurface_queries.py.  This pins the side the GPU subsurface test compares against.  Runs without a GPU.

It also pins what the reference does on purpose (kept, not fixed):
  - sample_s_r(1 - 2^-24) is exactly kMaxRadius in float32, so that probe is empty (sampled_radius >= r_max);
  - an empty probe (origin 0, direction 0) is still traced; the traversal ends and records nothing, even on a triangle through the
    world origin, because the triangle test's determinant is exactly 0 for a zero direction;
  - probes 1 and 2 of a gather on an axis-aligned plane travel in its plane and find nothing (determinant exactly 0).
"""
import numpy as np
import pytest
from scipy import integrate, stats

import subsurface_queries as sq
from etx_tracer_b200 import structs as S

K_SIGMA = 5.5
_cache = {}


@pytest.fixture(scope="module")
def ss_oracle(oracle_mod):
    if not oracle_mod.has_subsurface():
        pytest.skip("oracle/_ref predates oracle_subsurface (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


def _scene(case, spectral=False):
    if (case, spectral) not in _cache:
        _cache[(case, spectral)] = sq.scene(case, spectral)
    return _cache[(case, spectral)]


def _run(oracle_mod, case, q, reps=1, spectral=False):
    sd, _ = _scene(case, spectral)
    o = oracle_mod.Oracle(sd)
    r = o.subsurface(q, reps)
    o.close()
    return r


def _query(op, **fields):
    q = np.zeros(1, S.SUBSURFACE_QUERY)
    q["op"], q["seed"], q["material"], q["t_min"], q["t_max"], q["dir"] = op, 7, S.INVALID, sq.K_RAY_EPSILON, sq.K_MAX_FLOAT, (0, -1, 0)
    for k, v in fields.items():
        q[k] = v
    return q


def remap_model(color, distance):
    """remap_channel in float64"""
    a, b, c, d = 1.826052378200, 4.985111943850 + 0.12735595943800, 1.096861024240, 0.496310210422
    e, f = 4.231902997010 + 0.00310603949088, 2.406029994080
    color = np.maximum(0.0, color)
    blend = color ** 0.25
    albedo = (1 - blend) * a * np.arctan(b * color) ** c + blend * d * np.arctan(e * color) ** f
    albedo = np.clip(albedo, 0.0, 1.0 - float(sq.K_EPSILON))
    extinction = 1.0 / np.maximum(distance, 1.0 / 1024.0)
    return albedo, extinction, extinction * albedo


def s_r_model(rnd):
    """sample_s_r in float64 (with the reference's clamps)"""
    rnd = np.asarray(rnd, np.float64)
    lo = np.minimum(4.0 * rnd, 1.0 - float(sq.K_EPSILON))
    hi = np.minimum((rnd - 0.25) / 0.75, 1.0 - float(sq.K_EPSILON))
    return np.where(rnd < 0.25, -np.log1p(-lo), -3.0 * np.log1p(-hi))


def eval_model(d, r):
    """ss_evaluate in float64 for distance d"""
    r = np.maximum(r, float(sq.K_EPSILON))
    return (np.exp(-r / (3 * d)) + np.exp(-r / d)) / np.maximum(8 * np.pi * d * r, float(sq.K_EPSILON))


def _distances(sd, name):
    m = sd.materials[sd.material_names[name]]
    return sd.spectra[int(m["subsurface"]["spectrum_index"][0])]["integrated"][0].astype(np.float64)


def _color(sd, name):
    m = sd.materials[sd.material_names[name]]
    return sd.spectra[int(m["scattering"]["spectrum_index"][0])]["integrated"][0].astype(np.float64)


def test_remap_matches_float64(ss_oracle):
    sd, info, q, band, _ = sq.make("remap", False, 11)
    m = q["op"] == S.SUBSURFACE_REMAP
    r = _run(ss_oracle, "remap", q[m])[:, 0]
    al, ex, sc = remap_model(q["color"][m].astype(np.float64), q["distances"][m].astype(np.float64))
    np.testing.assert_allclose(r["albedo"], al, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(r["extinction"], ex, rtol=1e-7)
    np.testing.assert_allclose(r["scattering"], sc, rtol=3e-6, atol=1e-7)
    neg = q["color"][m][:, 0] <= 0
    assert (r["albedo"][neg, 0] == 0).all()
    # colors from about 0.95 to 1.1 reach the clamp at 1 - kEpsilon; 2 gives 0.922
    assert (r["albedo"] <= 1 - sq.K_EPSILON).all() and (r["albedo"][q["color"][m][:, 0] == 1, 0] == np.float32(1) - sq.K_EPSILON).all()
    assert (r["extinction"][q["distances"][m][:, 0] <= 2.0 ** -11, 0] == 1024.0).all()


def test_sample_s_r_bands_and_distribution(ss_oracle):
    rnd = np.array(list(sq.RND_BANDS.values()), np.float32)
    q = np.concatenate([_query(S.SUBSURFACE_PROFILE, triangle=0, rnd=x, radius=1.0, normal=(0, 1, 0)) for x in rnd])
    r = _run(ss_oracle, "remap", q)[:, 0]
    np.testing.assert_allclose(r["s_r"], s_r_model(rnd), rtol=2e-6)
    assert r["s_r"][0] == 0.0
    # the clamp: 3 logf(1 / kEpsilon) is the float32 value of kMaxRadius, so a probe there is empty (sampled_radius >= r_max)
    assert r["s_r"][list(sq.RND_BANDS).index("clamp")] == sq.K_MAX_RADIUS
    # KS test over 2^16 uniform draws against the mixture 0.25 Exp(1) + 0.75 Exp(1/3)
    n = 1 << 16
    u = ((np.arange(n) + np.random.default_rng(5).random(n)) / n).astype(np.float32)
    qq = np.repeat(q[:1], n)
    qq["rnd"] = u
    s = _run(ss_oracle, "remap", qq)[:, 0]["s_r"].astype(np.float64)
    cdf = lambda x: 1.0 - 0.25 * np.exp(-x) - 0.75 * np.exp(-x / 3.0)
    assert stats.kstest(s, cdf).pvalue > 1e-4
    # pointwise against the same steps with float32 roundings up to the logarithm (a float32 1 - x near 1 carries the error)
    f = np.float32
    x = np.where(u < f(0.25), np.minimum(f(4) * u, f(1) - sq.K_EPSILON), np.minimum((u - f(0.25)) / f(0.75), f(1) - sq.K_EPSILON)).astype(f)
    model = np.where(u < f(0.25), 1.0, 3.0) * np.log((f(1) / (f(1) - x)).astype(np.float64))
    np.testing.assert_allclose(s, model, rtol=2e-6, atol=1e-12)


def test_profile_integrates_to_one(ss_oracle):
    """2 pi r evaluate(r) over [0, r_max] is 1 - 0.75 exp(-kMaxRadius / 3) = 1 - 8.9e-8 per channel"""
    sd, info = _scene("plane")
    d = _distances(sd, "cb_grey")
    tri = info["cb_grey"][1]
    for c in range(3):
        r_max = float(d[c] * sq.K_MAX_RADIUS)
        radii = np.linspace(0.0, r_max, 8193)
        radii[0] = float(sq.K_EPSILON)  # 2 pi r evaluate(r) tends to 1 / (2 d) at 0; [0, kEpsilon] holds 1e-7 d of the integral
        q = np.repeat(_query(S.SUBSURFACE_PROFILE, triangle=tri, u=0.3, v=0.3, rnd=0.5, normal=(0, 1, 0)), radii.size)
        q["radius"] = radii
        e = _run(ss_oracle, "plane", q)[:, 0]["eval"][:, c].astype(np.float64)
        np.testing.assert_allclose(e, eval_model(d[c], radii), rtol=2e-6)
        total = integrate.simpson(2 * np.pi * radii * e, x=radii)
        expected = 1.0 - 0.75 * np.exp(-float(sq.K_MAX_RADIUS) / 3.0) - 0.25 * np.exp(-float(sq.K_MAX_RADIUS))
        assert abs(expected - (1.0 - 8.9e-8)) < 1e-9
        assert abs(total - expected) < 2e-6, (c, total)


def _tri_hits(sd, o, d, tmin, tmax, material):
    """float64 brute force over every triangle: (t, tri) of the candidates of `material` (None: any non-Void), sorted by t"""
    t = np.concatenate(sd.triangles)
    v = np.concatenate(sd.vertices)["pos"].astype(np.float64)
    p = v[t["i"]]
    e1, e2 = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    pv = np.cross(d, e2)
    det = (e1 * pv).sum(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / det
        tv = o - p[:, 0]
        u = (tv * pv).sum(-1) * inv
        qv = np.cross(tv, e1)
        vv = (qv * d).sum(-1) * inv
        tt = (e2 * qv).sum(-1) * inv
    with np.errstate(invalid="ignore"):
        ok = (np.abs(det) > 1e-12) & (u >= 0) & (u <= 1) & (vv >= 0) & (u + vv <= 1) & (tt > tmin) & (tt < tmax)
    mats = t["material_index"]
    void = np.array([int(sd.materials[int(k)]["cls"][0]) == S.MAT_VOID for k in mats])
    ok &= ~void if material is None else (mats == material)
    idx = np.flatnonzero(ok)
    return sorted(zip(tt[idx], idx))


@pytest.mark.parametrize("case", [c for c in sq.GEOMETRIES if c != "stack"])
def test_ray_queries_match_brute_force(ss_oracle, case):
    sd, info, q, band, _ = sq.make(case, False, 21)
    m = q["op"] <= S.SUBSURFACE_CONTINUOUS_TRACE
    q, band = q[m], band[m]
    r = _run(ss_oracle, case, q)[:, 0]
    for k in range(q.shape[0]):
        o, d = q["origin"][k].astype(np.float64), q["dir"][k].astype(np.float64)
        mat = None if q["material"][k] == S.INVALID else int(q["material"][k])
        cand = _tri_hits(sd, o, d, float(q["t_min"][k]), float(q["t_max"][k]), mat)
        # coincident copies of other materials make "any" ambiguous about which triangle: compare the distances there
        if q["op"][k] == S.SUBSURFACE_TRACE_MATERIAL:
            assert r["count"][k] == (1 if cand else 0), (band[k], cand)
            if cand:
                assert abs(r["hits"][k][0]["t"] - cand[0][0]) <= 1e-5 * max(1.0, cand[0][0]), band[k]
                if mat is not None:
                    assert r["hits"][k][0]["tri"] in [i for t, i in cand if abs(t - cand[0][0]) < 1e-5], band[k]
        else:
            n, mc = int(r["count"][k]), int(q["max_count"][k])
            assert n == min(mc, len(cand)), (band[k], n, len(cand))
            got = sorted(r["hits"][k][:n]["tri"].tolist())
            if mat is not None and n == len(cand):
                assert got == sorted(i for _, i in cand), band[k]
    if case in ("plane", "slab", "origin", "open_quad"):  # flat: a ray in the surface's plane meets nothing (det = 0 exactly)
        assert (r["count"][np.array([b.endswith("coplanar") for b in band])] == 0).all()


def test_zero_direction_traversal_records_nothing(ss_oracle):
    """an empty probe's ray (origin 0, direction 0, [kRayEpsilon, kMaxFloat]) on a triangle through the world origin"""
    sd, info = _scene("origin")
    q = np.concatenate([_query(op, origin=(0, 0, 0), dir=(0, 0, 0), max_count=8, material=mat)
                        for op in (S.SUBSURFACE_TRACE_MATERIAL, S.SUBSURFACE_CONTINUOUS_TRACE) for mat in (info["cb_zero"][0], S.INVALID)])
    r = _run(ss_oracle, "origin", q, reps=4)
    assert (r["count"] == 0).all() and (r["hits"]["tri"][:, :, 0][q["op"] == S.SUBSURFACE_TRACE_MATERIAL] == S.INVALID).all()
    assert (r["seed_end"] == r["seed_start"]).all()  # no candidate, so no alpha-test draw
    # the gathers there: RGB probes on the zero blue channel are empty; every weight stays finite
    _, _, qq, band, mats = sq.make("origin", False, 31)
    g = _run(ss_oracle, "origin", qq[(qq["op"] == S.SUBSURFACE_GATHER) & (mats == "cb_zero")], reps=64)
    empty = (g["probes"]["d"] == 0).all(-1)
    assert empty.any(), "no empty probe among the zero-channel gathers"
    assert np.isfinite(g["hits"]["weight"]).all() and np.isfinite(g["total_weight"]).all()


def test_plane_cb_gather_matches_model(ss_oracle):
    """On the flat plane a Christensen-Burley gather has at most one exit, from probe 0, at distance sampled_radius; its weight is
    base x eval(r) / avg(eval(sampled_radius)) (the geometric weight is 1); probes 1 and 2 find nothing."""
    sd, info, q, band, mats = sq.make("plane", False, 41)
    sel = (q["op"] == S.SUBSURFACE_GATHER) & (mats == "cb_grey")
    q = q[sel]
    r = _run(ss_oracle, "plane", q, reps=64)
    d, base = _distances(sd, "cb_grey"), _color(sd, "cb_grey")
    assert (r["count"] <= 1).all()
    assert (r["rays"] == 3).all()
    assert r["flag"].any()
    for i, k in np.argwhere(r["flag"] == 1):
        rec, p0 = r[i, k], r[i, k]["probes"][0]
        h = rec["hits"][0]
        pos = h["pos"].astype(np.float64)
        probe_pos = p0["o"].astype(np.float64) + h["t"] * p0["d"].astype(np.float64)
        assert np.abs(pos - probe_pos).max() < 1e-4 * max(1.0, float(p0["max_t"])), (i, k)
        entry_p = None
        p_a, p_b, p_c, _ = sq.triangle_frame(sd, int(q["triangle"][i]))
        entry_p = (1 - q["u"][i] - q["v"][i]) * p_a + q["u"][i] * p_b + q["v"][i] * p_c
        rr = np.linalg.norm(pos - entry_p)
        assert abs(rr - p0["sampled_radius"]) < 1e-4 * max(1.0, float(p0["sampled_radius"])), (i, k)
        expected = base * eval_model(d, rr) / eval_model(d, float(p0["sampled_radius"])).mean()
        np.testing.assert_allclose(rec["hits"][0]["weight"], expected, rtol=1e-3, atol=1e-30)
        assert rec["selected"] == 0 and rec["selected_sample_weight"] == 1.0


def _walk_checks(r, albedo):
    """every random-walk exit weight is albedo^k, k = rays - 1 scattering events (one trace per step, the last one finds the exit);
    k cannot be read from the sampler states alone: every candidate hit of the walk's traces draws once for the alpha test"""
    fails = []
    ok = r["flag"] == 1
    k = r["rays"].astype(np.float64) - 1.0
    expected = albedo[None, None, :] ** k[..., None]
    w = r["hits"][..., 0]["weight"].astype(np.float64)
    rel = np.where(ok[..., None], np.abs(w - expected) / np.maximum(expected, 1e-300), 0.0)
    bad = (rel > 2e-6 * (k[..., None] + 1.0)).any(-1)
    for idx in np.argwhere(bad)[:4]:
        fails.append(f"walk {tuple(idx)}: k {k[tuple(idx)]:.0f} weight {w[tuple(idx)]} expected {expected[tuple(idx)]}")
    fails += [f"walk {tuple(i)}: count {r['count'][tuple(i)]}" for i in np.argwhere(ok & (r["count"] != 1))[:2]]
    return fails


def _selection_checks(r, what):
    """the selection is unbiased: the mean of weights[selected] x selected_sample_weight equals the mean of the summed weights"""
    ok = r["flag"] == 1
    w = r["hits"]["weight"].astype(np.float64)
    picked = np.take_along_axis(w, r["selected"][..., None, None].astype(np.int64), axis=2)[..., 0, :] * r["selected_sample_weight"][..., None]
    total = w.sum(2)
    picked, total = np.where(ok[..., None], picked, 0.0), np.where(ok[..., None], total, 0.0)
    fails = []
    for i in range(r.shape[0]):
        diff = picked[i] - total[i]
        n = diff.shape[0]
        if np.abs(diff.mean(0)).max() > K_SIGMA * diff.std(0).max() / np.sqrt(n) + 1e-5 * np.abs(total[i].mean(0)).max():
            fails.append(f"{what} entry {i}: selected mean {picked[i].mean(0)} vs summed {total[i].mean(0)}")
    return fails


def test_grey_walk_weights_are_albedo_powers(ss_oracle):
    for case in ("box", "plane"):
        sd, info, q, band, mats = sq.make(case, False, 51)
        q = q[(q["op"] == S.SUBSURFACE_GATHER) & (mats == "rw_grey")]
        r = _run(ss_oracle, case, q, reps=128)
        albedo = remap_model(_color(sd, "rw_grey"), _distances(sd, "rw_grey"))[0]
        assert (r["flag"] == 1).mean() > 0.2
        assert not (f := _walk_checks(r, albedo)), f


def test_selection_is_unbiased(ss_oracle):
    for case in ("box", "sphere"):
        sd, info, q, band, mats = sq.make(case, False, 61)
        q = q[(q["op"] == S.SUBSURFACE_GATHER) & (mats == "cb_grey")][:6]
        r = _run(ss_oracle, case, q, reps=4096)
        assert (r["count"] > 1).any()
        assert not (f := _selection_checks(r, case)), f
