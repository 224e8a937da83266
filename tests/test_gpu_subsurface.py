"""The subsurface routines of dsss.cuh (trace_material, continuous_trace, remap, sample_s_r, ss_evaluate, ss_sample,
ss_geometric_weight, ss_gather and ss_exit_intersection) against the reference's own routines (the oracle, compiled in place), for every
case of subsurface_queries.CASES, RGB and spectral, on the product (`fast`) and the strict-IEEE (`parity`) builds.  Run with -m gpu.

(a) per query (subsurface_queries.make, REPS repetitions on the samplers (seed, r))
  parity   every word of every record bit for bit, sampler states included (a NaN matches a NaN)
  fast     seed_start equal.  A record is on the reference's decision path when its flag, count, selected, every hit's triangle and its
           end sampler state equal the reference's; the share of records off that path is bounded per op (FLIP_MAX).  On the path, every
           float is within the bounds below.  A non-finite output where the reference's is finite fails everywhere.  Random walks of more
           than one step (the reference's rays > 1) are compared as distributions only: a walk diverges after one rounding.
(b) as a distribution (fast only), N_DIST repetitions of subsurface_queries.distribution_queries, paired by repetition (the rule of
  test_gpu_bsdf_sample.compare_distribution): per exit-face bin (triangle mod 64) the indicator and weight x indicator per channel, the
  count and selected histograms, and the mean of weights[selected] x selected_sample_weight, each within K_SIGMA sigma / sqrt(N) plus
  RTOL_MEAN of the reference's mean.  The device's own records also pass test_oracle_subsurface's albedo^k and unbiased-selection checks.
(c) malformed queries are refused before any launch.
"""
import numpy as np
import pytest

import subsurface_queries as sq
import test_oracle_subsurface as tos
from etx_tracer_b200 import structs as S

pytestmark = pytest.mark.gpu

K_SIGMA = 5.5
REPS = 16
N_DIST = 1 << 16
RTOL_MEAN = 1e-3
NB = 64
# The product build's bounds (a), per op: RTOL relative for weights, profile values, remap outputs and s_r (below FTZ_ATOL absolute: the
# product build flushes denormals and its __expf underflows sooner); POS_RTOL for positions, t, probe origins and barycentric coordinates,
# relative beyond 1; DIR_ATOL for unit vectors (normals, w_i, probe directions and bases).  Measured on an H100 80GB HBM3 at 700 W (DESIGN
# §3); each bound is about twice the worst measured value.  What dominates: __logf near 1 in sample_s_r (small sampled radii, profile and
# gather values); __sinf / __cosf of phi times radii up to 4.8e4 (cb_huge) in the probe origins; make_intersection's normals at exits.
RTOL = {S.SUBSURFACE_TRACE_MATERIAL: 0.0, S.SUBSURFACE_CONTINUOUS_TRACE: 0.0, S.SUBSURFACE_REMAP: 8e-7, S.SUBSURFACE_PROFILE: 2e-2,
        S.SUBSURFACE_GATHER: 1e-2}  # measured 0, 0, 3.6e-7, 8.7e-3, 5.1e-3
POS_RTOL = {S.SUBSURFACE_TRACE_MATERIAL: 5e-7, S.SUBSURFACE_CONTINUOUS_TRACE: 7e-7, S.SUBSURFACE_REMAP: 0.0, S.SUBSURFACE_PROFILE: 4e-3,
            S.SUBSURFACE_GATHER: 7e-4}  # measured 2.1e-7, 3.6e-7, 0, 1.8e-3, 3.5e-4
DIR_ATOL = {S.SUBSURFACE_TRACE_MATERIAL: 0.0, S.SUBSURFACE_CONTINUOUS_TRACE: 0.0, S.SUBSURFACE_REMAP: 0.0, S.SUBSURFACE_PROFILE: 2.5e-7,
            S.SUBSURFACE_GATHER: 6e-5}  # measured 0, 0, 0, 1.2e-7, 3.1e-5
FTZ_ATOL = 1e-30
# A component below VEC_FLOOR of its field's largest in the record is held to that floor, not to itself: the profile's exp(-r / 3d) of a
# short-distance channel is a denormal the product build flushes before the division by d r, so a weight of (2.4, 9.5e-8, 1.3e-22) comes
# out as (2.4, 9.5e-8, 0) (plane, cb_tex: an exit 19 from an entry between black and white distance texels).
VEC_FLOOR = 1e-6
# The records off the reference's decision path, per op, at most (a share of the op's records).  Measured: none for the trace, remap and
# profile ops; 1 of 1999 gathers (plane, spectral, cb_tex: an entry on a texel boundary between black and white distance texels, where
# the product build's filtered distance rounds otherwise and the probe lands elsewhere).  continuous_trace records whose reference hits
# include one exactly on a triangle edge (u, v or u + v exactly 0 or 1) are not counted: the reference's strict Moeller-Trumbore gives
# the shared edge to both triangles (u = +-0 passes u >= 0), the product build's contracted barycentric puts it inside one and outside
# the other, so the buffer holds one hit fewer and the sampler one alpha-test draw fewer (measured on 768 of 4032 slab records, 416 of
# 8736 box records and 128 of 2688 open-quad records, all on rays through a quad's diagonal; DESIGN §3).
FLIP_MAX = {S.SUBSURFACE_TRACE_MATERIAL: 0.0, S.SUBSURFACE_CONTINUOUS_TRACE: 0.0, S.SUBSURFACE_REMAP: 0.0, S.SUBSURFACE_PROFILE: 0.0,
            S.SUBSURFACE_GATHER: 1e-3}
OP_NAMES = {S.SUBSURFACE_TRACE_MATERIAL: "trace", S.SUBSURFACE_CONTINUOUS_TRACE: "ctrace", S.SUBSURFACE_REMAP: "remap", S.SUBSURFACE_PROFILE: "profile",
            S.SUBSURFACE_GATHER: "gather"}
CASES = [(c, sp, fl) for c in sq.CASES for sp in (False, True) for fl in ("fast", "parity")]
WORDS = S.SUBSURFACE_RESULT.itemsize // 4


def _float_words(dt):
    """which 32-bit words of a record are float32: a NaN matches a NaN there (the device's and the host's default NaNs differ in sign)"""
    mask = np.zeros(dt.itemsize // 4, bool)

    def walk(d, base):
        for name in d.names:
            sub, off = d.fields[name][0], d.fields[name][1]
            inner, shape = (sub.subdtype if sub.subdtype else (sub, ()))
            n = int(np.prod(shape)) if shape else 1
            for k in range(n):
                start = base + off + k * inner.itemsize
                if inner.names:
                    walk(inner, start)
                elif inner.kind == "f":
                    mask[start // 4:(start + inner.itemsize) // 4] = True

    walk(dt, 0)
    return mask


FLOAT_WORDS = _float_words(S.SUBSURFACE_RESULT)
VALUES = ("selected_sample_weight", "total_weight", "albedo", "extinction", "scattering", "s_r", "eval", "geometric_weight", "probes.sampled_radius",
          "probes.max_t", "hits.weight")
POSITIONS = ("probes.o", "hits.t", "hits.u", "hits.v", "hits.pos")
DIRECTIONS = ("probes.d", "probes.u", "probes.v", "probes.w", "hits.w_i", "hits.nrm")

_cache = {}


def _setup(oracle_mod, case, spectral):
    key = (case, spectral)
    if key not in _cache:
        _cache.clear()
        index = sq.CASES.index(case)
        sd, info, q, band, mats = sq.make(case, spectral, seed=4001 * (1 + index) + int(spectral))
        o = oracle_mod.Oracle(sd)
        ref = o.subsurface(q, REPS)
        o.close()
        _cache[key] = (sd, info, q, band, mats, ref)
    return _cache[key]


def _field(x, name):
    a = x
    for part in name.split("."):
        a = a[part]
    return a.astype(np.float64).reshape(x.shape + (-1,))


def _multi_step_walk(q, mats, r):
    """gathers of random-walk materials whose reference walk took more than one step (compared as distributions only)"""
    rw = np.array([m.startswith("rw_") for m in mats])
    return (q["op"] == S.SUBSURFACE_GATHER)[:, None] & rw[:, None] & (r["rays"] > 1)


def compare(g, r, q, band, mats):
    """(a) on records shaped (n, REPS); returns (failures, report)"""
    fails = []
    report = {"records": int(g.size), "flips": {}, "worst": {}}
    op = np.broadcast_to(q["op"][:, None], g.shape)
    bnd = np.broadcast_to(band[:, None], g.shape)
    for idx in np.argwhere(g["seed_start"] != r["seed_start"])[:3]:
        fails.append(f"seed_start {tuple(idx)}: gpu {g[tuple(idx)]['seed_start']} ref {r[tuple(idx)]['seed_start']}")
    fields = VALUES + POSITIONS + DIRECTIONS
    fin = lambda x: np.stack([np.isfinite(_field(x, f)).all(-1) for f in fields], -1).all(-1)
    fg, fr = fin(g), fin(r)
    for idx in np.argwhere(fr & ~fg)[:4]:
        i = tuple(idx)
        fails.append(f"non-finite {i} ({bnd[i]} {mats[i[0]]})")
    walk = _multi_step_walk(q, mats, r)
    # continuous_trace records with a reference hit exactly on a triangle edge (see FLIP_MAX)
    valid = np.arange(24) < r["count"][..., None]
    hu, hv = r["hits"]["u"], r["hits"]["v"]
    on_edge = (valid & ((hu == 0) | (hv == 0) | (hu + hv == 1) | (hu == 1) | (hv == 1))).any(-1) & (op == S.SUBSURFACE_CONTINUOUS_TRACE)
    walk = walk | on_edge
    report["edge_records"] = int(on_edge.sum())
    on_path = ((g["flag"] == r["flag"]) & (g["count"] == r["count"]) & (g["selected"] == r["selected"]) & (g["seed_end"] == r["seed_end"]) &
               (g["hits"]["tri"] == r["hits"]["tri"]).all(-1) & (g["rays"] == r["rays"]) & fg & fr)
    for o, name in OP_NAMES.items():
        m = (op == o) & ~walk & fr
        if m.any():
            off = int((~on_path & m).sum())
            report["flips"][name] = f"{off}/{int(m.sum())}"
            if off:
                bands, counts = np.unique(bnd[~on_path & m], return_counts=True)
                report["flip_bands"] = report.get("flip_bands", {}) | {f"{name}:{b}": int(c) for b, c in zip(bands, counts)}
                i = tuple(np.argwhere(~on_path & m)[0])
                core = lambda x: (int(x["flag"]), int(x["count"]), int(x["rays"]), hex(int(x["seed_end"])), x["hits"]["tri"][:4].tolist(), x["hits"]["t"][:4].tolist(),
                                  x["hits"]["u"][:4].tolist(), x["hits"]["v"][:4].tolist())
                report["flip_example"] = report.get("flip_example", []) + [(name, i, bnd[i], mats[i[0]], q[i[0]]["origin"].tolist(), q[i[0]]["dir"].tolist(),
                                                                           "gpu", core(g[i]), "ref", core(r[i]))]
            if off > FLIP_MAX[o] * m.sum():
                i = tuple(np.argwhere(~on_path & m)[0])
                fails.append(f"{name}: {off} of {int(m.sum())} records off the reference's decision path; e.g. {i} ({bnd[i]} {mats[i[0]]})")
    ok = on_path & ~walk
    err = {}
    for kind, names in (("value", VALUES), ("pos", POSITIONS), ("dir", DIRECTIONS)):
        e = np.zeros(g.shape)
        for f in names:
            vg, vr = _field(g, f), _field(r, f)
            with np.errstate(invalid="ignore", over="ignore"):
                d = np.abs(vg - vr)
                d = np.where(vg == vr, 0.0, d)
                if kind == "value":  # relative, with a floor at VEC_FLOOR of the field's largest component in the record
                    d = d / np.maximum(np.maximum(np.abs(vr), VEC_FLOOR * np.abs(vr).max(-1, keepdims=True)), FTZ_ATOL)
                elif kind == "pos":
                    d = d / np.maximum(1.0, np.abs(vr))
            e = np.maximum(e, np.where(ok, d.max(-1), 0.0))
        err[kind] = e
        bound = np.vectorize(lambda o: {"value": RTOL, "pos": POS_RTOL, "dir": DIR_ATOL}[kind][o])(op)
        for idx in np.argwhere(ok & (e > bound))[:3]:
            i = tuple(idx)
            fails.append(f"{kind} {i} ({bnd[i]} {mats[i[0]]}): error {e[i]:.3g} > {bound[i]:.3g}")
    for o, name in OP_NAMES.items():
        for b in np.unique(band[q["op"] == o]):
            m = ok & (op == o) & (bnd == b)
            if m.any():
                report["worst"][b] = tuple(float(err[k][m].max()) for k in ("value", "pos", "dir"))
        m = ok & (op == o)
        if m.any():
            report["worst_op"] = report.get("worst_op", {})
            report["worst_op"][name] = tuple(float(err[k][m].max()) for k in ("value", "pos", "dir"))
    return fails, report


def _paired(what, xg, xr):
    """paired differences per repetition of per-sample quantities xg, xr shaped (n, bins); returns (failures, worst z)"""
    n = xg.shape[0]
    diff = xg - xr
    mean, ref_mean = diff.mean(0), xr.mean(0)
    sigma = diff.std(0)
    bound = K_SIGMA * sigma / np.sqrt(n) + RTOL_MEAN * np.abs(ref_mean)
    fails = [f"{what} bin {b}: mean difference {mean[b]:.4g} (reference {ref_mean[b]:.4g}), sigma/sqrt(N) {sigma[b] / np.sqrt(n):.3g}"
             for b in np.flatnonzero(np.abs(mean) > bound + 1e-300)[:3]]
    with np.errstate(divide="ignore", invalid="ignore"):
        z = np.where(sigma > 0, np.abs(mean) / (sigma / np.sqrt(n)), 0.0)
    return fails, float(z.max()) if z.size else 0.0


def _face_bins(rec):
    """(n, NB) indicator and (n, NB, 3) weight sums of the exits per face bin (triangle mod NB)"""
    n = rec.shape[0]
    valid = np.arange(24)[None, :] < np.where(rec["flag"] == 1, rec["count"], 0)[:, None]
    keys = (np.arange(n)[:, None] * NB + rec["hits"]["tri"].astype(np.int64) % NB)[valid]
    ind = np.bincount(keys, minlength=n * NB).reshape(n, NB).astype(np.float64)
    w = rec["hits"]["weight"].astype(np.float64)[valid]
    ws = np.stack([np.bincount(keys, w[:, c], n * NB).reshape(n, NB) for c in range(3)], -1)
    return ind, ws


def compare_distribution(what, g, r):
    """(b) for one entry's N_DIST records; returns (failures, worst z)"""
    fails, z = [], 0.0
    ig, wg = _face_bins(g)
    ir, wr = _face_bins(r)
    parts = [("exit face", ig, ir)] + [(f"exit face weight[{c}]", wg[..., c], wr[..., c]) for c in range(3)]
    hist = lambda x, nb: np.eye(nb)[np.minimum(x, nb - 1)]
    parts.append(("count", hist(np.where(g["flag"] == 1, g["count"], 0), 25), hist(np.where(r["flag"] == 1, r["count"], 0), 25)))
    parts.append(("selected", hist(np.where(g["flag"] == 1, g["selected"], 24), 25), hist(np.where(r["flag"] == 1, r["selected"], 24), 25)))

    def picked(x):
        w = x["hits"]["weight"].astype(np.float64)
        p = w[np.arange(x.shape[0]), x["selected"].astype(np.int64)] * x["selected_sample_weight"][:, None]
        return np.where((x["flag"] == 1)[:, None], p, 0.0)

    parts.append(("weights[selected] x selected_sample_weight", picked(g), picked(r)))
    for name, xg, xr in parts:
        f, zz = _paired(f"{what}: {name}", xg, xr)
        fails += f
        z = max(z, zz)
    return fails, z


@pytest.fixture(scope="module")
def ss_oracle(oracle_mod):
    if not oracle_mod.has_subsurface():
        pytest.skip("oracle/_ref predates oracle_subsurface (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


@pytest.mark.parametrize("case,spectral,flavor", CASES, ids=[f"{c}-{'spectral' if sp else 'rgb'}-{fl}" for c, sp, fl in CASES])
def test_subsurface_matches_reference(ss_oracle, case, spectral, flavor):
    from etx_tracer_b200.api import GPUVCM
    sd, info, q, band, mats, ref = _setup(ss_oracle, case, spectral)
    dev = GPUVCM(sd, flavor=flavor)
    g = dev.debug_subsurface(q, REPS)
    tag = f"{case}/{'spectral' if spectral else 'rgb'}/{flavor}"
    if flavor == "parity":
        wg = np.ascontiguousarray(g).view(np.uint32).reshape(g.shape + (WORDS,))
        wr = np.ascontiguousarray(ref).view(np.uint32).reshape(ref.shape + (WORDS,))
        exact = ((wg == wr) | (FLOAT_WORDS & np.isnan(wg.view(np.float32)) & np.isnan(wr.view(np.float32)))).all(-1)
        fails = [f"{tuple(i)} ({band[i[0]]} {mats[i[0]]})" for i in np.argwhere(~exact)[:8]]
        dev.close()
        print(f"\n[subsurface] {tag}: bit-exact {int(exact.sum())} of {exact.size}")
        assert not fails, f"{int((~exact).sum())} records differ:\n  " + "\n  ".join(fails)
        return
    fails, rep = compare(g, ref, q, band, mats)
    # the device's own walks and selections against the float64 rules of test_oracle_subsurface
    grey = (q["op"] == S.SUBSURFACE_GATHER) & (mats == "rw_grey")
    if grey.any() and not spectral:
        albedo = tos.remap_model(tos._color(sd, "rw_grey"), tos._distances(sd, "rw_grey"))[0]
        fails += tos._walk_checks(g[grey], albedo)
    z = 0.0
    if case in sq.DIST_MATERIALS:
        qd, _, dmats = sq.distribution_queries(case, spectral, 6007 * (1 + sq.CASES.index(case)) + int(spectral), sd, info)
        o = ss_oracle.Oracle(sd)
        for a in range(qd.shape[0]):
            rd = o.subsurface(qd[a:a + 1], N_DIST)[0]
            gd = dev.debug_subsurface(qd[a:a + 1], N_DIST)[0]
            f, zz = compare_distribution(f"{case} {dmats[a]}", gd, rd)
            fails += f
            z = max(z, zz)
            if dmats[a].startswith("cb_"):
                fails += tos._selection_checks(gd[None, :], f"{case} {dmats[a]} (device)")
        o.close()
    dev.close()
    worst = "; ".join(f"{k} {v[0]:.2e}/{v[1]:.2e}/{v[2]:.2e}" for k, v in rep["worst"].items())
    print(f"\n[subsurface] {tag}: off-path {rep['flips']} {rep.get('flip_bands', '')} {rep.get('flip_example', '')}; edge records {rep['edge_records']}; worst value rel / pos rel / dir abs per op {rep.get('worst_op')}; per band: {worst}; "
          f"worst bin z {z:.2f}")
    assert not fails, f"{len(fails)} findings:\n  " + "\n  ".join(fails[:24])


def test_malformed_queries_are_refused(ss_oracle):
    from etx_tracer_b200.api import GPUVCM, EtxbError
    sd, info = sq.scene("plane", False)
    dev = GPUVCM(sd, flavor="fast")
    m, first, _ = info["cb_grey"]
    good = np.zeros(1, S.SUBSURFACE_QUERY)
    good["op"], good["triangle"], good["u"], good["v"], good["dir"] = S.SUBSURFACE_GATHER, first, 0.3, 0.3, (0.0, -1.0, 0.0)
    good["t_min"], good["t_max"], good["max_count"], good["material"] = sq.K_RAY_EPSILON, sq.K_MAX_FLOAT, 8, m
    dev.debug_subsurface(good)
    plain = next(i for i, t in enumerate(np.concatenate(sd.triangles)) if int(sd.materials[int(t["material_index"])]["subsurface"]["cls"][0]) == 0)
    cases = {
        "op past 4": dict(op=5),
        "triangle past the count": dict(triangle=sum(t.shape[0] for t in sd.triangles)),
        "gather without a subsurface class": dict(triangle=plain),
        "gather zero direction": dict(dir=(0.0, 0.0, 0.0)),
        "gather NaN direction": dict(dir=(np.nan, -1.0, 0.0)),
        "gather NaN u": dict(u=np.nan),
        "profile probe direction 3": dict(op=S.SUBSURFACE_PROFILE, direction=3),
        "profile NaN rnd": dict(op=S.SUBSURFACE_PROFILE, rnd=np.nan),
        "profile infinite radius": dict(op=S.SUBSURFACE_PROFILE, radius=np.inf),
        "profile NaN normal": dict(op=S.SUBSURFACE_PROFILE, normal=(np.nan, 0.0, 0.0)),
        "trace material past the count": dict(op=S.SUBSURFACE_TRACE_MATERIAL, material=len(sd.materials)),
        "trace zero direction": dict(op=S.SUBSURFACE_TRACE_MATERIAL, dir=(0.0, 0.0, 0.0)),
        "trace NaN origin": dict(op=S.SUBSURFACE_TRACE_MATERIAL, origin=(np.nan, 0.0, 0.0)),
        "trace infinite t_max": dict(op=S.SUBSURFACE_TRACE_MATERIAL, t_max=np.inf),
        "continuous trace max_count 0": dict(op=S.SUBSURFACE_CONTINUOUS_TRACE, max_count=0),
        "continuous trace max_count 9": dict(op=S.SUBSURFACE_CONTINUOUS_TRACE, max_count=9),
        "remap NaN color": dict(op=S.SUBSURFACE_REMAP, color=(np.nan, 0.0, 0.0)),
        "remap infinite distance": dict(op=S.SUBSURFACE_REMAP, distances=(1.0, np.inf, 1.0)),
    }
    before = dev.counters()["kernel_launches"]
    for what, fields in cases.items():
        bad = good.copy()
        for k, v in fields.items():
            bad[k] = v
        with pytest.raises(EtxbError):
            dev.debug_subsurface(np.concatenate([good, bad]))
            pytest.fail(what)
    two, out = np.repeat(good, 2), np.zeros(1, S.SUBSURFACE_RESULT)
    assert dev.lib.etxb_debug_subsurface(dev.h, two.ctypes.data, 2, 1 << 30, out.ctypes.data) < 0
    assert dev.counters()["kernel_launches"] == before, "a refused query launched a kernel"
    ok = np.repeat(good, 3)
    ok["op"] = (S.SUBSURFACE_CONTINUOUS_TRACE, S.SUBSURFACE_TRACE_MATERIAL, S.SUBSURFACE_REMAP)
    ok["material"][1] = S.INVALID  # any material
    ok["dir"][2] = (0.0, 0.0, 0.0)  # remap ignores the ray
    dev.debug_subsurface(ok)
    dev.close()
