"""The media routines of dmedium.cuh (medium_intersects_bounds, medium_sample_density, medium_transmittance, sample_medium, the
Henyey-Greenstein phase function) and the shadow-ray walk through Boundary surfaces (trace_transmittance of dtrace.cuh) against the
reference's own routines (the oracle, compiled in place), for every case of medium_queries.CASES, RGB and spectral, on the product
(`fast`) and the strict-IEEE (`parity`) builds.  Run with -m gpu.

(a) per query (medium_queries.make, REPS repetitions on the samplers (seed, r))
  parity   every word of every record bit for bit, sampler states included (a NaN matches a NaN)
  fast     seed_start equal.  A record is on the reference's decision path when its end state, its bounds flag and the zero-ness of its
           value equal the reference's; the share of records off that path is bounded per op (FLIP_MAX): the product build's __logf
           can move a free-flight step across kRayEpsilon or t_max, a density across a Russian-roulette draw, an approximate slab test
           across a tangent.  On the path, every float is within the bounds below, zero exactly where the reference is zero.  A
           non-finite output where the reference's is finite fails in every band.
(b) as a distribution (fast only), N_DIST repetitions of medium_queries.distribution_queries: per bin of sampled_medium_t (32 bins over
  the ray) the paired differences of the indicator and of weight x indicator, and the mean transmittance, within K_SIGMA sigma / sqrt(N)
  plus RTOL_MEAN of the reference's mean (test_gpu_bsdf_sample.compare_distribution's rule).  The heterogeneous transmittance means
  are also held to the float64 model of test_oracle_medium.py (exp(-max_sigma x the optical depth)).
(c) malformed queries are refused before any launch.
"""
import numpy as np
import pytest

import medium_queries as mq
import test_oracle_medium as tom
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

K_SIGMA = 5.5
REPS = 16
N_DIST = 1 << 16
RTOL_MEAN = 1e-3
# a device weight against the float64 free-flight closed form: the oracle's own distance from it (2e-5) plus the product bound RTOL
WEIGHT_RTOL_MODEL = 5e-5
# The product build's bounds (a).  Measured on an H100 80GB HBM3 at 700 W (DESIGN §3); each bound is about twice the worst measured
# value.  RTOL relative for values, weights, transmittances and t; POS_ATOL absolute for positions and bounds (local units);
# MAX_ANGLE for directions; FTZ_ATOL for flushed denormals.  RTOL_PHASE_EDGE at |g| = 0.999, where 1 + g^2 - 2 g cos cancels to
# (1 - |g|)^2 = 1e-6 and the contracted product build rounds it otherwise; MAX_ANGLE_EDGE the sampled direction there.
# T_ATOL absolute for sampled_medium_t: __logf's absolute error near 1 (2^-21.4) over max_sigma, summed over the tracking steps.
# MAX_ANGLE_SHORT for the local direction of a segment just longer than kRayEpsilon (a float32 difference of two nearby local points);
# MAX_ANGLE_SMALL_G for the sampled direction at 1e-3 <= |g| <= 1e-2, where the Henyey-Greenstein inversion divides a rounded
# difference by 2 g.  A value below FLT_MIN counts as zero: the product build flushes denormals (-ftz=true).
RTOL, POS_ATOL, T_ATOL, MAX_ANGLE, FTZ_ATOL = 2e-5, 2.5e-5, 1e-6, 7e-6, 1e-30  # measured 9.6e-6, 1.2e-5, -, 3.3e-6 rad
# MAX_ANGLE_RND_EDGE at rnd.x = 0 or 1 - 2^-24, where the sampled cosine lies within ulps of +-1 and an absolute cosine error dc turns
# into an angle of sqrt(2 dc) (measured 6.9e-4 rad: the reference's cosine rounds to exactly 1 where the product build's is 1 - 2^-22).
RTOL_PHASE_EDGE, MAX_ANGLE_EDGE, MAX_ANGLE_SHORT, MAX_ANGLE_SMALL_G, MAX_ANGLE_RND_EDGE = 0.5, 1.4e-2, 5e-4, 4.5e-3, 1.5e-3  # measured 0.26, 6.8e-3, 2.3e-4, 2.1e-3, 6.9e-4
FLT_MIN = 1.17549435e-38
# the records off the reference's decision path, per op and case, at most (measured: none, in every case; DESIGN §3).  The product
# build flushes denormal inputs (-ftz=true): a density coordinate of -2^-149 is -0 to it, so those lookups are held to the reference's
# lookup at the flushed coordinate (the `below` band; ref_ftz in _setup).
FLIP_MAX = {S.MEDIUM_BOUNDS: 0, S.MEDIUM_DENSITY: 0, S.MEDIUM_TRANSMITTANCE: 0, S.MEDIUM_SAMPLE: 0, S.MEDIUM_PHASE: 0, S.MEDIUM_SEGMENT: 0}
OP_NAMES = {S.MEDIUM_BOUNDS: "bounds", S.MEDIUM_DENSITY: "density", S.MEDIUM_TRANSMITTANCE: "transmittance", S.MEDIUM_SAMPLE: "sample",
            S.MEDIUM_PHASE: "phase", S.MEDIUM_SEGMENT: "segment"}
CASES = [(c, sp, fl) for c in mq.CASES for sp in (False, True) for fl in ("fast", "parity")]
WORDS = S.MEDIUM_RESULT.itemsize // 4
FLOATS = ("value", "pos", "dir", "t_min", "t_max", "t")

_cache = {}


def _setup(oracle_mod, case, spectral):
    key = (case, spectral)
    if key not in _cache:
        _cache.clear()
        sd = mq.scene(spectral)
        index = mq.CASES.index(case)
        q, band = mq.make(sd, case, spectral, seed=3001 * (1 + index) + int(spectral))
        o = oracle_mod.Oracle(sd)
        ref = o.medium(q, REPS)
        # what the product build computes from its inputs: a denormal density coordinate flushed to a signed zero
        q_ftz = q.copy()
        den = (np.abs(q_ftz["origin"]) < FLT_MIN) & (q_ftz["origin"] != 0) & (q_ftz["op"] == S.MEDIUM_DENSITY)[:, None]
        q_ftz["origin"] = np.where(den, np.copysign(np.float32(0.0), q_ftz["origin"]), q_ftz["origin"])
        ref_ftz = np.where(den.any(-1)[:, None], o.medium(q_ftz, REPS), ref)
        qd = rd = None
        if case in mq.MEDIA:
            qd = mq.distribution_queries(case, spectral, seed=5003 * (1 + index) + int(spectral))
            rd = o.medium(qd, N_DIST)
        o.close()
        _cache[key] = (sd, q, band, ref, ref_ftz, qd, rd)
    return _cache[key]


def _angle(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=-1), (a * b).sum(-1))


def compare(g, r, q, band):
    """(a) on records shaped (n, REPS); returns (failures, report)"""
    fails = []
    wg = np.ascontiguousarray(g).view(np.uint32).reshape(g.shape + (WORDS,))
    wr = np.ascontiguousarray(r).view(np.uint32).reshape(r.shape + (WORDS,))
    report = {"records": int(g.size), "bit_exact": int((wg == wr).all(-1).sum()), "flips": {}, "worst": {}}
    op = np.broadcast_to(q["op"][:, None], g.shape)
    bnd = np.broadcast_to(band[:, None], g.shape)
    for idx in np.argwhere(g["seed_start"] != r["seed_start"])[:3]:
        fails.append(f"seed_start {tuple(idx)}: gpu {g[tuple(idx)]} ref {r[tuple(idx)]}")
    finite = lambda x: np.stack([np.isfinite(x[f]).reshape(x.shape + (-1,)).all(-1) for f in FLOATS], -1).all(-1)
    fg, fr = finite(g), finite(r)
    for idx in np.argwhere(fr & ~fg)[:4]:
        i = tuple(idx)
        fails.append(f"non-finite {i} ({OP_NAMES[int(op[i])]} {bnd[i]}): gpu {g[i]} ref {r[i]}")
    zero_g, zero_r = (np.abs(g["value"]) < FLT_MIN).all(-1), (np.abs(r["value"]) < FLT_MIN).all(-1)
    on_path = (g["seed_end"] == r["seed_end"]) & (g["flag"] == r["flag"]) & (zero_g == zero_r) & fg & fr
    for o, name in OP_NAMES.items():
        m = op == o
        if m.any():
            off = int((~on_path & m & fr).sum())
            report["flips"][name] = off
            if off > FLIP_MAX[o]:
                i = tuple(np.argwhere(~on_path & m & fr)[0])
                fails.append(f"{name}: {off} records off the reference's decision path (bound {FLIP_MAX[o]}); e.g. {i} ({bnd[i]}): gpu {g[i]} ref {r[i]}")
    edge = (op == S.MEDIUM_PHASE) & (np.abs(np.broadcast_to(q["g"][:, None], g.shape)) > 0.99)
    rtol = np.where(edge, RTOL_PHASE_EDGE, RTOL)
    gq = np.abs(np.broadcast_to(q["g"][:, None], g.shape))
    small_g = (op == S.MEDIUM_PHASE) & (gq >= 1e-3) & (gq <= 1e-2)
    rnd_x = np.broadcast_to(q["rnd"][:, 0][:, None], g.shape)
    rnd_edge = (op == S.MEDIUM_PHASE) & ((rnd_x == 0) | (rnd_x == mq.ONE_MINUS))
    max_angle = np.where(edge, MAX_ANGLE_EDGE, np.where(small_g, MAX_ANGLE_SMALL_G, np.where(bnd == "short", MAX_ANGLE_SHORT, MAX_ANGLE)))
    max_angle = np.where(rnd_edge, np.maximum(max_angle, MAX_ANGLE_RND_EDGE), max_angle)
    ok = on_path
    err = {}
    for f in ("value", "t"):
        vg, vr = g[f].astype(np.float64).reshape(g.shape + (-1,)), r[f].astype(np.float64).reshape(g.shape + (-1,))
        e = np.abs(vg - vr)
        flip = (vr == 0) & (vg != 0)
        atol = T_ATOL if f == "t" else FTZ_ATOL
        bad = ((e > rtol[..., None] * np.abs(vr) + atol) | flip).any(-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            err[f] = np.where(ok[..., None] & (np.abs(vr) >= FLT_MIN), e / np.abs(vr), 0.0).max(-1)
        for idx in np.argwhere(ok & bad)[:3]:
            i = tuple(idx)
            fails.append(f"{f} {i} ({OP_NAMES[int(op[i])]} {bnd[i]}): gpu {g[i]} ref {r[i]}")
    pos_e = np.zeros(g.shape)
    for f in ("pos", "t_min", "t_max"):
        vg, vr = g[f].astype(np.float64).reshape(g.shape + (-1,)), r[f].astype(np.float64).reshape(g.shape + (-1,))
        with np.errstate(invalid="ignore"):
            e = np.where(np.isinf(vr) & (vg == vr), 0.0, np.abs(vg - vr)).max(-1)
        e = np.where(op == S.MEDIUM_SAMPLE, e / np.maximum(1.0, np.abs(vr).max(-1)), e)  # world positions: relative beyond 1
        pos_e = np.maximum(pos_e, np.where(ok, e, 0.0))
        for idx in np.argwhere(ok & (e > POS_ATOL))[:3]:
            i = tuple(idx)
            fails.append(f"{f} {i} ({OP_NAMES[int(op[i])]} {bnd[i]}): gpu {g[i]} ref {r[i]}")
    has_dir = (np.abs(r["dir"]).sum(-1) > 0) & ok
    angle = np.where(has_dir, _angle(g["dir"], r["dir"]), 0.0)
    angle = np.where(np.isfinite(angle), angle, 0.0)
    for idx in np.argwhere(has_dir & (angle > max_angle))[:3]:
        i = tuple(idx)
        fails.append(f"dir {i} ({OP_NAMES[int(op[i])]} {bnd[i]}): {angle[i]:.3g} rad; gpu {g[i]} ref {r[i]}")
    for o, name in OP_NAMES.items():
        for b in np.unique(band):
            m = ok & (op == o) & (bnd == b)
            if m.any():
                report["worst"][f"{name}/{b}"] = (float(err["value"][m].max()), float(err["t"][m].max()), float(pos_e[m].max()), float(angle[m].max()))
    classes = {"edge": edge, "small_g": small_g & ~edge, "rnd_edge": rnd_edge & ~edge & ~small_g, "short": (bnd == "short") & ~rnd_edge,
               "other": ~edge & ~small_g & ~rnd_edge & (bnd != "short")}
    report["angle"] = {k: float(np.where(m, angle, 0.0).max()) for k, m in classes.items()}
    report["value_rel"] = {"edge": float(np.where(edge, err["value"], 0.0).max()), "other": float(np.where(~edge, err["value"], 0.0).max())}
    return fails, report


def _bins(q, rec):
    """32 bins of sampled_medium_t over the ray (heterogeneous: over the local t range), bin 32 for no scattering"""
    t = rec["t"].astype(np.float64)
    span = float(q["max_t"]) if q["medium"] < len(mq.HOMOGENEOUS) else 1.8
    b = np.minimum((t / span * 32).astype(np.int64), 31)
    return np.where(t > 0, b, 32)


def compare_distribution(case, spectral, qd, gd, rd):
    """(b): returns (failures, worst z)"""
    fails, z_max = [], 0.0
    for a in range(qd.shape[0]):
        g, r = gd[a], rd[a]
        n = g.shape[0]
        if qd["op"][a] == S.MEDIUM_TRANSMITTANCE:
            bg = br = np.zeros(n, np.int64)
            quantities = [("transmittance", g["value"][:, 0].astype(np.float64), r["value"][:, 0].astype(np.float64))]
            nb = 1
        else:
            bg, br = _bins(qd[a], g), _bins(qd[a], r)
            quantities = [("indicator", np.ones(n), np.ones(n))] + [(f"weight[{c}]", g["value"][:, c].astype(np.float64), r["value"][:, c].astype(np.float64)) for c in range(3)]
            nb = 33
        same = bg == br
        for name, xg, xr in quantities:
            sum_g, sum_r = np.bincount(bg, xg, nb), np.bincount(br, xr, nb)
            sq_same = np.bincount(bg[same], (xg - xr)[same] ** 2, nb)
            sq_diff = np.bincount(bg[~same], xg[~same] ** 2, nb) + np.bincount(br[~same], xr[~same] ** 2, nb)
            mean = (sum_g - sum_r) / n
            ref_mean = sum_r / n
            sigma = np.sqrt(np.maximum((sq_same + sq_diff) / n - mean ** 2, 0.0))
            bound = K_SIGMA * sigma / np.sqrt(n) + RTOL_MEAN * np.abs(ref_mean)
            for b in np.flatnonzero(np.abs(mean) > bound)[:3]:
                fails.append(f"{case} query {a}: bin {b} {name}: mean difference {mean[b]:.4g} (reference {ref_mean[b]:.4g}), sigma/sqrt(N) {sigma[b] / np.sqrt(n):.3g}")
            with np.errstate(divide="ignore", invalid="ignore"):
                z = np.where(sigma > 0, np.abs(mean) / (sigma / np.sqrt(n)), 0.0)
            z_max = max(z_max, float(z.max()))
        if qd["op"][a] == S.MEDIUM_SAMPLE and case in mq.HOMOGENEOUS and not spectral:
            # the device's own samples against the float64 free-flight model (RGB: the model takes the media's rgb coefficients)
            fails += tom.free_flight_fails(case, tuple(qd["throughput"][a]), float(qd["max_t"][a]), g, weight_rtol=WEIGHT_RTOL_MODEL)
        if qd["op"][a] == S.MEDIUM_TRANSMITTANCE and case in mq.HETEROGENEOUS and case != "zero_sigma":
            p, d, seg = tom._local(case, qd["origin"][a], qd["direction"][a], float(qd["max_t"][a]))
            _, t0, t1 = tom._slab(p, d, seg, inflate=False)
            expected = np.exp(-mq._HET[case][4] * tom._optical_depth(case, p, d, t0, t1))
            v = g["value"][:, 0].astype(np.float64)
            if abs(v.mean() - expected) > K_SIGMA * v.std() / np.sqrt(n) + 1e-4:
                fails.append(f"{case}: device transmittance mean {v.mean():.6g}, float64 model {expected:.6g}")
    return fails, z_max


@pytest.fixture(scope="module")
def medium_oracle(oracle_mod):
    if not oracle_mod.has_medium():
        pytest.skip("oracle/_ref predates oracle_medium (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


@pytest.mark.parametrize("case,spectral,flavor", CASES, ids=[f"{c}-{'spectral' if sp else 'rgb'}-{fl}" for c, sp, fl in CASES])
def test_medium_matches_reference(medium_oracle, case, spectral, flavor):
    from etx_tracer_b200.api import GPUVCM
    sd, q, band, ref, ref_ftz, qd, rd = _setup(medium_oracle, case, spectral)
    dev = GPUVCM(sd, flavor=flavor)
    g = dev.debug_medium(q, REPS)
    if flavor == "parity":
        wg = np.ascontiguousarray(g).view(np.uint32).reshape(g.shape + (WORDS,))
        wr = np.ascontiguousarray(ref).view(np.uint32).reshape(ref.shape + (WORDS,))
        exact = (wg == wr).all(-1)
        fails = [f"{tuple(i)} ({band[i[0]]}): gpu {g[tuple(i)]} ref {ref[tuple(i)]}" for i in np.argwhere(~exact)[:8]]
        dev.close()
        print(f"\n[medium] {case}/{'spectral' if spectral else 'rgb'}/parity: bit-exact {int(exact.sum())} of {exact.size}")
        assert not fails, f"{int((~exact).sum())} records differ:\n  " + "\n  ".join(fails)
        return
    fails, rep = compare(g, ref_ftz, q, band)
    z = 0.0
    if qd is not None:
        gd = dev.debug_medium(qd, N_DIST)
        f, z = compare_distribution(case, spectral, qd, gd, rd)
        fails += f
    dev.close()
    worst = "; ".join(f"{k} {v[0]:.2e}/{v[1]:.2e}/{v[2]:.2e}/{v[3]:.2e}" for k, v in rep["worst"].items())
    flips = ", ".join(f"{k} {v}" for k, v in rep["flips"].items())
    print(f"\n[medium] {case}/{'spectral' if spectral else 'rgb'}/fast: bit-exact {rep['bit_exact']} of {rep['records']}; off-path {flips}; "
          f"angle per class {rep['angle']}; value rel {rep['value_rel']}; "
          f"worst value rel / t rel / pos abs / angle per op and band: {worst}; worst bin z {z:.2f}")
    assert not fails, f"{len(fails)} findings:\n  " + "\n  ".join(fails[:24])


def test_malformed_queries_are_refused(medium_oracle):
    from etx_tracer_b200.api import GPUVCM, EtxbError
    sd = mq.scene(False)
    dev = GPUVCM(sd, flavor="fast")
    good = np.zeros(1, S.MEDIUM_QUERY)
    good["op"], good["medium"], good["direction"], good["max_t"] = S.MEDIUM_SAMPLE, mq.medium_index("fog"), (0.0, 0.0, 1.0), 1.0
    dev.debug_medium(good)
    cases = {
        "op past 5": dict(op=6),
        "medium past the count": dict(medium=len(mq.MEDIA)),
        "invalid medium for a sample": dict(medium=S.INVALID),
        "zero direction": dict(direction=(0.0, 0.0, 0.0)),
        "NaN direction": dict(direction=(np.nan, 0.0, 1.0)),
        "infinite direction": dict(direction=(np.inf, 0.0, 1.0)),
        "sample max_t below kRayEpsilon": dict(max_t=float(mq.K_RAY_EPSILON) * 0.5),
        "sample max_t NaN": dict(max_t=np.nan),
        "density of a homogeneous medium": dict(op=S.MEDIUM_DENSITY),
        "segment end not finite": dict(op=S.MEDIUM_SEGMENT, end=(np.inf, 0.0, 0.0)),
        "phase direction zero": dict(op=S.MEDIUM_PHASE, direction=(0.0, 0.0, 0.0)),
        # heterogeneous tracking that would never end: a NaN local segment (t >= t_max never true, a NaN density never ends ratio
        # tracking's roulette or delta tracking), an overflowing local length (a zero direction at one point), steps below an ulp of t
        "transmittance max_t NaN": dict(op=S.MEDIUM_TRANSMITTANCE, medium=mq.medium_index("cloud"), max_t=np.nan),
        "transmittance origin NaN": dict(op=S.MEDIUM_TRANSMITTANCE, medium=mq.medium_index("cloud"), origin=(np.nan, 0.0, 0.0)),
        "sample origin infinite": dict(medium=mq.medium_index("cloud"), origin=(0.0, -np.inf, 0.0)),
        "bounds origin NaN": dict(op=S.MEDIUM_BOUNDS, medium=mq.medium_index("cloud"), origin=(0.0, 0.0, np.nan)),
        "density coordinate NaN": dict(op=S.MEDIUM_DENSITY, medium=mq.medium_index("cloud"), origin=(np.nan, 0.5, 0.5)),
        "transmittance max_t 3e19": dict(op=S.MEDIUM_TRANSMITTANCE, medium=mq.medium_index("cloud"), max_t=3e19),
        "sample max_t 3e19": dict(medium=mq.medium_index("cloud"), max_t=3e19),
        "sample origin 1e16": dict(medium=mq.medium_index("cloud"), origin=(1e16, 0.0, 0.0)),
        "transmittance origin far from the medium": dict(op=S.MEDIUM_TRANSMITTANCE, medium=mq.medium_index("cloud"), origin=(0.0, 0.0, -1e5)),
        "sample throughput NaN": dict(throughput=(np.nan, 1.0, 1.0)),
        "segment end 1e16": dict(op=S.MEDIUM_SEGMENT, end=(1e16, 0.0, 0.0)),
        "segment far from a heterogeneous medium": dict(op=S.MEDIUM_SEGMENT, origin=(0.0, 1e5, 0.0), end=(0.0, 0.0, 0.0)),
    }
    before = dev.counters()["kernel_launches"]
    for what, fields in cases.items():
        bad = good.copy()
        for k, v in fields.items():
            bad[k] = v
        with pytest.raises(EtxbError):
            dev.debug_medium(np.concatenate([good, bad]))
            pytest.fail(what)
    # count x repetitions past 2^31: called without the wrapper, which would allocate the output first
    two, out = np.repeat(good, 2), np.zeros(1, S.MEDIUM_RESULT)
    assert dev.lib.etxb_debug_medium(dev.h, two.ctypes.data, 2, 1 << 30, out.ctypes.data) < 0
    assert dev.counters()["kernel_launches"] == before, "a refused query launched a kernel"
    # a segment may start outside every medium, and the phase op ignores the medium
    ok = np.zeros(2, S.MEDIUM_QUERY)
    ok["op"], ok["medium"], ok["end"] = (S.MEDIUM_SEGMENT, S.MEDIUM_PHASE), S.INVALID, (0.5, 0.0, 0.0)
    ok["direction"] = (0.0, 0.0, 1.0)
    dev.debug_medium(ok)
    far = good.copy()
    far["op"], far["medium"], far["max_t"] = S.MEDIUM_TRANSMITTANCE, mq.medium_index("cloud"), mq.K_MAX_FLOAT  # refused by the routine itself, not the hook
    dev.debug_medium(far)
    dev.close()
    # a homogeneous medium whose free-flight redraw loop (while t < kRayEpsilon) would run about exp(sigma kRayEpsilon) times
    thick = scenes.SceneData()
    m = thick.add_medium(absorption=(5e4, 5e4, 5e4), scattering=(5e4, 5e4, 5e4))
    thick.add_quad([-1, 0, 1], [1, 0, 1], [1, 0, -1], [-1, 0, -1], thick.add_material("floor", kd=[0.5, 0.5, 0.5]))
    light = thick.add_material("light", kd=[0, 0, 0], emission=scenes.spd_rgb_luminance([4.0, 4.0, 4.0]))
    thick.add_quad([-0.2, 2.0, -0.2], [0.2, 2.0, -0.2], [0.2, 2.0, 0.2], [-0.2, 2.0, 0.2], light)
    thick.set_camera([0.0, 1.0, 3.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0], 8, 8, 45.0)
    dev = GPUVCM(thick.finalize(samples=1, spectral=False), flavor="fast")
    q = good.copy()
    q["medium"] = m
    before = dev.counters()["kernel_launches"]
    with pytest.raises(EtxbError):
        dev.debug_medium(q)
    q["op"] = S.MEDIUM_TRANSMITTANCE  # no loop: accepted
    dev.debug_medium(q)
    assert dev.counters()["kernel_launches"] == before + 1
    dev.close()
