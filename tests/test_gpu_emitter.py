"""The emitter routines of dvcm.cuh (emitter selection, sample_emitter for next-event estimation, sample_emission at the start of every
light path, emitter_get_radiance when a path hits an emitter or escapes) against the reference's own routines (the oracle, compiled in
place), for every emitter form of emitter_queries.CASES, RGB and spectral, on the product (`fast`) and the strict-IEEE (`parity`) builds.
Run with -m gpu.

(a) per query (emitter_queries.make; emission_queries with EMISSION_REPS repetitions on the samplers (seed, r))
  parity   every word of every record bit for bit (a NaN matches a NaN)
  fast     indices, flags and sampler states equal; every other field within the bounds below, which are looser only for the
           fields and bands they are argued for; zero exactly where the reference is zero, except on a cone's edge, where the
           approximate dot product may land on either side.  A non-finite output where the reference's is finite fails in every band.
(b) as a distribution, per distant emitter of angular size > 0: N_DIST sample_in and N_DIST emission samples, binned by environment pixel
  (the true inverse of uv_to_direction) or by (r^2, phi) of a directional emitter's disk.  The device's counts are held to the float64
  pixel model of test_oracle_emitter.py (binomial, K_SIGMA) and to the oracle's paired samples (per bin, |mean difference| <= K_SIGMA
  sigma / sqrt(N) + 1e-3 |reference mean|, as test_gpu_bsdf_sample.compare_distribution).
(c) sample and evaluate agree: for every valid non-delta sample_in, the device's own radiance op at the sampled direction (from the sampled
  origin, for area emitters) reproduces the sample's pdf_dir and value within 1e-3 relative, 2e-2 in the first and last image rows.  The
  mirrored-and-rotated environment is the exception the reference defines (DESIGN §10); test_oracle_emitter.py pins it.  Environment
  samples within float32 rounding of a texel-row edge, of the u seam or of a pole are left out: the reference's pdf jumps there.
"""
import numpy as np
import pytest

import emitter_queries as eq
from etx_tracer_b200 import structs as S

pytestmark = pytest.mark.gpu

K_SIGMA = 5.5
EMISSION_REPS = 256
N_DIST = 1 << 17
# The product build's bounds (a).  Measured on an H100 80GB HBM3 at 700 W (DESIGN §3); each bound is about twice the worst measured value.
#   every field          RTOL relative, MAX_ANGLE for directions and normals, FTZ_ATOL absolute (-ftz flushes denormals); zero where the
#                        reference is zero and non-zero where it is not
#   pdf_dir, pdf_dir_out within 1e-4 of an area emitter (band near): RTOL_NEAR, the distance and cosine of nearby float32 points cancel
#                        collimated area emitters: a ratio within exp(COS_ABS x the exponent), the rounding of a float32 cosine
#                        raised to that power (at collimation 1, 8.4e6: a factor of 67, so there only zero against non-zero counts)
#                        The relative bounds of the two pdfs hold in both directions: gpu / ref and ref / gpu within 1 + bound.
#                        environment: SIN_ABS / sin(angle to the pole), the approximate sine's absolute error over the clamped sin_t;
#                        within POLE_FREE rad of a pole and on texel edges (cdf_edge) finiteness only: the reference's pdf divides by a
#                        sine clamped to kEpsilon there, or jumps across a texel-row edge, so a rounding changes it by any factor
#   sample_emission's direction at collimation 0.9 and 1: MAX_ANGLE_LOBE (an ulp of a sampled cosine next to 1 is 3.45e-4 rad)
#   origin               ORIGIN_ATOL_AREA, ORIGIN_ATOL_DISTANT (distance_to_sphere cancels near the bounding sphere), either root
#                        from a point on the sphere; barycentric BARY_ATOL
MAX_ANGLE, RTOL, FTZ_ATOL = 1e-4, 1e-4, 1e-30        # measured 1.3e-5 rad, 1.9e-5
RTOL_NEAR = 0.12                                     # measured 5.6e-2
COS_ABS = 5e-7                                       # measured 1.65e-7 at collimation 0.9, 2.5e-7 at 1 (a factor 8.4)
SIN_ABS = 1.1e-4                                     # measured 5.3e-5
POLE_FREE = 1e-3
MAX_ANGLE_LOBE = 7e-4                                # measured 3.45e-4
ORIGIN_ATOL_AREA, ORIGIN_ATOL_DISTANT, BARY_ATOL = 4e-7, 2.5e-4, 1.2e-7  # measured 1.8e-7, 1.2e-4, 6e-8
EDGE_VALUE_REL = 4e-6                                # about an ulp of a texel coordinate (32 texels) times the largest value
RTOL_EVAL, RTOL_EVAL_POLAR = 1e-3, 2e-2
CASES = [(c, sp, fl) for c in eq.CASES for sp in (False, True) for fl in ("fast", "parity")]
WORDS = S.EMITTER_RESULT.itemsize // 4

_cache = {}


def _setup(oracle_mod, case, spectral):
    key = (case, spectral)
    if key not in _cache:
        _cache.clear()
        sd = eq.scene(case, spectral)
        index = eq.CASES.index(case)
        q, band = eq.make(sd, case, spectral, seed=4001 * (1 + index) + int(spectral))
        qe = eq.emission_queries(5003 * (1 + index) + int(spectral), spectral)
        o = oracle_mod.Oracle(sd)
        ref, ref_e = o.emitter(q, 1), o.emitter(qe, EMISSION_REPS)
        dist = None
        if _distributed(sd):
            qd = eq.distribution_queries(sd, spectral, seed=6007 * (1 + index) + int(spectral), n=N_DIST)
            qde = eq.emission_queries(7001 * (1 + index) + int(spectral), spectral, count=1)
            dist = (qd, qde, o.emitter(qd, 1)[:, 0], o.emitter(qde, N_DIST)[0])
        o.close()
        _cache[key] = (sd, q, band, qe, ref, ref_e, dist)
    return _cache[key]


def _distributed(sd):
    cls = int(sd.a_emitters["cls"][0])
    return cls == S.EMITTER_ENVIRONMENT or (cls == S.EMITTER_DIRECTIONAL and float(sd.a_profiles["angular_size"][0]) > 0)


def _angle(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=-1), (a * b).sum(-1))


def compare(g, r, band, case, flavor, query_directions, sources, emission=False):
    """(a) on records of the same shape; returns (failures, report): bit-exact count and, per band, the worst angle, relative error (of the
    fields held relatively) and position error"""
    fails = []
    wg = np.ascontiguousarray(g).view(np.uint32).reshape(g.shape + (WORDS,))
    wr = np.ascontiguousarray(r).view(np.uint32).reshape(r.shape + (WORDS,))
    exact = (wg == wr).all(-1)
    report = {"records": int(g.size), "bit_exact": int(exact.sum()), "bands": {}}
    band = np.broadcast_to(band.reshape(band.shape + (1,) * (g.ndim - 1)), g.shape)
    sources = np.broadcast_to(sources.reshape(sources.shape[:1] + (1,) * (g.ndim - 1) + (3,)), g.shape + (3,)).astype(np.float64)
    query_directions = np.broadcast_to(query_directions.reshape(query_directions.shape[:1] + (1,) * (g.ndim - 1) + (3,)), g.shape + (3,))
    if flavor == "parity":
        for idx in np.argwhere(~exact)[:6]:
            i = tuple(idx)
            fails.append(f"{i} ({band[i]}): gpu {g[i]} ref {r[i]}")
        return fails, report
    for f in ("emitter_index", "triangle_index", "medium_index", "flags", "seed_start", "seed_end"):
        for idx in np.argwhere(g[f] != r[f])[:3]:
            fails.append(f"{f} {tuple(idx)} ({band[tuple(idx)]}): gpu {g[tuple(idx)]} ref {r[tuple(idx)]}")
    floats = ("value", "origin", "normal", "direction", "barycentric", "pdf_sample", "pdf_area", "pdf_dir", "pdf_dir_out")
    finite = lambda x: np.stack([np.isfinite(x[f]).reshape(x.shape + (-1,)).all(-1) for f in floats], -1).all(-1)
    fg, fr = finite(g), finite(r)
    for idx in np.argwhere(fr & ~fg)[:4]:
        fails.append(f"non-finite {tuple(idx)} ({band[tuple(idx)]}): gpu {g[tuple(idx)]} where the reference's is finite")
    ok = fg & fr
    env, area = case in eq.ENV_CASES, case in eq.AREA_CASES
    # the relative bound of pdf_dir and pdf_dir_out, per record (module docstring); every other field is held to RTOL
    pdf_tol = np.full(g.shape, RTOL)
    pdf_free = np.zeros(g.shape, bool)
    if area:
        pdf_tol = np.where(band == "near", RTOL_NEAR, np.maximum(pdf_tol, np.expm1(COS_ABS * eq.collimation_exponent(eq.AREA_CASES[case]))))
    if env:
        d = np.where((r["direction"] == 0).all(-1, keepdims=True), query_directions, r["direction"]).astype(np.float64)
        pole = np.arccos(np.clip(np.abs(d[..., 1]) / np.maximum(np.linalg.norm(d, axis=-1), 1e-30), 0.0, 1.0))
        pdf_tol = np.maximum(pdf_tol, SIN_ABS / np.maximum(np.sin(pole), 1e-30))
        pdf_free = (pole < POLE_FREE) | (band == "cdf_edge")
    max_angle = MAX_ANGLE_LOBE if (emission and area and eq.AREA_CASES[case] >= 0.9) else MAX_ANGLE
    angle = np.maximum(_angle(g["direction"], r["direction"]), _angle(g["normal"], r["normal"]))
    rel, pos_err = np.zeros(g.shape), np.zeros(g.shape)
    off = {"direction / normal": ok & (angle > max_angle)}
    edge_value_atol = EDGE_VALUE_REL * (np.abs(r["value"][ok]).max() if ok.any() else 0.0)
    for f in ("value", "pdf_sample", "pdf_area", "pdf_dir", "pdf_dir_out", "origin", "barycentric"):
        vg, vr = g[f].astype(np.float64).reshape(g.shape + (-1,)), r[f].astype(np.float64).reshape(r.shape + (-1,))
        err = np.abs(vg - vr)
        if f in ("origin", "barycentric"):
            atol = BARY_ATOL if f == "barycentric" else (ORIGIN_ATOL_AREA if area else ORIGIN_ATOL_DISTANT)
            bad = (err > atol).any(-1)
            if f == "origin" and not area:
                # from a point on the bounding sphere distance_to_sphere has a root at 0: a rounding picks it or the far side
                c, radius = eq.bounding_sphere(case)
                on_ray_end = (np.linalg.norm(vg - sources, axis=-1) < atol) | (np.abs(np.linalg.norm(vg - c, axis=-1) - radius) < atol)
                bad &= ~((band == "near") & on_ray_end)
                err = np.where(((band == "near") & on_ray_end)[..., None], 0.0, err)
            off[f] = ok & bad
            pos_err = np.maximum(pos_err, np.where(ok & ~bad, err.max(-1), 0.0))
            continue
        tol = pdf_tol if f in ("pdf_dir", "pdf_dir_out") else np.full(g.shape, RTOL)
        atol = np.full(g.shape, FTZ_ATOL)
        if f == "value" and env:  # a lookup on a texel edge beside a black texel takes a rounding-sized share of its neighbour
            atol = np.where(band == "cdf_edge", edge_value_atol, atol)
        flip = ((vr == 0) & (np.abs(vg) > atol[..., None])) | ((vr != 0) & (vg == 0) & (np.abs(vr) > atol[..., None]))
        scale = np.minimum(np.abs(vr), np.abs(vg)) if f in ("pdf_dir", "pdf_dir_out") else np.abs(vr)
        bad = ((err > tol[..., None] * scale + atol[..., None]) | flip).any(-1)
        if f in ("pdf_dir", "pdf_dir_out"):
            bad &= ~pdf_free
        # a cone's edge: the approximate dot product may put the direction on the other side (value and pdf 0 on one side only)
        other_side = np.zeros(g.shape, bool)
        if f in ("value", "pdf_area", "pdf_dir", "pdf_dir_out"):
            other_side = (band == "cone_edge") & ((vr == 0).all(-1) != (vg == 0).all(-1))
            bad &= ~other_side
        off[f] = ok & bad
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.where(ok[..., None] & (vr != 0), err / np.abs(vr), 0.0).max(-1)
        e = np.where(other_side | (pdf_free if f in ("pdf_dir", "pdf_dir_out") else False), 0.0, e)
        rel = np.maximum(rel, e)
    for name, v in off.items():
        for idx in np.argwhere(v)[:3]:
            i = tuple(idx)
            fails.append(f"{name} {i} ({band[i]}): gpu {g[i]} ref {r[i]}")
    for b in eq.BANDS:
        m = ok & (band == b)
        if m.any():
            report["bands"][b] = (float(angle[m].max()), float(rel[m].max()), float(pos_err[m].max()))
    return fails, report


def _bins(sd, d):
    """environment: the pixel of each direction's true uv; directional: 16 x 8 (r^2, phi) bins of the disk"""
    if int(sd.a_emitters["cls"][0]) == S.EMITTER_ENVIRONMENT:
        return eq.pixel_of(sd, d), eq.pixel_model(sd).reshape(-1)
    em_dir = sd.a_profiles["direction"][0].astype(np.float64)
    u, v = eq._basis(em_dir)
    d = d.astype(np.float64)
    r2 = (np.hypot(d @ u, d @ v) / (d @ em_dir) / np.tan(0.5 * float(sd.a_profiles["angular_size"][0]))) ** 2
    phi = np.arctan2(d @ v, d @ u)
    b = np.minimum((r2 * 16).astype(np.int64), 15) * 8 + np.minimum(((phi + np.pi) / (2 * np.pi) * 8).astype(np.int64), 7)
    return b, np.full(128, 1.0 / 128)


def compare_distribution(sd, g_dirs, r_dirs, what):
    """(b): device counts against the float64 model and against the oracle's paired samples; returns (failures, worst z)"""
    fails = []
    bg, p = _bins(sd, g_dirs)
    br, _ = _bins(sd, r_dirs)
    n, nb = bg.shape[0], p.shape[0]
    counts = np.bincount(bg, minlength=nb).astype(np.float64)
    sigma_model = np.sqrt(n * p * (1.0 - p))
    for b in np.flatnonzero(np.abs(counts - n * p) > K_SIGMA * sigma_model + 2.0)[:3]:
        fails.append(f"{what}: bin {b} count {counts[b]:.0f}, model {n * p[b]:.1f} (sigma {sigma_model[b]:.2f})")
    same = bg == br
    mean = (counts - np.bincount(br, minlength=nb)) / n
    sq = (np.bincount(bg[~same], minlength=nb) + np.bincount(br[~same], minlength=nb)) / n
    sigma = np.sqrt(np.maximum(sq - mean ** 2, 0.0))
    ref_mean = np.bincount(br, minlength=nb) / n
    for b in np.flatnonzero(np.abs(mean) > K_SIGMA * sigma / np.sqrt(n) + 1e-3 * ref_mean)[:3]:
        fails.append(f"{what}: bin {b} paired mean difference {mean[b]:.4g} (reference {ref_mean[b]:.4g})")
    with np.errstate(divide="ignore", invalid="ignore"):
        z = np.where(sigma > 0, np.abs(mean) / (sigma / np.sqrt(n)), 0.0)
        z_model = np.where(sigma_model > 0, np.abs(counts - n * p) / sigma_model, 0.0)
    return fails, float(max(z.max(), z_model.max()))


def compare_with_evaluate(dev, sd, case, q, g):
    """(c): returns (failures, checked, largest relative pdf gap)"""
    s = (q["op"] == S.EMITTER_SAMPLE_IN) & (g["pdf_dir"] > 0) & ((g["flags"] & S.EMITTER_FLAG_DELTA) == 0) & np.isfinite(g["pdf_dir"])
    if not s.any():
        return [], 0, 0.0
    gs = g[s]
    e = np.zeros(gs.shape[0], dtype=S.EMITTER_QUERY)
    e["op"], e["emitter"], e["wavelength"] = S.EMITTER_RADIANCE, q["emitter"][s], q["wavelength"][s]
    area = int(sd.a_emitters["cls"][0]) == S.EMITTER_AREA
    if area:
        # sample_emitter itself calls emitter_get_radiance with this source, target and uv: for area emitters (c) only confirms that
        # the op passes them through; its content is the environment round trip below
        e["source"], e["target"], e["uv"] = q["source"][s], gs["origin"], eq.area_uv(gs)
        polar = np.zeros(gs.shape[0], bool)
    else:
        e["direction"] = gs["direction"]
        rec, _, _ = eq.env_image(sd)
        w, h = float(rec["fsize"][0]), float(rec["fsize"][1])
        uv = eq.true_uv(gs["direction"], float(rec["offset"][0]), float(rec["scale"][0]))
        polar = (uv[:, 1] < 1.0 / h) | (uv[:, 1] > 1.0 - 1.0 / h)
        # the reference's pdf jumps where a lookup crosses a row edge (Image::evaluate weights the upper texel row by sin at v and the
        # lower by sin at v + 1/h) or the u seam (the column after the last is clamped, not wrapped), and its sin_t clamp makes it
        # arbitrarily steep within 1e-4 of a pole: a sample within float32 rounding of these is not held to its lookup
        row_edge = np.abs(uv[:, 1] * h - np.round(uv[:, 1] * h)) < 1e-4 * h if h > 1 else np.zeros(uv.shape[0], bool)
        seam = np.minimum(uv[:, 0], 1.0 - uv[:, 0]) * w < 1e-4
        pole = np.minimum(uv[:, 1], 1.0 - uv[:, 1]) < 1e-4
        skip = row_edge | seam | pole
        gs, e, polar = gs[~skip], e[~skip], polar[~skip]
    if gs.shape[0] == 0:
        return [], 0, 0.0
    ev = dev.debug_emitter(e)[:, 0]
    tol = np.where(polar, RTOL_EVAL_POLAR, RTOL_EVAL)
    gap = np.abs(ev["pdf_dir"].astype(np.float64) - gs["pdf_dir"]) / gs["pdf_dir"]
    vs = gs["value"].astype(np.float64)
    vgap = (np.abs(ev["value"] - vs) / np.maximum(np.abs(vs), 1e-30)).max(-1)
    fails = [f"sample {gs[j]}: evaluate pdf {ev['pdf_dir'][j]:.8g} value {ev['value'][j]}" for j in np.flatnonzero((gap > tol) | (vgap > tol))[:4]]
    return fails, int(gs.shape[0]), float(max(gap.max(), vgap.max()))


@pytest.fixture(scope="module")
def emitter_oracle(oracle_mod):
    if not oracle_mod.has_emitter():
        pytest.skip("oracle/_ref predates oracle_emitter (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


@pytest.mark.parametrize("case,spectral,flavor", CASES, ids=[f"{c}-{'spectral' if sp else 'rgb'}-{fl}" for c, sp, fl in CASES])
def test_emitter_matches_reference(emitter_oracle, case, spectral, flavor):
    from etx_tracer_b200.api import GPUVCM
    sd, q, band, qe, ref, ref_e, dist = _setup(emitter_oracle, case, spectral)
    dev = GPUVCM(sd, flavor=flavor)
    g, g_e = dev.debug_emitter(q), dev.debug_emitter(qe, EMISSION_REPS)
    fails, rep = compare(g, ref, band, case, flavor, q["direction"], q["source"])
    fails_e, rep_e = compare(g_e, ref_e, np.full(qe.shape[0], "uniform", dtype=object), case, flavor, qe["direction"], qe["source"], emission=True)
    fails += fails_e
    z_max = 0.0
    if dist is not None:
        qd, qde, ref_d, ref_de = dist
        g_d, g_de = dev.debug_emitter(qd)[:, 0], dev.debug_emitter(qde, N_DIST)[0]
        for what, gd, rd in (("sample_in", g_d["direction"], ref_d["direction"]), ("emission", -g_de["direction"], -ref_de["direction"])):
            keep = np.isfinite(gd).all(-1) & (np.abs(gd).sum(-1) > 0) & (np.abs(rd).sum(-1) > 0)
            f, z = compare_distribution(sd, gd[keep], rd[keep], what)
            fails += f
            z_max = max(z_max, z)
    elif int(sd.a_emitters["cls"][0]) == S.EMITTER_DIRECTIONAL:
        s = q["op"] == S.EMITTER_SAMPLE_IN
        if not (g["direction"][s, 0] == sd.a_profiles["direction"][0]).all():
            fails.append("a delta directional emitter sampled a direction other than its own")
    checked, gap = 0, 0.0
    if case != "env_mirrored_rotated":
        f, checked, gap = compare_with_evaluate(dev, sd, case, q, g[:, 0])
        fails += f
    dev.close()
    bands = ", ".join(f"{b} {a:.2e} rad / {r:.2e} rel / {o:.2e} abs" for b, (a, r, o) in rep["bands"].items())
    print(f"\n[emitter] {case}/{'spectral' if spectral else 'rgb'}/{flavor}: bit-exact {rep['bit_exact'] + rep_e['bit_exact']} of "
          f"{rep['records'] + rep_e['records']}; worst per band: {bands or '-'}; emission {rep_e['bands'].get('uniform', (0.0, 0.0, 0.0))}; "
          f"worst bin z {z_max:.2f}; sample/evaluate on {checked} samples, largest gap {gap:.3e}")
    assert not fails, f"{len(fails)} findings:\n  " + "\n  ".join(fails[:24])
