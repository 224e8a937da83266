"""The vertex closures of dclosure.cuh (make_closure + closure_evaluate: what the photon gather, the vertex connections and the emitter /
light-to-camera connections of the product build evaluate) against the reference's own bsdf::evaluate + bsdf::reverse_pdf (the oracle,
compiled in place), direction by direction, for every material class, in RGB and spectral, on the product (`fast`) and the strict-IEEE
(`parity`) builds.  The parity build separates restatement errors (algebra, branches, frames) from fast-math rounding.  Run with -m gpu.

Each query is evaluated N times on both sides, repetition r on the sampler (seed, r).  An output is deterministic on a side when its
variance over the repetitions is exactly 0, random otherwise (the microsurface walk; in RGB the thin-film wavelength jitter).
  deterministic on both  per query |gpu - ref| <= rtol |ref| + atol, and gpu == 0 exactly where ref == 0
  random on both         |mean_gpu - mean_ref| <= K sqrt(var_gpu / N + var_ref / N) + rtol |mean_ref|
  random on one side     a failure by itself: a draw or a branch one side does not have (unless its mean is zero on both sides)
  always                 finite wherever the reference is finite, pdf >= 0 and rev_pdf >= 0, func = bsdf = 0 wherever pdf = 0
"Zero" in the support test means at most 1e-6 x rtol of the output's largest reference value (the product build flushes denormal
intermediates).  Where the reference's own evaluation is invalid (pdf 0) but sets a func (TranslucentBSDF at n.w_o = 0), only the pdfs are
compared: every consumer drops an invalid evaluation, and the closure returns zero there.
Queries whose cosine lies within 1e-4 of a kEpsilon test (outside the exact axis-aligned set) or whose arrival direction lies within 1e-3 rad
of the critical angle form the boundary band: there float rounding may legitimately move a result across a threshold, so they keep only
the finiteness / sign / support checks of the last row.  Their number is printed.

Tolerances.  parity: 1e-4 relative (restated formulas differ in association order only).  fast: 1e-3 relative where both cosines are at
least 0.05 (approximate division / square root, special-function-unit transcendentals, the real-arithmetic dielectric Fresnel), 2e-2 in the
grazing range (a cosine below 0.05: 1 / cos and Smith Lambda amplify the relative error of the rounding there).
"""
import numpy as np
import pytest

import closure_queries as cq
from etx_tracer_b200 import scenes, structs as S

pytestmark = pytest.mark.gpu

K_SIGMA = 5.5
REPS_CLOSURE = 1024  # plastic, conductor, dielectric: the walk classes
REPS_OTHER = 256
RTOL = {"parity": 1e-4, "fast": 1e-3}
RTOL_GRAZING = {"parity": 1e-4, "fast": 2e-2}
RTOL_MEAN = {"parity": 1e-5, "fast": 1e-3}
ETA = {"glass": 1.5, "diamond": 2.42, "plastic": 1.5}

MATERIAL_BOX = "material_box"
SKY_ROOM = "sky_room"
# sky_room: textured Lambert floor (scattering image), plastic, conductor with a roughness image: make_closure's lookups at uv
SKY_ROOM_MATERIALS = {"floor": 0, "plastic": 1, "metal": 2}
# the query seeds follow the case's position in this list: the anisotropic kinds come last, so adding them keeps every other case's queries
ANISO_KINDS = [k for k in scenes.MATERIAL_KINDS if k.endswith("_aniso")]
CASES = ([(MATERIAL_BOX, k) for k in sorted(scenes.MATERIAL_KINDS) if k not in ANISO_KINDS] + [(SKY_ROOM, k) for k in sorted(SKY_ROOM_MATERIALS)]
         + [(MATERIAL_BOX, k) for k in ANISO_KINDS])


def _is_closure_class(m):
    cls, variation = int(m["cls"]), int(m["diffuse_variation"])
    return (cls == S.MAT_PLASTIC and variation == 0) or cls in (S.MAT_CONDUCTOR, S.MAT_DIELECTRIC)


_scene_cache = {}
_oracle_cache = {}


def _setup(where, kind, spectral):
    key = (where, kind, spectral)
    if key not in _scene_cache:
        if where == MATERIAL_BOX:
            sd, material = scenes.material_box(kind, spectral=spectral), 4
            spec = scenes.MATERIAL_KINDS[kind]
        else:
            sd, material = scenes.sky_room(spectral=spectral), SKY_ROOM_MATERIALS[kind]
            spec = {}
        m = sd.a_materials[material]
        closure = _is_closure_class(m)
        dielectric = int(m["cls"]) == S.MAT_DIELECTRIC
        alpha = float(max(m["roughness"]["value"][0], m["roughness"]["value"][1]))  # the wider axis steers the lobe set
        eta = ETA.get(spec.get("int_ior"), 1.5)
        q, band = cq.make(material, seed=7919 * (1 + CASES.index((where, kind))) + int(spectral), spectral=spectral, alpha=alpha, eta=eta,
                          dielectric=dielectric, count=48 if closure else 16)
        _scene_cache[key] = (sd, q, band, REPS_CLOSURE if closure else REPS_OTHER)
    return _scene_cache[key]


def _oracle(oracle_mod, key, sd, q, reps):
    if key not in _oracle_cache:
        o = oracle_mod.Oracle(sd)
        _oracle_cache[key] = o.bsdf_eval(q, reps)
        o.close()
    return _oracle_cache[key]


def compare(g, r, q, band, reps, flavor):
    """Every check of the module docstring; returns (failures, report)."""
    ci, co = cq.local(q)
    lowest = np.minimum(np.abs(ci), np.abs(co))
    boundary = ((lowest < 1e-4) & (band != "exact")) | (band == "critical")
    grazing = lowest < 0.05
    fails = []
    for name, col in (("non-finite", 24), ("pdf < 0", 25), ("func / bsdf without pdf", 26)):
        bad = np.flatnonzero((g[:, col] > 0) & (r[:, col] == 0))
        if bad.size:
            fails.append(f"{name} on {bad.size} queries, e.g. {bad[:5].tolist()}")
    # where the reference's evaluation is invalid (pdf 0) its func may still be set (TranslucentBSDF at n.w_o = 0): every consumer drops an
    # invalid evaluation, and the closure returns zero there (checked above through column 26), so only the pdfs are compared
    invalid_ref = r[:, 26] == reps
    rel_max, z_max, det_n, rnd_n, mismatch = 0.0, 0.0, 0, 0, 0
    for k, out in enumerate(S.CLOSURE_OUTPUTS):
        mg, mr, vg, vr = g[:, k], r[:, k], g[:, 8 + k], r[:, 8 + k]
        finite = np.isfinite(mr) & (r[:, 24] == 0) & (g[:, 24] == 0) & ~boundary & ~(invalid_ref & (k < 6))
        det_g, det_r = vg == 0, vr == 0
        scale = np.abs(mr[finite]).max() if finite.any() else 0.0
        tol_r = np.where(grazing, RTOL_GRAZING[flavor], RTOL[flavor])
        atol = 1e-6 * tol_r * scale  # values this far below the output's largest are "zero" (flushed denormal intermediates)
        # one side draws where the other does not (an output that is zero on both sides in that sense is not random on either)
        odd = np.flatnonzero(finite & (det_g != det_r) & ~((np.abs(mg) <= atol) & (np.abs(mr) <= atol)))
        mismatch += odd.size
        for i in odd[:3]:
            fails.append(f"{out}: q{i} ({band[i]}) random on {'gpu' if det_r[i] else 'reference'} only: gpu {mg[i]:.6g}/{vg[i]:.3g}, ref {mr[i]:.6g}/{vr[i]:.3g}")
        det = finite & det_g & det_r
        det_n += int(det.sum())
        support = np.flatnonzero(det & ((np.abs(mg) <= atol) != (np.abs(mr) <= atol)))
        for i in support[:3]:
            fails.append(f"{out}: q{i} ({band[i]}) support differs: gpu {mg[i]:.6g}, ref {mr[i]:.6g}")
        err = np.abs(mg - mr)
        bad = np.flatnonzero(det & (err > tol_r * np.abs(mr) + atol))
        for i in bad[:3]:
            fails.append(f"{out}: q{i} ({band[i]}, min |cos| {lowest[i]:.3g}) gpu {mg[i]:.8g} ref {mr[i]:.8g} rel {err[i] / max(abs(mr[i]), 1e-30):.3g}")
        if det.any():
            nz = det & (mr != 0)
            if nz.any():
                rel_max = max(rel_max, float((err[nz] / np.abs(mr[nz])).max()))
        rnd = finite & ~det_g & ~det_r
        rnd_n += int(rnd.sum())
        sigma = np.sqrt(vg / reps + vr / reps)
        bad = np.flatnonzero(rnd & (err > K_SIGMA * sigma + RTOL_MEAN[flavor] * np.abs(mr)))
        for i in bad[:3]:
            fails.append(f"{out}: q{i} ({band[i]}) mean gpu {mg[i]:.6g} ref {mr[i]:.6g}, z = {err[i] / sigma[i]:.2f}")
        if rnd.any():
            z_max = max(z_max, float((err[rnd] / sigma[rnd]).max()))
    rep0 = np.abs(g[:, 16:24] - r[:, 16:24]) <= 1e-4 * np.abs(r[:, 16:24]) + 1e-12
    report = dict(queries=q.shape[0], deterministic=det_n, random=rnd_n, boundary=int(boundary.sum()), max_rel=rel_max, max_z=z_max,
                  rep0_agree=float(rep0.all(axis=1).mean()), random_on_one_side=mismatch, invalid_ref=int(invalid_ref.sum()))
    return fails, report


@pytest.fixture(scope="module")
def bsdf_oracle(oracle_mod):
    if not oracle_mod.has_bsdf_eval():
        pytest.skip("oracle/_ref predates oracle_bsdf_eval (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


@pytest.mark.parametrize("flavor", ["fast", "parity"])
@pytest.mark.parametrize("spectral", [False, True], ids=["rgb", "spectral"])
@pytest.mark.parametrize("where,kind", CASES, ids=[f"{w}-{k}" for w, k in CASES])
def test_closure_matches_reference_bsdf(bsdf_oracle, where, kind, spectral, flavor):
    oracle_mod = bsdf_oracle
    from etx_tracer_b200.api import GPUVCM
    sd, q, band, reps = _setup(where, kind, spectral)
    r = _oracle(oracle_mod, (where, kind, spectral), sd, q, reps)
    dev = GPUVCM(sd, flavor=flavor)
    g = dev.debug_closure(q, reps)
    dev.close()
    fails, rep = compare(g, r, q, band, reps, flavor)
    print(f"\n[closure] {where}/{kind}/{'spectral' if spectral else 'rgb'}/{flavor}: {rep['queries']} queries x {reps}; "
          f"deterministic {rep['deterministic']} (max rel {rep['max_rel']:.3e}), random {rep['random']} (max z {rep['max_z']:.2f}), "
          f"boundary band {rep['boundary']}, reference value without pdf {rep['invalid_ref']}, repetition 0 agrees on {100 * rep['rep0_agree']:.1f} %")
    assert not fails, f"{len(fails)} findings:\n  " + "\n  ".join(fails[:24])
