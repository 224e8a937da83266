"""The oracle's BSDF export (oracle_bsdf_eval: the reference's bsdf::evaluate + bsdf::reverse_pdf compiled in place) against plain float64
formulas, on the query sets of closure_queries.py.  This pins the side the GPU closure tests compare against, and rehearses the query
conventions: the shading frame as interpolated, w_i pointing AT the surface, the reversed pair (w_i' = -w_o, w_o' = -w_i), the path source.
Runs without a GPU."""
import numpy as np
import pytest

import closure_queries as cq
from etx_tracer_b200 import scenes, structs as S

K_EPSILON = 1.192092896e-07
REPS = 4
RTOL = 2e-5


def _frame_local(q, v):
    v = v.astype(np.float64)
    return np.stack([(v * q[f].astype(np.float64)).sum(1) for f in ("tan", "btn", "nrm")], axis=1)


def _lambda(w, alpha):
    """RayInfo::updateDirection (bsdf_external.hxx:28-51)."""
    out = np.empty(w.shape[0])
    for i, (x, y, z) in enumerate(w):
        if z > 0.9999:
            out[i] = 0.0
        elif z < -0.9999:
            out[i] = -1.0
        else:
            s2 = 1.0 - z * z
            tan_t = np.sqrt(s2) / z
            av = np.sqrt((x * x / s2) * alpha[0] ** 2 + (y * y / s2) * alpha[1] ** 2)
            a = 1.0 / tan_t / av
            out[i] = 0.5 * (-1.0 + np.sign(a) * np.sqrt(1.0 + 1.0 / (a * a)))
    return out


def _d_ggx(wm, alpha):
    """D_ggx (bsdf_external.hxx:105-126)."""
    ax, ay, axy = (max(K_EPSILON, v) for v in (alpha[0] ** 2, alpha[1] ** 2, alpha[0] * alpha[1]))
    z = np.where(wm[:, 2] > K_EPSILON, wm[:, 2], 1.0)
    sx, sy = -wm[:, 0] / z, -wm[:, 1] / z
    tmp = 1.0 + sx * sx / ax + sy * sy / ay
    return np.where(wm[:, 2] > K_EPSILON, 1.0 / (np.pi * axy * tmp * tmp) / z ** 4, 0.0)


def _conductor_pdf(wi_l, wo_l, alpha):
    """ConductorBSDF::pdf (bsdf_conductor.hxx:106-126) on local directions already flipped towards the incoming side."""
    h = wi_l + wo_l
    h /= np.linalg.norm(h, axis=1, keepdims=True)
    p = _d_ggx(h, alpha) / (1.0 + _lambda(wi_l, alpha)) / (4.0 * wi_l[:, 2]) + wo_l[:, 2]
    return np.where((wi_l[:, 2] > K_EPSILON) & (wo_l[:, 2] > K_EPSILON), p, 0.0)


def _expected(q, kind, alpha):
    nrm = q["nrm"].astype(np.float64)
    w_i, w_o = q["w_i"].astype(np.float64), q["w_o"].astype(np.float64)
    entering = (nrm * w_i).sum(1) < 0.0        # the frame faces -w_i (BSDFData::get_normal_frame)
    entering_rev = (nrm * w_o).sum(1) > 0.0    # the reversed pair's incoming direction is -w_o
    s, s_rev = np.where(entering, 1.0, -1.0)[:, None], np.where(entering_rev, 1.0, -1.0)[:, None]
    if kind == "lambert":
        cos_o = s[:, 0] * (nrm * w_o).sum(1)
        cos_rev = s_rev[:, 0] * (nrm * -w_i).sum(1)
        pdf = np.where(cos_o > K_EPSILON, cos_o / np.pi, 0.0)
        rev = np.where(cos_rev > K_EPSILON, cos_rev / np.pi, 0.0)
    else:
        pdf = _conductor_pdf(_frame_local(q, -w_i) * s, _frame_local(q, w_o) * s, alpha)
        rev = _conductor_pdf(_frame_local(q, w_o) * s_rev, _frame_local(q, -w_i) * s_rev, alpha)
    return pdf, np.where(pdf > 0.0, rev, 0.0)  # reverse_pdf is only asked where the evaluation is valid


CASES = {
    # label: (scene factory, material index, kind)
    "lambert": (lambda sp: scenes.material_box("plastic", spectral=sp), 0, "lambert"),
    "conductor_rough": (lambda sp: scenes.material_box("conductor_rough", spectral=sp), 4, "conductor"),
    "conductor_thinfilm": (lambda sp: scenes.material_box("conductor_thinfilm", spectral=sp), 4, "conductor"),
}


@pytest.fixture(scope="module")
def bsdf_oracle(oracle_mod):
    if not oracle_mod.has_bsdf_eval():
        pytest.skip("oracle/_ref predates oracle_bsdf_eval (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


@pytest.mark.parametrize("spectral", [False, True], ids=["rgb", "spectral"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_bsdf_pdfs_match_float64_formulas(bsdf_oracle, case, spectral):
    oracle_mod = bsdf_oracle
    factory, material, kind = CASES[case]
    sd = factory(spectral)
    m = sd.a_materials[material]
    alpha = (float(m["roughness"]["value"][0]), float(m["roughness"]["value"][1]))
    q, band = cq.make(material, seed=1000 + material, spectral=spectral, alpha=alpha[0])
    o = oracle_mod.Oracle(sd)
    st = o.bsdf_eval(q, REPS)
    o.close()
    with np.errstate(all="ignore"):  # degenerate half vectors and normal incidence: the kEpsilon tests discard those terms
        pdf_ref, rev_ref = _expected(q, kind, alpha)
    ci, co = cq.local(q)
    edge = np.minimum(np.abs(ci), np.abs(co)) < 1e-5  # the kEpsilon tests: float32 inputs may land either side
    assert (st[:, 24:27] == 0).all(), "non-finite, negative or unsupported outputs"
    assert (st[:, 8 + 6] == 0).all() and (st[:, 8 + 7] == 0).all(), "pdf / rev_pdf vary with the sampler"
    for name, got, want in (("pdf", st[:, 6], pdf_ref), ("rev_pdf", st[:, 7], rev_ref)):
        assert ((got > 0) == (want > 0))[~edge].all(), f"{name}: support differs on {np.flatnonzero(((got > 0) != (want > 0)) & ~edge)[:8]}"
        ok = np.abs(got - want) <= RTOL * np.abs(want) + 1e-6 * max(1.0, np.abs(want).max() * 1e-3)
        bad = np.flatnonzero(~ok & ~edge)
        assert bad.size == 0, f"{name}: {bad.size} queries off, worst {[(band[i], got[i], want[i]) for i in bad[:5]]}"
    # the value is zero exactly where the pdf is (the oracle's own evaluate: pdf == 0 -> func == bsdf == 0)
    assert (st[:, 16:22][st[:, 22] == 0] == 0).all()
    print(f"\n[oracle bsdf] {case}/{'spectral' if spectral else 'rgb'}: {q.shape[0]} queries, {int((pdf_ref > 0).sum())} in the support, {int(edge.sum())} in the kEpsilon band")
