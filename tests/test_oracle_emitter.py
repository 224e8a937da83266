"""The oracle's emitter export (oracle_emitter: the reference's sample_emitter_index, sample_emitter, sample_emission and
emitter_get_radiance compiled in place) against plain float64 models, on the scenes and queries of emitter_queries.py.  This pins the side
the GPU emitter test compares against: the area, directional and environment pdfs, the emitter selection, the environment sampling tables
with their offset and mirroring, the normalisation of the environment pdf, and the reference's mirrored-and-rotated round trip
(DESIGN §10).  Runs without a GPU."""
import numpy as np
import pytest

import emitter_queries as eq
from etx_tracer_b200 import structs as S

K_SIGMA = 5.5
K_EPSILON = 1.192092896e-07
N_HIST = 1 << 17

# |integral of pdf_dir over the sphere - 1| per environment case.  The bilinear pdf of Image::evaluate is not exactly the sampled density
# (its two rows are weighted by sin at v and at v + 1/h, not at the texel centres), so the integral is not 1.  Measured on the query
# scenes' 32 x 16 images (1024 x 512 midpoint quadrature in uv): 4.65e-2 for plain, rotated, mirrored and mirrored-rotated, 5.41e-2
# black, 4.89e-2 RGBA8, 1.3e-3 the single row (flat pdf), 4e-6 the placeholder.  The bounds are about twice that.
NORMALISATION_BOUND = {"env_black": 0.11, "env_single_row": 3e-3, "env_placeholder": 1e-5}
NORMALISATION_BOUND_DEFAULT = 0.1


@pytest.fixture(scope="module")
def emitter_oracle(oracle_mod):
    if not oracle_mod.has_emitter():
        pytest.skip("oracle/_ref predates oracle_emitter (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


def _run(oracle_mod, sd, q, reps=1):
    o = oracle_mod.Oracle(sd)
    r = o.emitter(q, reps)
    o.close()
    return r if reps > 1 else r[:, 0]


def _binomial(counts, p, n, what):
    """each count within K_SIGMA binomial sigma of n p, plus 2 samples: a direction on a pixel edge may round into its neighbour"""
    sigma = np.sqrt(n * p * (1.0 - p))
    bad = np.flatnonzero(np.abs(counts - n * p) > K_SIGMA * sigma + 2.0)
    return [f"{what}: bin {b} count {counts[b]} expected {n * p[b]:.1f} (sigma {sigma[b]:.2f})" for b in bad[:6]]


@pytest.mark.parametrize("case", list(eq.AREA_CASES))
def test_area_pdfs_follow_the_float64_model(emitter_oracle, case):
    sd = eq.scene(case, False)
    q, band = eq.make(sd, case, False, seed=11)
    r = _run(emitter_oracle, sd, q)
    exponent = 1.0 / max(K_EPSILON, (1.0 - eq.AREA_CASES[case]) ** 4)
    # float32 cosines carry a few ulp; the power raises their relative error by the exponent
    rtol = 1e-5 + 6e-7 * exponent
    fails = []
    for op in (S.EMITTER_SAMPLE_IN, S.EMITTER_RADIANCE):
        m = q["op"] == op
        qq, rr = q[m], r[m]
        tri = np.array([eq._TRIANGLES[e] for e in qq["emitter"]], np.float64)
        area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
        src = qq["source"].astype(np.float64)
        tgt = rr["origin"].astype(np.float64) if op == S.EMITTER_SAMPLE_IN else qq["target"].astype(np.float64)
        visible = (qq["directly_visible"] != 0) & (op == S.EMITTER_RADIANCE)
        geo_n = np.array([0.0, -1.0, 0.0])
        back = (tgt - src) @ geo_n >= 0.0
        d2 = ((src - tgt) ** 2).sum(1)
        cos_t = np.abs((src - tgt) @ geo_n) / np.sqrt(d2)
        cos_tx = np.where(visible, cos_t, cos_t ** exponent)
        lit = ~back & (cos_tx > K_EPSILON)
        pdf_area = np.where(back, 0.0, 1.0 / area)
        pdf_dir = np.where(lit, pdf_area * d2 / np.maximum(cos_tx, 1e-300), 0.0)
        pdf_dir_out = np.where(lit, pdf_area * cos_tx / np.pi, 0.0)
        # where cos_tx is within the rounding of the kEpsilon threshold either decision is right
        with np.errstate(divide="ignore"):
            near_threshold = ~back & (np.abs(np.log(np.maximum(cos_tx, 1e-300) / K_EPSILON)) < rtol * 4)
        tol = np.where(visible, 1e-5, rtol)
        for name, model in (("pdf_area", pdf_area), ("pdf_dir", pdf_dir), ("pdf_dir_out", pdf_dir_out)):
            got = rr[name].astype(np.float64)
            off = (np.abs(got - model) > tol * np.abs(model)) | ((model == 0) != (got == 0))
            off &= ~near_threshold if name != "pdf_area" else True
            for i in np.flatnonzero(off)[:4]:
                fails.append(f"op {op} {name} ({band[m][i]}, visible {visible[i]}): oracle {got[i]:.8g} model {model[i]:.8g} cos_t {cos_t[i]:.9f}")
        zero = back & ((rr["value"] != 0).any(-1) | (rr["pdf_dir"] != 0))
        for i in np.flatnonzero(zero)[:2]:
            fails.append(f"op {op}: value or pdf on the back side: {rr[i]}")
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("case", list(eq.DIR_CASES))
def test_directional_pdfs_and_disk(emitter_oracle, case):
    sd = eq.scene(case, False)
    q, band = eq.make(sd, case, False, seed=12)
    r = _run(emitter_oracle, sd, q)
    em_dir = sd.a_profiles["direction"][0].astype(np.float64)
    cos_size = float(sd.a_profiles["angular_size_cosine"][0])
    size = float(sd.a_profiles["angular_size"][0])
    fails = []
    s = q["op"] == S.EMITTER_SAMPLE_IN
    if not ((r["pdf_dir"][s] == 1.0).all() and (r["flags"][s] == S.EMITTER_FLAG_DELTA).all()):
        fails.append("sample_in: pdf_dir 1 and the delta flag expected on every sample")
    m = q["op"] == S.EMITTER_RADIANCE
    dot = q["direction"][m].astype(np.float64) @ em_dir
    inside = (q["directly_visible"][m] != 0) & (size > 0) & (dot >= cos_size)
    ambiguous = np.abs(dot - cos_size) < 1e-6  # the float32 dot product may land on either side
    got = r["pdf_dir"][m]
    off = (got != np.where(inside, 1.0, 0.0)) & ~ambiguous
    for i in np.flatnonzero(off)[:4]:
        fails.append(f"radiance ({band[m][i]}): pdf_dir {got[i]} for dot - cos {dot[i] - cos_size:.3g}, visible {q['directly_visible'][m][i]}")
    if size > 0:
        qd = eq.distribution_queries(sd, False, seed=13, n=N_HIST)
        rd = _run(emitter_oracle, sd, qd)
        d = rd["direction"].astype(np.float64)
        u, v = eq._basis(em_dir)
        along = d @ em_dir
        radius = np.hypot(d @ u, d @ v) / along / np.tan(0.5 * size)  # the disk sample's radius
        phi = np.arctan2(d @ v, d @ u)
        fails.append("disk radius beyond 1") if radius.max() > 1.0 + 1e-4 else None
        b = np.minimum((radius ** 2 * 16).astype(int), 15) * 8 + np.minimum(((phi + np.pi) / (2 * np.pi) * 8).astype(int), 7)
        fails += _binomial(np.bincount(b, minlength=128), np.full(128, 1.0 / 128), N_HIST, "disk (r^2, phi)")
    assert not [f for f in fails if f], "\n".join(f for f in fails if f)


@pytest.mark.parametrize("case", ["area_textured", "area_c09"])
def test_emitter_selection_frequencies(emitter_oracle, case):
    sd = eq.scene(case, False)
    n = 1 << 20
    q = np.zeros(n, dtype=S.EMITTER_QUERY)
    q["op"] = S.EMITTER_SELECT
    q["rnd"][:, 0] = np.random.default_rng(14).random(n)
    r = _run(emitter_oracle, sd, q)
    w = sd.a_emitters["spectrum_weight"].astype(np.float64) * sd.a_emitters["additional_weight"].astype(np.float64)
    p = w / w.sum()
    assert len(set(np.round(p, 6))) == p.shape[0], "the emitters should have unequal weights"
    fails = _binomial(np.bincount(r["emitter_index"], minlength=p.shape[0]).astype(np.float64), p, n, "selection")
    pdf = r["pdf_sample"].astype(np.float64)
    if not np.allclose(pdf, p[r["emitter_index"]], rtol=1e-6, atol=0):
        fails.append("emitter_discrete_pdf differs from weight / total")
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("case", eq.ENV_CASES)
def test_environment_sampling_follows_the_pixels(emitter_oracle, case):
    """sample_in and sample_emission, histogrammed by the pixel the true inverse of uv_to_direction puts each direction in"""
    sd = eq.scene(case, False)
    p = eq.pixel_model(sd).reshape(-1)
    fails = []
    qd = eq.distribution_queries(sd, False, seed=15, n=N_HIST)
    rd = _run(emitter_oracle, sd, qd)
    fails += _binomial(np.bincount(eq.pixel_of(sd, rd["direction"]), minlength=p.size).astype(np.float64), p, N_HIST, "sample_in")
    re_ = _run(emitter_oracle, sd, eq.emission_queries(16, False, count=1), reps=N_HIST)[0]
    ok = re_["pdf_dir"] > 0
    fails += _binomial(np.bincount(eq.pixel_of(sd, -re_["direction"][ok].astype(np.float64)), minlength=p.size).astype(np.float64), p,
                       int(ok.sum()), "emission")
    if ok.sum() < N_HIST * (1.0 - 1e-3):
        fails.append(f"emission: {N_HIST - ok.sum()} samples with pdf 0")
    assert not fails, "\n".join(fails)


def _quadrature(emitter_oracle, sd, nu, nv):
    rec, _, _ = eq.env_image(sd)
    u, v = np.meshgrid((np.arange(nu) + 0.5) / nu, (np.arange(nv) + 0.5) / nv)
    uv = np.stack([u.reshape(-1), v.reshape(-1)], axis=-1)
    q = np.zeros(uv.shape[0], dtype=S.EMITTER_QUERY)
    q["op"] = S.EMITTER_RADIANCE
    q["direction"] = eq.uv_to_direction(uv, float(rec["offset"][0]), float(rec["scale"][0]))
    r = _run(emitter_oracle, sd, q)
    return float((r["pdf_dir"].astype(np.float64) * 2.0 * np.pi ** 2 * np.sin(np.pi * uv[:, 1])).sum() / (nu * nv))


@pytest.mark.parametrize("case", eq.ENV_CASES)
def test_environment_pdf_normalisation(emitter_oracle, case):
    sd = eq.scene(case, False)
    integral = _quadrature(emitter_oracle, sd, 1024, 512)
    bound = NORMALISATION_BOUND.get(case, NORMALISATION_BOUND_DEFAULT)
    print(f"\n[emitter] {case}: integral of pdf_dir over the sphere {integral:.6f} (error {abs(integral - 1.0):.3e}, bound {bound:g})")
    assert abs(integral - 1.0) <= bound


@pytest.mark.parametrize("case", ["env_plain", "env_rotated", "env_mirrored", "env_mirrored_rotated"])
def test_environment_round_trip(emitter_oracle, case):
    """emitter_get_radiance at a sampled direction looks the image up where the sample was taken, except with scale < 0 and offset != 0,
    where the reference's direction_to_uv lands at u + 2 offset (DESIGN §10): compared with the same image without offset and scale,
    looked up at the expected uv."""
    sd, twin = eq.scene(case, False), eq.scene(case, False, plain=True)
    rec, _, _ = eq.env_image(sd)
    offset, scale = float(rec["offset"][0]), float(rec["scale"][0])
    quirk = scale < 0 and offset != 0
    qd = eq.distribution_queries(sd, False, seed=17, n=4096)
    s = _run(emitter_oracle, sd, qd)
    uv = eq.true_uv(s["direction"], offset, scale)
    expected = uv + np.array([2.0 * offset if quirk else 0.0, 0.0])
    assert np.allclose(np.mod(eq.direction_to_uv(s["direction"], offset, scale)[:, 0] - expected[:, 0] + 0.5, 1.0), 0.5, atol=1e-5)
    # away from the poles (sin_t amplifies rounding) and the seam
    keep = (uv[:, 1] > 0.02) & (uv[:, 1] < 0.98) & (np.abs(np.mod(expected[:, 0] + 0.5, 1.0) - 0.5) > 1e-4)
    q = np.zeros(int(keep.sum()), dtype=S.EMITTER_QUERY)
    q["op"] = S.EMITTER_RADIANCE
    q["direction"] = s["direction"][keep]
    at_case = _run(emitter_oracle, sd, q)["pdf_dir"].astype(np.float64)
    q["direction"] = eq.uv_to_direction(np.mod(expected[keep], 1.0))
    at_twin = _run(emitter_oracle, twin, q)["pdf_dir"].astype(np.float64)
    err = np.abs(at_case - at_twin) / at_twin
    assert err.max() < 1e-3, f"lookup differs from the image at the expected uv by {err.max():.3g}"
    sample_pdf = s["pdf_dir"][keep].astype(np.float64)
    moved = np.abs(at_case - sample_pdf) > 1e-3 * sample_pdf
    if quirk:
        assert moved.mean() > 0.5, "the mirrored-and-rotated lookup was expected at u + 2 offset"
    else:
        assert not moved.any(), f"{int(moved.sum())} lookups disagree with their sample's pdf"
