"""The oracle's sampling export (oracle_bsdf_sample: the reference's bsdf::sample compiled in place) against plain float64 models, on the
query sets of sample_queries.py.  This pins the side the GPU sampling tests compare against and rehearses the query conventions: w_i
pointing AT the surface, the frame flipped towards the arrival, the fixed values of mode 0 and mode 1, the current medium, both path
sources.  It also pins which cases' sample pdf is the pdf bsdf::evaluate gives for the sampled direction (the GPU test's part (c)).
Runs without a GPU."""
import numpy as np
import pytest

import sample_queries as sq
from etx_tracer_b200 import scenes, structs as S

REPS = 16
K_EPSILON = 1.192092896e-07


def _flip(q):
    """+1 where the frame faces the arrival (BSDFData::get_normal_frame), -1 where it is flipped"""
    return np.where(sq.arrival_cos(q) > 0.0, 1.0, -1.0)


def _world(q, local):
    s = _flip(q)[:, None, None]
    return s * (local[..., :1] * q["tan"].astype(np.float64)[:, None] + local[..., 1:2] * q["btn"].astype(np.float64)[:, None]
                + local[..., 2:3] * q["nrm"].astype(np.float64)[:, None])


def _angle(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    c = (a * b).sum(-1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))
    return np.arccos(np.clip(c, -1.0, 1.0))


def _reflect(q):
    w = q["w_i"].astype(np.float64)
    n = q["nrm"].astype(np.float64)
    return w - 2.0 * (w * n).sum(1, keepdims=True) * n


def _stream(oracle_mod, q, draws):
    """the first `draws` values of Sampler(seed, r) for every query and repetition: float32 (n, REPS, draws)"""
    a = np.repeat(q["seed"], REPS)
    b = np.tile(np.arange(REPS, dtype=np.uint32), q.shape[0])
    return oracle_mod.sampler_kat(a, b, draws)[1].reshape(q.shape[0], REPS, draws)


def _fixed(oracle_mod, q):
    """(u, v, w) the sample sees as fixed values, and whether Smp::has_fixed holds: mode 0 pushes draws 0, 1 and 4 of the stream"""
    st = _stream(oracle_mod, q, 6)
    f = np.where((q["mode"] == S.SAMPLE_BOUNCE)[:, None, None], st[..., [0, 1, 4]], q["fixed"][:, None, :])
    f32 = f.astype(np.float32)
    has = (f32[..., 0] * f32[..., 0] + f32[..., 1] * f32[..., 1] + f32[..., 2] * f32[..., 2]) > np.float32(K_EPSILON)
    return f.astype(np.float64), has


def _fresnel(cos_i, eta):
    """unpolarised Fresnel reflectance of a smooth dielectric, light arriving at |cos_i| on the side where eta = n_t / n_i"""
    cos_i = np.abs(cos_i)
    sin2_t = (1.0 - cos_i ** 2) / eta ** 2
    cos_t = np.sqrt(np.maximum(0.0, 1.0 - sin2_t))
    rs = (cos_i - eta * cos_t) / (cos_i + eta * cos_t)
    rp = (eta * cos_i - cos_t) / (eta * cos_i + cos_t)
    return np.where(sin2_t >= 1.0, 1.0, 0.5 * (rs * rs + rp * rp))


@pytest.fixture(scope="module")
def sample_oracle(oracle_mod):
    if not oracle_mod.has_bsdf_sample():
        pytest.skip("oracle/_ref predates oracle_bsdf_sample (rebuild it with oracle/build_oracle.sh where the reference sources exist)")
    return oracle_mod


def _run(oracle_mod, sd, material, spectral, seed, **kw):
    q, band = sq.make(material, seed=seed, spectral=spectral, **kw)
    o = oracle_mod.Oracle(sd)
    r = o.bsdf_sample(q, REPS)
    o.close()
    return q, band, r


@pytest.mark.parametrize("spectral", [False, True], ids=["rgb", "spectral"])
def test_lambert_sample_is_the_cosine_lobe(sample_oracle, spectral):
    sd = scenes.material_box("plastic", spectral=spectral)
    q, band, r = _run(sample_oracle, sd, 0, spectral, 11, count=24)  # material 0: the white Lambert wall
    f, has = _fixed(sample_oracle, q)
    assert has.any() and (~has).any()
    cos_t = np.sqrt(np.maximum(f[..., 0], K_EPSILON))
    sin_t = np.sqrt(1.0 - cos_t ** 2)
    local = np.stack([np.cos(2.0 * np.pi * f[..., 1]) * sin_t, np.sin(2.0 * np.pi * f[..., 1]) * sin_t, cos_t], axis=-1)
    want = _world(q, local)
    angle = _angle(r["w_o"], want)
    assert (angle[has] < 2e-4).all(), f"direction off by up to {angle[has].max():.3g} rad"
    assert (r["properties"] == (S.BSDF_REFLECTION | S.BSDF_DIFFUSE)).all()
    ok = (r["pdf"] > 0) & has
    np.testing.assert_allclose(r["pdf"][ok], cos_t[ok] / np.pi, rtol=2e-5)
    # weight = bsdf / pdf = the reflectance: one value per query, whatever the direction
    w = r["weight"].astype(np.float64)
    assert np.allclose(w[ok], 1.0, rtol=0.0, atol=2e-2), (w[ok].min(), w[ok].max())
    if not spectral:
        assert np.ptp(w[ok], axis=0).max() < 1e-6
    # without the fixed values the lobe is sampled from the stream: only the two-sided-ness of the wall is visible
    assert (np.abs(sq.local(q, r["w_o"])[..., 2] * _flip(q)[:, None])[~has] >= 0).all()


@pytest.mark.parametrize("kind", ["mirror", "conductor_smooth"])
@pytest.mark.parametrize("spectral", [False, True], ids=["rgb", "spectral"])
def test_mirror_and_smooth_conductor_reflect_exactly(sample_oracle, kind, spectral):
    sd = scenes.material_box(kind, spectral=spectral)
    q, band, r = _run(sample_oracle, sd, 4, spectral, 13)
    valid = r["pdf"] > 0
    assert valid[band != "grazing"].all()
    angle = _angle(r["w_o"], np.broadcast_to(_reflect(q)[:, None, :], r["w_o"].shape))
    assert (angle[valid] < 2e-6).all(), f"reflection off by up to {angle[valid].max():.3g} rad"
    assert ((r["properties"] & (S.BSDF_REFLECTION | S.BSDF_DELTA)) == (S.BSDF_REFLECTION | S.BSDF_DELTA)).all()
    assert (r["eta"] == 1.0).all()


@pytest.mark.parametrize("kind", ["dielectric_smooth", "thinfilm"])
def test_smooth_dielectric_and_thinfilm_choose_by_fresnel(sample_oracle, kind):
    """spectral scenes: one wavelength per query, so the Fresnel term is one real number"""
    sd = scenes.material_box(kind, spectral=True)
    q, band, r = _run(sample_oracle, sd, 4, True, 17, dielectric=True, eta=2.42 if kind == "dielectric_smooth" else 1.5)
    refl = (r["properties"] & S.BSDF_REFLECTION) != 0
    trans = (r["properties"] & S.BSDF_TRANSMISSION) != 0
    assert (refl ^ trans).all() and ((r["properties"] & S.BSDF_DELTA) != 0).all()
    # directions: exact mirror reflection; transmission by Snell (dielectric) or straight through (thin film)
    angle_r = _angle(r["w_o"], np.broadcast_to(_reflect(q)[:, None, :], r["w_o"].shape))
    assert (angle_r[refl] < 2e-6).all(), angle_r[refl].max()
    cos_i = sq.arrival_cos(q)
    # media: a reflection keeps the current medium, a transmission enters the material's (none here)
    assert (r["medium_index"][refl] == q["medium"][:, None].repeat(REPS, 1)[refl]).all()
    assert (r["medium_index"][trans] == S.INVALID).all()
    st = _stream(sample_oracle, q, 8)
    if kind == "thinfilm":
        # ThinfilmBSDF::sample draws its choice from the stream, after the bounce's six draws in mode 0
        u = np.where((q["mode"] == S.SAMPLE_BOUNCE)[:, None], st[..., 6], st[..., 0]).astype(np.float64)
        f = np.where(refl, r["pdf"], 1.0 - r["pdf"]).astype(np.float64)
        assert np.allclose(f, f[:, :1], atol=1e-6), "the thin-film reflectance varies within a query"
        assert ((u <= f) == refl).all(), "reflection is not the choice u <= F"
        assert (r["w_o"][trans] == np.broadcast_to(q["w_i"][:, None, :], r["w_o"].shape)[trans]).all(), "a transmission leaves w_i"
        assert (r["eta"] == 1.0).all()
    else:
        # DielectricBSDF::sample at zero roughness: the walk scatters once at the geometric normal; the choice is fixed_w < F (the
        # stream's fourth draw where has_fixed fails: height, slope u, slope v, choice)
        fx, has = _fixed(sample_oracle, q)
        u = np.where(has, fx[..., 2], st[..., 3])
        eta_rel = r["eta"][trans]
        assert eta_rel.size and np.isfinite(eta_rel).all()
        eta_q = np.full(q.shape[0], np.nan)
        for i in range(q.shape[0]):
            e = r["eta"][i][trans[i]]
            if e.size:
                assert (e == e[0]).all()
                eta_q[i] = e[0]
        # a query with reflections only (total internal reflection) reflects from inside beyond the critical angle of its wavelength
        known = np.isfinite(eta_q)
        f = np.where(known, _fresnel(cos_i, np.where(known, eta_q, 1.0)), 1.0)[:, None]
        margin = np.abs(u - f) > 1e-5
        assert ((u < f) == refl)[margin & known[:, None]].all(), "reflection is not the choice u < F"
        assert refl[~known].all()
        # Snell: sin_t = sin_i / eta_rel on the other side, in the plane of incidence
        n = q["nrm"].astype(np.float64) * np.sign(cos_i)[:, None]
        w = -q["w_i"].astype(np.float64)
        ci = np.abs(cos_i)[:, None]
        e = np.where(known, eta_q, 1.0)[:, None]
        ct = np.sqrt(np.maximum(0.0, 1.0 - (1.0 - ci ** 2) / e ** 2))
        t = -w / e + (ci / e - ct) * n
        angle_t = _angle(r["w_o"], np.broadcast_to(t[:, None, :], r["w_o"].shape))
        assert (angle_t[trans] < 2e-5).all(), angle_t[trans].max()
        # weight: the reflectance (1) for a reflection, 1 / eta_rel^2 for a transmission, for camera and light paths alike
        w = r["weight"][..., 0].astype(np.float64)
        assert np.allclose(w[refl], 1.0, rtol=1e-4)
        assert np.allclose(w[trans], (1.0 / np.broadcast_to(e, w.shape) ** 2)[trans], rtol=1e-4)
        assert (r["eta"][refl] == 1.0).all()


def _eval_at_samples(oracle_mod, sd, q, r):
    ok = (r["pdf"] > 0) & ((r["properties"] & S.BSDF_DELTA) == 0) & np.isfinite(r["pdf"])
    qi, ki = np.nonzero(ok)
    cl = np.zeros(qi.size, dtype=S.CLOSURE_QUERY)
    for f in ("nrm", "tan", "btn", "w_i", "uv", "wavelength", "material", "path_source", "seed"):
        cl[f] = q[f][qi]
    cl["w_o"] = r["w_o"][qi, ki]
    o = oracle_mod.Oracle(sd)
    e = o.bsdf_eval(cl, 1)
    o.close()
    return r["pdf"][qi, ki].astype(np.float64), e[:, 6]


def _sample_pdf_is_evaluate_pdf(oracle_mod, where, kind, spectral):
    if where == "sky_room":
        sd, material = scenes.sky_room(spectral=spectral), {"floor": 0, "plastic": 1, "metal": 2}[kind]
    else:
        sd, material = scenes.material_box(kind, spectral=spectral), 4
    q, band, r = _run(oracle_mod, sd, material, spectral, 19, count=16)
    ps, pe = _eval_at_samples(oracle_mod, sd, q, r)
    if ps.size == 0:
        return None
    return bool((np.abs(ps - pe) <= 1e-4 * ps).all())


def test_which_sample_pdfs_are_evaluate_pdfs(sample_oracle):
    found = set()
    cases = [("material_box", k) for k in sorted(scenes.MATERIAL_KINDS)] + [("sky_room", k) for k in ("floor", "plastic", "metal")]
    for where, kind in cases:
        same = [_sample_pdf_is_evaluate_pdf(sample_oracle, where, kind, sp) for sp in (False, True)]
        if all(s is True for s in same):
            found.add(kind if where == "material_box" else f"{where}-{kind}")
    print(f"\n[oracle sample] sample pdf == evaluate pdf: {sorted(found)}")
    assert found == sq.SAMPLE_PDF_IS_EVALUATE_PDF
