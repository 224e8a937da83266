"""Seeded BSDF-sampling queries for the sampling tests (etxb_debug_bsdf_sample against the oracle's bsdf::sample).

make(material, ...) returns (queries, band): S.SAMPLE_QUERY records and, per query, the name of the set it belongs to.  Every arrival is
emitted twice, once per path source (camera, light).  `w_i` points AT the surface; the light arrives from -w_i.  Frames, uv and
wavelengths follow closure_queries.py.

Sets (mode 0, "bounce", unless named otherwise):
  uniform      arrivals uniform on the sphere: from outside and from inside
  normal       axis-aligned frames with exact zero components, arrival along +n and -n
  grazing      |cos| of the arrival in [2e-3, 5e-2], on either side
  critical     dielectrics: arrival from inside within 1e-3 rad of the critical angle, on both sides of it
  given        mode 1 on uniform arrivals: the fixed values of FIXED_EDGES, then uniform triples in [0, 1)

arrivals(...) returns the distribution test's arrival directions: normal, 30, 60, 80 and 88 degrees from outside, 45 degrees and
80 degrees from inside, and 5e-4 rad inside the critical angle (dielectrics) or 88 degrees from inside (the others).
"""
import numpy as np

import closure_queries as cq
from etx_tracer_b200 import structs as S

K_EPSILON = np.float32(1.192092896e-07)
_ONE_MINUS = np.nextafter(np.float32(1.0), np.float32(0.0))
# u^2 + v^2 + w^2 just below and just above the kEpsilon test of Smp::has_fixed (below: the walks draw from the stream instead)
_BELOW = np.float32(np.sqrt(K_EPSILON) * 0.999)
_ABOVE = np.float32(np.sqrt(K_EPSILON) * 1.001)
FIXED_EDGES = np.array([
    (0.0, 0.0, 0.0), (_ONE_MINUS, _ONE_MINUS, _ONE_MINUS), (0.0, _ONE_MINUS, 0.5), (_ONE_MINUS, 0.0, 0.5), (0.5, 0.5, 0.0),
    (0.5, 0.5, _ONE_MINUS), (0.0, 0.0, _ONE_MINUS), (_BELOW, 0.0, 0.0), (_ABOVE, 0.0, 0.0), (0.0, 0.0, _BELOW), (0.0, 0.0, _ABOVE),
    (0.0, _BELOW, 0.0), (0.0, _ABOVE, 0.0),
], dtype=np.float32)


# the cases (scenes.MATERIAL_KINDS names; sky_room-<material>) whose sample pdf is the pdf bsdf::evaluate returns for the sampled
# direction, in RGB and spectral scenes (test_oracle_bsdf_sample.py derives this set from the reference)
SAMPLE_PDF_IS_EVALUATE_PDF = {
    "conductor_rough", "conductor_thinfilm", "diffuse_rough", "plastic", "plastic_aniso", "plastic_rough_base", "plastic_vmf_base",
    "sss_refracted", "translucent", "velvet", "sky_room-metal", "sky_room-plastic",
}


def _fill(q, material, rng, spectral, medium):
    q["uv"] = rng.random((q.shape[0], 2))
    q["material"] = material
    q["seed"] = rng.integers(0, 2 ** 32, q.shape[0], dtype=np.uint64).astype(np.uint32)
    q["medium"] = medium
    wl = cq.spectral_sample(rng.random(q.shape[0]))
    wl[:4] = (390.0, 830.0, 390.0, 830.0)
    q["wavelength"] = wl if spectral else -1.0


def make(material, seed, spectral=False, eta=1.5, dielectric=False, count=32, medium=7):
    """Per-sample query set for one material index; `eta` (n_int / n_ext) steers the critical-angle set only.  `medium` is the current
    medium every query carries (Boundary and Void return it, reflections keep it)."""
    rng = np.random.default_rng(seed)
    sets = []  # (name, frames, w_i, mode, fixed)

    def add(name, frames, w_i, mode=S.SAMPLE_BOUNCE, fixed=None):
        n = w_i.shape[0]
        sets.append((name, frames, cq._unit(w_i), mode, np.zeros((n, 3), np.float32) if fixed is None else fixed))

    phi = lambda k: rng.uniform(0.0, 2.0 * np.pi, k)
    add("uniform", cq._random_frames(rng, 2 * count), cq._sphere(rng, 2 * count))

    axes = np.eye(3)
    frames, w_i = [], []
    for k in range(3):
        for s in (1.0, -1.0):
            nrm, tan = s * axes[k], axes[(k + 1) % 3]
            for w in (-nrm, nrm):
                frames.append((nrm, tan, np.cross(nrm, tan)))
                w_i.append(w)
    add("normal", tuple(np.array([f[j] for f in frames]) for j in range(3)), np.array(w_i))

    c = np.exp(rng.uniform(np.log(2e-3), np.log(5e-2), count)) * rng.choice([-1.0, 1.0], count)
    fr = cq._random_frames(rng, count)
    add("grazing", fr, -cq._to_world(fr, cq._local_dir(c, phi(count))))

    if dielectric:
        theta = np.arcsin(1.0 / eta) + rng.uniform(-1e-3, 1e-3, count)
        fr = cq._random_frames(rng, count)
        add("critical", fr, -cq._to_world(fr, cq._local_dir(-np.cos(theta), phi(count))))

    n = FIXED_EDGES.shape[0] + count
    fixed = np.concatenate([FIXED_EDGES, rng.random((count, 3)).astype(np.float32)])
    add("given", cq._random_frames(rng, n), cq._sphere(rng, n), S.SAMPLE_GIVEN, fixed)

    total = sum(s[2].shape[0] for s in sets)
    q = np.zeros(2 * total, dtype=S.SAMPLE_QUERY)
    band = np.empty(2 * total, dtype=object)
    k = 0
    for name, (nrm, tan, btn), w, mode, fx in sets:
        m = w.shape[0]
        for source in (S.PATH_CAMERA, S.PATH_LIGHT):
            sl = slice(k, k + m)
            q["nrm"][sl], q["tan"][sl], q["btn"][sl] = nrm, tan, btn
            q["w_i"][sl] = w
            q["path_source"][sl] = source
            q["mode"][sl] = mode
            q["fixed"][sl] = fx
            band[sl] = name
            k += m
    _fill(q, material, rng, spectral, medium)
    return q, band


ARRIVALS = ("0", "30", "60", "80", "88", "in45", "in80", "in-edge")


def arrivals(material, seed, spectral=False, eta=1.5, dielectric=False, medium=7):
    """The distribution test's queries: one per entry of ARRIVALS on a random frame, mode 0, alternating camera and light sources."""
    rng = np.random.default_rng(seed)
    deg = np.radians([0.0, 30.0, 60.0, 80.0, 88.0, 45.0, 80.0])
    cos_t = np.concatenate([np.cos(deg[:5]), -np.cos(deg[5:])])
    edge = np.arcsin(1.0 / eta) - 5e-4 if dielectric else np.radians(88.0)
    cos_t = np.append(cos_t, -np.cos(edge))
    n = cos_t.shape[0]
    fr = cq._random_frames(rng, n)
    q = np.zeros(n, dtype=S.SAMPLE_QUERY)
    q["nrm"], q["tan"], q["btn"] = fr
    q["w_i"] = -cq._to_world(fr, cq._local_dir(cos_t, rng.uniform(0.0, 2.0 * np.pi, n)))
    q["path_source"] = np.where(np.arange(n) % 2 == 0, S.PATH_CAMERA, S.PATH_LIGHT)
    q["mode"] = S.SAMPLE_BOUNCE
    _fill(q, material, rng, spectral, medium)
    return q


def local(q, w):
    """float64 coordinates of world directions w (n, ..., 3) in each query's frame {tan, btn, nrm} as interpolated (not flipped)."""
    w = np.asarray(w, np.float64)
    shape = (q.shape[0],) + (1,) * (w.ndim - 2) + (3,)
    return np.stack([(w * q[f].astype(np.float64).reshape(shape)).sum(-1) for f in ("tan", "btn", "nrm")], axis=-1)


def arrival_cos(q):
    """float64 cosine of the arrival direction -w_i against the interpolated normal."""
    return -(q["w_i"].astype(np.float64) * q["nrm"].astype(np.float64)).sum(1)
