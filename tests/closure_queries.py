"""Seeded direction pairs for the vertex-closure tests (etxb_debug_closure_eval against the oracle's bsdf::evaluate / reverse_pdf).

make(material, ...) returns (queries, band): S.CLOSURE_QUERY records and, per query, the name of the set it belongs to.  Every pair is
emitted twice, once per path source (camera, light).  `w_i` points AT the surface (BSDFData::w_i); `w_o` points away from it.  In the
local frame {tan, btn, nrm} the direction the light arrives from is -w_i.

Sets:
  uniform      w_i, w_o uniform on the sphere: both sides, entering and leaving, reflection and transmission
  lobe         w_o within a few alpha of the mirror reflection and of the refraction of -w_i (low roughness lobes)
  grazing      |cos| in [2e-3, 5e-2] for w_i, w_o or both
  exact        axis-aligned frames with exact zero components: normal incidence with w_o = n and w_o = -w_i, w_o in the tangent plane
  tangent      w_o in the tangent plane of a random frame (|cos| at float rounding: the kEpsilon band)
  critical     dielectrics: light arriving from inside, within 1e-3 rad of the critical angle on both sides of it
  straight     dielectrics: transmission pairs near the degenerate half vector (w_o ~ w_i, the straight-through direction)
Frames are random orthonormal (not axis-aligned) except in `exact`.  uv is uniform in [0, 1)^2.  Wavelengths follow the spectral sampling
(SpectralQuery::spectral_sample, debug_math fn 7) and include 390 and 830 nm exactly.
"""
import numpy as np

from etx_tracer_b200 import structs as S

_SPECTRAL_OFFSET = float.fromhex("0x1.35ce7a0000000p-5")


def spectral_sample(rnd):
    """SpectralQuery::spectral_sample (spectrum.hxx:234-239) in float64."""
    scale = 1.0 - _SPECTRAL_OFFSET
    return 538.0 - 138.888889 * np.arctanh(0.85691062 - 1.82750197 * (np.asarray(rnd, np.float64) * scale + _SPECTRAL_OFFSET))


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _sphere(rng, n):
    return _unit(rng.normal(size=(n, 3)))


def _random_frames(rng, n):
    nrm = _sphere(rng, n)
    tan = _unit(np.cross(nrm, _sphere(rng, n)))
    btn = np.cross(nrm, tan)
    return nrm, tan, btn


def _to_world(frames, local):
    nrm, tan, btn = frames
    return local[:, :1] * tan + local[:, 1:2] * btn + local[:, 2:3] * nrm


def _local_dir(cos_theta, phi):
    s = np.sqrt(np.maximum(0.0, 1.0 - cos_theta ** 2))
    return np.stack([s * np.cos(phi), s * np.sin(phi), cos_theta], axis=-1)


def _perturb(rng, d, spread):
    """d tilted by an angle ~ |N(0, spread)| about a random axis, renormalised."""
    axis = _unit(np.cross(d, _sphere(rng, d.shape[0])))
    ang = np.abs(rng.normal(size=(d.shape[0], 1))) * spread
    return _unit(d * np.cos(ang) + axis * np.sin(ang))


def _refract(wl, eta):
    """local arrival direction wl (z != 0, pointing away from the surface) -> refracted direction on the other side (None where TIR).
    eta = n_int / n_ext; for wl.z < 0 the light arrives from inside."""
    out = np.zeros_like(wl)
    ok = np.zeros(wl.shape[0], bool)
    for i, w in enumerate(wl):
        e = eta if w[2] > 0 else 1.0 / eta
        cos_i = abs(w[2])
        sin2_t = (1.0 - cos_i ** 2) / e ** 2
        if sin2_t >= 1.0:
            continue
        cos_t = np.sqrt(1.0 - sin2_t)
        t = -w / e
        t[2] = -np.sign(w[2]) * cos_t
        out[i] = _unit(t)
        ok[i] = True
    return out, ok


def make(material, seed, spectral=False, alpha=0.3, eta=1.5, dielectric=False, count=48):
    """Query set for one material index.  `alpha` (roughness) and `eta` (n_int / n_ext) steer the lobe / critical-angle sets only."""
    rng = np.random.default_rng(seed)
    alpha = max(float(alpha), 0.02)
    sets = []  # (name, frames, w_i, w_o)

    def add(name, frames, w_i, w_o):
        sets.append((name, frames, _unit(w_i), _unit(w_o)))

    n = 2 * count
    add("uniform", _random_frames(rng, n), _sphere(rng, n), _sphere(rng, n))

    # lobe: -w_i on either side, w_o near its mirror reflection / its refraction
    fr = _random_frames(rng, count)
    arr = _local_dir(rng.uniform(-1.0, 1.0, count), rng.uniform(0.0, 2.0 * np.pi, count))
    arr[:, 2] = np.where(np.abs(arr[:, 2]) < 0.05, 0.05 * np.sign(arr[:, 2] + 1e-9), arr[:, 2])
    arr = _unit(arr)
    mirror = arr * np.array([-1.0, -1.0, 1.0])
    spread = alpha * np.array([0.25, 1.0, 3.0])[rng.integers(0, 3, count)][:, None]
    add("lobe", fr, -_to_world(fr, arr), _to_world(fr, _perturb(rng, mirror, spread)))
    refr, ok = _refract(arr, eta)
    fr2 = tuple(f[ok] for f in fr)
    add("lobe", fr2, -_to_world(fr2, arr[ok]), _to_world(fr2, _perturb(rng, refr[ok], spread[ok])))

    # grazing: one direction or both with |cos| in [2e-3, 5e-2], on either side
    g = count
    c_gr = lambda k: np.exp(rng.uniform(np.log(2e-3), np.log(5e-2), k)) * rng.choice([-1.0, 1.0], k)
    c_any = lambda k: rng.uniform(-1.0, 1.0, k)
    phi = lambda k: rng.uniform(0.0, 2.0 * np.pi, k)
    which = rng.integers(0, 3, g)
    ci = np.where(which != 1, c_gr(g), c_any(g))
    co = np.where(which != 0, c_gr(g), c_any(g))
    fr = _random_frames(rng, g)
    add("grazing", fr, -_to_world(fr, _local_dir(ci, phi(g))), _to_world(fr, _local_dir(co, phi(g))))

    # exact geometry on axis-aligned frames (every component 0 or +-1); both orientations of the normal
    axes = np.eye(3)
    ex_frames, ex_wi, ex_wo = [], [], []
    for k in range(3):
        for s in (1.0, -1.0):
            nrm = s * axes[k]
            tan = axes[(k + 1) % 3]
            btn = np.cross(nrm, tan)
            for wi, wo in ((-nrm, nrm), (nrm, -nrm), (-nrm, -nrm), (nrm, nrm),  # normal incidence: w_o = n (reflection / transmission) and w_o = -w_i
                           (-nrm, tan), (nrm, btn), (_unit(-nrm + tan), tan), (_unit(nrm - btn), -tan),  # w_o exactly in the tangent plane
                           (_unit(-nrm + tan), _unit(nrm + tan)), (_unit(-nrm - btn), _unit(nrm + btn))):  # exact mirror pairs
                ex_frames.append((nrm, tan, btn))
                ex_wi.append(wi)
                ex_wo.append(wo)
    ex = tuple(np.array([f[j] for f in ex_frames]) for j in range(3))
    add("exact", ex, np.array(ex_wi), np.array(ex_wo))

    # w_o in the tangent plane of a random frame
    t = count // 2
    fr = _random_frames(rng, t)
    wo_l = _local_dir(np.zeros(t), phi(t))
    add("tangent", fr, -_to_world(fr, _local_dir(c_any(t), phi(t))), _to_world(fr, wo_l))

    if dielectric:
        # light from inside (local -w_i below the surface) within 1e-3 rad of the critical angle, w_o anywhere / near the refraction
        c = count
        theta_c = np.arcsin(1.0 / eta)
        theta = theta_c + rng.uniform(-1e-3, 1e-3, c)
        arr = _local_dir(-np.cos(theta), phi(c))
        fr = _random_frames(rng, c)
        wo = np.where(rng.random((c, 1)) < 0.5, _sphere(rng, c), _perturb(rng, arr * np.array([-1.0, -1.0, 1.0]), alpha))
        add("critical", fr, -_to_world(fr, arr), _to_world(fr, wo))
        # straight through: w_o ~ -(-w_i) continued, i.e. w_o ~ w_i, where w_i + eta w_o nearly cancels for eta near 1
        fr = _random_frames(rng, c)
        arr = _local_dir(rng.uniform(-1.0, 1.0, c), phi(c))
        add("straight", fr, -_to_world(fr, arr), _to_world(fr, _perturb(rng, -arr, 1e-3)))

    total = sum(s[2].shape[0] for s in sets)
    q = np.zeros(2 * total, dtype=S.CLOSURE_QUERY)
    band = np.empty(2 * total, dtype=object)
    k = 0
    for name, (nrm, tan, btn), w_i, w_o in sets:
        m = w_i.shape[0]
        for source in (S.PATH_CAMERA, S.PATH_LIGHT):
            sl = slice(k, k + m)
            q["nrm"][sl], q["tan"][sl], q["btn"][sl] = nrm, tan, btn
            q["w_i"][sl], q["w_o"][sl] = w_i, w_o
            q["path_source"][sl] = source
            band[sl] = name
            k += m
    q["uv"] = rng.random((q.shape[0], 2))
    q["material"] = material
    q["seed"] = rng.integers(0, 2 ** 32, q.shape[0], dtype=np.uint64).astype(np.uint32)
    wl = spectral_sample(rng.random(q.shape[0]))
    wl[:4] = (390.0, 830.0, 390.0, 830.0)
    q["wavelength"] = wl if spectral else -1.0
    return q, band


def local(q):
    """float64 local-frame cosines of the arrival direction -w_i and of w_o (frame as interpolated, not flipped)."""
    nrm = q["nrm"].astype(np.float64)
    return -(q["w_i"].astype(np.float64) * nrm).sum(1), (q["w_o"].astype(np.float64) * nrm).sum(1)
