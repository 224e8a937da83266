"""The scene and seeded queries for the media tests (etxb_debug_medium against the oracle's media routines).

scene(spectral) builds one scene with every medium of MEDIA, as the loader would (scenes.SceneData.add_medium):
  fog         homogeneous grey fog, g = 0.3
  absorber    chromatic pure absorber; its blue channel has zero extinction (in RGB)
  scatterer   pure scatterer (albedo 1), chromatic
  dense       extinction 1e4: the free-flight loop `while (t < kRayEpsilon)` repeats about ten times on average
  vacuum      absorption and scattering both 0
  invalid     absorption and scattering spectrum indices both invalid (0xffffffff)
  cloud       heterogeneous: the 16^3 fbm grid in non-cubic bounds 1 x 0.8 x 1.2
  grid1       heterogeneous 1 x 1 x 1 grid
  grid235     heterogeneous 2 x 3 x 5 grid in bounds 1 x 0.25 x 4
  ones        heterogeneous all-ones grid at max_sigma 40: ratio tracking's Russian roulette fires
  zero_sigma  heterogeneous with max_sigma = 0
Every heterogeneous max_sigma times the local diagonal (at most sqrt(3)) keeps a tracking loop under about a hundred steps.

Its geometry, for the segment op (trace_transmittance on the BVH): a Boundary box of fog (half size 1) around a Boundary box of cloud
(half size 0.5, fog outside), a stack of STACK thin Boundary quads facing -x at x = 3 + 0.02 k (scatterer inside, fog outside), a Void
quad at x = 2.5, an opaque quad at x = 5 and a small emitter far above.

make(sd, case, spectral, seed) returns (queries, band) for one case of CASES: a medium's name (its bounds, density, transmittance and
sample queries), "phase" or "segment".  Bands, one per query:
  inside, crossing, miss, axis (one or two zero direction components with the origin on a slab plane, where medium_bounds divides 0 by
  0), surface (origin on a face, edge or corner; or a direction tangent to a face), ends_inside, max_float (max_t = kMaxFloat),
  short (max_t just above kRayEpsilon), long (max_t = 1e4), throughput (zero channels of the sample op's throughput), uniform
  density: centre, face, zero (0 and -0), top (1 - 2^-24 and exactly 1), below (-2^-24 and the denormal -2^-149), uniform
  phase: g_small (|g| on either side of the 1e-3 switch), g_edge (g = +-0.999), rnd_edge (rnd 0 or 1 - 2^-24), pole (w_i = +-z), uniform
  segment: crossings_0 / 1 / 2 / 4, crossings_61 / 62 / 63, opaque, void, degenerate, nested (with and without a starting medium)
"""
import numpy as np

from etx_tracer_b200 import scenes, structs as S

f32 = np.float32
K_RAY_EPSILON = f32(15.0) / f32(65504.0 - 1.0)
K_MAX_FLOAT = f32(3.402823466e38)
ONE_MINUS = np.nextafter(f32(1.0), f32(0.0))
HOMOGENEOUS = ("fog", "absorber", "scatterer", "dense", "vacuum", "invalid")
HETEROGENEOUS = ("cloud", "grid1", "grid235", "ones", "zero_sigma")
MEDIA = HOMOGENEOUS + HETEROGENEOUS
CASES = MEDIA + ("phase", "segment")
STACK = 64
STACK_X0, STACK_DX = 3.0, 0.02
PHASE_G = (0.0, 5e-4, -5e-4, 9.99e-4, -9.99e-4, 1e-3, -1e-3, 0.3, -0.7, 0.9, 0.999, -0.999)
# the heterogeneous media: (grid, bounds, scattering, absorption, max_sigma)
_HET = {
    "cloud": (lambda: scenes.fbm_density(16), ([-0.5, -0.4, -0.5], [0.5, 0.4, 0.7]), (6.0, 5.0, 4.0), (0.5, 0.5, 0.5), 8.0),
    "grid1": (lambda: np.ones((1, 1, 1), f32), ([2.0, 2.0, 2.0], [3.0, 3.0, 3.0]), (2.0, 2.0, 2.0), (0.5, 0.5, 0.5), 3.0),
    "grid235": (lambda: np.random.default_rng(235).uniform(0.1, 1.0, (5, 3, 2)).astype(f32), ([-4.0, 0.0, 0.0], [-3.0, 0.25, 4.0]), (3.0, 2.0, 1.0),
                (0.2, 0.2, 0.2), 5.0),
    "ones": (lambda: np.ones((4, 4, 4), f32), ([2.0, -1.0, 2.0], [3.0, 0.0, 3.0]), (38.0, 38.0, 38.0), (2.0, 2.0, 2.0), 40.0),
    "zero_sigma": (lambda: scenes.fbm_density(8, seed=3), ([-3.0, -3.0, -3.0], [-2.0, -2.0, -2.0]), (2.0, 2.0, 2.0), (0.1, 0.1, 0.1), 0.0),
}


def scene(spectral):
    sd = scenes.SceneData()
    sd.name = f"media/{'spectral' if spectral else 'rgb'}"
    sd.add_medium(absorption=(0.1, 0.1, 0.1), scattering=(0.9, 0.9, 0.9), g=0.3)
    sd.add_medium(absorption=(0.5, 2.0, 0.0), scattering=(0.0, 0.0, 0.0))
    sd.add_medium(absorption=(0.0, 0.0, 0.0), scattering=(1.5, 1.0, 0.5), g=-0.4)
    sd.add_medium(absorption=(2000.0, 2000.0, 2000.0), scattering=(8000.0, 8000.0, 8000.0))
    sd.add_medium(absorption=(0.0, 0.0, 0.0), scattering=(0.0, 0.0, 0.0))
    sd.add_medium()
    sd._mediums[-1]["absorption_index"] = S.INVALID
    sd._mediums[-1]["scattering_index"] = S.INVALID
    for name in HETEROGENEOUS:
        grid, bounds, scattering, absorption, max_sigma = _HET[name]
        sd.add_medium(absorption=absorption, scattering=scattering, g=0.8, density=grid(), bounds=bounds, max_sigma=max_sigma)
    idx = {m: i for i, m in enumerate(MEDIA)}
    fog = sd.add_material("fog", cls=S.MAT_BOUNDARY, int_medium=idx["fog"])
    cloud = sd.add_material("cloud", cls=S.MAT_BOUNDARY, int_medium=idx["cloud"], ext_medium=idx["fog"])
    sheet = sd.add_material("sheet", cls=S.MAT_BOUNDARY, int_medium=idx["scatterer"], ext_medium=idx["fog"])
    void = sd.add_material("void", cls=S.MAT_VOID)
    wall = sd.add_material("wall", kd=[0.5, 0.5, 0.5])
    light = sd.add_material("light", kd=[0, 0, 0], emission=scenes.spd_rgb_luminance([4.0, 4.0, 4.0]))
    sd.add_box([0.0, 0.0, 0.0], (1.0, 1.0, 1.0), 0.0, fog)
    sd.add_box([0.0, 0.0, 0.0], (0.5, 0.5, 0.5), 0.0, cloud)

    def x_quad(x, mat):  # facing -x; its diagonal is y = z
        sd.add_quad([x, -0.5, -0.5], [x, -0.5, 0.5], [x, 0.5, 0.5], [x, 0.5, -0.5], mat)

    for k in range(STACK):
        x_quad(STACK_X0 + STACK_DX * k, sheet)
    x_quad(2.5, void)
    x_quad(5.0, wall)
    sd.add_quad([-0.2, 8.0, -0.2], [0.2, 8.0, -0.2], [0.2, 8.0, 0.2], [-0.2, 8.0, 0.2], light)
    sd.set_camera([0.0, 2.0, 6.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0], 8, 8, 45.0)
    return sd.finalize(samples=1, spectral=spectral)


def medium_index(name):
    return MEDIA.index(name)


def bounds(name):
    """the medium's bounds as the scene stores them (float32), in float64"""
    lo, hi = _HET[name][1]
    return np.array(lo, f32).astype(np.float64), np.array(hi, f32).astype(np.float64)


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


class _Builder:
    def __init__(self, spectral, rng):
        self.rows, self.bands, self.spectral, self.rng = [], [], spectral, rng

    def add(self, band, op, medium=0, origin=(0, 0, 0), direction=(0, 0, 1), max_t=1.0, end=(0, 0, 0), throughput=(1, 1, 1), g=0.0, rnd=(0.5, 0.5),
            w_o=(0, 0, 1)):
        q = np.zeros(1, S.MEDIUM_QUERY)
        q["op"], q["medium"], q["seed"] = op, medium, self.rng.integers(1, 2 ** 32 - 1)
        q["wavelength"] = self.rng.uniform(390.0, 760.0) if self.spectral else 0.0
        q["origin"], q["direction"], q["max_t"], q["end"] = origin, direction, max_t, end
        q["throughput"], q["g"], q["rnd"], q["w_o"] = throughput, g, rnd, w_o
        self.rows.append(q)
        self.bands.append(band)

    def done(self):
        return np.concatenate(self.rows), np.array(self.bands, dtype=object)


def _rays_heterogeneous(b, name, ops):
    """(band, origin, direction, max_t) rays about a heterogeneous medium's bounds, each for every op of `ops`"""
    rng = b.rng
    lo, hi = bounds(name)
    ext, mid = hi - lo, 0.5 * (lo + hi)
    diag = float(np.linalg.norm(ext))
    rays = []
    for _ in range(12):
        o = lo + ext * rng.random(3)
        rays.append(("inside", o, _unit(rng, 1)[0], rng.uniform(0.05, 2.0 * diag)))
    for _ in range(12):
        o = mid + _unit(rng, 1)[0] * diag * rng.uniform(0.8, 2.0)
        target = lo + ext * rng.random(3)
        d = (target - o) / np.linalg.norm(target - o)
        rays.append(("crossing", o, d, 3.0 * diag))
        rays.append(("miss", o, -d, 3.0 * diag))
        t_in = float(np.linalg.norm(target - o))
        rays.append(("ends_inside", o, d, t_in))
    for axes in ((0,), (1,), (2,), (0, 1), (1, 2), (0, 2)):
        for plane in (0.0, 1.0):
            o = lo + ext * rng.uniform(0.2, 0.8, 3)
            d = _unit(rng, 1)[0]
            for a in axes:
                o[a] = lo[a] if plane == 0.0 else hi[a]
                d[a] = 0.0
            rays.append(("axis", o, d / np.linalg.norm(d), rng.uniform(0.2, 2.0) * diag))
    for k in (1, 2, 3):  # a face, an edge, a corner
        for _ in range(4):
            o = lo + ext * rng.uniform(0.2, 0.8, 3)
            corner = rng.integers(0, 2, 3)
            for a in rng.permutation(3)[:k]:
                o[a] = hi[a] if corner[a] else lo[a]
            d = mid - o + 0.3 * ext * rng.normal(size=3)
            rays.append(("surface", o, d / np.linalg.norm(d), diag))
    o = lo + ext * rng.uniform(0.2, 0.8, 3)
    o[1] = lo[1]
    rays.append(("surface", o, np.array([0.6, 0.0, 0.8]), diag))  # tangent to the bottom face
    for _ in range(4):
        o = mid + 0.25 * ext * rng.normal(size=3)
        d = _unit(rng, 1)[0]
        rays.append(("max_float", o, d, K_MAX_FLOAT))
        rays.append(("short", o, d, np.nextafter(K_RAY_EPSILON, f32(1.0))))
        rays.append(("short", o, d, f32(1.5) * K_RAY_EPSILON))
        rays.append(("long", o, d, 1e4))
    for band, o, d, t in rays:
        for op in ops:
            b.add(band, op, medium_index(name), origin=o, direction=d, max_t=t, throughput=rng.uniform(0.2, 1.0, 3))


def _density_coords(b, name):
    rng = b.rng
    dims = np.array(_HET[name][0]().shape[::-1])
    m = medium_index(name)
    for _ in range(16):
        c = (rng.integers(0, dims) + 0.5) / dims
        b.add("centre", S.MEDIUM_DENSITY, m, origin=c)
        c2 = rng.integers(0, dims + 1) / dims
        b.add("face", S.MEDIUM_DENSITY, m, origin=np.minimum(c2, ONE_MINUS))
    specials = {"zero": (f32(0.0), f32(-0.0)), "top": (ONE_MINUS, f32(1.0)), "below": (f32(-2.0 ** -24), -np.nextafter(f32(0.0), f32(1.0)))}
    for band, values in specials.items():
        for v in values:
            for a in range(3):
                c = rng.uniform(0.1, 0.9, 3).astype(f32)
                c[a] = v
                b.add(band, S.MEDIUM_DENSITY, m, origin=c)
            b.add(band, S.MEDIUM_DENSITY, m, origin=(v, v, v))
    for _ in range(64):
        b.add("uniform", S.MEDIUM_DENSITY, m, origin=rng.random(3))


def _homogeneous(b, name):
    rng = b.rng
    m = medium_index(name)
    for op in (S.MEDIUM_TRANSMITTANCE, S.MEDIUM_SAMPLE):
        for _ in range(24):
            b.add("uniform", op, m, origin=rng.normal(size=3), direction=_unit(rng, 1)[0], max_t=10.0 ** rng.uniform(-3, 1), throughput=rng.uniform(0.1, 1.0, 3))
        for t in (K_MAX_FLOAT, 1e4, np.nextafter(K_RAY_EPSILON, f32(1.0)), f32(1.5) * K_RAY_EPSILON):
            band = "max_float" if t == K_MAX_FLOAT else ("long" if t == 1e4 else "short")
            for _ in range(3):
                b.add(band, op, m, origin=rng.normal(size=3), direction=_unit(rng, 1)[0], max_t=t, throughput=rng.uniform(0.1, 1.0, 3))
    for tp in ((1, 1, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0), (1e-30, 1, 1)):
        for t in (0.5, 20.0):
            b.add("throughput", S.MEDIUM_SAMPLE, m, origin=rng.normal(size=3), direction=_unit(rng, 1)[0], max_t=t, throughput=tp)


def _phase(b):
    rng = b.rng
    for g in PHASE_G:
        band = "g_edge" if abs(g) == 0.999 else ("g_small" if abs(g) <= 1e-3 else "uniform")
        for w_i in ((0, 0, 1), (0, 0, -1)):
            for x in (0.0, float(ONE_MINUS), 0.5):
                b.add("pole", S.MEDIUM_PHASE, direction=w_i, g=g, rnd=(x, rng.random()), w_o=_unit(rng, 1)[0])
        for x in (0.0, float(ONE_MINUS)):
            b.add("rnd_edge", S.MEDIUM_PHASE, direction=_unit(rng, 1)[0], g=g, rnd=(x, rng.random()), w_o=_unit(rng, 1)[0])
        b.add("rnd_edge", S.MEDIUM_PHASE, direction=_unit(rng, 1)[0], g=g, rnd=(0.5, float(ONE_MINUS)), w_o=_unit(rng, 1)[0])
        for _ in range(16):
            w_i = _unit(rng, 1)[0]
            w_o = w_i if _ == 0 else (-w_i if _ == 1 else _unit(rng, 1)[0])
            b.add(band, S.MEDIUM_PHASE, direction=w_i, g=g, rnd=rng.random(2), w_o=w_o)


def _segment(b):
    rng = b.rng
    fog, cloud, scat = medium_index("fog"), medium_index("cloud"), medium_index("scatterer")
    y, z = 0.2, -0.1

    def stack_end(n):  # between quad n - 1 and quad n
        return STACK_X0 + STACK_DX * (n - 0.5)

    for n in (0, 1, 2, 4, 61, 62, 63):
        for medium in (S.INVALID, fog):
            b.add(f"crossings_{n}", S.MEDIUM_SEGMENT, medium, origin=(STACK_X0 - 0.05, y, z), end=(stack_end(n), y + 0.01, z - 0.003))
    for medium in (S.INVALID, fog):
        b.add("opaque", S.MEDIUM_SEGMENT, medium, origin=(STACK_X0 + STACK_DX * 2.5, y, z), end=(5.5, y, z))
        b.add("void", S.MEDIUM_SEGMENT, medium, origin=(2.3, y, z), end=(2.9, y + 0.02, z))
        b.add("degenerate", S.MEDIUM_SEGMENT, medium, origin=(0.7, 0.7, 0.7), end=(0.7, 0.7, 0.7))
        b.add("degenerate", S.MEDIUM_SEGMENT, medium, origin=(0.7, 0.7, 0.7), end=(0.71, 0.7, 0.7))
    for _ in range(6):
        p_out = _unit(rng, 1)[0] * 1.8
        p_fog = rng.uniform(0.6, 0.95, 3) * rng.choice([-1, 1], 3)
        p_cloud = rng.uniform(-0.4, 0.4, 3)
        b.add("nested", S.MEDIUM_SEGMENT, S.INVALID, origin=p_out, end=-p_out + 0.1 * rng.normal(size=3))  # 4 crossings
        b.add("nested", S.MEDIUM_SEGMENT, fog, origin=p_fog, end=p_cloud)
        b.add("nested", S.MEDIUM_SEGMENT, cloud, origin=p_cloud, end=p_out)
        b.add("nested", S.MEDIUM_SEGMENT, fog, origin=p_fog, end=p_fog * np.array([1.0, 1.0, 1.0]) + 0.05 * rng.normal(size=3))
        b.add("nested", S.MEDIUM_SEGMENT, scat, origin=p_fog, end=p_out)  # a starting medium the geometry does not know


def make(sd, case, spectral, seed):
    b = _Builder(spectral, np.random.default_rng(seed))
    if case == "phase":
        _phase(b)
    elif case == "segment":
        _segment(b)
    elif case in HOMOGENEOUS:
        _homogeneous(b, case)
    else:
        _rays_heterogeneous(b, case, (S.MEDIUM_BOUNDS, S.MEDIUM_TRANSMITTANCE, S.MEDIUM_SAMPLE))  # every ray has max_t >= kRayEpsilon
        _density_coords(b, case)
    return b.done()


def distribution_queries(case, spectral, seed):
    """A few sample and transmittance queries whose results the GPU test bins over many repetitions: rays through the medium (homogeneous:
    max_t 2 from the origin)."""
    b = _Builder(spectral, np.random.default_rng(seed))
    m = medium_index(case)
    if case in HOMOGENEOUS:
        for tp in ((1.0, 1.0, 1.0), (0.3, 1.0, 0.6)):
            b.add("uniform", S.MEDIUM_SAMPLE, m, origin=(0.1, 0.2, 0.3), direction=(0.6, 0.0, 0.8), max_t=2.0 if case != "dense" else 1e-3, throughput=tp)
        b.add("uniform", S.MEDIUM_TRANSMITTANCE, m, origin=(0.1, 0.2, 0.3), direction=(0.6, 0.0, 0.8), max_t=0.5)
    else:
        lo, hi = bounds(case)
        mid, ext = 0.5 * (lo + hi), hi - lo
        o = mid - 0.9 * ext * np.array([0.8, 0.5, 0.6])
        d = (mid + 0.1 * ext - o) / np.linalg.norm(mid + 0.1 * ext - o)
        t = 2.0 * float(np.linalg.norm(ext))
        b.add("crossing", S.MEDIUM_SAMPLE, m, origin=o, direction=d, max_t=t, throughput=(1.0, 1.0, 1.0))
        b.add("crossing", S.MEDIUM_TRANSMITTANCE, m, origin=o, direction=d, max_t=t)
    return b.done()[0]
