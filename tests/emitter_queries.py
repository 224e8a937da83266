"""Scenes and seeded queries for the emitter tests (etxb_debug_emitter against the oracle's emitter routines).

CASES names one scene per emitter form; scene(case, spectral) builds it with scenes.SceneData, as the loader would:
  area_textured       three emitting triangles of unequal area under a textured emission image, collimation 0
  area_c05 / c09 / c1 the same triangles untextured at collimation 0.5, 0.9 and 1.0
  env_plain           a 32 x 16 lat-long image with a bright spot, sampling table built, wrapping in u (loader.py parse_env)
  env_rotated         the same with offset 0.3 ("rotation")
  env_mirrored        the same with scale -1
  env_mirrored_rotated  scale -1 and offset 0.3: the pinned reference quirk (DESIGN §10)
  env_black           black polar rows and a black column band: zero-width CDF steps, zero pdf
  env_single_row      a 32 x 1 image: Image::evaluate's flat pdf (fsize_y == 1)
  env_rgba8           an 8-bit image (Image::Format::RGBA8)
  env_placeholder     the 1 x 1 white image a missing file becomes
  dir_delta           a directional emitter of angular size 0
  dir_05 / dir_10     angular size 0.5 and 10 degrees
  dir_10_image        10 degrees with an image over its disk

make(sd, case, spectral, seed) returns (queries, band): S.EMITTER_QUERY records of the select, sample_in and radiance ops and, per query,
its band: polar, seam, cone_edge, near (within 1e-4 of an area emitter, or on the bounding sphere), grazing, axis (within 1e-3 rad
of an area emitter's normal), cdf_edge or uniform.  emission_queries(...) returns the emission op's queries.
"""
import math

import numpy as np

from etx_tracer_b200 import scenes, structs as S

f32 = np.float32
ONE_MINUS = np.nextafter(f32(1.0), f32(0.0))  # 1 - 2^-24
ENV_OFFSET = 0.3
BANDS = ("polar", "seam", "cone_edge", "near", "grazing", "axis", "cdf_edge", "uniform")

AREA_CASES = {"area_textured": 0.0, "area_c05": 0.5, "area_c09": 0.9, "area_c1": 1.0}
ENV_CASES = ("env_plain", "env_rotated", "env_mirrored", "env_mirrored_rotated", "env_black", "env_single_row", "env_rgba8", "env_placeholder")
DIR_CASES = {"dir_delta": 0.0, "dir_05": 0.5, "dir_10": 10.0, "dir_10_image": 10.0}
CASES = tuple(AREA_CASES) + ENV_CASES + tuple(DIR_CASES)
SUN_DIRECTION = (0.3, 0.8, 0.5)

# the emitting triangles: (p0, p1, p2) at y = 1, facing down (geometric normal -y), areas 0.08, 0.18 and 0.405
_TRIANGLES = [((-0.9, 1.0, -0.4), (-0.5, 1.0, -0.4), (-0.9, 1.0, 0.0)), ((-0.3, 1.0, -0.3), (0.3, 1.0, -0.3), (-0.3, 1.0, 0.3)),
              ((0.0, 1.0, 0.1), (0.9, 1.0, 0.1), (0.0, 1.0, 1.0))]
_TRI_UV = [(0.0, 0.0), (1.0, 0.0), (0.0, 1.0)]


def env_pixels(w=32, h=16, seed=17):
    """A smooth sky with a bright spot at (u, v) = (0.7, 0.3) and +-30% pixel noise, RGBA32F."""
    rng = np.random.default_rng(seed)
    v, u = np.meshgrid((np.arange(h) + 0.5) / h, (np.arange(w) + 0.5) / w, indexing="ij")
    base = np.stack([0.4 + 0.3 * u, 0.5 + 0.2 * np.cos(v * np.pi), 0.6 + 0.1 * v], axis=-1)
    spot = 20.0 * np.exp(-(((u - 0.7) * w) ** 2 + ((v - 0.3) * h) ** 2) / 4.0)
    img = base * (0.7 + 0.6 * rng.random((h, w, 1))) + spot[..., None] * np.array([1.0, 0.8, 0.6])
    return np.concatenate([img, np.ones((h, w, 1))], axis=-1).astype(f32)


def _disk_pixels(n=16):
    yy, xx = np.mgrid[0:n, 0:n]
    r = np.hypot((xx + 0.5) / n - 0.5, (yy + 0.5) / n - 0.5) * 2.0
    img = np.stack([1.0 - 0.6 * r, 0.8 - 0.3 * r, 0.3 + 0.5 * r], axis=-1).clip(0.05, None)
    return np.concatenate([img, np.ones((n, n, 1))], axis=-1).astype(f32)


def scene(case, spectral, plain=False):
    """`plain`: an environment case's image without its offset and scale (the lookups of a correct round trip)"""
    sd = scenes.SceneData()
    sd.name = f"emitters/{case}/{'spectral' if spectral else 'rgb'}"
    floor = sd.add_material("floor", kd=[0.5, 0.5, 0.5])
    sd.add_quad([-1, 0, 1], [1, 0, 1], [1, 0, -1], [-1, 0, -1], floor)
    if case in AREA_CASES:
        light = sd.add_material("light", kd=[0, 0, 0], emission=scenes.spd_rgb_luminance([4.0, 3.0, 2.0]), collimation=AREA_CASES[case])
        if case == "area_textured":
            sd.materials[light]["emission"]["image_index"] = sd.add_image(scenes.checker_image(8), repeat=True)
        for tri in _TRIANGLES:
            sd.add_mesh(tri, [(0.0, -1.0, 0.0)] * 3, [(0, 1, 2)], light, uvs=_TRI_UV)
    elif case in ENV_CASES:
        kw = dict(repeat=True, repeat_v=False, build_table=True)
        px = env_pixels()
        if case == "env_rotated":
            kw["offset"] = (ENV_OFFSET, 0.0)
        elif case == "env_mirrored":
            kw["scale"] = (-1.0, 1.0)
        elif case == "env_mirrored_rotated":
            kw.update(offset=(ENV_OFFSET, 0.0), scale=(-1.0, 1.0))
        elif case == "env_black":
            px[:2, :, :3] = 0.0
            px[-2:, :, :3] = 0.0
            px[:, 10:14, :3] = 0.0
        elif case == "env_single_row":
            px = px[5:6]
        elif case == "env_rgba8":
            px = (np.clip(px / px[..., :3].max(), 0.0, 1.0) * 255.0).astype(np.uint8)
            px[..., 3] = 255
        elif case == "env_placeholder":
            px = np.ones((1, 1, 4), f32)
            kw["repeat_v"] = True
        if plain:
            kw.update(offset=(0.0, 0.0), scale=(1.0, 1.0))
        sd.add_environment_emitter(sd.add_image(px, **kw), rgb=(1.0, 0.9, 0.8))
    else:
        image = sd.add_image(_disk_pixels(), repeat=False) if case == "dir_10_image" else S.INVALID
        sd.add_directional_emitter(SUN_DIRECTION, rgb=(3.0, 2.8, 2.5), angular_size_deg=DIR_CASES[case], image_index=image)
    sd.set_camera([0.0, 1.2, 3.6], [0.0, 0.5, 0.0], [0.0, 1.0, 0.0], 8, 8, 45.0)
    return sd.finalize(samples=1, spectral=spectral)


def collimation_exponent(c):
    """collimation_to_exponent (scene.hxx:67-71) in float64"""
    return 1.0 / max(1.192092896e-07, (1.0 - min(max(c, 0.0), 1.0)) ** 4)


def bounding_sphere(case):
    """centre and radius of the query scenes' bounding sphere (the floor quad's; the emitters lie inside it)"""
    sd = scene(case, False)
    return sd.scene["bounding_sphere_center"][0].astype(np.float64), float(sd.scene["bounding_sphere_radius"][0])


def env_image(sd):
    """(image record, pixels, (row entries, row-selection entries)) of the scene's environment emitter"""
    i = int(sd.a_profiles["emission"]["image_index"][int(sd.a_emitters["profile"][0])])
    return sd._images[i][0], sd._image_px[i], sd._image_tables[i]


# ---- float64 models of the lat-long mapping (math.hxx uv_to_direction / direction_to_uv) -------------------------------------------
def uv_to_direction(uv, offset=0.0, scale=1.0):
    u = np.asarray(uv[..., 0], np.float64)
    if scale < 0:
        u = 1.0 - u
    u = np.mod(u - offset, 1.0)
    phi, theta = (2.0 * u - 1.0) * np.pi, (0.5 - np.asarray(uv[..., 1], np.float64)) * np.pi
    return np.stack([np.cos(phi) * np.cos(theta), np.sin(theta), np.sin(phi) * np.cos(theta)], axis=-1)


def true_uv(d, offset=0.0, scale=1.0):
    """the inverse of uv_to_direction: the uv whose image the sampler picked"""
    d = np.asarray(d, np.float64)
    d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    u = np.mod(np.arctan2(d[..., 2], d[..., 0]) / (2.0 * np.pi) + 0.5 + offset, 1.0)
    if scale < 0:
        u = 1.0 - u
    v = 0.5 - np.arcsin(np.clip(d[..., 1], -1.0, 1.0)) / np.pi
    return np.stack([u, v], axis=-1)


def direction_to_uv(d, offset=0.0, scale=1.0):
    """the reference's direction_to_uv in float64: differs from true_uv when scale < 0 and offset != 0"""
    d = np.asarray(d, np.float64)
    d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    u = np.arctan2(d[..., 2], d[..., 0]) / (2.0 * np.pi) + 0.5
    if scale < 0:
        u = 1.0 - u
    u = np.mod(u + offset, 1.0)
    return np.stack([u, 0.5 - np.arcsin(np.clip(d[..., 1], -1.0, 1.0)) / np.pi], axis=-1)


def pixel_model(sd):
    """float64 probability of each environment pixel (h, w) under Image::sample: the luminance of the mean of the 2 x 2 texels from each
    pixel (wrapping in u, clamped in v) times sin((y + 0.5) / h pi), normalised; a black image is uniform."""
    rec, px, _ = env_image(sd)
    px = px[..., :3].astype(np.float64)
    h, w = px.shape[:2]
    xs, ys = (np.arange(w) + 1) % w, np.minimum(np.arange(h) + 1, h - 1)
    if int(rec["options"]) & 4:  # RepeatV: the placeholder
        ys = (np.arange(h) + 1) % h
    avg = 0.25 * (px + px[:, xs] + px[ys] + px[ys][:, xs])
    lum = avg @ np.array([0.212671, 0.715160, 0.072169])
    p = lum * np.sin((np.arange(h)[:, None] + 0.5) / h * np.pi)
    return p / p.sum() if p.sum() > 0 else np.full(p.shape, 1.0 / p.size)


def pixel_of(sd, d):
    """the pixel (flat index) each direction's true uv lies in"""
    rec, _, _ = env_image(sd)
    w, h = (int(x) for x in rec["isize"])
    uv = true_uv(d, float(rec["offset"][0]), float(rec["scale"][0]))
    x = np.clip(np.floor(uv[..., 0] * w), 0, w - 1).astype(np.int64)
    y = np.clip(np.floor(uv[..., 1] * h), 0, h - 1).astype(np.int64)
    return y * w + x


# ---- queries ------------------------------------------------------------------------------------------------------------------------
def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _sphere(rng, n):
    return _unit(rng.normal(size=(n, 3)))


def _basis(n):
    n = _unit(n)
    a = np.array([1.0, 0.0, 0.0]) if abs(n[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    u = _unit(np.cross(n, a))
    return u, np.cross(n, u)


def _wavelengths(rng, n):
    wl = rng.uniform(390.0, 830.0, n)
    wl[:2] = (390.0, 830.0)[:n]
    return wl


def _queries(op, n):
    q = np.zeros(n, dtype=S.EMITTER_QUERY)
    q["op"] = op
    return q


def _pole_directions():
    """exactly at the poles, and |y| = 1 - k 2^-24 (k = 1..8) with the rest in tiny x and z, both poles"""
    out = []
    for s in (1.0, -1.0):
        out.append((0.0, s, 0.0))
        out.append((1e-30, s, -1e-30))
        for k in range(1, 9):
            y = 1.0 - k * 2.0 ** -24
            r = math.sqrt(1.0 - y * y)
            for phi in (0.3, 2.5, -1.9):
                out.append((r * math.cos(phi), s * y, r * math.sin(phi)))
    return np.array(out)


def _seam_directions(rng):
    """phi = +-pi: x < 0 with z = +0, -0 and +-1 ulp, at several heights"""
    out = []
    for y in (0.0, 0.5, -0.7, 0.95):
        x = -math.sqrt(1.0 - y * y)
        for z in (0.0, -0.0, 1e-8, -1e-8, np.nextafter(f32(0), f32(1)), -np.nextafter(f32(0), f32(1))):
            out.append((x, y, z))
    return np.array(out)


def _sampler_values(x):
    """values a sampler can return: 0 and [2^-24, 1) (the product build flushes the denormal neighbours of 0 to 0)"""
    return (x == 0) | ((x >= 2.0 ** -24) & (x < 1))


def make(sd, case, spectral, seed, count=256):
    rng = np.random.default_rng(seed)
    parts = []  # (band, queries)
    center, radius = sd.scene["bounding_sphere_center"][0].astype(np.float64), float(sd.scene["bounding_sphere_radius"][0])
    ne = sd.a_emitters.shape[0]

    # select: rnd at 0, 1 - 2^-24, on every CDF entry (zero-width steps included) and uniform
    cdf = sd.a_dist["cdf"].astype(f32)
    edge = np.concatenate([[0.0, ONE_MINUS], cdf, np.nextafter(cdf, f32(0)), np.nextafter(cdf, f32(2))]).astype(f32)
    edge = edge[_sampler_values(edge)]
    q = _queries(S.EMITTER_SELECT, edge.shape[0])
    q["rnd"][:, 0] = edge
    parts.append(("cdf_edge", q))
    q = _queries(S.EMITTER_SELECT, count)
    q["rnd"][:, 0] = rng.random(count)
    parts.append(("uniform", q))

    def sample_in(band, rnd, from_point, emitter=0):
        q = _queries(S.EMITTER_SAMPLE_IN, rnd.shape[0])
        q["rnd"], q["source"], q["emitter"] = rnd, from_point, emitter
        parts.append((band, q))

    def radiance(band, direction, source=(0.0, 0.0, 0.0), target=(0.0, 0.0, 0.0), uv=(0.0, 0.0), emitter=0):
        n = np.asarray(direction).shape[0]
        for visible in (0, 1):
            q = _queries(S.EMITTER_RADIANCE, n)
            q["direction"], q["source"], q["target"], q["uv"], q["emitter"] = direction, source, target, uv, emitter
            q["directly_visible"] = visible
            parts.append((band, q))

    if case in AREA_CASES:
        tri_of = np.arange(ne)
        for e in tri_of:
            p = np.array(_TRIANGLES[e], np.float64)
            centroid = p.mean(0)
            # below the triangle (the emitting side), on its back, grazing its plane, within 1e-4 of it
            below = np.column_stack([rng.uniform(-1, 1, count), rng.uniform(0.0, 0.9, count), rng.uniform(-1, 1, count)])
            sample_in("uniform", rng.random((count, 2)), below, e)
            above = np.column_stack([rng.uniform(-1, 1, 32), rng.uniform(1.05, 2.0, 32), rng.uniform(-1, 1, 32)])
            sample_in("uniform", rng.random((32, 2)), above, e)
            far = centroid + np.column_stack([np.cos(a := rng.uniform(0, 2 * np.pi, 32)) * 3.0, -rng.uniform(1e-3, 5e-2, 32), np.sin(a) * 3.0])
            sample_in("grazing", rng.random((32, 2)), far, e)
            near = centroid + np.column_stack([rng.uniform(-0.05, 0.05, 32), -np.exp(rng.uniform(np.log(1e-6), np.log(1e-4), 32)), rng.uniform(-0.05, 0.05, 32)])
            sample_in("near", rng.random((32, 2)), near, e)
            edges = np.array([(0.0, 0.0), (ONE_MINUS, ONE_MINUS), (0.0, ONE_MINUS), (ONE_MINUS, 0.0), (0.5, 0.0), (0.0, 0.5)], f32)
            sample_in("cdf_edge", edges, np.tile(centroid - (0.0, 0.5, 0.0), (edges.shape[0], 1)), e)
            # radiance: targets on the triangle from sources on both sides, grazing and near
            bc = rng.dirichlet((1.0, 1.0, 1.0), count)
            target = bc @ p
            radiance("uniform", np.zeros((count, 3)), below, target, rng.random((count, 2)), e)
            radiance("uniform", np.zeros((32, 3)), above, target[:32], rng.random((32, 2)), e)
            radiance("grazing", np.zeros((32, 3)), far, target[:32], rng.random((32, 2)), e)
            radiance("near", np.zeros((32, 3)), near, target[:32], rng.random((32, 2)), e)
        # on the normal through a point of each triangle, 2e-4 to 8e-4 rad off it: where a collimated emitter's pdf is not 0
        for e in tri_of:
            p = np.array(_TRIANGLES[e], np.float64)
            target = rng.dirichlet((1.0, 1.0, 1.0), 32) @ p
            a, ph, dist = rng.uniform(2e-4, 8e-4, 32), rng.uniform(0, 2 * np.pi, 32), rng.uniform(0.3, 0.9, 32)
            source = target + dist[:, None] * np.column_stack([np.sin(a) * np.cos(ph), -np.cos(a), np.sin(a) * np.sin(ph)])
            radiance("axis", np.zeros((32, 3)), source, target, rng.random((32, 2)), e)
    elif case in ENV_CASES:
        rec, _, (rows, ey) = env_image(sd)
        h = rows.shape[0]
        inside = center + _sphere(rng, count) * (radius * rng.random((count, 1)) ** (1 / 3))
        sample_in("uniform", rng.random((count, 2)), inside)
        sample_in("near", rng.random((16, 2)), center + _sphere(rng, 16) * radius)  # on the bounding sphere
        sample_in("uniform", rng.random((16, 2)), center + _sphere(rng, 16) * (2.0 * radius))
        # rnd.y on the row-selection CDF (either side of each entry), rnd.x on the CDF of the row it selects
        ycdf = ey["cdf"][:h].astype(f32)
        ys = np.concatenate([ycdf, np.nextafter(ycdf, f32(2)), np.nextafter(ycdf, f32(0))])
        ys = ys[_sampler_values(ys)]
        ry = rng.integers(0, h, ys.shape[0])
        xcdf = rows["cdf"][ry, rng.integers(0, rows.shape[1] - 1, ys.shape[0])].astype(f32)
        rnd = np.column_stack([xcdf, ys])
        extreme = (rnd[:, 1] == 0) | (rnd[:, 1] >= ONE_MINUS)
        sample_in("cdf_edge", rnd[~extreme], np.tile(center, (int((~extreme).sum()), 1)))
        poles = np.array([(0.0, 0.0), (ONE_MINUS, 0.0), (0.5, 0.0), (0.0, ONE_MINUS), (ONE_MINUS, ONE_MINUS), (0.5, ONE_MINUS)], f32)
        sample_in("polar", np.concatenate([poles, rnd[extreme]]), np.tile(center, (poles.shape[0] + int(extreme.sum()), 1)))
        radiance("uniform", _sphere(rng, count))
        radiance("polar", _pole_directions())
        radiance("seam", _seam_directions(rng))
        # on texel edges (a single-row image: at mid-height)
        row = rng.integers(1, h, 32) / float(rec["fsize"][1]) if h > 1 else np.full(32, 0.5)
        texel = np.column_stack([rng.integers(0, int(rec["isize"][0]), 32) / float(rec["fsize"][0]), row])
        radiance("cdf_edge", uv_to_direction(texel, float(rec["offset"][0]), float(rec["scale"][0])))
    else:
        em_dir = np.array(sd.a_profiles["direction"][0], np.float64)
        half = 0.5 * float(sd.a_profiles["angular_size"][0])
        u, v = _basis(em_dir)
        inside = center + _sphere(rng, count) * (radius * rng.random((count, 1)) ** (1 / 3))
        sample_in("uniform", rng.random((count, 2)), inside)
        sample_in("near", rng.random((16, 2)), center + _sphere(rng, 16) * radius)  # on the bounding sphere
        sample_in("uniform", rng.random((16, 2)), center + _sphere(rng, 16) * (2.0 * radius))
        edges = np.array([(0.0, 0.0), (ONE_MINUS, ONE_MINUS), (0.0, ONE_MINUS), (ONE_MINUS, 0.0), (0.5, 0.0), (0.0, 0.5)], f32)
        sample_in("cdf_edge", edges, np.tile(center, (edges.shape[0], 1)))
        phi = rng.uniform(0, 2 * np.pi, count)
        ang = half * np.sqrt(rng.random(count)) if half > 0 else np.zeros(count)
        cone = lambda a, ph: _unit(np.cos(a)[:, None] * em_dir + np.sin(a)[:, None] * (np.cos(ph)[:, None] * u + np.sin(ph)[:, None] * v))
        radiance("uniform", np.concatenate([cone(ang, phi), cone(rng.uniform(half, np.pi, 64), phi[:64])]))
        # either side of the cone's edge: a few ulps of angle around half the angular size
        k = np.arange(-8, 9, dtype=np.float64)
        a = np.clip(half + k * 1.2e-7 * max(half, 1e-3), 0.0, None)
        radiance("cone_edge", cone(np.tile(a, 4), np.repeat(rng.uniform(0, 2 * np.pi, 4), k.shape[0])))
        radiance("cone_edge", np.tile(em_dir, (4, 1)))
    q = np.concatenate([p for _, p in parts])
    band = np.concatenate([np.full(p.shape[0], b, dtype=object) for b, p in parts])
    q["seed"] = rng.integers(0, 2 ** 32, q.shape[0], dtype=np.uint64).astype(np.uint32)
    q["wavelength"] = _wavelengths(rng, q.shape[0]) if spectral else -1.0
    return q, band


def emission_queries(seed, spectral, count=16):
    """the emission op on `count` random seeds (the repetitions run on the sampler (seed, r))"""
    rng = np.random.default_rng(seed)
    q = _queries(S.EMITTER_EMISSION, count)
    q["seed"] = rng.integers(0, 2 ** 32, count, dtype=np.uint64).astype(np.uint32)
    q["wavelength"] = _wavelengths(rng, count) if spectral else -1.0
    return q


def distribution_queries(sd, spectral, seed, n):
    """n sample_in queries from the bounding sphere's centre with uniform rnd, for the distribution tests"""
    rng = np.random.default_rng(seed)
    q = _queries(S.EMITTER_SAMPLE_IN, n)
    q["rnd"] = rng.random((n, 2))
    q["source"] = sd.scene["bounding_sphere_center"][0]
    q["wavelength"] = _wavelengths(rng, n) if spectral else -1.0
    return q


def area_uv(r):
    """the uv sample_emitter looks the emission image up at: the vertex uvs interpolated at the sample's barycentric"""
    b = r["barycentric"].astype(np.float64)
    return b @ np.array(_TRI_UV)
