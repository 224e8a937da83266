"""The scenes and seeded queries for the subsurface tests (etxb_debug_subsurface against the oracle's subsurface routines).

One scene per geometry of GEOMETRIES, RGB or spectral.  Each holds its geometry once per material of the case, all copies in the same
place: the gathers and both ray queries only see triangles of one material, so the copies never meet.
  plane      a flat axis-aligned 40 x 40 quad at y = 0 (probes 1 and 2 of a gather at normal incidence lie in its plane)
  slab       two parallel quads at y = 0 and y = -0.05 facing apart (a thin slab)
  box        a closed box of half size 0.5
  sphere     a smooth-normal UV sphere of radius 0.5
  stack      STACK quads facing +y at y = -0.01 k; between them a Void quad, two alpha-tested quads (texel alpha 0 and 0.5) and a quad
             of another material (all on the entry material's own texture, uv fixed per quad)
  origin     a triangle through the world origin (an empty probe starts there: origin 0, direction 0)
  open_quad  one 1 x 1 quad: most random walks leave through nothing and end on a failure
and "remap" (no geometry of its own: the remap op).

Materials (MATERIALS; each case takes its list from CASE_MATERIALS):
  cb_grey        Christensen-Burley, grey distances 0.3
  cb_zero        Christensen-Burley, distances (0.5, 0.2, 0): an RGB probe on the blue channel is empty
  cb_tiny        Christensen-Burley at distance scale 1e-6
  cb_huge        Christensen-Burley at distance scale 1e3
  cb_tex         Christensen-Burley with a distance image of black and white texels
  rw_grey        random walk, diffuse entry, grey color 0.5 and distances 0.2 (every exit weight is albedo^k)
  rw_diffuse     random walk, diffuse entry, chromatic
  rw_refracted   random walk, refracted entry (the walk starts along the entry's w_i)
  rw_medium_g    random walk over an int_medium with g = 0.7
  rw_medium_zero random walk over an int_medium whose blue channel has zero extinction (max_t = kMaxFloat there)
  rw_tex         random walk with a textured scattering color
  rw_tiny        random walk at distance scale 1e-6 (extinction 1024: the walk runs into its 1024-step cap or its throughput floor)
  rw_huge        random walk at distance scale 1e3
The stack case uses cb_alpha and rw_alpha: cb_grey and rw_grey on the alpha texture.

make(case, spectral, seed) returns (scene, queries, band, material_of_query); bands name the op and the edge each query sits on:
  trace/<material|any>/<kind> and ctrace/<max_count>/<kind> (kind: hit, miss, coplanar, grazing, stack)
  remap/<color band>/<distance band>
  s_r/<rnd band>, profile/<direction>/<radius band>/<entry>, gather/<entry> (entry: face, edge, vertex x normal, grazing)
"""
import numpy as np

from etx_tracer_b200 import scenes, structs as S

f32 = np.float32
K_EPSILON = f32(1.192092896e-07)
K_RAY_EPSILON = f32(15.0) / f32(65504.0 - 1.0)
K_MAX_FLOAT = f32(3.402823466e38)
K_MAX_RADIUS = f32(47.827155457397595950044717258511)
ONE_MINUS = np.nextafter(f32(1.0), f32(0.0))  # 1 - 2^-24
RND_BANDS = {"zero": f32(0.0), "below_quarter": f32(0.25) - f32(2.0 ** -26), "quarter": f32(0.25), "clamp": ONE_MINUS, "mid": f32(0.6)}
COLOR_BANDS = {"neg": f32(-1.0), "zero": f32(0.0), "one": f32(1.0), "two": f32(2.0)}
DISTANCE_BANDS = {"zero": f32(0.0), "min": f32(2.0 ** -11), "one": f32(1.0)}
STACK = 12
GEOMETRIES = ("plane", "slab", "box", "sphere", "stack", "origin", "open_quad")
CASES = GEOMETRIES + ("remap",)
MATERIALS = {
    "cb_grey": dict(kd=[0.5, 0.5, 0.5], subsurface=dict(cls="burley", distances=[0.3, 0.3, 0.3])),
    "cb_zero": dict(kd=[0.9, 0.5, 0.2], subsurface=dict(cls="burley", distances=[0.5, 0.2, 0.0])),
    "cb_tiny": dict(kd=[0.7, 0.6, 0.5], subsurface=dict(cls="burley", distances=[1.0, 0.4, 0.15], scale=1e-6)),
    "cb_huge": dict(kd=[0.7, 0.6, 0.5], subsurface=dict(cls="burley", distances=[1.0, 0.4, 0.15], scale=1e3)),
    "cb_tex": dict(kd=[0.8, 0.7, 0.6], subsurface=dict(cls="burley", distances=[0.4, 0.3, 0.2], image="distance_checker")),
    "rw_grey": dict(kd=[0.5, 0.5, 0.5], subsurface=dict(cls="random_walk", path="diffuse", distances=[0.2, 0.2, 0.2])),
    "rw_diffuse": dict(kd=[0.8, 0.6, 0.4], subsurface=dict(cls="random_walk", path="diffuse", distances=[1.0, 0.4, 0.15], scale=0.12)),
    "rw_refracted": dict(kd=[0.9, 0.8, 0.7], subsurface=dict(cls="random_walk", path="refracted", distances=[0.3, 0.6, 1.0], scale=0.1)),
    "rw_medium_g": dict(kd=[0.8, 0.8, 0.8], int_medium="hg", subsurface=dict(cls="random_walk", path="diffuse")),
    "rw_medium_zero": dict(kd=[0.8, 0.8, 0.8], int_medium="zero_blue", subsurface=dict(cls="random_walk", path="diffuse")),
    "rw_tex": dict(kd=[1.0, 1.0, 1.0], scattering_image="color_checker", subsurface=dict(cls="random_walk", path="diffuse", distances=[0.5, 0.3, 0.2], scale=0.2)),
    "rw_tiny": dict(kd=[0.8, 0.6, 0.4], subsurface=dict(cls="random_walk", path="diffuse", distances=[1.0, 0.4, 0.15], scale=1e-6)),
    "rw_huge": dict(kd=[0.8, 0.6, 0.4], subsurface=dict(cls="random_walk", path="diffuse", distances=[1.0, 0.4, 0.15], scale=1e3)),
    "cb_alpha": dict(kd=[1.0, 1.0, 1.0], scattering_image="alpha_strip", subsurface=dict(cls="burley", distances=[0.3, 0.3, 0.3])),
    "rw_alpha": dict(kd=[1.0, 1.0, 1.0], scattering_image="alpha_strip", subsurface=dict(cls="random_walk", path="diffuse", distances=[0.2, 0.2, 0.2])),
}
_ALL = ("cb_grey", "cb_zero", "cb_tiny", "cb_huge", "cb_tex", "rw_grey", "rw_diffuse", "rw_refracted", "rw_medium_g", "rw_medium_zero", "rw_tex",
        "rw_tiny", "rw_huge")
CASE_MATERIALS = {
    "plane": _ALL, "slab": ("cb_grey", "cb_zero", "rw_grey", "rw_diffuse", "rw_refracted", "rw_medium_g"),
    "box": _ALL, "sphere": ("cb_grey", "cb_zero", "rw_grey", "rw_diffuse", "rw_refracted", "rw_medium_zero", "rw_tex"),
    "stack": ("cb_alpha", "rw_alpha"), "origin": ("cb_zero", "cb_grey", "rw_grey"), "open_quad": ("rw_grey", "rw_diffuse", "rw_refracted", "cb_grey"),
    "remap": ("rw_grey",),
}
# the materials whose gathers the distribution test runs 2^16 times per entry, per case
DIST_MATERIALS = {"plane": ("cb_grey", "rw_grey"), "slab": ("cb_zero", "rw_diffuse"), "box": ("cb_grey", "rw_diffuse", "rw_medium_g"),
                  "sphere": ("cb_zero", "rw_refracted"), "stack": ("cb_alpha", "rw_alpha"), "origin": ("cb_zero",), "open_quad": ("rw_grey",)}
# the alpha strip's texels (u = 0.125, 0.375, 0.625, 0.875): opaque, opaque, alpha 0, alpha 0.5
STACK_UV = {"opaque": (0.125, 0.5), "alpha0": (0.625, 0.5), "alpha_half": (0.875, 0.5)}


def _images(sd):
    checker = np.ones((4, 4, 4), f32)
    yy, xx = np.mgrid[0:4, 0:4]
    checker[((xx + yy) % 2) == 1, :3] = 0.0  # black texels: zero distances there
    colors = np.concatenate([np.random.default_rng(11).uniform(0.05, 1.0, (4, 4, 3)), np.ones((4, 4, 1))], -1).astype(f32)
    strip = np.ones((1, 4, 4), f32)
    strip[0, :, :3] = 0.5
    strip[0, 2, 3], strip[0, 3, 3] = 0.0, 0.5
    return {"distance_checker": sd.add_image(checker), "color_checker": sd.add_image(colors), "alpha_strip": sd.add_image(strip)}


def _add_material(sd, name, images, mediums):
    kw = dict(MATERIALS[name])
    ss = dict(kw.pop("subsurface"))
    if "image" in ss:
        ss["image"] = images[ss["image"]]
    tex = kw.pop("scattering_image", None)
    if "int_medium" in kw:
        kw["int_medium"] = mediums[kw["int_medium"]]
    m = sd.add_material(name, subsurface=ss, **kw)
    if tex is not None:
        sd.materials[m]["scattering"]["image_index"] = images[tex]
    return m


def _quad_uv(sd, p0, p1, p2, p3, mat, uv):
    """a quad whose four vertices share one texture coordinate (one texel of the entry material's image)"""
    p = np.array([p0, p1, p2, p3], np.float64)
    n = np.cross(p[1] - p[0], p[3] - p[0])
    sd.add_mesh(p, np.tile(n / np.linalg.norm(n), (4, 1)), np.array([(0, 1, 2), (0, 2, 3)]), mat, uvs=np.tile(np.array(uv, np.float64), (4, 1)))


def _geometry(sd, case, mat, other, void):
    if case == "plane":
        sd.add_quad([-20, 0, 20], [20, 0, 20], [20, 0, -20], [-20, 0, -20], mat)
    elif case == "slab":
        sd.add_quad([-20, 0, 20], [20, 0, 20], [20, 0, -20], [-20, 0, -20], mat)
        sd.add_quad([-20, -0.05, -20], [20, -0.05, -20], [20, -0.05, 20], [-20, -0.05, 20], mat)
    elif case == "box":
        sd.add_box([0.0, 0.0, 0.0], (0.5, 0.5, 0.5), 0.0, mat)
    elif case == "sphere":
        sd.add_uv_sphere([0.0, 0.0, 0.0], 0.5, 16, 9, mat)
    elif case == "stack":
        def y_quad(y, m, uv):
            _quad_uv(sd, [-1, y, 1], [1, y, 1], [1, y, -1], [-1, y, -1], m, uv)

        for k in range(STACK):
            y_quad(-0.01 * k, mat, STACK_UV["opaque"])
        y_quad(-0.005, void, STACK_UV["opaque"])
        y_quad(-0.015, mat, STACK_UV["alpha0"])
        y_quad(-0.025, mat, STACK_UV["alpha_half"])
        y_quad(-0.035, other, STACK_UV["opaque"])
    elif case == "origin":
        sd.add_mesh([[-1.0, 0.0, -1.0], [2.0, 0.0, 0.5], [-1.0, 0.0, 1.5]], [[0, 1, 0]] * 3, [(0, 2, 1)], mat, uvs=[[0, 0], [1, 0], [0, 1]])
    elif case == "open_quad":
        sd.add_quad([-0.5, 0, 0.5], [0.5, 0, 0.5], [0.5, 0, -0.5], [-0.5, 0, -0.5], mat)


def scene(case, spectral):
    """(SceneData finalized, {material name: (material index, first triangle, triangle count)})"""
    sd = scenes.SceneData()
    sd.name = f"subsurface/{case}/{'spectral' if spectral else 'rgb'}"
    images = _images(sd)
    mediums = {"hg": sd.add_medium(absorption=(0.2, 0.2, 0.2), scattering=(6.0, 5.0, 4.0), g=0.7),
               "zero_blue": sd.add_medium(absorption=(0.5, 1.0, 0.0), scattering=(4.0, 2.0, 0.0), g=-0.3)}
    other = sd.add_material("other", kd=[0.5, 0.5, 0.5])
    void = sd.add_material("void", cls=S.MAT_VOID)
    light = sd.add_material("light", kd=[0, 0, 0], emission=scenes.spd_rgb_luminance([4.0, 4.0, 4.0]))
    sd.add_quad([-0.2, 60.0, -0.2], [0.2, 60.0, -0.2], [0.2, 60.0, 0.2], [-0.2, 60.0, 0.2], light)
    info = {}
    for name in CASE_MATERIALS[case]:
        m = _add_material(sd, name, images, mediums)
        first = sum(t.shape[0] for t in sd.triangles)
        _geometry(sd, case if case != "remap" else "open_quad", m, other, void)
        info[name] = (m, first, sum(t.shape[0] for t in sd.triangles) - first)
    sd.set_camera([0.0, 2.0, 6.0], [0.0, 0.0, 0.0], [0.0, 1.0, 0.0], 8, 8, 45.0)
    return sd.finalize(samples=1, spectral=spectral), info


def triangle_frame(sd, tri):
    """(p0, p1, p2, geometric normal) of a triangle, float64"""
    t = np.concatenate(sd.triangles)[tri]
    v = np.concatenate(sd.vertices)["pos"].astype(np.float64)
    p = v[t["i"]]
    return p[0], p[1], p[2], t["geo_n"].astype(np.float64)


def _unit(v):
    return v / np.linalg.norm(v)


class _Builder:
    def __init__(self, spectral, rng):
        self.rows, self.bands, self.mats, self.spectral, self.rng = [], [], [], spectral, rng

    def add(self, band, mat_name, op, **fields):
        q = np.zeros(1, S.SUBSURFACE_QUERY)
        q["op"], q["seed"], q["material"] = op, self.rng.integers(1, 2 ** 32 - 1), S.INVALID
        q["wavelength"] = self.rng.uniform(390.0, 760.0) if self.spectral else 0.0
        q["t_min"], q["t_max"], q["dir"] = K_RAY_EPSILON, K_MAX_FLOAT, (0.0, -1.0, 0.0)
        for k, v in fields.items():
            q[k] = v
        self.rows.append(q)
        self.bands.append(band)
        self.mats.append(mat_name)

    def done(self):
        return np.concatenate(self.rows), np.array(self.bands, dtype=object), np.array(self.mats, dtype=object)


def entries(sd, info, name, rng, triangles=2):
    """(entry band, triangle, u, v, w_i) on `triangles` triangles of the material: face, edge and vertex coordinates at normal and grazing
    incidence (w_i points into the surface, against the geometric normal)"""
    m, first, n = info[name]
    out = []
    for tri in rng.choice(np.arange(first, first + n), size=min(triangles, n), replace=False):
        p0, p1, p2, gn = triangle_frame(sd, int(tri))
        e = _unit(p1 - p0)
        for loc, (u, v) in (("face", tuple(rng.dirichlet((1, 1, 1))[1:])), ("edge", (0.0, float(rng.random()))), ("edge", (0.5, 0.5)),
                            ("vertex", (0.0, 0.0)), ("vertex", (1.0, 0.0)), ("vertex", (0.0, 1.0))):
            for inc, w in (("normal", -gn), ("grazing", _unit(-0.02 * gn + e))):
                out.append((f"{loc}/{inc}", int(tri), u, v, w))
    return out


def make(case, spectral, seed):
    sd, info = scene(case, spectral)
    b = _Builder(spectral, np.random.default_rng(seed))
    rng = b.rng
    if case == "remap":
        for cn, c in COLOR_BANDS.items():
            for dn, d in DISTANCE_BANDS.items():
                b.add(f"remap/{cn}/{dn}", "", S.SUBSURFACE_REMAP, color=(c, c * f32(0.5), rng.uniform(0, 1)), distances=(d, d * f32(2.0), rng.uniform(0, 2)))
        for _ in range(32):
            b.add("remap/uniform", "", S.SUBSURFACE_REMAP, color=rng.uniform(-0.2, 1.2, 3), distances=10.0 ** rng.uniform(-5, 2, 3))
        for rn, r in RND_BANDS.items():
            b.add(f"s_r/{rn}", "rw_grey", S.SUBSURFACE_PROFILE, triangle=0, rnd=r, radius=1.0, normal=(0, 1, 0), dir=(0, -1, 0))
        for r in np.linspace(0, 1, 64, endpoint=False):
            b.add("s_r/uniform", "rw_grey", S.SUBSURFACE_PROFILE, triangle=0, rnd=r, radius=1.0, normal=(0, 1, 0), dir=(0, -1, 0))
        q, band, mats = b.done()
        return sd, info, q, band, mats
    for name in CASE_MATERIALS[case]:
        m, first, n = info[name]
        for eb, tri, u, v, w in entries(sd, info, name, rng):
            b.add(f"gather/{eb}", name, S.SUBSURFACE_GATHER, triangle=tri, u=u, v=v, dir=w)
            if eb.endswith("normal"):
                for d in range(3):
                    for rn, r in (("zero", 0.0), ("eps", K_EPSILON), ("r_max", K_MAX_RADIUS * f32(0.3)), ("mid", rng.uniform(0.01, 1.0))):
                        b.add(f"profile/{d}/{rn}/{eb.split('/')[0]}", name, S.SUBSURFACE_PROFILE, triangle=tri, u=u, v=v, dir=w, direction=d, radius=r,
                              rnd=rng.random(), normal=_unit(rng.normal(size=3)))
        # ray queries: down onto the geometry from above, up from below, grazing, and along its plane
        p0, p1, p2, gn = triangle_frame(sd, first)
        centre = (p0 + p1 + p2) / 3.0
        for mat_band, mat in ((name, m), ("any", S.INVALID)):
            for kind, o, d in (("hit", centre + 2.0 * gn, -gn), ("hit", centre - 3.0 * gn + 0.01 * rng.normal(size=3), gn), ("miss", centre + 2.0 * gn, gn),
                               ("grazing", centre + 0.01 * gn - 2.0 * _unit(p1 - p0), _unit(p1 - p0) - 0.004 * gn),
                               ("coplanar", centre - 2.0 * _unit(p1 - p0), _unit(p1 - p0))):
                b.add(f"trace/{'own' if mat_band == name else 'any'}/{kind}", name, S.SUBSURFACE_TRACE_MATERIAL, material=mat, origin=o, dir=_unit(d))
                for mc in (1, 7, 8):
                    b.add(f"ctrace/{mc}/{kind}", name, S.SUBSURFACE_CONTINUOUS_TRACE, material=mat, origin=o, dir=_unit(d), max_count=mc)
                    if kind == "hit":  # the ray interval ends before the farthest candidate
                        b.add(f"ctrace/{mc}/short", name, S.SUBSURFACE_CONTINUOUS_TRACE, material=mat, origin=o, dir=_unit(d), max_count=mc, t_max=2.5)
    q, band, mats = b.done()
    return sd, info, q, band, mats


def distribution_queries(case, spectral, seed, sd, info):
    """One gather at normal incidence on a face per material of DIST_MATERIALS[case], for the distribution test."""
    b = _Builder(spectral, np.random.default_rng(seed))
    for name in DIST_MATERIALS[case]:
        m, first, n = info[name]
        p0, p1, p2, gn = triangle_frame(sd, first)
        b.add("gather/face/normal", name, S.SUBSURFACE_GATHER, triangle=first, u=0.3, v=0.3, dir=-gn)
    return b.done()
