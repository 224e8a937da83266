"""Deterministic synthetic scene generators for the BASELINE.json configs.

They fill the reference's Scene/Camera PODs (etx_tracer_b200/structs.py) the way the reference's loader would
(sources/etx/render/host/scene_representation.cxx: commit():420, add_area_emitters_for_triangle:840,
build_emitters_distribution:2460, validate_materials:262, build_camera:579) so that the same arrays can be handed
to the CUDA module (etxb_upload_scene) and to the CPU oracle.  No file IO besides the committed data tables.
"""
import math
import os

import numpy as np

from . import structs as S

f32 = np.float32
DATA_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")

_tables = {}


def tables(name):
    if name not in _tables:
        _tables[name] = dict(np.load(os.path.join(DATA_DIR, name + ".npz")))
    return _tables[name]


K_RGB_LUMINANCE_SCALE = np.array([0.817660332, 1.05418909, 1.09945524], dtype=f32)  # spectrum.hxx:450
WAVELENGTHS = np.arange(390, 831, dtype=f32)


def luminance(rgb):
    rgb = np.asarray(rgb, dtype=f32)
    return f32(f32(f32(rgb[0] * f32(0.212671)) + f32(rgb[1] * f32(0.715160))) + f32(rgb[2] * f32(0.072169)))  # math.hxx:729


def _spd(power441, integrated):
    s = np.zeros(1, dtype=S.SPECTRUM)
    s["entries"]["wavelength"][0] = WAVELENGTHS
    s["entries"]["power"][0] = np.asarray(power441, dtype=f32)
    s["entry_count"] = 441
    s["integrated"][0] = np.asarray(integrated, dtype=f32)
    return s


def spd_constant(value):
    """SpectralDistribution::constant (render/host/spectrum.cxx:108-116)."""
    return _spd(np.full(441, value, dtype=f32), [value, value, value])


def spd_rgb_reflectance(rgb):
    """SpectralDistribution::rgb_reflectance (spectrum.cxx:135-148) via rgb_response (spectrum.cxx:399-)."""
    rgb = np.asarray(rgb, dtype=f32)
    if luminance(rgb) == 0.0:
        return spd_constant(0.0)
    w = tables("color_tables")["rgb_response_391x3"].astype(f32)
    p = (rgb[0] * w[:, 0]).astype(f32)
    p = (p + (rgb[1] * w[:, 1]).astype(f32)).astype(f32)
    p = (p + (rgb[2] * w[:, 2]).astype(f32)).astype(f32)
    power = np.concatenate([p, np.full(441 - 391, p[-1], dtype=f32)])  # from_samples clamps beyond the last sample
    return _spd(power, rgb)


def spd_rgb_luminance(rgb):
    """SpectralDistribution::rgb_luminance (spectrum.cxx:150-154)."""
    rgb = np.asarray(rgb, dtype=f32)
    s = spd_rgb_reflectance((rgb * K_RGB_LUMINANCE_SCALE).astype(f32))
    s["integrated"][0] = rgb
    return s


def spd_named_ior(name):
    t = tables("spectra")
    eta = _spd(t[f"{name}.eta_power"], t[f"{name}.eta_rgb"])
    k = _spd(t[f"{name}.k_power"], t[f"{name}.k_rgb"])
    return eta, k, int(t[f"{name}.cls"][0])


def spd_named_emission(name):
    t = tables("spectra")
    return _spd(t[f"{name}.power"], t[f"{name}.rgb"])


class SceneData:
    """Owns every array a Scene POD points to."""

    def __init__(self):
        self.vertices = []
        self.triangles = []
        self.materials = []
        self.spectra = []
        self.material_names = {}
        self.scene = np.zeros(1, dtype=S.SCENE)
        self.camera = np.zeros(1, dtype=S.CAMERA)
        self.name = ""
        self._keep = []

    # -- spectra / materials ---------------------------------------------------------------------
    def add_spectrum(self, spd):
        self.spectra.append(spd)
        return len(self.spectra) - 1

    def add_material(self, name, cls=S.MAT_DIFFUSE, kd=None, ks=None, roughness=0.0, emission=None, two_sided=0, int_ior=None,
                     thinfilm=None, collimation=0.0, int_medium=S.INVALID, ext_medium=S.INVALID, diffuse_variation=0, metalness=0.0, transmission=0.0,
                     subsurface=None):
        m = np.zeros(1, dtype=S.MATERIAL)
        for fld in ("reflectance", "scattering", "emission"):
            m[fld]["spectrum_index"] = S.INVALID
            m[fld]["image_index"] = S.INVALID
        for fld in ("roughness", "metalness", "transmission"):
            m[fld]["image_index"] = S.INVALID
            m[fld]["channel"] = S.INVALID
        m["subsurface"]["spectrum_index"] = S.INVALID
        m["subsurface"]["image_index"] = S.INVALID
        m["thinfilm"]["ior"]["eta_index"] = S.INVALID
        m["thinfilm"]["ior"]["k_index"] = S.INVALID
        m["thinfilm"]["thickness_image"] = S.INVALID
        for fld in ("ext_ior", "int_ior"):
            m[fld]["eta_index"] = S.INVALID
            m[fld]["k_index"] = S.INVALID
        m["cls"] = cls
        m["int_medium"] = int_medium
        m["ext_medium"] = ext_medium
        m["normal_image_index"] = S.INVALID
        m["diffuse_variation"] = diffuse_variation
        m["two_sided"] = two_sided
        m["normal_scale"] = 1.0
        m["opacity"] = 1.0
        m["emission_collimation"] = collimation
        if kd is not None:
            m["scattering"]["spectrum_index"] = self.add_spectrum(spd_rgb_reflectance(kd))
        if ks is not None:
            m["reflectance"]["spectrum_index"] = self.add_spectrum(spd_rgb_reflectance(ks))
        # "Pr u" or "Pr u v", each axis squared by the loader (scene_representation.cxx:1731-1738); a scalar sets both axes
        ru, rv = (roughness, roughness) if np.isscalar(roughness) else roughness
        m["roughness"]["value"][0][:2] = (f32(ru) * f32(ru), f32(rv) * f32(rv))
        m["metalness"]["value"][0][:] = metalness
        m["transmission"]["value"][0][:] = transmission
        if emission is not None:
            m["emission"]["spectrum_index"] = self.add_spectrum(emission)
        if int_ior is not None:
            eta, k, cls_ior = spd_named_ior(int_ior)
            m["int_ior"]["cls"] = cls_ior
            m["int_ior"]["eta_index"] = self.add_spectrum(eta)
            m["int_ior"]["k_index"] = self.add_spectrum(k)
        if thinfilm is not None:
            name_ior, tmin, tmax = thinfilm
            eta, k, cls_ior = spd_named_ior(name_ior)
            m["thinfilm"]["ior"]["cls"] = cls_ior
            m["thinfilm"]["ior"]["eta_index"] = self.add_spectrum(eta)
            m["thinfilm"]["ior"]["k_index"] = self.add_spectrum(k)
            m["thinfilm"]["min_thickness"] = tmin
            m["thinfilm"]["max_thickness"] = tmax
        if subsurface is not None:
            # "subsurface [refracted|diffuse-path] [burley] distances r g b scale s" (scene_representation.cxx:1972-2007)
            m["subsurface"]["cls"] = {"random_walk": 1, "burley": 2}[subsurface.get("cls", "random_walk")]
            m["subsurface"]["path"] = {"diffuse": 0, "refracted": 1}[subsurface.get("path", "diffuse")]
            spd = spd_rgb_reflectance(subsurface.get("distances", [1.0, 0.2, 0.04]))
            scale = f32(subsurface.get("scale", 1.0))
            spd["entries"]["power"][0] = (spd["entries"]["power"][0] * scale).astype(f32)
            spd["integrated"][0] = (spd["integrated"][0] * scale).astype(f32)
            m["subsurface"]["spectrum_index"] = self.add_spectrum(spd)
            # an image index scales the distances per texel (apply_image of the SubsurfaceMaterial)
            m["subsurface"]["image_index"] = subsurface.get("image", S.INVALID)
        self.materials.append(m)
        self.material_names[name] = len(self.materials) - 1
        return len(self.materials) - 1

    # -- images / distant emitters ------------------------------------------------------------------
    def add_image(self, pixels, repeat=True, build_table=False, uniform_table=False, offset=(0.0, 0.0), scale=(1.0, 1.0), has_alpha=None, repeat_v=None):
        """ImagePool::add_from_data + build_image_sampling_table (render/host/image_pool.cxx:226-259), RGBA32F."""
        u8 = np.asarray(pixels).dtype == np.uint8  # Image::Format::RGBA8 (8-bit files stay 8-bit, image_pool.cxx:188-205); float pixels: RGBA32F
        store = np.ascontiguousarray(pixels, dtype=np.uint8) if u8 else None
        px = (store.astype(f32) / f32(255.0)).astype(f32) if u8 else np.ascontiguousarray(pixels, dtype=f32)  # to_float4(ubyte4) (math.hxx:709-711)
        h, w = px.shape[:2]
        assert px.shape[2] == 4
        img = np.zeros(1, dtype=S.IMAGE)
        repeat_v = repeat if repeat_v is None else repeat_v  # Image::RepeatU / RepeatV are separate bits (an environment map wraps in u only)
        opts = (2 if repeat else 0) | (4 if repeat_v else 0) | (1 if build_table else 0) | (32 if uniform_table else 0)
        if has_alpha is None:
            has_alpha = bool((px[..., 3] < 1.0).any())
        if has_alpha:
            opts |= 16
        img["pixels"]["a"] = store.ctypes.data if u8 else px.ctypes.data
        img["pixels"]["count"] = w * h
        img["fsize"][0] = (w, h)
        img["isize"][0] = (w, h)
        img["offset"][0] = offset
        img["scale"][0] = scale
        img["options"] = opts
        img["format"] = 2 if u8 else 1
        img["data_size"] = store.nbytes if u8 else px.nbytes
        keep = [px, store]
        table = None
        if build_table:
            # Image::read at texel centres = mean of the 2x2 neighbourhood (image.hxx:173-186)
            xs1 = (np.arange(w) + 1) % w if repeat else np.minimum(np.arange(w) + 1, w - 1)
            ys1 = (np.arange(h) + 1) % h if repeat_v else np.minimum(np.arange(h) + 1, h - 1)
            rgb = px[..., :3]
            avg = (rgb * f32(0.25) + rgb[:, xs1] * f32(0.25) + rgb[ys1] * f32(0.25) + rgb[ys1][:, xs1] * f32(0.25)).astype(f32)
            lum = (avg[..., 0] * f32(0.212671) + avg[..., 1] * f32(0.715160) + avg[..., 2] * f32(0.072169)).astype(f32)

            def build(values):
                n = values.shape[0]
                e = np.zeros(n + 1, dtype=S.DIST_ENTRY)
                e["value"][:n] = values
                c = np.concatenate([[0.0], np.cumsum(values.astype(np.float64))]).astype(f32)
                total = f32(c[n])
                if total == 0:
                    e["value"][:n] = 1.0
                    e["pdf"][:n] = f32(1.0 / n)
                    e["cdf"][:n] = (np.arange(n) / n).astype(f32)
                else:
                    e["pdf"][:n] = (values / total).astype(f32)
                    e["cdf"][:n] = (c[:n] / total).astype(f32)
                e["cdf"][n] = 1.0
                return e, total

            rows = np.zeros(h, dtype=S.DISTRIBUTION)
            row_values = np.zeros(h, dtype=f32)
            for y in range(h):
                e, total = build(lum[y])
                keep.append(e)
                rows["values"]["a"][y] = e.ctypes.data
                rows["values"]["count"][y] = w + 1
                rows["total_weight"][y] = total
                v = (y + 0.5) / h
                row_values[y] = f32(lum[y].astype(np.float64).sum()) * f32(1.0 if uniform_table else math.sin(v * math.pi))
            ey, total_y = build(row_values)
            keep += [rows, ey]
            table = (np.stack(keep[2:2 + h]), ey)
            img["x_distributions"]["a"] = rows.ctypes.data
            img["x_distributions"]["count"] = h
            img["y_distribution"]["values"]["a"] = ey.ctypes.data
            img["y_distribution"]["values"]["count"] = h + 1
            img["y_distribution"]["total_weight"] = total_y
            img["normalization"] = f32(row_values.astype(np.float64).sum()) / f32(w * h)
        self._keep.append(keep)
        if not hasattr(self, "_images"):
            self._images = []
        if not hasattr(self, "_image_px"):
            self._image_px = {}
        self._images.append(img)
        self._image_px[len(self._images) - 1] = px  # the pixels as Image::pixel() returns them (float4)
        if not hasattr(self, "_image_tables"):
            self._image_tables = {}
        self._image_tables[len(self._images) - 1] = table  # (h, w + 1) row entries and the h + 1 row-selection entries, or None
        return len(self._images) - 1

    def image_evaluate(self, index, uv):
        """Image::evaluate(uv, nullptr) (render/shared/image.hxx:51-88): bilinear gather with the image's repeat / clamp flags; uv = (N, 2) float32."""
        rec, px = self._images[index], self._image_px[index]
        w, h = int(rec["isize"][0][0]), int(rec["isize"][0][1])
        fw, fh = f32(w), f32(h)
        opts = int(rec["options"][0])

        def coord(t, size, rep):
            if rep:
                x = np.fmod(t, size).astype(f32)
                return np.where(x < 0, (x + size).astype(f32), x).astype(f32)
            return np.clip(t, f32(0.0), np.nextafter(size, f32(0.0), dtype=f32)).astype(f32)
        x0 = coord((uv[:, 0] * fw).astype(f32), fw, bool(opts & 2))
        y0 = coord((uv[:, 1] * fh).astype(f32), fh, bool(opts & 4))
        dx, dy = (x0 - np.floor(x0)).astype(f32), (y0 - np.floor(y0)).astype(f32)
        r0 = np.clip(y0.astype(np.uint32), 0, h - 1)
        r1 = np.clip(r0 + 1, 0, h - 1)
        c0 = np.clip(x0.astype(np.uint32), 0, w - 1)
        c1 = np.clip(c0 + 1, 0, w - 1)
        one = f32(1.0)
        p00 = ((px[r0, c0] * (one - dx)[:, None]).astype(f32) * (one - dy)[:, None]).astype(f32)
        p01 = ((px[r0, c1] * dx[:, None]).astype(f32) * (one - dy)[:, None]).astype(f32)
        p10 = ((px[r1, c0] * (one - dx)[:, None]).astype(f32) * dy[:, None]).astype(f32)
        p11 = ((px[r1, c1] * dx[:, None]).astype(f32) * dy[:, None]).astype(f32)
        return (((p00 + p01).astype(f32) + p10).astype(f32) + p11).astype(f32)

    def _texture_emission(self, image_index, tex):
        """The emission-image factor of an area emitter's weight (add_area_emitters_for_triangle, scene_representation.cxx:855-872): 1 + the image's
        luminance x alpha averaged over a barycentric grid of the triangle (the inner loop of the reference steps by dv, kept)."""
        rec = self._images[image_index]
        fs = rec["fsize"][0]
        mn, mx = tex.min(axis=0), tex.max(axis=0)
        u_size = f32(4.0) * max(f32(1.0), f32(np.ceil(f32(f32(mx[0] - mn[0]) * fs[0]))))
        v_size = f32(4.0) * max(f32(1.0), f32(np.ceil(f32(f32(mx[1] - mn[1]) * fs[1]))))
        du, dv = f32(1.0) / u_size, f32(1.0) / v_size
        steps, t = [], f32(0.0)
        while t < f32(1.0):
            steps.append(t)
            t = f32(t + dv)
        g = np.array(steps, dtype=f32)
        v, u = np.repeat(g, len(g)), np.tile(g, len(g))
        r1 = np.sqrt(u).astype(f32)
        bc = np.stack([(f32(1.0) - r1).astype(f32), (r1 * (f32(1.0) - v).astype(f32)).astype(f32), (r1 * v).astype(f32)], 1)
        uv = ((tex[0][None, :] * bc[:, 0:1]).astype(f32) + (tex[1][None, :] * bc[:, 1:2]).astype(f32)).astype(f32)
        uv = (uv + (tex[2][None, :] * bc[:, 2:3]).astype(f32)).astype(f32)
        val = self.image_evaluate(image_index, uv)
        lum = ((val[:, 0] * f32(0.212671)).astype(f32) + (val[:, 1] * f32(0.715160)).astype(f32)).astype(f32) + (val[:, 2] * f32(0.072169)).astype(f32)
        terms = (((lum.astype(f32) * du).astype(f32) * dv).astype(f32) * val[:, 3]).astype(f32)
        return f32(np.cumsum(np.concatenate([[f32(1.0)], terms]).astype(f32), dtype=f32)[-1])

    def add_environment_emitter(self, image_index, rgb=(1.0, 1.0, 1.0)):
        """et::env with an image (scene_representation.cxx: environment profile + one instance)."""
        p = np.zeros(1, dtype=S.EMITTER_PROFILE)
        p["emission"]["spectrum_index"] = self.add_spectrum(spd_rgb_luminance(rgb))
        p["emission"]["image_index"] = image_index
        p["cls"] = S.EMITTER_ENVIRONMENT
        p["angular_size_cosine"] = 1.0
        e = np.zeros(1, dtype=S.EMITTER)
        e["cls"] = S.EMITTER_ENVIRONMENT
        e["triangle_index"] = S.INVALID
        if not hasattr(self, "_distant_emitters"):
            self._distant_emitters = []
        self._distant_emitters.append((p, e))

    def add_directional_emitter(self, direction, rgb, angular_size_deg=0.0, image_index=S.INVALID):
        """et::dir (finite angular size allowed, optionally an image over its disk); equivalent_disk_size / angular_size_cosine as
        build_emitters_distribution (:2463-2466)."""
        d = np.asarray(direction, dtype=f32)
        d = (d / f32(math.sqrt(float(np.dot(d, d))))).astype(f32)
        ang = f32(math.radians(angular_size_deg))
        p = np.zeros(1, dtype=S.EMITTER_PROFILE)
        p["emission"]["spectrum_index"] = self.add_spectrum(spd_rgb_luminance(rgb))
        p["emission"]["image_index"] = image_index
        p["direction"][0] = d
        p["cls"] = S.EMITTER_DIRECTIONAL
        p["angular_size"] = ang
        p["equivalent_disk_size"] = f32(2.0 * math.tan(float(ang) / 2.0))
        p["angular_size_cosine"] = f32(math.cos(float(ang) / 2.0))
        e = np.zeros(1, dtype=S.EMITTER)
        e["cls"] = S.EMITTER_DIRECTIONAL
        e["triangle_index"] = S.INVALID
        if not hasattr(self, "_distant_emitters"):
            self._distant_emitters = []
        self._distant_emitters.append((p, e))

    def add_medium(self, absorption=(0.0, 0.0, 0.0), scattering=(0.8, 0.8, 0.8), g=0.0, explicit_connections=True, density=None, bounds=None, max_sigma=None):
        """MediumPool::add (render/host/medium_pool.cxx:23-60): homogeneous, or heterogeneous with a dense grid normalised to max 1."""
        m = np.zeros(1, dtype=S.MEDIUM)
        m["absorption_index"] = self.add_spectrum(spd_rgb_reflectance(absorption))
        m["scattering_index"] = self.add_spectrum(spd_rgb_reflectance(scattering))
        m["phase_function_g"] = g
        m["enable_explicit_connections"] = 1 if explicit_connections else 0
        ext = np.asarray(absorption, dtype=f32) + np.asarray(scattering, dtype=f32)
        m["max_sigma"] = f32(max_sigma if max_sigma is not None else float(ext.max()))
        if density is not None:
            d = np.ascontiguousarray(density, dtype=f32)
            d = (d / max(float(d.max()), 1e-20)).astype(f32)
            m["cls"] = 1
            m["density"]["a"] = d.ctypes.data
            m["density"]["count"] = d.size
            m["dimensions"][0] = (d.shape[2], d.shape[1], d.shape[0])  # x fastest
            lo, hi = bounds
            m["bounds_min"][0] = lo
            m["bounds_max"][0] = hi
            self._keep.append(d)
        if not hasattr(self, "_mediums"):
            self._mediums = []
        self._mediums.append(m)
        return len(self._mediums) - 1

    # -- geometry --------------------------------------------------------------------------------
    def add_mesh(self, positions, normals, indices, material_index, uvs=None):
        positions = np.asarray(positions, dtype=f32).reshape(-1, 3)
        normals = np.asarray(normals, dtype=f32).reshape(-1, 3)
        indices = np.asarray(indices, dtype=np.uint32).reshape(-1, 3)
        n = positions.shape[0]
        v = np.zeros(n, dtype=S.VERTEX)
        v["pos"] = positions
        nl = np.linalg.norm(normals, axis=1, keepdims=True).astype(f32)
        nrm = (normals / np.maximum(nl, f32(1e-20))).astype(f32)
        v["nrm"] = nrm
        # tangent frame: any vector orthogonal to the normal (the loader runs MikkTSpace; a fixed rule is enough here)
        helper = np.where(np.abs(nrm[:, 1:2]) < 0.9, np.array([[0, 1, 0]], dtype=f32), np.array([[1, 0, 0]], dtype=f32))
        tan = np.cross(helper, nrm).astype(f32)
        tan = (tan / np.linalg.norm(tan, axis=1, keepdims=True)).astype(f32)
        btn = np.cross(nrm, tan).astype(f32)
        btn = (btn / np.linalg.norm(btn, axis=1, keepdims=True)).astype(f32)
        v["tan"] = tan
        v["btn"] = btn
        if uvs is not None:
            v["tex"] = np.asarray(uvs, dtype=f32).reshape(-1, 2)
        base = sum(a.shape[0] for a in self.vertices)
        t = np.zeros(indices.shape[0], dtype=S.TRIANGLE)
        t["i"] = indices + np.uint32(base)
        t["material_index"] = material_index
        p0, p1, p2 = positions[indices[:, 0]], positions[indices[:, 1]], positions[indices[:, 2]]
        gn = np.cross(p1 - p0, p2 - p0).astype(f32)
        gl = np.linalg.norm(gn, axis=1, keepdims=True).astype(f32)
        t["geo_n"] = (gn / np.maximum(gl, f32(1e-30))).astype(f32)
        self.vertices.append(v)
        self.triangles.append(t)

    def add_quad(self, p0, p1, p2, p3, material_index, subdiv=1):
        """Quad p0,p1,p2,p3 (counter-clockwise seen from the side the normal points to), optionally tessellated."""
        p0, p1, p2, p3 = [np.asarray(p, dtype=np.float64) for p in (p0, p1, p2, p3)]
        n = np.cross(p1 - p0, p3 - p0)
        n = n / np.linalg.norm(n)
        s = subdiv
        us, vs = np.meshgrid(np.linspace(0, 1, s + 1), np.linspace(0, 1, s + 1), indexing="xy")
        us, vs = us.reshape(-1, 1), vs.reshape(-1, 1)
        pos = (1 - us) * (1 - vs) * p0 + us * (1 - vs) * p1 + us * vs * p2 + (1 - us) * vs * p3
        idx = []
        for j in range(s):
            for i in range(s):
                a = j * (s + 1) + i
                b, c, d = a + 1, a + s + 2, a + s + 1
                idx.append((a, b, c))
                idx.append((a, c, d))
        self.add_mesh(pos, np.tile(n, (pos.shape[0], 1)), np.array(idx), material_index, uvs=np.hstack([us, vs]))

    def add_box(self, center, half, yaw_deg, material_index, subdiv=1):
        c = np.asarray(center, dtype=np.float64)
        hx, hy, hz = half
        a = math.radians(yaw_deg)
        rot = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])

        def P(x, y, z):
            return c + rot @ np.array([x * hx, y * hy, z * hz])

        self.add_quad(P(-1, 1, 1), P(1, 1, 1), P(1, 1, -1), P(-1, 1, -1), material_index, subdiv)      # top
        self.add_quad(P(-1, -1, -1), P(1, -1, -1), P(1, -1, 1), P(-1, -1, 1), material_index, subdiv)  # bottom
        self.add_quad(P(-1, -1, 1), P(1, -1, 1), P(1, 1, 1), P(-1, 1, 1), material_index, subdiv)      # +z
        self.add_quad(P(1, -1, -1), P(-1, -1, -1), P(-1, 1, -1), P(1, 1, -1), material_index, subdiv)  # -z
        self.add_quad(P(1, -1, 1), P(1, -1, -1), P(1, 1, -1), P(1, 1, 1), material_index, subdiv)      # +x
        self.add_quad(P(-1, -1, -1), P(-1, -1, 1), P(-1, 1, 1), P(-1, 1, -1), material_index, subdiv)  # -x

    def add_uv_sphere(self, center, radius, segments, rings, material_index, displace=None):
        """UV sphere with 2*segments*(rings-1) triangles, smooth normals."""
        c = np.asarray(center, dtype=np.float64)
        pos, nrm, uv = [], [], []
        for r in range(rings + 1):
            theta = math.pi * r / rings
            for s in range(segments + 1):
                phi = 2.0 * math.pi * s / segments
                d = np.array([math.sin(theta) * math.cos(phi), math.cos(theta), math.sin(theta) * math.sin(phi)])
                rr = radius if displace is None else radius * displace(d)
                pos.append(c + rr * d)
                nrm.append(d)
                uv.append((s / segments, r / rings))
        idx = []
        for r in range(rings):
            for s in range(segments):
                a = r * (segments + 1) + s
                b = a + 1
                d = a + segments + 1
                e = d + 1
                if r != 0:
                    idx.append((a, b, d))  # outward-facing winding (counter-clockwise from outside)
                if r != rings - 1:
                    idx.append((b, e, d))
        self.add_mesh(np.array(pos), np.array(nrm), np.array(idx), material_index, uvs=np.array(uv))

    # -- finalisation ----------------------------------------------------------------------------
    def set_camera(self, origin, target, up, width, height, fov_deg, clip_near=1.0 / 256.0, clip_far=1024.0, lens_radius=0.0, focal_distance=0.0, f32_trig=False):
        """build_camera (scene_representation.cxx:579-598) with float32 arithmetic."""
        cam = self.camera
        cam[:] = 0
        cam["clip_near"] = clip_near
        cam["clip_far"] = clip_far
        cam["lens_image"] = S.INVALID
        cam["medium_index"] = S.INVALID
        cam["lens_radius"] = lens_radius
        cam["focal_distance"] = focal_distance
        o, t, u = [np.asarray(x, dtype=f32) for x in (origin, target, up)]

        def nz(v):
            return (v / f32(math.sqrt(float(np.dot(v, v))))).astype(f32)

        f = nz(t - o)
        s = nz(np.cross(f, u).astype(f32))
        uu = np.cross(s, f).astype(f32)
        view = np.zeros((4, 4), dtype=f32)  # view[col][row]
        view[0][0], view[1][0], view[2][0] = s
        view[0][1], view[1][1], view[2][1] = uu
        view[0][2], view[1][2], view[2][2] = -f
        view[3][0] = -np.dot(s, o)
        view[3][1] = -np.dot(uu, o)
        view[3][2] = np.dot(f, o)
        view[3][3] = 1.0
        fov = f32(fov_deg) * f32(math.pi) / f32(180.0)
        if f32_trig:  # perspective() divides cosf by sinf (vector_math.hxx:118): the scene-file loader follows it to the bit
            half = f32(f32(0.5) * fov)
            w = f32(np.cos(half, dtype=f32) / np.sin(half, dtype=f32))
        else:        # the generators' cameras (and the golden renders made with them) use the double-precision quotient
            w = f32(math.cos(0.5 * float(fov)) / math.sin(0.5 * float(fov)))
        aspect = f32(width) / f32(height)
        zn, zf = f32(clip_near), f32(clip_far)
        proj = np.zeros((4, 4), dtype=f32)
        proj[0][0] = w
        proj[1][1] = w * aspect
        proj[2][2] = zf / (zn - zf)
        proj[2][3] = -1.0
        proj[3][2] = -(zf * zn) / (zf - zn)
        # column-major product proj * view: result.col[j] = sum_k proj.col[k] * view.col[j][k]
        vp = np.zeros((4, 4), dtype=f32)
        for j in range(4):
            acc = np.zeros(4, dtype=f32)
            for k in range(4):
                acc = (acc + proj[k] * view[j][k]).astype(f32)
            vp[j] = acc
        cam["view_proj"][0] = vp.reshape(-1)
        cam["target"][0] = t
        cam["position"][0] = o  # inverse(view).col[3] == origin
        cam["side"][0] = s
        cam["up"][0] = uu
        cam["direction"][0] = f
        cam["tan_half_fov"] = f32(1.0) / abs(w)
        cam["aspect"] = proj[1][1] / proj[0][0]
        thf = cam["tan_half_fov"][0]
        cam["area"] = (f32(2.0) * thf) * (f32(2.0) * thf / cam["aspect"][0])
        cam["film_size"][0] = (width, height)
        cam["image_plane"] = f32(width) / (f32(2.0) * thf)

    def finalize(self, samples, spectral, max_path_length=1023, min_path_length=0, random_path_termination=6):
        """validate_materials + commit + rebuild_area_emitters + build_emitters_distribution."""
        sc = self.scene
        sc[:] = 0
        white = self.add_spectrum(spd_rgb_reflectance([1.0, 1.0, 1.0]))
        black = self.add_spectrum(spd_constant(0.0))
        one = self.add_spectrum(spd_constant(1.0))
        sss = self.add_spectrum(spd_rgb_reflectance([1.0, 0.2, 0.04]))
        glass_eta, glass_k, _ = spd_named_ior("glass")
        def_diel = self.add_spectrum(glass_eta)
        gold_eta, gold_k, _ = spd_named_ior("gold")
        def_cond_eta, def_cond_k = self.add_spectrum(gold_eta), self.add_spectrum(gold_k)
        ss_scatter = ss_exit = S.INVALID
        if any(int(m["subsurface"]["cls"][0]) != 0 for m in self.materials):
            # init_default_values (scene_representation.cxx:216-224)
            ss_scatter = self.add_material("etx::subsurface-scatter", cls=S.MAT_TRANSLUCENT)
            self.materials[ss_scatter]["reflectance"]["spectrum_index"] = black
            self.materials[ss_scatter]["scattering"]["spectrum_index"] = white
            ss_exit = self.add_material("etx::subsurface-exit", cls=S.MAT_DIFFUSE)
            self.materials[ss_exit]["reflectance"]["spectrum_index"] = white
            self.materials[ss_exit]["scattering"]["spectrum_index"] = white
        for m in self.materials:
            if m["reflectance"]["spectrum_index"][0] == S.INVALID:
                m["reflectance"]["spectrum_index"] = white
            if m["scattering"]["spectrum_index"][0] == S.INVALID:
                m["scattering"]["spectrum_index"] = white
            if m["subsurface"]["spectrum_index"][0] == S.INVALID:
                m["subsurface"]["spectrum_index"] = sss
            if m["emission"]["spectrum_index"][0] == S.INVALID:
                m["emission"]["spectrum_index"] = black
            r = m["roughness"]["value"][0]
            if r[0] > 0 or r[1] > 0:
                r[0] = max(f32(1e-6), r[0])
                r[1] = max(f32(1e-6), r[1])
            if m["int_ior"]["eta_index"][0] == S.INVALID:
                m["int_ior"]["eta_index"] = def_cond_eta if m["cls"][0] == S.MAT_CONDUCTOR else def_diel
            if m["int_ior"]["k_index"][0] == S.INVALID:
                m["int_ior"]["k_index"] = def_cond_k if m["cls"][0] == S.MAT_CONDUCTOR else black
            if m["thinfilm"]["ior"]["k_index"][0] == S.INVALID:
                m["thinfilm"]["ior"]["k_index"] = black
            if m["thinfilm"]["ior"]["eta_index"][0] == S.INVALID:
                m["thinfilm"]["ior"]["eta_index"] = one

        self.finalize_arrays(samples, spectral, max_path_length, min_path_length, random_path_termination)
        sc["black_spectrum"] = black
        sc["white_spectrum"] = white
        for fld in ("rayleigh_spectrum", "mie_spectrum", "ozone_spectrum"):
            sc[fld] = S.INVALID
        sc["subsurface_scatter_material"] = ss_scatter
        sc["subsurface_exit_material"] = ss_exit
        sc["default_dielectric_eta"] = def_diel
        sc["default_conductor_eta"] = def_cond_eta
        sc["default_conductor_k"] = def_cond_k
        return self

    def finalize_arrays(self, samples, spectral, max_path_length=1023, min_path_length=0, random_path_termination=6, distant_first=False):
        """commit (scene_representation.cxx:420-455) + rebuild_area_emitters + build_emitters_distribution on validated materials: the flat arrays and
        the Scene record (the default-spectrum / subsurface-material indices are the caller's)."""
        sc = self.scene
        self.a_vertices = np.concatenate(self.vertices) if self.vertices else np.zeros(0, S.VERTEX)
        self.a_triangles = np.concatenate(self.triangles) if self.triangles else np.zeros(0, S.TRIANGLE)
        self.a_materials = np.concatenate(self.materials)
        self.a_spectra = np.concatenate(self.spectra)
        nt = self.a_triangles.shape[0]

        # bounding sphere (commit():431-444)
        tri_pos = self.a_vertices["pos"][self.a_triangles["i"].reshape(-1)]
        bmin, bmax = tri_pos.min(axis=0).astype(f32), tri_pos.max(axis=0).astype(f32)
        center = (f32(0.5) * (bmin + bmax)).astype(f32)
        d = (bmax - center).astype(f32)
        radius = f32(math.sqrt(float(f32(f32(f32(d[0] * d[0]) + f32(d[1] * d[1])) + f32(d[2] * d[2])))))

        # area emitters (add_area_emitters_for_triangle:840-903)
        tri_to_emitter = np.full(nt, S.INVALID, dtype=np.uint32)
        profiles, instances, mat_to_profile = [], [], {}
        lum = {}

        def add_distant():
            for (p, e) in getattr(self, "_distant_emitters", []):
                e = e.copy()
                e["cls"] = p["cls"]
                e["profile"] = len(profiles)
                e["additional_weight"] = f32(math.pi) * radius * radius
                e["spectrum_weight"] = luminance(self.a_spectra["integrated"][int(p["emission"]["spectrum_index"][0])])
                profiles.append(p)
                instances.append(e)
        if distant_first:  # a scene FILE declares its et::env / et::dir emitters before commit() instances the area emitters (scene_representation.cxx:1308-1378, 956)
            add_distant()
        for ti in range(nt):
            mi = int(self.a_triangles["material_index"][ti])
            m = self.a_materials[mi]
            si = int(m["emission"]["spectrum_index"])
            if si not in lum:
                lum[si] = luminance(self.a_spectra["integrated"][si])
            if lum[si] <= 0.0:
                continue
            i0, i1, i2 = self.a_triangles["i"][ti]
            p0, p1, p2 = self.a_vertices["pos"][i0], self.a_vertices["pos"][i1], self.a_vertices["pos"][i2]
            cr = np.cross((p1 - p0).astype(f32), (p2 - p0).astype(f32)).astype(f32)
            area = f32(0.5) * f32(math.sqrt(float(np.dot(cr, cr))))
            tex_em = f32(1.0)
            if int(m["emission"]["image_index"]) != S.INVALID:
                tex_em = self._texture_emission(int(m["emission"]["image_index"]), self.a_vertices["tex"][[i0, i1, i2]])
            add_w = f32((2.0 if m["two_sided"] else 1.0)) * f32(area * f32(math.pi)) * tex_em
            if mi not in mat_to_profile:
                p = np.zeros(1, dtype=S.EMITTER_PROFILE)
                p["emission"] = m["emission"]
                p["cls"] = S.EMITTER_AREA
                p["angular_size_cosine"] = 1.0
                mat_to_profile[mi] = len(profiles)
                profiles.append(p)
            e = np.zeros(1, dtype=S.EMITTER)
            e["cls"] = S.EMITTER_AREA
            e["profile"] = mat_to_profile[mi]
            e["triangle_index"] = ti
            e["triangle_area"] = area
            e["additional_weight"] = add_w
            e["spectrum_weight"] = lum[si]
            tri_to_emitter[ti] = len(instances)
            instances.append(e)
        if not distant_first:
            add_distant()
        assert instances, "scene needs at least one emitter (the loader would synthesise an atmosphere otherwise)"
        self.a_profiles = np.concatenate(profiles)
        self.a_emitters = np.concatenate(instances)
        self.a_tri_to_emitter = tri_to_emitter

        # emitter distribution (DistributionBuilder::finalize, distribution_builder.hxx:30-58)
        ne = self.a_emitters.shape[0]
        dist = np.zeros(ne + 1, dtype=S.DIST_ENTRY)
        total = f32(0.0)
        env = []
        for i in range(ne):
            w = f32(self.a_emitters["spectrum_weight"][i] * self.a_emitters["additional_weight"][i])
            dist["value"][i] = w
            dist["cdf"][i] = total
            total = f32(total + w)
            if self.a_emitters["cls"][i] != S.EMITTER_AREA and w > 0:
                env.append(i)
        dist["pdf"][:ne] = (dist["value"][:ne] / total).astype(f32)
        dist["cdf"][:ne] = (dist["cdf"][:ne] / total).astype(f32)
        dist["cdf"][ne] = 1.0
        self.a_dist = dist

        def view(field, arr):
            sc[field]["a"] = arr.ctypes.data if arr.size else 0
            sc[field]["count"] = arr.shape[0]

        view("vertices", self.a_vertices)
        view("triangles", self.a_triangles)
        view("triangle_to_emitter", self.a_tri_to_emitter)
        view("materials", self.a_materials)
        view("emitter_profiles", self.a_profiles)
        view("emitter_instances", self.a_emitters)
        self.a_images = np.concatenate(self._images) if getattr(self, "_images", None) else np.zeros(0, dtype=S.IMAGE)
        self.a_mediums = np.concatenate(self._mediums) if getattr(self, "_mediums", None) else np.zeros(0, dtype=S.MEDIUM)
        view("images", self.a_images)
        view("mediums", self.a_mediums)
        view("spectrums", self.a_spectra)
        sc["emitters_distribution"]["values"]["a"] = dist.ctypes.data
        sc["emitters_distribution"]["values"]["count"] = ne + 1
        sc["emitters_distribution"]["total_weight"] = total
        sc["environment_emitter_count"] = len(env)
        for k, i in enumerate(env):
            sc["environment_emitters"][0][k] = i
        sc["bounding_sphere_center"][0] = center
        sc["bounding_sphere_radius"] = radius
        sc["pixel_sampler_image"] = S.INVALID
        sc["pixel_sampler_radius"] = 1.5
        sc["min_path_length"] = min_path_length
        sc["max_path_length"] = max_path_length
        sc["samples"] = samples
        sc["random_path_termination"] = random_path_termination
        sc["noise_threshold"] = 0.1
        sc["radiance_clamp"] = 0.0
        sc["flags"] = S.SCENE_COMMITTED | (S.SCENE_SPECTRAL if spectral else 0)
        return self

    @property
    def width(self):
        return int(self.camera["film_size"][0][0])

    @property
    def height(self):
        return int(self.camera["film_size"][0][1])

    @property
    def triangle_count(self):
        return int(self.a_triangles.shape[0])


# ---------------------------------------------------------------------------------------------------
# BASELINE.json configs
# ---------------------------------------------------------------------------------------------------
def cornell_box(width=512, height=512, samples=16, spectral=False, sphere=False, sphere_segments=128, sphere_rings=81, wall_subdiv=1,
                sphere_roughness=0.0, max_path_length=1023, tall_box_material="diffuse", finalize=True):
    """C1 (sphere=False, spectral=False) / C2 (sphere=True, spectral=True): SURVEY.md §8(d).

    Closed box x,z in [-1,1], y in [0,2] (the reference asset's dimensions, bin/assets/cornellbox/cornellbox.json:9-34 camera),
    all-diffuse walls and two boxes, one `light` quad emitter (color 10.018 3.918 0.932, two-sided).
    """
    sd = SceneData()
    sd.name = "cornell" + ("+sphere" if sphere else "") + ("/spectral" if spectral else "/rgb")
    white = sd.add_material("white", kd=[1.0, 1.0, 1.0], two_sided=1)
    grey = sd.add_material("grey", kd=[0.906, 0.906, 0.906], two_sided=1)
    red = sd.add_material("leftWall", kd=[1.0, 0.0, 0.0], two_sided=1)
    green = sd.add_material("rightWall", kd=[0.0, 1.0, 0.0], two_sided=1)
    light = sd.add_material("light", kd=[0.0, 0.0, 0.0], emission=spd_rgb_luminance([10.018, 3.918, 0.932]), two_sided=1)
    s = wall_subdiv
    zf = 4.0  # the box is closed behind the camera (camera sits at z = 3.82)
    sd.add_quad([-1, 0, zf], [1, 0, zf], [1, 0, -1], [-1, 0, -1], white, s)    # floor (normal +y)
    sd.add_quad([-1, 2, -1], [1, 2, -1], [1, 2, zf], [-1, 2, zf], white, s)    # ceiling (normal -y)
    sd.add_quad([-1, 0, -1], [1, 0, -1], [1, 2, -1], [-1, 2, -1], grey, s)     # back wall (normal +z)
    sd.add_quad([-1, 0, zf], [-1, 0, -1], [-1, 2, -1], [-1, 2, zf], red, s)    # left wall (normal +x)
    sd.add_quad([1, 0, -1], [1, 0, zf], [1, 2, zf], [1, 2, -1], green, s)      # right wall (normal -x)
    sd.add_quad([-1, 0, zf], [-1, 2, zf], [1, 2, zf], [1, 0, zf], grey, s)     # wall behind the camera (normal -z)
    sd.add_quad([-0.24, 1.98, -0.22], [0.23, 1.98, -0.22], [0.23, 1.98, 0.16], [-0.24, 1.98, 0.16], light, 1)  # light (normal -y)
    if tall_box_material == "diffuse":
        tall = grey
    else:
        tall = sd.add_material("tallBox", cls=S.MAT_CONDUCTOR, ks=[1, 1, 1], int_ior="silver", two_sided=1)
    sd.add_box([-0.33, 0.6, -0.29], (0.3, 0.6, 0.3), 17.0, tall, s)
    if sphere:
        glass = sd.add_material("glass", cls=S.MAT_DIELECTRIC, roughness=sphere_roughness, int_ior="glass")
        sd.add_uv_sphere([0.33, 0.301, 0.35], 0.3, sphere_segments, sphere_rings, glass)
    else:
        sd.add_box([0.33, 0.3, 0.35], (0.3, 0.3, 0.3), -17.0, grey, s)
    sd.set_camera([0.0, 1.0, 3.82], [0.0, 1.0, -6.18], [0.0, 1.0, 0.0], width, height, 39.597755335771296, clip_near=0.1, clip_far=100.0)
    if not finalize:
        return sd  # the caller still changes the camera / adds images
    return sd.finalize(samples=samples, spectral=spectral, max_path_length=max_path_length)


MATERIAL_KINDS = {
    # name: add_material kwargs — one entry per Material::Class the device implements (material.hxx:53-68)
    "conductor_rough": dict(cls=S.MAT_CONDUCTOR, ks=[1.0, 1.0, 1.0], roughness=0.45, int_ior="gold"),
    "conductor_smooth": dict(cls=S.MAT_CONDUCTOR, ks=[0.9, 0.9, 0.9], roughness=0.0, int_ior="silver"),
    "conductor_thinfilm": dict(cls=S.MAT_CONDUCTOR, ks=[1.0, 1.0, 1.0], roughness=0.3, int_ior="copper", thinfilm=("water", 320.0, 320.0)),
    "plastic": dict(cls=S.MAT_PLASTIC, kd=[0.2, 0.4, 0.8], ks=[1.0, 1.0, 1.0], roughness=0.55, int_ior="plastic"),
    "plastic_thinfilm": dict(cls=S.MAT_PLASTIC, kd=[0.7, 0.7, 0.7], ks=[1.0, 1.0, 1.0], roughness=0.4, int_ior="plastic", thinfilm=("glass", 300.0, 700.0)),
    "dielectric_rough": dict(cls=S.MAT_DIELECTRIC, roughness=0.4, int_ior="glass"),
    "dielectric_smooth": dict(cls=S.MAT_DIELECTRIC, roughness=0.0, int_ior="diamond"),
    "thinfilm": dict(cls=S.MAT_THINFILM, kd=[0.9, 0.9, 0.9], ks=[1.0, 1.0, 1.0], int_ior="glass", thinfilm=("water", 250.0, 450.0)),
    "mirror": dict(cls=S.MAT_MIRROR, kd=[0.9, 0.9, 0.9]),
    "translucent": dict(cls=S.MAT_TRANSLUCENT, kd=[0.5, 0.5, 0.4], ks=[0.3, 0.4, 0.3]),
    "velvet": dict(cls=S.MAT_VELVET, kd=[0.6, 0.1, 0.1], ks=[0.5, 0.5, 0.5], roughness=0.7),
    "principled": dict(cls=S.MAT_PRINCIPLED, kd=[0.8, 0.5, 0.2], ks=[1.0, 1.0, 1.0], roughness=0.5, metalness=0.4, transmission=0.3),
    "void": dict(cls=S.MAT_VOID),
    "diffuse_rough": dict(kd=[0.8, 0.7, 0.5], roughness=0.6, diffuse_variation=1),  # Heitz rough diffuse: random walk in sample AND evaluate
    # vMF diffuse fit (diffuse_variation 2): the three branches of its cross section — m > 0.9, 0.25 <= m <= 0.9, m < 0.25 (m = -log(1 - Pr))
    "diffuse_vmf": dict(kd=[0.8, 0.7, 0.5], roughness=0.62, diffuse_variation=2),
    "diffuse_vmf_mid": dict(kd=[0.6, 0.7, 0.8], roughness=0.4, diffuse_variation=2),
    "diffuse_vmf_low": dict(kd=[0.8, 0.8, 0.8], roughness=0.15, diffuse_variation=2),
    # the diffuse variations as the base layer of PlasticBSDF::evaluate (bsdf_plastic.hxx:136)
    "plastic_rough_base": dict(cls=S.MAT_PLASTIC, kd=[0.3, 0.6, 0.4], ks=[1.0, 1.0, 1.0], roughness=0.5, int_ior="plastic", diffuse_variation=1),
    "plastic_vmf_base": dict(cls=S.MAT_PLASTIC, kd=[0.7, 0.4, 0.3], ks=[1.0, 1.0, 1.0], roughness=0.45, int_ior="plastic", diffuse_variation=2),
    # subsurface scattering on top of a diffuse-lobe class (material.hxx:36-51)
    "sss_random_walk": dict(kd=[0.8, 0.6, 0.4], subsurface=dict(cls="random_walk", path="diffuse", distances=[1.0, 0.4, 0.15], scale=0.12)),
    "sss_refracted": dict(cls=S.MAT_PLASTIC, kd=[0.7, 0.8, 0.6], ks=[1.0, 1.0, 1.0], roughness=0.3, int_ior="plastic",
                          subsurface=dict(cls="random_walk", path="refracted", distances=[0.3, 0.6, 1.0], scale=0.1)),
    "sss_burley": dict(kd=[0.9, 0.5, 0.4], subsurface=dict(cls="burley", distances=[1.0, 0.3, 0.1], scale=0.08)),
    # anisotropic roughness ("Pr u v"): the microsurface walk with alpha_x != alpha_y
    "conductor_aniso": dict(cls=S.MAT_CONDUCTOR, ks=[1.0, 1.0, 1.0], roughness=(0.15, 0.6), int_ior="gold"),
    "dielectric_aniso": dict(cls=S.MAT_DIELECTRIC, roughness=(0.5, 0.1), int_ior="glass"),
    "plastic_aniso": dict(cls=S.MAT_PLASTIC, kd=[0.3, 0.5, 0.7], ks=[1.0, 1.0, 1.0], roughness=(0.2, 0.65), int_ior="plastic"),
}


def material_box(kind, width=32, height=32, samples=16, spectral=False, sphere_segments=16, sphere_rings=9):
    """Cornell box whose tall box and a sphere carry one material class — the per-class parity scenes."""
    sd = SceneData()
    sd.name = f"material_box[{kind}]" + ("/spectral" if spectral else "/rgb")
    white = sd.add_material("white", kd=[1.0, 1.0, 1.0], two_sided=1)
    red = sd.add_material("leftWall", kd=[1.0, 0.0, 0.0], two_sided=1)
    green = sd.add_material("rightWall", kd=[0.0, 1.0, 0.0], two_sided=1)
    light = sd.add_material("light", kd=[0.0, 0.0, 0.0], emission=spd_rgb_luminance([10.018, 3.918, 0.932]), two_sided=1)
    test = sd.add_material("test", **MATERIAL_KINDS[kind])
    zf = 4.0
    sd.add_quad([-1, 0, zf], [1, 0, zf], [1, 0, -1], [-1, 0, -1], white)
    sd.add_quad([-1, 2, -1], [1, 2, -1], [1, 2, zf], [-1, 2, zf], white)
    sd.add_quad([-1, 0, -1], [1, 0, -1], [1, 2, -1], [-1, 2, -1], white)
    sd.add_quad([-1, 0, zf], [-1, 0, -1], [-1, 2, -1], [-1, 2, zf], red)
    sd.add_quad([1, 0, -1], [1, 0, zf], [1, 2, zf], [1, 2, -1], green)
    sd.add_quad([-1, 0, zf], [-1, 2, zf], [1, 2, zf], [1, 0, zf], white)
    sd.add_quad([-0.24, 1.98, -0.22], [0.23, 1.98, -0.22], [0.23, 1.98, 0.16], [-0.24, 1.98, 0.16], light)
    sd.add_box([-0.33, 0.6, -0.29], (0.3, 0.6, 0.3), 17.0, test)
    sd.add_uv_sphere([0.38, 0.351, 0.35], 0.35, sphere_segments, sphere_rings, test)
    sd.set_camera([0.0, 1.0, 3.82], [0.0, 1.0, -6.18], [0.0, 1.0, 0.0], width, height, 39.597755335771296, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=samples, spectral=spectral)


CAMERA_KINDS = ("thin_lens", "lens_image", "equirectangular")


def camera_box(kind, width=32, height=32, samples=16, spectral=False):
    """Cornell box seen through the camera variants of scene_camera.hxx: thin lens (disk aperture), aperture image, equirectangular."""
    sd = cornell_box(width, height, samples=samples, spectral=spectral, sphere=False, finalize=False)
    sd.name = f"camera_box[{kind}]" + ("/spectral" if spectral else "/rgb")
    if kind == "equirectangular":
        sd.set_camera([0.0, 1.0, 1.5], [0.0, 1.0, -6.18], [0.0, 1.0, 0.0], width, height, 39.597755335771296, clip_near=0.1, clip_far=100.0)
        sd.camera["cls"] = 1
    else:
        sd.set_camera([0.0, 1.0, 3.82], [0.0, 1.0, -6.18], [0.0, 1.0, 0.0], width, height, 39.597755335771296, clip_near=0.1, clip_far=100.0,
                      lens_radius=0.08, focal_distance=3.9)
        if kind == "lens_image":
            # a hexagon-ish aperture with a bright rim (the loader builds the table with BuildSamplingTable | UniformSamplingTable,
            # scene_representation.cxx:1137)
            n = 16
            yy, xx = np.mgrid[0:n, 0:n]
            cx, cy = (xx + 0.5) / n * 2 - 1, (yy + 0.5) / n * 2 - 1
            r = np.maximum(np.abs(cx), np.abs(cx) * 0.5 + np.abs(cy) * 0.866)
            v = np.where(r < 0.9, 0.3 + 0.7 * (r / 0.9) ** 4, 0.0)
            px = np.stack([v, v, v, np.ones_like(v)], axis=-1).astype(f32)
            sd.camera["lens_image"] = sd.add_image(px, repeat=False, build_table=True, uniform_table=True)
    return sd.finalize(samples=samples, spectral=spectral)


def sky_image(width=64, height=32, seed=1234):
    """Procedural RGBA32F lat-long sky: vertical gradient + a sun blob (BASELINE config 3's env map in miniature)."""
    rng = np.random.default_rng(seed)
    v, u = np.meshgrid((np.arange(height) + 0.5) / height, (np.arange(width) + 0.5) / width, indexing="ij")
    up = np.cos(v * np.pi)
    sky = np.stack([0.25 + 0.35 * np.clip(up, 0, 1), 0.35 + 0.45 * np.clip(up, 0, 1), 0.55 + 0.6 * np.clip(up, 0, 1)], axis=-1)
    ground = np.array([0.12, 0.10, 0.08])
    img = np.where(up[..., None] > 0, sky, ground)
    su, sv = 0.3, 0.22
    blob = 40.0 * np.exp(-(((u - su) * 2 * np.cos((v - 0.5) * np.pi)) ** 2 + (v - sv) ** 2) / (2 * 0.015 ** 2))
    img = img + blob[..., None] * np.array([1.0, 0.9, 0.7])
    img = img * (1.0 + 0.02 * rng.random(img.shape))
    return np.concatenate([img, np.ones((height, width, 1))], axis=-1).astype(f32)


def checker_image(n=16, a=(0.8, 0.8, 0.8), b=(0.2, 0.3, 0.6), alpha_holes=False):
    yy, xx = np.mgrid[0:n, 0:n]
    m = ((xx // 2 + yy // 2) % 2).astype(bool)
    img = np.where(m[..., None], np.array(a), np.array(b))
    alpha = np.ones((n, n, 1))
    if alpha_holes:
        alpha[(xx % 4 == 0) & (yy % 4 == 0)] = 0.25
    return np.concatenate([img, alpha], axis=-1).astype(f32)


def sky_room(width=32, height=32, samples=16, spectral=False, textures=True, sun=True, env=True, area_light=True):
    """Open scene under an importance-sampled environment map + a finite-size sun, textured / normal-mapped floor, plastic and conductor props."""
    sd = SceneData()
    sd.name = "sky_room" + ("/spectral" if spectral else "/rgb")
    floor_kw = dict(kd=[1.0, 1.0, 1.0])
    floor = sd.add_material("floor", **floor_kw)
    plastic = sd.add_material("plastic", cls=S.MAT_PLASTIC, kd=[0.7, 0.2, 0.2], ks=[1, 1, 1], roughness=0.5, int_ior="plastic")
    metal = sd.add_material("metal", cls=S.MAT_CONDUCTOR, ks=[1, 1, 1], roughness=0.4, int_ior="gold")
    panel = sd.add_material("panel", kd=[0.9, 0.9, 0.9], two_sided=1)
    light = sd.add_material("light", kd=[0, 0, 0], emission=spd_rgb_luminance([6.0, 5.0, 4.0]), two_sided=1)
    if textures:
        checker = sd.add_image(checker_image(16), repeat=True)
        holes = sd.add_image(checker_image(8, alpha_holes=True), repeat=True)
        nrm_px = np.zeros((8, 8, 4), dtype=f32)
        yy, xx = np.mgrid[0:8, 0:8]
        nrm_px[..., 0] = 0.5 + 0.2 * np.sin(xx * np.pi / 4)
        nrm_px[..., 1] = 0.5 + 0.2 * np.cos(yy * np.pi / 4)
        nrm_px[..., 2] = 0.9
        nrm_px[..., 3] = 1.0
        nmap = sd.add_image(nrm_px, repeat=True)
        rough = sd.add_image(np.concatenate([np.tile(np.linspace(0.3, 1.0, 8, dtype=f32)[None, :, None], (8, 1, 3)), np.ones((8, 8, 1), f32)], axis=-1), repeat=True)
        sd.materials[floor]["scattering"]["image_index"] = checker
        sd.materials[floor]["normal_image_index"] = nmap
        sd.materials[floor]["normal_scale"] = 0.7
        sd.materials[panel]["scattering"]["image_index"] = holes
        sd.materials[metal]["roughness"]["image_index"] = rough
        sd.materials[metal]["roughness"]["channel"] = 0
    sd.add_quad([-2, 0, 2], [2, 0, 2], [2, 0, -2], [-2, 0, -2], floor, 2)
    sd.add_box([-0.5, 0.4, -0.3], (0.35, 0.4, 0.35), 20.0, plastic)
    sd.add_uv_sphere([0.55, 0.4, 0.2], 0.4, 16, 9, metal)
    sd.add_quad([-1.2, 0.0, -1.2], [1.2, 0.0, -1.2], [1.2, 1.4, -1.2], [-1.2, 1.4, -1.2], panel)
    if area_light:
        sd.add_quad([-0.3, 1.6, -0.3], [0.3, 1.6, -0.3], [0.3, 1.6, 0.3], [-0.3, 1.6, 0.3], light)
    if env:
        sky = sd.add_image(sky_image(64, 32), repeat=True, build_table=True)
        sd.add_environment_emitter(sky, rgb=(1.0, 1.0, 1.0))
    if sun:
        sd.add_directional_emitter([0.3, 0.8, 0.5], rgb=(3.0, 2.8, 2.5), angular_size_deg=2.0)
    sd.set_camera([0.0, 1.2, 3.6], [0.0, 0.5, 0.0], [0.0, 1.0, 0.0], width, height, 45.0, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=samples, spectral=spectral)


def _grid_mesh(p00, du, dv, nu, nv):
    """Vectorised tessellated parallelogram: positions, normals, uvs, indices (two triangles per cell)."""
    p00, du, dv = [np.asarray(x, dtype=np.float64) for x in (p00, du, dv)]
    us, vs = np.meshgrid(np.linspace(0, 1, nu + 1), np.linspace(0, 1, nv + 1), indexing="xy")
    pos = p00 + us[..., None] * du + vs[..., None] * dv
    n = np.cross(du, dv)
    n = n / np.linalg.norm(n)
    i = (np.arange(nv)[:, None] * (nu + 1) + np.arange(nu)[None, :]).reshape(-1)
    a, b, c, d = i, i + 1, i + nu + 2, i + nu + 1
    idx = np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)])
    return pos.reshape(-1, 3), np.tile(n, (pos.shape[0] * pos.shape[1], 1)), np.stack([us, vs], -1).reshape(-1, 2), idx


def _sphere_mesh(center, radius, segments, rings, bump=0.0, seed=0):
    """Vectorised UV sphere (2*segments*(rings-1) triangles) with optional low-frequency radial displacement."""
    theta = np.pi * np.arange(rings + 1) / rings
    phi = 2 * np.pi * np.arange(segments + 1) / segments
    st, ct = np.sin(theta)[:, None], np.cos(theta)[:, None]
    d = np.stack([st * np.cos(phi)[None, :], ct * np.ones_like(phi)[None, :], st * np.sin(phi)[None, :]], -1)
    r = radius * (1.0 + bump * np.sin(3 * phi + seed)[None, :] * np.sin(2 * theta + 0.5 * seed)[:, None])
    pos = np.asarray(center, dtype=np.float64) + d * r[..., None]
    rr, ss = np.meshgrid(np.arange(rings), np.arange(segments), indexing="ij")
    a = (rr * (segments + 1) + ss).reshape(-1)
    b, dd, e = a + 1, a + segments + 1, a + segments + 2
    rflat = rr.reshape(-1)
    t1 = np.stack([a, b, dd], 1)[rflat != 0]
    t2 = np.stack([b, e, dd], 1)[rflat != rings - 1]
    uv = np.stack(np.meshgrid(np.arange(segments + 1) / segments, np.arange(rings + 1) / rings, indexing="xy"), -1)
    return pos.reshape(-1, 3), d.reshape(-1, 3), uv.reshape(-1, 2), np.concatenate([t1, t2])


def procedural_room(width=1920, height=1080, samples=1024, spectral=True, target_triangles=1_000_000, props=200, env_size=(2048, 1024), seed=1234):
    """BASELINE config 3: ~1 M-triangle room — tessellated floor/walls + `props` displaced spheres with materials round-robin
    {plastic, conductor (gold), plastic + thin film, diffuse}, lit by a procedural sky/sun environment map through an open roof
    plus one area light (SURVEY.md 8(d))."""
    rng = np.random.default_rng(seed)
    sd = SceneData()
    sd.name = f"room{target_triangles // 1000}k" + ("/spectral" if spectral else "/rgb")
    wall = sd.add_material("wall", kd=[0.8, 0.8, 0.8], two_sided=1)
    floor = sd.add_material("floor", kd=[0.6, 0.5, 0.4], two_sided=1)
    mats = [
        sd.add_material("plastic", cls=S.MAT_PLASTIC, kd=[0.7, 0.25, 0.2], ks=[1, 1, 1], roughness=0.3, int_ior="plastic"),
        sd.add_material("gold", cls=S.MAT_CONDUCTOR, ks=[1, 1, 1], roughness=0.2, int_ior="gold"),
        sd.add_material("plastic_film", cls=S.MAT_PLASTIC, kd=[0.2, 0.3, 0.7], ks=[1, 1, 1], roughness=0.3, int_ior="plastic", thinfilm=("glass", 300.0, 700.0)),
        sd.add_material("diffuse", kd=[0.3, 0.7, 0.3]),
    ]
    light = sd.add_material("light", kd=[0, 0, 0], emission=spd_rgb_luminance([12.0, 10.0, 8.0]), two_sided=1)
    rings = 24
    segments = 48
    per_prop = 2 * segments * (rings - 1)
    structure = max(target_triangles - props * per_prop, 6 * 2)
    n = max(1, int(math.sqrt(structure / (2 * 5.0))))  # 5 tessellated surfaces
    X, Y, Z = 4.0, 3.0, 4.0
    surfaces = [
        ([-X, 0, Z], [2 * X, 0, 0], [0, 0, -2 * Z], floor),          # floor (+y)
        ([-X, 0, -Z], [2 * X, 0, 0], [0, Y, 0], wall),               # back wall (+z)
        ([-X, 0, Z], [0, 0, -2 * Z], [0, Y, 0], wall),               # left wall (+x)
        ([X, 0, -Z], [0, 0, 2 * Z], [0, Y, 0], wall),                # right wall (-x)
        ([-X, Y, -Z], [2 * X, 0, 0], [0, 0, 0.9 * Z], wall),         # half ceiling (-y), rest open to the sky
    ]
    for p00, du, dv, mat in surfaces:
        pos, nrm, uv, idx = _grid_mesh(p00, du, dv, n, n)
        sd.add_mesh(pos, nrm, idx, mat, uvs=uv)
    for k in range(props):
        cx, cz = rng.uniform(-X + 0.4, X - 0.4), rng.uniform(-Z + 0.4, Z - 0.4)
        r = rng.uniform(0.12, 0.28)
        cy = r * 1.02 + (rng.uniform(0, 1.5) if k % 5 == 0 else 0.0)
        pos, nrm, uv, idx = _sphere_mesh([cx, cy, cz], r, segments, rings, bump=0.12, seed=k)
        sd.add_mesh(pos, nrm, idx, mats[k % 4], uvs=uv)
    sd.add_quad([-0.6, Y - 0.02, -2.6], [0.6, Y - 0.02, -2.6], [0.6, Y - 0.02, -1.4], [-0.6, Y - 0.02, -1.4], light)
    sky = sd.add_image(sky_image(env_size[0], env_size[1], seed=seed), repeat=True, build_table=True)
    sd.add_environment_emitter(sky, rgb=(1.0, 1.0, 1.0))
    sd.set_camera([0.0, 1.6, 3.8], [0.0, 1.0, 0.0], [0.0, 1.0, 0.0], width, height, 55.0, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=samples, spectral=spectral)


def fbm_density(n=16, seed=42):
    """Deterministic value-noise fBm on an n^3 grid, normalised to max 1 (BASELINE config 5's cloud in miniature)."""
    rng = np.random.default_rng(seed)
    total = np.zeros((n, n, n))
    amp, freq = 1.0, 2
    z, y, x = np.mgrid[0:n, 0:n, 0:n] / n
    while freq <= n:
        lattice = rng.random((freq + 1, freq + 1, freq + 1))
        fx, fy, fz = x * freq, y * freq, z * freq
        ix, iy, iz = fx.astype(int), fy.astype(int), fz.astype(int)
        tx, ty, tz = fx - ix, fy - iy, fz - iz
        def L(a, b, c):
            return lattice[iz + c, iy + b, ix + a]
        v = ((L(0, 0, 0) * (1 - tx) + L(1, 0, 0) * tx) * (1 - ty) + (L(0, 1, 0) * (1 - tx) + L(1, 1, 0) * tx) * ty) * (1 - tz) + \
            ((L(0, 0, 1) * (1 - tx) + L(1, 0, 1) * tx) * (1 - ty) + (L(0, 1, 1) * (1 - tx) + L(1, 1, 1) * tx) * ty) * tz
        total += amp * v
        amp *= 0.5
        freq *= 2
    r = np.sqrt((x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2)
    total = np.clip(total * np.clip(1.0 - 2.0 * r, 0, 1) - 0.15, 0, None)
    return (total / total.max()).astype(f32)


def media_box(kind="fog", width=32, height=32, samples=16, spectral=False):
    """Cornell box with participating media behind Boundary materials:
    fog      — homogeneous scattering medium in a box (boundary crossings, medium light vertices, explicit connections)
    cloud    — heterogeneous fBm density (delta tracking / ratio tracking), anisotropic phase function
    tinted   — absorbing homogeneous medium inside a smooth dielectric sphere + thin fog without explicit connections
    camera   — the camera itself sits inside a homogeneous medium that fills the room"""
    sd = SceneData()
    sd.name = f"media_box[{kind}]" + ("/spectral" if spectral else "/rgb")
    white = sd.add_material("white", kd=[1.0, 1.0, 1.0], two_sided=1)
    red = sd.add_material("leftWall", kd=[1.0, 0.0, 0.0], two_sided=1)
    green = sd.add_material("rightWall", kd=[0.0, 1.0, 0.0], two_sided=1)
    light = sd.add_material("light", kd=[0.0, 0.0, 0.0], emission=spd_rgb_luminance([10.018, 3.918, 0.932]), two_sided=1)
    zf = 4.0
    sd.add_quad([-1, 0, zf], [1, 0, zf], [1, 0, -1], [-1, 0, -1], white)
    sd.add_quad([-1, 2, -1], [1, 2, -1], [1, 2, zf], [-1, 2, zf], white)
    sd.add_quad([-1, 0, -1], [1, 0, -1], [1, 2, -1], [-1, 2, -1], white)
    sd.add_quad([-1, 0, zf], [-1, 0, -1], [-1, 2, -1], [-1, 2, zf], red)
    sd.add_quad([1, 0, -1], [1, 0, zf], [1, 2, zf], [1, 2, -1], green)
    sd.add_quad([-1, 0, zf], [-1, 2, zf], [1, 2, zf], [1, 0, zf], white)
    sd.add_quad([-0.24, 1.98, -0.22], [0.23, 1.98, -0.22], [0.23, 1.98, 0.16], [-0.24, 1.98, 0.16], light)
    cam_medium = S.INVALID
    if kind == "fog":
        fog = sd.add_medium(absorption=(0.05, 0.05, 0.05), scattering=(1.6, 1.4, 1.2), g=0.3)
        b = sd.add_material("fog", cls=S.MAT_BOUNDARY, int_medium=fog)
        sd.add_box([0.0, 0.7, 0.0], (0.6, 0.55, 0.6), 10.0, b)
        sd.add_box([-0.3, 0.3, 0.2], (0.15, 0.3, 0.15), 30.0, white)  # an object inside the fog
    elif kind == "cloud":
        cloud = sd.add_medium(absorption=(0.2, 0.2, 0.2), scattering=(18.0, 18.0, 18.0), g=0.8, density=fbm_density(16), bounds=([-0.6, 0.4, -0.6], [0.6, 1.6, 0.6]), max_sigma=18.2)
        b = sd.add_material("cloud", cls=S.MAT_BOUNDARY, int_medium=cloud)
        sd.add_box([0.0, 1.0, 0.0], (0.6, 0.6, 0.6), 0.0, b)
    elif kind == "tinted":
        tint = sd.add_medium(absorption=(0.2, 1.5, 3.0), scattering=(0.0, 0.0, 0.0))
        thin = sd.add_medium(absorption=(0.0, 0.0, 0.0), scattering=(0.5, 0.5, 0.5), explicit_connections=False)
        glass = sd.add_material("glass", cls=S.MAT_DIELECTRIC, roughness=0.0, int_ior="glass", int_medium=tint)
        sd.add_uv_sphere([0.35, 0.41, 0.3], 0.4, 16, 9, glass)
        b = sd.add_material("haze", cls=S.MAT_BOUNDARY, int_medium=thin)
        sd.add_box([-0.4, 0.9, -0.2], (0.35, 0.8, 0.35), 0.0, b)
    elif kind == "camera":
        room = sd.add_medium(absorption=(0.02, 0.02, 0.02), scattering=(0.25, 0.25, 0.3), g=0.0)
        cam_medium = room
        for m in sd.materials:
            m["ext_medium"] = room  # emitters start their paths in the room's medium (emitter_external_medium_index)
        sd.add_box([0.3, 0.3, 0.2], (0.3, 0.3, 0.3), -17.0, white)
    else:
        raise KeyError(kind)
    sd.set_camera([0.0, 1.0, 3.82], [0.0, 1.0, -6.18], [0.0, 1.0, 0.0], width, height, 39.597755335771296, clip_near=0.1, clip_far=100.0)
    sd.camera["medium_index"] = cam_medium
    return sd.finalize(samples=samples, spectral=spectral)


def fbm_density_fast(n=256, seed=42):
    """fbm_density for large grids (float32, one z-slab at a time; same recipe, its own lattice order) — BASELINE config 5 uses 256^3."""
    rng = np.random.default_rng(seed)
    total = np.zeros((n, n, n), dtype=f32)
    c = ((np.arange(n, dtype=f32) + f32(0.0)) / f32(n)).astype(f32)
    amp, freq = f32(1.0), 2
    while freq <= n:
        lattice = rng.random((freq + 1, freq + 1, freq + 1), dtype=f32)
        f = c * f32(freq)
        i0 = f.astype(np.int64)
        t = (f - i0).astype(f32)
        i1 = i0 + 1
        # separable trilinear interpolation: z, then y, then x
        a = lattice[i0] * (1 - t)[:, None, None] + lattice[i1] * t[:, None, None]            # (n, F, F)
        a = a[:, i0, :] * (1 - t)[None, :, None] + a[:, i1, :] * t[None, :, None]          # (n, n, F)
        a = a[:, :, i0] * (1 - t)[None, None, :] + a[:, :, i1] * t[None, None, :]          # (n, n, n)
        total += amp * a.astype(f32)
        amp *= f32(0.5)
        freq *= 2
    r2 = (c[:, None, None] - f32(0.5)) ** 2 + (c[None, :, None] - f32(0.5)) ** 2 + (c[None, None, :] - f32(0.5)) ** 2
    total = np.clip(total * np.clip(1.0 - 2.0 * np.sqrt(r2), 0, 1) - f32(0.15), 0, None).astype(f32)
    return (total / total.max()).astype(f32)


def sss_dragon(width=1024, height=1024, samples=512, spectral=True, target_triangles=871_000, seed=7):
    """BASELINE config 4: the dragon stand-in — one displaced sphere of ~871 k triangles, `material class plastic` with
    `subsurface distances 1.0 0.2 0.04 scale 0.1` (random walk, diffuse entry: the loader's defaults, scene_representation.cxx:1972-2007),
    on a diffuse floor/backdrop, lit by three area emitters (SURVEY.md 8(d))."""
    sd = SceneData()
    sd.name = f"sss_dragon{target_triangles // 1000}k" + ("/spectral" if spectral else "/rgb")
    floor = sd.add_material("floor", kd=[0.7, 0.7, 0.7], two_sided=1)
    skin = sd.add_material("dragon", cls=S.MAT_PLASTIC, kd=[0.8, 0.75, 0.6], ks=[1, 1, 1], roughness=0.3, int_ior="plastic",
                           subsurface=dict(cls="random_walk", path="diffuse", distances=[1.0, 0.2, 0.04], scale=0.1))
    lights = [sd.add_material(f"light{k}", kd=[0, 0, 0], emission=spd_rgb_luminance(rgb), two_sided=1)
              for k, rgb in enumerate(([14.0, 12.0, 10.0], [4.0, 6.0, 10.0], [10.0, 5.0, 3.0]))]
    # 2*segments*(rings-1) triangles with segments = 2*rings
    rings = max(4, int(round(math.sqrt(target_triangles / 4.0))))
    segments = 2 * rings
    pos, nrm, uv, idx = _sphere_mesh([0.0, 0.75, 0.0], 0.62, segments, rings, bump=0.0)
    # "dragon" relief: three octaves of low-frequency lobes along the smooth normal (positions only; shading normals stay the sphere's)
    d = nrm
    relief = (0.10 * np.sin(5.0 * d[:, 0] + 0.3 * seed) * np.sin(4.0 * d[:, 1] + 1.1) + 0.05 * np.sin(11.0 * d[:, 2] + 0.7 * seed) * np.cos(9.0 * d[:, 0])
              + 0.02 * np.sin(23.0 * d[:, 1]) * np.sin(19.0 * d[:, 2] + seed))
    pos = pos + d * (0.62 * relief)[:, None]
    sd.add_mesh(pos, nrm, idx, skin, uvs=uv)
    sd.add_quad([-3, 0, 3], [3, 0, 3], [3, 0, -3], [-3, 0, -3], floor, 2)
    sd.add_quad([-3, 0, -1.6], [3, 0, -1.6], [3, 3, -1.6], [-3, 3, -1.6], floor, 2)
    sd.add_quad([-0.5, 2.4, -0.5], [0.5, 2.4, -0.5], [0.5, 2.4, 0.5], [-0.5, 2.4, 0.5], lights[0])          # key, overhead (faces down: two-sided)
    sd.add_quad([-1.9, 0.3, 0.2], [-1.9, 0.3, 1.0], [-1.9, 1.3, 1.0], [-1.9, 1.3, 0.2], lights[1])          # cool fill from the left
    sd.add_quad([1.7, 0.2, -0.9], [1.7, 0.2, -0.3], [1.7, 1.5, -0.3], [1.7, 1.5, -0.9], lights[2])          # warm rim from behind right
    sd.set_camera([0.0, 1.0, 3.2], [0.0, 0.75, 0.0], [0.0, 1.0, 0.0], width, height, 40.0, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=samples, spectral=spectral)


def cloud_box(width=1024, height=1024, samples=256, spectral=True, grid=256, seed=42):
    """BASELINE config 5: unit-cube `boundary` mesh holding a heterogeneous cloud (fBm density grid^3 normalised to max 1 like
    medium_pool.cxx:44-55; scattering : absorption = 0.9 : 0.01; majorant max_sigma = 20, i.e. ~20 tracking steps with 8-tap density
    gathers per crossing; g = 0.8) under a sun (directional emitter) and a sky environment map, over a diffuse ground plane.
    The reference's tracker attenuates every segment by the medium's FULL extinction whatever the local density
    (scene_medium.hxx:306-346), so sigma_t is kept at ~2 per unit length (the cube stays translucent) while max_sigma sets the step rate.
    Rendered connect-only (`vcm-merging` off = volumetric BDPT); the caller sets that option (workload_options)."""
    sd = SceneData()
    sd.name = f"cloud{grid}" + ("/spectral" if spectral else "/rgb")
    ground = sd.add_material("ground", kd=[0.35, 0.4, 0.3], two_sided=1)
    k = 2.0 / 0.91
    density = fbm_density(grid, seed) if grid <= 32 else fbm_density_fast(grid, seed)
    cloud = sd.add_medium(absorption=(0.01 * k,) * 3, scattering=(0.9 * k,) * 3, g=0.8, density=density,
                          bounds=([-0.5, 0.6, -0.5], [0.5, 1.6, 0.5]), max_sigma=20.0)
    b = sd.add_material("cloud", cls=S.MAT_BOUNDARY, int_medium=cloud)
    sd.add_box([0.0, 1.1, 0.0], (0.5, 0.5, 0.5), 0.0, b)
    sd.add_quad([-6, 0, 6], [6, 0, 6], [6, 0, -6], [-6, 0, -6], ground, 2)
    sky = sd.add_image(sky_image(256 if grid > 32 else 64, 128 if grid > 32 else 32, seed=1234), repeat=True, build_table=True)
    sd.add_environment_emitter(sky, rgb=(1.0, 1.0, 1.0))
    sd.add_directional_emitter([0.35, 0.8, 0.45], rgb=(6.0, 5.6, 5.0), angular_size_deg=1.0)
    sd.set_camera([0.0, 1.0, 3.4], [0.0, 1.1, 0.0], [0.0, 1.0, 0.0], width, height, 35.0, clip_near=0.1, clip_far=100.0)
    return sd.finalize(samples=samples, spectral=spectral)


def workload_options(name):
    """Integrator options a named config runs with beyond the defaults (vcm_shared.cxx:6-28)."""
    return {"vcm-merging": 0.0} if name == "C5" else {}


def config(name, scale=1.0):
    """Named BASELINE.json configs. `scale` < 1 shrinks resolution for CPU-sized tests (geometry unchanged)."""
    def dim(v):
        return max(16, int(round(v * scale)))
    if name == "C1":
        return cornell_box(dim(512), dim(512), samples=16, spectral=False, sphere=False)
    if name == "C2":
        return cornell_box(dim(1024), dim(1024), samples=256, spectral=True, sphere=True)
    if name == "C3":
        return procedural_room(dim(1920), dim(1080), samples=1024, spectral=True)
    if name == "C4":
        return sss_dragon(dim(1024), dim(1024), samples=512, spectral=True)
    if name == "C5":
        return cloud_box(dim(1024), dim(1024), samples=256, spectral=True)
    raise KeyError(name)
