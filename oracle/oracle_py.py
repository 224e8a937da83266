"""ctypes binding of the CPU oracle (oracle/_ref/liboracle_*.so).  TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
The product package (etx_tracer_b200) never does.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def lib_path(flavor="parity"):
    return os.path.join(HERE, "_ref", f"liboracle_{flavor}.so")


def available(flavor="parity"):
    return os.path.exists(lib_path(flavor))


_libs = {}


def load(flavor="parity"):
    if flavor in _libs:
        return _libs[flavor]
    lib = C.CDLL(lib_path(flavor))
    vp, u32, u64, f32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_float
    lib.oracle_create.restype = vp
    lib.oracle_create.argtypes = [vp, u64, vp, u64]
    lib.oracle_destroy.argtypes = [vp]
    lib.oracle_set_options.argtypes = [vp, vp]
    lib.oracle_begin.argtypes = [vp, u32]
    lib.oracle_run_iterations.restype = C.c_double
    lib.oracle_run_iterations.argtypes = [vp, u32, u32]
    lib.oracle_read_film.argtypes = [vp, u32, vp, u64]
    if hasattr(lib, "oracle_set_integrator"):
        lib.oracle_set_integrator.argtypes = [vp, u32]
        lib.oracle_pt_set_options.argtypes = [vp, vp]
        lib.oracle_pt_get_status.argtypes = [vp, vp]
        lib.oracle_set_scene_settings.argtypes = [vp, f32, f32]
    lib.oracle_read_buffer.argtypes = [vp, u32, vp, u64, C.POINTER(u64)]
    lib.oracle_get_counters.argtypes = [vp, vp]
    lib.oracle_trace.argtypes = [vp, vp, vp, u32, vp, vp]
    lib.oracle_bvh_info.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]
    if hasattr(lib, "oracle_bsdf_eval"):  # an oracle/_ref built before this export still serves every other test
        lib.oracle_bsdf_eval.argtypes = [vp, vp, u32, u32, u32, vp]
    if hasattr(lib, "oracle_bsdf_sample"):
        lib.oracle_bsdf_sample.argtypes = [vp, vp, u32, u32, u32, vp]
    if hasattr(lib, "oracle_emitter"):
        lib.oracle_emitter.argtypes = [vp, vp, u32, u32, u32, vp]
    if hasattr(lib, "oracle_medium"):
        lib.oracle_medium.argtypes = [vp, vp, u32, u32, u32, vp]
    if hasattr(lib, "oracle_subsurface"):
        lib.oracle_subsurface.argtypes = [vp, vp, u32, u32, u32, vp]
    if hasattr(lib, "oracle_merge"):
        lib.oracle_merge.argtypes = [vp, vp, u32, vp, vp, u32, u32, u32, vp, vp]
    lib.oracle_sampler.argtypes = [vp, vp, u32, u32, vp, vp]
    lib.oracle_math.argtypes = [u32, vp, vp, u32, vp]
    lib.oracle_offset_ray.argtypes = [vp, vp, vp]
    lib.oracle_grid_cell_index.restype = u32
    lib.oracle_grid_cell_index.argtypes = [u32, C.c_int32, C.c_int32, C.c_int32]
    lib.oracle_spectrum_rgb_reflectance.argtypes = [vp, vp]
    lib.oracle_spectrum_rgb_luminance.argtypes = [vp, vp]
    lib.oracle_spectrum_constant.argtypes = [f32, vp]
    lib.oracle_spectrum_blackbody.argtypes = [f32, f32, C.c_int, vp]
    lib.oracle_spectrum_load_ior.restype = C.c_int
    lib.oracle_spectrum_load_ior.argtypes = [C.c_char_p, vp, vp]
    lib.oracle_spectrum_luminance.restype = f32
    lib.oracle_spectrum_luminance.argtypes = [vp]
    lib.oracle_color_tables.argtypes = [vp, vp, vp]
    lib.oracle_build_camera.argtypes = [vp, vp, vp, vp, u32, u32, f32]
    lib.oracle_sizeof.restype = u32
    lib.oracle_sizeof.argtypes = [u32]
    _libs[flavor] = lib
    return lib


def has_bsdf_eval(flavor="parity"):
    """Whether the built oracle exports oracle_bsdf_eval (oracle/_ref is older than the export where the reference could not rebuild it)."""
    return hasattr(load(flavor), "oracle_bsdf_eval")


def has_bsdf_sample(flavor="parity"):
    """Whether the built oracle exports oracle_bsdf_sample."""
    return hasattr(load(flavor), "oracle_bsdf_sample")


def has_emitter(flavor="parity"):
    """Whether the built oracle exports oracle_emitter."""
    return hasattr(load(flavor), "oracle_emitter")


def has_medium(flavor="parity"):
    """Whether the built oracle exports oracle_medium."""
    return hasattr(load(flavor), "oracle_medium")


def has_subsurface(flavor="parity"):
    """Whether the built oracle exports oracle_subsurface."""
    return hasattr(load(flavor), "oracle_subsurface")


def has_merge(flavor="parity"):
    """Whether the built oracle exports oracle_merge."""
    return hasattr(load(flavor), "oracle_merge")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


REFERENCE_ROOT = os.environ.get("ETX_REFERENCE", "/root/reference")


class ReferenceScene:
    """A scene file loaded by the reference's OWN loader (oracle/_ref/libreference_loader.so = scene_representation.cxx and friends compiled
    in place, oracle/ref_loader.cxx).  Exposes what Oracle / GPUVCM read from a SceneData: `.scene` and `.camera` as numpy views over the
    Scene / Camera PODs the loader owns (528 / 176 bytes, host pointers inside), plus width / height / triangle_count.  Only usable where the
    reference tree (assets, IOR database) exists; `resize()` rebuilds the camera for a smaller film (build_camera, same view)."""

    _lib = None

    @classmethod
    def available(cls):
        return os.path.exists(os.path.join(HERE, "_ref", "libreference_loader.so")) and os.path.isdir(os.path.join(REFERENCE_ROOT, "bin", "assets"))

    @classmethod
    def lib(cls):
        if cls._lib is None:
            lib = C.CDLL(os.path.join(HERE, "_ref", "libreference_loader.so"))
            lib.refloader_load.restype = C.c_void_p
            lib.refloader_load.argtypes = [C.c_char_p, C.c_char_p]
            lib.refloader_free.argtypes = [C.c_void_p]
            lib.refloader_free.restype = None
            for fn in (lib.refloader_scene, lib.refloader_camera):
                fn.restype = C.c_void_p
                fn.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
            lib.refloader_material_index.restype = C.c_uint32
            lib.refloader_material_index.argtypes = [C.c_void_p, C.c_char_p]
            cls._lib = lib
        return cls._lib

    def __init__(self, scene_file, data_folder=None):
        from etx_tracer_b200 import structs as S
        lib = self.lib()
        path = scene_file if os.path.isabs(scene_file) else os.path.join(REFERENCE_ROOT, "bin", scene_file)
        self.h = lib.refloader_load((data_folder or os.path.join(REFERENCE_ROOT, "bin")).encode(), path.encode())
        if not self.h:
            raise RuntimeError(f"the reference loader rejected {path}")
        n = C.c_uint64(0)
        sp = lib.refloader_scene(self.h, C.byref(n))
        assert n.value == S.SCENE.itemsize, (n.value, S.SCENE.itemsize)
        self.scene = np.frombuffer((C.c_char * S.SCENE.itemsize).from_address(sp), dtype=S.SCENE)
        cp = lib.refloader_camera(self.h, C.byref(n))
        assert n.value == S.CAMERA.itemsize, (n.value, S.CAMERA.itemsize)
        self.camera = np.frombuffer((C.c_char * S.CAMERA.itemsize).from_address(cp), dtype=S.CAMERA).copy()  # resize() edits the copy
        self.name = "reference:" + os.path.basename(path)

    @property
    def width(self):
        return int(self.camera["film_size"][0][0])

    @property
    def height(self):
        return int(self.camera["film_size"][0][1])

    @property
    def triangle_count(self):
        return int(self.scene["triangles"]["count"][0])

    def material_index(self, name):
        return int(self.lib().refloader_material_index(self.h, name.encode()))

    def resize(self, width, height, origin, target, up, fov):
        """build_camera (scene_representation.cxx:579-598) for another film size, through the oracle's export of the reference function."""
        o, t, u = (np.asarray(v, dtype=np.float32) for v in (origin, target, up))
        load("parity").oracle_build_camera(_p(self.camera), _p(o), _p(t), _p(u), int(width), int(height), C.c_float(fov))
        return self

    def close(self):
        if getattr(self, "h", None):
            self.lib().refloader_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Oracle:
    """One oracle instance bound to a SceneData (etx_tracer_b200.scenes.SceneData) or a ReferenceScene."""

    def __init__(self, scene_data, flavor="parity"):
        from etx_tracer_b200 import structs as S

        self.lib = load(flavor)
        self.scene_data = scene_data  # keeps the numpy arrays alive
        self.S = S
        self.h = self.lib.oracle_create(_p(scene_data.scene), scene_data.scene.nbytes, _p(scene_data.camera), scene_data.camera.nbytes)
        if not self.h:
            raise RuntimeError("oracle_create failed (layout mismatch)")
        self.width = int(scene_data.camera["film_size"][0][0])
        self.height = int(scene_data.camera["film_size"][0][1])

    def close(self):
        if self.h:
            self.lib.oracle_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_options(self, opts):
        self.lib.oracle_set_options(self.h, _p(opts))

    def set_integrator(self, integrator):
        """0 = VCM (default), 1 = the reference's path tracer (run_path_iteration compiled in place + the restated CPUPathTracing driver)."""
        self.lib.oracle_set_integrator(self.h, integrator)

    def pt_set_options(self, opts):
        self.lib.oracle_pt_set_options(self.h, _p(opts))

    def pt_status(self):
        st = np.zeros(1, dtype=self.S.PT_STATUS)
        self.lib.oracle_pt_get_status(self.h, _p(st))
        return {k: st[k][0].item() for k in st.dtype.names}

    def set_scene_settings(self, noise_threshold, radiance_clamp=0.0):
        self.lib.oracle_set_scene_settings(self.h, C.c_float(noise_threshold), C.c_float(radiance_clamp))

    def begin(self, first_iteration=0):
        self.lib.oracle_begin(self.h, first_iteration)

    def run(self, iterations, threads=1):
        return self.lib.oracle_run_iterations(self.h, iterations, threads)

    def film(self, layer=0):
        out = np.zeros((self.height, self.width, 4), dtype=np.float32)
        rc = self.lib.oracle_read_film(self.h, layer, _p(out), out.nbytes)
        assert rc == 0
        return out

    def buffer(self, buf_id, dtype):
        n = C.c_uint64(0)
        rc = self.lib.oracle_read_buffer(self.h, buf_id, None, 0, C.byref(n))
        assert rc == 0, rc
        out = np.zeros(n.value // np.dtype(dtype).itemsize, dtype=dtype)
        if n.value:
            rc = self.lib.oracle_read_buffer(self.h, buf_id, _p(out), out.nbytes, C.byref(n))
            assert rc == 0, rc
        return out

    def counters(self):
        c = np.zeros(1, dtype=self.S.COUNTERS)
        self.lib.oracle_get_counters(self.h, _p(c))
        return c

    def trace(self, rays, seeds):
        rays = np.ascontiguousarray(rays, dtype=np.float32)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint32).copy()
        n = rays.shape[0]
        uvt = np.zeros((n, 3), dtype=np.float32)
        tri = np.zeros(n, dtype=np.uint32)
        self.lib.oracle_trace(self.h, _p(rays), _p(seeds), n, _p(uvt), _p(tri))
        return uvt, tri, seeds

    def bsdf_eval(self, queries, repetitions, threads=None):
        """The reference's bsdf::evaluate + bsdf::reverse_pdf for S.CLOSURE_QUERY records, `repetitions` samplers Sampler(seed, r) per query;
        float64 (n, S.CLOSURE_STATS) in the layout of GPUVCM.debug_closure."""
        queries = np.ascontiguousarray(queries, dtype=self.S.CLOSURE_QUERY)
        out = np.zeros((queries.shape[0], self.S.CLOSURE_STATS), dtype=np.float64)
        self.lib.oracle_bsdf_eval(self.h, _p(queries), queries.shape[0], int(repetitions), int(threads or os.cpu_count() or 1), _p(out))
        return out

    def bsdf_sample(self, queries, repetitions, threads=None):
        """The reference's bsdf::sample for S.SAMPLE_QUERY records, repetition r of each on Sampler(seed, r); S.SAMPLE_RESULT records
        shaped (n, repetitions), in the layout of GPUVCM.debug_bsdf_sample."""
        queries = np.ascontiguousarray(queries, dtype=self.S.SAMPLE_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=self.S.SAMPLE_RESULT)
        self.lib.oracle_bsdf_sample(self.h, _p(queries), queries.shape[0], int(repetitions), int(threads or os.cpu_count() or 1), _p(out))
        return out

    def emitter(self, queries, repetitions=1, threads=None):
        """The reference's emitter routines for S.EMITTER_QUERY records, repetition r of each emission query on Sampler(seed, r); S.EMITTER_RESULT
        records shaped (n, repetitions), in the layout of GPUVCM.debug_emitter."""
        queries = np.ascontiguousarray(queries, dtype=self.S.EMITTER_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=self.S.EMITTER_RESULT)
        self.lib.oracle_emitter(self.h, _p(queries), queries.shape[0], int(repetitions), int(threads or os.cpu_count() or 1), _p(out))
        return out

    def medium(self, queries, repetitions=1, threads=None):
        """The reference's media routines for S.MEDIUM_QUERY records, repetition r of each query on Sampler(seed, r); S.MEDIUM_RESULT records
        shaped (n, repetitions), in the layout of GPUVCM.debug_medium."""
        queries = np.ascontiguousarray(queries, dtype=self.S.MEDIUM_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=self.S.MEDIUM_RESULT)
        self.lib.oracle_medium(self.h, _p(queries), queries.shape[0], int(repetitions), int(threads or os.cpu_count() or 1), _p(out))
        return out

    def subsurface(self, queries, repetitions=1, threads=None):
        """The reference's subsurface routines for S.SUBSURFACE_QUERY records, repetition r of each query on Sampler(seed, r);
        S.SUBSURFACE_RESULT records shaped (n, repetitions), in the layout of GPUVCM.debug_subsurface."""
        queries = np.ascontiguousarray(queries, dtype=self.S.SUBSURFACE_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=self.S.SUBSURFACE_RESULT)
        self.lib.oracle_subsurface(self.h, _p(queries), queries.shape[0], int(repetitions), int(threads or os.cpu_count() or 1), _p(out))
        return out

    def merge(self, records, light_wavelengths, queries, repetitions=1, threads=None):
        """The reference's VCMSpatialGridData::gather for etxb_debug_merge's inputs (S.LIGHT_VERTEX_REC records, a wavelength per light path index,
        S.MERGE_QUERY records) at the current options and iteration, `repetitions` samplers Sampler(seed, r) per query.  Returns float64 (n, 8):
        mean rgb, variance rgb, the sampler state after repetition 0, 0; and the grid as a dict like GPUVCM.debug_merge's."""
        records = np.ascontiguousarray(records, dtype=self.S.LIGHT_VERTEX_REC)
        wl = np.zeros(self.width * self.height, dtype=np.float32)
        wl[:len(light_wavelengths)] = light_wavelengths
        queries = np.ascontiguousarray(queries, dtype=self.S.MERGE_QUERY)
        out = np.zeros((queries.shape[0], 8), dtype=np.float64)
        g = np.zeros(10, dtype=np.float64)
        self.lib.oracle_merge(self.h, _p(records), records.shape[0], _p(wl), _p(queries), queries.shape[0], int(repetitions), int(threads or os.cpu_count() or 1),
                              _p(out), _p(g))
        grid = {"bbox_min": g[0:3].astype(np.float32), "bbox_max": g[3:6].astype(np.float32), "cell_size": float(g[6]), "radius_squared": float(g[7]),
                "hash_table_mask": int(g[8]), "photon_count": int(g[9])}
        return out, grid

    def bvh_info(self):
        a, b = C.c_uint32(0), C.c_uint32(0)
        self.lib.oracle_bvh_info(self.h, C.byref(a), C.byref(b))
        return a.value, b.value


def sampler_kat(a, b, draws, flavor="parity"):
    lib = load(flavor)
    a = np.ascontiguousarray(a, dtype=np.uint32)
    b = np.ascontiguousarray(b, dtype=np.uint32)
    n = a.shape[0]
    seeds = np.zeros((n, draws + 1), dtype=np.uint32)
    vals = np.zeros((n, draws), dtype=np.float32)
    lib.oracle_sampler(_p(a), _p(b), n, draws, _p(seeds), _p(vals))
    return seeds, vals


def math_kat(fn, x, y=None, flavor="parity"):
    lib = load(flavor)
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.zeros_like(x)
    if y is not None:
        y = np.ascontiguousarray(y, dtype=np.float32)
    lib.oracle_math(fn, _p(x), _p(y) if y is not None else None, x.shape[0], _p(out))
    return out
