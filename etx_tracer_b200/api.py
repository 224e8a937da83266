"""ctypes binding of the C ABI (include/etx_b200.h) + `GPUVCM`, the Python mirror of the reference's
Integrator interface for this path (sources/etx/rt/integrators/integrator.hxx:12-98, vcm_cpu.cxx:247-310).

There is no CPU fallback: loading fails loudly if the CUDA library is missing, and every call raises
EtxbError with the module's message when the device path cannot do what was asked.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build
from . import scenes as _scenes
from . import structs as S

_libs = {}


class EtxbError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"etxb error {code}: {message}")
        self.code = code


def load_library(flavor="fast"):
    if flavor in _libs:
        return _libs[flavor]
    path = _build.lib_path(flavor)
    if not os.path.exists(path):
        raise EtxbError(-100, f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
    lib = C.CDLL(path)
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    lib.etxb_build_flavor.restype = C.c_char_p
    lib.etxb_last_error.restype = C.c_char_p
    lib.etxb_last_error.argtypes = [vp]
    lib.etxb_create.argtypes = [C.POINTER(vp), vp]
    lib.etxb_destroy.argtypes = [vp]
    lib.etxb_destroy.restype = None
    lib.etxb_upload_scene.argtypes = [vp, vp, u64, vp, u64]
    lib.etxb_update_scene.argtypes = [vp, vp, u64, vp, u64, vp]
    lib.etxb_group_update_scene.argtypes = [vp, vp, u64, vp, u64, vp]
    lib.etxb_upload_blue_noise.argtypes = [vp, vp, vp, vp]
    lib.etxb_upload_color_tables.argtypes = [vp, vp, vp]
    lib.etxb_scene_file_load.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(vp), C.c_char_p, u64]
    lib.etxb_scene_file_free.argtypes = [vp]
    lib.etxb_scene_file_free.restype = None
    lib.etxb_scene_file_set_samples.argtypes = [vp, u32]
    lib.etxb_scene_file_set_samples.restype = None
    lib.etxb_scene_file_commit.argtypes = [vp, vp]
    lib.etxb_scene_file_table.argtypes = [vp, C.c_char_p, C.POINTER(u64)]
    lib.etxb_scene_file_table.restype = vp
    lib.etxb_atmosphere_images.argtypes = [C.c_char_p, vp, C.c_float, vp, u32, u32, vp, vp]
    lib.etxb_options_file_string.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, u64]
    lib.etxb_mesh_tangents.argtypes = [vp, u64, vp, u64]
    lib.etxb_image_file_read.argtypes = [C.c_char_p, vp, vp, vp, vp, u64, C.c_char_p, u64]
    lib.etxb_nvdb_density.argtypes = [C.c_char_p, vp, vp, u64, C.c_char_p, u64]
    for fn in (lib.etxb_scene_file_scene, lib.etxb_scene_file_camera):
        fn.argtypes = [vp]
        fn.restype = vp
    for fn in (lib.etxb_scene_file_warning_count, lib.etxb_scene_file_material_count):
        fn.argtypes = [vp]
        fn.restype = u32
    for fn in (lib.etxb_scene_file_warning, lib.etxb_scene_file_material_name):
        fn.argtypes = [vp, u32]
        fn.restype = C.c_char_p
    lib.etxb_options_default.argtypes = [vp]
    lib.etxb_options_default.restype = None
    lib.etxb_options_set_key.argtypes = [vp, C.c_char_p, C.c_double]
    lib.etxb_set_options.argtypes = [vp, vp]
    lib.etxb_set_next_iteration.argtypes = [vp, u32]
    lib.etxb_group_create.argtypes = [C.POINTER(vp), vp, u32]
    lib.etxb_group_destroy.argtypes = [vp]
    lib.etxb_group_destroy.restype = None
    lib.etxb_group_lanes.argtypes = [vp]
    lib.etxb_group_lanes.restype = u32
    lib.etxb_group_lane.argtypes = [vp, u32]
    lib.etxb_group_lane.restype = vp
    lib.etxb_group_last_error.argtypes = [vp]
    lib.etxb_group_last_error.restype = C.c_char_p
    lib.etxb_group_begin.argtypes = [vp, u32]
    lib.etxb_group_enqueue.argtypes = [vp, u32]
    lib.etxb_group_wait.argtypes = [vp]
    lib.etxb_group_poll.argtypes = [vp, vp]
    lib.etxb_group_read_film.argtypes = [vp, u32, vp, u64]
    lib.etxb_comm_unique_id.argtypes = [vp, u64]
    lib.etxb_comm_init.argtypes = [vp, u32, u32, vp, u64]
    lib.etxb_comm_world.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]
    lib.etxb_comm_reduce_film.argtypes = [vp, u32, vp, u64]
    lib.etxb_group_comm_init.argtypes = [vp, u32, u32, vp, u32]
    lib.etxb_group_comm_reduce_film.argtypes = [vp, u32, vp, u64]
    lib.etxb_group_comm_init_replicas.argtypes = [vp, u32, u32, vp, u64]
    lib.etxb_group_reserve_split_lane.argtypes = [vp]
    lib.etxb_debug_group_plan.argtypes = [u32, u32, u32, u32, C.c_int, vp, u32, vp, u32]
    lib.etxb_set_integrator.argtypes = [vp, u32]
    lib.etxb_pt_options_default.argtypes = [vp]
    lib.etxb_pt_options_default.restype = None
    lib.etxb_pt_options_set_key.argtypes = [vp, C.c_char_p, C.c_double]
    lib.etxb_pt_set_options.argtypes = [vp, vp]
    lib.etxb_pt_get_status.argtypes = [vp, vp]
    lib.etxb_set_scene_settings.argtypes = [vp, C.c_float, C.c_float]
    lib.etxb_set_partition.argtypes = [vp, u32, u32]
    lib.etxb_begin.argtypes = [vp, u32]
    lib.etxb_set_film_pixel_size.argtypes = [vp, u32]
    lib.etxb_group_set_film_pixel_size.argtypes = [vp, u32]
    lib.etxb_enqueue_iteration.argtypes = [vp]
    lib.etxb_poll.argtypes = [vp, vp]
    lib.etxb_wait.argtypes = [vp]
    lib.etxb_stop.argtypes = [vp, C.c_int]
    lib.etxb_read_film.argtypes = [vp, u32, vp, u64]
    lib.etxb_film_size.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]
    lib.etxb_read_film_ldr.argtypes = [vp, u32, C.c_float, vp, u64]
    lib.etxb_denoise.argtypes = [vp, u32]
    lib.etxb_debug_denoise.argtypes = [vp, vp, vp, vp, vp, vp, vp, u32, u32, vp, vp]
    lib.etxb_debug_noise_estimate.argtypes = [vp, u32, u32, u32, C.c_float, vp, vp, vp, vp, vp, vp]
    lib.etxb_save_film.argtypes = [vp, u32, C.c_char_p, u32, C.c_float]
    lib.etxb_write_exr.argtypes = [C.c_char_p, vp, u32, u32]
    lib.etxb_write_png.argtypes = [C.c_char_p, vp, u32, u32]
    lib.etxb_tonemap_rgba8.argtypes = [vp, u64, C.c_float, vp]
    lib.etxb_get_counters.argtypes = [vp, vp]
    lib.etxb_get_kernel_times.argtypes = [vp, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.POINTER(u32), u32]
    lib.etxb_read_buffer.argtypes = [vp, u32, vp, u64, C.POINTER(u64)]
    lib.etxb_stream.restype = vp
    lib.etxb_stream.argtypes = [vp]
    lib.etxb_debug_trace.argtypes = [vp, vp, vp, u32, vp, vp]
    lib.etxb_debug_select_tree.argtypes = [vp, C.c_int]
    lib.etxb_debug_build_trees.argtypes = [vp, vp, u32, vp, u32, u32, vp]
    lib.etxb_debug_occluded.argtypes = [vp, vp, u32, vp]
    lib.etxb_debug_sampler.argtypes = [vp, vp, vp, u32, u32, vp, vp]
    lib.etxb_debug_math.argtypes = [vp, u32, vp, vp, u32, vp]
    lib.etxb_debug_closure_eval.argtypes = [vp, vp, u32, u32, vp]
    lib.etxb_debug_bsdf_sample.argtypes = [vp, vp, u32, u32, vp]
    lib.etxb_debug_emitter.argtypes = [vp, vp, u32, u32, vp]
    lib.etxb_debug_medium.argtypes = [vp, vp, u32, u32, vp]
    lib.etxb_debug_subsurface.argtypes = [vp, vp, u32, u32, vp]
    lib.etxb_debug_set_thresholds.argtypes = [vp, vp]
    lib.etxb_debug_get_branch_counts.argtypes = [vp, vp]
    lib.etxb_debug_merge.argtypes = [vp, vp, u32, vp, vp, u32, vp, vp]
    _libs[flavor] = lib
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _fields(a):
    """A one-record struct array as a dict: Python scalars, and copies of its array fields."""
    return {k: (a[k][0].copy() if a[k][0].ndim else a[k][0].item()) for k in a.dtype.names}


def _device_config(device, max_light_vertices, profile):
    cfg = np.zeros(1, dtype=S.DEVICE_CONFIG)
    cfg["device_index"] = device
    cfg["max_light_vertices"] = max_light_vertices
    cfg["flags"] = 1 if profile else 0
    return cfg


def read_image(file_name, flavor="fast"):
    """The module's image readers (PNG in every form, OpenEXR, Radiance HDR, PFM): (H, W, 4) uint8 or float32, rows in file order."""
    lib = load_library(flavor)
    w, h, eight = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    err = C.create_string_buffer(512)
    if lib.etxb_image_file_read(os.fsencode(file_name), C.byref(w), C.byref(h), C.byref(eight), None, 0, err, len(err)) != 0:
        raise EtxbError(-4, err.value.decode(errors="replace"))
    out = np.zeros((h.value, w.value, 4), dtype=np.uint8 if eight.value else np.float32)
    if lib.etxb_image_file_read(os.fsencode(file_name), C.byref(w), C.byref(h), C.byref(eight), _p(out), out.nbytes, err, len(err)) != 0:
        raise EtxbError(-4, err.value.decode(errors="replace"))
    return out


def write_exr(file_name, rgba, flavor="fast"):
    """float4 image (H, W, 4) -> OpenEXR (32-bit float A, B, G, R channels, scan lines, no compression); host code of the module."""
    rgba = np.ascontiguousarray(rgba, dtype=np.float32)
    rc = load_library(flavor).etxb_write_exr(os.fsencode(file_name), _p(rgba), rgba.shape[1], rgba.shape[0])
    if rc != 0:
        raise EtxbError(rc, f"could not write {file_name}")


def write_png(file_name, rgba8, flavor="fast"):
    rgba8 = np.ascontiguousarray(rgba8, dtype=np.uint8)
    rc = load_library(flavor).etxb_write_png(os.fsencode(file_name), _p(rgba8), rgba8.shape[1], rgba8.shape[0])
    if rc != 0:
        raise EtxbError(rc, f"could not write {file_name}")


def tonemap(rgba, exposure=1.0, flavor="fast"):
    """The reference's LDR tone map on the host (app.cxx:268-282): 1 - exp(-exposure c), sRGB curve, 8 bits."""
    rgba = np.ascontiguousarray(rgba, dtype=np.float32)
    out = np.zeros(rgba.shape[:-1] + (4,), dtype=np.uint8)
    load_library(flavor).etxb_tonemap_rgba8(_p(rgba), rgba.size // 4, C.c_float(exposure), _p(out))
    return out


class SceneFile:
    """A scene file read by the module's C++ loader (csrc/scene_loader.cpp; replaces SceneRepresentation::load_from_file,
    render/host/scene_representation.cxx:679-838).  Duck-types scenes.SceneData for GPUVCM / GPUPathTracing / GPUVCMGroup: `.scene`, `.camera`
    (numpy views of the Scene / Camera PODs the loader object owns), width / height / triangle_count, `.warnings`, `.material_names`."""

    def __init__(self, file_name, flavor="fast", data_folder=None):
        self.lib = load_library(flavor)
        self.h = C.c_void_p()
        err = C.create_string_buffer(1024)
        rc = self.lib.etxb_scene_file_load(os.fsencode(file_name), os.fsencode(data_folder) if data_folder else None, C.byref(self.h), err, len(err))
        if rc != 0:
            self.h = C.c_void_p()
            raise EtxbError(rc, err.value.decode(errors="replace") or f"could not load {file_name}")
        self.scene = np.frombuffer((C.c_char * S.SCENE.itemsize).from_address(self.lib.etxb_scene_file_scene(self.h)), dtype=S.SCENE)
        self.camera = np.frombuffer((C.c_char * S.CAMERA.itemsize).from_address(self.lib.etxb_scene_file_camera(self.h)), dtype=S.CAMERA).copy()
        self.warnings = [self.lib.etxb_scene_file_warning(self.h, i).decode(errors="replace") for i in range(self.lib.etxb_scene_file_warning_count(self.h))]
        self.material_names = {self.lib.etxb_scene_file_material_name(self.h, i).decode(errors="replace"): i for i in range(self.lib.etxb_scene_file_material_count(self.h))}
        self.name = os.path.basename(os.fsdecode(file_name))

    @property
    def width(self):
        return int(self.camera["film_size"][0][0])

    @property
    def height(self):
        return int(self.camera["film_size"][0][1])

    @property
    def triangle_count(self):
        return int(self.scene["triangles"]["count"][0])

    def table(self, name, dtype=np.uint8):
        """a table of tables.bin by name ("bluenoise/sobol", "color_tables/xyz_441x3", ...), None when absent"""
        n = C.c_uint64(0)
        p = self.lib.etxb_scene_file_table(self.h, name.encode(), C.byref(n))
        return np.frombuffer((C.c_char * n.value).from_address(p), dtype=dtype).copy() if p else None

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.scene = None
            self.lib.etxb_scene_file_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def load_scene_file(file_name, flavor="fast"):
    return SceneFile(file_name, flavor=flavor)


COMM_ID_BYTES = 128


def _bn_variant(samples):
    """BNSampler variant = next_power(min(samples, 256)) (thirdparty/bluenoise/bluenoise.cxx:73-95)"""
    spp = 1
    while spp < min(max(samples, 1), 256):
        spp *= 2
    return spp


def comm_unique_ids(count, flavor="fast"):
    """`count` NCCL unique ids (ETXB_COMM_ID_BYTES each) from the module, for rank 0 to hand to the other ranks by any transport."""
    lib = load_library(flavor)
    ids = np.zeros(count * COMM_ID_BYTES, dtype=np.uint8)
    for k in range(count):
        rc = lib.etxb_comm_unique_id(ids[k * COMM_ID_BYTES:].ctypes.data_as(C.c_void_p), COMM_ID_BYTES)
        if rc != 0:
            raise EtxbError(rc, "etxb_comm_unique_id failed (libnccl.so.2 missing?)")
    return ids


class GPUVCM:
    """`name()/run()/update()/stop()/status()/options` like the reference's CPUVCM, driving the CUDA module."""

    def __init__(self, scene_data=None, flavor="fast", device=0, max_light_vertices=0, profile=False, _adopt=None):
        self.lib = load_library(flavor)
        self.flavor = flavor
        self.h = C.c_void_p()
        self._owned = _adopt is None
        if _adopt is not None:
            self.h = C.c_void_p(_adopt)  # a lane of an etxb_group: the group owns the context
        else:
            rc = self.lib.etxb_create(C.byref(self.h), _p(_device_config(device, max_light_vertices, profile)))
            if rc != 0:
                raise EtxbError(rc, "etxb_create failed (no CUDA device? the module has no CPU fallback)")
        self.options = S.default_vcm_options()
        self.scene_data = None
        self._running = False
        self._target_iterations = 0
        ct = _scenes.tables("color_tables")
        self._xyz = np.ascontiguousarray(ct["xyz_441x3"], dtype=np.float32)
        self._rgbr = np.ascontiguousarray(ct["rgb_response_391x3"], dtype=np.float32)
        self._check(self.lib.etxb_upload_color_tables(self.h, _p(self._xyz), _p(self._rgbr)))
        if scene_data is not None:
            self.set_scene(scene_data)

    # -- plumbing ---------------------------------------------------------------------------------
    def _check(self, rc):
        if rc < 0:
            raise EtxbError(rc, self.lib.etxb_last_error(self.h).decode())
        return rc

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            if self._owned:
                self.lib.etxb_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- Integrator surface -------------------------------------------------------------------------
    @staticmethod
    def name():
        return "VCM (B200)"

    def _upload_blue_noise(self, samples):
        spp = _bn_variant(samples)
        bn = _scenes.tables("bluenoise")
        self._bn = [np.ascontiguousarray(bn[k], dtype=np.uint8) for k in ("sobol", f"scrambling_{spp}", f"ranking_{spp}")]
        self._check(self.lib.etxb_upload_blue_noise(self.h, _p(self._bn[0]), _p(self._bn[1]), _p(self._bn[2])))
        self._bn_spp = spp

    def _read_film_size(self):
        w, h = C.c_uint32(0), C.c_uint32(0)
        self._check(self.lib.etxb_film_size(self.h, C.byref(w), C.byref(h)))
        self.width, self.height = w.value, h.value

    def set_scene(self, scene_data):
        """Raytracing::link_scene/link_camera + commit_changes."""
        self.scene_data = scene_data
        self._upload_blue_noise(int(scene_data.scene["samples"][0]))
        self._check(self.lib.etxb_upload_scene(self.h, _p(scene_data.scene), scene_data.scene.nbytes, _p(scene_data.camera), scene_data.camera.nbytes))
        self._read_film_size()

    def update_scene(self, scene_data):
        """The restart after an edit of the scene or camera (etxb_update_scene): renders what set_scene(scene_data) would, keeping on the device
        what the edit did not change.  The film is cleared and armed at iteration 0; a render that was running goes on with the new scene.
        Returns the etxb_update_info fields as a dict."""
        info = np.zeros(1, dtype=S.UPDATE_INFO)
        self._check(self.lib.etxb_update_scene(self.h, _p(scene_data.scene), scene_data.scene.nbytes, _p(scene_data.camera), scene_data.camera.nbytes, _p(info)))
        self._after_update(scene_data)
        return _fields(info)

    def _after_update(self, scene_data):
        self.scene_data = scene_data
        samples = int(scene_data.scene["samples"][0])
        if _bn_variant(samples) != getattr(self, "_bn_spp", None):
            self._upload_blue_noise(samples)
        self._read_film_size()
        self._target_iterations = samples

    def set_option(self, key, value):
        """Integrator::options() keys: vcm-initial_radius, vcm-radius_decay, vcm-blue_noise, vcm-kernel, vcm-direct_hit, ..."""
        rc = self.lib.etxb_options_set_key(_p(self.options), key.encode(), float(value))
        if rc != 0:
            raise EtxbError(rc, f"unknown option key {key}")

    def set_partition(self, rank, world):
        self._check(self.lib.etxb_set_partition(self.h, rank, world))

    def comm_init(self, world, rank, comm_id):
        """Pixel tiles over `world` processes (one GPU each): collective; comm_id = the 128 bytes rank 0 got from comm_unique_ids(1)."""
        comm_id = np.ascontiguousarray(comm_id, dtype=np.uint8)
        self._check(self.lib.etxb_comm_init(self.h, world, rank, _p(comm_id), comm_id.nbytes))

    def comm_reduce_film(self, layer=S.FILM_RESULT, out=None):
        """Collective: the whole frame on rank 0 (returned there; None elsewhere).  Result, Camera, Light, and the path tracer's Normals, Albedo
        and CameraAdaptive layers."""
        w, r = C.c_uint32(1), C.c_uint32(0)
        self._check(self.lib.etxb_comm_world(self.h, C.byref(w), C.byref(r)))
        if (out is None) and (r.value == 0):
            out = np.zeros((self.height, self.width, 4), dtype=np.float32)
        self._check(self.lib.etxb_comm_reduce_film(self.h, layer, _p(out) if r.value == 0 else None, out.nbytes if r.value == 0 else 0))
        return out if r.value == 0 else None

    def set_film_pixel_size(self, size):
        """Film::set_pixel_size: the coarse preview the application renders while the camera moves (8), and full resolution (1).  Clamped to
        [1, 1024]; takes effect at the next run() or update_scene().  At size s an iteration traces ceil(W / s) x ceil(H / s) paths and every
        s x s block of the film takes its path's value; the film stays W x H."""
        self._check(self.lib.etxb_set_film_pixel_size(self.h, size))

    def _push_options(self):
        self._check(self.lib.etxb_set_options(self.h, _p(self.options)))

    def _converged(self, st):
        """Whether every pixel has converged, which ends the run before scene.samples: never for the VCM."""
        return False

    def run(self, first_iteration=0):
        """CPUVCM::run -> CPUVCMImpl::start: clears the film and arms iteration 0."""
        self._push_options()
        self._check(self.lib.etxb_begin(self.h, first_iteration))
        self._running = True
        self._target_iterations = int(self.scene_data.scene["samples"][0])

    def update(self):
        """One pump of the integrator, non-blocking like CPUVCM::update (vcm_cpu.cxx:264-276): queues the next iteration once the previous one has
        finished; stops at scene.samples like the reference, or earlier when _converged() says so."""
        if not self._running:
            return False
        st = self.status()
        if st["iteration_in_flight"]:
            return True
        if self._converged(st) or (st["completed_iterations"] >= self._target_iterations):
            self._running = False
            return False
        self._check(self.lib.etxb_enqueue_iteration(self.h))
        return True

    def render(self, iterations, first_iteration=0):
        self.run(first_iteration)
        for _ in range(iterations):
            self._check(self.lib.etxb_enqueue_iteration(self.h))
        self._check(self.lib.etxb_wait(self.h))
        return self.status()

    def iterate(self):
        self._check(self.lib.etxb_enqueue_iteration(self.h))

    def stop(self, wait_for_iteration=True):
        self._running = False
        self._check(self.lib.etxb_stop(self.h, 1 if wait_for_iteration else 0))

    def wait(self):
        self._check(self.lib.etxb_wait(self.h))

    def status(self):
        st = np.zeros(1, dtype=S.STATUS)
        self._check(self.lib.etxb_poll(self.h, _p(st)))
        return _fields(st)

    # -- results --------------------------------------------------------------------------------------
    def film(self, layer=S.FILM_RESULT, out=None):
        if out is None:
            out = np.zeros((self.height, self.width, 4), dtype=np.float32)
        self._check(self.lib.etxb_read_film(self.h, layer, _p(out), out.nbytes))
        return out

    def film_ldr(self, layer=S.FILM_RESULT, exposure=1.0):
        """The tone-mapped 8-bit frame of the reference's viewer / LDR export (app.cxx:268-282), tone-mapped on the device."""
        out = np.zeros((self.height, self.width, 4), dtype=np.uint8)
        self._check(self.lib.etxb_read_film_ldr(self.h, layer, C.c_float(exposure), _p(out), out.nbytes))
        return out

    def save_image(self, file_name, layer=S.FILM_RESULT, tonemapped=False, exposure=1.0):
        """RTApplication::on_save_image_selected (app.cxx:261-295): the float layer as OpenEXR, or tone-mapped as PNG."""
        self._check(self.lib.etxb_save_film(self.h, layer, os.fsencode(file_name), 1 if tonemapped else 0, C.c_float(exposure)))

    def denoise(self, layer=S.FILM_RESULT):
        """Film::denoise(layer): filters the Result or Camera layer into S.FILM_DENOISED on the device (DESIGN §13: non-local means with a
        two-half-buffer variance estimate, guided by the normal and albedo layers under the path tracer).  Needs two iterations on the film."""
        self._check(self.lib.etxb_denoise(self.h, layer))

    def counters(self):
        c = np.zeros(1, dtype=S.COUNTERS)
        self._check(self.lib.etxb_get_counters(self.h, _p(c)))
        return _fields(c)

    def kernel_times(self):
        cap = self._check(self.lib.etxb_get_kernel_times(self.h, None, None, None, 0))  # the module's number of timed kernels
        names = (C.c_char_p * cap)()
        ms = (C.c_float * cap)()
        launches = (C.c_uint32 * cap)()
        n = self._check(self.lib.etxb_get_kernel_times(self.h, names, ms, launches, cap))
        return {names[i].decode(): (float(ms[i]), int(launches[i])) for i in range(n)}

    def buffer(self, buf_id, dtype):
        n = C.c_uint64(0)
        self._check(self.lib.etxb_read_buffer(self.h, buf_id, None, 0, C.byref(n)))
        out = np.zeros(n.value // np.dtype(dtype).itemsize, dtype=dtype)
        if n.value:
            self._check(self.lib.etxb_read_buffer(self.h, buf_id, _p(out), out.nbytes, C.byref(n)))
        return out

    def stream(self):
        return self.lib.etxb_stream(self.h)

    # -- unit entry points (parity tests) -----------------------------------------------------------------
    def debug_select_tree(self, wide):
        """etxb_debug_trace / etxb_debug_occluded walk the BVH2 (False) or the product build's 4-wide quantised tree (True); returns whether that
        tree exists."""
        return self.lib.etxb_debug_select_tree(self.h, 1 if wide else 0) == 1

    def debug_build_trees(self, positions, indices, device):
        """Both trees of a triangle soup (positions float[V, 3], indices uint32[T, 3]) without committing a scene: built by the host builder
        (device=False, the specification) or on the device (device=True, what an upload runs).  Returns a dict: bvh_nodes (S.BVH_NODE),
        tri_pos (float32[3 * slots, 4]), tri_index (uint32[slots]), wide_nodes (S.WIDE_NODE), max_depth, max_stack, seconds."""
        positions = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
        indices = np.ascontiguousarray(indices, dtype=np.uint32).reshape(-1, 3)
        cap = max(1, indices.shape[0])
        nodes = np.zeros(cap, dtype=S.BVH_NODE)
        tri_pos = np.zeros((cap * 3, 4), dtype=np.float32)
        tri_index = np.zeros(cap, dtype=np.uint32)
        wide = np.zeros(cap, dtype=S.WIDE_NODE)

        class Trees(C.Structure):
            _fields_ = [("bvh_nodes", C.c_void_p), ("tri_pos", C.c_void_p), ("tri_index", C.c_void_p), ("wide_nodes", C.c_void_p),
                        ("bvh_node_count", C.c_uint32), ("slot_count", C.c_uint32), ("wide_node_count", C.c_uint32), ("max_depth", C.c_uint32),
                        ("max_stack", C.c_uint32), ("pad", C.c_uint32), ("seconds", C.c_double)]

        t = Trees(_p(nodes), _p(tri_pos), _p(tri_index), _p(wide))
        self._check(self.lib.etxb_debug_build_trees(self.h, _p(positions), positions.shape[0], _p(indices), indices.shape[0], 1 if device else 0,
                                                    C.byref(t)))
        return {"bvh_nodes": nodes[:t.bvh_node_count], "tri_pos": tri_pos[:t.slot_count * 3], "tri_index": tri_index[:t.slot_count],
                "wide_nodes": wide[:t.wide_node_count], "max_depth": int(t.max_depth), "max_stack": int(t.max_stack), "seconds": float(t.seconds)}

    def debug_trace(self, rays, seeds):
        rays = np.ascontiguousarray(rays, dtype=np.float32)
        seeds = np.ascontiguousarray(seeds, dtype=np.uint32).copy()
        n = rays.shape[0]
        uvt = np.zeros((n, 3), dtype=np.float32)
        tri = np.zeros(n, dtype=np.uint32)
        self._check(self.lib.etxb_debug_trace(self.h, _p(rays), _p(seeds), n, _p(uvt), _p(tri)))
        return uvt, tri, seeds

    def debug_occluded(self, segments):
        """segments: float32 (n, 6) rows {p0, p1}; returns a bool per segment: is a non-Void surface between p0 and p1?"""
        segments = np.ascontiguousarray(segments, dtype=np.float32)
        n = segments.shape[0]
        out = np.zeros(n, dtype=np.uint32)
        self._check(self.lib.etxb_debug_occluded(self.h, _p(segments), n, _p(out)))
        return out != 0

    def debug_denoise(self, color, camera, half, counts, normals=None, albedo=None):
        """etxb_denoise's kernels on host arrays: color / camera / half (and the optional guides) float32 (H, W, 3 or 4), counts uint32 (H, W).
        Returns (denoised float32 (H, W, 4), smoothed variance of the mean float32 (H, W, 4))."""
        def rgba(a):
            a = np.asarray(a, dtype=np.float32)
            out = np.zeros(a.shape[:2] + (4,), dtype=np.float32)
            out[..., :a.shape[2]] = a
            return np.ascontiguousarray(out)
        c, f, hh = rgba(color), rgba(camera), rgba(half)
        h, w = c.shape[:2]
        n = np.ascontiguousarray(counts, dtype=np.uint32).reshape(h, w)
        g = [rgba(x) if x is not None else None for x in (normals, albedo)]
        out = np.zeros((h, w, 4), dtype=np.float32)
        var = np.zeros((h, w, 4), dtype=np.float32)
        self._check(self.lib.etxb_debug_denoise(self.h, _p(c), _p(f), _p(hh), _p(n), _p(g[0]) if g[0] is not None else None,
                                                _p(g[1]) if g[1] is not None else None, w, h, _p(out), _p(var)))
        return out, var

    def debug_noise_estimate(self, camera, adaptive, info, threshold, world=1):
        """The path tracer's noise estimate as `world` pixel-tile ranks run it (etxb_debug_noise_estimate) on storage-order arrays: camera and
        adaptive (H, W, 4) float32, info (H, W) uint32 S.BUF_PIXEL_INFO words.  Returns (info, error level, converged count, error sum)."""
        camera = np.ascontiguousarray(camera, dtype=np.float32)
        adaptive = np.ascontiguousarray(adaptive, dtype=np.float32)
        info = np.ascontiguousarray(info, dtype=np.uint32)
        h, w = info.shape
        assert camera.shape == (h, w, 4) and adaptive.shape == (h, w, 4)
        info_out = np.zeros((h, w), dtype=np.uint32)
        error = np.zeros((h, w), dtype=np.float32)
        stats = np.zeros(2, dtype=np.uint32)
        self._check(self.lib.etxb_debug_noise_estimate(self.h, w, h, world, C.c_float(threshold), _p(camera), _p(adaptive), _p(info), _p(info_out), _p(error),
                                                       _p(stats)))
        return info_out, error, int(stats[0]), float(stats[1:2].view(np.float32)[0])

    def debug_sampler(self, a, b, draws):
        a = np.ascontiguousarray(a, dtype=np.uint32)
        b = np.ascontiguousarray(b, dtype=np.uint32)
        n = a.shape[0]
        seeds = np.zeros((n, draws + 1), dtype=np.uint32)
        vals = np.zeros((n, max(draws, 1)), dtype=np.float32)
        self._check(self.lib.etxb_debug_sampler(self.h, _p(a), _p(b), n, draws, _p(seeds), _p(vals)))
        return seeds, vals[:, :draws]

    def debug_math(self, fn, x, y=None):
        x = np.ascontiguousarray(x, dtype=np.float32)
        out = np.zeros_like(x)
        yy = np.ascontiguousarray(y, dtype=np.float32) if y is not None else None
        self._check(self.lib.etxb_debug_math(self.h, fn, _p(x), _p(yy) if yy is not None else None, x.shape[0], _p(out)))
        return out

    def debug_closure(self, queries, repetitions):
        """The vertex closures (make_closure + closure_evaluate) for S.CLOSURE_QUERY records on the uploaded scene, `repetitions` fresh
        samplers per query; returns float64 (n, S.CLOSURE_STATS), laid out as etxb_debug_closure_eval documents (include/etx_b200.h)."""
        queries = np.ascontiguousarray(queries, dtype=S.CLOSURE_QUERY)
        out = np.zeros((queries.shape[0], S.CLOSURE_STATS), dtype=np.float64)
        self._check(self.lib.etxb_debug_closure_eval(self.h, _p(queries), queries.shape[0], int(repetitions), _p(out)))
        return out

    def debug_bsdf_sample(self, queries, repetitions):
        """bsdf_sample for S.SAMPLE_QUERY records on the uploaded scene, repetition r of each on the sampler (seed, r); returns
        S.SAMPLE_RESULT records shaped (n, repetitions), laid out as etxb_debug_bsdf_sample documents (include/etx_b200.h)."""
        queries = np.ascontiguousarray(queries, dtype=S.SAMPLE_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=S.SAMPLE_RESULT)
        self._check(self.lib.etxb_debug_bsdf_sample(self.h, _p(queries), queries.shape[0], int(repetitions), _p(out)))
        return out

    def debug_emitter(self, queries, repetitions=1):
        """The emitter routines for S.EMITTER_QUERY records on the uploaded scene, repetition r of each emission query on the sampler (seed, r);
        returns S.EMITTER_RESULT records shaped (n, repetitions), laid out as etxb_debug_emitter documents (include/etx_b200.h)."""
        queries = np.ascontiguousarray(queries, dtype=S.EMITTER_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=S.EMITTER_RESULT)
        self._check(self.lib.etxb_debug_emitter(self.h, _p(queries), queries.shape[0], int(repetitions), _p(out)))
        return out

    def debug_medium(self, queries, repetitions=1):
        """The media routines for S.MEDIUM_QUERY records on the uploaded scene, repetition r of each query on the sampler (seed, r); returns
        S.MEDIUM_RESULT records shaped (n, repetitions), laid out as etxb_debug_medium documents (include/etx_b200.h)."""
        queries = np.ascontiguousarray(queries, dtype=S.MEDIUM_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=S.MEDIUM_RESULT)
        self._check(self.lib.etxb_debug_medium(self.h, _p(queries), queries.shape[0], int(repetitions), _p(out)))
        return out

    def debug_subsurface(self, queries, repetitions=1):
        """The subsurface routines for S.SUBSURFACE_QUERY records on the uploaded scene, repetition r of each query on the sampler (seed, r);
        returns S.SUBSURFACE_RESULT records shaped (n, repetitions), laid out as etxb_debug_subsurface documents (include/etx_b200.h)."""
        queries = np.ascontiguousarray(queries, dtype=S.SUBSURFACE_QUERY)
        out = np.zeros((queries.shape[0], int(repetitions)), dtype=S.SUBSURFACE_RESULT)
        self._check(self.lib.etxb_debug_subsurface(self.h, _p(queries), queries.shape[0], int(repetitions), _p(out)))
        return out

    def debug_thresholds(self, **fields):
        """The queue sizes from which the passes take their large-queue branches (etxb_debug_set_thresholds): keyword fields of
        S.DEBUG_THRESHOLDS, the others at their defaults; 0 = always, S.NEVER = never.  No argument restores the defaults."""
        unknown = set(fields) - set(S.DEFAULT_THRESHOLDS)
        if unknown:
            raise ValueError(f"unknown thresholds {sorted(unknown)}")
        t = np.zeros(1, dtype=S.DEBUG_THRESHOLDS)
        for k, v in dict(S.DEFAULT_THRESHOLDS, **fields).items():
            t[k] = v
        self._check(self.lib.etxb_debug_set_thresholds(self.h, _p(t)))

    def debug_branch_counts(self):
        """etxb_debug_get_branch_counts as a dict; `merge_qpw` maps queries per warp (1 .. 32) to gather launches."""
        c = np.zeros(1, dtype=S.DEBUG_BRANCH_COUNTS)
        self._check(self.lib.etxb_debug_get_branch_counts(self.h, _p(c)))
        out = {k: int(c[k][0]) for k in ("merge_sorts", "connect_launches", "pair_sorts", "queue_sorts")}
        out["merge_qpw"] = {q: int(n) for q, n in zip(S.MERGE_QPW, c["merge_launches"][0])}
        return out

    def debug_merge(self, records, light_wavelengths, queries):
        """The photon gather query by query (etxb_debug_merge): S.LIGHT_VERTEX_REC records, one wavelength per light path index (path_count of
        them), S.MERGE_QUERY records; returns (S.MERGE_RESULT per query, S.MERGE_GRID as a dict).  Leaves the context to etxb_begin."""
        records = np.ascontiguousarray(records, dtype=S.LIGHT_VERTEX_REC)
        wl = np.zeros(self.width * self.height, dtype=np.float32)
        wl[:len(light_wavelengths)] = light_wavelengths
        queries = np.ascontiguousarray(queries, dtype=S.MERGE_QUERY)
        out = np.zeros(queries.shape[0], dtype=S.MERGE_RESULT)
        grid = np.zeros(1, dtype=S.MERGE_GRID)
        self._check(self.lib.etxb_debug_merge(self.h, _p(records), records.shape[0], _p(wl), _p(queries), queries.shape[0], _p(out), _p(grid)))
        return out, _fields(grid)


class GPUPathTracing(GPUVCM):
    """`name()/run()/update()/stop()/status()/options` like the reference's CPUPathTracing (rt/integrators/path_tracing.cxx:122-170) on the same CUDA
    context type: one path per active pixel and iteration, normal / albedo layers, adaptive sampling (Film::estimate_noise_levels)."""

    def __init__(self, scene_data=None, flavor="fast", device=0, profile=False):
        super().__init__(scene_data, flavor=flavor, device=device, profile=profile)
        self.pt_options = S.default_pt_options()
        self._check(self.lib.etxb_set_integrator(self.h, S.INTEGRATOR_PT))

    @staticmethod
    def name():
        return "Path Tracing (B200)"

    def set_option(self, key, value):
        """The reference's option ids: "direct", "nee", "mis", "bn" (path_tracing.cxx:36-39)."""
        rc = self.lib.etxb_pt_options_set_key(_p(self.pt_options), key.encode(), float(value))
        if rc != 0:
            raise EtxbError(rc, f"unknown option key {key}")

    def set_scene_settings(self, noise_threshold, radiance_clamp=0.0):
        """Scene::noise_threshold / radiance_clamp without a new upload."""
        self._check(self.lib.etxb_set_scene_settings(self.h, C.c_float(noise_threshold), C.c_float(radiance_clamp)))

    def _push_options(self):
        """The path tracer's options, read by CPUPathTracingImpl::start (path_tracing.cxx:35-48)."""
        self._check(self.lib.etxb_pt_set_options(self.h, _p(self.pt_options)))

    def _converged(self, st):
        """CPUPathTracingImpl::update (path_tracing.cxx:85-110): an iteration that processed no pixel (all converged) ends the run.  With a
        communicator pixels_processed counts every rank's pixels, so all ranks stop at the same iteration."""
        return (st["completed_iterations"] > 0) and (self.pt_status()["pixels_processed"] == 0)

    def pt_status(self):
        """etxb_pt_get_status; over all ranks on a context with a communicator."""
        st = np.zeros(1, dtype=S.PT_STATUS)
        self._check(self.lib.etxb_pt_get_status(self.h, _p(st)))
        return _fields(st)


class GPUVCMGroup:
    """Several iterations in flight on one device (etxb_group): `lanes` contexts, one host thread each inside the module, each popping
    iteration indices from its lane's queue, which enqueue fills (on one GPU all lanes share one queue, so a free lane takes the next index).
    Same Integrator-style surface as GPUVCM: run / enqueue / wait / status / film."""

    def __init__(self, scene_data, lanes=4, flavor="fast", device=0, max_light_vertices=0, profile=False):
        self.lib = load_library(flavor)
        self.h = C.c_void_p()
        rc = self.lib.etxb_group_create(C.byref(self.h), _p(_device_config(device, max_light_vertices, profile)), lanes)
        if rc != 0:
            raise EtxbError(rc, "etxb_group_create failed (no CUDA device? the module has no CPU fallback)")
        self.lanes = [GPUVCM(scene_data, flavor=flavor, _adopt=self.lib.etxb_group_lane(self.h, k)) for k in range(lanes)]
        self.options = self.lanes[0].options
        self.scene_data = scene_data
        self.width, self.height = self.lanes[0].width, self.lanes[0].height

    def _check(self, rc):
        if rc < 0:
            raise EtxbError(rc, self.lib.etxb_group_last_error(self.h).decode() or self.lib.etxb_last_error(self.lanes[0].h).decode())
        return rc

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            for g in self.lanes:
                g.close()
            self.lib.etxb_group_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_integrator(self, integrator, pt_options=None):
        """Every lane renders with the VCM (default) or the path-tracing algorithm.  With iterations in flight each lane keeps its own film and per-pixel
        history, so the path tracer's adaptive sampling is switched off here (noise threshold 0: every pixel gets one sample per iteration, like the
        reference with `noise_threshold 0`); the combined film is the mean over the iterations of all lanes.  A group in pixel-tile mode
        (comm_init with world >= 2) refuses the path tracer."""
        for g in self.lanes:
            g._check(self.lib.etxb_set_integrator(g.h, integrator))
            if integrator == S.INTEGRATOR_PT:
                g._check(self.lib.etxb_pt_set_options(g.h, _p(pt_options if pt_options is not None else S.default_pt_options())))
                g._check(self.lib.etxb_set_scene_settings(g.h, C.c_float(0.0), C.c_float(float(self.scene_data.scene["radiance_clamp"][0]))))

    def set_film_pixel_size(self, size):
        """GPUVCM.set_film_pixel_size for every lane (etxb_group_set_film_pixel_size): applied by the next run() or update_scene()."""
        self._check(self.lib.etxb_group_set_film_pixel_size(self.h, size))

    def set_options(self):
        """Pushes self.options (the Integrator options) to every lane."""
        for g in self.lanes:
            g._check(self.lib.etxb_set_options(g.h, _p(self.options)))

    def run(self, first_iteration=0):
        self.set_options()
        self._check(self.lib.etxb_group_begin(self.h, first_iteration))

    def update_scene(self, scene_data):
        """GPUVCM.update_scene for every lane (etxb_group_update_scene): hashed once, then the group is idle and armed at iteration 0.  Returns
        lane 0's etxb_update_info fields, `kept` being what every lane kept."""
        info = np.zeros(1, dtype=S.UPDATE_INFO)
        self._check(self.lib.etxb_group_update_scene(self.h, _p(scene_data.scene), scene_data.scene.nbytes, _p(scene_data.camera), scene_data.camera.nbytes,
                                                     _p(info)))
        for g in self.lanes:
            g._after_update(scene_data)
        self.scene_data = scene_data
        self.width, self.height = self.lanes[0].width, self.lanes[0].height
        return _fields(info)

    def comm_init(self, world, rank, comm_ids):
        """Pixel tiles over `world` processes with len(self.lanes) iterations in flight on each: collective; comm_ids = the (lanes + 1) x 128
        bytes rank 0 got from comm_unique_ids(lanes + 1)."""
        comm_ids = np.ascontiguousarray(comm_ids, dtype=np.uint8)
        self._check(self.lib.etxb_group_comm_init(self.h, world, rank, _p(comm_ids), comm_ids.nbytes // COMM_ID_BYTES))
        self.comm_rank, self.comm_world = rank, world

    def comm_init_replicas(self, world, rank, comm_id, split_lane=False):
        """Whole-frame iterations dealt to `world` processes (the job's j-th iteration on rank j % world); enqueue(n) then counts iterations of
        the job.  Collective; comm_id = the 128 bytes rank 0 got from comm_unique_ids(1).  split_lane: reserve the last lane for camera-split
        iterations (the remainder of an enqueue that is not a multiple of `world`)."""
        if split_lane:
            self._check(self.lib.etxb_group_reserve_split_lane(self.h))
        comm_id = np.ascontiguousarray(comm_id, dtype=np.uint8)
        self._check(self.lib.etxb_group_comm_init_replicas(self.h, world, rank, _p(comm_id), comm_id.nbytes))
        self.comm_rank, self.comm_world = rank, world

    def comm_reduce_film(self, layer=S.FILM_RESULT, out=None):
        """Collective: the whole frame (mean over the iterations finished so far) on rank 0; None elsewhere."""
        rank = getattr(self, "comm_rank", 0)
        if (out is None) and (rank == 0):
            out = np.zeros((self.height, self.width, 4), dtype=np.float32)
        self._check(self.lib.etxb_group_comm_reduce_film(self.h, layer, _p(out) if rank == 0 else None, out.nbytes if rank == 0 else 0))
        return out if rank == 0 else None

    def enqueue(self, iterations=1):
        self._check(self.lib.etxb_group_enqueue(self.h, iterations))

    def wait(self):
        self._check(self.lib.etxb_group_wait(self.h))

    def render(self, iterations, first_iteration=0):
        self.run(first_iteration)
        self.enqueue(iterations)
        self.wait()
        return self.status()

    def status(self):
        st = np.zeros(1, dtype=S.STATUS)
        self._check(self.lib.etxb_group_poll(self.h, _p(st)))
        return _fields(st)

    def film(self, layer=S.FILM_RESULT, out=None):
        if out is None:
            out = np.zeros((self.height, self.width, 4), dtype=np.float32)
        self._check(self.lib.etxb_group_read_film(self.h, layer, _p(out), out.nbytes))
        return out

    def counters(self):
        total = {}
        for g in self.lanes:
            for k, v in g.counters().items():
                total[k] = total.get(k, 0) + v
        return total

    def kernel_times(self):
        total = {}
        for g in self.lanes:
            for k, (ms, n) in g.kernel_times().items():
                a = total.get(k, (0.0, 0))
                total[k] = (a[0] + ms, a[1] + n)
        return total
