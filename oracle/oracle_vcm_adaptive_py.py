"""ctypes binding of the oracle with the VCM's CameraAdaptive layer (oracle/_ref/liboracle_vcm_adaptive_parity.so, built from
oracle_vcm_adaptive.cxx).  TEST INFRASTRUCTURE.

The library is the coarse-preview oracle (oracle_preview.cxx) whose VCM iterations also keep Film's CameraAdaptive layer (film.cxx:173-230).
"""
import ctypes as C

from oracle import oracle_py

FLAVOR = "vcm_adaptive_parity"


def available():
    return oracle_py.available(FLAVOR)


def _lib():
    lib = oracle_py.load(FLAVOR)
    if not getattr(lib, "_adaptive_bound", False):
        lib.oracle_set_film_pixel_size.argtypes = [C.c_void_p, C.c_uint32]
        lib.oracle_adaptive_run_iterations.restype = C.c_double
        lib.oracle_adaptive_run_iterations.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        lib._adaptive_bound = True
    return lib


class Oracle(oracle_py.Oracle):
    """oracle_py.Oracle with the Film pixel size, whose VCM iterations keep the CameraAdaptive layer."""

    def __init__(self, scene_data):
        _lib()
        super().__init__(scene_data, flavor=FLAVOR)

    def set_film_pixel_size(self, size):
        """Film::set_pixel_size: clamped to [1, 1024], applied by the next begin()."""
        self.lib.oracle_set_film_pixel_size(self.h, size)

    def run(self, iterations, threads=1):
        return self.lib.oracle_adaptive_run_iterations(self.h, iterations, threads)
