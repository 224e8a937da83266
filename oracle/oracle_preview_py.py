"""ctypes binding of the coarse-preview oracle (oracle/_ref/liboracle_preview_parity.so, built from oracle_preview.cxx).  TEST INFRASTRUCTURE.

The library is the parity oracle with Film::set_pixel_size added; at pixel size 1 it runs oracle_vcm.cxx's own code.
"""
import ctypes as C

import numpy as np

from oracle import oracle_py

FLAVOR = "preview_parity"


def available():
    return oracle_py.available(FLAVOR)


def _lib():
    lib = oracle_py.load(FLAVOR)
    if not getattr(lib, "_preview_bound", False):
        lib.oracle_set_film_pixel_size.argtypes = [C.c_void_p, C.c_uint32]
        lib.oracle_preview_offset.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        lib._preview_bound = True
    return lib


class Oracle(oracle_py.Oracle):
    """oracle_py.Oracle with the Film pixel size."""

    def __init__(self, scene_data):
        _lib()
        super().__init__(scene_data, flavor=FLAVOR)

    def set_film_pixel_size(self, size):
        """Film::set_pixel_size: clamped to [1, 1024], applied by the next begin()."""
        self.lib.oracle_set_film_pixel_size(self.h, size)


def preview_offset(index, iteration, size):
    """pm::preview_offset (etx_tracer_b200/csrc/portable_math.h) for arrays of path indices and iterations: (dx, dy) inside the size x size block."""
    lib = _lib()
    index = np.ascontiguousarray(index, dtype=np.uint32)
    iteration = np.ascontiguousarray(np.broadcast_to(np.asarray(iteration, dtype=np.uint32), index.shape))
    dx, dy = np.zeros_like(index), np.zeros_like(index)
    lib.oracle_preview_offset(index.ctypes.data_as(C.c_void_p), iteration.ctypes.data_as(C.c_void_p), index.size, size,
                              dx.ctypes.data_as(C.c_void_p), dy.ctypes.data_as(C.c_void_p))
    return dx, dy
