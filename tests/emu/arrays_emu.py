"""ctypes front end of tests/emu/libmeao_emu_arrays.so -- one CUDA-ARRAY frame (meao_render_arrays) through the host-compiled array
kernel sources, with the depth and the AO in emulated 2-D / layered / cube-map arrays.  TEST INFRASTRUCTURE ONLY (see cuda_emu.h)."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_arrays_emu  # noqa: E402
from layered_emu import LayeredFrame  # noqa: E402

SHAPES = {"2d": 0, "layered": 1, "cube": 2}
_lib: C.CDLL | None = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        l = C.CDLL(build_arrays_emu.build())
        l.lemu_create.restype = C.c_void_p
        l.lemu_create.argtypes = [C.c_int, C.c_int, C.c_int]
        l.lemu_destroy.argtypes = [C.c_void_p]
        l.lemu_set_constants.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float] + [C.c_int] * 6
        l.lemu_get_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        l.lemu_tma_box_loads.restype = C.c_longlong
        l.aemu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_int, C.c_longlong]
        l.aemu_surface_accesses.restype = C.c_longlong
        _lib = l
    return _lib


class ArrayFrame(LayeredFrame):
    """LayeredFrame's arena and constants in the array library; run() takes the depth as an emulated array and returns the AO array."""

    def __init__(self, plan, *, linear: bool = False, use_tma: bool = True):
        import layered_emu
        saved, layered_emu._lib = layered_emu._lib, lib()      # the base class builds its arena through layered_emu.lib()
        try:
            super().__init__(plan, linear=linear, use_tma=use_tma)
        finally:
            layered_emu._lib = saved

    def surface_accesses(self) -> int:
        return int(self._lib.aemu_surface_accesses())

    def run_arrays(self, depth: np.ndarray, depth_shape: str = "2d", ao_shape: str | None = None, pad: int = 24) -> np.ndarray:
        """depth [layers, H, W] (float32 / uint16 D16 codes).  Each array gets rows `pad` elements wider than W, and its bytes outside
        the image are filled with a marker that must survive.  Returns the AO [layers, H, W]."""
        fmt = {"float32": 0, "uint16": 1}[depth.dtype.name]
        L, H, W = depth.shape
        assert (L, H, W) == (self.layers, self.H, self.W)
        d = np.full((L, H, W + pad), 7, depth.dtype)
        d[:, :, :W] = depth
        ao = np.full((L, H, W + pad), 0xA5, np.uint8)
        ao_shape = ao_shape or depth_shape
        self._lib.aemu_run(self._h, d.ctypes.data, fmt, SHAPES[depth_shape], d.strides[1], ao.ctypes.data, SHAPES[ao_shape], ao.strides[1])
        assert (ao[:, :, W:] == 0xA5).all(), "a store outside the image"
        return ao[:, :, :W].copy()
