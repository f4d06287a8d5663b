"""ctypes front end of tests/emu/libmeao_emu_layered.so -- one LAYERED frame (meao_set_layers) through the host-compiled layered
kernel sources.  TEST INFRASTRUCTURE ONLY (see cuda_emu.h); the layered twin of emu.EmulatedFrame."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_layered_emu  # noqa: E402
from emu.emu import linearize_zero  # noqa: E402

_lib: C.CDLL | None = None


def _aligned(a: np.ndarray) -> np.ndarray:
    """16-byte aligned C-contiguous copy (the kernels use 128-bit loads on the input)."""
    raw = np.empty(a.nbytes + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    out = raw[off:off + a.nbytes].view(a.dtype).reshape(a.shape)
    out[...] = a
    return out


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        l = C.CDLL(build_layered_emu.build())
        l.lemu_create.restype = C.c_void_p
        l.lemu_create.argtypes = [C.c_int, C.c_int, C.c_int]
        l.lemu_destroy.argtypes = [C.c_void_p]
        l.lemu_set_constants.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float] + [C.c_int] * 6
        l.lemu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        l.lemu_get_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        l.lemu_tma_box_loads.restype = C.c_longlong
        _lib = l
    return _lib



class LayeredFrame:
    """One layered frame through the host-compiled layered kernels, planned by a plan-only libmeao context (device = -1) whose
    `layers` property gives the layer count."""

    def __init__(self, plan, *, linear: bool = False, use_tma: bool = True):
        """use_tma: interior tiles take the kernels' TMA path (emulated box loads); False forces the gather path everywhere."""
        from miniengineao_b200 import _native as N
        self._lib = lib()
        plan.LateUpdate()
        self.plan = plan
        self.W, self.H, self.layers = plan._width, plan._height, int(plan.layers)
        nl = N.lib()
        rc, rcw, uc = (C.c_float * 112)(), (C.c_float * 112)(), (C.c_float * 32)()
        zb = (C.c_float * 4)()
        for k in range(1, 5):
            N.check(plan._ctx, nl.meao_render_constants(plan._ctx, k, C.cast(C.byref(rc, 112 * (k - 1)), C.POINTER(C.c_float))))
            N.check(plan._ctx, nl.meao_render_constants_wide(plan._ctx, k, C.cast(C.byref(rcw, 112 * (k - 1)), C.POINTER(C.c_float))))
            N.check(plan._ctx, nl.meao_upsample_constants(plan._ctx, k, C.cast(C.byref(uc, 32 * (k - 1)), C.POINTER(C.c_float))))
        N.check(plan._ctx, nl.meao_zbuffer_params(plan._ctx, zb))
        rz = bool(plan.camera.usesReversedZBuffer)
        pad12 = 0.0 if linear else (1e5 if rz else linearize_zero(zb))     # Linearize(OOB load = 0): DS1:40-45
        self._h = self._lib.lemu_create(self.W, self.H, self.layers)
        self._lib.lemu_set_constants(self._h, rc, rcw, uc, zb, pad12, int(not linear), int(rz), int(plan.highQualityMask),
                                     int(plan.sampleExhaustively), int(plan.singleScale), int(use_tma))

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.lemu_destroy(self._h)
            self._h = None

    def run(self, depth: np.ndarray) -> None:
        """depth [layers, H, W] (float32 / uint16 D16 codes / uint32 D24S8 words), stacked at a stride of one image."""
        fmt = {"float32": 0, "uint16": 1, "uint32": 2}[depth.dtype.name]
        d = _aligned(np.ascontiguousarray(depth))
        assert d.shape == (self.layers, self.H, self.W)
        self._lib.lemu_run(self._h, d.ctypes.data, fmt)

    def tma_box_loads(self) -> int:
        """Emulated TMA box loads issued by this library instance so far (process-wide counter)."""
        return int(self._lib.lemu_tma_box_loads())

    def buffer(self, bid: int, layer: int) -> np.ndarray:
        d = self.plan.buffer_desc(bid)
        dt = {1: np.uint8, 2: np.float16, 4: np.float32}[d.elem_bytes]
        shape = (d.slices, d.height, d.width) if d.slices > 1 else (d.height, d.width)
        out = np.zeros(shape, dt)
        assert self._lib.lemu_get_buffer(self._h, bid, layer, out.ctypes.data) == 0
        return out
