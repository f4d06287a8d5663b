"""ctypes front end of tests/emu/libmeao_emu.so -- the kernel SOURCES of miniengineao_b200/csrc compiled for the host.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h): used by the CPU test-suite to check the kernels' logic against the oracle
without a GPU.  Nothing outside tests/ may import this; libmeao.so never links or loads it.
"""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_emu  # noqa: E402

_lib: C.CDLL | None = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        l = C.CDLL(build_emu.build())
        l.emu_create.restype = C.c_void_p
        l.emu_create.argtypes = [C.c_int, C.c_int]
        l.emu_destroy.argtypes = [C.c_void_p]
        l.emu_set_constants.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int]
        l.emu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        l.emu_set_tma.argtypes = [C.c_void_p, C.c_int]
        l.emu_tma_box_loads.restype = C.c_longlong
        l.emu_set_band.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        l.emu_poison_low.argtypes = [C.c_void_p]
        l.emu_band_phase_a.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        l.emu_halo.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        l.emu_band_phase_b.argtypes = [C.c_void_p]
        l.emu_get_buffer.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        l.emu_debug_view.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        l.emu_set_render_tile.argtypes = [C.c_void_p, C.c_int]
        l.emu_set_single_scale.argtypes = [C.c_void_p, C.c_int]
        l.emu_band_exchange.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        l.emu_band_flags.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        l.emu_composite.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int]
        l.emu_composite_debug.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int]
        _lib = l
    return _lib


def _aligned(a: np.ndarray) -> np.ndarray:
    """16-byte aligned C-contiguous copy (the kernels use 128-bit loads on the input)."""
    raw = np.empty(a.nbytes + 64, np.uint8)
    off = (-raw.ctypes.data) % 64
    out = raw[off:off + a.nbytes].view(a.dtype).reshape(a.shape)
    out[...] = a
    return out


def linearize_zero(zb) -> float:
    """Linearize(0) of a standard-Z camera, the value of the padding texels (DS1:40): 1 / fma(zbx, 0, zby), as libmeao forms it --
    NaN when zbx is infinite (far / near overflowed f32), not 1 / zby."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.float32(1) / (np.float32(zb[0]) * np.float32(0) + np.float32(zb[1])))


class EmulatedFrame:
    """One frame through the host-compiled kernels, planned by a plan-only libmeao context (device = -1)."""

    def __init__(self, plan, *, linear: bool = False, use_tma: bool = True, render_tile: int = -1):
        """plan: miniengineao_b200.AmbientOcclusion(camera, device=-1) with parameters / variants already set.
        use_tma: interior tiles take the kernels' TMA path (emulated box loads) -- what runs on the GPU; False forces the
        gather path everywhere (libmeao's MEAO_DISABLE_TMA=1)."""
        from miniengineao_b200 import _native as N
        self._lib = lib()
        plan.LateUpdate()
        self.plan = plan
        self.W, self.H = plan._width, plan._height
        nl = N.lib()
        rc, rcw, uc = (C.c_float * 112)(), (C.c_float * 112)(), (C.c_float * 32)()
        zb = (C.c_float * 4)()
        for k in range(1, 5):
            N.check(plan._ctx, nl.meao_render_constants(plan._ctx, k, C.cast(C.byref(rc, 112 * (k - 1)), C.POINTER(C.c_float))))
            N.check(plan._ctx, nl.meao_render_constants_wide(plan._ctx, k, C.cast(C.byref(rcw, 112 * (k - 1)), C.POINTER(C.c_float))))
            N.check(plan._ctx, nl.meao_upsample_constants(plan._ctx, k, C.cast(C.byref(uc, 32 * (k - 1)), C.POINTER(C.c_float))))
        N.check(plan._ctx, nl.meao_zbuffer_params(plan._ctx, zb))
        rz = bool(plan.camera.usesReversedZBuffer)
        if linear:
            pad12 = 0.0
        else:       # Linearize(OOB load = 0): DS1:40-45
            pad12 = 1e5 if rz else linearize_zero(zb)
        self._h = self._lib.emu_create(self.W, self.H)
        self._lib.emu_set_tma(self._h, int(use_tma))
        self._lib.emu_set_render_tile(self._h, int(render_tile))       # -1: the planner's rule; 0 / 1 / 2: force 64x32 / 64x16 / 64x8 tiles
        self._lib.emu_set_single_scale(self._h, int(getattr(plan, "singleScale", False)))
        self._lib.emu_set_constants(self._h, rc, rcw, uc, zb, pad12, int(not linear), int(rz), int(plan.highQualityMask), int(plan.sampleExhaustively))

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.emu_destroy(self._h)
            self._h = None

    def run(self, depth: np.ndarray) -> np.ndarray:
        fmt = {"float32": 0, "uint16": 1, "uint32": 2}[depth.dtype.name]
        d = _aligned(np.ascontiguousarray(depth))
        assert d.shape == (self.H, self.W)
        self._lib.emu_run(self._h, d.ctypes.data, fmt)
        return self.buffer(17)

    # ---- row bands: the plan must already carry the band (plan.set_row_band) -----------------------------------------
    def use_plan_band(self) -> None:
        rows = self.plan.band_rows()
        prod = (C.c_int * 10)(*[v for lohi in rows["produce"] for v in lohi])
        self.band = rows["produce"][0]
        self._lib.emu_set_band(self._h, self.band[0], self.band[1], prod)
        self._lib.emu_poison_low(self._h)

    def band_phase_a(self, depth_band: np.ndarray) -> None:
        d = _aligned(np.ascontiguousarray(depth_band, np.float32))
        assert d.shape == (self.band[1] - self.band[0], self.W)
        self._lib.emu_band_phase_a(self._h, d.ctypes.data, 0)

    def halo_pack(self, side: int) -> np.ndarray:
        rows = self.plan.halo_rows(side, True)
        buf = _aligned(np.zeros(max(self.plan.halo_bytes(side) // 4, 1), np.float32))
        self._lib.emu_halo(self._h, (C.c_int * 8)(*[v for lohi in rows for v in lohi]), buf.ctypes.data, 1)
        return buf[:self.plan.halo_bytes(side) // 4]

    def halo_unpack(self, side: int, packed: np.ndarray) -> None:
        rows = self.plan.halo_rows(side, False)
        buf = _aligned(np.ascontiguousarray(packed, np.float32)) if packed.size else _aligned(np.zeros(1, np.float32))
        assert packed.size * 4 == self.plan.halo_recv_bytes(side)
        self._lib.emu_halo(self._h, (C.c_int * 8)(*[v for lohi in rows for v in lohi]), buf.ctypes.data, 0)

    # ---- native neighbour exchange (band_exchange.cu): peers are other EmulatedFrame objects of the same frame size ---------
    def exchange(self, up=None, down=None, timeout_polls: int = 1000) -> int:
        """Runs band_exchange_kernel for this band: pushes its border rows straight into the neighbours' LowDepth buffers and
        handshakes through the epoch flags.  Returns the sticky error (0 = ok)."""
        ru = (C.c_int * 8)(*[v for lohi in self.plan.halo_rows(0, True) for v in lohi])
        rd = (C.c_int * 8)(*[v for lohi in self.plan.halo_rows(1, True) for v in lohi])
        return int(self._lib.emu_band_exchange(self._h, up._h if up is not None else None, down._h if down is not None else None, ru, rd, timeout_polls))

    def flags(self, set_ready_ack=None) -> dict:
        out = (C.c_int * 8)()
        arr = (C.c_int * 4)(*set_ready_ack) if set_ready_ack is not None else None
        self._lib.emu_band_flags(self._h, arr, out)
        return {"ready": (out[0], out[1]), "ack": (out[2], out[3]), "epoch": out[4], "done": out[5], "error": out[6], "host_error": out[7]}

    def band_phase_b(self) -> np.ndarray:
        """-> the band's rows of the AO texture"""
        self._lib.emu_band_phase_b(self._h)
        return self.buffer(17)[self.band[0]:self.band[1]]

    def tma_box_loads(self) -> int:
        """Emulated TMA box loads issued by this library instance so far (process-wide counter)."""
        return int(self._lib.emu_tma_box_loads())

    def buffer(self, bid: int) -> np.ndarray:
        d = self.plan.buffer_desc(bid)
        dt = {1: np.uint8, 2: np.float16, 4: np.float32}[d.elem_bytes]
        shape = (d.slices, d.height, d.width) if d.slices > 1 else (d.height, d.width)
        out = np.zeros(shape, dt)
        assert self._lib.emu_get_buffer(self._h, bid, out.ctypes.data) == 0
        return out

    def debug_view(self, bid: int) -> np.ndarray:
        out = np.zeros((self.H, self.W), np.uint8)
        assert self._lib.emu_debug_view(self._h, bid, out.ctypes.data) == 0
        return out


def composite(ao: np.ndarray, color: np.ndarray, *, rgb: bool, alpha: bool, one_minus: bool) -> np.ndarray:
    out = _aligned(np.ascontiguousarray(color))
    a = _aligned(np.ascontiguousarray(ao, np.uint8))
    lib().emu_composite(a.ctypes.data, out.ctypes.data, a.size, int(out.dtype == np.float16), int(rgb), int(alpha), int(one_minus))
    return out.copy()


def composite_debug(view: np.ndarray, like: np.ndarray) -> np.ndarray:
    v = _aligned(np.ascontiguousarray(view, np.uint8))
    out = _aligned(np.zeros(v.shape + (4,), like.dtype))
    lib().emu_composite_debug(v.ctypes.data, out.ctypes.data, v.size, int(out.dtype == np.float16))
    return out.copy()
