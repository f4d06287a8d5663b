"""ctypes front end of tests/emu/libmeao_emu.so -- the kernel SOURCES of miniengineao_b200/csrc compiled for the host.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h): used by the CPU test-suite to check the kernels' logic against the oracle
without a GPU.  Nothing outside tests/ may import this; libmeao.so never links or loads it.
"""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_emu  # noqa: E402

_lib: C.CDLL | None = None

KINDS = {"float32": 0, "uint16": 2, "uint32": 3}        # MEAO_DEPTH_RAW_F32 / _RAW_D16_UNORM / _RAW_D24S8 (a float32 linear frame: 1)
SHAPES = {"2d": 0, "layered": 1, "cube": 2}


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        l = C.CDLL(build_emu.build())
        P, I, LL = C.c_void_p, C.c_int, C.c_longlong
        l.frame_create.restype = P
        l.frame_create.argtypes = [I, I, I]
        l.frame_destroy.argtypes = [P]
        l.frame_arena_bytes.restype = C.c_size_t
        l.frame_arena_bytes.argtypes = [P]
        l.frame_resize.argtypes = [P, I, I]
        l.frame_set_plan.argtypes = [P, P, P, P, P, P] + [I] * 6
        l.frame_null_tables.argtypes = [P]
        l.frame_zero_pitches.argtypes = [P, I]
        l.frame_run.argtypes = [P, P, I, I, LL, LL, P, LL, LL, I, I]
        l.frame_prepare_low.argtypes = [P, P, I]
        l.frame_run_arrays.argtypes = [P, P, I, I, LL, P, I, LL]
        l.frame_set_band.argtypes = [P, I, I, P]
        l.frame_band_phase_a.argtypes = [P, P, I]
        l.frame_band_phase_b.argtypes = [P]
        l.frame_halo.argtypes = [P, P, P, I]
        l.frame_band_exchange.argtypes = [P, P, P, P, P, I]
        l.frame_band_flags.argtypes = [P, P, P]
        l.frame_poison.argtypes = [P, I]
        l.frame_get_buffer.argtypes = [P, I, I, P]
        l.frame_debug_view.argtypes = [P, I, P]
        l.frame_composite.argtypes = [P, P, LL, I, I, I, I]
        l.frame_composite_debug.argtypes = [P, P, LL, I]
        l.frame_schedule_export.argtypes = [P, P, P, I]
        l.frame_kernel_units.argtypes = [P, P, I]
        l.frame_tma_box_loads.restype = LL
        l.frame_surface_accesses.restype = LL
        l.frame_ledger_read.argtypes = [P, P, P, P, I]
        _lib = l
    return _lib


def _aligned(a: np.ndarray, offset: int = 0) -> np.ndarray:
    """C-contiguous copy `offset` bytes past a 64-byte boundary (the kernels use 128-bit loads on the input; offset 4: a depth
    pointer that is not 16-byte aligned)."""
    raw = np.empty(a.nbytes + 128, np.uint8)
    off = (-raw.ctypes.data) % 64 + offset
    out = raw[off:off + a.nbytes].view(a.dtype).reshape(a.shape)
    out[...] = a
    return out


def linearize_zero(zb) -> float:
    """Linearize(0) of a standard-Z camera, the value of the padding texels (DS1:40): 1 / fma(zbx, 0, zby), as libmeao forms it --
    NaN when zbx is infinite (far / near overflowed f32), not 1 / zby."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.float32(1) / (np.float32(zb[0]) * np.float32(0) + np.float32(zb[1])))


class Frame:
    """Frames through the host-compiled kernels, launched as libmeao launches them (csrc/frame_record.h), with the plan of a plan-only
    libmeao context (device = -1) whose parameters, variants, layers and cameras are already set."""

    def __init__(self, plan, *, linear: bool = False, use_tma: bool = True, render_tile: int = -1, max_size=None,
                 null_tables: bool = False):
        """linear: float32 depth is already linear (MEAO_DEPTH_LINEAR_F32).  use_tma: interior tiles take the kernels' TMA path
        (emulated box loads) -- what runs on the GPU; False forces the gather path everywhere (libmeao's MEAO_DISABLE_TMA=1).
        render_tile: -1 the planner's rule; 0 / 1 / 2 force 64x32 / 64x16 / 64x8 render tiles.  max_size: (W, H) the arena is laid
        out for (meao_reserve; default: the plan's size).  null_tables: pin the layered kernels' path without camera tables."""
        self._lib = lib()
        self.linear, self.use_tma, self.render_tile, self.null_tables = linear, use_tma, render_tile, null_tables
        plan.LateUpdate()
        self.layers = int(plan.layers)
        self._h = self._lib.frame_create(*(max_size or (plan._width, plan._height)), self.layers)
        self._load(plan)

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.frame_destroy(self._h)
            self._h = None

    def load(self, plan) -> None:
        """Places the buffers of the plan's size in the arena and takes its constants, each layer's from the per-layer getters."""
        plan.LateUpdate()
        self._load(plan)

    def _load(self, plan) -> None:
        from miniengineao_b200 import _native as N
        self.plan, self.W, self.H = plan, plan._width, plan._height
        self._ao = None             # the caller's AO of the last run_fused, if it had none of its own
        assert int(plan.layers) == self.layers and self._lib.frame_resize(self._h, self.W, self.H) == 0
        nl, ctx, L = N.lib(), plan._ctx, self.layers
        rc, rcw, uc, zb, pad = (C.c_float * (112 * L))(), (C.c_float * (112 * L))(), (C.c_float * 32)(), (C.c_float * (4 * L))(), (C.c_float * L)()
        at = lambda buf, n: C.cast(C.byref(buf, 4 * n), C.POINTER(C.c_float))
        rz = bool(plan.camera.usesReversedZBuffer)
        for l in range(L):
            for k in range(1, 5):
                N.check(ctx, nl.meao_render_constants_layer(ctx, l, k, 0, at(rc, 28 * (4 * l + k - 1))))
                N.check(ctx, nl.meao_render_constants_layer(ctx, l, k, 1, at(rcw, 28 * (4 * l + k - 1))))
            N.check(ctx, nl.meao_zbuffer_params_layer(ctx, l, at(zb, 4 * l)))
            pad[l] = 1e5 if rz else linearize_zero(zb[4 * l:4 * l + 2])      # Linearize(OOB load = 0): DS1:40-45
        for k in range(1, 5):
            N.check(ctx, nl.meao_upsample_constants(ctx, k, at(uc, 8 * (k - 1))))
        self.zb = np.array(zb[:2])
        self._lib.frame_set_plan(self._h, rc, rcw, uc, zb, pad, int(rz), int(plan.highQualityMask), int(plan.sampleExhaustively),
                                 int(getattr(plan, "singleScale", False)), int(self.use_tma), int(self.render_tile))
        if self.null_tables:
            self._lib.frame_null_tables(self._h)

    def _kind(self, depth) -> int:
        return 1 if self.linear and depth.dtype == np.float32 else KINDS[depth.dtype.name]

    def _counted(self, run) -> None:
        n0 = self.tma_box_loads()
        run()
        self.tma_loads_in_run = self.tma_box_loads() - n0

    def _shape(self, depth) -> tuple:
        return (self.H, self.W) if self.layers == 1 and depth.ndim == 2 else (self.layers, self.H, self.W)

    # ---- frame forms ---------------------------------------------------------------------------------------------------------
    def run(self, depth: np.ndarray) -> np.ndarray:
        """prepare_depth -> LinearDepth -> the final upsample (the stage API's frame).  depth [H, W] or [layers, H, W] (float32 /
        uint16 D16 codes / uint32 D24S8 words).  Returns the AO of layer 0."""
        self._ao = None
        d = _aligned(np.ascontiguousarray(depth))
        assert d.shape == self._shape(d)
        self._counted(lambda: self._lib.frame_run(self._h, d.ctypes.data, self._kind(d), 0, 0, 0, None, 0, 0, 0, 0))
        return self.buffer(17)

    def run_fused(self, depth, *, offset=0, rows=(0, 0), depth_row=0, depth_layer=0, ao=None, ao_row=0, ao_layer=0) -> None:
        """The frame meao_render records: low-only prepare_depth and the final upsample that reads and linearises the raw depth.
        offset: the depth copy starts this many bytes past a 64-byte boundary.  rows = (row0, row1), row1 > row0: only the final
        level's rows [row0, row1) take the fused kernel (see frame_run).  depth_row != 0: `depth` is a flat aligned buffer holding the
        frame at these ELEMENT pitches, and `ao` a flat uint8 buffer holding the AO at these byte pitches.  Without `ao` the AO goes
        to a tight [layers, H, W] array of the caller's, as meao_render stores it, and buffer(17) returns that array."""
        if ao is None and not depth_row:
            self._ao = _aligned(np.zeros((self.layers, self.H, self.W), np.uint8))
            ao = self._ao.reshape(-1)[rows[0] * self.W:]
        if depth_row:
            es = depth.itemsize
            d, p = depth, (depth_row * es, depth_layer * es, ao_row, ao_layer)
        else:
            d, p = _aligned(np.ascontiguousarray(depth), offset), (0, 0, 0, 0)
            assert d.shape == self._shape(d)
        self._keep = (d, ao)
        self._counted(lambda: self._lib.frame_run(self._h, d.ctypes.data, self._kind(d), 1, p[0], p[1], None if ao is None else ao.ctypes.data,
                                                  p[2], p[3], rows[0], rows[1]))

    def run_pitched(self, dv, av, rows=(0, 0), zero=False) -> None:
        """The fused frame from the depth view `dv` into the AO view `av` (objects with .ptr, .row, .layer byte pitches and .arr).
        zero: the tight views with zero pitches in the argument blocks (the launchers' "zero means tight")."""
        self._ao = None
        self._lib.frame_zero_pitches(self._h, int(zero))
        p = (0, 0, 0, 0) if zero else (dv.row, dv.layer, av.row, av.layer)
        self._lib.frame_run(self._h, dv.ptr, self._kind(dv.arr), 1, p[0], p[1], av.ptr, p[2], p[3], rows[0], rows[1])
        self._lib.frame_zero_pitches(self._h, 0)

    def run_arrays(self, depth: np.ndarray, depth_shape: str = "2d", ao_shape: str | None = None, pad: int = 24) -> np.ndarray:
        """A CUDA-array frame.  depth [layers, H, W] (float32 / uint16 D16 codes).  Each array gets rows `pad` elements wider than W,
        and its bytes outside the image are filled with a marker that must survive.  Returns the AO [layers, H, W]."""
        self._ao = None
        L, H, W = depth.shape
        assert (L, H, W) == (self.layers, self.H, self.W)
        d = np.full((L, H, W + pad), 7, depth.dtype)
        d[:, :, :W] = depth
        ao = np.full((L, H, W + pad), 0xA5, np.uint8)
        ao_shape = ao_shape or depth_shape
        self._lib.frame_run_arrays(self._h, d.ctypes.data, self._kind(d), SHAPES[depth_shape], d.strides[1], ao.ctypes.data, SHAPES[ao_shape],
                                   ao.strides[1])
        assert (ao[:, :, W:] == 0xA5).all(), "a store outside the image"
        return ao[:, :, :W].copy()

    def prepare_low(self, depth) -> None:
        """The low-only prepare_depth alone."""
        self._ao = None
        d = _aligned(np.ascontiguousarray(depth))
        self._lib.frame_prepare_low(self._h, d.ctypes.data, self._kind(d))

    # ---- poison and fill -------------------------------------------------------------------------------------------------------
    def fill(self) -> None:
        """Every image byte of the arena := 0xFF (NaN in every f16 / f32)."""
        self._lib.frame_poison(self._h, 0)

    def poison_lin(self) -> None:
        self._lib.frame_poison(self._h, 1)

    def poison_low(self) -> None:
        self._lib.frame_poison(self._h, 2)

    def arena_bytes(self) -> int:
        return int(self._lib.frame_arena_bytes(self._h))

    # ---- row bands: the plan must already carry the band (plan.set_row_band) -----------------------------------------
    def use_plan_band(self) -> None:
        rows = self.plan.band_rows()
        prod = (C.c_int * 10)(*[v for lohi in rows["produce"] for v in lohi])
        self.band = rows["produce"][0]
        self._lib.frame_set_band(self._h, self.band[0], self.band[1], prod)
        self.poison_low()

    def band_phase_a(self, depth_band: np.ndarray) -> None:
        d = _aligned(np.ascontiguousarray(depth_band, np.float32))
        assert d.shape == (self.band[1] - self.band[0], self.W)
        self._lib.frame_band_phase_a(self._h, d.ctypes.data, 0)

    def halo_pack(self, side: int) -> np.ndarray:
        rows = self.plan.halo_rows(side, True)
        buf = _aligned(np.zeros(max(self.plan.halo_bytes(side) // 4, 1), np.float32))
        self._lib.frame_halo(self._h, (C.c_int * 8)(*[v for lohi in rows for v in lohi]), buf.ctypes.data, 1)
        return buf[:self.plan.halo_bytes(side) // 4]

    def halo_unpack(self, side: int, packed: np.ndarray) -> None:
        rows = self.plan.halo_rows(side, False)
        buf = _aligned(np.ascontiguousarray(packed, np.float32)) if packed.size else _aligned(np.zeros(1, np.float32))
        assert packed.size * 4 == self.plan.halo_recv_bytes(side)
        self._lib.frame_halo(self._h, (C.c_int * 8)(*[v for lohi in rows for v in lohi]), buf.ctypes.data, 0)

    # ---- native neighbour exchange (band_exchange.cu): peers are other Frame objects of the same frame size ---------
    def exchange(self, up=None, down=None, timeout_polls: int = 1000) -> int:
        """Runs band_exchange_kernel for this band: pushes its border rows straight into the neighbours' LowDepth buffers and
        handshakes through the epoch flags.  Returns the sticky error (0 = ok)."""
        ru = (C.c_int * 8)(*[v for lohi in self.plan.halo_rows(0, True) for v in lohi])
        rd = (C.c_int * 8)(*[v for lohi in self.plan.halo_rows(1, True) for v in lohi])
        return int(self._lib.frame_band_exchange(self._h, up._h if up is not None else None, down._h if down is not None else None, ru, rd, timeout_polls))

    def flags(self, set_ready_ack=None) -> dict:
        out = (C.c_int * 8)()
        arr = (C.c_int * 4)(*set_ready_ack) if set_ready_ack is not None else None
        self._lib.frame_band_flags(self._h, arr, out)
        return {"ready": (out[0], out[1]), "ack": (out[2], out[3]), "epoch": out[4], "done": out[5], "error": out[6], "host_error": out[7]}

    def band_phase_b(self) -> np.ndarray:
        """-> the band's rows of the AO texture"""
        self._ao = None
        self._lib.frame_band_phase_b(self._h)
        return self.buffer(17)[self.band[0]:self.band[1]]

    # ---- reading back -----------------------------------------------------------------------------------------------------
    def tma_box_loads(self) -> int:
        """Emulated TMA box loads issued by this library instance so far (process-wide counter)."""
        return int(self._lib.frame_tma_box_loads())

    def surface_accesses(self) -> int:
        return int(self._lib.frame_surface_accesses())

    def buffer(self, bid: int, layer: int = 0) -> np.ndarray:
        if bid == 17 and self._ao is not None:
            return self._ao[layer].copy()
        d = self.plan.buffer_desc(bid)
        dt = {1: np.uint8, 2: np.float16, 4: np.float32}[d.elem_bytes]
        shape = (d.slices, d.height, d.width) if d.slices > 1 else (d.height, d.width)
        out = np.zeros(shape, dt)
        assert self._lib.frame_get_buffer(self._h, bid, layer, out.ctypes.data) == 0
        return out

    def debug_view(self, bid: int) -> np.ndarray:
        out = np.zeros((self.H, self.W), np.uint8)
        assert self._lib.frame_debug_view(self._h, bid, out.ctypes.data) == 0
        return out


STAGES = ("prepare", "render", "render_wide", "upsample")    # frame_record.h FrameStage
PDL = ("never", ">=1", ">=2")                                # frame_record.h PdlClass


def schedule(variants=(0, 0, 0, 0)) -> list:
    """frame_record.h frame_schedule of MeaoVariants (single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale): one
    (stage, level, branch, wait, pdl, name) per launch in serial order; wait is the index of the launch waited for, or None."""
    cap = 32
    out, names = (C.c_int * (5 * cap))(), C.create_string_buffer(32 * cap)
    n = lib().frame_schedule_export((C.c_int * 4)(*variants), out, names, cap)
    assert 0 < n <= cap
    rows = []
    for i in range(n):
        stage, level, branch, wait, pdl = out[5 * i:5 * i + 5]
        rows.append((STAGES[stage], level, branch, None if wait < 0 else wait, PDL[pdl], names.raw[32 * i:32 * (i + 1)].split(b"\0")[0].decode()))
    return rows


def kernel_units() -> dict:
    """kernels.h kKernelUnits as the emulator builds them: unit file -> the number of kernels in its table."""
    cap = 32
    names, counts = C.create_string_buffer(32 * cap), (C.c_int * cap)()
    n = lib().frame_kernel_units(names, counts, cap)
    assert 0 < n <= cap
    return {names.raw[32 * i:32 * (i + 1)].split(b"\0")[0].decode(): counts[i] for i in range(n)}


_symbols: dict | None = None
_KERNEL = re.compile(r"(?:void )?meao::\(anonymous namespace\)::(\w+_kernel(?:<[^()]*>)?)\([^()]*\)")


def _kernel_symbols() -> dict:
    """library-relative address -> 'name<template args>' of every kernel of the library (one nm run, cached).  The kernels are
    meao::(anonymous namespace)::*_kernel functions: local symbols, in the symbol table but not among the dynamic ones."""
    global _symbols
    if _symbols is None:
        out = subprocess.run(["nm", "-C", "--defined-only", build_emu.build()], capture_output=True, text=True, check=True).stdout
        _symbols = {}
        for line in out.splitlines():
            parts = line.split(" ", 2)
            m = _KERNEL.fullmatch(parts[2]) if len(parts) == 3 and parts[1] in "tT" else None
            if m:
                _symbols[int(parts[0], 16)] = m.group(1)
    return _symbols


def emulated_kernels() -> set:
    """The name of every kernel the emulator builds ('render_ao_kernel<0, true, 32>', 'halo_copy_kernel')."""
    return set(_kernel_symbols().values())


def ledger_reset() -> None:
    lib().frame_ledger_reset()


def _ledger() -> dict:
    """{library-relative kernel address: (launches, TMA box loads issued during them, CTAs of their grids)} since ledger_reset()."""
    cap = 256
    off, n_launch, n_tma, n_cta = (C.c_ulonglong * cap)(), (C.c_longlong * cap)(), (C.c_longlong * cap)(), (C.c_longlong * cap)()
    n = lib().frame_ledger_read(off, n_launch, n_tma, n_cta, cap)
    assert 0 <= n <= cap
    return {off[i]: (n_launch[i], n_tma[i], n_cta[i]) for i in range(n)}


def kernel_ledger() -> dict:
    """The kernels launched since ledger_reset() in this process: {name: (launches, TMA box loads issued during them)}."""
    names = _kernel_symbols()
    return {names.get(off, hex(off)): e[:2] for off, e in _ledger().items()}


def library_symbols(path: str) -> dict:
    """library-relative address -> 'name<template args>' of every kernel of the library at `path` (one nm run)."""
    out = subprocess.run(["nm", "-C", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    syms = {}
    for line in out.splitlines():
        parts = line.split(" ", 2)
        m = _KERNEL.fullmatch(parts[2]) if len(parts) == 3 and parts[1] in "tT" else None
        if m:
            syms[int(parts[0], 16)] = m.group(1)
    return syms


def unit_ledger(names: dict) -> dict:
    """The ledger entries of one library's kernels (`names`: its library_symbols): {name: (launches, TMA box loads, CTAs)}.  The
    ledger keys a kernel by its address relative to its own library, so the libraries' kernels must not share an offset
    (tests/test_unit_matrix_emulated.py checks that they do not)."""
    return {names[off]: e for off, e in _ledger().items() if off in names}


def composite(ao: np.ndarray, color: np.ndarray, *, rgb: bool, alpha: bool, one_minus: bool) -> np.ndarray:
    out = _aligned(np.ascontiguousarray(color))
    a = _aligned(np.ascontiguousarray(ao, np.uint8))
    lib().frame_composite(a.ctypes.data, out.ctypes.data, a.size, int(out.dtype == np.float16), int(rgb), int(alpha), int(one_minus))
    return out.copy()


def composite_debug(view: np.ndarray, like: np.ndarray) -> np.ndarray:
    v = _aligned(np.ascontiguousarray(view, np.uint8))
    out = _aligned(np.zeros(v.shape + (4,), like.dtype))
    lib().frame_composite_debug(v.ctypes.data, out.ctypes.data, v.size, int(out.dtype == np.float16))
    return out.copy()
