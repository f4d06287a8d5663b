"""ctypes front end of tests/emu/libmeao_emu_mixed.so: layered frames whose layers mix both projections (meao_set_layer_projections) in
the emulator.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h).  The library holds one driver (frame_mixed.cpp) and the mixed kernels' translation units
(build.py MIXED_SOURCES), and links against libmeao_emu.so, so every other kernel, the surface-access counter and the launch
ledger are those of the emulator the other CPU tests use.  It is built like that one: through a private temporary directory and an
atomic rename."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import emu

build_emu = emu.build_emu
HERE = build_emu.HERE

from miniengineao_b200.build import MIXED_SOURCES  # noqa: E402

SRC = os.path.join(HERE, "frame_mixed.cpp")
LIB = os.path.join(HERE, "libmeao_emu_mixed.so")
_lib: C.CDLL | None = None


def _stale(base: str) -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [base, SRC] + [os.path.join(build_emu.CSRC, f) for f in os.listdir(build_emu.CSRC)] + \
           [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith(".h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _build(base: str) -> str:
    if not _stale(base):
        return LIB
    tmp = tempfile.mkdtemp(prefix="meao_emu_mixed_")
    try:
        srcs = [(SRC, [])] + [(os.path.join(build_emu.CSRC, k), ["-x", "c++"]) for k in MIXED_SOURCES]

        def compile_one(src_lang):
            src, lang = src_lang
            obj = os.path.join(tmp, os.path.basename(src) + ".o")
            p = subprocess.run(["g++"] + build_emu.FLAGS + lang + ["-c", src, "-o", obj], capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise RuntimeError(f"emulator build failed: {os.path.basename(src)}")
            return obj

        with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as pool:
            objs = list(pool.map(compile_one, srcs))
        out = os.path.join(tmp, "lib.so")
        subprocess.check_call(["g++", "-shared", "-o", out] + objs + ["-L", HERE, "-l:" + os.path.basename(base), "-Wl,-rpath,$ORIGIN"])
        staged = f"{LIB}.tmp{os.getpid()}"
        shutil.copyfile(out, staged)
        os.replace(staged, LIB)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return LIB


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        emu.lib()                                   # builds and loads libmeao_emu.so first: this library shares that instance
        l = C.CDLL(_build(build_emu.LIB))
        P, I, LL = C.c_void_p, C.c_int, C.c_longlong
        l.frame_mixed_set.argtypes = [P, C.POINTER(C.c_int32)]
        l.frame_mixed_is_mixed.argtypes = [P]
        l.frame_run_mixed.argtypes = [P, P, I, I, P, I]
        l.frame_run_arrays_mixed.argtypes = [P, P, I, I, LL, P, I, LL, I]
        l.frame_mixed_tiled.argtypes = [P, I, I, I, P]
        l.frame_mixed_kernel_units.argtypes = [C.c_char_p, C.POINTER(C.c_int), I]
        _lib = l
    return _lib


def frame(plan, table, **kw) -> emu.Frame:
    """An emu.Frame on the plan of `plan` (a plan-only layered context whose projection table is `table`), with the layers' projections
    (frame_mixed_set)."""
    f = emu.Frame(plan, **kw)
    lib().frame_mixed_set(f._h, (C.c_int32 * len(table))(*table))
    return f


def is_mixed(f: emu.Frame) -> bool:
    return lib().frame_mixed_is_mixed(f._h) == 1


def run(f: emu.Frame, depth: np.ndarray, *, fused: bool, ren_tile: int = -1) -> None:
    """A whole frame: fused (meao_render's frame, AO into a tight array of the caller's, returned by f.buffer(17)) or the stage API's
    frame (prepare_depth -> LinearDepth -> final upsample).  depth [H, W] or [layers, H, W] (float32 / uint16 D16 / uint32 D24S8)."""
    d = emu._aligned(np.ascontiguousarray(depth))
    assert d.shape == f._shape(d)
    ao = emu._aligned(np.zeros((f.layers, f.H, f.W), np.uint8)) if fused else None
    f._ao, f._keep = ao, (d, ao)
    rc = lib().frame_run_mixed(f._h, d.ctypes.data, f._kind(d), int(fused), None if ao is None else ao.ctypes.data, ren_tile)
    assert rc == 0, f"a launch failed ({rc})"


def run_arrays(f: emu.Frame, depth: np.ndarray, shape: str = "2d", ren_tile: int = -1, pad: int = 24) -> np.ndarray:
    """A CUDA-array frame.  depth [layers, H, W] (float32 / uint16 D16 codes).  Each array gets rows `pad` elements wider than W, and
    its bytes outside the image must keep their marker.  Returns the AO [layers, H, W]."""
    f._ao = None
    L, H, W = depth.shape
    d = np.full((L, H, W + pad), 7, depth.dtype)
    d[:, :, :W] = depth
    ao = np.full((L, H, W + pad), 0xA5, np.uint8)
    rc = lib().frame_run_arrays_mixed(f._h, d.ctypes.data, f._kind(d), emu.SHAPES[shape], d.strides[1], ao.ctypes.data, emu.SHAPES[shape],
                                      ao.strides[1], ren_tile)
    assert rc == 0, f"a launch failed ({rc})"
    assert (ao[:, :, W:] == 0xA5).all(), "a store outside the image"
    return ao[:, :, :W].copy()


def buffer(f: emu.Frame, bid: int, layer: int, kind: int) -> np.ndarray:
    """f.buffer(bid, layer), with TiledDepth1..4 (ids 6-9) synthesised with the atlas padding of depth kind `kind` (MEAO_DEPTH_*)."""
    if not 6 <= bid <= 9:
        return f.buffer(bid, layer)
    d = f.plan.buffer_desc(bid)
    out = np.zeros((d.slices, d.height, d.width), np.float16)
    lib().frame_mixed_tiled(f._h, bid - 5, layer, kind, out.ctypes.data)
    return out


def kernel_units() -> dict:
    """The mixed units as the emulator builds them: unit file -> the number of kernels in its table."""
    cap = 8
    names, counts = C.create_string_buffer(32 * cap), (C.c_int * cap)()
    n = lib().frame_mixed_kernel_units(names, counts, cap)
    return {names.raw[32 * i:32 * (i + 1)].split(b"\0")[0].decode(): counts[i] for i in range(n)}


_symbols: dict | None = None


def _kernel_symbols() -> dict:
    """library-relative address -> 'name<template args>' of every kernel this library builds (one nm run, cached)"""
    global _symbols
    if _symbols is None:
        out = subprocess.run(["nm", "-C", "--defined-only", lib()._name], capture_output=True, text=True, check=True).stdout
        _symbols = {}
        for line in out.splitlines():
            parts = line.split(" ", 2)
            m = emu._KERNEL.fullmatch(parts[2]) if len(parts) == 3 and parts[1] in "tT" else None
            if m:
                _symbols[int(parts[0], 16)] = m.group(1)
    return _symbols


def kernels() -> set:
    """The name of every kernel this library builds ('prepare_depth_low_mixed_layered_kernel<true, false, 2>', ...)."""
    return set(_kernel_symbols().values())


def launched() -> set:
    """The kernels of this library in the emulator's launch ledger (emu.kernel_ledger) since its last reset.  The ledger keeps each
    kernel's address relative to its own library, and names only libmeao_emu.so's; the others are named here."""
    names = _kernel_symbols()
    return {names[int(k, 16)] for k in emu.kernel_ledger() if k.startswith("0x") and int(k, 16) in names}


def ledger() -> dict:
    """launched() with each kernel's ledger entry: {name: (launches, TMA box loads issued during them, CTAs of their grids)}."""
    return emu.unit_ledger(_kernel_symbols())
