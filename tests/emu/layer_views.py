"""ctypes front end of tests/emu/libmeao_emu_layer_views.so: layered CUDA-array and pointer frames with a layer-viewport table
(meao_set_layer_viewports) in the emulator.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h).  The library holds one driver (frame_layer_views.cpp) and the table kernels' translation
units (build.py VIEW_SOURCES), and links against libmeao_emu.so, so every other kernel, the surface-access counter and the launch
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

from miniengineao_b200.build import VIEW_SOURCES  # noqa: E402

SRC = os.path.join(HERE, "frame_layer_views.cpp")
LIB = os.path.join(HERE, "libmeao_emu_layer_views.so")
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
    tmp = tempfile.mkdtemp(prefix="meao_emu_layer_views_")
    try:
        srcs = [(SRC, [])] + [(os.path.join(build_emu.CSRC, k), ["-x", "c++"]) for k in VIEW_SOURCES]

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
        l.frame_run_arrays_views.argtypes = [P, P, I, I, I, I, I, LL, P, I, I, I, I, LL, P]
        l.frame_run_pitched_views.argtypes = [P, P, I, LL, LL, P, LL, LL, P]
        l.frame_view_kernel_units.argtypes = [C.c_char_p, C.POINTER(C.c_int), I]
        _lib = l
    return _lib


def _note_kind(frame: emu.Frame, dtype) -> None:
    """The emulator's driver pads its tiled debug views by the ingest kind of the last prepare it ran (as libmeao does by the last
    frame's): one low-only prepare of a zero depth of this kind tells it.  The table frame then rewrites every intermediate."""
    zero = np.zeros((frame.layers, frame.H, frame.W), dtype)
    emu.lib().frame_prepare_low(frame._h, zero.ctypes.data, frame._kind(zero))


def run_arrays_views(frame: emu.Frame, depth: np.ndarray, ao: np.ndarray, views, depth_shape: str = "2d", ao_shape: str | None = None) -> None:
    """A layered CUDA-array frame on `frame` with the layer-viewport table `views` (one (depth_x, depth_y, depth_slice, ao_x, ao_y,
    ao_slice) per layer).  depth: the whole emulated depth array [slices, h, w] (float32 / uint16 D16 codes); ao: the whole AO array
    [slices, h', w'] (uint8), written in place.  A cube map has 6 slices.  The arrays' rows are exactly their width."""
    assert depth.flags.c_contiguous and ao.flags.c_contiguous and ao.dtype == np.uint8
    assert len(views) == frame.layers
    ao_shape = ao_shape or depth_shape
    table = np.ascontiguousarray(np.asarray(views, np.int32).reshape(frame.layers, 6))
    _note_kind(frame, depth.dtype)
    lib().frame_run_arrays_views(frame._h, depth.ctypes.data, frame._kind(depth), emu.SHAPES[depth_shape], depth.shape[2], depth.shape[1],
                                 depth.shape[0], depth.strides[1], ao.ctypes.data, emu.SHAPES[ao_shape], ao.shape[2], ao.shape[1],
                                 ao.shape[0], ao.strides[1], table.ctypes.data)


def run_pitched_views(frame: emu.Frame, depth: np.ndarray, depth_pitches, ao: np.ndarray, ao_pitches, views) -> None:
    """The fused pointer frame (meao_render_pitched) on `frame` with the table `views`.  depth / ao: flat buffers (any dtype of the
    depth kind / uint8) holding every rectangle at the BYTE pitches depth_pitches = (row, slice) and ao_pitches = (row, slice)."""
    assert depth.flags.c_contiguous and ao.flags.c_contiguous and ao.dtype == np.uint8
    table = np.ascontiguousarray(np.asarray(views, np.int32).reshape(frame.layers, 6))
    frame._keep = (depth, ao, table)
    _note_kind(frame, depth.dtype)
    lib().frame_run_pitched_views(frame._h, depth.ctypes.data, frame._kind(depth), depth_pitches[0], depth_pitches[1], ao.ctypes.data,
                                  ao_pitches[0], ao_pitches[1], table.ctypes.data)


def kernel_units() -> dict:
    """The table kernels' units as the emulator builds them: unit file -> the number of kernels in its table."""
    cap = 8
    names, counts = C.create_string_buffer(32 * cap), (C.c_int * cap)()
    n = lib().frame_view_kernel_units(names, counts, cap)
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
    """The name of every kernel this library builds ('prepare_depth_low_views_kernel<true, false, 2>', ...)."""
    return set(_kernel_symbols().values())


def launched() -> set:
    """The kernels of this library in the emulator's launch ledger (emu.kernel_ledger) since its last reset.  The ledger keeps each
    kernel's address relative to its own library, and names only libmeao_emu.so's; the others are named here."""
    names = _kernel_symbols()
    return {names[int(k, 16)] for k in emu.kernel_ledger() if k.startswith("0x") and int(k, 16) in names}


def ledger() -> dict:
    """launched() with each kernel's ledger entry: {name: (launches, TMA box loads issued during them, CTAs of their grids)}."""
    return emu.unit_ledger(_kernel_symbols())
