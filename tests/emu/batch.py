"""ctypes front end of tests/emu/libmeao_emu_batch.so: batches over CUDA arrays and device buffers (meao_render_arrays_batch /
meao_render_batch) in the emulator.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h).  The library holds one driver (frame_batch.cpp) and the batch kernels' translation units
(build.py BATCH_SOURCES), and links against libmeao_emu.so, so every other kernel, the surface-access counter and the launch
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

from miniengineao_b200.build import BATCH_SOURCES  # noqa: E402

SRC = os.path.join(HERE, "frame_batch.cpp")
LIB = os.path.join(HERE, "libmeao_emu_batch.so")
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
    tmp = tempfile.mkdtemp(prefix="meao_emu_batch_")
    try:
        srcs = [(SRC, [])] + [(os.path.join(build_emu.CSRC, k), ["-x", "c++"]) for k in BATCH_SOURCES]

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
        P = C.c_void_p
        l.frame_run_arrays_batch.argtypes = [P, C.c_int] + [P] * 10
        l.frame_run_pointers_batch.argtypes = [P, C.c_int, P, P, P, P]
        l.frame_batch_kernel_units.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.c_int]
        _lib = l
    return _lib


def _ptrs(arrs):
    return (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])


def _note_kind(frame: emu.Frame, dtype) -> None:
    """The emulator's driver pads its tiled debug views by the ingest kind of the last prepare it ran (as libmeao does by the last
    frame's): one low-only prepare of a zero depth of this kind tells it.  The batch frame then rewrites every intermediate."""
    zero = np.zeros((frame.layers, frame.H, frame.W), dtype)
    emu.lib().frame_prepare_low(frame._h, zero.ctypes.data, frame._kind(zero))


def run_arrays_batch(frame: emu.Frame, depths, aos, depth_shapes=None, ao_shapes=None) -> None:
    """An array batch on `frame`: layer l reads the emulated 2-D array depths[l] ([h, w], float32 / uint16 D16 codes, at least W x H)
    and writes aos[l] ([h', w'] uint8) in place.  depth_shapes / ao_shapes: "2d" or "layered" (of one layer) per layer."""
    L = frame.layers
    assert len(depths) == L and len(aos) == L and all(a.dtype == np.uint8 and a.flags.c_contiguous for a in aos)
    assert all(d.flags.c_contiguous for d in depths)
    ds, as_ = depth_shapes or ["2d"] * L, ao_shapes or ["2d"] * L
    _note_kind(frame, depths[0].dtype)
    ints = lambda v: (C.c_int * L)(*v)                  # noqa: E731
    lls = lambda v: (C.c_longlong * L)(*v)              # noqa: E731
    lib().frame_run_arrays_batch(frame._h, frame._kind(depths[0]), _ptrs(depths), ints([emu.SHAPES[s] for s in ds]),
                                 ints([d.shape[1] for d in depths]), ints([d.shape[0] for d in depths]), lls([d.strides[0] for d in depths]),
                                 _ptrs(aos), ints([emu.SHAPES[s] for s in as_]), ints([a.shape[1] for a in aos]),
                                 ints([a.shape[0] for a in aos]), lls([a.strides[0] for a in aos]))


def run_pointers_batch(frame: emu.Frame, depths, depth_rows, aos, ao_rows) -> None:
    """A pointer batch (the fused frame of meao_render_batch) on `frame`: layer l reads the buffer depths[l] (any dtype of the depth
    kind, rows depth_rows[l] BYTES apart from its first element) and writes aos[l] (a uint8 buffer, rows ao_rows[l] bytes apart).
    Entries are numpy arrays whose first element is the view's first pixel (a base may be misaligned on purpose)."""
    L = frame.layers
    lls = lambda v: (C.c_longlong * L)(*v)              # noqa: E731
    frame._keep = (depths, aos)
    _note_kind(frame, depths[0].dtype)
    lib().frame_run_pointers_batch(frame._h, frame._kind(depths[0]), _ptrs(depths), lls(depth_rows), _ptrs(aos), lls(ao_rows))


def kernel_units() -> dict:
    """The batch kernels' units as the emulator builds them: unit file -> the number of kernels in its table."""
    cap = 8
    names, counts = C.create_string_buffer(32 * cap), (C.c_int * cap)()
    n = lib().frame_batch_kernel_units(names, counts, cap)
    return {names.raw[32 * i:32 * (i + 1)].split(b"\0")[0].decode(): counts[i] for i in range(n)}


_symbols: dict | None = None


def _kernel_symbols() -> dict:
    """library-relative address -> 'name<template args>' of every kernel this library builds (one nm run, cached)"""
    global _symbols
    if _symbols is None:
        out = subprocess.run(["nm", "-C", "--defined-only", _build(build_emu.LIB)], capture_output=True, text=True, check=True).stdout
        _symbols = {}
        for line in out.splitlines():
            parts = line.split(" ", 2)
            m = emu._KERNEL.fullmatch(parts[2]) if len(parts) == 3 and parts[1] in "tT" else None
            if m:
                _symbols[int(parts[0], 16)] = m.group(1)
    return _symbols


def kernels() -> set:
    """The name of every kernel this library builds ('prepare_depth_low_batch_kernel<true, false, 2>', ...)."""
    return set(_kernel_symbols().values())


def launched() -> set:
    """The kernels of this library in the emulator's launch ledger (emu.kernel_ledger) since its last reset.  The ledger keeps each
    kernel's address relative to its own library, and names only libmeao_emu.so's; the others are named here."""
    names = _kernel_symbols()
    return {names[int(k, 16)] for k in emu.kernel_ledger() if k.startswith("0x") and int(k, 16) in names}
