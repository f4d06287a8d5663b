"""ctypes front end of tests/emu/libmeao_emu_views.so: CUDA-array viewport frames (meao_render_arrays_at) in the emulator.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h).  The library holds one driver (frame_views.cpp) and links against libmeao_emu.so, so the
kernels that run, the surface-access counter and the launch ledger are those of the emulator the other CPU tests use.  It is built
like that one: through a private temporary directory and an atomic rename."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

from . import emu

build_emu = emu.build_emu
HERE = build_emu.HERE

SRC = os.path.join(HERE, "frame_views.cpp")
LIB = os.path.join(HERE, "libmeao_emu_views.so")
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
    tmp = tempfile.mkdtemp(prefix="meao_emu_views_")
    try:
        obj, out = os.path.join(tmp, "frame_views.o"), os.path.join(tmp, "lib.so")
        p = subprocess.run(["g++"] + build_emu.FLAGS + ["-c", SRC, "-o", obj], capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise RuntimeError("emulator build failed: frame_views.cpp")
        subprocess.check_call(["g++", "-shared", "-o", out, obj, "-L", HERE, "-l:" + os.path.basename(base), "-Wl,-rpath,$ORIGIN"])
        staged = f"{LIB}.tmp{os.getpid()}"
        shutil.copyfile(out, staged)
        os.replace(staged, LIB)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return LIB


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        emu.lib()                                   # builds and loads libmeao_emu.so first: the views library shares that instance
        l = C.CDLL(_build(build_emu.LIB))
        P, I, LL = C.c_void_p, C.c_int, C.c_longlong
        l.frame_run_arrays_at.argtypes = [P, P, I, I, I, I, LL, I, I, P, I, I, I, LL, I, I]
        _lib = l
    return _lib


def run_arrays_at(frame: emu.Frame, depth: np.ndarray, depth_origin, ao: np.ndarray, ao_origin, depth_shape: str = "2d",
                  ao_shape: str | None = None) -> None:
    """A CUDA-array frame of viewports on `frame`.  depth: the whole emulated depth array [layers, h, w] (float32 / uint16 D16 codes),
    read at depth_origin = (x, y); ao: the whole AO array [layers, h', w'] (uint8), written in place at ao_origin.  The arrays' rows are
    exactly their width: only the emulator's range check of each array's own extent stands between a stray access and a wrong byte."""
    assert depth.flags.c_contiguous and ao.flags.c_contiguous and ao.dtype == np.uint8
    ao_shape = ao_shape or depth_shape
    (dx, dy), (ax, ay) = depth_origin, ao_origin
    lib().frame_run_arrays_at(frame._h, depth.ctypes.data, frame._kind(depth), emu.SHAPES[depth_shape], depth.shape[2], depth.shape[1],
                              depth.strides[1], dx, dy, ao.ctypes.data, emu.SHAPES[ao_shape], ao.shape[2], ao.shape[1], ao.strides[1],
                              ax, ay)
