"""ctypes front end of tests/emu/libmeao_emu_depth.so: the hierarchy depth (meao_set_hierarchy_depth) of emulated frames.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h).  The library holds frame_depth.cpp and links against libmeao_emu.so, so it sets the depth on
the frames of every emulator front end (emu.Frame and the frames of ortho.py, mixed.py, batch.py, device_cameras.py, ...).  It is built
like that one: through a private temporary directory and an atomic rename."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

from . import emu

build_emu = emu.build_emu
HERE = build_emu.HERE

SRC = os.path.join(HERE, "frame_depth.cpp")
LIB = os.path.join(HERE, "libmeao_emu_depth.so")
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
    tmp = tempfile.mkdtemp(prefix="meao_emu_depth_")
    try:
        obj, out = os.path.join(tmp, "frame_depth.o"), os.path.join(tmp, "lib.so")
        p = subprocess.run(["g++"] + build_emu.FLAGS + ["-c", SRC, "-o", obj], capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise RuntimeError("emulator build failed: frame_depth.cpp")
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
        emu.lib()                                   # builds and loads libmeao_emu.so first: this library shares that instance
        l = C.CDLL(_build(build_emu.LIB))
        P, I = C.c_void_p, C.c_int
        l.frame_set_levels.argtypes = [P, I]
        l.frame_schedule_levels.argtypes = [P, I, I, P, P, I]
        _lib = l
    return _lib


def set_levels(frame: emu.Frame, levels: int) -> emu.Frame:
    """The hierarchy depth of `frame` (any front end's emu.Frame), after its plan was loaded; returns the frame."""
    lib().frame_set_levels(frame._h, int(levels))
    return frame


def schedule(variants=(0, 0, 0, 0), levels=4, device_cameras=False) -> list:
    """frame_record.h frame_schedule of MeaoVariants (single_pass_stereo, sample_exhaustively, high_quality_mask, single_scale) at
    hierarchy depth `levels`, with the camera stage when device_cameras: one (stage, level, branch, wait, pdl, name) per launch in serial
    order; wait is the index of the launch waited for, or None."""
    cap = 32
    out, names = (C.c_int * (5 * cap))(), C.create_string_buffer(32 * cap)
    n = lib().frame_schedule_levels((C.c_int * 4)(*variants), int(levels), int(device_cameras), out, names, cap)
    assert 0 < n <= cap
    stages = emu.STAGES + ("camera",)
    rows = []
    for i in range(n):
        stage, level, branch, wait, pdl = out[5 * i:5 * i + 5]
        rows.append((stages[stage], level, branch, None if wait < 0 else wait, emu.PDL[pdl], names.raw[32 * i:32 * (i + 1)].split(b"\0")[0].decode()))
    return rows
