"""ctypes front end of tests/emu/libmeao_emu_cameras.so: device cameras (meao_bind_device_cameras) in the emulator -- the camera tables
derived by the host-compiled camera kernel, and whole bound frames.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h).  The library holds one driver (frame_device_cameras.cpp) and the camera unit (build.py
CAMERA_SOURCES), and links against libmeao_emu.so, libmeao_emu_ortho.so and libmeao_emu_mixed.so (the orthographic and mixed kernels
of bound frames with orthographic layers), so every other kernel, the surface-access counter and the launch ledger are those of the
emulator the other CPU tests use.  It is built like that one: through a private temporary directory and an atomic rename."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

from . import emu, mixed, ortho

build_emu = emu.build_emu
HERE = build_emu.HERE

from miniengineao_b200.build import CAMERA_SOURCES  # noqa: E402

SRC = os.path.join(HERE, "frame_device_cameras.cpp")
LIB = os.path.join(HERE, "libmeao_emu_cameras.so")
STATUS_WORDS = 6                    # kernels.h kCameraStatusWords
LAYER_RENDER_FLOATS = 32            # kernels.h LayerRender: 128 bytes
_lib: C.CDLL | None = None


def _stale(deps) -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = list(deps) + [SRC] + [os.path.join(build_emu.CSRC, f) for f in os.listdir(build_emu.CSRC)] + \
        [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith(".h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _build(base: str, others) -> str:
    if not _stale([base] + list(others)):
        return LIB
    tmp = tempfile.mkdtemp(prefix="meao_emu_cameras_")
    try:
        objs = []
        for src, lang in [(SRC, [])] + [(os.path.join(build_emu.CSRC, k), ["-x", "c++"]) for k in CAMERA_SOURCES]:
            obj = os.path.join(tmp, os.path.basename(src) + ".o")
            p = subprocess.run(["g++"] + build_emu.FLAGS + lang + ["-c", src, "-o", obj], capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise RuntimeError(f"emulator build failed: {os.path.basename(src)}")
            objs.append(obj)
        out = os.path.join(tmp, "lib.so")
        subprocess.check_call(["g++", "-shared", "-o", out] + objs + ["-L", HERE] + ["-l:" + os.path.basename(o) for o in others] +
                              ["-l:" + os.path.basename(base), "-Wl,-rpath,$ORIGIN"])
        staged = f"{LIB}.tmp{os.getpid()}"
        shutil.copyfile(out, staged)
        os.replace(staged, LIB)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return LIB


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        ortho.lib()                                 # builds and loads libmeao_emu.so and the libraries this one links first: shared
        mixed.lib()                                 # instances
        l = C.CDLL(_build(build_emu.LIB, [ortho.LIB, mixed.LIB]))
        P, I = C.c_void_p, C.c_int
        l.frame_cams_plan.argtypes = [P, I, C.POINTER(C.c_int32)]
        l.frame_cams_expected.argtypes = [P, P, P]
        l.frame_cams_tables.argtypes = [P, P, P]
        l.frame_cams_clobber.argtypes = [P, I]
        l.frame_cams_derive.argtypes = [P, P, P]
        l.frame_cams_run.argtypes = [P, P, P, P, I, I, P, I]
        l.frame_cams_tiled.argtypes = [P, I, I, I, P]
        l.frame_cams_kernel_unit.argtypes = [C.c_char_p]
        _lib = l
    return _lib


def frame(plan, table, stereo=False, **kw) -> emu.Frame:
    """An emu.Frame on the plan of `plan` (a plan-only context whose host cameras, variants and projections are set), with the layers'
    projections `table` and single-pass stereo, as libmeao plans them (frame_cams_plan)."""
    f = emu.Frame(plan, **kw)
    lib().frame_cams_plan(f._h, int(stereo), (C.c_int32 * len(table))(*table))
    return f


def _tables(fn, f: emu.Frame):
    zb = np.zeros((f.layers, 2), np.float32)
    ren = np.zeros((8, f.layers, LAYER_RENDER_FLOATS), np.float32)
    fn(f._h, zb.ctypes.data, ren.ctypes.data)
    return zb, ren


def expected(f: emu.Frame):
    """camera_tables() of the frame's plan: (LayerZ [L, 2], LayerRender [8, L, 32]) as float32 arrays (compare them as bytes)."""
    return _tables(lib().frame_cams_expected, f)


def tables(f: emu.Frame):
    """The arena's camera tables as they stand, shaped like expected()."""
    return _tables(lib().frame_cams_tables, f)


def clobber(f: emu.Frame, fill: int = 0xA5) -> None:
    lib().frame_cams_clobber(f._h, fill)


def new_status() -> np.ndarray:
    return np.zeros(STATUS_WORDS, np.uint32)


def derive(f: emu.Frame, cams: np.ndarray, status: np.ndarray) -> None:
    """The camera stage alone, from cams [L, 3] float32 (near, far, tan_half_fov_h)."""
    c = np.ascontiguousarray(cams, np.float32)
    assert c.shape == (f.layers, 3) or (c.ndim == 2 and c.shape[0] >= f.layers and c.shape[1] == 3)
    rc = lib().frame_cams_derive(f._h, c.ctypes.data, status.ctypes.data)
    assert rc == 0, f"the camera launch failed ({rc})"


def run(f: emu.Frame, cams: np.ndarray, status: np.ndarray, depth: np.ndarray, *, fused: bool = True, ren_tile: int = -1) -> None:
    """A whole bound frame (the camera stage, then the schedule with the layered kernels at every layer count).  fused: meao_render's
    frame, AO into a tight array of the caller's (f.buffer(17)); otherwise the stage API's frame.  depth [H, W] or [layers, H, W].
    ren_tile: -1 the planner's rule; 0 / 1 / 2 force 64x32 / 64x16 / 64x8 render tiles."""
    c = np.ascontiguousarray(cams, np.float32)
    d = emu._aligned(np.ascontiguousarray(depth))
    assert d.shape == f._shape(d)
    ao = emu._aligned(np.zeros((f.layers, f.H, f.W), np.uint8)) if fused else None
    f._ao, f._keep = ao, (c, d, ao)
    rc = lib().frame_cams_run(f._h, c.ctypes.data, status.ctypes.data, d.ctypes.data, f._kind(d), int(fused),
                              None if ao is None else ao.ctypes.data, ren_tile)
    assert rc == 0, f"a launch failed ({rc})"


def buffer(f: emu.Frame, bid: int, layer: int, kind: int) -> np.ndarray:
    """f.buffer(bid, layer), with TiledDepth1..4 (ids 6-9) synthesised with the padding of the layer's derived camera table row for
    depth kind `kind` (MEAO_DEPTH_*), as meao_get_buffer reads them while a buffer is bound."""
    if not 6 <= bid <= 9:
        return f.buffer(bid, layer)
    d = f.plan.buffer_desc(bid)
    out = np.zeros((d.slices, d.height, d.width), np.float16)
    lib().frame_cams_tiled(f._h, bid - 5, layer, kind, out.ctypes.data)
    return out


def kernel_unit() -> tuple:
    """(the camera unit's file, the number of kernels in its table) as this library builds it."""
    name = C.create_string_buffer(32)
    n = lib().frame_cams_kernel_unit(name)
    return name.value.decode(), n


_symbols: dict | None = None


def _kernel_symbols() -> dict:
    global _symbols
    if _symbols is None:
        _symbols = emu.library_symbols(lib()._name)
    return _symbols


def kernels() -> set:
    """The name of every kernel this library builds (camera_tables_kernel, camera_tables_mixed_kernel)."""
    return set(_kernel_symbols().values())


def ledger() -> dict:
    """This library's kernels in the emulator's launch ledger since its last reset: {name: (launches, TMA box loads, CTAs)}."""
    return emu.unit_ledger(_kernel_symbols())
