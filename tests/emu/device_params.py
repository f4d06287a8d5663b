"""ctypes front end of tests/emu/libmeao_emu_params.so: device parameters (meao_bind_device_params) in the emulator -- the slot derived
by the host-compiled parameter stage, and whole frames through the *_params_layered render twins.

TEST INFRASTRUCTURE ONLY (see cuda_emu.h).  The library holds one driver (frame_device_params.cpp) and the device-parameter units
(build.py PARAM_SOURCES), and links against libmeao_emu_cameras.so, libmeao_emu_ortho.so, libmeao_emu_mixed.so and libmeao_emu.so, so
every other kernel (the camera stage of frames with device cameras too), the surface-access counter and the launch ledger are those of
the emulator the other CPU tests use.  It is built like that one: through a private temporary directory and an atomic rename."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

from . import device_cameras, emu, mixed, ortho

build_emu = emu.build_emu
HERE = build_emu.HERE

from miniengineao_b200.build import PARAM_SOURCES  # noqa: E402

SRC = os.path.join(HERE, "frame_device_params.cpp")
LIB = os.path.join(HERE, "libmeao_emu_params.so")
SLOT_WORDS = 4                  # {reject_fadeoff, intensity} and kernels.h kParamStatusWords status words
_lib: C.CDLL | None = None


def _stale(deps) -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = list(deps) + [SRC] + [os.path.join(build_emu.CSRC, f) for f in os.listdir(build_emu.CSRC)] + \
        [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith(".h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _build(others) -> str:
    if not _stale(others):
        return LIB
    tmp = tempfile.mkdtemp(prefix="meao_emu_params_")
    try:
        objs = []
        for src, lang in [(SRC, [])] + [(os.path.join(build_emu.CSRC, k), ["-x", "c++"]) for k in PARAM_SOURCES]:
            obj = os.path.join(tmp, os.path.basename(src) + ".o")
            p = subprocess.run(["g++"] + build_emu.FLAGS + lang + ["-c", src, "-o", obj], capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise RuntimeError(f"emulator build failed: {os.path.basename(src)}")
            objs.append(obj)
        out = os.path.join(tmp, "lib.so")
        subprocess.check_call(["g++", "-shared", "-o", out] + objs + ["-L", HERE] + ["-l:" + os.path.basename(o) for o in others] +
                              ["-Wl,-rpath,$ORIGIN"])
        staged = f"{LIB}.tmp{os.getpid()}"
        shutil.copyfile(out, staged)
        os.replace(staged, LIB)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return LIB


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        device_cameras.lib()                        # builds and loads the libraries this one links first: shared instances
        l = C.CDLL(_build([device_cameras.LIB, ortho.LIB, mixed.LIB, build_emu.LIB]))
        P, I = C.c_void_p, C.c_int
        l.frame_params_derive.argtypes = [P, P]
        l.frame_params_run.argtypes = [P, P, P, P, P, P, I, I, P, I]
        l.frame_params_kernel_units.argtypes = [P, P, I]
        _lib = l
    return _lib


def new_slot(reject_fadeoff: float, intensity: float) -> np.ndarray:
    """The context's slot as meao_bind_device_params writes it: the host's derived values, the status words zero (as float32 words)."""
    s = np.zeros(SLOT_WORDS, np.float32)
    s[0], s[1] = reject_fadeoff, intensity
    return s


def status(slot: np.ndarray) -> list:
    return [int(w) for w in slot[2:].view(np.uint32)]


def derive(params, slot: np.ndarray) -> None:
    """The parameter stage alone, from params (thickness_modifier, intensity) into slot."""
    p = np.ascontiguousarray(params, np.float32)
    assert p.shape == (2,)
    rc = lib().frame_params_derive(p.ctypes.data, slot.ctypes.data)
    assert rc == 0, f"the parameter launch failed ({rc})"


def run(f: emu.Frame, depth: np.ndarray, *, params=None, slot=None, cams=None, cam_status=None, fused: bool = True,
        ren_tile: int = -1) -> None:
    """A whole frame of f's plan (device_cameras.frame) with the schedule of its bindings: params (thickness_modifier, intensity) with
    slot, and / or cams [L, 3] with cam_status; None: the plan's host values.  fused and ren_tile as device_cameras.run."""
    p = None if params is None else np.ascontiguousarray(params, np.float32)
    c = None if cams is None else np.ascontiguousarray(cams, np.float32)
    d = emu._aligned(np.ascontiguousarray(depth))
    assert d.shape == f._shape(d)
    ao = emu._aligned(np.zeros((f.layers, f.H, f.W), np.uint8)) if fused else None
    f._ao, f._keep = ao, (p, c, d, ao)
    ptr = lambda a: None if a is None else a.ctypes.data     # noqa: E731
    rc = lib().frame_params_run(f._h, ptr(p), ptr(slot), ptr(c), ptr(cam_status), d.ctypes.data, f._kind(d), int(fused), ptr(ao), ren_tile)
    assert rc == 0, f"a launch failed ({rc})"


def kernel_units() -> dict:
    """The device-parameter units as this library builds them: unit file -> the number of kernels in its table."""
    cap = 8
    names, counts = C.create_string_buffer(48 * cap), (C.c_int * cap)()
    n = lib().frame_params_kernel_units(names, counts, cap)
    return {names.raw[48 * i:48 * (i + 1)].split(b"\0")[0].decode(): counts[i] for i in range(n)}


_symbols: dict | None = None


def _kernel_symbols() -> dict:
    global _symbols
    if _symbols is None:
        _symbols = emu.library_symbols(lib()._name)
    return _symbols


def kernels() -> set:
    """The name of every kernel this library builds (render_params_kernel and the 36 *_params_layered_kernel instantiations)."""
    return set(_kernel_symbols().values())


def ledger() -> dict:
    """This library's kernels in the emulator's launch ledger since its last reset: {name: (launches, TMA box loads, CTAs)}."""
    return emu.unit_ledger(_kernel_symbols())
