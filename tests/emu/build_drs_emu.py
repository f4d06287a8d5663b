"""Builds tests/emu/libmeao_emu_drs.so: the kernel sources of a fused frame (build_lin_emu.KERNELS) with drs_driver.cpp, which runs
frames of several sizes inside one arena laid out for the largest (meao_reserve), compiled by g++ for the host (-DMEAO_EMULATE), with
the fiber runtime.  TEST INFRASTRUCTURE ONLY (see cuda_emu.h).

The same compiler flags as build_emu.py; the build goes through a private temporary directory and an atomic rename, so test processes
that build it at the same time never see a half-written library."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_emu  # noqa: E402
import build_lin_emu  # noqa: E402

CSRC = build_emu.CSRC
LIB = os.path.join(HERE, "libmeao_emu_drs.so")
KERNELS = build_lin_emu.KERNELS


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".h", ".cpp", ".py"))]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    tmp = tempfile.mkdtemp(prefix="meao_emu_drs_")
    try:
        objs = []
        for src, lang in [(os.path.join(HERE, "emu_runtime.cpp"), []), (os.path.join(HERE, "drs_driver.cpp"), [])] + \
                         [(os.path.join(CSRC, k), ["-x", "c++"]) for k in KERNELS]:
            obj = os.path.join(tmp, os.path.basename(src) + ".o")
            p = subprocess.run(["g++"] + build_emu.FLAGS + lang + ["-c", src, "-o", obj], capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise RuntimeError(f"dynamic-resolution emulator build failed: {os.path.basename(src)}")
            objs.append(obj)
        out = os.path.join(tmp, "lib.so")
        subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", out] + objs)
        staged = f"{LIB}.tmp{os.getpid()}"
        shutil.copyfile(out, staged)            # the temporary directory may be on another file system
        os.replace(staged, LIB)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return LIB


if __name__ == "__main__":
    print(build(force=True))
