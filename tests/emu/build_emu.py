"""Builds tests/emu/libmeao_emu.so: the kernel SOURCES of miniengineao_b200/csrc compiled by g++ for the host
(-DMEAO_EMULATE) plus the fiber runtime and the frame driver.  TEST INFRASTRUCTURE ONLY (see cuda_emu.h)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(os.path.dirname(HERE)), "miniengineao_b200", "csrc")
LIB = os.path.join(HERE, "libmeao_emu.so")
KERNELS = ["prepare_depth.cu", "render_ao.cu", "blur_upsample.cu", "debug_view.cu", "composite.cu", "halo.cu", "band_exchange.cu"]
FLAGS = ["-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-DMEAO_EMULATE", "-I", HERE, "-Wno-unknown-pragmas", "-Wno-unused-function"]


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".h", ".cpp", ".py"))]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    objs = []
    for src, lang in [(os.path.join(HERE, "emu_runtime.cpp"), []), (os.path.join(HERE, "emu_driver.cpp"), [])] + \
                     [(os.path.join(CSRC, k), ["-x", "c++"]) for k in KERNELS]:
        obj = os.path.join(HERE, f"libmeao_emu_{os.path.basename(src)}.o")
        cmd = ["g++"] + FLAGS + lang + ["-c", src, "-o", obj]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stdout + p.stderr)
            raise RuntimeError(f"emulator build failed: {os.path.basename(src)}")
        objs.append(obj)
    subprocess.check_call(["g++", "-shared", "-o", LIB] + objs)
    for o in objs:
        os.remove(o)
    return LIB


if __name__ == "__main__":
    print(build(force=True))
