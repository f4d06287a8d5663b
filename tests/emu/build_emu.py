"""Builds tests/emu/libmeao_emu.so: the kernel translation units libmeao.so is built from (miniengineao_b200/build.py SOURCES, less the
context and the GPU self test) compiled by g++ for the host (-DMEAO_EMULATE), with the fiber runtime and the frame driver.  TEST
INFRASTRUCTURE ONLY (see cuda_emu.h).

The build goes through a private temporary directory and an atomic rename, so test processes that build it at the same time never
see a half-written library."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from miniengineao_b200.build import SOURCES  # noqa: E402

CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")
LIB = os.path.join(HERE, "libmeao_emu.so")
KERNELS = [s for s in SOURCES if s not in ("meao_api.cu", "selftest.cu")]
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
    tmp = tempfile.mkdtemp(prefix="meao_emu_")
    try:
        srcs = [(os.path.join(HERE, "emu_runtime.cpp"), []), (os.path.join(HERE, "frame_driver.cpp"), [])] + \
               [(os.path.join(CSRC, k), ["-x", "c++"]) for k in KERNELS]

        def compile_one(src_lang):
            src, lang = src_lang
            obj = os.path.join(tmp, os.path.basename(src) + ".o")
            p = subprocess.run(["g++"] + FLAGS + lang + ["-c", src, "-o", obj], capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise RuntimeError(f"emulator build failed: {os.path.basename(src)}")
            return obj

        with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as pool:
            objs = list(pool.map(compile_one, srcs))
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
