"""Builds libmeao.so (CUDA, sm_90a only) in-tree with nvcc.

nvcc cross-compiles without a GPU, so this also runs in the CPU-only build container.
-fmad=false: fused multiply-adds appear only where the sources call fmaf() (the arithmetic
contract shared with the oracle); -prec-div / -prec-sqrt stay at their IEEE defaults.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmeao.so")
SOURCES = ["meao_api.cu", "prepare_depth.cu", "render_ao.cu", "blur_upsample.cu", "selftest.cu", "halo.cu", "band_exchange.cu", "composite.cu", "debug_view.cu",
           "prepare_depth_layered.cu", "render_ao_layered.cu", "blur_upsample_layered.cu", "prepare_depth_array.cu", "blur_upsample_array.cu",
           "blur_upsample_lin.cu"]
# The layer-viewport kernels (meao_set_layer_viewports): compiled into libmeao.so with SOURCES; the CPU emulator builds them into a
# library of their own (tests/emu/layer_views.py), and tests/test_layer_viewports_units.py audits them.
VIEW_SOURCES = ["prepare_depth_array_views.cu", "blur_upsample_array_views.cu", "prepare_depth_views.cu", "blur_upsample_lin_views.cu"]
# The orthographic-projection kernels (meao_set_projection): compiled into libmeao.so with SOURCES, each a textual include of an existing
# kernel body under MEAO_ORTHO, so the SOURCES kernels keep their code; tests/test_ortho_units.py audits them.
ORTHO_SOURCES = ["prepare_depth_ortho.cu", "prepare_depth_ortho_layered.cu", "prepare_depth_array_ortho.cu", "render_ao_ortho.cu",
                 "render_ao_ortho_layered.cu", "blur_upsample_lin_ortho.cu"]
# The batch kernels (meao_render_arrays_batch / meao_render_batch: each layer with its own depth and AO): compiled into libmeao.so with
# SOURCES; the CPU emulator builds them into a library of their own (tests/emu/batch.py), and tests/test_batch_units.py audits them.
BATCH_SOURCES = ["prepare_depth_array_batch.cu", "blur_upsample_array_batch.cu", "prepare_depth_batch.cu", "blur_upsample_lin_batch.cu"]
# The per-layer projection kernels (meao_set_layer_projections: a layered frame whose layers mix both projections): compiled into
# libmeao.so with SOURCES, each a textual include of an existing kernel body under MEAO_ORTHO 2, so the other kernels keep their code; the
# CPU emulator builds them into a library of their own (tests/emu/mixed.py), and tests/test_layer_projections_units.py audits them.
MIXED_SOURCES = ["prepare_depth_mixed_layered.cu", "prepare_depth_array_mixed.cu", "render_ao_mixed_layered.cu", "blur_upsample_lin_mixed.cu"]
# The device-camera kernel (meao_bind_device_cameras: the per-layer camera tables derived on the device at the head of every frame):
# compiled into libmeao.so with SOURCES; tests/test_device_cameras_units.py audits it, and the CPU emulator builds it into a library of its
# own (tests/emu/device_cameras.py).
CAMERA_SOURCES = ["camera_tables.cu"]
# The device-parameter kernels (meao_bind_device_params: reject_fadeoff and intensity derived on the device ahead of the renders, and the
# layered render kernels that read them): compiled into libmeao.so with SOURCES, the renders each a textual include of an existing kernel
# body under MEAO_DEVICE_PARAMS, so the other kernels keep their code; tests/test_device_params_units.py audits them, and the CPU emulator
# builds them into a library of their own (tests/emu/device_params.py).
PARAM_SOURCES = ["render_params.cu", "render_ao_params_layered.cu", "render_ao_ortho_params_layered.cu", "render_ao_mixed_params_layered.cu"]
HEADERS = ["common.cuh", "kernels.h", "prepare_depth_kernel.inc", "render_ao_kernel.inc", "render_ao_groups.inc", "render_ao_sample.inc", "blur_upsample_device.inc", "blur_upsample_kernel.inc",
           "blur_upsample_layer_args.inc", "blur_upsample_lin_device.inc", "surface_io.cuh", "depth_in.cuh", "arena_layout.h", "frame_record.h",
           os.path.join("..", "..", "include", "meao.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false",
    "-Xcompiler", "-fPIC,-O2,-fvisibility=hidden",
    "-Xptxas", "-v",
    "-shared", "-cudart", "static", "--threads", "0",
    "-Xlinker", "--exclude-libs,ALL", "-Xlinker", "-Bsymbolic",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in SOURCES + VIEW_SOURCES + ORTHO_SOURCES + BATCH_SOURCES + MIXED_SOURCES + CAMERA_SOURCES + PARAM_SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    extra = os.environ.get("MEAO_NVCC_DEFS", "").split()      # tuning experiments, e.g. "-DMEAO_REN_MINB=12"
    cmd = [_nvcc()] + NVCC_FLAGS + extra + ["-o", LIB] + [os.path.join(CSRC, f) for f in SOURCES + VIEW_SOURCES + ORTHO_SOURCES + BATCH_SOURCES + MIXED_SOURCES + CAMERA_SOURCES + PARAM_SOURCES]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed building libmeao.so")
    with open(os.path.join(HERE, "build_ptxas.log"), "w") as f:
        f.write(proc.stdout + proc.stderr)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print(LIB)
