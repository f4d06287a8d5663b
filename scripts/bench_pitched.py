"""Pitched frames (meao_render_pitched) against the tight frame and against the copies a host needs without them, in microseconds per
frame (all L layers):

  (a) tight    meao_render on tight device buffers
  (b) pitched  meao_render_pitched on the same images with every row padded to a multiple of 256 bytes (a D3D12 placed footprint),
               or, with a Wmax, as the corner of a Wmax-wide target (dynamic resolution)
  (c) copies   the workaround on one stream: cudaMemcpy2DAsync of the padded depth into a tight buffer, meao_render, cudaMemcpy2DAsync of
               the AO back into the padded AO

The arms alternate over several rounds (CUDA events around `frames` back-to-back frames, after a warm-up); the median round and the
spread (max - min) are reported.  The AO of all three arms is compared bit for bit.  Prints the GPU's name and power limit, then one
JSON line per configuration.

    python scripts/bench_pitched.py [--frames 100] [--rounds 7] [--configs 1366x768x1,1920x1080x1,1920x1080x2,3840x2160x1:4096]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D2D = 3


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def run_config(torch, rt, W, H, L, frames, rounds, wmax=0, row_align=256):
    from miniengineao_b200 import AmbientOcclusion, Camera, synth
    from miniengineao_b200 import _native as N
    lib = N.lib()
    ao = AmbientOcclusion(Camera(W, H), device=0)
    ao.layers = L
    ao.LateUpdate()
    ctx = ao._ctx
    depth_np = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    wp = max(W, wmax)               # wmax: the frame is the corner of a target this wide (dynamic resolution)
    dpitch, apitch = (wp * 4 + row_align - 1) // row_align * row_align, (wp + row_align - 1) // row_align * row_align
    tight_d = torch.from_numpy(depth_np).cuda()
    tight_a = {k: torch.empty((L, H, W), dtype=torch.uint8, device="cuda") for k in "ac"}
    pad_d = torch.full((L, H, dpitch // 4), float("nan"), dtype=torch.float32, device="cuda")
    pad_d[:, :, :W] = tight_d
    pad_a = {k: torch.zeros((L, H, apitch), dtype=torch.uint8, device="cuda") for k in "bc"}
    stream = torch.cuda.Stream()
    sh = C.c_void_p(stream.cuda_stream)
    rows = L * H                    # the layers are H rows apart: one 2-D copy covers them all

    def arm_a(n):
        for _ in range(n):
            N.check(ctx, lib.meao_render(ctx, tight_d.data_ptr(), 0, tight_a["a"].data_ptr(), sh))

    def arm_b(n):
        for _ in range(n):
            N.check(ctx, lib.meao_render_pitched(ctx, pad_d.data_ptr(), dpitch, H * dpitch, 0, pad_a["b"].data_ptr(), apitch, H * apitch, sh))

    def arm_c(n):
        for _ in range(n):
            assert rt.cudaMemcpy2DAsync(C.c_void_p(tight_d.data_ptr()), W * 4, C.c_void_p(pad_d.data_ptr()), dpitch, W * 4, rows, D2D, sh) == 0
            N.check(ctx, lib.meao_render(ctx, tight_d.data_ptr(), 0, tight_a["c"].data_ptr(), sh))
            assert rt.cudaMemcpy2DAsync(C.c_void_p(pad_a["c"].data_ptr()), apitch, C.c_void_p(tight_a["c"].data_ptr()), W, W, rows, D2D, sh) == 0

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn(frames)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / frames

    arms = {"a_tight": arm_a, "b_pitched": arm_b, "c_copies": arm_c}
    for fn in arms.values():
        fn(5)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn))
    torch.cuda.synchronize()
    a = tight_a["a"].cpu().numpy()
    identical = bool(np.array_equal(pad_a["b"][:, :, :W].cpu().numpy(), a) and np.array_equal(pad_a["c"][:, :, :W].cpu().numpy(), a)
                     and np.array_equal(tight_a["c"].cpu().numpy(), a))
    ao.close()
    row = {"W": W, "H": H, "layers": L, "depth_row_pitch": dpitch, "ao_row_pitch": apitch, "frames": frames, "rounds": rounds,
           "outputs_identical": identical}
    for k, v in res.items():
        row[k + "_us"] = round(float(np.median(v)), 2)
        row[k + "_spread_us"] = round(float(max(v) - min(v)), 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100, help="frames per timed window and arm")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--configs", default="1366x768x1,1920x1080x1,1920x1080x2,3840x2160x1,3840x2160x1:4096",
                    help="WxHxL[:Wmax], Wmax: the width of the target the frame is the corner of (sets the row pitch)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_pitched.py needs a GPU")
    torch.cuda.init()
    rt = C.CDLL("libcudart.so.12")
    rt.cudaMemcpy2DAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p]
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for cfg in args.configs.split(","):
        size, _, wmax = cfg.partition(":")
        W, H, L = (int(v) for v in size.split("x"))
        print(json.dumps(run_config(torch, rt, W, H, L, args.frames, args.rounds, int(wmax or 0))), flush=True)


if __name__ == "__main__":
    main()
