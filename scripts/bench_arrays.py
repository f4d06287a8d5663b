"""CUDA-array frames (meao_render_arrays) against the linear-buffer frame and against the copies a host needs without them, in
microseconds per frame (all L layers):

  (a) pointers  meao_render on linear device buffers
  (b) arrays    meao_render_arrays: the depth read from and the AO written into CUDA arrays by the first and last kernel
  (c) copies    the workaround on one stream: copy the depth out of its array (cudaMemcpy3DAsync), meao_render, copy the AO into its array

The arms alternate over several rounds (CUDA events around `frames` back-to-back frames, after a warm-up); the median round and the
spread (max - min) are reported.  The AO of all three arms is compared bit for bit.  Prints the GPU's name and power limit, then one
JSON line per configuration.

    python scripts/bench_arrays.py [--frames 100] [--rounds 7]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

D2D = 3


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def run_config(torch, rt, W, H, L, shape, frames, rounds):
    from gpu_harness import Array, Extent, Memcpy3DParms, PitchedPtr   # the ctypes CUDA-array helpers of the GPU tests
    from miniengineao_b200 import AmbientOcclusion, Camera, synth
    ao = AmbientOcclusion(Camera(W, H), device=0)
    ao.layers = L
    ao.LateUpdate()
    depth_np = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    depth = torch.from_numpy(depth_np if L > 1 else depth_np[0]).cuda()
    out = {k: torch.empty(depth.shape, dtype=torch.uint8, device="cuda") for k in "ac"}
    dstage = torch.empty_like(depth)
    da, aa_b, aa_c = Array(rt, W, H, np.float32, shape, L), Array(rt, W, H, np.uint8, shape, L), Array(rt, W, H, np.uint8, shape, L)
    da.fill(depth_np)
    stream = torch.cuda.Stream()
    sh = C.c_void_p(stream.cuda_stream)

    def copy(arr, dev, elem, to_array):
        p = Memcpy3DParms()
        pp = PitchedPtr(dev.data_ptr(), W * elem, W, H)
        if to_array:
            p.srcPtr, p.dstArray = pp, arr.handle
        else:
            p.srcArray, p.dstPtr = arr.handle, pp
        p.extent, p.kind = Extent(W, H, arr.layers), D2D
        assert rt.cudaMemcpy3DAsync(C.byref(p), sh) == 0

    def arm_a(n):
        for _ in range(n):
            ao.render(depth, out["a"], stream=stream)

    def arm_b(n):
        for _ in range(n):
            ao.render_arrays(da.handle, aa_b.handle, stream=stream)

    def arm_c(n):
        for _ in range(n):
            copy(da, dstage, 4, False)
            ao.render(dstage, out["c"], stream=stream)
            copy(aa_c, out["c"], 1, True)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn(frames)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / frames

    arms = {"a_pointers": arm_a, "b_arrays": arm_b, "c_copies": arm_c}
    for fn in arms.values():
        fn(5)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn))
    torch.cuda.synchronize()
    a = out["a"].cpu().numpy().reshape(L, H, W)
    identical = bool(np.array_equal(aa_b.read(), a) and np.array_equal(aa_c.read(), a) and np.array_equal(out["c"].cpu().numpy().reshape(L, H, W), a))
    for x in (da, aa_b, aa_c):
        ao.release_array(x.handle)
        x.free()
    ao.close()
    row = {"W": W, "H": H, "layers": L, "array": shape, "frames": frames, "rounds": rounds, "outputs_identical": identical}
    for k, v in res.items():
        row[k + "_us"] = round(float(np.median(v)), 2)
        row[k + "_spread_us"] = round(float(max(v) - min(v)), 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100, help="frames per timed window and arm")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--configs", default="1920x1080x1:2d,1920x1080x2:layered,3840x2160x1:2d,3840x2160x2:layered,1024x1024x6:cube")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_arrays.py needs a GPU")
    torch.cuda.init()
    from gpu_harness import Memcpy3DParms, runtime
    rt = runtime()
    rt.cudaMemcpy3DAsync.argtypes = [C.POINTER(Memcpy3DParms), C.c_void_p]
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for cfg in args.configs.split(","):
        size, shape = cfg.split(":")
        W, H, L = (int(v) for v in size.split("x"))
        print(json.dumps(run_config(torch, rt, W, H, L, shape, args.frames, args.rounds)), flush=True)


if __name__ == "__main__":
    main()
