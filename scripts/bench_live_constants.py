"""The cost of live frame constants: a camera and an intensity that change on every frame, against a static camera.

One context per arm renders frames back to back on one stream (synthetic corridor depth, every layer its own frame of it).  Arms,
alternated over rounds:
  (a) static     the same camera and MeaoParams every frame: graph replays
  (b) animated   a new field of view (30 -> 90 degrees), near plane and intensity every frame: the constants are planned again on the
                 host, the camera tables are written on the stream and the frame's graph is re-targeted (capture + cudaGraphExecUpdate)
  (c) before     (b) on another build of libmeao.so (--lib-before), e.g. one from before live constants, where a change re-planned
Configurations: 1920 x 1080 and 3840 x 2160, with 1 and 6 layers.  Per arm: device time per frame (CUDA events around the whole
back-to-back run of --frames frames, so an idle gap between frames counts) and the host time of one meao_render call (which holds
the re-target), each the median over --rounds rounds, with the spread of the device time.  Prints the GPU's name and power limit, then
one JSON line per configuration.

    python scripts/bench_live_constants.py [--rounds 5] [--frames 200] [--lib-before path/to/libmeao.so]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [(1920, 1080, 1), (3840, 2160, 1), (1920, 1080, 6), (3840, 2160, 6)]


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def load(path: str) -> C.CDLL:
    """A libmeao.so with every signature of include/meao.h bound (miniengineao_b200._native's table)."""
    from miniengineao_b200 import _native as N
    if path == N.LIB_PATH:
        return N.lib()
    lib = C.CDLL(path)
    for name, (res, args) in N.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib


class Arm:
    def __init__(self, lib, W, H, L, animated):
        from miniengineao_b200 import _native as N
        self.N, self.lib, self.W, self.H, self.animated = N, lib, W, H, animated
        h = C.c_void_p()
        assert lib.meao_create(C.byref(N.MeaoDeviceCfg(0, 0)), C.byref(h)) == 0
        self.ctx = h
        assert lib.meao_set_layers(h, L) >= 0
        assert lib.meao_resize(h, W, H) >= 0
        self.params = N.MeaoParams()
        lib.meao_default_params(C.byref(self.params))
        self.i = 0

    def frame(self, depth, out, stream) -> float:
        """One frame; returns the host time (s) of its meao_render call."""
        lib = self.lib
        if self.animated:
            t = (self.i % 61) / 60.0
            fov = math.radians(30.0 + 60.0 * t)
            cam = self.N.MeaoCamera(0.1 + 0.2 * t, 1000.0, math.tan(fov / 2) * self.W / self.H, 1)
            assert lib.meao_set_camera(self.ctx, C.byref(cam)) == 0
            self.params.intensity = 0.5 + t
            assert lib.meao_set_params(self.ctx, C.byref(self.params)) >= 0
        self.i += 1
        t0 = time.perf_counter()
        rc = lib.meao_render(self.ctx, C.c_void_p(depth.data_ptr()), 0, C.c_void_p(out.data_ptr()), stream)
        dt = time.perf_counter() - t0
        assert rc == 0, lib.meao_last_error(self.ctx)
        return dt

    def close(self):
        self.lib.meao_destroy(self.ctx)


def run(torch, arm, n, depth, out, s):
    """n frames back to back: (device ms per frame, median host us per meao_render call)."""
    sh = C.c_void_p(s.cuda_stream)
    s.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    host = [arm.frame(depth, out, sh) for _ in range(n)]
    e1.record(s)
    s.synchronize()
    return e0.elapsed_time(e1) / n, float(np.median(host)) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--lib-before", default=None, help="another libmeao.so for arm (c)")
    args = ap.parse_args()
    import torch
    from miniengineao_b200 import _native as N, build, synth
    assert torch.cuda.is_available(), "needs a GPU"
    build.build()
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    libs = {"static": load(N.LIB_PATH), "animated": load(N.LIB_PATH)}
    if args.lib_before:
        libs["before"] = load(os.path.abspath(args.lib_before))
    s = torch.cuda.Stream()
    for W, H, L in CONFIGS:
        depth = torch.from_numpy(np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=l)) for l in range(L)]).astype(np.float32)).cuda()
        arms = {k: Arm(lib, W, H, L, k != "static") for k, lib in libs.items()}
        outs = {k: torch.empty((L, H, W), dtype=torch.uint8, device="cuda") for k in arms}
        for k, arm in arms.items():
            run(torch, arm, 20, depth, outs[k], s)                    # warm-up: module loads, the first capture
        stats = {k: ([], []) for k in arms}
        for _ in range(args.rounds):
            for k, arm in arms.items():
                dev, host = run(torch, arm, args.frames, depth, outs[k], s)
                stats[k][0].append(dev)
                stats[k][1].append(host)
        res = {"width": W, "height": H, "layers": L, "frames": args.frames, "rounds": args.rounds, "gpu": info["name"],
               "power_limit_w": info["power_limit_w"]}
        for k, (dev, host) in stats.items():
            r = N.MeaoReservation()
            arms[k].lib.meao_reservation(arms[k].ctx, C.byref(r))
            res[k] = {"device_us_per_frame": round(1e3 * float(np.median(dev)), 1),
                      "device_us_spread": [round(1e3 * min(dev), 1), round(1e3 * max(dev), 1)],
                      "host_us_per_render": round(float(np.median(host)), 1), "graph_instantiations": r.graph_instantiations}
        for arm in arms.values():
            arm.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
