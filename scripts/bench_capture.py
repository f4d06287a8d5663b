"""Frames inside the caller's CUDA graph: what a host gains by recording the AO frame into its own torch graph.

One context per configuration renders back to back on one stream (synthetic corridor depth, every layer its own frame of it).  Arms,
alternated over rounds:
  (a) render          each frame one meao_render call (the context replays its own cached graph)
  (b) graph           each frame one replay of a torch graph that holds the AO frame (recorded by ao.render inside torch.cuda.graph)
  (c) separate        each frame AO + a frame-buffer composite + a small torch op (a colour grade on a 256-element tensor), three calls
  (d) one graph       the same three recorded into one torch graph, one replay per frame
Configurations: 1920 x 1080 and 3840 x 2160, with 1 and 6 layers.  Per arm: device time per frame (CUDA events around the whole
back-to-back run of --frames frames, so idle gaps between frames count) and the host time of one frame's calls, each the median over
--rounds rounds, with the spread of the device time.  Prints the GPU's name and power limit, then one JSON line per configuration.

    python scripts/bench_capture.py [--rounds 5] [--frames 200]
"""
from __future__ import annotations

import argparse
import json
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


def run(torch, frame, n, s):
    """n frames back to back on stream s: (device us per frame, median host us per frame)."""
    s.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    host = []
    with torch.cuda.stream(s):
        e0.record(s)
        for _ in range(n):
            t0 = time.perf_counter()
            frame()
            host.append(time.perf_counter() - t0)
        e1.record(s)
    s.synchronize()
    return 1e3 * e0.elapsed_time(e1) / n, float(np.median(host)) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=200)
    args = ap.parse_args()
    import torch
    from miniengineao_b200 import AmbientOcclusion, Camera, build, synth
    assert torch.cuda.is_available(), "needs a GPU"
    build.build()
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    s = torch.cuda.Stream()
    for W, H, L in CONFIGS:
        ao = AmbientOcclusion(Camera(W, H), device=0)
        ao.layers = L
        shape = (L, H, W) if L > 1 else (H, W)
        depth = torch.from_numpy(np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=l)) for l in range(L)]).astype(np.float32)
                                 .reshape(shape)).cuda()
        out = torch.empty(shape, dtype=torch.uint8, device="cuda")
        color = torch.full(shape + (4,), 200, dtype=torch.uint8, device="cuda")
        grade = torch.ones(256, device="cuda")

        def ao_frame():
            ao.render(depth, out)

        def full_frame():
            ao.render(depth, out)
            ao.composite_framebuffer(out, color)
            grade.mul_(1.0001).clamp_(0.0, 2.0)

        graphs = {}
        for name, fn in (("graph", ao_frame), ("one_graph", full_frame)):
            run(torch, fn, 3, s)                                        # warm-up: module loads, the context's first capture
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                fn()
            graphs[name] = g
        arms = {"render": ao_frame, "graph": graphs["graph"].replay, "separate": full_frame, "one_graph": graphs["one_graph"].replay}
        for fn in arms.values():
            run(torch, fn, 20, s)
        stats = {k: ([], []) for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                dev, host = run(torch, fn, args.frames, s)
                stats[k][0].append(dev)
                stats[k][1].append(host)
        res = {"width": W, "height": H, "layers": L, "frames": args.frames, "rounds": args.rounds, "gpu": info["name"],
               "power_limit_w": info["power_limit_w"]}
        for k, (dev, host) in stats.items():
            res[k] = {"device_us_per_frame": round(float(np.median(dev)), 1), "device_us_spread": [round(min(dev), 1), round(max(dev), 1)],
                      "host_us_per_frame": round(float(np.median(host)), 1)}
        del graphs, arms
        torch.cuda.synchronize()
        ao.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
