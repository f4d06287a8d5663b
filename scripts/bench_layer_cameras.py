"""Per-layer cameras (meao_set_layer_cameras) against a shared camera and against the workaround, in microseconds per view.

  (a) shared     one context with L layers and one camera, frames back to back on one stream (one graph of 9 kernels per frame)
  (b) per-layer  the same context shape with a table of L distinct cameras (near / far / field of view differ per layer)
  (c) workaround L single-layer contexts, each with its own camera, the L views rendered one after another on one stream

The arms alternate over several rounds (CUDA events, after a warm-up of every context); the median round and the spread (max - min)
are reported.  (b) and (c) must produce bit-identical AO.  The parent commit's layered frame -- arm (d) -- is measured by running
scripts/bench_layers.py of that checkout in the same call.  Prints the GPU's name and power limit, then one JSON line per configuration.

    python scripts/bench_layer_cameras.py [--frames 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CAMS = [(0.1, 50.0, 40.0), (0.3, 100.0, 60.0), (1.0, 1000.0, 90.0), (0.2, 300.0, 75.0)]


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def run_config(torch, W, H, L, frames, rounds):
    from miniengineao_b200 import AmbientOcclusion, Camera, synth
    cams = [Camera(W, H, nearClipPlane=CAMS[i % 4][0], farClipPlane=CAMS[i % 4][1], fieldOfView=CAMS[i % 4][2]) for i in range(L)]
    depth = torch.from_numpy(np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])).cuda()
    stream = torch.cuda.Stream()
    shared = AmbientOcclusion(Camera(W, H), device=0)
    shared.layers = L
    per = AmbientOcclusion(Camera(W, H), device=0)
    per.layers = L
    per.layerCameras = cams
    singles = [AmbientOcclusion(c, device=0) for c in cams]
    out_a, out_b, out_c = (torch.empty((L, H, W), dtype=torch.uint8, device="cuda") for _ in range(3))

    def arm_a(n):
        for _ in range(n):
            shared.render(depth, out_a, stream=stream)

    def arm_b(n):
        for _ in range(n):
            per.render(depth, out_b, stream=stream)

    def arm_c(n):
        for _ in range(n):
            for l in range(L):
                singles[l].render(depth[l], out_c[l], stream=stream)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn(frames)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (frames * L)             # us per view

    arms = {"a_shared": arm_a, "b_per_layer": arm_b, "c_single_contexts": arm_c}
    for fn in arms.values():                                           # warm-up: graph capture of every context
        fn(3)
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn))
    identical = bool(torch.equal(out_b, out_c))
    assert identical, f"{W}x{H} L={L}: per-layer cameras differ from the single-layer contexts"
    for c in [shared, per] + singles:
        c.close()
    row = {"W": W, "H": H, "layers": L, "frames": frames, "rounds": rounds, "b_equals_c": identical}
    for k, v in res.items():
        row[k + "_us_per_view"] = round(float(np.median(v)), 2)
        row[k + "_spread_us"] = round(float(max(v) - min(v)), 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50, help="frames per timed window and arm")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--configs", default="1920x1080x2,1920x1080x6,1920x1080x8,3840x2160x2")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_layer_cameras.py needs a GPU")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for cfg in args.configs.split(","):
        W, H, L = (int(v) for v in cfg.split("x"))
        print(json.dumps(run_config(torch, W, H, L, args.frames, args.rounds)), flush=True)


if __name__ == "__main__":
    main()
