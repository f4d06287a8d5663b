"""Layered frames (meao_set_layers) against the ways a host renders L same-size views without them, in microseconds per view.

  (a) layered   one context with L layers on one stream, frames back to back (one graph of 9 kernels per frame)
  (b) serial    one single-layer context, the L views rendered one after the other (L graphs per frame)
  (c) throughput: 5 layered contexts on 5 streams, against 5 single-layer contexts on 5 streams rendering L views each

The arms alternate over several rounds (CUDA events, after a warm-up of every context); the median round is reported.  The
outputs of all arms are compared bit for bit on the same inputs.  Prints the GPU's name and power limit, then one JSON line per
configuration.

    python scripts/bench_layers.py [--frames 50] [--rounds 5]
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

STREAMS = 5


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def _ctx(W, H, layers):
    from miniengineao_b200 import AmbientOcclusion, Camera
    ao = AmbientOcclusion(Camera(W, H), device=0)
    ao.layers = layers
    ao.LateUpdate()
    return ao


def run_config(torch, W, H, L, frames, rounds):
    from miniengineao_b200 import synth
    depth_np = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    depth = torch.from_numpy(depth_np).cuda()
    streams = [torch.cuda.Stream() for _ in range(STREAMS)]
    lay = [_ctx(W, H, L) for _ in range(STREAMS)]
    one = [_ctx(W, H, 1) for _ in range(STREAMS)]
    out_l = [torch.empty((L, H, W), dtype=torch.uint8, device="cuda") for _ in range(STREAMS)]
    out_1 = [torch.empty((L, H, W), dtype=torch.uint8, device="cuda") for _ in range(STREAMS)]

    def layered(n_ctx, n):
        d = depth if L > 1 else depth[0]                                # a single-layer context takes [H, W]
        for _ in range(n):
            for c in range(n_ctx):
                lay[c].render(d, out_l[c] if L > 1 else out_l[c][0], stream=streams[c])

    def serial(n_ctx, n):
        for _ in range(n):
            for c in range(n_ctx):
                for l in range(L):
                    one[c].render(depth[l], out_1[c][l], stream=streams[c])

    def timed(fn, n_ctx):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(streams[0])
        for s in streams[1:n_ctx]:
            s.wait_event(e0)
        fn(n_ctx, frames)
        for s in streams[1:n_ctx]:
            ev = torch.cuda.Event()
            ev.record(s)
            streams[0].wait_event(ev)
        e1.record(streams[0])
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (frames * L * n_ctx)       # us per view

    arms = {"a_layered": (layered, 1), "b_serial": (serial, 1), "c_layered_x5": (layered, STREAMS), "c_single_x5": (serial, STREAMS)}
    for fn, n in arms.values():                                         # warm-up: graph capture of every context and buffer pair
        fn(STREAMS, 3)
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, (fn, n) in arms.items():
            res[k].append(timed(fn, n))
    ref = out_1[0].cpu().numpy()
    identical = all(np.array_equal(o.cpu().numpy(), ref) for o in out_l + out_1)
    for c in lay + one:
        c.close()
    row = {"W": W, "H": H, "layers": L, "frames": frames, "rounds": rounds, "outputs_identical": bool(identical)}
    for k, v in res.items():
        row[k + "_us_per_view"] = round(float(np.median(v)), 2)
        row[k + "_spread_us"] = round(float(max(v) - min(v)), 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50, help="frames per timed window and arm")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--configs", default="1920x1080x1,1920x1080x2,1920x1080x6,1920x1080x8,3840x2160x2")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_layers.py needs a GPU")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for cfg in args.configs.split(","):
        W, H, L = (int(v) for v in cfg.split("x"))
        print(json.dumps(run_config(torch, W, H, L, args.frames, args.rounds)), flush=True)


if __name__ == "__main__":
    main()
