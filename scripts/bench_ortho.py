"""Orthographic against perspective frames on one GPU: a 4K perspective context and a 4K orthographic context render the same raw
depth, alternating in one process (so both see the same clocks and neighbours), and meao_profile_frame gives each context's per-kernel
times of the four render levels.  Prints the card name and power limit with the numbers; writes nothing.

    python scripts/bench_ortho.py [--rounds 8] [--frames 200] [--size 3840x2160]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from miniengineao_b200 import AmbientOcclusion, Camera, synth  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--size", default="3840x2160")
    ap.add_argument("--profile-repeats", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ortho.py needs a CUDA device")
    W, H = (int(v) for v in a.size.split("x"))
    depth = torch.from_numpy(synth.lin01_to_raw(synth.corridor(W, H)).astype(np.float32)).cuda()
    ctx = {"perspective": AmbientOcclusion(Camera(W, H), device=0),
           "orthographic": AmbientOcclusion(Camera(W, H, orthographic=True, orthographicSize=20.0), device=0)}
    out = {name: torch.empty((H, W), dtype=torch.uint8, device="cuda") for name in ctx}
    for name, ao in ctx.items():               # warm-up: plan, graph instantiation, module loads
        for _ in range(20):
            ao.render(depth, out[name])
    torch.cuda.synchronize()
    us = {name: [] for name in ctx}
    for _ in range(a.rounds):
        for name, ao in ctx.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.frames):
                ao.render(depth, out[name])
            t1.record()
            t1.synchronize()
            us[name].append(1000.0 * t0.elapsed_time(t1) / a.frames)
    render_ms = {}
    for name, ao in ctx.items():
        prof = ao.profile_frame(depth, out[name], repeats=a.profile_repeats)
        render_ms[name] = {n: round(ms * 1000.0, 2) for n, ms in prof if n.startswith("render_ao")}
    res = {"card": card(), "size": f"{W}x{H}", "rounds": a.rounds, "frames_per_round": a.frames,
           "us_per_frame_median": {n: round(statistics.median(v), 2) for n, v in us.items()},
           "us_per_frame_rounds": {n: [round(x, 2) for x in v] for n, v in us.items()},
           "render_us_per_level (meao_profile_frame)": render_ms}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
