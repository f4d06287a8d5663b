"""What the hierarchy depth (meao_set_hierarchy_depth) costs and saves on the GPU.

For depths 1-4 at 1920x1080 and 3840x2160: device microseconds per frame (one context per depth, the arms alternated over several
rounds, each round a CUDA-event pair around `--frames` graph frames, medians over rounds), the per-kernel times of meao_profile_frame,
and the host cost of a depth change (set the depth, render one frame, synchronise, minus a steady frame of the new depth) -- the re-plan
a host pays per toggle.  Prints one JSON document and writes it to --out.

    python scripts/bench_hierarchy_depth.py --rounds 9 --frames 200 --out /tmp/hierarchy_depth.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from miniengineao_b200 import AmbientOcclusion, Camera, synth  # noqa: E402

SIZES = [(1920, 1080), (3840, 2160)]
DEPTHS = [1, 2, 3, 4]


def gpu_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"gpu": q, "torch_device": torch.cuda.get_device_name(0)}


def frames_us(ao, d, out, n) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        ao.render(d, out)
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--replans", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_hierarchy_depth.py measures on the GPU"
    result = {"info": gpu_info(), "rounds": args.rounds, "frames_per_round": args.frames, "sizes": {}}
    for W, H in SIZES:
        depth = torch.from_numpy(synth.lin01_to_raw(synth.corridor(W, H))).cuda()
        ctxs, outs = {}, {}
        for n in DEPTHS:
            ao = AmbientOcclusion(Camera(W, H), device=0)
            ao.hierarchyDepth = n
            outs[n] = torch.empty((H, W), dtype=torch.uint8, device="cuda")
            for _ in range(20):                                    # warm-up: plan, capture, instantiate, clocks
                ao.render(depth, outs[n])
            ctxs[n] = ao
        torch.cuda.synchronize()
        per = {n: [] for n in DEPTHS}
        for r in range(args.rounds):
            order = DEPTHS if r % 2 == 0 else DEPTHS[::-1]            # alternate the arms' order every round
            for n in order:
                per[n].append(frames_us(ctxs[n], depth, outs[n], args.frames))
        entry = {}
        for n in DEPTHS:
            ao = ctxs[n]
            ao.profile_frame(depth, outs[n], repeats=20)
            prof = ao.profile_frame(depth, outs[n], repeats=20)
            entry[f"depth{n}"] = {"us_per_frame_median": round(statistics.median(per[n]), 2),
                                  "us_per_frame_min": round(min(per[n]), 2), "us_per_frame_max": round(max(per[n]), 2),
                                  "kernels_per_frame": ao.kernels_per_frame,
                                  "profile_us": {name: round(ms * 1e3, 2) for name, ms in prof}}
        full = statistics.median(per[4])
        for n in DEPTHS:
            entry[f"depth{n}"]["saving_vs_depth4_pct"] = round(100.0 * (full - statistics.median(per[n])) / full, 1)
        # the re-plan of a depth change: one context toggled between 4 and 2, each toggle's set + frame + synchronise on the host clock,
        # minus the median steady frame of the new depth
        ao = ctxs[4]
        steady = {4: statistics.median(per[4]), 2: statistics.median(per[2])}
        host = []
        for i in range(args.replans):
            n = 2 if i % 2 == 0 else 4
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ao.hierarchyDepth = n
            ao.render(depth, outs[4])
            torch.cuda.synchronize()
            host.append((time.perf_counter() - t0) * 1e6 - steady[n])
        entry["depth_change_host_us_median"] = round(statistics.median(host), 1)
        entry["depth_change_host_us_max"] = round(max(host), 1)
        for c in ctxs.values():
            c.close()
        result["sizes"][f"{W}x{H}"] = entry
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
