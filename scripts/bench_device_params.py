"""An AO fade -- thickness_modifier and intensity that change every frame -- on one GPU.  Per size (1920x1080, 3840x2160) and layer count
(1, 6), four arms alternated in one process (so all see the same clocks and neighbours), medians over rounds:
  (a) host parameters on the context's own graph: meao_set_params every frame, which the next frame takes as live constants (the own
      graph is re-targeted, not re-captured);
  (b) device parameters on the context's own graph (meao_bind_device_params): the host writes the bound tensor with copy_ every frame;
  (c_host) a caller's torch.cuda.graph with host parameters: every change moves meao_frame_generation, so the frame is captured into a
      new graph and instantiated before its replay;
  (c_device) a caller's torch.cuda.graph with device parameters: one graph captured once, the tensor written with copy_ before each replay.
For each arm: device microseconds per frame (CUDA events around the frames) and host microseconds per frame (the issue loop, before the
final synchronise), with the spread over rounds.  After the timed rounds every arm renders the same values once and the AO is compared.
meao_profile_frame gives the per-kernel times of a bound and an unbound context.  Prints the card name and power limit with the numbers;
writes nothing.

    python scripts/bench_device_params.py [--rounds 6] [--frames 40]
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def values(i):
    """(thickness_modifier, intensity) of frame i: a fade in and out, and a thickness that moves with it."""
    t = (i % 20) / 19.0
    return 0.5 + 2.0 * t, 1.5 * (1.0 - abs(2.0 * t - 1.0))


def context(W, H, L):
    ao = AmbientOcclusion(Camera(W, H, nearClipPlane=0.3, farClipPlane=1000.0), device=0)
    ao.layers = L
    return ao


def bench(W, H, L, rounds, frames, repeats):
    raw = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    depth = torch.from_numpy(raw if L > 1 else raw[0]).cuda()
    shape = (L, H, W) if L > 1 else (H, W)
    outs = {k: torch.empty(shape, dtype=torch.uint8, device="cuda") for k in ("a", "b", "ch", "cd")}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    inputs = [torch.tensor(values(i), dtype=torch.float32).pin_memory() for i in range(frames)]

    def host_set(ao, i):
        ao.thicknessModifier, ao.intensity = values(i)

    a = context(W, H, L)

    def frame_a(i):
        host_set(a, i)
        a.render(depth, outs["a"], stream=s)

    b = context(W, H, L)
    b.deviceParams = torch.tensor(values(0), dtype=torch.float32, device="cuda")

    def frame_b(i):
        with torch.cuda.stream(s):
            b.deviceParams.copy_(inputs[i], non_blocking=True)
        b.render(depth, outs["b"], stream=s)

    ch = context(W, H, L)

    def frame_ch(i):
        host_set(ch, i)
        with torch.cuda.stream(s):
            ch.render(depth, outs["ch"], stream=s)      # settles the new constants outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ch.render(depth, outs["ch"], stream=s)
        g.replay()
        return g

    cd = context(W, H, L)
    cd.deviceParams = torch.tensor(values(0), dtype=torch.float32, device="cuda")
    with torch.cuda.stream(s):
        cd.render(depth, outs["cd"], stream=s)
    s.synchronize()
    gcd = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gcd, stream=s):
        cd.render(depth, outs["cd"], stream=s)

    def frame_cd(i):
        with torch.cuda.stream(s):
            cd.deviceParams.copy_(inputs[i], non_blocking=True)
            gcd.replay()

    arms = {"a_host_params_own_graph": frame_a, "b_device_params_own_graph": frame_b, "c_host_params_recapture": frame_ch,
            "c_device_params_replay": frame_cd}
    for fn in arms.values():
        for i in range(3):
            fn(i)
    torch.cuda.synchronize()
    dev = {n: [] for n in arms}
    host = {n: [] for n in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            keep = []
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record(s)
            h0 = time.perf_counter()
            for i in range(frames):
                keep.append(fn(i))
            h1 = time.perf_counter()
            t1.record(s)
            t1.synchronize()
            dev[name].append(1000.0 * t0.elapsed_time(t1) / frames)
            host[name].append(1e6 * (h1 - h0) / frames)
            del keep
    last = frames - 1
    for fn in arms.values():
        fn(last)
    torch.cuda.synchronize()
    equal = all(torch.equal(outs["a"], outs[k]) for k in ("b", "ch", "cd"))
    prof = {}
    for name, ao in (("bound", b), ("unbound", a)):
        prof[name] = {n: round(ms * 1000.0, 2) for n, ms in ao.profile_frame(depth, outs["a"], repeats=repeats)}

    def spread(v):
        return [round(min(v), 1), round(max(v), 1)]
    return {"size": f"{W}x{H}", "layers": L, "rounds": rounds, "frames_per_round": frames, "ao_equal_between_arms": equal,
            "device_us_per_frame_median": {n: round(statistics.median(v), 1) for n, v in dev.items()},
            "device_us_per_frame_min_max": {n: spread(v) for n, v in dev.items()},
            "host_us_per_frame_median": {n: round(statistics.median(v), 1) for n, v in host.items()},
            "host_us_per_frame_min_max": {n: spread(v) for n, v in host.items()},
            "kernel_us (meao_profile_frame)": prof}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--profile-repeats", type=int, default=20)
    ap.add_argument("--sizes", default="1920x1080,3840x2160")
    ap.add_argument("--layers", default="1,6")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_params.py needs a CUDA device")
    res = {"card": card(), "results": []}
    for size in a.sizes.split(","):
        W, H = (int(v) for v in size.split("x"))
        for L in (int(x) for x in a.layers.split(",")):
            res["results"].append(bench(W, H, L, a.rounds, a.frames, a.profile_repeats))
            print(json.dumps(res["results"][-1]), flush=True)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
