"""Perspective and orthographic views in one frame against the two-context recipe, on one GPU.  Per size (4 x 960x540: the panes of a
1080p quad view; 4 x 1920x1080), one perspective view plus three orthographic views of the same raw depth, four arms alternated in one
process (so all see the same clocks and neighbours), medians over rounds:
  (a) one layered frame with a projection table [P, O, O, O] (meao_set_layer_projections);
  (b) two contexts, a perspective one of 1 layer and an orthographic one of 3 layers, on one stream;
  (c) the same two contexts on two streams;
  (d) a 4-layer all-perspective frame of the same depth: what the mixed kernels cost against their twins.
meao_profile_frame gives the per-kernel times of (a) and (d).  Prints the card name and power limit with the numbers; writes nothing.

    python scripts/bench_mixed_projection.py [--rounds 8] [--frames 100]
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


def persp(W, H):
    return Camera(W, H, nearClipPlane=0.3, farClipPlane=1000.0)


def ortho(W, H, size):
    return Camera(W, H, nearClipPlane=0.3, farClipPlane=1000.0, orthographic=True, orthographicSize=size)


def context(cam, layers=1, layer_cameras=None, per_layer=False):
    ao = AmbientOcclusion(cam, device=0)
    ao.layers, ao.layerCameras, ao.perLayerProjection = layers, layer_cameras, per_layer
    return ao


def bench_size(W, H, rounds, frames, repeats):
    raw = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(4)])
    depth = torch.from_numpy(raw).cuda()
    out = torch.empty((4, H, W), dtype=torch.uint8, device="cuda")
    cams = [persp(W, H)] + [ortho(W, H, s) for s in (8.0, 12.0, 20.0)]
    mixed = context(cams[0], 4, cams, per_layer=True)
    one_p = context(cams[0])
    three_o = context(cams[1], 3, cams[1:])
    all_p = context(cams[0], 4, [persp(W, H) for _ in range(4)])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    main = torch.cuda.current_stream()

    def arm_a():
        mixed.render(depth, out)

    def arm_b():
        one_p.render(depth[0], out[0])
        three_o.render(depth[1:], out[1:])

    def arm_c():
        s1.wait_stream(main)
        s2.wait_stream(main)
        one_p.render(depth[0], out[0], stream=s1)
        three_o.render(depth[1:], out[1:], stream=s2)
        main.wait_stream(s1)
        main.wait_stream(s2)

    def arm_d():
        all_p.render(depth, out)

    arms = {"a_mixed_frame": arm_a, "b_two_contexts_one_stream": arm_b, "c_two_contexts_two_streams": arm_c, "d_all_perspective": arm_d}
    for fn in arms.values():                    # warm-up: plan, graph instantiation, module loads
        for _ in range(20):
            fn()
    torch.cuda.synchronize()
    # the mixed frame's AO equals the two contexts' layer for layer
    arm_a(); ref_a = out.clone()
    arm_b(); torch.cuda.synchronize()
    identical = bool(torch.equal(ref_a, out))
    us = {n: [] for n in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(frames):
                fn()
            t1.record()
            t1.synchronize()
            us[name].append(1000.0 * t0.elapsed_time(t1) / frames)
    prof = {}
    for name, ao in (("a_mixed_frame", mixed), ("d_all_perspective", all_p)):
        prof[name] = {n: round(ms * 1000.0, 2) for n, ms in ao.profile_frame(depth, out, repeats=repeats)}
    return {"views": f"4 x {W}x{H} (1 perspective + 3 orthographic)", "rounds": rounds, "frames_per_round": frames,
            "mixed_equals_two_contexts": identical,
            "us_per_frame_median": {n: round(statistics.median(v), 2) for n, v in us.items()},
            "us_per_frame_rounds": {n: [round(x, 2) for x in v] for n, v in us.items()},
            "kernel_us (meao_profile_frame)": prof}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--profile-repeats", type=int, default=20)
    ap.add_argument("--sizes", default="960x540,1920x1080")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed_projection.py needs a CUDA device")
    res = {"card": card(), "results": []}
    for size in a.sizes.split(","):
        W, H = (int(v) for v in size.split("x"))
        res["results"].append(bench_size(W, H, a.rounds, a.frames, a.profile_repeats))
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
