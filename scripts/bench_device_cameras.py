"""A camera that moves every frame, recorded into the caller's torch.cuda.graph, on one GPU.  Per size (1920x1080, 3840x2160) and layer
count (1, 6), three arms alternated in one process (so all see the same clocks and neighbours), medians over rounds:
  (a) host cameras: every camera change moves meao_frame_generation, so the frame is captured into a new graph and instantiated before
      its replay (the recipe without device cameras);
  (b) device cameras (meao_bind_device_cameras): one graph captured once; a torch op inside it writes the frame's cameras into the bound
      tensor from a per-frame input, which the host updates with copy_ before each replay;
  (c) a static camera: one graph captured once and replayed (the floor).
For each arm: device microseconds per frame (CUDA events around the frames) and host microseconds per frame (the issue loop, before the
final synchronise).  After the timed rounds every arm renders the same cameras once and the AO is compared.  meao_profile_frame gives
the per-kernel times of a bound context (the camera stage, and the layered kernels at L = 1) and of an unbound one (the single-image
kernels at L = 1).  Prints the card name and power limit with the numbers; writes nothing.

    python scripts/bench_device_cameras.py [--rounds 6] [--frames 40]
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


def camera_rows(W, H, L, i):
    """The cameras of frame i: a field of view and planes that move every frame."""
    rows = []
    for l in range(L):
        c = Camera(W, H, nearClipPlane=0.3 + 0.01 * ((i + l) % 7), farClipPlane=1000.0 - (i % 5), fieldOfView=55.0 + 0.5 * ((i + 3 * l) % 11))
        rows.append((c.nearClipPlane, c.farClipPlane, 1.0 / c.projection00))
    return rows


def host_cams(W, H, rows):
    return [Camera(W, H, nearClipPlane=float(n), farClipPlane=float(f), fieldOfView=float(np.degrees(2 * np.arctan(t / (W / H)))))
            for n, f, t in rows]


def context(W, H, L):
    ao = AmbientOcclusion(Camera(W, H, nearClipPlane=0.3, farClipPlane=1000.0), device=0)
    ao.layers = L
    return ao


def bench(W, H, L, rounds, frames, repeats):
    raw = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    depth = torch.from_numpy(raw if L > 1 else raw[0]).cuda()
    shape = (L, H, W) if L > 1 else (H, W)
    outs = {k: torch.empty(shape, dtype=torch.uint8, device="cuda") for k in "abc"}
    s = torch.cuda.Stream()
    inputs = [torch.tensor(camera_rows(W, H, L, i), dtype=torch.float32).pin_memory() for i in range(frames)]

    # (a) host cameras, one capture and instantiation per camera change
    a = context(W, H, L)
    a.layerCameras = host_cams(W, H, camera_rows(W, H, L, 0)) if L > 1 else None

    def set_host(i):
        cams = host_cams(W, H, inputs[i].tolist())
        if L > 1:
            a.layerCameras = cams
        else:
            a.camera.nearClipPlane, a.camera.farClipPlane, a.camera.fieldOfView = cams[0].nearClipPlane, cams[0].farClipPlane, cams[0].fieldOfView

    def frame_a(i):
        set_host(i)
        with torch.cuda.stream(s):
            a.render(depth, outs["a"], stream=s)        # settles the new constants outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            a.render(depth, outs["a"], stream=s)
        g.replay()
        return g

    # (b) device cameras: one capture; the op inside it copies the frame's input into the bound tensor
    b = context(W, H, L)
    cam_in = torch.empty((L, 3), dtype=torch.float32, device="cuda")
    cam_in.copy_(inputs[0])
    b.deviceCameras = torch.empty((L, 3), dtype=torch.float32, device="cuda")
    b.deviceCameras.copy_(cam_in)
    with torch.cuda.stream(s):
        b.render(depth, outs["b"], stream=s)
    s.synchronize()
    gb = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gb, stream=s):
        b.deviceCameras.copy_(cam_in)
        b.render(depth, outs["b"], stream=s)

    def frame_b(i):
        cam_in.copy_(inputs[i], non_blocking=True)
        gb.replay()

    # (c) a static camera
    c = context(W, H, L)
    with torch.cuda.stream(s):
        c.render(depth, outs["c"], stream=s)
    s.synchronize()
    gc = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gc, stream=s):
        c.render(depth, outs["c"], stream=s)

    def frame_c(i):
        gc.replay()

    arms = {"a_recapture_per_change": frame_a, "b_device_cameras": frame_b, "c_static_camera": frame_c}
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
            t0.record()
            h0 = time.perf_counter()
            for i in range(frames):
                keep.append(fn(i))
            h1 = time.perf_counter()
            t1.record()
            t1.synchronize()
            dev[name].append(1000.0 * t0.elapsed_time(t1) / frames)
            host[name].append(1e6 * (h1 - h0) / frames)
            del keep
    # the same cameras through every arm: (a) and (c) with host cameras, (b) from the tensor
    last = frames - 1
    frame_a(last)
    frame_b(last)
    c.layerCameras = host_cams(W, H, inputs[last].tolist()) if L > 1 else None
    if L == 1:
        hc = host_cams(W, H, inputs[last].tolist())[0]
        c.camera.nearClipPlane, c.camera.farClipPlane, c.camera.fieldOfView = hc.nearClipPlane, hc.farClipPlane, hc.fieldOfView
    c.render(depth, outs["c"])
    torch.cuda.synchronize()
    equal = bool(torch.equal(outs["a"], outs["b"]) and torch.equal(outs["b"], outs["c"]))
    prof = {}
    for name, ao in (("bound", b), ("unbound", c)):
        prof[name] = {n: round(ms * 1000.0, 2) for n, ms in ao.profile_frame(depth, outs["c"], repeats=repeats)}
    return {"size": f"{W}x{H}", "layers": L, "rounds": rounds, "frames_per_round": frames, "ao_equal_between_arms": equal,
            "device_us_per_frame_median": {n: round(statistics.median(v), 1) for n, v in dev.items()},
            "host_us_per_frame_median": {n: round(statistics.median(v), 1) for n, v in host.items()},
            "device_us_per_frame_rounds": {n: [round(x, 1) for x in v] for n, v in dev.items()},
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
        raise SystemExit("bench_device_cameras.py needs a CUDA device")
    res = {"card": card(), "results": []}
    for size in a.sizes.split(","):
        W, H = (int(v) for v in size.split("x"))
        for L in (int(x) for x in a.layers.split(",")):
            res["results"].append(bench(W, H, L, a.rounds, a.frames, a.profile_repeats))
            print(json.dumps(res["results"][-1]), flush=True)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
