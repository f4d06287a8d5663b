"""The cost of a change in the number of views, with and without a layer reservation (meao_reserve_layers), at 1920 x 1080 per view.

Arms, alternated over rounds:
  (a) unreserved  meao_set_layers re-allocates at every count change (what a host did before meao_reserve_layers)
  (b) reserved    meao_reserve_layers(max) once; a count change inside it allocates and synchronises nothing
  (c) fixed       the maximum count every frame: what a host that never changes the count renders
Schedules:
  split    split-screen players 1 -> 2 -> 3 -> 4 -> 2 -> 1, a change every 8 frames, 96 frames.  Every player is a quadrant of one shared
           3840 x 2160 depth and AO target, placed by the layer-viewport table (meao_render_pitched over the shared targets); each
           change is meao_set_layers + meao_set_layer_cameras + meao_set_layer_viewports.  (c) renders all four quadrants every frame.
  batches  a torch-style stream of batches of 64 views (meao_render_batch over a list of [1080, 1920] tensors) with a short final
           batch of 37 in every epoch of 3 x 64 + 37 views, 3 epochs.  (c) pads the short batch to 64.
Per arm: the host time of each change frame (the count change and the frame call, no synchronise: median, max) and the back-to-back
device time of the whole schedule (CUDA events, one synchronise at the end).  The AO of every frame that follows a change is compared
bit for bit between (a) and (b).  Prints the GPU's name and power limit, then one JSON line per schedule.

    python scripts/bench_dynamic_layers.py [--rounds 5]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H = 1920, 1080
PLAYERS = [1, 2, 3, 4, 2, 1]
FRAMES_PER_PHASE = 8
EPOCH = [64, 64, 64, 37]
EPOCHS = 3
QUADS = [(0, 0), (W, 0), (0, H), (W, H)]


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def cams(n):
    from miniengineao_b200 import _native as N
    return (N.MeaoCamera * n)(*[N.MeaoCamera(0.1 + 0.05 * l, 500.0 + 100.0 * l, 0.55 + 0.05 * l, 1) for l in range(n)])


class Ctx:
    def __init__(self, kind: str, max_layers: int):
        from miniengineao_b200 import _native as N
        self.N, self.lib = N, N.lib()
        h = C.c_void_p()
        assert self.lib.meao_create(C.byref(N.MeaoDeviceCfg(0, 0)), C.byref(h)) == 0
        self.h, self.kind, self.max_layers = h, kind, max_layers
        assert self.lib.meao_set_camera(h, C.byref(N.MeaoCamera(0.3, 1000.0, 0.5774, 1))) == 0
        if kind == "reserved":
            assert self.lib.meao_reserve_layers(h, max_layers) == 1
        assert self.lib.meao_resize(h, W, H) == 1

    def check(self, rc):
        if rc < 0:
            raise RuntimeError(self.lib.meao_last_error(self.h).decode())
        return rc

    def set_layers(self, n):
        """The count this arm renders for n views, its cameras and (split) its viewports; True if the count changed."""
        n = self.max_layers if self.kind == "fixed" else n
        changed = self.check(self.lib.meao_set_layers(self.h, n)) == 1
        self.check(self.lib.meao_set_layer_cameras(self.h, cams(n), n))
        return n, changed

    def close(self):
        self.lib.meao_destroy(self.h)


def run_split(torch, ctx, depth, ao, stream, keep):
    """One pass of the split-screen schedule; returns (host µs of each change frame, device ms of the schedule)."""
    N, lib = ctx.N, ctx.lib
    s = C.c_void_p(stream.cuda_stream)
    host, kept = [], []
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    for players in PLAYERS:
        for f in range(FRAMES_PER_PHASE):
            t0 = time.perf_counter()
            if f == 0:
                n, _ = ctx.set_layers(players)
                views = (N.MeaoLayerViewport * n)(*[N.MeaoLayerViewport(x, y, 0, x, y, 0) for (x, y) in QUADS[:n]])
                ctx.check(lib.meao_set_layer_viewports(ctx.h, views, n))
            ctx.check(lib.meao_render_pitched(ctx.h, C.c_void_p(depth.data_ptr()), 2 * W * 4, 2 * W * 2 * H * 4, 0,
                                              C.c_void_p(ao.data_ptr()), 2 * W, 2 * W * 2 * H, s))
            if f == 0:
                host.append((time.perf_counter() - t0) * 1e6)
                if keep:
                    with torch.cuda.stream(stream):
                        kept.append(torch.cat([ao[y:y + H, x:x + W].reshape(-1) for (x, y) in QUADS[:players]]).clone())
    end.record(stream)
    torch.cuda.synchronize()
    return host, start.elapsed_time(end), kept


def run_batches(torch, ctx, depth, outs, stream, keep):
    """One pass of the batch stream; returns (host µs of each change frame, device ms of the schedule)."""
    lib = ctx.lib
    s = C.c_void_p(stream.cuda_stream)
    host, kept = [], []
    I64 = C.c_int64
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    for _ in range(EPOCHS):
        for views in EPOCH:
            t0 = time.perf_counter()
            n, changed = ctx.set_layers(views)
            P = C.c_void_p * n
            ctx.check(lib.meao_render_batch(ctx.h, P(*[depth[l].data_ptr() for l in range(n)]), (I64 * n)(*[W * 4] * n), 0,
                                            P(*[outs[l].data_ptr() for l in range(n)]), (I64 * n)(*[W] * n), n, s))
            if changed or (ctx.kind == "fixed" and views != n):
                host.append((time.perf_counter() - t0) * 1e6)
            if keep and views != EPOCH[0]:
                with torch.cuda.stream(stream):
                    kept.append(outs[:views].clone())
    end.record(stream)
    torch.cuda.synchronize()
    return host, start.elapsed_time(end), kept


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    from miniengineao_b200 import synth
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    stream = torch.cuda.Stream()
    lin = synth.corridor(2 * W, 2 * H)
    depth_split = torch.from_numpy(synth.lin01_to_raw(lin).astype(np.float32)).cuda()
    ao_split = torch.zeros((2 * H, 2 * W), dtype=torch.uint8, device="cuda")
    one = torch.from_numpy(synth.lin01_to_raw(synth.corridor(W, H)).astype(np.float32)).cuda()
    depth_batch = torch.stack([torch.roll(one, 7 * l, dims=1) for l in range(64)]).contiguous()
    outs = torch.zeros((64, H, W), dtype=torch.uint8, device="cuda")

    for name, runner, max_layers, args_ in (("split", run_split, 4, (depth_split, ao_split)), ("batches", run_batches, 64, (depth_batch, outs))):
        arms = {k: Ctx(k, max_layers) for k in ("unreserved", "reserved", "fixed")}
        kept = {}
        for k, c in arms.items():                                   # warm-up pass: every (W, H, L) planned, every graph captured
            kept[k] = runner(torch, c, *args_, stream, keep=k != "fixed")[2]
        same = all(torch.equal(a, b) for a, b in zip(kept["unreserved"], kept["reserved"])) and len(kept["unreserved"]) == len(kept["reserved"])
        del kept
        host = {k: [] for k in arms}
        dev = {k: [] for k in arms}
        for r in range(args.rounds):
            order = list(arms) if r % 2 == 0 else list(arms)[::-1]
            for k in order:
                h, ms, _ = runner(torch, arms[k], *args_, stream, keep=False)
                host[k] += h
                dev[k].append(ms)
        res = {"schedule": name, "rounds": args.rounds, "ao_identical_a_b": bool(same)}
        for k in arms:
            res[k] = {"change_frame_host_us_median": float(np.median(host[k])) if host[k] else None,
                      "change_frame_host_us_max": float(np.max(host[k])) if host[k] else None,
                      "schedule_device_ms_median": float(np.median(dev[k])), "schedule_device_ms_min": float(np.min(dev[k])),
                      "schedule_device_ms_max": float(np.max(dev[k]))}
            r_ = arms[k].N.MeaoReservation()
            arms[k].lib.meao_reservation(arms[k].h, C.byref(r_))
            res[k]["arena_allocations"] = int(r_.arena_allocations)
            res[k]["graph_instantiations"] = int(r_.graph_instantiations)
        print(json.dumps(res), flush=True)
        for c in arms.values():
            c.close()


if __name__ == "__main__":
    main()
