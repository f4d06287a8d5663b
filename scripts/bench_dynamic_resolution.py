"""The cost of a dynamic-resolution size change, with and without a reservation (meao_reserve), at a 3840 x 2160 target.

One context renders frames back to back on one stream from a max-size depth target (synthetic corridor depth) into a max-size AO
target, each frame a corner view rt[:h, :w] through meao_render_pitched, after meao_resize(w, h).  Arms, alternated over rounds:
  (a) unreserved  meao_resize re-allocates at every size change (what a host did before meao_reserve)
  (b) reserved    meao_reserve(3840, 2160) once; a size change inside it allocates and synchronises nothing
  (c) fixed       3840 x 2160 every frame: the floor
Schedules:
  stepped     scale 1.0 -> 0.7 -> 1.0 in steps of 0.1, a change every 4 frames, 400 frames
  continuous  a new width every frame, 8 px apart (3840 -> 1920 -> 3840, height at 16:9), 480 frames
Per arm: frame times from a host clock around resize + frame + stream synchronise (median, max), the mean extra cost of a change frame
over the median steady frame (stepped only; for (b) split into the first visit of a size and a revisit), and the back-to-back time of the whole
schedule (one synchronise at the end, CUDA events) -- where a device synchronise inside a resize ends CPU/GPU overlap.  The last AO
frame of (a) and (b) is compared bit for bit at every size of the schedule.  Prints the GPU's name and power limit, then one JSON line
per schedule.

    python scripts/bench_dynamic_resolution.py [--rounds 3]
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

MAXW, MAXH = 3840, 2160


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def schedule(name: str) -> list:
    if name == "stepped":
        scales = [1.0, 0.9, 0.8, 0.7, 0.8, 0.9]
        return [(int(MAXW * scales[(i // 4) % 6] + 0.5), int(MAXH * scales[(i // 4) % 6] + 0.5)) for i in range(400)]
    widths = [MAXW - 8 * i for i in range(240)] + [1920 + 8 * i for i in range(240)]
    return [(w, w * 9 // 16) for w in widths]


class Arm:
    def __init__(self, torch, kind: str):
        from miniengineao_b200 import _native as N
        self.N, self.lib, self.kind = N, N.lib(), kind
        h = C.c_void_p()
        assert self.lib.meao_create(C.byref(N.MeaoDeviceCfg(0, 0)), C.byref(h)) == 0
        self.ctx = h
        if kind == "reserved":
            assert self.lib.meao_reserve(h, MAXW, MAXH) == 1
        self.seen = set()

    def frame(self, w, h, depth, out, stream):
        lib = self.lib
        if self.kind == "fixed":
            w, h = MAXW, MAXH
        assert lib.meao_resize(self.ctx, w, h) >= 0
        rc = lib.meao_render_pitched(self.ctx, C.c_void_p(depth.data_ptr()), MAXW * 4, MAXW * MAXH * 4, 0, C.c_void_p(out.data_ptr()), MAXW,
                                     MAXW * MAXH, stream)
        assert rc == 0, lib.meao_last_error(self.ctx)

    def reservation(self):
        r = self.N.MeaoReservation()
        self.lib.meao_reservation(self.ctx, C.byref(r))
        return r

    def close(self):
        self.lib.meao_destroy(self.ctx)


def run_synced(torch, arm, sched, depth, out, s):
    """Per-frame host times (ms) around resize + frame + synchronise; per frame: was it a size change, a first visit?"""
    sh = C.c_void_p(s.cuda_stream)
    times, change, first = [], [], []
    prev = None
    for (w, h) in sched:
        key = (w, h) if arm.kind != "fixed" else (MAXW, MAXH)
        t0 = time.perf_counter()
        arm.frame(w, h, depth, out, sh)
        s.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        change.append(prev is not None and key != prev)
        first.append(key not in arm.seen)
        arm.seen.add(key)
        prev = key
    return np.array(times), np.array(change), np.array(first)


def run_back_to_back(torch, arm, sched, depth, out, s):
    sh = C.c_void_p(s.cuda_stream)
    s.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record(s)
    for (w, h) in sched:
        arm.frame(w, h, depth, out, sh)
    e1.record(s)
    s.synchronize()
    return (time.perf_counter() - t0) * 1e3, e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from miniengineao_b200 import synth
    assert torch.cuda.is_available(), "needs a GPU"
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    depth = torch.from_numpy(synth.lin01_to_raw(synth.corridor(MAXW, MAXH)).astype(np.float32)).cuda()
    s = torch.cuda.Stream()
    for name in ("stepped", "continuous"):
        sched = schedule(name)
        arms = {k: Arm(torch, k) for k in ("unreserved", "reserved", "fixed")}
        outs = {k: torch.zeros((MAXH, MAXW), dtype=torch.uint8, device="cuda") for k in arms}
        stats = {k: {"synced": [], "b2b_host": [], "b2b_dev": []} for k in arms}
        for r in range(args.rounds):
            for k, arm in arms.items():
                stats[k]["synced"].append(run_synced(torch, arm, sched, depth, outs[k], s))
                th, td = run_back_to_back(torch, arm, sched, depth, outs[k], s)
                stats[k]["b2b_host"].append(th)
                stats[k]["b2b_dev"].append(td)
        # (a) and (b) produce the same AO at every size of the schedule
        identical = True
        for (w, h) in sorted(set(sched)):
            for k in ("unreserved", "reserved"):
                arms[k].frame(w, h, depth, outs[k], C.c_void_p(s.cuda_stream))
            s.synchronize()
            identical &= bool(torch.equal(outs["unreserved"][:h, :w], outs["reserved"][:h, :w]))
        res = {"schedule": name, "frames": len(sched), "rounds": args.rounds, "gpu": info["name"], "power_limit_w": info["power_limit_w"],
               "ao_identical_unreserved_vs_reserved": identical}
        for k in arms:
            t = np.concatenate([x[0] for x in stats[k]["synced"]])
            ch = np.concatenate([x[1] for x in stats[k]["synced"]])
            fv = np.concatenate([x[2] for x in stats[k]["synced"]])
            steady = float(np.median(t[~ch])) if (~ch).any() else float("nan")
            d = {"median_ms": round(float(np.median(t)), 4), "max_ms": round(float(t.max()), 3), "steady_median_ms": round(steady, 4),
                 "b2b_host_ms": round(float(np.median(stats[k]["b2b_host"])), 2), "b2b_device_ms": round(float(np.median(stats[k]["b2b_dev"])), 2),
                 "b2b_spread_ms": round(float(np.ptp(stats[k]["b2b_host"])), 2)}
            if ch.any() and (~ch).sum() >= 10:             # the continuous schedule has no steady frames to compare with
                d["change_extra_ms"] = round(float(t[ch].mean() - steady), 4)
                if (ch & fv).any():
                    d["change_extra_first_visit_ms"] = round(float(t[ch & fv].mean() - steady), 4)
                if (ch & ~fv).any():
                    d["change_extra_revisit_ms"] = round(float(t[ch & ~fv].mean() - steady), 4)
            r = arms[k].reservation()
            d["arena_allocations"], d["graph_instantiations"], d["graphs_held"] = r.arena_allocations, r.graph_instantiations, r.graphs_held
            res[k] = d
        for arm in arms.values():
            arm.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
