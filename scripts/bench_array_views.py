"""Dynamic resolution on interop textures: viewport frames (meao_render_arrays_at) against the copies a host needs without them, at a
3840 x 2160 maximum, in milliseconds per schedule.

One reserved context (meao_reserve(3840, 2160)) renders frames back to back on one stream; a frame is meao_resize(w, h) and then:
  (a) viewports  meao_render_arrays_at from and into the top-left w x h of one max-size depth / AO array pair, registered once
  (b) copies     today's workaround: copy the depth corner into an exact-size array (cudaMemcpy3DAsync, the stream-ordered
                 cudaMemcpy2DArrayToArray), meao_render_arrays, copy the AO back into the corner of the max-size AO array; the exact-size
                 arrays are released (meao_release_array, a device synchronise), freed and allocated again at every size change
  (c) fixed      3840 x 2160 meao_render_arrays frames on max-size arrays every frame: the floor
The schedules are those of scripts/bench_dynamic_resolution.py: stepped (scale 1.0 -> 0.7 -> 1.0 in steps of 0.1, a change every 4
frames, 400 frames) and continuous (a new width every frame, 8 px apart, 480 frames).  Per arm and schedule: the back-to-back time of the
whole schedule (CUDA events, one synchronise at the end) and the slowest frame (host clock around one frame and a stream synchronise),
the median over the rounds.  The last frame's AO corner of (a) and (b) is compared bit for bit.  Prints the GPU's name and power limit,
read in the same run, then one JSON line per schedule.

    python scripts/bench_array_views.py [--rounds 3]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

MAXW, MAXH = 3840, 2160
D2D = 3


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
    def __init__(self, rt, kind: str, depth_max, ao_max):
        from gpu_harness import Array
        from miniengineao_b200 import _native as N
        self.N, self.lib, self.rt, self.kind, self.Array = N, N.lib(), rt, kind, Array
        self.dmax, self.amax = depth_max, ao_max
        h = C.c_void_p()
        assert self.lib.meao_create(C.byref(N.MeaoDeviceCfg(0, 0)), C.byref(h)) == 0
        self.ctx = h
        assert self.lib.meao_reserve(h, MAXW, MAXH) == 1
        self.exact, self.exact_size = None, None

    def _copy(self, src, dst, w, h, s):
        from gpu_harness import Extent, Memcpy3DParms
        p = Memcpy3DParms()
        p.srcArray, p.dstArray, p.extent, p.kind = src, dst, Extent(w, h, 1), D2D
        assert self.rt.cudaMemcpy3DAsync(C.byref(p), s) == 0

    def frame(self, w, h, s):
        lib, ctx = self.lib, self.ctx
        if self.kind == "fixed":
            w, h = MAXW, MAXH
        assert lib.meao_resize(ctx, w, h) >= 0
        if self.kind == "viewports":
            rc = lib.meao_render_arrays_at(ctx, C.c_void_p(self.dmax.handle), 0, 0, 0, C.c_void_p(self.amax.handle), 0, 0, s)
        elif self.kind == "fixed":
            rc = lib.meao_render_arrays(ctx, C.c_void_p(self.dmax.handle), 0, C.c_void_p(self.amax.handle), s)
        else:
            if self.exact_size != (w, h):
                self._drop_exact()
                self.exact = (self.Array(self.rt, w, h, np.float32), self.Array(self.rt, w, h, np.uint8))
                self.exact_size = (w, h)
            de, ae = self.exact
            self._copy(self.dmax.handle, de.handle, w, h, s)
            rc = lib.meao_render_arrays(ctx, C.c_void_p(de.handle), 0, C.c_void_p(ae.handle), s)
            self._copy(ae.handle, self.amax.handle, w, h, s)
        assert rc == 0, lib.meao_last_error(ctx)

    def _drop_exact(self):
        if self.exact:
            for a in self.exact:
                self.lib.meao_release_array(self.ctx, C.c_void_p(a.handle))
                a.free()
        self.exact, self.exact_size = None, None

    def close(self):
        self._drop_exact()
        for a in (self.dmax, self.amax):
            self.lib.meao_release_array(self.ctx, C.c_void_p(a.handle))
        self.lib.meao_destroy(self.ctx)


def run_back_to_back(torch, arm, sched, s):
    sh = C.c_void_p(s.cuda_stream)
    s.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for (w, h) in sched:
        arm.frame(w, h, sh)
    e1.record(s)
    s.synchronize()
    return e0.elapsed_time(e1)


def slowest_frame(arm, sched, s):
    sh = C.c_void_p(s.cuda_stream)
    worst = 0.0
    for (w, h) in sched:
        t0 = time.perf_counter()
        arm.frame(w, h, sh)
        s.synchronize()
        worst = max(worst, (time.perf_counter() - t0) * 1e3)
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    from gpu_harness import Array, runtime
    from miniengineao_b200 import synth
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    rt = runtime()
    rt.cudaMemcpy3DAsync.argtypes = [C.c_void_p, C.c_void_p]
    dmax, amax = Array(rt, MAXW, MAXH, np.float32), Array(rt, MAXW, MAXH, np.uint8)
    dmax.fill(synth.lin01_to_raw(synth.corridor(MAXW, MAXH)).astype(np.float32))
    s = torch.cuda.Stream()
    for name in ("stepped", "continuous"):
        sched = schedule(name)
        res = {k: {"ms": [], "slowest_ms": []} for k in ("viewports", "copies", "fixed")}
        last = {}
        for r in range(args.rounds):
            for kind in res:
                arm = Arm(rt, kind, dmax, amax)
                for (w, h) in sched[:8]:                # warm-up: the first sizes' graphs
                    arm.frame(w, h, C.c_void_p(s.cuda_stream))
                res[kind]["ms"].append(run_back_to_back(torch, arm, sched, s))
                res[kind]["slowest_ms"].append(slowest_frame(arm, sched, s))
                w, h = sched[-1]
                if kind != "fixed":
                    last[kind] = amax.read()[0, :h, :w].copy()
                arm.close()
        out = {"schedule": name, "frames": len(sched), "rounds": args.rounds,
               "ao_identical": bool(np.array_equal(last["viewports"], last["copies"]))}
        for kind, v in res.items():
            out[kind] = {"ms": round(float(np.median(v["ms"])), 2), "ms_spread": round(float(np.ptp(v["ms"])), 2),
                         "slowest_frame_ms": round(float(np.median(v["slowest_ms"])), 3)}
        print(json.dumps(out), flush=True)
    dmax.free()
    amax.free()


if __name__ == "__main__":
    main()
