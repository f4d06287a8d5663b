"""Split-screen in one frame: N players as the N layers of one context with a camera table and a viewport table
(meao_set_layer_viewports), against the recipe without it, in microseconds per frame.

The players share one depth target and one AO target: N views of W x H side by side (2 players: two 960 x 1080 halves of 1920 x 1080)
or in quadrants (4 players: four 1920 x 1080 quadrants of 3840 x 2160), each with its own camera.  Arms, each one frame of all players:
  (a) table    one context with N layers, the camera table and the viewport table: one call, 9 launches
  (b) one      N single-layer contexts, one call each on one stream (meao_render_arrays_at / meao_render_pitched at the player's
               rectangle): today's recipe, 9 N launches in order
  (c) streams  the same N contexts, each on its own stream, joined back to the first
for CUDA arrays (2-D arrays, registered once) and for pitched buffers (one depth image, one AO image).  The arms alternate inside each
round; a round times `frames` back-to-back frames with CUDA events; the median over the rounds is reported, with every round's value.
The AO of (a) and (b) is compared bit for bit.

--parent LIB: also time table-less fixed-size frames (meao_render_arrays and meao_render_pitched, 1080p and 4K, L = 1 and 2) of this
build against the library at LIB (the parent commit's libmeao.so, loaded side by side), alternating, and compare their AO bit for bit.

Prints the GPU's name and power limit, read in the same run, then one JSON line per measurement.

    python scripts/bench_layer_viewports.py [--rounds 7] [--frames 200] [--parent path/to/parent/libmeao.so]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CAMS = [(0.3, 100.0, 0.577), (0.1, 1000.0, 1.0), (0.5, 50.0, 0.364), (0.2, 300.0, 0.767)]     # near, far, tan(half horizontal fov)


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def load(path: str) -> C.CDLL:
    from miniengineao_b200 import _native as N
    l = C.CDLL(path)
    for name, (res, args) in N.SIGNATURES.items():
        if hasattr(l, name):
            getattr(l, name).restype, getattr(l, name).argtypes = res, args
    return l


def context(lib, W, H, L, cams):
    from miniengineao_b200 import _native as N
    h = C.c_void_p()
    assert lib.meao_create(C.byref(N.MeaoDeviceCfg(0, 0)), C.byref(h)) == 0
    assert lib.meao_set_layers(h, L) >= 0 and lib.meao_resize(h, W, H) >= 0
    if cams is not None:
        t = (N.MeaoCamera * L)(*[N.MeaoCamera(n, f, t, 1) for n, f, t in cams])
        assert lib.meao_set_layer_cameras(h, t, L) >= 0, lib.meao_last_error(h)
    return h


class Setup:
    """N players of W x H in one target of (cols x W) x (rows x H): arrays or pitched buffers, and the contexts of the three arms."""

    def __init__(self, torch, rt, N_, W, H, io):
        from gpu_harness import Array
        from miniengineao_b200 import _native as Nat
        import harness
        self.torch, self.N, self.W, self.H, self.io, self.lib = torch, N_, W, H, io, Nat.lib()
        cols, rows = (2, 1) if N_ == 2 else (2, 2)
        self.TW, self.TH = cols * W, rows * H
        self.org = [((i % cols) * W, (i // cols) * H) for i in range(N_)]
        depth = harness.frames(self.TW, self.TH, 1, seed=N_)[0]
        if io == "arrays":
            self.da, self.aa = Array(rt, self.TW, self.TH, np.float32), Array(rt, self.TW, self.TH, np.uint8)
            self.da.fill(depth[None])
            self.d, self.a = self.da.handle, self.aa.handle
        else:
            self.dt = torch.from_numpy(depth).cuda()
            self.at = torch.zeros((self.TH, self.TW), dtype=torch.uint8, device="cuda")
            self.d, self.a = self.dt.data_ptr(), self.at.data_ptr()
        cams = CAMS[:N_]
        self.table = context(self.lib, W, H, N_, cams)
        vt = (Nat.MeaoLayerViewport * N_)(*[Nat.MeaoLayerViewport(x, y, 0, x, y, 0) for x, y in self.org])
        assert self.lib.meao_set_layer_viewports(self.table, vt, N_) == 1
        self.single = [context(self.lib, W, H, 1, [cams[i]]) for i in range(N_)]
        self.streams = [torch.cuda.Stream() for _ in range(N_)]

    def _one(self, ctx, i, s):
        x, y = self.org[i]
        if self.io == "arrays":
            rc = self.lib.meao_render_arrays_at(ctx, C.c_void_p(self.d), x, y, 0, C.c_void_p(self.a), x, y, s)
        else:
            rc = self.lib.meao_render_pitched(ctx, C.c_void_p(self.d + 4 * (y * self.TW + x)), 4 * self.TW, 4 * self.TW * self.H, 0,
                                              C.c_void_p(self.a + y * self.TW + x), self.TW, self.TW * self.H, s)
        assert rc == 0, self.lib.meao_last_error(ctx)

    def frame(self, arm, s):
        if arm == "table":
            if self.io == "arrays":
                rc = self.lib.meao_render_arrays(self.table, C.c_void_p(self.d), 0, C.c_void_p(self.a), s)
            else:
                rc = self.lib.meao_render_pitched(self.table, C.c_void_p(self.d), 4 * self.TW, 4 * self.TW * self.TH, 0, C.c_void_p(self.a),
                                                  self.TW, self.TW * self.TH, s)
            assert rc == 0, self.lib.meao_last_error(self.table)
        elif arm == "one":
            for i, c in enumerate(self.single):
                self._one(c, i, s)
        else:
            torch = self.torch
            main = torch.cuda.current_stream()
            for i, c in enumerate(self.single):
                st = self.streams[i]
                st.wait_stream(main)
                self._one(c, i, C.c_void_p(st.cuda_stream))
            for st in self.streams:
                main.wait_stream(st)

    def ao(self):
        self.torch.cuda.synchronize()
        return self.aa.read()[0] if self.io == "arrays" else self.at.cpu().numpy()


def timed(torch, run, frames):
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(frames):
        run()
    s1.record()
    s1.synchronize()
    return 1000.0 * s0.elapsed_time(s1) / frames


def split_screen(torch, rt, args):
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for N_, W, H, label in ((2, 960, 1080, "2 players 1080p"), (4, 1920, 1080, "4 players 4K")):
        for io in ("arrays", "pitched"):
            st = Setup(torch, rt, N_, W, H, io)
            for arm in ("table", "one", "streams"):
                for _ in range(3):
                    st.frame(arm, s)
            st.frame("one", s)
            ref = st.ao()
            st.frame("table", s)
            same = bool(np.array_equal(st.ao(), ref))
            res = {a: [] for a in ("table", "one", "streams")}
            for _ in range(args.rounds):
                for arm in res:
                    res[arm].append(timed(torch, lambda: st.frame(arm, s), args.frames))
            med = {a: statistics.median(v) for a, v in res.items()}
            print(json.dumps({"case": label, "io": io, "us_per_frame": {a: round(v, 1) for a, v in med.items()},
                              "rounds": {a: [round(x, 1) for x in v] for a, v in res.items()},
                              "speedup_vs_one": round(med["one"] / med["table"], 3), "speedup_vs_streams": round(med["streams"] / med["table"], 3),
                              "ao_identical": same}), flush=True)


def parent_compare(torch, rt, args):
    """Table-less fixed-size frames: this build against the parent library, alternating, AO compared."""
    from gpu_harness import Array
    import harness
    libs = {"this": load(os.path.join(ROOT, "miniengineao_b200", "libmeao.so")), "parent": load(args.parent)}
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for W, H, L in ((1920, 1080, 1), (1920, 1080, 2), (3840, 2160, 1), (3840, 2160, 2)):
        depth = harness.frames(W, H, L, seed=L)
        for io in ("arrays", "pitched"):
            ctxs = {k: context(l, W, H, L, None) for k, l in libs.items()}
            if io == "arrays":
                shape = "2d" if L == 1 else "layered"
                da = Array(rt, W, H, np.float32, shape, L)
                da.fill(depth)
                outs = {k: Array(rt, W, H, np.uint8, shape, L) for k in libs}

                def run(k):
                    assert libs[k].meao_render_arrays(ctxs[k], C.c_void_p(da.handle), 0, C.c_void_p(outs[k].handle), s) == 0

                def read(k):
                    return outs[k].read()
            else:
                dt = torch.from_numpy(depth).cuda()
                outs = {k: torch.zeros((L, H, W), dtype=torch.uint8, device="cuda") for k in libs}

                def run(k):
                    assert libs[k].meao_render(ctxs[k], C.c_void_p(dt.data_ptr()), 0, C.c_void_p(outs[k].data_ptr()), s) == 0

                def read(k):
                    return outs[k].cpu().numpy()
            for k in libs:
                for _ in range(3):
                    run(k)
            torch.cuda.synchronize()
            same = bool(np.array_equal(read("this"), read("parent")))
            res = {k: [] for k in libs}
            for _ in range(args.rounds):
                for k in libs:
                    res[k].append(timed(torch, lambda: run(k), args.frames))
            med = {k: statistics.median(v) for k, v in res.items()}
            print(json.dumps({"case": f"{W}x{H} L={L} fixed", "io": io, "us_per_frame": {k: round(v, 1) for k, v in med.items()},
                              "rounds": {k: [round(x, 1) for x in v] for k, v in res.items()}, "ao_identical": same}), flush=True)
            torch.cuda.synchronize()
            for k, l in libs.items():
                if io == "arrays":
                    l.meao_release_array(ctxs[k], C.c_void_p(da.handle))
                    l.meao_release_array(ctxs[k], C.c_void_p(outs[k].handle))
                    outs[k].free()
                l.meao_destroy(ctxs[k])
            if io == "arrays":
                da.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--parent", default=None)
    args = ap.parse_args()
    import torch
    from gpu_harness import runtime
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    rt = runtime()
    split_screen(torch, rt, args)
    if args.parent:
        parent_compare(torch, rt, args)


if __name__ == "__main__":
    main()
