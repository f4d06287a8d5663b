"""Several cameras, each with its own targets: N views of 1920 x 1080 as one batch (meao_render_arrays_batch / meao_render_batch) against
the recipes without it, in microseconds of device time per frame of all N views.

Every view has its own depth and AO resource and its own camera.  Arms, each one frame of all views:
  (a) batch    one context with N layers and a camera table: one call over the list, 9 launches
  (b) one      N single-layer contexts, one call each on one stream (meao_render_arrays / meao_render)
  (c) streams  the same N contexts, each on its own stream, joined back to the first
  (d) copy     a copy of every view into one stacked allocation (a layered array / a [N, H, W] tensor), one layered frame of the
               N-layer context, and a copy of every view's AO back out
for CUDA arrays (2-D arrays, registered once) and for device buffers (separate torch tensors).  The arms alternate inside each round;
a round times `frames` back-to-back frames with CUDA events; the median over the rounds is reported, with every round's value.  The
AO of (a) is compared bit for bit with (b)'s.

Prints the GPU's name and power limit, read in the same run, then one JSON line per measurement.

    python scripts/bench_batch.py [--rounds 7] [--frames 200] [--views 4 8 64]
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
D2D = 3


def gpu_info() -> dict:
    f = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip().split(",")
    return {"name": f[0].strip(), "power_limit_w": float(f[1])}


def context(lib, W, H, L, cams):
    from miniengineao_b200 import _native as N
    h = C.c_void_p()
    assert lib.meao_create(C.byref(N.MeaoDeviceCfg(0, 0)), C.byref(h)) == 0
    assert lib.meao_set_layers(h, L) >= 0 and lib.meao_resize(h, W, H) >= 0
    t = (N.MeaoCamera * L)(*[N.MeaoCamera(n, f, t, 1) for n, f, t in cams])
    assert lib.meao_set_layer_cameras(h, t, L) >= 0, lib.meao_last_error(h)
    return h


class Setup:
    """N views of W x H, each in its own resource, and the contexts and staging of the four arms."""

    def __init__(self, torch, rt, N_, W, H, io):
        from gpu_harness import Array
        from miniengineao_b200 import _native as Nat
        import harness
        self.torch, self.rt, self.N, self.W, self.H, self.io, self.lib = torch, rt, N_, W, H, io, Nat.lib()
        cams = [CAMS[i % len(CAMS)] for i in range(N_)]
        depth = [harness.frames(W, H, 1, seed=i)[0] for i in range(N_)]
        if io == "arrays":
            self.da = [Array(rt, W, H, np.float32) for _ in range(N_)]
            self.aa = [Array(rt, W, H, np.uint8) for _ in range(N_)]
            for a, d in zip(self.da, depth):
                a.fill(d[None])
            self.sd, self.sa = Array(rt, W, H, np.float32, "layered", N_), Array(rt, W, H, np.uint8, "layered", N_)
            self.d = (C.c_void_p * N_)(*[a.handle for a in self.da])
            self.a = (C.c_void_p * N_)(*[a.handle for a in self.aa])
        else:
            self.dt = [torch.from_numpy(d).cuda() for d in depth]
            self.at = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(N_)]
            self.sd = torch.empty((N_, H, W), dtype=torch.float32, device="cuda")
            self.sa = torch.empty((N_, H, W), dtype=torch.uint8, device="cuda")
            self.d = (C.c_void_p * N_)(*[t.data_ptr() for t in self.dt])
            self.a = (C.c_void_p * N_)(*[t.data_ptr() for t in self.at])
            self.zero = (C.c_int64 * N_)(*([0] * N_))
        self.batch = context(self.lib, W, H, N_, cams)
        self.single = [context(self.lib, W, H, 1, [cams[i]]) for i in range(N_)]
        self.streams = [torch.cuda.Stream() for _ in range(N_)]
        if io == "arrays":
            from gpu_harness import Extent, Memcpy3DParms, Pos
            self.copies_in, self.copies_out = [], []
            for i in range(N_):
                p = Memcpy3DParms()
                p.srcArray, p.dstArray, p.dstPos, p.extent, p.kind = self.da[i].handle, self.sd.handle, Pos(0, 0, i), Extent(W, H, 1), D2D
                self.copies_in.append(p)
                q = Memcpy3DParms()
                q.srcArray, q.srcPos, q.dstArray, q.extent, q.kind = self.sa.handle, Pos(0, 0, i), self.aa[i].handle, Extent(W, H, 1), D2D
                self.copies_out.append(q)
            rt.cudaMemcpy3DAsync.argtypes = [C.POINTER(Memcpy3DParms), C.c_void_p]

    def _one(self, ctx, i, s):
        if self.io == "arrays":
            rc = self.lib.meao_render_arrays(ctx, C.c_void_p(self.da[i].handle), 0, C.c_void_p(self.aa[i].handle), s)
        else:
            rc = self.lib.meao_render(ctx, C.c_void_p(self.dt[i].data_ptr()), 0, C.c_void_p(self.at[i].data_ptr()), s)
        assert rc == 0, self.lib.meao_last_error(ctx)

    def frame(self, arm, s):
        torch, lib = self.torch, self.lib
        if arm == "batch":
            if self.io == "arrays":
                rc = lib.meao_render_arrays_batch(self.batch, self.d, 0, self.a, self.N, s)
            else:
                rc = lib.meao_render_batch(self.batch, self.d, self.zero, 0, self.a, self.zero, self.N, s)
            assert rc == 0, lib.meao_last_error(self.batch)
        elif arm == "one":
            for i, c in enumerate(self.single):
                self._one(c, i, s)
        elif arm == "streams":
            main = torch.cuda.current_stream()
            for i, c in enumerate(self.single):
                st = self.streams[i]
                st.wait_stream(main)
                self._one(c, i, C.c_void_p(st.cuda_stream))
            for st in self.streams:
                main.wait_stream(st)
        elif self.io == "arrays":
            for p in self.copies_in:
                assert self.rt.cudaMemcpy3DAsync(C.byref(p), s) == 0
            rc = lib.meao_render_arrays(self.batch, C.c_void_p(self.sd.handle), 0, C.c_void_p(self.sa.handle), s)
            assert rc == 0, lib.meao_last_error(self.batch)
            for p in self.copies_out:
                assert self.rt.cudaMemcpy3DAsync(C.byref(p), s) == 0
        else:
            torch.stack(self.dt, out=self.sd)
            rc = lib.meao_render(self.batch, C.c_void_p(self.sd.data_ptr()), 0, C.c_void_p(self.sa.data_ptr()), s)
            assert rc == 0, lib.meao_last_error(self.batch)
            torch._foreach_copy_(self.at, list(self.sa.unbind(0)))

    def ao(self):
        self.torch.cuda.synchronize()
        return np.stack([a.read()[0] for a in self.aa]) if self.io == "arrays" else np.stack([t.cpu().numpy() for t in self.at])

    def close(self):
        self.torch.cuda.synchronize()
        for c in [self.batch] + self.single:
            if self.io == "arrays":
                for a in self.da + self.aa + [self.sd, self.sa]:
                    self.lib.meao_release_array(c, C.c_void_p(a.handle))
            self.lib.meao_destroy(c)
        if self.io == "arrays":
            for a in self.da + self.aa + [self.sd, self.sa]:
                a.free()


def timed(torch, run, frames):
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(frames):
        run()
    s1.record()
    s1.synchronize()
    return 1000.0 * s0.elapsed_time(s1) / frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--views", type=int, nargs="+", default=[4, 8, 64])
    args = ap.parse_args()
    import torch
    from gpu_harness import runtime
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    rt = runtime()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    W, H = 1920, 1080
    arms = ("batch", "one", "streams", "copy")
    for n in args.views:
        for io in ("arrays", "pointers"):
            st = Setup(torch, rt, n, W, H, io)
            for arm in arms:
                for _ in range(3):
                    st.frame(arm, s)
            st.frame("one", s)
            ref = st.ao()
            st.frame("batch", s)
            same = bool(np.array_equal(st.ao(), ref))
            res = {a: [] for a in arms}
            for _ in range(args.rounds):
                for arm in arms:
                    res[arm].append(timed(torch, lambda: st.frame(arm, s), args.frames))
            med = {a: statistics.median(v) for a, v in res.items()}
            print(json.dumps({"case": f"{n} x 1080p", "io": io, "us_per_frame": {a: round(v, 1) for a, v in med.items()},
                              "rounds": {a: [round(x, 1) for x in v] for a, v in res.items()},
                              "speedup_vs_one": round(med["one"] / med["batch"], 3), "speedup_vs_streams": round(med["streams"] / med["batch"], 3),
                              "speedup_vs_copy": round(med["copy"] / med["batch"], 3), "ao_identical": same}), flush=True)
            st.close()


if __name__ == "__main__":
    main()
