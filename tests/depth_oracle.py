"""The oracles of a frame of hierarchy depth n (include/meao.h meao_set_hierarchy_depth).  Test infrastructure: not collected by pytest.

A frame of depth n renders levels 1..n (and the wide renders of the high_quality_mask bits <= n) and upsamples n..1; its first upsample
reads Occlusion<n> where the depth-4 frame's lo-level-4 upsample reads Occlusion4.  The oracles state this with their own stages:
  - run(o, depth, n): the thread-group oracle (oracle/meao_oracle.c) stage by stage.  Its upsample of lo level k < 4 reads Combined<k> as
    LoResAO1, so for n < 4 Combined<n> is first loaded with Occlusion<n> -- a buffer the frame of depth n never writes itself;
  - OrthoDepthOracle: the same walk over the orthographic oracle's render (tests/ortho_oracle.py);
  - direct(...): the global per-pixel restatement (oracle/direct_formulation.py) walked the same way, the independent cross-check.
At n = 4 each is its depth-4 frame, step for step."""
from __future__ import annotations

import numpy as np

import harness
from oracle import direct_formulation as D
from ortho_oracle import OrthoOracle, interleaved_tap, render_core, wide_tap


def written_ids(n, mask):
    """The buffers a frame of depth n writes: LinearDepth, LowDepth1..4 and their tiled views, Occlusion1..n, Combined1..n-1, the AO, and
    HighQuality<k> of the mask bits k <= n.  The others have unspecified contents."""
    return ([1, 2, 3, 4, 5, 6, 7, 8, 9] + [9 + k for k in range(1, n + 1)] + [13 + k for k in range(1, n)] + [17]
            + [17 + k for k in range(1, n + 1) if (mask >> (k - 1)) & 1])


def _upsample_chain(o, n):
    if n < 4:
        o.set_buffer(13 + n, o.buffer(9 + n))           # LoResAO1 of the first upsample: Occlusion<n>
    for lo in range(n, 0, -1):
        o.upsample(lo)


def run(o, depth, n, mask=0):
    """The frame of depth n on the Oracle `o` (constructed with high_quality_mask = mask); returns the AO codes."""
    o.downsample(np.ascontiguousarray(depth, np.float32))
    for k in range(1, n + 1):
        o.render(k)
    for k in range(1, n + 1):
        if (mask >> (k - 1)) & 1:
            o.render_wide(k)
    _upsample_chain(o, n)
    return o.ao_u8()


class DepthOracle:
    """A perspective Oracle (harness.oracle keywords) that runs frames of depth n; buffer() / codes() serve harness.compare_buffers."""

    def __init__(self, W, H, n, **kw):
        self.n, self.mask = n, int(kw.get("high_quality_mask", 0))
        self.o = harness.oracle(W, H, **kw)

    def run(self, depth):
        return run(self.o, depth, self.n, self.mask)

    def buffer(self, bid):
        return self.o.buffer(bid)

    def codes(self, bid):
        return self.o.codes(bid)


class OrthoDepthOracle(OrthoOracle):
    """OrthoOracle's frame at depth n: its projection-dependent steps, the perspective oracle's upsample chain of depth n."""

    def __init__(self, W, H, n, **kw):
        super().__init__(W, H, **kw)
        self.n = n

    def run(self, depth):
        from ortho_oracle import linearize
        lin = np.asarray(depth, np.float32) if self.linear else linearize(depth, self.near, self.far, self.reversed_z)
        o = self.o
        o.downsample(lin)
        exh = bool(self.kw.get("sample_exhaustively", False))
        hq = int(self.kw.get("high_quality_mask", 0))
        for k in range(1, 5):
            sw, sh = self.dims[k + 2]
            o.set_buffer(5 + k, D.tiled_view(o.buffer(1 + k), sw, sh, self.pad(k)))
        for k in range(1, self.n + 1):
            sw, sh = self.dims[k + 2]
            rc = o.render_constants(k)
            codes = render_core(interleaved_tap(o.buffer(1 + k), sw, sh, self.pad(k)), self.dims[k][::-1], self.inv_thickness(k),
                                rc["sample_weight"], rc["reject_fadeoff"], rc["intensity"], exh)
            o.set_buffer(9 + k, D._u8load(codes))
            if (hq >> (k - 1)) & 1:
                rw = o.render_constants(k, wide=True)
                codes = render_core(wide_tap(o.buffer(1 + k)), self.dims[k][::-1], self.inv_thickness(k, wide=True),
                                    rw["sample_weight"], rw["reject_fadeoff"], rw["intensity"], exh)
                o.set_buffer(17 + k, D._u8load(codes))
        _upsample_chain(o, self.n)
        return o.ao_u8()


def for_camera(cam, n, linear=False, threads=4, **kw):
    """The oracle of depth n for one layer with camera `cam`: orthographic or perspective."""
    if cam.orthographic:
        return OrthoDepthOracle(cam.pixelWidth, cam.pixelHeight, n, near=cam.nearClipPlane, far=cam.farClipPlane,
                                tan_half_fov_h_=1.0 / cam.projection00, reversed_z=cam.usesReversedZBuffer, linear=linear, threads=threads, **kw)
    return DepthOracle(cam.pixelWidth, cam.pixelHeight, n, camera=cam, linear=linear, threads=threads, **kw)


def direct(depth, render_consts, upsample_consts, zb, n, *, reversed_z=True, linear=False, exhaustive=False, high_quality_mask=0,
           render_consts_wide=None):
    """oracle/direct_formulation.py's whole pipe at depth n: {"occ", "hq", "comb"} like its run(return_all=True)."""
    H, W = depth.shape
    dims = D.level_dims(W, H)
    lin_h, low = D.prepare_depth(depth, zb, reversed_z, linear)
    pad12 = np.float32(0) if linear else (np.float32(1e5) if reversed_z else np.float32(np.float32(1) / np.float32(zb[1])))
    occ, hq, comb = [None] * 5, [None] * 5, [None] * 4
    for k in range(1, n + 1):
        sw, sh = dims[k + 2]
        occ[k] = D.render_ao(low[k], sw, sh, pad12 if k <= 2 else np.float32(0), render_consts[k], exhaustive)
        if (high_quality_mask >> (k - 1)) & 1:
            hq[k] = D.render_ao_wide(low[k], render_consts_wide[k], exhaustive)
    lo_ao = occ[n]
    for lo in range(n, 0, -1):
        hi = lo - 1
        comb[hi] = D.blur_upsample(low[lo], lo_ao, lin_h if hi == 0 else low[hi], None if hi == 0 else occ[hi], upsample_consts[lo], hq[lo])
        lo_ao = comb[hi]
    return {"occ": occ, "hq": hq, "comb": comb}
