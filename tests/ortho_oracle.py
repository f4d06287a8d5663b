"""The CPU oracle of an orthographic projection (include/meao.h meao_set_projection).  Test infrastructure: not collected by pytest.

Under an orthographic projection two steps of the pipe change, and this module states them:
  - linearisation: lin = fma(zb.x, d, zb.y) with zb = {1 - r, r} (reversed Z: {r - 1, 1}), r = near / far; the sky rule of DS1:41-44 and
    the atlas padding of levels 1-2 (the linearisation of raw depth 0: r, reversed 1e5) follow;
  - render: invRange = it_i = (far / ThicknessMultiplier) / SampleThickness[i] and -frontDepth = fma(-centre, it_i, 0.5), the disocclusion
    fma(S, it_i, -frontDepth); everything else of Render.compute:60-177 as in the perspective oracle.
Everything that does not depend on the projection -- the point-sampled mips, the blur and upsample, the debug views -- is the perspective
oracle's own code (oracle/meao_oracle.c, fed the linearised depth), so an orthographic frame differs from a perspective one exactly in the
two steps above.  The render is restated per pixel in numpy (the global form of oracle/direct_formulation.py) with an exact float32
fused multiply-add (fma32); tests/test_ortho_plan.py checks the restatement against meao_oracle.c with perspective constants.
"""
from __future__ import annotations

import numpy as np

from oracle import direct_formulation as D
from oracle.oracle import Oracle

F = np.float32


def fma32(a, b, c):
    """float32 fma(a, b, c), correctly rounded: the product is exact in float64, the sum is rounded to odd in float64 (TwoSum error
    term), and a round-to-odd result with 53 >= 24 + 2 bits rounds to the correctly rounded float32."""
    a, b, c = (np.asarray(x, F) for x in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)
        fix = np.isfinite(s) & np.isfinite(e) & (e != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(F)


def zbuffer_params(near, far, reversed_z):
    r = F(near) / F(far)
    return (F(r - F(1)), F(1)) if reversed_z else (F(F(1) - r), r)


def linearize(d, near, far, reversed_z):
    """Raw depth -> eye depth / far (float32), sky (d == 1, reversed d == 0) -> 1e5."""
    zx, zy = zbuffer_params(near, far, reversed_z)
    d = np.asarray(d, F)
    lin = fma32(zx, d, zy)
    return np.where(d == (F(0) if reversed_z else F(1)), F(1e5), lin).astype(F)


def thickness_multiplier(tan_half_fov_h, src_w, wide, stereo):
    """ThicknessMultiplier, AO.cs:671-683, in the float32 order the planner evaluates it."""
    tm = F(F(F(2) * F(tan_half_fov_h)) * F(10)) / F(src_w)
    if wide:
        tm = F(tm * F(2))                   # AO.cs:679 (!source.isTiled)
    if stereo:
        tm = F(tm * F(2))                   # AO.cs:680
    return tm


def inv_thickness(far, tan_half_fov_h, src_w, thick, wide=False, stereo=False):
    """it_i = (far / ThicknessMultiplier) / SampleThickness[i], the 12 table slots."""
    with np.errstate(over="ignore"):                     # a tiny half-width overflows it_i to inf, as the planner's float32 does
        irf = F(far) / thickness_multiplier(tan_half_fov_h, src_w, wide, stereo)
    return (irf / np.asarray(thick, F)).astype(F)


def render_core(tap, shape, it, weight, rf, intensity, exhaustive, perspective=False):
    """UNORM8 codes of one render level.  tap(di, dj): the source value at sample offset (di, dj) of every pixel (tap(0, 0): the centre as
    the reference's LDS holds it).  it / weight: the 12 table slots.  perspective=True evaluates the perspective formulas with the same
    code (invRange = it / centre, -frontDepth = -(it - 0.5)): the cross-check against meao_oracle.c."""
    lh, lw = shape
    rf, intensity = F(rf), F(intensity)
    ctr = tap(0, 0)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv = (F(1) / ctr).astype(F) if perspective else None

        def pair(ir, nf, ox, oy):                                                   # REN:60-75, the order of pair_eval2
            d1 = fma32(tap(ox, oy), ir, nf)
            d2 = fma32(tap(-ox, -oy), ir, nf)
            p1, p2 = D._sat((rf * d1).astype(F)), D._sat((rf * d2).astype(F))
            c1 = np.fmax(D._sat(d1), p2).astype(F)
            c2 = np.fmin(np.fmax(d2, p1), F(1)).astype(F)
            return D._sat(fma32(-p1, p2, (c1 + c2).astype(F)))

        ao = np.zeros((lh, lw), F)
        for idx, (x, y) in (D.SAMPLES_EXHAUSTIVE if exhaustive else D.SAMPLES_CHECKER):
            i = F(it[idx])
            if perspective:
                ir, nf = (i * inv).astype(F), np.full((lh, lw), -(i - F(0.5)), F)
            else:
                ir, nf = np.full((lh, lw), i, F), fma32(-ctr, i, F(0.5))
            if y == 0:
                g = (F(0.5) * (pair(ir, nf, x, 0) + pair(ir, nf, 0, x))).astype(F)
            elif x == y:
                g = (F(0.5) * (pair(ir, nf, -x, x) + pair(ir, nf, x, x))).astype(F)
            else:
                t = ((pair(ir, nf, x, y) + pair(ir, nf, -x, y)) + pair(ir, nf, y, x)) + pair(ir, nf, -y, x)
                g = (F(0.25) * t.astype(F)).astype(F)
            ao = fma32(F(weight[idx]), g, ao)
        out = fma32(intensity, (ao - F(1)).astype(F), F(1))                          # REN:176
    return D._unorm8(out)


def interleaved_tap(low_k, sw, sh, pad):
    """Kernel main_interleaved's taps: the f16 atlas of level k + 2 over LowDepth<k>, `pad` outside the level (SURVEY.md P3)."""
    lh, lw = low_k.shape
    lowh = D._f16r(np.asarray(low_k, F))
    padh = D._f16r(np.asarray(pad, F))
    Y, X = np.meshgrid(np.arange(lh), np.arange(lw), indexing="ij")
    I, J, SX, SY = X >> 2, Y >> 2, X & 3, Y & 3

    def tap(di, dj):
        cx = 4 * np.clip(I + di, 0, sw - 1) + SX
        cy = 4 * np.clip(J + dj, 0, sh - 1) + SY
        ok = (cx < lw) & (cy < lh)
        return np.where(ok, lowh[np.minimum(cy, lh - 1), np.minimum(cx, lw - 1)], padh).astype(F)
    return tap


def wide_tap(low_k):
    """Kernel main's taps: the f32 LowDepth<k> at twice the offsets, clamped to the level."""
    lh, lw = low_k.shape
    Y, X = np.meshgrid(np.arange(lh), np.arange(lw), indexing="ij")
    return lambda di, dj: np.asarray(low_k, F)[np.clip(Y + 2 * dj, 0, lh - 1), np.clip(X + 2 * di, 0, lw - 1)]


class OrthoOracle:
    """An oracle frame of W x H under an orthographic camera: near / far / tan_half_fov_h_ (the view volume's half-width) / reversed_z;
    linear: the input is eye depth / far already.  The other keywords are Oracle's (params and variants).  After run(depth), buffer() and
    codes() serve harness.compare_buffers, debug_view() the views."""

    def __init__(self, W, H, *, near=0.3, far=100.0, tan_half_fov_h_=5.0, reversed_z=True, linear=False, threads=4, **kw):
        self.W, self.H = W, H
        self.near, self.far, self.thfh, self.reversed_z, self.linear = F(near), F(far), F(tan_half_fov_h_), bool(reversed_z), linear
        self.kw = kw
        self.o = Oracle(W, H, depth_is_linear=True, near=near, far=far, tan_half_fov_h_=tan_half_fov_h_, reversed_z=reversed_z,
                        threads=threads, **kw)
        self.dims = D.level_dims(W, H)

    # the planner's constants under the projection
    def zbuffer_params(self):
        return np.array(zbuffer_params(self.near, self.far, self.reversed_z) + (0, 0), F)

    def inv_thickness(self, level, wide=False):
        src_w = self.dims[level][0] if wide else self.dims[level + 2][0]
        return inv_thickness(self.far, self.thfh, src_w, self.o.sample_thickness(), wide, self.kw.get("single_pass_stereo", False))

    def pad(self, level):
        """The f16-rounded atlas padding value of render level `level`."""
        if self.linear or level > 2:
            return F(0)
        return D._f16r(np.asarray(F(1e5) if self.reversed_z else zbuffer_params(self.near, self.far, False)[1], F))[()]

    def run(self, depth):
        lin = np.asarray(depth, F) if self.linear else linearize(depth, self.near, self.far, self.reversed_z)
        o = self.o
        o.downsample(lin)
        exh = bool(self.kw.get("sample_exhaustively", False))
        hq = int(self.kw.get("high_quality_mask", 0))
        levels = [1] if self.kw.get("single_scale", False) else [1, 2, 3, 4]
        for k in range(1, 5):
            sw, sh = self.dims[k + 2]
            o.set_buffer(5 + k, D.tiled_view(o.buffer(1 + k), sw, sh, self.pad(k)))       # TiledDepth<k> with this projection's padding
        for k in levels:
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
        for lo in levels[::-1]:
            o.upsample(lo)
        return o.ao_u8()

    def buffer(self, bid):
        return self.o.buffer(bid)

    def codes(self, bid):
        return self.o.codes(bid)

    def debug_view(self, bid):
        return self.o.debug_view(bid)
