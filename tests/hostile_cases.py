"""The hostile-input case table shared by tests/test_hostile_inputs_emulated.py (fiber emulator) and tests/test_hostile_inputs_gpu.py
(H100): depth values, cameras and parameters at and beyond the edges of the range the kernels' fast paths are guarded for.

Every fast path in the kernels replaces IEEE division by a reciprocal that is only valid for positive normal operands in
[2^-60, 2^60) and tests that range once for a whole group (eight pixels of linearize8, a render pair, four upsample texels, the
bilateral pair sums); outside it the group must take the plain IEEE operators and give the oracle's bits.  So the values below sit at
every lane of those groups, at tile seams, on the texels LowDepth1..4 sample, in solid blocks and in a checkerboard with ordinary
depth.  The comparison helper treats two NaNs as equal whatever their sign or payload (the GPU returns the canonical NaN, the oracle
keeps payloads) and everything else -- signed zeros and infinities included -- bit for bit."""
from __future__ import annotations

import math

import numpy as np

from miniengineao_b200 import synth


def f32(bits: int) -> np.float32:
    return np.array([bits], np.uint32).view(np.float32)[0]


def _ulp_below(x: float) -> np.float32:
    return np.nextafter(np.float32(x), np.float32(0))


# ---- depth values -------------------------------------------------------------------------------------------------------------
# linear f32 ingest: the value reaches LowDepth<k> unchanged and LinearDepth as f16
LINEAR = np.array([
    0.0, -0.0, -1e-3, -0.5, -1e30,
    f32(0x000116c2), -f32(0x000116c2), f32(0x00000001),     # subnormals: +-1e-40, 1e-45
    2.0 ** -61, 1e-30, 2.0 ** -60, _ulp_below(2.0 ** -60),
    _ulp_below(2.0 ** 60), 2.0 ** 60, 1e30,
    65504.0, 65519.99, 65520.0, 7e4, 1e5,                                  # f16 max, the rounding edge to inf, beyond
    3e-8, 1e-5,                                                            # f16-subnormal lin01
    np.inf, -np.inf,
    f32(0x7fc00000), f32(0xffc00000), f32(0x7f800001),                     # NaN: quiet, negative quiet, signalling pattern
], np.float32)


def zero_crossing(zb, n_ulps: int = 3) -> np.ndarray:
    """Raw depths around the root of fma(zbx, d, zby) (the linearisation's denominator), computed in float64 from zbuffer_params():
    the nearest float32 and n_ulps float32 steps either side."""
    zbx, zby = float(zb[0]), float(zb[1])
    if zbx == 0 or not math.isfinite(zbx) or not math.isfinite(zby):
        return np.zeros(0, np.float32)
    d = np.float32(-zby / zbx)
    out = [d]
    lo = hi = d
    for _ in range(n_ulps):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        out += [lo, hi]
    return np.array(out, np.float32)


def raw_values(zb) -> np.ndarray:
    """Raw f32 ingest (either Z direction): the sky / far-plane sentinels, out-of-range depths, specials, and the values where the
    linearisation's denominator crosses zero for this camera."""
    base = np.array([0.0, -0.0, 1.0, 2.0, -1.0, f32(0x000116c2), f32(0x7fc00000), np.inf, -np.inf], np.float32)
    return np.concatenate([base, zero_crossing(zb)])


def unorm_codes(bits: int) -> np.ndarray:
    """D16 / D24 sentinels: code 0 and 2^n - 1 (sky in one Z direction, the far plane in the other)."""
    return np.array([0, (1 << bits) - 1], np.uint32)


STENCILS = (0x00, 0xFF)


# ---- placement ------------------------------------------------------------------------------------------------------------------
def salt(base: np.ndarray, values: np.ndarray, seed: int = 0) -> np.ndarray:
    """`base` [H, W] with `values` placed where the grouped guards can go wrong:
      * rows 0, 1 and H - 1: value i at x = i (mod 8) of consecutive 8-pixel groups, so each value lands on every lane of a linearize8
        group, including the partial last group when W % 8 != 0; pairs (2m, 2m + 1) of equal and of different values
      * single pixels on the lattice of multiples of 16 (sampled by LowDepth1..4 at every level) and on their right neighbour
      * the tile seams x = 63 / 64 / 65 and y = 31 / 32 / 33
      * a solid 48 x 48 block aligned to 16 (whole texels of every level; more where the frame is larger)
      * a checkerboard of values and ordinary depth, so in-range and out-of-range lanes share one group"""
    H, W = base.shape
    a = base.astype(base.dtype, copy=True)
    v = np.asarray(values, dtype=base.dtype)
    n = len(v)
    rng = np.random.default_rng(seed)
    for y in {0, 1 % H, H - 1}:
        for x in range(W):
            g, lane = divmod(x, 8)
            if y == 0:
                a[y, x] = v[(g + lane) % n]                   # value (g + lane) at lane `lane`: each value visits each lane
            elif y == 1 % H:
                a[y, x] = v[(x // 2) % n]                     # equal pairs
            else:
                a[y, x] = v[(g * 3 + lane * 5) % n]
    ys, xs = np.meshgrid(np.arange(0, H, 16), np.arange(0, W, 16), indexing="ij")
    k = rng.integers(0, n, size=ys.shape)
    a[ys, xs] = v[k]
    right = xs + 1 < W
    a[ys[right], xs[right] + 1] = v[(k[right] + 1) % n]
    for x in (63, 64, 65):
        if x < W:
            a[2:H - 1:3, x] = v[(np.arange(2, H - 1, 3) + x) % n]
    for y in (31, 32, 33):
        if 1 < y < H - 1:
            a[y, 2::3] = v[(np.arange(2, W, 3) + y) % n]
    by, bx = min(32, max(0, H - 48)) // 16 * 16, min(48, max(0, W - 48)) // 16 * 16
    blk = max(48, (min(H, W) // 4) // 16 * 16)
    a[by:by + blk, bx:bx + blk] = v[rng.integers(0, n)]
    cy0, cx0 = H // 2, W // 2
    cb = a[cy0:cy0 + 24, cx0:cx0 + 40]
    yy, xx = np.indices(cb.shape)
    sel = (yy + xx) % 2 == 0
    cb[sel] = v[rng.integers(0, n, size=int(sel.sum()))]
    return a


def hostile_linear(W: int, H: int, seed: int = 0) -> np.ndarray:
    return salt(synth.random_depth(W, H, seed=seed).astype(np.float32), LINEAR, seed)


def hostile_raw(W: int, H: int, zb, reversed_z: bool, seed: int = 0) -> np.ndarray:
    raw = synth.lin01_to_raw(synth.random_depth(W, H, seed=seed), reversed_z=reversed_z).astype(np.float32)
    return salt(raw, raw_values(zb), seed)


def hostile_unorm(W: int, H: int, bits: int, reversed_z: bool, seed: int = 0):
    """(codes in the ingest format, the float32 the oracle sees): D16 (bits 16) or D24S8 words (bits 24, stencil 0x00 / 0xFF)."""
    raw = synth.lin01_to_raw(synth.random_depth(W, H, seed=seed), reversed_z=reversed_z).astype(np.float64)
    full = (1 << bits) - 1
    codes = salt(np.clip(np.rint(raw * full), 1, full - 1).astype(np.uint32), unorm_codes(bits), seed)
    seen = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
    if bits == 16:
        return codes.astype(np.uint16), seen
    stencil = np.where((np.indices(codes.shape).sum(axis=0) % 3) == 0, STENCILS[0], STENCILS[1]).astype(np.uint32)
    return codes | (stencil << np.uint32(24)), seen


# ---- cameras ------------------------------------------------------------------------------------------------------------------
def fov_for_tan_half_h(t: float, W: int, H: int) -> float:
    """Vertical field of view (degrees) whose tan_half_fov_h (aspect * tan(fov / 2)) is t."""
    return math.degrees(2.0 * math.atan(t * H / W))


# name -> (near, far, tan_half_fov_h or None for the default 60 degree camera)
CAMERAS = {
    "far_near_1p2m20": (1.0, 1.0 + 2.0 ** -20, None),       # far / near = 1 + 2^-20: ZBufferParams.x is 2^-20 (or -2^-20)
    "far_near_1e7": (0.01, 1e5, None),
    "far_near_overflows": (1e-30, 1e30, None),              # far / near overflows f32 to inf; the validator accepts it
    "tan_half_fov_1em6": (0.3, 100.0, 1e-6),
    "tan_half_fov_1e6": (0.3, 100.0, 1e6),
}


def camera(name: str, W: int, H: int, reversed_z: bool):
    from miniengineao_b200 import Camera
    near, far, t = CAMERAS[name]
    kw = {} if t is None else {"fieldOfView": fov_for_tan_half_h(t, W, H)}
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, **kw)


def oracle_camera_kw(cam) -> dict:
    return dict(near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00, reversed_z=cam.usesReversedZBuffer)


# ---- parameters ---------------------------------------------------------------------------------------------------------------
# upsample_tolerance -16.55 / -16.56 put 10^x on either side of 2^-55; 0 and +20 (10^20 >= 2^60) on either side of the top;
# noise_filter_tolerance 15.65 / 15.66 put noise_filter_strength on either side of 2^-52
PARAMS = [
    dict(upsample_tolerance=-16.55), dict(upsample_tolerance=-16.56), dict(upsample_tolerance=0.0), dict(upsample_tolerance=20.0),
    dict(noise_filter_tolerance=15.65), dict(noise_filter_tolerance=15.66),
    dict(blur_tolerance=1.0), dict(blur_tolerance=-30.0),
    dict(thickness_modifier=1e-6), dict(thickness_modifier=1e6), dict(intensity=100.0),
]


def fast_div_ok(tol: float, nfs: float) -> bool:
    """upsample_fast_div_ok (csrc/kernels.h) stated in float64: 2^-55 <= tol < 2^60 and 2^-52 <= nfs < 2^58."""
    return 2.0 ** -55 <= tol < 2.0 ** 60 and 2.0 ** -52 <= nfs < 2.0 ** 58


def fast_div_sides(plan) -> set:
    """Which side of upsample_fast_div_ok the plan's four upsample levels fall on, from upsample_constants()."""
    out = set()
    for lo in range(1, 5):
        uc = plan.upsample_constants(lo)
        out.add(fast_div_ok(float(uc["upsample_tolerance"]), float(uc["noise_filter_strength"])))
    return out


# ---- comparison -----------------------------------------------------------------------------------------------------------------
def n_diff(got: np.ndarray, ref: np.ndarray) -> int:
    """Elements that differ: unorm8 codes exactly; f16 / f32 bit for bit, except that any two NaNs match."""
    if got.dtype == np.uint8:
        return int((got != ref).sum())
    if got.dtype == np.float16:
        with np.errstate(over="ignore", invalid="ignore"):
            ref = np.asarray(ref).astype(np.float16)
        same = got.view(np.uint16) == ref.view(np.uint16)
    else:
        ref = np.asarray(ref, np.float32)
        same = got.view(np.uint32) == ref.view(np.uint32)
    return int((~(same | (np.isnan(got) & np.isnan(ref)))).sum())


def buffer_ids(high_quality_mask: int = 0, single_scale: bool = False) -> list:
    if single_scale:
        return [1, 2, 3, 4, 5, 10, 17]
    return list(range(1, 18)) + [17 + k for k in range(1, 5) if (high_quality_mask >> (k - 1)) & 1]


def compare_buffers(get, orc, tag: str, ids) -> None:
    """get(bid) -> the kernel's buffer; orc: an Oracle that has run the same frame."""
    bad = []
    for bid in ids:
        got = get(bid)
        ref = orc.codes(bid) if got.dtype == np.uint8 else orc.buffer(bid)
        n = n_diff(got, ref)
        if n:
            bad.append((bid, n, got.size))
    assert not bad, f"{tag}: mismatching buffers (id, #diff, size): {bad}"
