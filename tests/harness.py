"""Shared CPU helpers of the test suite: contexts, oracles, depth inputs and the bit-exact buffer comparison.  Every test module and
script takes these from here, so a change to one of them changes every test that uses it knowingly.  No torch here: the CPU-only
tests import this module.  Nothing in it is collected by pytest."""
import ctypes as C
import os

import numpy as np

from miniengineao_b200 import AmbientOcclusion, Camera, synth
from miniengineao_b200 import _native as N
from oracle.oracle import Oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the MeaoParams fields: the oracle's keyword (also the name tests use) -> the AmbientOcclusion property
PARAMS = {"noise_filter_tolerance": "noiseFilterTolerance", "blur_tolerance": "blurTolerance", "upsample_tolerance": "upsampleTolerance",
          "thickness_modifier": "thicknessModifier", "intensity": "intensity"}
PROPERTIES = {v: k for k, v in PARAMS.items()}


# ---- contexts and oracles ---------------------------------------------------------------------------------------------------------
def context(camera, H=None, *, device=-1, layers=1, layer_cameras=None, use_graph=True, stereo=False, max_resolution=None,
            reversed_z=True, sample_exhaustively=False, high_quality_mask=0, single_scale=False, **params):
    """An AmbientOcclusion (device -1: plan only) for `camera`, or for a Camera(W, H) when called as context(W, H, ...): then stereo
    makes W the double-wide eye pair of a W / 2 stereo camera and reversed_z is its Z direction.  stereo also registers one draw of
    both eyes (OnPreRender).  params: the MeaoParams fields by their PARAMS names."""
    if H is not None:
        camera = Camera(camera // 2 if stereo else camera, H, stereoEnabled=stereo, usesReversedZBuffer=reversed_z)
    unknown = set(params) - set(PARAMS)
    if unknown:
        raise TypeError(f"context() got unknown keywords {sorted(unknown)}")
    ao = AmbientOcclusion(camera, device=device, use_graph=use_graph)
    for py, prop in PARAMS.items():
        if py in params:
            setattr(ao, prop, params[py])
    ao.sampleExhaustively, ao.highQualityMask, ao.singleScale = sample_exhaustively, high_quality_mask, single_scale
    ao.layers, ao.layerCameras, ao.maxResolution = layers, layer_cameras, max_resolution
    if stereo:
        ao.OnPreRender()
    return ao


def oracle_camera_kw(cam) -> dict:
    return dict(near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00, reversed_z=cam.usesReversedZBuffer)


def oracle(W, H, *, camera=None, linear=False, stereo=False, threads=4, **kw):
    """An Oracle of W x H.  camera: take its near / far / field of view / Z direction (None: the oracle's own default camera, with
    reversed_z from kw); linear: linear depth in; stereo: single-pass stereo; kw: the other Oracle keywords (params, variants)."""
    if camera is not None:
        kw.update(oracle_camera_kw(camera))
    if linear:
        kw["depth_is_linear"] = True
    if stereo:
        kw["single_pass_stereo"] = True
    return Oracle(W, H, threads=threads, **kw)


def context_and_oracle(W, H, *, device=0, use_graph=True, single_pass_stereo=False, threads=8, **kw):
    """context(W, H) and an oracle with the same params, variants and Z direction; the oracle keeps its default camera, except that
    under single-pass stereo (W the double-wide eye pair) it takes the eye camera's field of view."""
    ao = context(W, H, device=device, use_graph=use_graph, stereo=single_pass_stereo, **kw)
    if single_pass_stereo:
        kw["tan_half_fov_h_"] = 1.0 / ao.camera.projection00
    return ao, oracle(W, H, stereo=single_pass_stereo, threads=threads, **kw)


# ---- depth inputs -----------------------------------------------------------------------------------------------------------------
def contrasting_layers(W, H, n, seed=0):
    """Linear depth in [0, 1) of n layers that differ sharply at every boundary; layer 2 carries a sky patch (raw depth 0)."""
    out = []
    for i in range(n):
        kind = i % 4
        if kind == 0:
            lin = synth.corridor(W, H, frame=i)
        elif kind == 1:
            lin = np.full((H, W), 0.37, np.float32)
        elif kind == 2:
            lin = synth.random_depth(W, H, seed=seed + 17 * i, lo=0.05, hi=0.6)
        else:
            lin = synth.random_depth(W, H, seed=seed + 31 * i)
        out.append(lin.astype(np.float32))
    return np.stack(out)


def raw(lin, reversed_z=True):
    """Raw depth of the layers `lin`; layer 2, if there is one, gets a sky patch."""
    out = np.stack([synth.lin01_to_raw(l, reversed_z=reversed_z) for l in lin])
    if len(out) > 2:
        H, W = out.shape[1:]
        out[2, H // 4: H // 2, W // 5: W // 2] = 0.0          # sky: raw 0 -> 1e5 -> inf in f16 -> NaN paths
    return out


def frames(W, H, L, seed=0, reversed_z=True):
    """L contrasting raw-depth layers: corridors of distinct frames, constant depth, a sky patch, random depth."""
    out = []
    for i in range(L):
        k = (i + seed) % 4
        if k == 0:
            lin = synth.corridor(W, H, frame=i + seed)
        elif k == 1:
            lin = np.full((H, W), 0.37, np.float32)
        else:
            lin = synth.random_depth(W, H, seed=seed * 13 + i)
        r = synth.lin01_to_raw(lin, reversed_z=reversed_z).astype(np.float32)
        if k == 2:
            r[H // 4: H // 2, W // 5: W // 2] = 0.0
        out.append(r)
    return np.stack(out)


def corridor_depth(W, H, frame=0, L=1):
    """Raw depth of corridor frames frame .. frame + L - 1: [L, H, W], or [H, W] for L = 1."""
    d = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=frame + l)).astype(np.float32) for l in range(L)])
    return d if L > 1 else d[0]


def raw_with_sky(W, H, seed, reversed_z=True):
    r = synth.lin01_to_raw(synth.random_depth(W, H, seed=seed), reversed_z=reversed_z).astype(np.float32)
    r[H // 4: H // 2 + 1, W // 5: W // 2 + 1] = 0.0 if reversed_z else 1.0          # sky
    return r


def ingest(r, kind, stencil=0xA5):
    """(depth in the ingest format of `kind`, the float32 the oracle sees) for float depth `r`: "f32" and "linear" are `r` itself,
    "d16" uint16 codes, "d24s8" uint32 words of a 24-bit code under the stencil byte."""
    if kind in ("f32", "linear"):
        return r, r
    bits = 16 if kind == "d16" else 24
    full = (1 << bits) - 1
    codes = np.clip(np.rint(r.astype(np.float64) * full), 0, full).astype(np.uint32)
    as_float = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
    return (codes.astype(np.uint16) if bits == 16 else codes | (np.uint32(stencil) << np.uint32(24))), as_float


# ---- comparison -------------------------------------------------------------------------------------------------------------------
def buffer_ids(high_quality_mask=0, single_scale=False) -> list:
    """The debug buffers a frame produces: ids 1-17, 18-21 for its high-quality levels; a single-scale frame has only level 1's."""
    if single_scale:
        return [1, 2, 3, 4, 5, 10, 17]
    return list(range(1, 18)) + [17 + k for k in range(1, 5) if (high_quality_mask >> (k - 1)) & 1]


def n_diff(got: np.ndarray, ref: np.ndarray, nan_equal=False) -> int:
    """Elements that differ: unorm8 codes exactly; f16 / f32 bit for bit, NaN payloads included.  nan_equal: any two NaNs match."""
    if got.dtype == np.uint8:
        return int((got != ref).sum())
    if got.dtype == np.float16:
        with np.errstate(over="ignore", invalid="ignore"):
            ref = np.asarray(ref).astype(np.float16)
        same = got.view(np.uint16) == ref.view(np.uint16)
    else:
        ref = np.asarray(ref, np.float32)
        same = got.view(np.uint32) == ref.view(np.uint32)
    if nan_equal:
        same |= np.isnan(got) & np.isnan(ref)
    return int((~same).sum())


def compare_buffers(get, orc, tag: str, ids, nan_equal=False) -> None:
    """get(bid) -> the kernel's buffer; orc: an Oracle that has run the same frame.  Unorm8 buffers against the oracle's codes."""
    bad = []
    for bid in ids:
        got = get(bid)
        n = n_diff(got, orc.codes(bid) if got.dtype == np.uint8 else orc.buffer(bid), nan_equal)
        if n:
            bad.append((bid, n, got.size))
    assert not bad, f"{tag}: mismatching buffers (id, #diff, size): {bad}"


# ---- frames of the emulator ---------------------------------------------------------------------------------------------------
def fused_frame(plan, **kw):
    """An emulator Frame whose LinearDepth is NaN first, so every element the fused frame does not write shows."""
    from emu.emu import Frame
    f = Frame(plan, **kw)
    f.poison_lin()
    return f


def band_frames(W, H, nb, **kw):
    """nb emulator Frames of the row bands of a W x H frame (rowtile.partition), each on its own plan-only context."""
    from emu.emu import Frame
    from miniengineao_b200 import rowtile
    cuts = rowtile.partition(H, nb)
    out = []
    for i in range(nb):
        plan = context(W, H, **kw)
        plan.set_row_band(cuts[i], cuts[i + 1], *rowtile.neighbours(cuts, i))
        f = Frame(plan)
        f.use_plan_band()
        out.append(f)
    return cuts, out


SENTINEL = 0xA5


class View:
    """`shape` = (layers, rows, W) elements of `dtype` at byte pitches (row, layer), `base` bytes past a 256-byte boundary of a backing
    allocation filled with `fill`."""

    def __init__(self, shape, dtype, row, layer, base=0, fill=0xFF):
        L, rows, W = shape
        es = np.dtype(dtype).itemsize
        self.extent = (L - 1) * layer + (rows - 1) * row + W * es
        self.raw = np.empty(base + self.extent + 512, np.uint8)
        off = (-self.raw.ctypes.data) % 256
        self.back = self.raw[off:off + base + self.extent + 256]
        self.back[...] = fill
        self.base, self.row, self.layer = base, row, layer
        self.arr = np.ndarray(shape, dtype, buffer=self.back, offset=base, strides=(layer, row, es))

    @property
    def ptr(self):
        return self.back.ctypes.data + self.base

    def outside(self):
        """The backing bytes that are not part of the view."""
        mask = np.ones(self.back.size, bool)
        L, rows, W = self.arr.shape
        es = self.arr.itemsize
        for l in range(L):
            for r in range(rows):
                s = self.base + l * self.layer + r * self.row
                mask[s:s + W * es] = False
        return self.back[mask]


# ---- the plan's constants and the C client ----------------------------------------------------------------------------------------
def plan_constants(h, layers):
    """Every constant getter of the plan `h`, as one byte string."""
    lib = N.lib()
    parts = []
    for k in range(1, 5):
        for getter, n in ((lib.meao_render_constants, 28), (lib.meao_render_constants_wide, 28), (lib.meao_upsample_constants, 8)):
            out = (C.c_float * n)()
            assert getter(h, k, out) == 0
            parts.append(bytes(out))
        for l in range(layers):
            for wide in (0, 1):
                out = (C.c_float * 28)()
                assert lib.meao_render_constants_layer(h, l, k, wide, out) == 0
                parts.append(bytes(out))
    out = (C.c_float * 4)()
    assert lib.meao_zbuffer_params(h, out) == 0
    parts.append(bytes(out))
    for l in range(layers):
        assert lib.meao_zbuffer_params_layer(h, l, out) == 0
        parts.append(bytes(out))
    return b"".join(parts)


def build_c_client(tmp_path):
    """tests/c_abi/smoke.c compiled as C99 against include/meao.h and linked against libmeao.so; the executable's path."""
    import subprocess
    exe = os.path.join(str(tmp_path), "meao_c_smoke")
    libdir = os.path.dirname(N.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c_abi", "smoke.c"), "-o", exe,
                           "-L", libdir, "-l:libmeao.so", f"-Wl,-rpath,{libdir}"])
    return exe
