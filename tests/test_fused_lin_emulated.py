"""CPU tests of the fused frame: prepare_depth in its low-only form (LowDepth1..4 from the even depth rows, no LinearDepth) and the
final blur_upsample reading the raw depth, linearising it and writing LinearDepth itself (csrc/blur_upsample_lin.cu).

The kernel sources run in the fiber emulator (tests/emu/lin_driver.cpp) and every buffer must be bit-identical to the oracle's: the
depth kinds, both Z directions, widths and depth pointers that rule out the 128-bit loads, sky patches (the grouped range test falls
back), premin, single-scale, layered frames and a row band.  LinearDepth is poisoned with NaN first, so every element the frame does
not write shows.  Also here: the packed-contraction audit of the new translation unit."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from miniengineao_b200 import _native as N
from miniengineao_b200 import synth
from oracle.oracle import Oracle

from emu import build_lin_emu  # noqa: E402  (tests/ is on sys.path via conftest)
from emu.emu import linearize_zero
from test_layers_emulated import _compare_layer, _plan, contrasting_layers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")

_lib = None


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(build_lin_emu.build())
        l.lemu_create.restype = C.c_void_p
        l.lemu_create.argtypes = [C.c_int, C.c_int, C.c_int]
        l.lemu_destroy.argtypes = [C.c_void_p]
        l.lemu_set_constants.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float] + [C.c_int] * 6
        l.lemu_get_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        l.femu_poison_lin.argtypes = [C.c_void_p]
        l.femu_prepare_low.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        l.femu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        _lib = l
    return _lib


class FusedFrame:
    """One frame in the fused form, planned by a plan-only libmeao context (device = -1); the set-up of emu.layered_emu.LayeredFrame."""

    def __init__(self, plan, *, linear=False):
        self._lib = lib()
        plan.LateUpdate()
        self.plan = plan
        self.W, self.H, self.layers = plan._width, plan._height, int(plan.layers)
        nl = N.lib()
        rc, rcw, uc, zb = (C.c_float * 112)(), (C.c_float * 112)(), (C.c_float * 32)(), (C.c_float * 4)()
        for k in range(1, 5):
            N.check(plan._ctx, nl.meao_render_constants(plan._ctx, k, C.cast(C.byref(rc, 112 * (k - 1)), C.POINTER(C.c_float))))
            N.check(plan._ctx, nl.meao_render_constants_wide(plan._ctx, k, C.cast(C.byref(rcw, 112 * (k - 1)), C.POINTER(C.c_float))))
            N.check(plan._ctx, nl.meao_upsample_constants(plan._ctx, k, C.cast(C.byref(uc, 32 * (k - 1)), C.POINTER(C.c_float))))
        N.check(plan._ctx, nl.meao_zbuffer_params(plan._ctx, zb))
        rz = bool(plan.camera.usesReversedZBuffer)
        pad12 = 0.0 if linear else (1e5 if rz else linearize_zero(zb))
        self._h = self._lib.lemu_create(self.W, self.H, self.layers)
        self._lib.lemu_set_constants(self._h, rc, rcw, uc, zb, pad12, int(not linear), int(rz), int(plan.highQualityMask),
                                     int(plan.sampleExhaustively), int(plan.singleScale), 1)
        self._lib.femu_poison_lin(self._h)

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.lemu_destroy(self._h)
            self._h = None

    @staticmethod
    def _input(depth, offset):
        """C-contiguous copy `offset` bytes past a 64-byte boundary (offset 4: the depth pointer is not 16-byte aligned)."""
        raw = np.empty(depth.nbytes + 128, np.uint8)
        off = (-raw.ctypes.data) % 64 + offset
        out = raw[off:off + depth.nbytes].view(depth.dtype).reshape(depth.shape)
        out[...] = depth
        return out

    def run(self, depth, *, offset=0, rows=(0, 0)):
        fmt = {"float32": 0, "uint16": 1, "uint32": 2}[depth.dtype.name]
        d = self._input(np.ascontiguousarray(depth), offset)
        self._lib.femu_run(self._h, d.ctypes.data, fmt, rows[0], rows[1])

    def prepare_low(self, depth):
        fmt = {"float32": 0, "uint16": 1, "uint32": 2}[depth.dtype.name]
        d = self._input(np.ascontiguousarray(depth), 0)
        self._lib.femu_prepare_low(self._h, d.ctypes.data, fmt)

    def buffer(self, bid, layer=0):
        d = self.plan.buffer_desc(bid)
        dt = {1: np.uint8, 2: np.float16, 4: np.float32}[d.elem_bytes]
        shape = (d.slices, d.height, d.width) if d.slices > 1 else (d.height, d.width)
        out = np.zeros(shape, dt)
        assert self._lib.lemu_get_buffer(self._h, bid, layer, out.ctypes.data) == 0
        return out


def _raw_with_sky(W, H, seed, reversed_z=True):
    raw = synth.lin01_to_raw(synth.random_depth(W, H, seed=seed), reversed_z=reversed_z).astype(np.float32)
    raw[H // 4: H // 2 + 1, W // 5: W // 2 + 1] = 0.0 if reversed_z else 1.0          # sky
    return raw


def _ingest(raw, kind):
    """(depth in the ingest format, the float32 the oracle sees)."""
    if kind in ("f32", "linear"):
        return raw, raw
    bits = 16 if kind == "d16" else 24
    full = (1 << bits) - 1
    codes = np.clip(np.rint(raw.astype(np.float64) * full), 0, full).astype(np.uint32)
    as_float = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
    return (codes.astype(np.uint16) if bits == 16 else codes | (np.uint32(0xA5) << np.uint32(24))), as_float


def _check(f, seen, tag, layer=0, single_scale=False, **okw):
    orc = Oracle(f.W, f.H, threads=4, single_scale=single_scale, **okw)
    ref = orc.run(seen)
    assert np.array_equal(f.buffer(17, layer), ref), tag
    ids = [1, 2, 3, 4, 5, 10, 17] if single_scale else None
    _compare_layer(f, layer, orc, tag, okw.get("high_quality_mask", 0), ids)


@pytest.mark.parametrize("kind", ["f32", "d16", "d24s8", "linear"])
@pytest.mark.parametrize("W,H", [(1, 1), (3, 5), (161, 93), (250, 131), (37, 1000)])
def test_fused_frame_equals_oracle(W, H, kind):
    rz = (W * H) % 2 == 1
    raw = synth.random_depth(W, H, seed=W + H).astype(np.float32) if kind == "linear" else _raw_with_sky(W, H, W + H, rz)
    depth, seen = _ingest(raw, kind)
    f = FusedFrame(_plan(W, H, reversed_z=rz, intensity=1.1), linear=(kind == "linear"))
    f.run(depth)
    _check(f, seen, f"{kind} {W}x{H}", intensity=1.1, reversed_z=rz, depth_is_linear=(kind == "linear"))


@pytest.mark.parametrize("kind", ["f32", "d16"])
def test_unaligned_depth_pointer(kind):
    """vec_ok false although W % 8 == 0: the depth pointer is 4 bytes past a 16-byte boundary."""
    W, H = 136, 72
    depth, seen = _ingest(_raw_with_sky(W, H, 2), kind)
    f = FusedFrame(_plan(W, H, intensity=1.1))
    f.run(depth, offset=4)
    _check(f, seen, f"unaligned {kind}", intensity=1.1)


@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(single_scale=True)])
def test_fused_variants(kw):
    W, H = 250, 131
    raw = _raw_with_sky(W, H, 5)
    f = FusedFrame(_plan(W, H, intensity=1.1, **kw))
    f.run(raw)
    _check(f, raw, str(kw), intensity=1.1, **kw)


@pytest.mark.parametrize("layers", [2, 6])
def test_fused_layered(layers):
    W, H = 130, 70
    lin = contrasting_layers(W, H, layers, seed=layers)
    raw = np.stack([synth.lin01_to_raw(l) for l in lin]).astype(np.float32)
    raw[min(2, layers - 1), H // 4: H // 2, W // 5: W // 2] = 0.0
    f = FusedFrame(_plan(W, H, layers, intensity=1.1, high_quality_mask=1))
    f.run(raw)
    for l in range(layers):
        _check(f, raw[l], f"layer {l}", layer=l, intensity=1.1, high_quality_mask=1)


def test_fused_row_band():
    """The final level's rows [32, 96) through the fused kernel with the band's own depth rows (depth_row0 = 32)."""
    W, H = 161, 130
    raw = _raw_with_sky(W, H, 8)
    f = FusedFrame(_plan(W, H, intensity=1.1))
    f.run(raw, rows=(32, 96))
    ref = Oracle(W, H, threads=4, intensity=1.1).run(raw)
    assert np.array_equal(f.buffer(17)[32:96], ref[32:96])


def test_low_only_prepare_writes_no_linear_depth_and_reads_only_even_rows():
    """The low-only prepare_depth leaves the NaN-poisoned LinearDepth alone and gives the LowDepth1..4 of the clean depth when every
    odd row is NaN; the whole frame then writes every LinearDepth element."""
    W, H = 250, 131
    raw = _raw_with_sky(W, H, 4)
    odd_nan = raw.copy()
    odd_nan[1::2] = np.nan
    f = FusedFrame(_plan(W, H, intensity=1.1))
    f.prepare_low(odd_nan)
    assert np.isnan(f.buffer(1).astype(np.float32)).all()
    orc = Oracle(W, H, threads=4, intensity=1.1)
    orc.run(raw)
    for bid in (2, 3, 4, 5):
        assert np.array_equal(f.buffer(bid).view(np.uint32), orc.buffer(bid).view(np.uint32)), bid
    f.run(raw)
    assert np.array_equal(f.buffer(1).view(np.uint16), orc.buffer(1).astype(np.float16).view(np.uint16))


# ---- packed-contraction audit of the new translation unit (the method of test_no_packed_contraction.py) ------------------------
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false"]
EXPECTED = {"blur_upsample_lin.cu": 22}     # FMULs of the div.rn / rcp.rn expansions of its 12 kernels (blur_upsample.cu: 12 for 8)


@pytest.mark.parametrize("tu", sorted(EXPECTED))
def test_fused_unit_has_only_the_audited_contractions(tu, tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    src = os.path.join(CSRC, tu)
    ptx, cubin = os.path.join(str(tmp_path), "k.ptx"), os.path.join(str(tmp_path), "k.cubin")
    subprocess.check_call([nvcc] + FLAGS + ["-ptx", "-o", ptx, src], stderr=subprocess.DEVNULL)
    subprocess.check_call([nvcc] + FLAGS + ["-cubin", "-o", cubin, src], stderr=subprocess.DEVNULL)
    p = open(ptx).read()
    s = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True).stdout
    assert "f32x2" not in p, tu
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", s), tu
    n_mul = len(re.findall(r"\bmul\.rn\.f32\b", p))
    n_fmul = len(re.findall(r"\bFMUL\b", s))
    assert n_mul > 0, tu
    assert n_fmul - n_mul == EXPECTED[tu], (tu, n_mul, n_fmul)
