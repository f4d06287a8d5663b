"""CPU tests of pitched frames (meao_render_pitched): the depth and the AO are views inside larger allocations, each with its own row and
layer pitch.  The kernel sources of a fused frame run in the fiber emulator (tests/emu/pitched_driver.cpp) with the argument blocks
meao_api.cu fills for such views.

Every backing byte of the depth outside its view is 0xff (NaN as f32, the far-plane code as D16 / D24S8), so a bit-exact AO proves the
padding is never read; every AO byte outside its view holds a sentinel that must survive.  AO, LinearDepth and LowDepth1..4 of every
layer must equal the oracle's on the tight depth, over the depth kinds, both Z directions, ragged sizes, D3D12-style 256-byte row
pitches, row pitches that rule out the 128-bit loads, a sub-rectangle at x0 = 1, a dynamic-resolution corner of a larger layered
target, premin, single-scale and a row band.  Zero pitches in the argument blocks must keep meaning the tight views.  Also here: the
packed-contraction audit of the changed translation units and a spill check of the fused final-level and prepare kernels."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from miniengineao_b200 import _native as N
from oracle.oracle import Oracle

from emu import build_pitched_emu  # noqa: E402  (tests/ is on sys.path via conftest)
from test_fused_lin_emulated import _ingest, _raw_with_sky
from test_layers_emulated import _compare_layer, _plan, contrasting_layers
from miniengineao_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")
SENTINEL = 0xA5

_lib = None


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(build_pitched_emu.build())
        l.lemu_create.restype = C.c_void_p
        l.lemu_create.argtypes = [C.c_int, C.c_int, C.c_int]
        l.lemu_destroy.argtypes = [C.c_void_p]
        l.lemu_set_constants.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float] + [C.c_int] * 6
        l.lemu_get_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        l.femu_poison_lin.argtypes = [C.c_void_p]
        l.pemu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_longlong, C.c_void_p, C.c_longlong, C.c_longlong,
                               C.c_int, C.c_int]
        _lib = l
    return _lib


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


class PitchedFrame:
    """One fused frame on views, planned by a plan-only libmeao context (device = -1); the set-up of FusedFrame."""

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
        pad12 = 0.0 if linear else (1e5 if rz else float(np.float32(1) / np.float32(zb[1])))
        self._h = self._lib.lemu_create(self.W, self.H, self.layers)
        self._lib.lemu_set_constants(self._h, rc, rcw, uc, zb, pad12, int(not linear), int(rz), int(plan.highQualityMask),
                                     int(plan.sampleExhaustively), int(plan.singleScale), 1)
        self._lib.femu_poison_lin(self._h)

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.lemu_destroy(self._h)
            self._h = None

    def run(self, dv: View, av: View, rows=(0, 0), zero=False):
        fmt = {"float32": 0, "uint16": 1, "uint32": 2}[dv.arr.dtype.name]
        p = (0, 0, 0, 0) if zero else (dv.row, dv.layer, av.row, av.layer)
        self._lib.pemu_run(self._h, dv.ptr, fmt, p[0], p[1], av.ptr, p[2], p[3], rows[0], rows[1])

    def buffer(self, bid, layer=0):
        d = self.plan.buffer_desc(bid)
        dt = {1: np.uint8, 2: np.float16, 4: np.float32}[d.elem_bytes]
        shape = (d.slices, d.height, d.width) if d.slices > 1 else (d.height, d.width)
        out = np.zeros(shape, dt)
        assert self._lib.lemu_get_buffer(self._h, bid, layer, out.ctypes.data) == 0
        return out


def _frame(depth, seen, *, drow=None, dlayer=None, dbase=0, arow=None, alayer=None, abase=0, linear=False, rz=True, rows=(0, 0),
           zero=False, **kw):
    """Run depth [L, H, W] (ingest format) through views with the given byte pitches (None: tight) and check every layer against the
    oracle on `seen` (float32 [L, H, W]).  Returns the frame."""
    L, H, W = depth.shape
    es = depth.dtype.itemsize
    drow = drow or W * es
    dlayer = dlayer or H * drow
    arow = arow or W
    alayer = alayer or H * arow
    f = PitchedFrame(_plan(W, H, L, reversed_z=rz, intensity=1.1, **kw), linear=linear)
    band = rows[1] > rows[0]
    dv = View(depth.shape, depth.dtype, drow, dlayer, dbase)
    dv.arr[...] = depth
    ashape = (L, rows[1] - rows[0], W) if band else (L, H, W)
    av = View(ashape, np.uint8, arow, alayer, abase, fill=SENTINEL)
    f.run(dv, av, rows, zero)
    assert (av.outside() == SENTINEL).all(), "a byte outside the AO view was written"
    assert (dv.outside() == 0xFF).all()
    okw = dict(intensity=1.1, reversed_z=rz, depth_is_linear=linear, **kw)
    for l in range(L):
        orc = Oracle(W, H, threads=4, **okw)
        ref = orc.run(seen[l])
        if band:
            assert np.array_equal(av.arr[l], ref[rows[0]:rows[1]]), f"band layer {l}"
            continue
        assert np.array_equal(av.arr[l], ref), f"AO view layer {l}"
        _compare_layer(f, l, orc, f"layer {l}", ids=[1, 2, 3, 4, 5])       # LinearDepth, LowDepth1..4
    return f


def _one(W, H, kind, seed, rz=True):
    raw = synth.random_depth(W, H, seed=seed).astype(np.float32) if kind == "linear" else _raw_with_sky(W, H, seed, rz)
    depth, seen = _ingest(raw, kind)
    return depth[None], seen[None]


def _up(x, a):
    return (x + a - 1) // a * a


@pytest.mark.parametrize("kind", ["f32", "d16", "d24s8", "linear"])
@pytest.mark.parametrize("W,H", [(1, 1), (3, 5), (161, 93), (250, 131)])
def test_d3d12_row_pitch_equals_oracle(W, H, kind):
    """Rows rounded up to 256 bytes (a D3D12 placed footprint) for the depth and the AO; both Z directions over the sizes."""
    rz = (W * H) % 2 == 1
    depth, seen = _one(W, H, kind, W + H, rz)
    es = depth.dtype.itemsize
    _frame(depth, seen, drow=_up(W * es, 256), arow=_up(W, 256), linear=(kind == "linear"), rz=rz)


@pytest.mark.parametrize("kind", ["f32", "d16", "d24s8"])
def test_row_pitch_off_the_16_byte_grid_takes_the_scalar_path(kind):
    """A row pitch that is a multiple of the element size but not of 16 bytes (no 128-bit loads), and an AO pitch that is not a
    multiple of 8 (no 64-bit stores): the same bits."""
    W, H = 136, 72
    depth, seen = _one(W, H, kind, 3)
    es = depth.dtype.itemsize
    _frame(depth, seen, drow=W * es + es, arow=W + 3)


def test_sub_rectangle_at_x0_1():
    """A viewport inside an atlas at x0 = 1: the depth pointer is 4 bytes past a 16-byte boundary, the AO pointer 1 byte past one."""
    W, H = 160, 90
    depth, seen = _one(W, H, "f32", 6)
    _frame(depth, seen, drow=1024, dbase=4, arow=256, abase=1)


@pytest.mark.parametrize("layers", [2, 6])
def test_dynamic_resolution_corner_of_a_layered_target(layers):
    """[L, Hmax, Wmax][:, :H, :W]: the layer pitch is the whole max-size image, larger than rows x row pitch; premin on level 1."""
    W, H, Wmax, Hmax = 130, 70, 200, 96
    lin = contrasting_layers(W, H, layers, seed=layers)
    raw = np.stack([synth.lin01_to_raw(l) for l in lin]).astype(np.float32)
    raw[min(2, layers - 1), H // 4: H // 2, W // 5: W // 2] = 0.0
    _frame(raw, raw, drow=Wmax * 4, dlayer=Hmax * Wmax * 4, arow=Wmax, alayer=Hmax * Wmax, high_quality_mask=1)


def test_layered_d16_layer_pitch_off_the_grid():
    """Layer pitches that are not multiples of 16 (depth) or 8 (AO) bytes although the rows are: the layered vector-path rule."""
    W, H, L = 64, 40, 3
    raws = [_raw_with_sky(W, H, 20 + l) for l in range(L)]
    pairs = [_ingest(r, "d16") for r in raws]
    depth, seen = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    _frame(depth, seen, drow=256, dlayer=256 * H + 2, arow=64, alayer=64 * H + 4)


@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(single_scale=True)])
def test_pitched_variants(kw):
    W, H = 250, 131
    depth, seen = _one(W, H, "f32", 5)
    _frame(depth, seen, drow=1024, arow=256, **kw)


def test_pitched_row_band():
    """The final level's rows [32, 96) read from the band's own depth rows of a pitched view and stored into a pitched band AO view."""
    W, H = 161, 130
    depth, seen = _one(W, H, "f32", 8)
    _frame(depth, seen, drow=768, arow=192, rows=(32, 96))


@pytest.mark.parametrize("kind", ["f32", "d16"])
def test_zero_pitches_in_the_argument_blocks_mean_tight(kind):
    """The drivers written before the pitch fields zero-fill PrepareArgs / DepthIn: zero pitches on tight views give the tight
    frame, for one layer and for a layered frame."""
    W, H = 136, 72
    depth, seen = _one(W, H, kind, 11)
    _frame(depth, seen, zero=True)
    raws = [_raw_with_sky(W, H, 30 + l) for l in range(2)]
    pairs = [_ingest(r, kind) for r in raws]
    _frame(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]), zero=True)


# ---- audits of the changed translation units ---------------------------------------------------------------------------------
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false"]
EXPECTED = {"prepare_depth.cu": 0, "prepare_depth_layered.cu": 0, "blur_upsample_lin.cu": 22}   # the values of the existing audits


def _nvcc():
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    return nvcc


@pytest.mark.parametrize("tu", sorted(EXPECTED))
def test_changed_unit_has_only_the_audited_contractions(tu, tmp_path):
    nvcc = _nvcc()
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


# translation unit -> (kernel-name pattern, number of kernels): the pitch replaces the W multiplier and must not cost a spill
SPILL_FREE = {"blur_upsample_lin.cu": (r"blur_upsample_\w*lin\w*_kernel", 12), "prepare_depth.cu": (r"prepare_depth_\w*kernel", 14),
              "prepare_depth_layered.cu": (r"prepare_depth_\w*kernel", 14)}


@pytest.mark.parametrize("tu", sorted(SPILL_FREE))
def test_pitched_kernels_do_not_spill(tu, tmp_path):
    """-Xptxas -v of the fused final-level kernels (48-register cap) and of both prepare forms: 0 bytes of spill each."""
    nvcc = _nvcc()
    cubin = os.path.join(str(tmp_path), "k.cubin")
    out = subprocess.run([nvcc] + FLAGS + ["-Xptxas", "-v", "-cubin", "-o", cubin, os.path.join(CSRC, tu)], capture_output=True,
                         text=True)
    assert out.returncode == 0, out.stderr
    ents = re.findall(r"Compiling entry function '([^']+)'[^\n]*\n(?:[^\n]*\n)*?[^\n]*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                      out.stdout + out.stderr)
    pat, n = SPILL_FREE[tu]
    mine = [(name, int(st), int(ld)) for name, st, ld in ents if re.search(pat, name)]
    assert len(mine) == n, (tu, [m[0] for m in mine])
    assert all(st == 0 and ld == 0 for _, st, ld in mine), mine


def test_python_pitches_of_size_one_dimensions():
    """render()'s byte pitches of a tensor view: a dimension of size 1 is never stepped along, so its stride is taken as the tight one
    -- torch.empty(1, H).t() (shape (H, 1), strides (1, H)) is contiguous and must be accepted as a one-pixel-wide image."""
    import torch
    from miniengineao_b200 import AmbientOcclusion
    pitches = AmbientOcclusion._pitches
    assert pitches(None, torch.empty(1, 16).t(), "depth") == (4, 64)
    assert pitches(None, torch.empty(16, 1, dtype=torch.uint8), "out") == (1, 16)
    assert pitches(None, torch.empty(4, 1, 9)[:, :, :5], "depth") == (20, 36)        # one row per layer, layers 9 floats apart
    assert pitches(None, torch.empty(2, 8, 16)[:, :5, :3], "depth") == (64, 512)
    with pytest.raises(ValueError):
        pitches(None, torch.empty(5, 6)[:, ::2], "depth")                              # last stride 2
    with pytest.raises(ValueError):
        pitches(None, torch.empty(6, 5).t(), "depth")
