"""CPU tests of pitched frames (meao_render_pitched): the depth and the AO are views inside larger allocations, each with its own row and
layer pitch.  The kernel sources of a fused frame run in the fiber emulator (tests/emu/frame_driver.cpp) with the argument blocks
libmeao fills for such views.

Every backing byte of the depth outside its view is 0xff (NaN as f32, the far-plane code as D16 / D24S8), so a bit-exact AO proves the
padding is never read; every AO byte outside its view holds a sentinel that must survive.  AO, LinearDepth and LowDepth1..4 of every
layer must equal the oracle's on the tight depth, over the depth kinds, both Z directions, ragged sizes, D3D12-style 256-byte row
pitches, row pitches that rule out the 128-bit loads, a sub-rectangle at x0 = 1, a dynamic-resolution corner of a larger layered
target, premin, single-scale and a row band.  Zero pitches in the argument blocks must keep meaning the tight views."""

import numpy as np
import pytest

from miniengineao_b200 import synth

import harness
from harness import SENTINEL, View, fused_frame


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
    f = fused_frame(harness.context(W, H, layers=L, reversed_z=rz, intensity=1.1, **kw), linear=linear)
    band = rows[1] > rows[0]
    dv = View(depth.shape, depth.dtype, drow, dlayer, dbase)
    dv.arr[...] = depth
    ashape = (L, rows[1] - rows[0], W) if band else (L, H, W)
    av = View(ashape, np.uint8, arow, alayer, abase, fill=SENTINEL)
    f.run_pitched(dv, av, rows, zero)
    assert (av.outside() == SENTINEL).all(), "a byte outside the AO view was written"
    assert (dv.outside() == 0xFF).all()
    okw = dict(intensity=1.1, reversed_z=rz, depth_is_linear=linear, **kw)
    for l in range(L):
        orc = harness.oracle(W, H, **okw)
        ref = orc.run(seen[l])
        if band:
            assert np.array_equal(av.arr[l], ref[rows[0]:rows[1]]), f"band layer {l}"
            continue
        assert np.array_equal(av.arr[l], ref), f"AO view layer {l}"
        harness.compare_buffers(lambda bid: f.buffer(bid, l), orc, f"layer {l}", [1, 2, 3, 4, 5])       # LinearDepth, LowDepth1..4
    return f


def _one(W, H, kind, seed, rz=True):
    raw = synth.random_depth(W, H, seed=seed).astype(np.float32) if kind == "linear" else harness.raw_with_sky(W, H, seed, rz)
    depth, seen = harness.ingest(raw, kind)
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
    lin = harness.contrasting_layers(W, H, layers, seed=layers)
    raw = np.stack([synth.lin01_to_raw(l) for l in lin]).astype(np.float32)
    raw[min(2, layers - 1), H // 4: H // 2, W // 5: W // 2] = 0.0
    _frame(raw, raw, drow=Wmax * 4, dlayer=Hmax * Wmax * 4, arow=Wmax, alayer=Hmax * Wmax, high_quality_mask=1)


def test_layered_d16_layer_pitch_off_the_grid():
    """Layer pitches that are not multiples of 16 (depth) or 8 (AO) bytes although the rows are: the layered vector-path rule."""
    W, H, L = 64, 40, 3
    raws = [harness.raw_with_sky(W, H, 20 + l) for l in range(L)]
    pairs = [harness.ingest(r, "d16") for r in raws]
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
    """The launchers resolve zero pitches in PrepareArgs / DepthIn to the tight views (the blocks are built as libmeao builds them,
    then their pitches zeroed): zero pitches on tight views give the tight frame, for one layer and for a layered frame."""
    W, H = 136, 72
    depth, seen = _one(W, H, kind, 11)
    _frame(depth, seen, zero=True)
    raws = [harness.raw_with_sky(W, H, 30 + l) for l in range(2)]
    pairs = [harness.ingest(r, kind) for r in raws]
    _frame(np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]), zero=True)


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
