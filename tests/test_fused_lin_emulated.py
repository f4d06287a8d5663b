"""CPU tests of the fused frame: prepare_depth in its low-only form (LowDepth1..4 from the even depth rows, no LinearDepth) and the
final blur_upsample reading the raw depth, linearising it and writing LinearDepth itself (csrc/blur_upsample_lin.cu).

The kernel sources run in the fiber emulator (tests/emu/frame_driver.cpp) and every buffer must be bit-identical to the oracle's: the
depth kinds, both Z directions, widths and depth pointers that rule out the 128-bit loads, sky patches (the grouped range test falls
back), premin, single-scale, layered frames and a row band.  LinearDepth is poisoned with NaN first, so every element the frame does
not write shows."""

import numpy as np
import pytest

from miniengineao_b200 import synth
from oracle.oracle import Oracle

from emu.emu import Frame  # noqa: E402  (tests/ is on sys.path via conftest)
from test_layers_emulated import _compare_layer, _plan, contrasting_layers



def fused_frame(plan, **kw):
    """A Frame whose LinearDepth is NaN first, so every element the fused frame does not write shows."""
    f = Frame(plan, **kw)
    f.poison_lin()
    return f


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
    f = fused_frame(_plan(W, H, reversed_z=rz, intensity=1.1), linear=(kind == "linear"))
    f.run_fused(depth)
    _check(f, seen, f"{kind} {W}x{H}", intensity=1.1, reversed_z=rz, depth_is_linear=(kind == "linear"))


@pytest.mark.parametrize("kind", ["f32", "d16"])
def test_unaligned_depth_pointer(kind):
    """vec_ok false although W % 8 == 0: the depth pointer is 4 bytes past a 16-byte boundary."""
    W, H = 136, 72
    depth, seen = _ingest(_raw_with_sky(W, H, 2), kind)
    f = fused_frame(_plan(W, H, intensity=1.1))
    f.run_fused(depth, offset=4)
    _check(f, seen, f"unaligned {kind}", intensity=1.1)


@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(single_scale=True)])
def test_fused_variants(kw):
    W, H = 250, 131
    raw = _raw_with_sky(W, H, 5)
    f = fused_frame(_plan(W, H, intensity=1.1, **kw))
    f.run_fused(raw)
    _check(f, raw, str(kw), intensity=1.1, **kw)


@pytest.mark.parametrize("layers", [2, 6])
def test_fused_layered(layers):
    W, H = 130, 70
    lin = contrasting_layers(W, H, layers, seed=layers)
    raw = np.stack([synth.lin01_to_raw(l) for l in lin]).astype(np.float32)
    raw[min(2, layers - 1), H // 4: H // 2, W // 5: W // 2] = 0.0
    f = fused_frame(_plan(W, H, layers, intensity=1.1, high_quality_mask=1))
    f.run_fused(raw)
    for l in range(layers):
        _check(f, raw[l], f"layer {l}", layer=l, intensity=1.1, high_quality_mask=1)


def test_fused_row_band():
    """The final level's rows [32, 96) through the fused kernel with the band's own depth rows (depth_row0 = 32)."""
    W, H = 161, 130
    raw = _raw_with_sky(W, H, 8)
    f = fused_frame(_plan(W, H, intensity=1.1))
    f.run_fused(raw, rows=(32, 96))
    ref = Oracle(W, H, threads=4, intensity=1.1).run(raw)
    assert np.array_equal(f.buffer(17)[32:96], ref[32:96])


def test_low_only_prepare_writes_no_linear_depth_and_reads_only_even_rows():
    """The low-only prepare_depth leaves the NaN-poisoned LinearDepth alone and gives the LowDepth1..4 of the clean depth when every
    odd row is NaN; the whole frame then writes every LinearDepth element."""
    W, H = 250, 131
    raw = _raw_with_sky(W, H, 4)
    odd_nan = raw.copy()
    odd_nan[1::2] = np.nan
    f = fused_frame(_plan(W, H, intensity=1.1))
    f.prepare_low(odd_nan)
    assert np.isnan(f.buffer(1).astype(np.float32)).all()
    orc = Oracle(W, H, threads=4, intensity=1.1)
    orc.run(raw)
    for bid in (2, 3, 4, 5):
        assert np.array_equal(f.buffer(bid).view(np.uint32), orc.buffer(bid).view(np.uint32)), bid
    f.run_fused(raw)
    assert np.array_equal(f.buffer(1).view(np.uint16), orc.buffer(1).astype(np.float16).view(np.uint16))
