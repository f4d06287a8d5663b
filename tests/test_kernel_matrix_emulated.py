"""Every kernel of every kernel table, run in the CPU emulator as the instantiation its slot stands for (tests/kernel_matrix.py).

Each case resets the emulator's launch ledger, runs, and must have launched exactly the kernels kernel_matrix.expected_kernels names --
a table entry swapped with another launches the wrong kernel, which a ragged frame's output does not always show (a taller render tile
on a shorter tile's grid only rewrites rows the next CTA writes again).  A frame must then equal the oracle bit for bit in every layer:
the AO and every intermediate.  At 640 x 360 every render and upsample kernel the case launched must have issued TMA box loads, so
the TMA-fed interior tiles ran too.  The matrix as a whole must name every kernel the emulator builds."""
import numpy as np
import pytest

from miniengineao_b200 import synth
from oracle import oracle as O
from oracle.oracle import Oracle

import kernel_matrix as km  # noqa: E402  (tests/ is on sys.path via conftest)
from emu import emu  # noqa: E402
from emu.emu import Frame, composite, composite_debug  # noqa: E402
from test_kernel_logic_emulated import _band_frames  # noqa: E402
from test_layers_emulated import _compare_layer, _plan  # noqa: E402


def _ran(expected: set, tag: str) -> dict:
    ledger = emu.kernel_ledger()
    assert set(ledger) == expected, f"{tag}: launched {sorted(set(ledger) - expected)} unexpectedly, never launched {sorted(expected - set(ledger))}"
    return ledger


def _frame_case(c: km.Case) -> None:
    W, H = c.size
    depth, seen = km.depth(c)
    plan = _plan(W, H, c.layers, single_scale=c.single_scale, reversed_z=c.reversed_z, intensity=1.1, high_quality_mask=c.hq,
                 sample_exhaustively=c.exhaustive)
    f = Frame(plan, linear=c.kind == "linear", render_tile=c.tile)
    ao = None
    emu.ledger_reset()
    if c.form == "stage":
        f.run(depth)
    elif c.form == "fused":
        f.run_fused(depth)
    else:
        ao = f.run_arrays(depth, "layered" if c.layers > 1 else "2d")
    ledger = _ran(km.expected_kernels(c), c.id)
    if c.size == km.TMA_FED:
        untouched = [k for k, (_, tma) in ledger.items() if k.startswith(("render_ao", "blur_upsample")) and tma == 0]
        assert not untouched, f"{c.id}: no TMA box loads in {untouched}"
    for l in range(c.layers):
        orc = Oracle(W, H, threads=4, **c.oracle_kw())
        ref = orc.run(seen[l])
        if ao is not None:
            assert np.array_equal(ao[l], ref), f"{c.id}: the AO array of layer {l} differs from the oracle"
        _compare_layer(f, l, orc, c.id, c.hq, c.buffer_ids())


def _composite(c: km.Case) -> None:
    rng = np.random.default_rng(0)
    ao = rng.integers(0, 256, size=(45, 67), dtype=np.uint8)
    c8 = rng.integers(0, 256, size=(45, 67, 4), dtype=np.uint8)
    c16 = (rng.uniform(0, 4, size=(45, 67, 4)) ** 3).astype(np.float16)
    emu.ledger_reset()
    got = [composite(ao, col, rgb=True, alpha=True, one_minus=False) for col in (c8, c16)]
    _ran(km.expected_kernels(c), c.id)
    for g, col in zip(got, (c8, c16)):
        assert np.array_equal(g.view(np.uint8), O.composite_framebuffer(ao, col).view(np.uint8)), col.dtype


def _debug_composite(c: km.Case) -> None:
    v = np.random.default_rng(1).integers(0, 256, size=(45, 67), dtype=np.uint8)
    likes = (np.zeros(1, np.uint8), np.zeros(1, np.float16))
    emu.ledger_reset()
    got = [composite_debug(v, like) for like in likes]
    _ran(km.expected_kernels(c), c.id)
    for g, like in zip(got, likes):
        assert np.array_equal(g.view(np.uint8), O.composite_debug(v, like).view(np.uint8)), like.dtype


def _debug_view(c: km.Case) -> None:
    """A plain view (Occlusion2), a tiled one (TiledDepth2, synthesised from LowDepth2 by the view kernel) and the TiledDepth2 buffer
    itself (synth_tiled_kernel), after a frame."""
    W, H = c.size
    depth, seen = km.depth(c)
    f = Frame(_plan(W, H, intensity=1.1))
    f.run(depth)
    orc = Oracle(W, H, threads=4, **c.oracle_kw())
    orc.run(seen[0])
    emu.ledger_reset()
    plain, tiled, atlas = f.debug_view(11), f.debug_view(7), f.buffer(7)
    _ran(km.expected_kernels(c), c.id)
    assert np.array_equal(plain, orc.debug_view(11)) and np.array_equal(tiled, orc.debug_view(7))
    assert np.array_equal(atlas.view(np.uint16), orc.buffer(7).astype(np.float16).view(np.uint16))


def _band_depth(W, H):
    return synth.lin01_to_raw(synth.random_depth(W, H, seed=3))


def _halo(c: km.Case) -> None:
    """Two bands swap their halo rows through pack (LowDepth1..4 -> a contiguous message) and unpack; each band's AO must then equal
    its rows of the whole-frame oracle."""
    W, H = 200, 528
    depth = _band_depth(W, H)
    cuts, (a, b) = _band_frames(W, H, 2, intensity=1.1)
    a.band_phase_a(depth[cuts[0]:cuts[1]])
    b.band_phase_a(depth[cuts[1]:cuts[2]])
    emu.ledger_reset()
    b.halo_unpack(0, a.halo_pack(1))
    a.halo_unpack(1, b.halo_pack(0))
    _ran(km.expected_kernels(c), c.id)
    ref = Oracle(W, H, threads=4, intensity=1.1).run(depth)
    for i, f in enumerate((a, b)):
        assert np.array_equal(f.band_phase_b(), ref[cuts[i]:cuts[i + 1]]), i


def _band_exchange(c: km.Case) -> None:
    """Two bands through the native exchange kernel (peer stores + epoch flags); the flags the band below would have raised by the
    time the first band runs are preset, as in test_kernel_logic_emulated.py."""
    W, H = 200, 528
    depth = _band_depth(W, H)
    cuts, (a, b) = _band_frames(W, H, 2, intensity=1.1)
    a.band_phase_a(depth[cuts[0]:cuts[1]])
    b.band_phase_a(depth[cuts[1]:cuts[2]])
    emu.ledger_reset()
    fl = a.flags()
    a.flags(set_ready_ack=(fl["ready"][0], 1, fl["ack"][0], 1))
    assert a.exchange(None, b) == 0 and b.exchange(a, None) == 0
    _ran(km.expected_kernels(c), c.id)
    ref = Oracle(W, H, threads=4, intensity=1.1).run(depth)
    for i, f in enumerate((a, b)):
        assert np.array_equal(f.band_phase_b(), ref[cuts[i]:cuts[i + 1]]), i


UNITS = {"composite": _composite, "debug_view": _debug_view, "debug_composite": _debug_composite, "halo": _halo,
         "band_exchange": _band_exchange}


@pytest.mark.parametrize("case", km.CASES, ids=lambda c: c.id)
def test_case_launches_its_kernels_and_matches_the_oracle(case):
    if case.frame:
        _frame_case(case)
    else:
        UNITS[case.form](case)


def test_the_matrix_launches_every_kernel_the_emulator_builds():
    named = set().union(*(km.expected_kernels(c) for c in km.CASES))
    built = emu.emulated_kernels()
    assert named == built, f"never launched: {sorted(built - named)}; not built: {sorted(named - built)}"
    assert len(built) == 87
