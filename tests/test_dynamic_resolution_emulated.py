"""CPU tests of dynamic resolution (meao_reserve): frames of smaller, ragged sizes run inside ONE arena laid out for the largest size,
at the offsets and pitches of arena_layout (csrc/arena_layout.h, shared with meao_api.cu), through the host-compiled kernel sources
(tests/emu/frame_driver.cpp).  The arena first holds stale data -- the buffers of a hostile frame at the maximum size, or an 0xFF
poison (NaN in every f16 / f32) -- where a fresh context's arena holds zeros; any kernel that read a byte its frame did not write
(pitch padding, rows beyond the frame) would change bits.  AO and every debug buffer of every layer must equal the oracle's, for single
and layered frames, with and without the fused final level, and for the premin and single-scale variants."""
import numpy as np
import pytest

import harness
import hostile_cases as HC
from emu.emu import Frame, lib  # noqa: E402  (tests/ is on sys.path via conftest)

MAX = (330, 190)
SIZES = [(1, 1), (33, 17), (97, 61), (329, 189), (257, 131), (64, 32)]


def test_layout_is_the_librarys():
    """The arena the driver allocates is the one meao_reserve reports for the same reservation and layer count."""
    for L in (1, 3):
        p = harness.context(64, 32, layers=L)
        p.maxResolution = MAX
        p.LateUpdate()
        f = Frame(p, max_size=MAX)
        assert f.arena_bytes() == p.reservation()["arena_bytes"]
        assert lib().frame_resize(f._h, MAX[0] + 1, MAX[1]) == -1


CASES = {
    "single_fused": dict(layers=1, fused=True),
    "single_full": dict(layers=1, fused=False),
    "layered_fused": dict(layers=3, fused=True),
    "layered_full": dict(layers=3, fused=False),
    "premin_fused": dict(layers=1, fused=True, high_quality_mask=1),
    "premin_layered_full": dict(layers=2, fused=False, high_quality_mask=15),
    "single_scale_fused": dict(layers=1, fused=True, single_scale=True),
    "single_scale_layered_full": dict(layers=3, fused=False, single_scale=True),
}


@pytest.mark.parametrize("stale", ["max_frame", "poison"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_smaller_frames_in_a_stale_arena_match_the_oracle(case, stale):
    kw = dict(CASES[case])
    L, fused = kw.pop("layers"), kw.pop("fused")
    f = Frame(harness.context(*MAX, layers=L, intensity=1.1, **kw), max_size=MAX)
    run = f.run_fused if fused else f.run
    if stale == "max_frame":
        run(np.stack([HC.hostile_raw(*MAX, f.zb, True, seed=l) for l in range(L)]).astype(np.float32))
    else:
        f.fill()
    ids = harness.buffer_ids(kw.get("high_quality_mask", 0), kw.get("single_scale", False))
    for i, (W, H) in enumerate(SIZES):
        f.load(harness.context(W, H, layers=L, intensity=1.1, **kw))
        depth = harness.raw(harness.contrasting_layers(W, H, L, seed=i)).astype(np.float32)
        run(depth)
        for l in range(L):
            orc = harness.oracle(W, H, intensity=1.1, **kw)
            ref = orc.run(depth[l])
            assert np.array_equal(f.buffer(17, l), ref), (case, stale, W, H, l)
            harness.compare_buffers(lambda bid: f.buffer(bid, l), orc, f"{case} {stale} {W}x{H} layer {l}", ids)
