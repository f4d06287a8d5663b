"""The oracles of the hierarchy depth (tests/depth_oracle.py): the thread-group oracle (oracle/meao_oracle.c) walked at depth n against the
global per-pixel restatement (oracle/direct_formulation.py) walked the same way, for depths 1-4 with high-quality masks; single_scale as
depth 1; and at depth 4 the committed golden fixtures bit for bit."""
import glob
import os

import numpy as np
import pytest

import depth_oracle as DO
from miniengineao_b200 import synth
from oracle.oracle import Oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def run_both(W, H, seed, n, **kw):
    o = Oracle(W, H, variant="nofma", threads=4, **kw)
    depth = synth.lin01_to_raw(synth.random_depth(W, H, seed=seed))
    ao = DO.run(o, depth, n, kw.get("high_quality_mask", 0))
    rc = {k: o.render_constants(k) for k in range(1, 5)}
    rcw = {k: o.render_constants(k, wide=True) for k in range(1, 5)}
    uc = {k: o.upsample_constants(k) for k in range(1, 5)}
    r = DO.direct(depth, rc, uc, o.zbuffer_params(), n, exhaustive=kw.get("sample_exhaustively", False),
                  high_quality_mask=kw.get("high_quality_mask", 0), render_consts_wide=rcw)
    return o, ao, r


@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("W,H,kw", [
    (97, 61, dict()),
    (130, 70, dict(high_quality_mask=0b1111, sample_exhaustively=True, intensity=1.2)),
    (64, 48, dict(high_quality_mask=0b0101)),
    (33, 17, dict(high_quality_mask=0b1010, thickness_modifier=3.0)),
])
def test_direct_formulation_equals_thread_group_oracle(W, H, kw, n):
    """Every buffer the frame of depth n writes: Occlusion and HighQuality of levels 1..n, Combined below n, the AO."""
    o, ao, r = run_both(W, H, W * 7 + H + n, n, **kw)
    mask = kw.get("high_quality_mask", 0)
    for k in range(1, n + 1):
        assert np.array_equal(r["occ"][k], o.codes(9 + k)), f"Occlusion{k}"
        if (mask >> (k - 1)) & 1:
            assert np.array_equal(r["hq"][k], o.codes(17 + k)), f"HighQuality{k}"
    for k in range(n + 1, 5):
        assert r["occ"][k] is None and r["hq"][k] is None
    for k in range(1, n):
        assert np.array_equal(r["comb"][k], o.codes(13 + k)), f"Combined{k}"
    assert np.array_equal(r["comb"][0], ao)


def test_depth_four_is_the_oracles_own_frame_and_depths_differ():
    W, H = 160, 90
    depth = synth.lin01_to_raw(synth.corridor(W, H))
    aos = [DO.run(Oracle(W, H), depth, n) for n in (1, 2, 3, 4)]
    for i in range(4):
        for j in range(i):
            assert not np.array_equal(aos[i], aos[j]), (i + 1, j + 1)
    assert np.array_equal(aos[3], Oracle(W, H).run(depth))


def test_single_scale_is_depth_one():
    """The oracle's single_scale frame (DS1 + REN 1 + the final-style UPS on Occlusion1) is the frame of depth 1."""
    W, H = 256, 256
    depth = synth.lin01_to_raw(synth.flat_sphere(W, H))
    assert np.array_equal(DO.run(Oracle(W, H, intensity=1.1), depth, 1), Oracle(W, H, intensity=1.1, single_scale=True).run(depth))


def test_depth_one_with_high_quality_level_one():
    """single_scale = 0, n = 1, mask bit 0: the premin final upsample on Occlusion1 + HighQuality1 (both restatements)."""
    o, ao, r = run_both(81, 53, 11, 1, high_quality_mask=1)
    assert np.array_equal(r["hq"][1], o.codes(18))
    assert np.array_equal(r["comb"][0], ao)
    plain = DO.run(Oracle(81, 53, variant="nofma"), synth.lin01_to_raw(synth.random_depth(81, 53, seed=11)), 1)
    assert not np.array_equal(ao, plain)


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "*.npz"))))
def test_depth_four_reproduces_golden_fixture(path):
    """The walk at depth 4 (depth 1 for the single-scale fixture) reproduces every committed fixture."""
    g = np.load(path)
    H, W = g["depth"].shape
    p = g["params"]
    v = np.zeros(4, np.int32)
    if "variants" in g.files:
        v[:len(g["variants"])] = g["variants"]
    o = Oracle(W, H, noise_filter_tolerance=float(p[0]), blur_tolerance=float(p[1]), upsample_tolerance=float(p[2]),
               thickness_modifier=float(p[3]), intensity=float(p[4]), single_pass_stereo=bool(v[0]), sample_exhaustively=bool(v[1]),
               high_quality_mask=int(v[2]))
    assert np.array_equal(DO.run(o, g["depth"], 1 if v[3] else 4, int(v[2])), g["ao"])
    for bid in [int(k[3:]) for k in g.files if k.startswith("buf")]:
        if v[3] and bid == 14:
            continue                                    # Combined1 is no buffer of the depth-1 frame (it holds the walk's LoResAO1)
        ref = g[f"buf{bid}"]
        if ref.dtype == np.uint8:
            assert np.array_equal(o.codes(bid), ref), bid
        elif ref.dtype == np.float16:
            with np.errstate(over="ignore"):
                assert np.array_equal(o.buffer(bid).astype(np.float16).view(np.uint16), ref.view(np.uint16)), bid
        else:
            assert np.array_equal(o.buffer(bid), ref), bid
