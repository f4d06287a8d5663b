"""CPU tests of batches (meao_render_arrays_batch / meao_render_batch): each layer of a layered frame reads its own depth and writes
its own AO, in CUDA arrays or in device buffers of their own.

The batch kernels (build.py BATCH_SOURCES) run in the fiber emulator (tests/emu/frame_batch.cpp, linked against the emulator the other
CPU tests use).  A case matrix covers arrays and pointers, every depth format each supports, both Z directions, the plain and the
premin final level, per-layer cameras, and layers with a misaligned base or an odd row pitch.  In every case each layer is bit-exact to
the oracle's single-layer frame with that layer's camera, on the AO and on every debug buffer (ids 1-21), and every byte of an
oversized AO target outside W x H keeps its poison.  The launch ledger of the matrix holds every one of the 20 batch kernels."""
import numpy as np
import pytest

from miniengineao_b200 import Camera

import harness
from emu import batch, emu  # noqa: E402  (tests/ is on sys.path via conftest)
from emu.emu import Frame  # noqa: E402

POISON = 0x5C
# (near, far, vertical field of view): every layer its own camera
CAMS = [(0.3, 100.0, 60.0), (0.1, 1000.0, 90.0), (0.5, 50.0, 40.0)]


def _cameras(W, H, L, reversed_z):
    return [Camera(W, H, nearClipPlane=n, farClipPlane=f, fieldOfView=v, usesReversedZBuffer=reversed_z) for n, f, v in CAMS[:L]]


def _depth(W, H, L, kind, reversed_z, seed):
    """(the layers' depth in the format of `kind` [L, H, W], the float32 the oracle reads, linear?)"""
    lin = harness.contrasting_layers(W, H, L, seed=seed)
    if kind == "linear_f32":
        return lin, lin, True
    r = harness.raw(lin, reversed_z=reversed_z)
    if kind in ("d16", "d24s8"):
        codes, as_float = harness.ingest(r, kind)
        return codes, as_float, False
    return r, r, False


def _compare(f, W, H, cams, oracle_depth, ao, linear, hq, tag):
    """Each layer l against the oracle's single-layer frame with camera l: ao[l] ([H, W]) and the debug buffers of layer l"""
    ids = [b for b in harness.buffer_ids(hq) if b != harness.buffer_ids()[-1]]     # id 17 is the caller's AO here, compared directly
    for l, cam in enumerate(cams):
        orc = harness.oracle(W, H, camera=cam, linear=linear, high_quality_mask=hq)
        ref = orc.run(oracle_depth[l])
        assert np.array_equal(ao[l], ref), f"{tag}: layer {l}'s AO differs from the oracle's single-layer frame"
        harness.compare_buffers(lambda bid: f.buffer(bid, l), orc, f"{tag} layer {l}", ids)


def _arrays_case(kind, reversed_z, hq, W=61, H=37, L=3, seed=1):
    """An array batch: layer 0 exact-size 2-D arrays, layer 1 oversized 2-D arrays, layer 2 oversized layered arrays of one layer; the
    depth outside W x H holds NaN / inf, the AO the poison byte."""
    depth, odepth, linear = _depth(W, H, L, kind, reversed_z, seed)
    ext = [(H, W), (H + 3, W + 5), (H + 1, W + 2)]
    shapes = ["2d", "2d", "layered"]
    fill = np.float32(np.nan) if depth.dtype == np.float32 else 0
    ds, aos = [], []
    for l in range(L):
        d = np.full(ext[l], fill, depth.dtype)
        if depth.dtype == np.float32 and ext[l] != (H, W):
            d[H:] = np.inf
        d[:H, :W] = depth[l]
        ds.append(d)
        aos.append(np.full(ext[l], POISON, np.uint8))
    cams = _cameras(W, H, L, reversed_z)
    f = Frame(harness.context(W, H, layers=L, layer_cameras=cams, reversed_z=reversed_z, high_quality_mask=hq), linear=linear)
    n0 = f.surface_accesses()
    batch.run_arrays_batch(f, ds, aos, shapes, shapes[::-1])
    assert f.surface_accesses() - n0 == 2 * L * W * H, "a surface access outside W x H, or one missing"
    tag = f"arrays {W}x{H} {kind} reversed_z={reversed_z} hq={hq}"
    for l, a in enumerate(aos):
        assert (a[H:] == POISON).all() and (a[:, W:] == POISON).all(), f"{tag}: layer {l} stored outside W x H"
    _compare(f, W, H, cams, odepth, [a[:H, :W] for a in aos], linear, hq, tag)


def _pointers_case(kind, reversed_z, hq, W=61, H=37, L=3, seed=2):
    """A pointer batch: layer 0 tight and aligned, layer 1 at an odd row pitch, layer 2 at a base that misses the vector alignment; each
    AO view inside a poisoned buffer of its own."""
    depth, odepth, linear = _depth(W, H, L, kind, reversed_z, seed)
    es = depth.itemsize
    drow = [W, W + 3, W]                    # elements
    arow = [W, W + 5, W + 1]                # bytes
    doff = [0, 0, 1]                        # elements past a 64-byte boundary
    aoff = [0, 0, 3]                        # bytes
    ds, abufs, aviews = [], [], []
    for l in range(L):
        buf = np.zeros(H * drow[l] + doff[l], depth.dtype)
        for r in range(H):
            buf[doff[l] + r * drow[l]:][:W] = depth[l, r]
        buf = emu._aligned(buf)
        ds.append(buf[doff[l]:])
        a = emu._aligned(np.full(H * arow[l] + aoff[l] + 7, POISON, np.uint8))
        abufs.append(a)
        aviews.append(a[aoff[l]:])
    cams = _cameras(W, H, L, reversed_z)
    f = Frame(harness.context(W, H, layers=L, layer_cameras=cams, reversed_z=reversed_z, high_quality_mask=hq), linear=linear)
    batch.run_pointers_batch(f, ds, [r * es for r in drow], aviews, arow)
    tag = f"pointers {W}x{H} {kind} reversed_z={reversed_z} hq={hq}"
    ao = []
    for l in range(L):
        written = np.zeros(abufs[l].shape, bool)
        for r in range(H):
            written[aoff[l] + r * arow[l]:][:W] = True
        assert (abufs[l][~written] == POISON).all(), f"{tag}: layer {l} stored outside its view"
        ao.append(np.stack([aviews[l][r * arow[l]:][:W] for r in range(H)]))
    _compare(f, W, H, cams, odepth, ao, linear, hq, tag)


# (io, depth kind, reversed Z, high_quality_mask): together they select every slot of the four batch units' tables -- the five prepare
# forms of an array, the seven of a pointer (D24S8 too), both Z directions, and the plain and premin final level of every depth format
CASES = [("arrays", "linear_f32", True, 0), ("arrays", "raw_f32", True, 1), ("arrays", "raw_f32", False, 0),
         ("arrays", "d16", True, 0), ("arrays", "d16", False, 1),
         ("pointers", "linear_f32", True, 0), ("pointers", "raw_f32", True, 1), ("pointers", "raw_f32", False, 0),
         ("pointers", "d16", True, 0), ("pointers", "d16", False, 1), ("pointers", "d24s8", True, 1), ("pointers", "d24s8", False, 0)]


def _case(io, kind, reversed_z, hq):
    (_arrays_case if io == "arrays" else _pointers_case)(kind, reversed_z, hq)


@pytest.mark.parametrize("io,kind,reversed_z,hq", CASES)
def test_each_layer_matches_the_oracle(io, kind, reversed_z, hq):
    _case(io, kind, reversed_z, hq)


def test_the_cases_launch_every_batch_kernel():
    """The launch ledger of the cases above holds every kernel the batch units build, and nothing else of theirs"""
    built = batch.kernels()
    assert len(built) == 20, sorted(built)
    ran = set()
    for c in CASES:
        emu.ledger_reset()
        _case(*c)
        ran |= batch.launched()
    assert ran == built, sorted(built - ran)


def test_one_layer_batch_of_a_large_ragged_frame():
    """One layer of 133 x 75 (ragged in both directions at every level) over an oversized array and over a misaligned pointer"""
    W, H = 133, 75
    depth, odepth, _ = _depth(W, H, 1, "raw_f32", True, 9)
    cams = _cameras(W, H, 1, True)
    f = Frame(harness.context(W, H, layers=1, layer_cameras=cams), linear=False)
    d = np.full((H + 2, W + 9), np.nan, np.float32)
    d[:H, :W] = depth[0]
    a = np.full((H + 2, W + 9), POISON, np.uint8)
    batch.run_arrays_batch(f, [d], [a])
    assert (a[H:] == POISON).all() and (a[:, W:] == POISON).all()
    _compare(f, W, H, cams, odepth, [a[:H, :W]], False, 0, "one layer, array")
