"""CPU tests of batches (meao_render_arrays_batch / meao_render_batch): each layer of a layered frame reads its own depth and writes
its own AO, in CUDA arrays or in device buffers of their own.

The batch kernels (build.py BATCH_SOURCES) run in the fiber emulator (tests/emu/frame_batch.cpp, linked against the emulator the other
CPU tests use).  Here: one layer of a large ragged frame over an oversized array and a misaligned pointer, bit-exact to the oracle's
single-layer frame on the AO and every debug buffer.  The case matrix over arrays and pointers, every depth format, both Z directions,
the plain and the premin final level, per-layer cameras and layers with a misaligned base or an odd row pitch -- launching every batch
kernel -- is tests/unit_matrix.py's, run by test_unit_matrix_emulated.py."""
import numpy as np

from miniengineao_b200 import Camera

import harness
from emu import batch  # noqa: E402  (tests/ is on sys.path via conftest)
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
