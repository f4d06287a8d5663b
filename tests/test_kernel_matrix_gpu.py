"""The frames of the kernel case matrix (tests/kernel_matrix.py) through libmeao on the H100: the stage entry points (prepare, render,
wide render, upsample: the final level unfused), meao_render (the fused final level) and meao_render_arrays.  Every layer's AO and
every intermediate must equal the oracle bit for bit.

The emulated twin (test_kernel_matrix_emulated.py) proves which kernel each case launches; the host code that chooses it (frame_record.h
and the launchers) is the same source here, and MEAO_REN_TILE fixes the one choice that depends on the device, the render tile height.
What this adds is the hardware: real TMA boxes at layer boundaries and at every tile height, MUFU reciprocals, surface stores.  A fresh
context per case, because MEAO_REN_TILE is read when a frame is recorded and a cached graph would keep another case's tile."""
import numpy as np
import pytest

import harness  # noqa: E402  (tests/ is on sys.path via conftest)
import kernel_matrix as km  # noqa: E402
from gpu_harness import Array, rt, torch_cuda  # noqa: E402,F401  (the fixtures)

pytestmark = pytest.mark.gpu

ARRAY_KINDS = {"linear": "linear_f32", "f32": "raw_f32", "d16": "d16"}


def _tensor(torch, depth):
    if depth.dtype == np.uint16:
        return torch.from_numpy(depth.view(np.int16)).cuda().view(torch.uint16)
    if depth.dtype == np.uint32:
        return torch.from_numpy(depth.view(np.int32)).cuda()
    return torch.from_numpy(depth).cuda()


def _stage_frame(torch, ao, c, depth):
    from miniengineao_b200 import _native as N
    d = _tensor(torch, depth if c.layers > 1 else depth[0])
    kind = ao._kind(str(d.dtype).replace("torch.", ""), c.kind == "linear")
    ao._update(False)
    ao._check(N.lib().meao_stage_downsample(ao._ctx, d.data_ptr(), kind, ao._stream()))
    levels = [1] if c.single_scale else [1, 2, 3, 4]
    for k in levels:
        ao.stage_render(k)
    for k in levels:
        if (c.hq >> (k - 1)) & 1:
            ao.stage_render_wide(k)
    for lo in reversed(levels):
        ao.stage_upsample(lo)
    ao.synchronize()
    return ao.debug_buffer(17).reshape(depth.shape)


def _fused_frame(torch, ao, c, depth):
    d = _tensor(torch, depth if c.layers > 1 else depth[0])
    out = ao.render(d, linear=c.kind == "linear")
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(depth.shape)


def _array_frame(torch, rt, ao, c, depth):
    W, H = c.size
    shape = "layered" if c.layers > 1 else "2d"
    da = Array(rt, W, H, depth.dtype, shape, c.layers)
    aa = Array(rt, W, H, np.uint8, shape, c.layers)
    try:
        da.fill(depth)
        aa.fill(np.full(depth.shape, 0x5A, np.uint8))
        ao.render_arrays(da.handle, aa.handle, kind=ARRAY_KINDS[c.kind])
        torch.cuda.synchronize()
        return aa.read()
    finally:
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()


@pytest.mark.parametrize("case", km.FRAME_CASES, ids=lambda c: c.id)
def test_case_matches_the_oracle(torch_cuda, rt, case, monkeypatch):
    c = case
    monkeypatch.setenv("MEAO_REN_TILE", str(c.tile))
    W, H = c.size
    depth, seen = km.depth(c)
    ao = harness.context(W, H, device=0, layers=c.layers, reversed_z=c.reversed_z, sample_exhaustively=c.exhaustive, high_quality_mask=c.hq,
              single_scale=c.single_scale, intensity=1.1)
    if c.form == "stage":
        got = _stage_frame(torch_cuda, ao, c, depth)
    elif c.form == "fused":
        got = _fused_frame(torch_cuda, ao, c, depth)
    else:
        got = _array_frame(torch_cuda, rt, ao, c, depth)
    bufs = {bid: ao.debug_buffer(bid) for bid in c.buffer_ids()}
    for l in range(c.layers):
        orc = harness.oracle(W, H, threads=8, **c.oracle_kw())
        n = int((got[l] != orc.run(seen[l])).sum())
        assert n == 0, f"{c.id}: the AO of layer {l} differs from the oracle in {n} pixels"
        harness.compare_buffers(lambda bid: bufs[bid][l] if c.layers > 1 else bufs[bid], orc, f"{c.id} layer {l}", c.buffer_ids())
