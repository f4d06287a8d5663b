"""The frames of the satellite units' case matrix (tests/unit_matrix.py) through libmeao on the H100: orthographic, mixed-projection and
bound-camera frames through the stage entry points, meao_render and meao_render_arrays; batches over tensors and CUDA arrays of each
layer's own; layer-viewport frames over CUDA arrays and pitched buffers.  Every layer's AO and every intermediate must equal its oracle
bit for bit, each layer against its own camera.

The emulated twin (test_unit_matrix_emulated.py) proves which kernel each case launches, that its interior tiles take TMA boxes and
that its tile-loop cases run the persistent upsample loop; the host code that makes those choices is the same source here.  What this
adds is the hardware: TMA boxes at layer boundaries and at every render tile height, MUFU reciprocals, surface stores, and the tile
loop's atomics and barriers with CTAs really in flight together.  A fresh context per case, because MEAO_REN_TILE and
MEAO_UPS_PERSIST_MIN_WAVES are read when a frame is recorded and a cached graph would keep another case's choice.  The tile-loop cases
run three frames through one context (half of them replaying a recorded graph), so the counters the last CTA re-arms are used again.
Last, one frame per unit at a size where the planner chooses the tile loop itself: a 4K orthographic frame, three 1080p layers of
mixed projections, and three 1080p batch layers as tensors and as CUDA arrays."""
import numpy as np
import pytest

import harness
import unit_matrix as um  # noqa: E402  (tests/ is on sys.path via conftest)
from gpu_harness import Array, rt, torch_cuda  # noqa: E402,F401  (the fixtures)
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

pytestmark = pytest.mark.gpu

POISON = 0xA7
DTYPES = {"f32": np.float32, "linear": np.float32, "d16": np.uint16, "d24s8": np.uint32}


def _tensor(torch, a):
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16)).cuda().view(torch.uint16)
    if a.dtype == np.uint32:
        return torch.from_numpy(a.view(np.int32)).cuda()
    return torch.from_numpy(a).cuda()


def _context(torch, c, use_graph=True):
    cams = c.cameras()
    kw = dict(device=0, layers=c.layers, sample_exhaustively=c.exhaustive, high_quality_mask=c.hq, use_graph=use_graph)
    if c.unit == "camera":
        # the host cameras are other ones: a bound frame must read the buffer's
        host = [Camera(k.pixelWidth, k.pixelHeight, nearClipPlane=1.0, farClipPlane=500.0, usesReversedZBuffer=c.reversed_z,
                       **(dict(orthographic=True, orthographicSize=2.0) if k.orthographic else dict(fieldOfView=70.0))) for k in cams]
        ao = harness.context(host[0], layer_cameras=host, **kw)
        ao.perLayerProjection = True
        ao.deviceCameras = torch.tensor([(k.nearClipPlane, k.farClipPlane, 1.0 / k.projection00) for k in cams], dtype=torch.float32,
                                        device="cuda")
        return ao, cams
    ao = harness.context(cams[0], layer_cameras=cams if c.layers > 1 else None, **kw)
    if c.unit == "mixed":
        ao.perLayerProjection = True
    return ao, cams


def _stage_frame(torch, ao, c, depth):
    d = _tensor(torch, depth if c.layers > 1 else depth[0])
    kind = ao._kind(str(d.dtype).replace("torch.", ""), c.linear)
    ao._update(False)
    ao._check(N.lib().meao_stage_downsample(ao._ctx, d.data_ptr(), kind, ao._stream()))
    for k in range(1, 5):
        ao.stage_render(k)
    for k in range(1, 5):
        if (c.hq >> (k - 1)) & 1:
            ao.stage_render_wide(k)
    for lo in range(4, 0, -1):
        ao.stage_upsample(lo)
    ao.synchronize()
    return ao.debug_buffer(17).reshape(depth.shape)


def _fused_frame(torch, ao, c, depth):
    out = ao.render(_tensor(torch, np.ascontiguousarray(depth if c.layers > 1 else depth[0])), linear=c.linear)
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(depth.shape)


def _array_frame(torch, rt, ao, c, depth):
    W, H = c.size
    shape = "layered" if c.layers > 1 else "2d"
    da, aa = Array(rt, W, H, depth.dtype, shape, c.layers), Array(rt, W, H, np.uint8, shape, c.layers)
    try:
        da.fill(depth)
        aa.fill(np.full(depth.shape, POISON, np.uint8))
        ao.render_arrays(da.handle, aa.handle, kind=um.ARRAY_KINDS[c.kind])
        torch.cuda.synchronize()
        return aa.read()
    finally:
        for a in (da, aa):
            ao.release_array(a.handle)
            a.free()


def _batch_pointers(torch, rt, ao, c, depth):
    W, H = c.size
    ds, outs, backs = [], [], []
    for l, (drow, doff, arow, aoff) in enumerate(um.batch_pointer_layout(c)):
        flat = np.zeros(H * drow + doff, depth.dtype)
        flat[doff:].reshape(H, drow)[:, :W] = depth[l]
        ds.append(_tensor(torch, flat)[doff:].view(H, drow)[:, :W])
        back = torch.full((H * arow + aoff + 7,), POISON, dtype=torch.uint8, device="cuda")
        outs.append(back[aoff:aoff + H * arow].view(H, arow)[:, :W])
        backs.append((back, aoff, arow))
    ao.render_batch(ds, outs, linear=c.linear)
    torch.cuda.synchronize()
    for l, (back, aoff, arow) in enumerate(backs):
        b = back.cpu().numpy()
        written = np.zeros(b.shape, bool)
        written[aoff:aoff + H * arow].reshape(H, arow)[:, :W] = True
        assert (b[~written] == POISON).all(), f"{c.id}: layer {l} stored outside its view"
    return np.stack([o.cpu().numpy() for o in outs])


def _batch_arrays(torch, rt, ao, c, depth):
    W, H = c.size
    da, aa = [], []
    try:
        for l, ((h, w), dshape, ashape) in enumerate(um.batch_array_layout(c)):
            img = np.full((h, w), np.inf if depth.dtype == np.float32 else 0, depth.dtype)
            img[:H, :W] = depth[l]
            d, a = Array(rt, w, h, depth.dtype, dshape), Array(rt, w, h, np.uint8, ashape)
            da.append(d)
            aa.append(a)
            d.fill(img[None])
            a.fill(np.full((1, h, w), POISON, np.uint8))
        ao.render_arrays_batch([d.handle for d in da], [a.handle for a in aa], kind=um.ARRAY_KINDS[c.kind])
        torch.cuda.synchronize()
        got = [a.read()[0] for a in aa]
        for l, g in enumerate(got):
            assert (g[H:] == POISON).all() and (g[:, W:] == POISON).all(), f"{c.id}: layer {l} stored outside W x H"
        return np.stack([g[:H, :W] for g in got])
    finally:
        for x in da + aa:
            ao.release_array(x.handle)
            x.free()


def _views_arrays(torch, rt, ao, c, depth):
    W, H = c.size
    table, dshape, (ds, dh, dw), ashape, (as_, ah, aw) = um.view_arrays_layout(c)
    dimg = np.full((ds, dh, dw), np.inf if depth.dtype == np.float32 else 0, depth.dtype)
    written = np.zeros((as_, ah, aw), bool)
    for l, (dx, dy, dsl, ax, ay, asl) in enumerate(table):
        dimg[dsl, dy:dy + H, dx:dx + W] = depth[l]
        written[asl, ay:ay + H, ax:ax + W] = True
    da, aa = Array(rt, dw, dh, depth.dtype, dshape, ds), Array(rt, aw, ah, np.uint8, ashape, as_)
    try:
        da.fill(dimg)
        aa.fill(np.full((as_, ah, aw), POISON, np.uint8))
        ao.layerViewports = table
        ao.render_arrays(da.handle, aa.handle, kind=um.ARRAY_KINDS[c.kind])
        torch.cuda.synchronize()
        got = aa.read()
    finally:
        for x in (da, aa):
            ao.release_array(x.handle)
            x.free()
    assert (got[~written] == POISON).all(), f"{c.id}: a store outside the AO rectangles"
    return np.stack([got[asl, ay:ay + H, ax:ax + W] for _, _, _, ax, ay, asl in table])


def _views_pitched(torch, rt, ao, c, depth):
    W, H = c.size
    table, drow, dsl, arow, asl, slices = um.view_pitched_layout(c)
    es = depth.itemsize
    dflat = np.zeros(slices * dsl, depth.dtype)
    written = np.zeros(slices * asl, bool)
    for l, (dx, dy, ds, ax, ay, as_) in enumerate(table):
        for r in range(H):
            o = ds * dsl + (dy + r) * drow + dx
            dflat[o:o + W] = depth[l, r]
            o = as_ * asl + (ay + r) * arow + ax
            written[o:o + W] = True
    d = _tensor(torch, dflat)
    out = torch.full((slices * asl,), POISON, dtype=torch.uint8, device="cuda")
    ao.layerViewports = table
    ao.LateUpdate()
    kind = ao._kind(str(d.dtype).replace("torch.", ""), c.linear)
    ao._check(ao._lib.meao_render_pitched(ao._ctx, d.data_ptr(), drow * es, dsl * es, kind, out.data_ptr(), arow, asl, ao._stream()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert (got[~written] == POISON).all(), f"{c.id}: a store outside the AO rectangles"
    return np.stack([np.stack([got[as_ * asl + (ay + r) * arow + ax:][:W] for r in range(H)]) for _, _, _, ax, ay, as_ in table])


FRAMES = {"stage": lambda torch, rt, ao, c, d: _stage_frame(torch, ao, c, d), "fused": lambda torch, rt, ao, c, d: _fused_frame(torch, ao, c, d),
          "arrays": lambda torch, rt, ao, c, d: _array_frame(torch, rt, ao, c, d)}
TARGETS = {("batch", "pointers"): _batch_pointers, ("batch", "arrays"): _batch_arrays, ("views", "arrays"): _views_arrays,
           ("views", "pitched"): _views_pitched}


def _run(torch, rt, c, use_graph=True, frames=None, buffers=True):
    W, H = c.size
    ao, cams = _context(torch, c, use_graph)
    try:
        for n in range(frames or c.frames):
            depth, seen = um.depth(c, n)
            run = TARGETS.get((c.unit, c.form)) or FRAMES[c.form]
            got = run(torch, rt, ao, c, depth)
            ids = c.buffer_ids() if buffers else []
            bufs = {bid: ao.debug_buffer(bid) for bid in ids}
            for l, cam in enumerate(cams):
                ref = um.oracle(c, cam, threads=8)
                want = ref.run(seen[l])
                bad = int((got[l] != want).sum())
                assert bad == 0, f"{c.id} frame {n}: the AO of layer {l} differs from the oracle in {bad} pixels"
                assert int(got[l].astype(np.uint64).sum()) == int(want.astype(np.uint64).sum())
                harness.compare_buffers(lambda bid: bufs[bid][l] if c.layers > 1 else bufs[bid], ref, f"{c.id} frame {n} layer {l}", ids)
    finally:
        ao.close()


@pytest.mark.parametrize("case", um.CASES, ids=lambda c: c.id)
def test_case_matches_the_oracle(torch_cuda, rt, case, monkeypatch):
    c = case
    monkeypatch.setenv("MEAO_REN_TILE", str(c.tile))
    if c.persist:
        monkeypatch.setenv("MEAO_UPS_PERSIST_MIN_WAVES", "0.0001")
    # the tile-loop cases alternate between launching each frame and replaying the recorded graph
    _run(torch_cuda, rt, c, use_graph=not (c.persist and c.hq & 1))


# one frame per unit at a size where the planner takes the persistent tile loop itself (2 waves of tiles or more)
NATURAL = [um.Case("ortho", "fused", 1, (um.O,), "f32", size=(3840, 2160)),
           um.Case("mixed", "fused", 3, (um.P, um.O, um.P), "d16", size=(1920, 1080)),
           um.Case("batch", "pointers", 3, (um.P,) * 3, "f32", size=(1920, 1080)),
           um.Case("batch", "arrays", 3, (um.P,) * 3, "d16", hq=1, size=(1920, 1080))]


@pytest.mark.parametrize("case", NATURAL, ids=lambda c: c.id.replace("-tile8", ""))
def test_the_planners_own_tile_loop_matches_the_oracle(torch_cuda, rt, case, monkeypatch):
    monkeypatch.delenv("MEAO_UPS_PERSIST_MIN_WAVES", raising=False)
    monkeypatch.delenv("MEAO_REN_TILE", raising=False)
    assert um.loop_tiles(case) >= 2 * 132 * 5
    _run(torch_cuda, rt, case, frames=2, buffers=case.unit != "ortho")
