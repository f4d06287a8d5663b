"""GPU tests of the hierarchy depth (include/meao.h meao_set_hierarchy_depth) on the H100.  For every depth 1-4 each frame form must equal the
oracle of that depth bit for bit, on the AO and on every debug buffer the frame writes: pointer frames (graph, MEAO_FLAG_NO_GRAPH,
pitched views), host frames (synchronous and asynchronous), CUDA arrays and their viewports, layered frames, batches, orthographic and
[P, O] mixed frames and a bound device camera buffer.  Also: torch.cuda.graph capture after one settling frame, a depth change inside
reservations (one arena allocation, no instantiation on returning to a planned (W, H, L, depth)), 2-3 row bands on one GPU, and
refusals that launch nothing."""
import numpy as np
import pytest

import depth_oracle as DO
import harness
from gpu_harness import Array, native_bands, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import Camera, synth
from miniengineao_b200 import _native as N

pytestmark = pytest.mark.gpu

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
DEPTHS = [1, 2, 3, 4]


def camera(W, H, l=0, reversed_z=True, ortho_=False):
    near, far = 0.2 + 0.15 * l, 60.0 + 40.0 * l
    if ortho_:
        return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, orthographic=True, orthographicSize=3.0 + 2.5 * l)
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, fieldOfView=50.0 + 7.0 * l)


def oracle(cam, n, linear=False, **kw):
    return DO.for_camera(cam, n, linear=linear, threads=8, **kw)


def context(cam, n, **kw):
    ao = harness.context(cam, device=0, **kw)
    ao.hierarchyDepth = n
    return ao


def check(ao, cams, depth, got, n, tag, buffers=True, **kw):
    """Layer l of `got` (and of every written debug buffer) against the oracle of cams[l] at depth n."""
    L = len(cams)
    ids = DO.written_ids(n, kw.get("high_quality_mask", 0)) if buffers else []
    bufs = {bid: ao.debug_buffer(bid) for bid in ids}
    for l, cam in enumerate(cams):
        orc = oracle(cam, n, **kw)
        ref = orc.run(depth[l])
        assert np.array_equal(got[l], ref), f"{tag}: layer {l} AO ({int((got[l] != ref).sum())} codes differ)"
        harness.compare_buffers(lambda bid: bufs[bid][l] if L > 1 else bufs[bid], orc, f"{tag} layer {l}", ids)


def cuda(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---- single-layer perspective frames --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", DEPTHS)
@pytest.mark.parametrize("reversed_z,kw", [(True, dict()), (False, dict(high_quality_mask=0b1011, sample_exhaustively=True))],
                         ids=["plain", "hq11-exh-stdz"])
def test_pointer_and_host_frames(torch_cuda, n, reversed_z, kw):
    torch = torch_cuda
    W, H = 333, 187
    cam = camera(W, H, reversed_z=reversed_z)
    d = harness.frames(W, H, 1, seed=n, reversed_z=reversed_z)
    ao = context(cam, n, **kw)
    check(ao, [cam], d, ao.render(cuda(torch, d[0])).cpu().numpy()[None], n, f"graph n={n}", **kw)
    assert ao.launch_count == ao.kernels_per_frame == 1 + 2 * n + bin(kw.get("high_quality_mask", 0) & ((1 << n) - 1)).count("1")
    check(ao, [cam], d, ao.render_host(d[0])[None], n, f"host n={n}", buffers=False, **kw)
    # a pitched view: the corner of a larger target
    big = torch.full((H + 5, W + 40), 0.5, dtype=torch.float32, device="cuda")
    big[:H, :W] = cuda(torch, d[0])
    out = torch.full((H + 3, W + 24), 7, dtype=torch.uint8, device="cuda")
    ao.render(big[:H, :W], out[:H, :W])
    check(ao, [cam], d, out[:H, :W].cpu().numpy()[None], n, f"pitched n={n}", buffers=False, **kw)
    assert (out[H:] == 7).all() and (out[:, W:] == 7).all()
    ao.close()
    ng = context(cam, n, use_graph=False, **kw)
    check(ng, [cam], d, ng.render(cuda(torch, d[0])).cpu().numpy()[None], n, f"no graph n={n}", **kw)
    ng.close()


@pytest.mark.parametrize("n", DEPTHS)
def test_host_async(torch_cuda, n):
    W, H = 200, 120
    cam = camera(W, H)
    ao = context(cam, n, high_quality_mask=n)
    frames = [harness.frames(W, H, 1, seed=20 + i) for i in range(3)]
    outs = [np.zeros((H, W), np.uint8) for _ in range(3)]
    ao.LateUpdate()                                     # the raw calls below do not apply the properties
    for i in range(3):
        ao._check(ao._lib.meao_render_host_async(ao._ctx, frames[i][0].ctypes.data, 0, outs[i].ctypes.data, i % 2))
        if i >= 1:
            ao._check(ao._lib.meao_host_wait(ao._ctx, (i - 1) % 2))
    ao._check(ao._lib.meao_host_wait(ao._ctx, 0))
    for i in range(3):
        check(ao, [cam], frames[i], outs[i][None], n, f"async n={n} frame {i}", buffers=False, high_quality_mask=n)
    ao.close()


# ---- layered frames, CUDA arrays and batches ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", DEPTHS)
def test_layered_arrays_and_batches(torch_cuda, rt, n):
    torch = torch_cuda
    W, H, L = 160, 96, 3
    cams = [camera(W, H, l) for l in range(L)]
    kw = dict(high_quality_mask=0b0110)
    d = harness.frames(W, H, L, seed=40 + n)
    ao = context(cams[0], n, layers=L, layer_cameras=cams, **kw)
    check(ao, cams, d, ao.render(cuda(torch, d)).cpu().numpy(), n, f"layered n={n}", **kw)
    da, aa = Array(rt, W, H, np.float32, "layered", L), Array(rt, W, H, np.uint8, "layered", L)
    da.fill(d)
    ao.render_arrays(da.handle, aa.handle)
    torch.cuda.synchronize()
    check(ao, cams, d, aa.read(), n, f"arrays n={n}", **kw)
    # a viewport of larger arrays
    db, ab = Array(rt, W + 17, H + 9, np.float32, "layered", L), Array(rt, W + 11, H + 5, np.uint8, "layered", L)
    big = np.full((L, H + 9, W + 17), 0.25, np.float32)
    big[:, 9:, 17:] = d
    db.fill(big)
    ao.render_arrays(db.handle, ab.handle, depth_origin=(17, 9), ao_origin=(11, 5))
    torch.cuda.synchronize()
    check(ao, cams, d, ab.read()[:, 5:, 11:], n, f"arrays_at n={n}", buffers=False, **kw)
    outs = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(L)]
    ao.render_batch([cuda(torch, x) for x in d], outs)
    check(ao, cams, d, np.stack([o.cpu().numpy() for o in outs]), n, f"batch n={n}", buffers=False, **kw)
    for a in (da, aa, db, ab):
        ao.release_array(a.handle)
        a.free()
    ao.close()


@pytest.mark.parametrize("n", DEPTHS)
def test_layer_viewports(torch_cuda, rt, n):
    torch = torch_cuda
    W, H, L = 120, 80, 2
    cams = [camera(W, H, l) for l in range(L)]
    d = harness.frames(W, H, L, seed=60 + n)
    ao = context(cams[0], n, layers=L, layer_cameras=cams)
    ao.layerViewports = [(0, 0, 0, W, 0, 0), (W, 0, 0, 0, 0, 0)]           # side by side in one image, the AO halves swapped
    da, aa = Array(rt, 2 * W, H, np.float32), Array(rt, 2 * W, H, np.uint8)
    da.fill(np.concatenate([d[0], d[1]], axis=1)[None])
    ao.render_arrays(da.handle, aa.handle)
    torch.cuda.synchronize()
    o = aa.read()[0]
    check(ao, cams, d, np.stack([o[:, W:], o[:, :W]]), n, f"viewports n={n}", buffers=False)
    for a in (da, aa):
        ao.release_array(a.handle)
        a.free()
    ao.close()


# ---- orthographic, mixed and device cameras ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", DEPTHS)
def test_orthographic_and_mixed(torch_cuda, n):
    torch = torch_cuda
    W, H = 211, 117
    kw = dict(high_quality_mask=0b1100, sample_exhaustively=True)
    cam = camera(W, H, ortho_=True)
    d = harness.frames(W, H, 1, seed=80 + n)
    ao = context(cam, n, **kw)
    check(ao, [cam], d, ao.render(cuda(torch, d[0])).cpu().numpy()[None], n, f"ortho n={n}", **kw)
    ao.close()
    cams = [camera(W, H, 0), camera(W, H, 1, ortho_=True)]
    d = harness.frames(W, H, 2, seed=90 + n)
    ao = context(cams[0], n, layers=2, layer_cameras=cams, **kw)
    ao.perLayerProjection = True
    check(ao, cams, d, ao.render(cuda(torch, d)).cpu().numpy(), n, f"mixed n={n}", **kw)
    ao.close()


@pytest.mark.parametrize("n", DEPTHS)
def test_device_cameras(torch_cuda, n):
    torch = torch_cuda
    W, H, L = 150, 90, 2
    cams = [camera(W, H, l) for l in range(L)]
    host = [Camera(W, H, nearClipPlane=1.0, farClipPlane=500.0, fieldOfView=70.0) for _ in range(L)]
    d = harness.frames(W, H, L, seed=100 + n)
    ao = context(host[0], n, layers=L, layer_cameras=host, high_quality_mask=15)
    ao.deviceCameras = torch.tensor([(c.nearClipPlane, c.farClipPlane, 1.0 / c.projection00) for c in cams], dtype=torch.float32, device="cuda")
    check(ao, cams, d, ao.render(cuda(torch, d)).cpu().numpy(), n, f"device cameras n={n}", high_quality_mask=15)
    assert ao.kernels_per_frame == 2 + 2 * n + n
    ao.close()


# ---- capture, reservations and row bands ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", DEPTHS)
def test_torch_graph_capture(torch_cuda, n):
    torch = torch_cuda
    W, H = 256, 144
    cam = camera(W, H)
    ao = context(cam, n)
    d = harness.frames(W, H, 2, seed=110 + n)
    dt, out = cuda(torch, d[0]), torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    ao.render(dt, out)                                  # the settling frame
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ao.render(dt, out, stream=s)
    gen = ao.frame_generation
    for i in (1, 0):
        dt.copy_(cuda(torch, d[i]))
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert ao.frame_generation == gen
        check(ao, [cam], d[i:i + 1], out.cpu().numpy()[None], n, f"capture n={n} frame {i}", buffers=False)
    ao.close()


def test_depth_change_inside_reservations(torch_cuda):
    torch = torch_cuda
    sizes = [(320, 180), (256, 160)]
    ao = harness.context(320, 180, device=0, max_resolution=(320, 180))
    ao.maxLayers = 2
    depth = {s: harness.frames(s[0], s[1], 1, seed=s[0]) for s in sizes}

    def frame(n, size):
        ao.camera.pixelWidth, ao.camera.pixelHeight = size
        ao.hierarchyDepth = n
        got = ao.render(cuda(torch, depth[size][0])).cpu().numpy()
        check(ao, [Camera(*size)], depth[size], got[None], n, f"reserved n={n} {size}", buffers=False)

    for n in (4, 2, 1, 3):
        for size in sizes:
            frame(n, size)
        before = ao.reservation()
        for size in sizes:                              # back to planned (W, H, L, n): no instantiation
            frame(n, size)
        after = ao.reservation()
        assert after["graph_instantiations"] == before["graph_instantiations"], n
        assert after["arena_allocations"] == 1, n
    ao.close()


@pytest.mark.parametrize("n,bands", [(1, 2), (2, 3), (3, 2)])
def test_row_bands(torch_cuda, n, bands):
    """The native exchange under the existing scheduling contract: every band's graph on its own stream; the halo rows are those of the
    depth-4 frame."""
    torch = torch_cuda
    W, H = 1920, 1080
    cuts, ctxs, streams = native_bands(torch, W, H, bands, intensity=1.1, hierarchyDepth=n)
    outs = [torch.zeros((cuts[i + 1] - cuts[i], W), dtype=torch.uint8, device="cuda") for i in range(bands)]
    orc = DO.DepthOracle(W, H, n, threads=8, intensity=1.1)
    for frame in range(2):
        depth = synth.lin01_to_raw(synth.corridor(W, H, frame=frame))
        ref = orc.run(depth)
        bufs = [torch.from_numpy(depth[cuts[i]:cuts[i + 1]]).cuda() for i in range(bands)]
        torch.cuda.synchronize()
        for i, a in enumerate(ctxs):
            a.band_step(bufs[i], outs[i], stream=streams[i])
        torch.cuda.synchronize()
        assert [a.band_status()["error"] for a in ctxs] == [0] * bands
        got = np.concatenate([o.cpu().numpy() for o in outs])
        assert np.array_equal(got, ref), f"bands n={n} frame {frame}: {int((got != ref).sum())} codes differ"
    for a in ctxs:
        a.close()


# ---- refusals --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3])
def test_refusals_launch_nothing(torch_cuda, n):
    torch = torch_cuda
    W, H = 128, 96
    cam = camera(W, H)
    ao = context(cam, n)
    d = harness.frames(W, H, 1, seed=130 + n)
    ao.render(cuda(torch, d[0]))
    torch.cuda.synchronize()
    before = ao.launch_count
    ao.stage_downsample(cuda(torch, d[0]))
    for k in range(1, 5):
        ao.stage_render(k)                              # unchanged: every level may be rendered
    for lo in range(4, n, -1):
        mid = ao.launch_count
        assert ao._lib.meao_stage_upsample(ao._ctx, lo, None, None) == N.MEAO_ERR_INVALID
        assert "hierarchy depth" in ao._lib.meao_last_error(ao._ctx).decode()
        assert ao.launch_count == mid
    for lo in range(n, 0, -1):
        ao.stage_upsample(lo)
    torch.cuda.synchronize()
    assert ao.launch_count == before + 1 + 4 + n
    orc = oracle(cam, n)
    assert np.array_equal(ao.debug_buffer(17), orc.run(d[0]))        # the stage frame of depth n: Occlusion<n> read at lo = n
    gen = ao._lib.meao_frame_generation(ao._ctx)
    assert ao._lib.meao_set_hierarchy_depth(ao._ctx, 0) == N.MEAO_ERR_INVALID
    assert ao._lib.meao_frame_generation(ao._ctx) == gen and ao.launch_count == before + 1 + 4 + n
    ao.close()
