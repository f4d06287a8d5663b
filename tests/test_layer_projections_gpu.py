"""GPU tests of per-layer projections (meao_set_layer_projections) on the H100: a layered frame whose layers mix perspective and
orthographic cameras must give, layer by layer, the AO and every debug buffer (ids 1-21) of a single-layer frame of that layer's depth on a
context with that projection and camera -- through pointer frames of every depth kind and Z direction, every variant, pitched views,
host frames (synchronous and the asynchronous two-slot stream), CUDA
arrays (layered and cube-map, and _at viewports), MEAO_FLAG_NO_GRAPH, the plugin event and torch.cuda.graph capture.  An orthographic zoom
and a field-of-view change take effect at the next frame without a graph instantiation, a layer change inside a reservation that clears
the table neither waits for the GPU nor allocates, uniform tables launch the kernels of the context projection, and the refusals launch nothing."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, backlog, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

pytestmark = pytest.mark.gpu

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
LINEAR = {"f32": False, "linear": True, "d16": False, "d24s8": False}


def cameras(W, H, table, reversed_z=True):
    """One camera per layer, each with planes and a field of view (half-width) of its own."""
    out = []
    for l, p in enumerate(table):
        near, far = 0.2 + 0.15 * l, 60.0 + 40.0 * l
        if p == O:
            out.append(Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, orthographic=True,
                              orthographicSize=3.0 + 2.5 * l))
        else:
            out.append(Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, fieldOfView=50.0 + 7.0 * l))
    return out


def mixed_context(cams, **kw):
    ao = harness.context(cams[0], device=0, layers=len(cams), layer_cameras=cams, **kw)
    ao.perLayerProjection = True
    return ao


def depth_of(W, H, kind, reversed_z, L, seed=0):
    """(the [L, H, W] depth in the ingest format of `kind`, the same as the single-layer contexts read it)."""
    if kind == "linear":
        return harness.contrasting_layers(W, H, L, seed=seed)
    return harness.ingest(harness.frames(W, H, L, seed=seed, reversed_z=reversed_z), kind)[0]


def to_tensor(torch, d):
    if d.dtype == np.uint32:
        d = d.view(np.int32)
    return torch.from_numpy(np.ascontiguousarray(d)).cuda()


def reference(torch, cam, depth, ids, linear=False, **kw):
    """The AO and buffers `ids` of one single-layer frame of `depth` on a fresh context with the camera's projection and camera."""
    ao = harness.context(cam, device=0, **kw)
    out = ao.render(to_tensor(torch, depth), linear=linear).cpu().numpy()
    bufs = {bid: ao.debug_buffer(bid) for bid in ids}
    assert ao._lib.meao_get_projection(ao._ctx) == (O if cam.orthographic else P)
    ao.close()
    return out, bufs


def check_layers(torch, ao, cams, depth, got, tag, linear=False, **kw):
    ids = harness.buffer_ids(kw.get("high_quality_mask", 0), kw.get("single_scale", False))
    bufs = {bid: ao.debug_buffer(bid) for bid in ids}
    for l, cam in enumerate(cams):
        ref, rbufs = reference(torch, cam, depth[l], ids, linear=linear, **kw)
        assert np.array_equal(got[l], ref), f"{tag}: layer {l} AO"
        for bid in ids:
            a, b = bufs[bid][l], rbufs[bid]
            view = {1: np.uint8, 2: np.uint16, 4: np.uint32}[a.dtype.itemsize]
            assert a.dtype == b.dtype and np.array_equal(a.view(view), b.view(view)), f"{tag}: layer {l} buffer {bid}"


def table_of(ao):
    out = (C.c_int32 * 64)()
    n = ao._lib.meao_get_layer_projections(ao._ctx, out, 64)
    return list(out[:n])


@pytest.mark.parametrize("reversed_z", [True, False])
@pytest.mark.parametrize("kind", list(LINEAR))
@pytest.mark.parametrize("table", [[P, O], [O, P, O, O]])
def test_pointer_frames(torch_cuda, table, kind, reversed_z):
    W, H = 161, 93
    cams = cameras(W, H, table, reversed_z)
    d = depth_of(W, H, kind, reversed_z, len(table), seed=3)
    ao = mixed_context(cams)
    got = ao.render(to_tensor(torch_cuda, d), linear=LINEAR[kind]).cpu().numpy()
    assert table_of(ao) == table
    check_layers(torch_cuda, ao, cams, d, got, f"{table} {kind} rz={reversed_z}", linear=LINEAR[kind])


@pytest.mark.parametrize("params", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True),
                                    dict(high_quality_mask=5, sample_exhaustively=True, use_graph=False)])
def test_variants_host_and_no_graph(torch_cuda, params):
    W, H = 333, 187
    table = [O, P, O]
    cams = cameras(W, H, table)
    d = depth_of(W, H, "f32", True, 3, seed=5)
    ao = mixed_context(cams, **params)
    got = ao.render(to_tensor(torch_cuda, d)).cpu().numpy()
    ref_kw = {k: v for k, v in params.items() if k != "use_graph"}
    check_layers(torch_cuda, ao, cams, d, got, f"variant {params}", **ref_kw)
    got = ao.render_host(d)
    check_layers(torch_cuda, ao, cams, d, got, f"host variant {params}", **ref_kw)


def test_cube_alternating_and_live_constants(torch_cuda):
    """A 6-face cube of 512 x 512 faces with alternating projections, then an orthographic zoom and a field-of-view change from one
    frame to the next: frame constants, so no graph instantiation, each taking effect at the very next frame."""
    W, H = 512, 512
    table = [P, O] * 3
    cams = cameras(W, H, table)
    d = depth_of(W, H, "f32", True, 6, seed=7)
    ao = mixed_context(cams)
    t = to_tensor(torch_cuda, d)
    got = ao.render(t).cpu().numpy()
    check_layers(torch_cuda, ao, cams, d, got, "cube")
    before = ao.reservation()["graph_instantiations"]
    for step in range(2):
        cams[1].orthographicSize *= 1.7
        cams[2].fieldOfView += 9.0
        got = ao.render(t).cpu().numpy()
        for l in (1, 2, 3):
            ref, _ = reference(torch_cuda, cams[l], d[l], [])
            assert np.array_equal(got[l], ref), (step, l)
    assert ao.reservation()["graph_instantiations"] == before


@pytest.mark.parametrize("shape,table", [("layered", [O, P]), ("cube", [P, O, O, P, O, P])])
def test_cuda_arrays(torch_cuda, rt, shape, table):
    L = len(table)
    W, H = (61, 61) if shape == "cube" else (83, 61)
    cams = cameras(W, H, table)
    for kind, dtype, ikind in (("raw_f32", np.float32, "f32"), ("d16", np.uint16, "d16"), ("linear_f32", np.float32, "linear")):
        d = depth_of(W, H, ikind, True, L, seed=L)
        dep = Array(rt, W, H, dtype, shape=shape, layers=L)
        aoa = Array(rt, W, H, np.uint8, shape=shape, layers=L)
        dep.fill(d.astype(dtype))
        ao = mixed_context(cams)
        ao.render_arrays(dep.handle, aoa.handle, kind=kind)
        torch_cuda.cuda.synchronize()
        check_layers(torch_cuda, ao, cams, d, aoa.read().reshape(L, H, W), f"{shape} {kind}", linear=ikind == "linear")
        ao.close()
        dep.free(); aoa.free()


def test_arrays_at_viewport(torch_cuda, rt):
    W, H, L = 64, 40, 2
    table = [P, O]
    cams = cameras(W, H, table)
    d = depth_of(W, H, "f32", True, L, seed=9)
    big = np.full((L, H + 10, W + 20), 0.25, np.float32)
    big[:, 4:4 + H, 7:7 + W] = d
    dep = Array(rt, W + 20, H + 10, np.float32, shape="layered", layers=L)
    aoa = Array(rt, W + 30, H + 6, np.uint8, shape="layered", layers=L)
    dep.fill(big)
    aoa.fill(np.full((L, H + 6, W + 30), 9, np.uint8))
    ao = mixed_context(cams)
    ao.render_arrays(dep.handle, aoa.handle, depth_origin=(7, 4), ao_origin=(11, 2))
    torch_cuda.cuda.synchronize()
    got = aoa.read().reshape(L, H + 6, W + 30)
    check_layers(torch_cuda, ao, cams, d, got[:, 2:2 + H, 11:11 + W], "arrays_at")
    mask = np.ones(got.shape, bool)
    mask[:, 2:2 + H, 11:11 + W] = False
    assert (got[mask] == 9).all()
    dep.free(); aoa.free()


def test_plugin_event_and_torch_graph_capture(torch_cuda):
    torch = torch_cuda
    W, H = 256, 144
    table = [O, P, O, O]
    cams = cameras(W, H, table)
    d = depth_of(W, H, "d24s8", True, 4, seed=4)
    ao = mixed_context(cams, high_quality_mask=2)
    depth = to_tensor(torch, d)
    out = torch.empty((4, H, W), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ao.render(depth, out, stream=s)     # one settling frame
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    out.fill_(0)
    with torch.cuda.graph(g, stream=s):
        ao.render(depth, out, stream=s)
    g.replay()
    torch.cuda.synchronize()
    check_layers(torch, ao, cams, d, out.cpu().numpy(), "captured", high_quality_mask=2)
    lib = N.lib()
    o = torch.zeros((4, H, W), dtype=torch.uint8, device="cuda")
    assert lib.meao_bind_event(ao._ctx, 95, C.c_void_p(depth.data_ptr()), N.MEAO_DEPTH_RAW_D24S8, C.c_void_p(o.data_ptr()), None) == 0
    lib.meao_get_render_event_func()(95)
    torch.cuda.synchronize()
    assert np.array_equal(o.cpu().numpy(), out.cpu().numpy())
    assert lib.meao_bind_event(ao._ctx, 95, None, 0, None, None) == 0


def test_dynamic_layer_counts_inside_a_reservation(torch_cuda):
    """Inside a layer reservation a layer change clears the table as host bookkeeping: behind a half-second backlog of the GPU it waits
    for nothing and allocates nothing, a revisited count without a table replays its graph, and every frame equals fresh single-layer
    frames of the projections then in effect.  Setting a table again is structural (include/meao.h): it re-plans behind a device
    synchronise, so that step drains the backlog."""
    torch = torch_cuda
    s = torch.cuda.Stream()
    W, H = 200, 120
    table4 = [P, O, O, P]
    cams4 = cameras(W, H, table4)
    d = depth_of(W, H, "f32", True, 4, seed=13)
    dev = {L: to_tensor(torch, d[:L]) for L in (2, 3, 4)}
    out = {L: torch.empty((L, H, W), dtype=torch.uint8, device="cuda") for L in dev}
    ao = mixed_context(cams4)
    ao.maxLayers = 4
    ao.render(dev[4], out[4], stream=s)
    s.synchronize()
    check_layers(torch, ao, cams4, d, out[4].cpu().numpy(), "L=4")
    r0 = ao.reservation()
    main = cams4[0]                             # the context's camera (perspective), which every layer takes once the tables are gone
    e = backlog(torch, s, ao, dev[4], out[4])
    ao.layers, ao.layerCameras, ao.perLayerProjection = 3, None, False     # the change clears the projection table
    ao.render(dev[3], out[3], stream=s)
    assert not e.query(), "a layer change that cleared the projection table waited for the GPU"
    ao.layers = 2
    ao.render(dev[2], out[2], stream=s)
    assert not e.query(), "a layer change without a table waited for the GPU"
    inst = ao.reservation()["graph_instantiations"]
    ao.layers = 3                               # a planned count without a table: a plain replay
    ao.render(dev[3], out[3], stream=s)
    assert not e.query(), "a change to a planned layer count waited for the GPU"
    assert ao.reservation()["graph_instantiations"] == inst
    s.synchronize()
    got3 = out[3].cpu().numpy()
    for l in range(3):
        ref, _ = reference(torch, main, d[l], [])
        assert np.array_equal(got3[l], ref), ("no table", l)
    # setting a table again is a structural input: the re-plan synchronises the device
    e = backlog(torch, s, ao, dev[3], out[3])
    cams2 = cameras(W, H, [O, P])
    ao.layers, ao.layerCameras, ao.perLayerProjection = 2, cams2, True
    ao.render(dev[2], out[2], stream=s)
    assert e.query(), "setting a projection table is expected to re-plan behind a device synchronise"
    s.synchronize()
    assert table_of(ao) == [O, P]
    check_layers(torch, ao, cams2, d[:2], out[2].cpu().numpy(), "L=2 [O, P]")
    assert ao.reservation()["arena_allocations"] == r0["arena_allocations"]


def test_pitched_views_and_host_frames(torch_cuda):
    """meao_render_pitched on views of larger tensors (own row and layer pitches; nothing outside the view written), and the host frame
    stream (meao_render_host_async over both staging slots)."""
    torch = torch_cuda
    W, H, L = 130, 70, 3
    table = [O, P, O]
    cams = cameras(W, H, table, reversed_z=False)
    d = depth_of(W, H, "f32", False, L, seed=2)
    big = torch.full((L + 1, H + 3, W + 37), 0.5, dtype=torch.float32, device="cuda")
    big[1:, 1:H + 1, 5:W + 5] = torch.from_numpy(d).cuda()
    out_big = torch.full((L, H + 2, W + 19), 7, dtype=torch.uint8, device="cuda")
    ao = mixed_context(cams)
    ao.render(big[1:, 1:H + 1, 5:W + 5], out_big[:, 1:H + 1, 3:W + 3])
    got = out_big.cpu().numpy()
    check_layers(torch, ao, cams, d, got[:, 1:H + 1, 3:W + 3], "pitched")
    mask = np.ones(got.shape, bool)
    mask[:, 1:H + 1, 3:W + 3] = False
    assert (got[mask] == 7).all(), "a store outside the view"
    d2 = depth_of(W, H, "f32", False, L, seed=6)
    depths = [np.ascontiguousarray(x) for x in (d, d2, d)]
    outs = [np.zeros((L, H, W), np.uint8) for _ in depths]
    ao.render_host_batch(depths, outs)
    for i, (x, o) in enumerate(zip(depths, outs)):
        for l, cam in enumerate(cams):
            ref, _ = reference(torch, cam, x[l], [])
            assert np.array_equal(o[l], ref), ("host async", i, l)


def test_uniform_tables_launch_the_context_projections_kernels(torch_cuda):
    W, H = 160, 96
    d = depth_of(W, H, "f32", True, 3, seed=2)
    for proj in (P, O):
        cams = cameras(W, H, [proj] * 3)
        ao = mixed_context(cams)
        t = to_tensor(torch_cuda, d)
        out = torch_cuda.empty((3, H, W), dtype=torch_cuda.uint8, device="cuda")
        names = [n for n, _ in ao.profile_frame(t, out)]
        got = out.cpu().numpy()
        check_layers(torch_cuda, ao, cams, d, got, f"uniform {proj}")
        ref = harness.context(cams[0], device=0, layers=3, layer_cameras=cams)
        ref.render(t)
        assert names == [n for n, _ in ref.profile_frame(t, out)]
        assert ao._lib.meao_kernels_per_frame(ao._ctx) == ref._lib.meao_kernels_per_frame(ref._ctx)
        assert np.array_equal(out.cpu().numpy(), got)
        ao.close(); ref.close()


def test_refusals_launch_nothing(torch_cuda):
    W, H = 128, 64
    cams = cameras(W, H, [P, O])
    ao = mixed_context(cams)
    d = to_tensor(torch_cuda, depth_of(W, H, "f32", True, 2))
    ao.render(d)
    lib, ctx = ao._lib, ao._ctx
    n0, g0 = lib.meao_launch_count(ctx), lib.meao_frame_generation(ctx)
    views = (N.MeaoLayerViewport * 2)(N.MeaoLayerViewport(0, 0, 0, 0, 0, 0), N.MeaoLayerViewport(0, 0, 1, 0, 0, 1))
    assert lib.meao_set_layer_viewports(ctx, views, 2) == N.MEAO_ERR_UNSUPPORTED
    assert b"orthographic layer" in lib.meao_last_error(ctx)
    with pytest.raises(Exception, match="orthographic layer"):
        ao.render_batch([d[0], d[1]])
    outs = [torch_cuda.empty((H, W), dtype=torch_cuda.uint8, device="cuda") for _ in range(2)]
    ptrs = (C.c_void_p * 2)(d[0].data_ptr(), d[1].data_ptr())
    pitches = (C.c_int64 * 2)(W * 4, W * 4)
    optrs = (C.c_void_p * 2)(outs[0].data_ptr(), outs[1].data_ptr())
    opitches = (C.c_int64 * 2)(W, W)
    assert lib.meao_render_batch(ctx, ptrs, pitches, N.MEAO_DEPTH_RAW_F32, optrs, opitches, 2, None) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_launch_count(ctx) == n0 and lib.meao_frame_generation(ctx) == g0
    assert lib.meao_get_layer_viewports(ctx, None, 0) == 0
    # with the table cleared the same batch runs
    ao.perLayerProjection = False
    ao.layerCameras = None
    ao.LateUpdate()
    assert lib.meao_render_batch(ctx, ptrs, pitches, N.MEAO_DEPTH_RAW_F32, optrs, opitches, 2, None) == 0
