"""GPU tests of device cameras (meao_bind_device_cameras) on the H100: with the cameras in a CUDA float32 tensor and host cameras that
differ from them, every layer's AO and debug buffers (ids 1-21) must equal, bit for bit, the same frame on a context whose host cameras
are the tensor's -- through pointer frames of every depth kind and Z direction, the variants, L = 1 (the layered kernels with one layer)
and L = 3, orthographic and mixed projection tables, pitched views, host frames, CUDA arrays and _at viewports, a layer-viewport table,
batches, the plugin event, MEAO_FLAG_NO_GRAPH and the stage calls.  A torch.cuda.graph captured once follows the tensor at every replay
(written by a torch op inside the graph and by copy_ outside it) without moving meao_frame_generation or instantiating a graph.  An
invalid camera is reported by the status with every other layer exact, and the refusals launch nothing."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

pytestmark = pytest.mark.gpu

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
LINEAR = {"f32": False, "linear": True, "d16": False, "d24s8": False}


def cameras(W, H, L, reversed_z=True, table=None, shift=0.0):
    """L cameras with planes and fields of view of their own (table: each layer's projection, default perspective)."""
    out = []
    for l in range(L):
        near, far = 0.2 + 0.15 * l + shift, 60.0 + 40.0 * l + 30 * shift
        if table and table[l] == O:
            out.append(Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, orthographic=True,
                              orthographicSize=3.0 + 2.5 * l + shift))
        else:
            out.append(Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, fieldOfView=50.0 + 7.0 * l + 10 * shift))
    return out


def cam_tensor(torch, cams, n=None):
    """The device camera buffer of `cams` (n rows, the extra ones a valid filler)."""
    rows = [(c.nearClipPlane, c.farClipPlane, 1.0 / c.projection00) for c in cams]
    rows += [(1.0, 2.0, 1.0)] * ((n or len(cams)) - len(cams))
    return torch.tensor(rows, dtype=torch.float32, device="cuda")


def host_context(cams, table=None, **kw):
    """A context whose host cameras are `cams` (and whose projections are `table`)."""
    L = len(cams)
    ao = harness.context(cams[0], device=0, layers=L, layer_cameras=cams if L > 1 else None, **kw)
    if table is not None and L > 1:
        ao.perLayerProjection = True
    return ao


def bound_context(torch, cams, table=None, **kw):
    """A context whose host cameras differ from `cams` (same Z direction and projections) and whose device buffer holds `cams`."""
    W, H = cams[0].pixelWidth, cams[0].pixelHeight
    other = cameras(W, H, len(cams), cams[0].usesReversedZBuffer, table, shift=0.7)
    ao = host_context(other, table, **kw)
    ao.deviceCameras = cam_tensor(torch, cams)
    return ao


def depth_of(W, H, kind, reversed_z, L, seed=0):
    if kind == "linear":
        return harness.contrasting_layers(W, H, L, seed=seed)
    return harness.ingest(harness.frames(W, H, L, seed=seed, reversed_z=reversed_z), kind)[0]


def to_tensor(torch, d):
    if d.dtype == np.uint32:
        d = d.view(np.int32)
    return torch.from_numpy(np.ascontiguousarray(d)).cuda()


def same_buffers(a, b, ids, tag):
    for bid in ids:
        x, y = a.debug_buffer(bid), b.debug_buffer(bid)
        view = {1: np.uint8, 2: np.uint16, 4: np.uint32}[x.dtype.itemsize]
        assert x.dtype == y.dtype and np.array_equal(x.view(view), y.view(view)), f"{tag}: buffer {bid}"


def check(torch, ao, ref, got, want, tag, **kw):
    assert np.array_equal(np.asarray(got), np.asarray(want)), f"{tag}: AO"
    same_buffers(ao, ref, harness.buffer_ids(kw.get("high_quality_mask", 0), kw.get("single_scale", False)), tag)


@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("reversed_z", [True, False])
@pytest.mark.parametrize("kind", list(LINEAR))
def test_pointer_frames(torch_cuda, kind, reversed_z, L):
    W, H = 161, 93
    cams = cameras(W, H, L, reversed_z)
    d = depth_of(W, H, kind, reversed_z, L, seed=3)
    d = d if L > 1 else d[0]
    ao, ref = bound_context(torch_cuda, cams), host_context(cams)
    got = ao.render(to_tensor(torch_cuda, d), linear=LINEAR[kind]).cpu().numpy()
    want = ref.render(to_tensor(torch_cuda, d), linear=LINEAR[kind]).cpu().numpy()
    check(torch_cuda, ao, ref, got, want, f"{kind} rz={reversed_z} L={L}")
    assert ao.deviceCameraStatus() == (0, 0, 0)


@pytest.mark.parametrize("params", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True),
                                    dict(high_quality_mask=5, sample_exhaustively=True, use_graph=False)])
@pytest.mark.parametrize("L", [1, 3])
def test_variants_host_frames_and_no_graph(torch_cuda, params, L):
    W, H = 333, 187
    cams = cameras(W, H, L)
    d = depth_of(W, H, "f32", True, L, seed=5)
    d = d if L > 1 else d[0]
    ao, ref = bound_context(torch_cuda, cams, **params), host_context(cams, **params)
    kw = {k: v for k, v in params.items() if k != "use_graph"}
    check(torch_cuda, ao, ref, ao.render(to_tensor(torch_cuda, d)).cpu().numpy(), ref.render(to_tensor(torch_cuda, d)).cpu().numpy(),
          f"{params} L={L}", **kw)
    check(torch_cuda, ao, ref, ao.render_host(d), ref.render_host(d), f"host {params} L={L}", **kw)


@pytest.mark.parametrize("table", [[O], [O, O], [P, O, O], [O, P, O, P, O, P]])
def test_orthographic_and_mixed_tables(torch_cuda, table):
    W, H = 128, 80
    L = len(table)
    cams = cameras(W, H, L, table=table)
    for kind in ("f32", "d16", "linear"):
        d = depth_of(W, H, kind, True, L, seed=L)
        d = d if L > 1 else d[0]
        ao, ref = bound_context(torch_cuda, cams, table=table), host_context(cams, table=table)
        got = ao.render(to_tensor(torch_cuda, d), linear=LINEAR[kind]).cpu().numpy()
        want = ref.render(to_tensor(torch_cuda, d), linear=LINEAR[kind]).cpu().numpy()
        check(torch_cuda, ao, ref, got, want, f"{table} {kind}")
        ao.close(); ref.close()


def test_arrays_pitched_viewports_batches_and_events(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 96, 64, 3
    cams = cameras(W, H, L)
    d = depth_of(W, H, "f32", True, L, seed=9)
    ao, ref = bound_context(torch, cams), host_context(cams)
    # CUDA arrays, whole and at viewports
    for a in (ao, ref):
        dep = Array(rt, W + 8, H + 4, np.float32, shape="layered", layers=L)
        big = np.full((L, H + 4, W + 8), 0.25, np.float32)
        big[:, 3:3 + H, 5:5 + W] = d
        dep.fill(big)
        aoa = Array(rt, W + 2, H + 6, np.uint8, shape="layered", layers=L)
        aoa.fill(np.full((L, H + 6, W + 2), 9, np.uint8))
        a.render_arrays(dep.handle, aoa.handle, depth_origin=(5, 3), ao_origin=(1, 2))
        torch.cuda.synchronize()
        a._arr = aoa.read()
        a.release_array(dep.handle); a.release_array(aoa.handle)
        dep.free(); aoa.free()
    check(torch, ao, ref, ao._arr, ref._arr, "arrays_at")
    # pitched views of larger tensors
    outs = []
    for a in (ao, ref):
        bigd = torch.full((L + 1, H + 3, W + 37), 0.5, dtype=torch.float32, device="cuda")
        bigd[1:, 1:H + 1, 5:W + 5] = torch.from_numpy(d).cuda()
        out_big = torch.full((L, H + 2, W + 19), 7, dtype=torch.uint8, device="cuda")
        a.render(bigd[1:, 1:H + 1, 5:W + 5], out_big[:, 1:H + 1, 3:W + 3])
        outs.append(out_big.cpu().numpy())
    check(torch, ao, ref, outs[0], outs[1], "pitched")
    # a layer-viewport table over one shared buffer
    views = [(0, 0, l, 0, 0, l) for l in range(L)]
    for a in (ao, ref):
        a.layerViewports = views
        a._out = a.render(to_tensor(torch, d)).cpu().numpy()
        a.layerViewports = None
    check(torch, ao, ref, ao._out, ref._out, "viewport table")
    # pointer and array batches
    for a in (ao, ref):
        a._out = [o.cpu().numpy() for o in a.render_batch([to_tensor(torch, d[l]) for l in range(L)])]
    check(torch, ao, ref, ao._out, ref._out, "batch")
    # the plugin event
    lib = N.lib()
    dt = to_tensor(torch, d)
    res = []
    for i, a in enumerate((ao, ref)):
        o = torch.zeros((L, H, W), dtype=torch.uint8, device="cuda")
        assert lib.meao_bind_event(a._ctx, 70 + i, C.c_void_p(dt.data_ptr()), N.MEAO_DEPTH_RAW_F32, C.c_void_p(o.data_ptr()), None) == 0
        lib.meao_get_render_event_func()(70 + i)
        torch.cuda.synchronize()
        res.append(o.cpu().numpy())
        assert lib.meao_bind_event(a._ctx, 70 + i, None, 0, None, None) == 0
    check(torch, ao, ref, res[0], res[1], "event")


@pytest.mark.parametrize("L", [1, 3])
def test_stage_calls(torch_cuda, L):
    """meao_stage_downsample derives the tables; the later stage calls read them."""
    W, H = 128, 72
    cams = cameras(W, H, L)
    d = depth_of(W, H, "f32", True, L, seed=11)
    d = d if L > 1 else d[0]
    ao, ref = bound_context(torch_cuda, cams), host_context(cams)
    lib = N.lib()
    n0 = lib.meao_launch_count(ao._ctx)
    for a in (ao, ref):
        a.stage_downsample(to_tensor(torch_cuda, d))
        for k in (1, 2, 3, 4):
            a.stage_render(k)
        for lo in (4, 3, 2, 1):
            a.stage_upsample(lo)
    torch_cuda.cuda.synchronize()
    assert lib.meao_launch_count(ao._ctx) - n0 == 10          # the camera stage, the prepare, four renders, four upsamples
    same_buffers(ao, ref, harness.buffer_ids(), f"stages L={L}")


def test_torch_graph_follows_the_camera_tensor(torch_cuda):
    """One capture; every replay equals a fresh host-camera frame of the cameras the tensor then holds, whether a torch op inside the
    graph or a copy_ outside it wrote them.  Neither the generation nor the instantiation count moves."""
    torch = torch_cuda
    W, H, L = 192, 108, 2
    cams = cameras(W, H, L)
    d = depth_of(W, H, "d24s8", True, L, seed=4)
    depth = to_tensor(torch, d)
    ao = bound_context(torch, cams, high_quality_mask=2)
    cam_t = ao.deviceCameras
    base = cam_t.clone()
    scale = torch.ones((L, 3), dtype=torch.float32, device="cuda")
    out = torch.empty((L, H, W), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ao.render(depth, out, stream=s)         # one settling frame: binds the tensor and plans
    s.synchronize()
    lib = N.lib()
    gen, inst = lib.meao_frame_generation(ao._ctx), ao.reservation()["graph_instantiations"]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        torch.mul(base, scale, out=cam_t)       # the cameras written by a torch op inside the graph
        ao.render(depth, out, stream=s)

    def expect(rows, tag):
        """The replay against a fresh context whose HOST cameras are the float32 rows, and against a fresh bound context."""
        host = harness.context(cams[0], device=0, layers=L, high_quality_mask=2)
        host.LateUpdate()
        mc = (N.MeaoCamera * L)(*[N.MeaoCamera(*r, 1) for r in rows])
        assert lib.meao_set_layer_cameras(host._ctx, mc, L) == 1
        host_out = torch.empty((L, H, W), dtype=torch.uint8, device="cuda")
        assert lib.meao_render(host._ctx, C.c_void_p(depth.data_ptr()), N.MEAO_DEPTH_RAW_D24S8, C.c_void_p(host_out.data_ptr()), None) == 0
        ref = host_context(cams, high_quality_mask=2)
        ref.deviceCameras = torch.tensor(rows, dtype=torch.float32, device="cuda")
        ref_out = ref.render(depth).cpu().numpy()
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), host_out.cpu().numpy()), f"{tag}: replay against the host cameras"
        assert np.array_equal(out.cpu().numpy(), ref_out), f"{tag}: replay against a fresh bound context"
        host.close(); ref.close()

    for step, factors in enumerate(([1.0, 1.0, 1.0], [1.3, 1.7, 0.8], [0.6, 3.0, 1.9])):
        scale.copy_(torch.tensor([factors] * L, dtype=torch.float32))
        g.replay()
        torch.cuda.synchronize()
        expect((base * scale).cpu().numpy().tolist(), f"op step {step}")
    # copy_ outside the graph: the op inside it writes base * scale, so the new cameras go into base
    base.copy_(cam_tensor(torch, cameras(W, H, L, shift=1.3)))
    scale.fill_(1.0)
    g.replay()
    torch.cuda.synchronize()
    expect(base.cpu().numpy().tolist(), "copy_")
    assert lib.meao_frame_generation(ao._ctx) == gen
    assert ao.reservation()["graph_instantiations"] == inst


def test_context_graph_follows_the_buffer_without_instantiation(torch_cuda):
    """The context's own graph replays with the new cameras: no generation, no instantiation, each change at the next frame."""
    torch = torch_cuda
    W, H, L = 160, 96, 3
    d = depth_of(W, H, "f32", True, L, seed=8)
    t = to_tensor(torch, d)
    ao = bound_context(torch, cameras(W, H, L))
    ao.render(t)
    lib = N.lib()
    gen, inst = lib.meao_frame_generation(ao._ctx), ao.reservation()["graph_instantiations"]
    for shift in (0.3, 1.1, 2.9):
        cams = cameras(W, H, L, shift=shift)
        ao.deviceCameras.copy_(cam_tensor(torch, cams))
        got = ao.render(t).cpu().numpy()
        ref = host_context(cams)
        assert np.array_equal(got, ref.render(t).cpu().numpy()), shift
        ref.close()
    assert lib.meao_frame_generation(ao._ctx) == gen
    assert ao.reservation()["graph_instantiations"] == inst


@pytest.mark.parametrize("bad,field", [((0.0, 50.0, 1.0), 1), ((2.0, 2.0, 1.0), 2), ((0.5, 50.0, float("nan")), 3),
                                       ((float("nan"), 50.0, 1.0), 1), ((0.5, 50.0, -1.0), 3)])
def test_invalid_camera_is_reported_and_other_layers_stay_exact(torch_cuda, bad, field):
    torch = torch_cuda
    W, H, L = 128, 64, 4
    cams = cameras(W, H, L)
    d = depth_of(W, H, "f32", True, L, seed=1)
    t = to_tensor(torch, d)
    ao = bound_context(torch, cams)
    ao.render(t)
    assert ao.deviceCameraStatus() == (0, 0, 0)
    ao.deviceCameras[2] = torch.tensor(bad, dtype=torch.float32)
    got = ao.render(t).cpu().numpy()
    ref = host_context(cams)
    want = ref.render(t).cpu().numpy()
    for l in (0, 1, 3):
        assert np.array_equal(got[l], want[l]), l
    assert ao.deviceCameraStatus() == (1, 2, field)
    ao.deviceCameras[0] = torch.tensor(bad, dtype=torch.float32)
    ao.render(t)
    assert ao.deviceCameraStatus() == (2, 0, field)
    ao.deviceCameras.copy_(cam_tensor(torch, cams))
    got = ao.render(t).cpu().numpy()
    assert np.array_equal(got, want)
    assert ao.deviceCameraStatus() == (2, 0, field)             # counts since the bind


def test_profile_names_the_camera_stage(torch_cuda):
    W, H = 128, 64
    cams = cameras(W, H, 2)
    ao = bound_context(torch_cuda, cams)
    t = to_tensor(torch_cuda, depth_of(W, H, "f32", True, 2))
    out = torch_cuda.empty((2, H, W), dtype=torch_cuda.uint8, device="cuda")
    names = [n for n, _ in ao.profile_frame(t, out)]
    assert names[0] == "camera_tables" and names[1] == "prepare_depth"
    assert len(names) == N.lib().meao_kernels_per_frame(ao._ctx)


def test_refusals_launch_nothing(torch_cuda):
    torch = torch_cuda
    W, H = 128, 64
    lib = N.lib()
    cams = cameras(W, H, 4)
    ao = bound_context(torch, cams[:2])
    ao.maxLayers = 4
    d = to_tensor(torch, depth_of(W, H, "f32", True, 4))
    ao.render(d[:2])
    ctx = ao._ctx
    n0 = lib.meao_launch_count(ctx)
    # a frame with more layers than the buffer holds
    assert lib.meao_set_layers(ctx, 4) == 1
    out = torch.empty((4, H, W), dtype=torch.uint8, device="cuda")
    assert lib.meao_render(ctx, C.c_void_p(d.data_ptr()), N.MEAO_DEPTH_RAW_F32, C.c_void_p(out.data_ptr()), None) == N.MEAO_ERR_INVALID
    assert b"holds 2 cameras" in lib.meao_last_error(ctx)
    host = np.zeros((4, H, W), np.float32)
    hout = np.zeros((4, H, W), np.uint8)
    assert lib.meao_render_host(ctx, host.ctypes.data, N.MEAO_DEPTH_RAW_F32, hout.ctypes.data) == N.MEAO_ERR_INVALID
    assert lib.meao_stage_downsample(ctx, C.c_void_p(d.data_ptr()), N.MEAO_DEPTH_RAW_F32, None) == N.MEAO_ERR_INVALID
    assert lib.meao_set_layers(ctx, 2) == 1
    g0 = lib.meao_frame_generation(ctx)
    # the TiledDepth debug views
    view = torch.empty((2, H, W), dtype=torch.uint8, device="cuda")
    for bid in (6, 7, 8, 9):
        assert lib.meao_debug_view(ctx, bid, C.c_void_p(view.data_ptr()), None) == N.MEAO_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert lib.meao_launch_count(ctx) == n0
    assert lib.meao_frame_generation(ctx) == g0
    # a single-layer context with a row band refuses the binding, and a bound one refuses the band
    one = harness.context(W, H, device=0)
    one.render(d[0])
    assert one._lib.meao_set_row_band(one._ctx, 0, 32, -1, H) == 0
    assert lib.meao_bind_device_cameras(one._ctx, C.c_void_p(ao.deviceCameras.data_ptr()), 1) == N.MEAO_ERR_UNSUPPORTED
    one.close()
    one = harness.context(W, H, device=0)
    one.render(d[0])
    assert lib.meao_bind_device_cameras(one._ctx, C.c_void_p(ao.deviceCameras.data_ptr()), 1) == 1
    assert lib.meao_set_row_band(one._ctx, 0, 32, -1, H) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_bind_device_cameras(one._ctx, None, 0) == 1
    one.close()
    # host memory is refused
    hcams = np.ones((2, 3), np.float32)
    assert lib.meao_bind_device_cameras(ctx, C.c_void_p(hcams.ctypes.data), 2) == N.MEAO_ERR_INVALID


HOSTILE = [("far_near_1p2m20", 1.0, 1.0 + 2.0 ** -20, None), ("far_near_1e7", 0.01, 1e5, None), ("far_near_overflows", 1e-30, 1e30, None),
           ("tan_half_fov_1em6", 0.3, 100.0, 1e-6), ("tan_half_fov_1e6", 0.3, 100.0, 1e6), ("subnormal_tm", 0.3, 100.0, 3e-38),
           ("ortho_it_inf", 1e-3, 3e38, 1e-6)]


@pytest.mark.parametrize("stereo", [False, True])
@pytest.mark.parametrize("rz", [True, False])
@pytest.mark.parametrize("name,near,far,tan", HOSTILE, ids=[h[0] for h in HOSTILE])
def test_hostile_cameras_and_stereo(torch_cuda, name, near, far, tan, rz, stereo):
    """The extreme cameras of tests/hostile_cases.py and ones whose products go subnormal or overflow, perspective and orthographic
    layers, both Z directions, with and without single-pass stereo (the ThicknessMultiplier doubling): the derived tables make the same
    frame as the host planner's, on the AO and every buffer (NaN where the host's is NaN)."""
    import math
    W, H = 96, 64
    table = [P, O, P]
    cams = []
    for p in table:
        t = 1.0 if tan is None else tan
        if p == O:
            cams.append(Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True,
                               orthographicSize=t * H / W, stereoEnabled=stereo))
        else:
            cams.append(Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, stereoEnabled=stereo,
                               fieldOfView=math.degrees(2.0 * math.atan(t * H / W))))
    d = depth_of(2 * W if stereo else W, H, "f32", rz, 3, seed=6)
    ao, ref = bound_context(torch_cuda, cams, table=table), host_context(cams, table=table)
    if stereo:
        ao.camera.stereoEnabled = True          # the bound context's own host camera is another one: single-pass stereo as well
        ao.OnPreRender(); ref.OnPreRender()
    got = ao.render(to_tensor(torch_cuda, d)).cpu().numpy()
    want = ref.render(to_tensor(torch_cuda, d)).cpu().numpy()
    assert np.array_equal(got, want), f"{name}: AO"
    for bid in harness.buffer_ids():
        x, y = ao.debug_buffer(bid), ref.debug_buffer(bid)
        if x.dtype == np.uint8:
            assert np.array_equal(x, y), f"{name}: buffer {bid}"
        else:
            assert np.array_equal(x, y, equal_nan=True), f"{name}: buffer {bid}"
