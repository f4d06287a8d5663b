"""GPU tests of orthographic cameras (meao_set_projection) on the H100: every buffer of an orthographic frame must be bit-identical to
the orthographic oracle (tests/ortho_oracle.py) through each frame form -- pointer frames of every depth kind and Z direction, pitched
views, host frames, CUDA arrays, layered frames with per-layer cameras, every variant, a reserved context across sizes and a frame
recorded into torch.cuda.graph -- an orthographic zoom must take effect at the next frame without a graph instantiation, and the
refused combinations must launch nothing."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N
from ortho_oracle import OrthoOracle

pytestmark = pytest.mark.gpu

KINDS = {"f32": False, "linear": True, "d16": False, "d24s8": False}


def ortho_camera(W, H, reversed_z=True, near=0.5, far=80.0, size=6.0):
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, orthographic=True, orthographicSize=size)


def ortho_context(cam, **kw):
    return harness.context(cam, device=0, **kw)


def ortho_oracle(cam, linear=False, **kw):
    return OrthoOracle(cam.pixelWidth, cam.pixelHeight, near=cam.nearClipPlane, far=cam.farClipPlane,
                       tan_half_fov_h_=1.0 / cam.projection00, reversed_z=cam.usesReversedZBuffer, linear=linear, threads=8, **kw)


def depth_of(W, H, kind, reversed_z, seed=0, L=1):
    """(the depth in the ingest format of `kind`, the float32 the oracle sees), [L, H, W] or [H, W]."""
    if kind == "linear":
        lin = harness.contrasting_layers(W, H, max(L, 1), seed=seed)
        d = lin if L > 1 else lin[0]
        return d, d
    r = harness.frames(W, H, L, seed=seed, reversed_z=reversed_z)
    r = r if L > 1 else r[0]
    return harness.ingest(r, kind)


def variant_kw(params):
    return {k: params[k] for k in ("sample_exhaustively", "high_quality_mask", "single_scale") if k in params}


def check_frame(ao, cam, fdepth, tag, linear=False, layer_cams=None, **params):
    ids = harness.buffer_ids(params.get("high_quality_mask", 0), params.get("single_scale", False))
    got = {bid: ao.debug_buffer(bid) for bid in ids}
    cams = layer_cams or [cam]
    for l, c in enumerate(cams):
        orc = ortho_oracle(c, linear=linear, single_pass_stereo=False, **variant_kw(params))
        orc.run(fdepth[l] if len(cams) > 1 else fdepth)
        harness.compare_buffers((lambda bid: got[bid][l]) if len(cams) > 1 else (lambda bid: got[bid]), orc, f"{tag} layer {l}", ids)
    return cams


@pytest.mark.parametrize("reversed_z", [True, False])
@pytest.mark.parametrize("kind", list(KINDS))
def test_pointer_frames_every_kind(torch_cuda, kind, reversed_z):
    W, H = 161, 93
    cam = ortho_camera(W, H, reversed_z)
    d, fd = depth_of(W, H, kind, reversed_z, seed=3)
    ao = ortho_context(cam)
    out = ao.render(torch_cuda.from_numpy(np.ascontiguousarray(d)).cuda(), linear=KINDS[kind]).cpu().numpy()
    assert ao._lib.meao_get_projection(ao._ctx) == N.MEAO_PROJECTION_ORTHOGRAPHIC
    check_frame(ao, cam, fd, f"{kind} rz={reversed_z}", linear=KINDS[kind])
    orc = ortho_oracle(cam, linear=KINDS[kind])
    assert (out == orc.run(fd)).all()
    # the debug views of every buffer (the AO regeneration of id 17 included)
    for bid in (1, 6, 10, 14, 17):
        assert (ao.debug_view(bid).cpu().numpy() == orc.debug_view(bid)).all(), bid


@pytest.mark.parametrize("params", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True),
                                    dict(reversed_z=False, high_quality_mask=5, sample_exhaustively=True)])
def test_variants(torch_cuda, params):
    W, H = 333, 187
    rz = params.pop("reversed_z", True)
    cam = ortho_camera(W, H, rz, near=0.1, far=500.0, size=40.0)
    d, fd = depth_of(W, H, "f32", rz, seed=5)
    ao = ortho_context(cam, **params)
    ao.render(torch_cuda.from_numpy(d).cuda())
    check_frame(ao, cam, fd, f"variant {params}", **params)
    ao.render_host(d)                       # the host path, the same frame
    check_frame(ao, cam, fd, f"host variant {params}", **params)


def test_1080p_and_graph_replay_equals_direct_launches(torch_cuda):
    W, H = 1920, 1080
    cam = ortho_camera(W, H, size=12.5)
    d, fd = depth_of(W, H, "f32", True, seed=7)
    ref = ortho_oracle(cam).run(fd)
    for use_graph in (True, False):
        ao = harness.context(cam, device=0, use_graph=use_graph)
        for _ in range(2):
            out = ao.render(torch_cuda.from_numpy(d).cuda()).cpu().numpy()
            assert (out == ref).all(), f"use_graph={use_graph}"
        ao.close()


@pytest.mark.parametrize("kind", ["f32", "linear", "d16"])
def test_layered_with_layer_cameras(torch_cuda, kind):
    W, H, L = 200, 120, 3
    cams = [ortho_camera(W, H, near=n, far=f, size=s) for n, f, s in ((0.5, 80.0, 6.0), (1.0, 300.0, 25.0), (0.1, 20.0, 2.0))]
    d, fd = depth_of(W, H, kind, True, seed=11, L=L)
    ao = harness.context(cams[0], device=0, layers=L, layer_cameras=cams)
    ao.render(torch_cuda.from_numpy(np.ascontiguousarray(d)).cuda(), linear=KINDS[kind])
    check_frame(ao, cams[0], fd, f"layered {kind}", linear=KINDS[kind], layer_cams=cams)
    # without a table every layer takes the main camera
    ao.layerCameras = None
    ao.render(torch_cuda.from_numpy(np.ascontiguousarray(d)).cuda(), linear=KINDS[kind])
    check_frame(ao, cams[0], fd, f"layered {kind} one camera", linear=KINDS[kind], layer_cams=[cams[0]] * L)


def test_pitched_views(torch_cuda):
    W, H = 130, 70
    cam = ortho_camera(W, H, reversed_z=False)
    d, fd = depth_of(W, H, "f32", False, seed=2)
    big = torch_cuda.full((H + 3, W + 37), 0.5, dtype=torch_cuda.float32, device="cuda")
    big[1:H + 1, 5:W + 5] = torch_cuda.from_numpy(d).cuda()
    out_big = torch_cuda.full((H + 2, W + 19), 7, dtype=torch_cuda.uint8, device="cuda")
    ao = ortho_context(cam)
    ao.render(big[1:H + 1, 5:W + 5], out_big[1:H + 1, 3:W + 3])
    got = out_big.cpu().numpy()
    assert (got[1:H + 1, 3:W + 3] == ortho_oracle(cam).run(fd)).all()
    assert (got[0] == 7).all() and (got[:, :3] == 7).all() and (got[:, W + 3:] == 7).all()
    check_frame(ao, cam, fd, "pitched")


@pytest.mark.parametrize("shape,L", [("2d", 1), ("layered", 2), ("cube", 6)])
def test_cuda_arrays(torch_cuda, rt, shape, L):
    W, H = (61, 61) if shape == "cube" else (83, 61)
    cam = ortho_camera(W, H)
    for kind, dtype, ikind in (("raw_f32", np.float32, "f32"), ("d16", np.uint16, "d16"), ("linear_f32", np.float32, "linear")):
        d, fd = depth_of(W, H, ikind, True, seed=L, L=L)
        dep = Array(rt, W, H, dtype, shape=shape, layers=L)
        aoa = Array(rt, W, H, np.uint8, shape=shape, layers=L)
        dep.fill(np.ascontiguousarray(d).astype(dtype))
        ao = harness.context(cam, device=0, layers=L)
        ao.render_arrays(dep.handle, aoa.handle, kind=kind)
        torch_cuda.cuda.synchronize()
        got = aoa.read().reshape(L, H, W)
        fdl = fd if L > 1 else fd[None]
        bufs = {bid: ao.debug_buffer(bid) for bid in range(1, 17)}
        for l in range(L):
            orc = ortho_oracle(cam, linear=ikind == "linear")
            assert (got[l] == orc.run(fdl[l])).all(), f"{shape} {kind} layer {l}"
            harness.compare_buffers(lambda bid: bufs[bid][l] if L > 1 else bufs[bid], orc, f"{shape} {kind} layer {l}", range(1, 17))
        ao.close()
        dep.free(); aoa.free()


def test_arrays_at_viewport(torch_cuda, rt):
    W, H = 64, 40
    cam = ortho_camera(W, H)
    d, fd = depth_of(W, H, "f32", True, seed=9)
    big = np.full((H + 10, W + 20), 0.25, np.float32)
    big[4:4 + H, 7:7 + W] = d
    dep = Array(rt, W + 20, H + 10, np.float32)
    aoa = Array(rt, W + 30, H + 6, np.uint8)
    dep.fill(big)
    aoa.fill(np.full((H + 6, W + 30), 9, np.uint8))
    ao = ortho_context(cam)
    ao.render_arrays(dep.handle, aoa.handle, depth_origin=(7, 4), ao_origin=(11, 2))
    torch_cuda.cuda.synchronize()
    got = aoa.read().reshape(H + 6, W + 30)
    orc = ortho_oracle(cam)
    assert (got[2:2 + H, 11:11 + W] == orc.run(fd)).all()
    harness.compare_buffers(ao.debug_buffer, orc, "arrays_at", range(1, 17))
    dep.free(); aoa.free()


def test_reserved_sizes_and_live_zoom(torch_cuda):
    cam = ortho_camera(640, 360)
    ao = harness.context(cam, device=0, max_resolution=(640, 360))
    sizes = [(640, 360), (401, 233), (640, 360), (97, 61)]
    inst = None
    for i, (W, H) in enumerate(sizes):
        cam.pixelWidth, cam.pixelHeight = W, H
        cam.orthographicSize = 3.0 + i           # a zoom every frame: a frame constant
        d, fd = depth_of(W, H, "f32", True, seed=i)
        out = ao.render(torch_cuda.from_numpy(d).cuda()).cpu().numpy()
        assert (out == ortho_oracle(cam).run(fd)).all(), (W, H)
        if i == 2:
            inst = ao.reservation()["graph_instantiations"]
    # back at a planned size, zooming frame after frame: no graph instantiation, each zoom in the very next frame
    cam.pixelWidth, cam.pixelHeight = 640, 360
    d, fd = depth_of(640, 360, "f32", True, seed=0)
    ao.render(torch_cuda.from_numpy(d).cuda())
    before = ao.reservation()["graph_instantiations"]
    for z in (2.0, 2.5, 40.0):
        cam.orthographicSize = z
        out = ao.render(torch_cuda.from_numpy(d).cuda()).cpu().numpy()
        assert (out == ortho_oracle(cam).run(fd)).all(), z
    after = ao.reservation()["graph_instantiations"]
    assert after == before and inst is not None


def test_torch_graph_capture(torch_cuda):
    torch = torch_cuda
    W, H = 256, 144
    cam = ortho_camera(W, H)
    d, fd = depth_of(W, H, "d24s8", True, seed=4)
    ao = ortho_context(cam)
    depth = torch.from_numpy(d.view(np.int32)).cuda()
    out = torch.empty((H, W), dtype=torch.uint8, device="cuda")
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
    assert (out.cpu().numpy() == ortho_oracle(cam).run(fd)).all()


def test_stage_api_and_profile(torch_cuda):
    W, H = 150, 90
    cam = ortho_camera(W, H)
    d, fd = depth_of(W, H, "f32", True, seed=8)
    ao = ortho_context(cam, high_quality_mask=2)
    lib, ctx = ao._lib, ao._ctx
    ao.LateUpdate()
    t = torch_cuda.from_numpy(d).cuda()
    out = torch_cuda.empty((H, W), dtype=torch_cuda.uint8, device="cuda")
    assert lib.meao_stage_downsample(ctx, t.data_ptr(), N.MEAO_DEPTH_RAW_F32, None) == 0
    for k in range(1, 5):
        assert lib.meao_stage_render(ctx, k, None) == 0
    assert lib.meao_stage_render_wide(ctx, 2, None) == 0
    for lo in range(4, 0, -1):
        assert lib.meao_stage_upsample(ctx, lo, out.data_ptr() if lo == 1 else None, None) == 0
    torch_cuda.cuda.synchronize()
    orc = ortho_oracle(cam, high_quality_mask=2)
    assert (out.cpu().numpy() == orc.run(fd)).all()
    harness.compare_buffers(ao.debug_buffer, orc, "stage", harness.buffer_ids(2))
    names = [n for n, _ in ao.profile_frame(t, out)]
    assert sum(n.startswith("render_ao") for n in names) == 5, names
    assert (out.cpu().numpy() == orc.codes(17)).all()
    harness.compare_buffers(ao.debug_buffer, orc, "profile", harness.buffer_ids(2))


def test_refusals_launch_nothing(torch_cuda):
    W, H = 128, 64
    cam = ortho_camera(W, H)
    ao = harness.context(cam, device=0, layers=2)
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    n0 = lib.meao_launch_count(ctx)
    views = (N.MeaoLayerViewport * 2)(N.MeaoLayerViewport(0, 0, 0, 0, 0, 0), N.MeaoLayerViewport(0, 0, 1, 0, 0, 1))
    assert lib.meao_set_layer_viewports(ctx, views, 2) == N.MEAO_ERR_UNSUPPORTED
    assert b"orthographic" in lib.meao_last_error(ctx)
    assert lib.meao_get_layer_viewports(ctx, None, 0) == 0
    assert lib.meao_set_projection(ctx, N.MEAO_PROJECTION_PERSPECTIVE) == 1
    assert lib.meao_set_layer_viewports(ctx, views, 2) == 1
    assert lib.meao_set_projection(ctx, N.MEAO_PROJECTION_ORTHOGRAPHIC) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_get_projection(ctx) == N.MEAO_PROJECTION_PERSPECTIVE
    assert lib.meao_launch_count(ctx) == n0


def test_single_pass_stereo_and_plugin_event(torch_cuda):
    """A single-pass stereo pair (the double-wide frame, ThicknessMultiplier x 2) and the plugin event (meao_bind_event) under the
    projection: every buffer against the oracle."""
    W, H = 2 * 96, 80
    cam = Camera(W // 2, H, nearClipPlane=0.5, farClipPlane=80.0, orthographic=True, orthographicSize=6.0, stereoEnabled=True)
    ao = harness.context(cam, device=0, high_quality_mask=3)
    ao.OnPreRender()
    d, fd = depth_of(W, H, "f32", True, seed=12)
    t = torch_cuda.from_numpy(d).cuda()
    out = ao.render(t).cpu().numpy()
    orc = OrthoOracle(W, H, near=0.5, far=80.0, tan_half_fov_h_=1.0 / cam.projection00, reversed_z=True, threads=8, single_pass_stereo=True,
                      high_quality_mask=3)
    assert (out == orc.run(fd)).all()
    harness.compare_buffers(ao.debug_buffer, orc, "stereo", harness.buffer_ids(3))
    lib = N.lib()
    o = torch_cuda.zeros((H, W), dtype=torch_cuda.uint8, device="cuda")
    assert lib.meao_bind_event(ao._ctx, 93, C.c_void_p(t.data_ptr()), 0, C.c_void_p(o.data_ptr()), None) == 0
    lib.meao_get_render_event_func()(93)
    torch_cuda.cuda.synchronize()
    assert (o.cpu().numpy() == orc.codes(17)).all()
    harness.compare_buffers(ao.debug_buffer, orc, "event", harness.buffer_ids(3))
    assert lib.meao_bind_event(ao._ctx, 93, None, 0, None, None) == 0


def test_golden_fixture(torch_cuda):
    """tests/golden/ortho/*.npz (make_golden_ortho.py): the CUDA path reproduces the committed AO and intermediates bit for bit."""
    import glob
    import os
    paths = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ortho", "*.npz")))
    assert paths
    for path in paths:
        g = np.load(path)
        H, W = g["depth"].shape
        near, far, size, rz = (float(v) for v in g["camera"])
        cam = Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=bool(rz), orthographic=True, orthographicSize=size)
        ao = ortho_context(cam, intensity=float(g["params"][4]))
        got = ao.render(torch_cuda.from_numpy(g["depth"]).cuda()).cpu().numpy()
        assert np.array_equal(got, g["ao"]), path
        for key in g.files:
            if key.startswith("buf"):
                buf, ref = ao.debug_buffer(int(key[3:])), g[key]
                view = {1: np.uint8, 2: np.uint16, 4: np.uint32}[ref.dtype.itemsize]
                assert buf.dtype == ref.dtype and np.array_equal(buf.view(view), ref.view(view)), (path, key)
