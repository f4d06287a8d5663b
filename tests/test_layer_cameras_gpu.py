"""GPU tests of per-layer cameras (meao_set_layer_cameras) on the H100: layer l of a layered frame with per-layer cameras must be
bit-identical to a single-layer context with camera l, and to the oracle run on that layer with camera l, through every public path
(graph replay, direct launches, host buffers, events, pitched views, CUDA arrays, debug buffers and views)."""
import ctypes as C

import numpy as np
import pytest

from test_arrays_gpu import Array, rt, torch_cuda  # noqa: F401  (fixtures)
from test_layers_gpu import _frames

pytestmark = pytest.mark.gpu

CAMS = [(0.1, 50.0, 40.0), (0.3, 100.0, 60.0), (1.0, 1000.0, 90.0), (0.2, 300.0, 75.0)]


def cameras(W, H, n, reversed_z=True, shift=0):
    from miniengineao_b200 import Camera
    return [Camera(W, H, nearClipPlane=CAMS[(i + shift) % 4][0], farClipPlane=CAMS[(i + shift) % 4][1],
                   fieldOfView=CAMS[(i + shift) % 4][2], usesReversedZBuffer=reversed_z) for i in range(n)]


def _setup(ao, **params):
    ao.sampleExhaustively = bool(params.get("sample_exhaustively", False))
    ao.highQualityMask = int(params.get("high_quality_mask", 0))
    ao.singleScale = bool(params.get("single_scale", False))
    return ao


def _layered(W, H, cams, use_graph=True, **params):
    from miniengineao_b200 import AmbientOcclusion, Camera
    ao = _setup(AmbientOcclusion(Camera(W, H, usesReversedZBuffer=params.get("reversed_z", True)), device=0, use_graph=use_graph), **params)
    ao.layers = len(cams)
    ao.layerCameras = cams
    return ao


def _single(cam, **params):
    from miniengineao_b200 import AmbientOcclusion
    return _setup(AmbientOcclusion(cam, device=0), **params)


def _oracle(W, H, cam, linear=False, **params):
    from oracle.oracle import Oracle
    okw = {k: params[k] for k in ("sample_exhaustively", "high_quality_mask", "single_scale") if k in params}
    return Oracle(W, H, threads=8, near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00,
                  reversed_z=cam.usesReversedZBuffer, depth_is_linear=linear, **okw)


def _singles(torch, cams, depth, linear=False, **params):
    out = []
    for l, cam in enumerate(cams):
        s = _single(cam, **params)
        out.append(s.render(torch.from_numpy(np.ascontiguousarray(depth[l])).cuda(), linear=linear).cpu().numpy())
        s.close()
    return out


def _check(got, refs, tag):
    for l, ref in enumerate(refs):
        n = int((got[l] != ref).sum())
        assert n == 0, f"{tag}: layer {l} differs in {n} pixels"


def _ids(params):
    mask = params.get("high_quality_mask", 0)
    return [1, 2, 3, 4, 5, 10, 17] if params.get("single_scale") else list(range(1, 18)) + [17 + k for k in range(1, 5) if (mask >> (k - 1)) & 1]


def _compare_buffers(ao, W, H, cams, depth, tag, linear=False, oracle_depth=None, **params):
    ids = _ids(params)
    got = {bid: ao.debug_buffer(bid) for bid in ids}
    for l, cam in enumerate(cams):
        orc = _oracle(W, H, cam, linear=linear, **params)
        orc.run(depth[l] if oracle_depth is None else oracle_depth[l])
        bad = []
        for bid in ids:
            g = got[bid][l]
            if g.dtype == np.uint8:
                n = int((g != orc.codes(bid)).sum())
            elif g.dtype == np.float16:
                with np.errstate(over="ignore"):
                    n = int((g.view(np.uint16) != orc.buffer(bid).astype(np.float16).view(np.uint16)).sum())
            else:
                n = int((g.view(np.uint32) != orc.buffer(bid).view(np.uint32)).sum())
            if n:
                bad.append((bid, n))
        assert not bad, f"{tag} layer {l}: (id, #diff) {bad}"


@pytest.mark.parametrize("L", [2, 6, 8])
def test_1080p_distinct_frames_and_cameras(torch_cuda, L):
    W, H = 1920, 1080
    cams = cameras(W, H, L)
    depth = _frames(W, H, L, seed=L)
    ao = _layered(W, H, cams)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    singles = _singles(torch_cuda, cams, depth)
    _check(got, singles, f"1080p L={L} vs single-layer contexts")
    if L == 2:
        _check(got, [_oracle(W, H, c).run(depth[l]) for l, c in enumerate(cams)], "1080p L=2 vs oracle")


def test_4k_two_layers(torch_cuda):
    W, H = 3840, 2160
    cams = cameras(W, H, 2, shift=2)
    depth = _frames(W, H, 2, seed=3)
    ao = _layered(W, H, cams)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    _check(got, _singles(torch_cuda, cams, depth), "4K vs single-layer contexts")
    _check(got, [_oracle(W, H, c).run(depth[l]) for l, c in enumerate(cams)], "4K vs oracle")


@pytest.mark.parametrize("params", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True),
                                    dict(reversed_z=False, high_quality_mask=3)])
def test_ragged_all_buffers_and_variants(torch_cuda, params):
    W, H = 333, 187
    rz = params.get("reversed_z", True)
    cams = cameras(W, H, 4, reversed_z=rz)
    depth = _frames(W, H, 4, seed=5, reversed_z=rz)
    ao = _layered(W, H, cams, **params)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    _check(got, _singles(torch_cuda, cams, depth, **params), f"ragged {params}")
    _compare_buffers(ao, W, H, cams, depth, f"ragged {params}", **params)
    # meao_debug_view of every TiledDepth (each layer with its own padding value) and of the AO after the frame
    for bid in (6, 7, 8, 9, 17):
        v = ao.debug_view(bid).cpu().numpy()
        for l, cam in enumerate(cams):
            s = _single(cam, **params)
            s.render(torch_cuda.from_numpy(np.ascontiguousarray(depth[l])).cuda())
            assert np.array_equal(v[l], s.debug_view(bid).cpu().numpy()), (bid, l)
            s.close()


@pytest.mark.parametrize("kind", ["linear", "d16", "d24s8"])
def test_depth_kinds(torch_cuda, kind):
    from miniengineao_b200 import synth
    W, H, L = 640, 360, 3
    cams = cameras(W, H, L)
    raw = _frames(W, H, L, seed=7).astype(np.float64)
    if kind == "linear":
        depth = np.stack([synth.random_depth(W, H, seed=i) for i in range(L)]).astype(np.float32)
        odepth = depth
    else:
        bits = 16 if kind == "d16" else 24
        full = (1 << bits) - 1
        codes = np.clip(np.rint(raw * full), 0, full).astype(np.uint32)
        odepth = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
        depth = codes.astype(np.uint16) if bits == 16 else (codes | (np.uint32(0x5A) << np.uint32(24))).view(np.int32)
    lin = kind == "linear"
    ao = _layered(W, H, cams)
    got = ao.render(torch_cuda.from_numpy(depth).cuda(), linear=lin).cpu().numpy()
    _check(got, _singles(torch_cuda, cams, depth, linear=lin), kind)
    _compare_buffers(ao, W, H, cams, depth, kind, linear=lin, oracle_depth=odepth)


def test_pitched_views(torch_cuda):
    W, H, L = 1366, 768, 2
    cams = cameras(W, H, L, shift=1)
    depth = _frames(W, H, L, seed=9)
    big = torch_cuda.full((L, H + 8, 1408), float("nan"), device="cuda")
    big[:, :H, :W] = torch_cuda.from_numpy(depth).cuda()
    out = torch_cuda.full((L, H + 4, 1536), 0xA7, dtype=torch_cuda.uint8, device="cuda")
    ao = _layered(W, H, cams)
    ao.render(big[:, :H, :W], out[:, :H, :W])
    got = out[:, :H, :W].cpu().numpy()
    assert int((out[:, :H, W:] != 0xA7).sum()) == 0
    _check(got, _singles(torch_cuda, cams, depth), "pitched")


@pytest.mark.parametrize("shape,L", [("layered", 3), ("cube", 6)])
def test_cuda_arrays(torch_cuda, rt, shape, L):  # noqa: F811
    W, H = (192, 192) if shape == "cube" else (400, 224)
    cams = cameras(W, H, L)
    depth = _frames(W, H, L, seed=11)
    da, aa = Array(rt, W, H, np.float32, shape, L), Array(rt, W, H, np.uint8, shape, L)
    try:
        da.fill(depth)
        ao = _layered(W, H, cams)
        ao.render_arrays(da.handle, aa.handle)
        torch_cuda.cuda.synchronize()
        got = aa.read()
        _check(got, _singles(torch_cuda, cams, depth), f"arrays {shape}")
        _compare_buffers(ao, W, H, cams, depth, f"arrays {shape}")
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        ao.close()
    finally:
        da.free()
        aa.free()


def test_replay_camera_changes_clear_and_identical_tables(torch_cuda):
    from miniengineao_b200 import AmbientOcclusion, Camera
    W, H, L = 960, 540, 3
    cams = cameras(W, H, L)
    frames = [torch_cuda.from_numpy(_frames(W, H, L, seed=s)).cuda() for s in range(3)]
    ao = _layered(W, H, cams)
    out = torch_cuda.empty((L, H, W), dtype=torch_cuda.uint8, device="cuda")
    for i, d in enumerate(frames):                 # graph capture, then replay on new contents of the same pointers
        src = frames[0]
        src.copy_(d) if i else None
        ao.render(src, out)
        _check(out.cpu().numpy(), _singles(torch_cuda, cams, d.cpu().numpy()), f"replay frame {i}")
    # one layer's camera changes: the next frame re-plans and follows it
    cams2 = list(cams)
    cams2[1] = Camera(W, H, nearClipPlane=0.05, farClipPlane=20.0, fieldOfView=100.0)
    ao.layerCameras = cams2
    assert ao.LateUpdate() is True
    ao.render(frames[0], out)
    _check(out.cpu().numpy(), _singles(torch_cuda, cams2, frames[0].cpu().numpy()), "after a camera change")
    # clearing the table gives exactly the shared-camera frame
    shared = AmbientOcclusion(Camera(W, H), device=0)
    shared.layers = L
    ref = shared.render(frames[0]).cpu().numpy()
    ao.layerCameras = None
    ao.render(frames[0], out)
    assert np.array_equal(out.cpu().numpy(), ref)
    # a table of L identical cameras gives exactly the frame without a table
    ao.layerCameras = [Camera(W, H)] * L
    ao.render(frames[0], out)
    assert np.array_equal(out.cpu().numpy(), ref)


def test_no_graph_host_async_event_and_buffers(torch_cuda):
    from miniengineao_b200 import _native as N
    W, H, L = 512, 288, 3
    cams = cameras(W, H, L)
    depth = _frames(W, H, L, seed=13)
    singles = _singles(torch_cuda, cams, depth)
    ng = _layered(W, H, cams, use_graph=False)
    _check(ng.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy(), singles, "MEAO_FLAG_NO_GRAPH")
    ao = _layered(W, H, cams)
    _check(ao.render_host(depth), singles, "host")
    outs = [np.zeros((L, H, W), np.uint8) for _ in range(3)]
    ao.render_host_batch([depth] * 3, outs)
    for o in outs:
        _check(o, singles, "async host")
    # the plugin event
    lib = N.lib()
    d = torch_cuda.from_numpy(depth).cuda()
    o = torch_cuda.zeros((L, H, W), dtype=torch_cuda.uint8, device="cuda")
    ao.LateUpdate()
    assert lib.meao_bind_event(ao._ctx, 91, C.c_void_p(d.data_ptr()), 0, C.c_void_p(o.data_ptr()), None) == 0
    lib.meao_get_render_event_func()(91)
    torch_cuda.cuda.synchronize()
    _check(o.cpu().numpy(), singles, "event")
    # meao_get_buffer / meao_debug_view of TiledDepth1-4 and the AO after a frame into the caller's buffer
    _compare_buffers(ao, W, H, cams, depth, "buffers after the event frame", **{})
    assert lib.meao_bind_event(ao._ctx, 91, None, 0, None, None) == 0
