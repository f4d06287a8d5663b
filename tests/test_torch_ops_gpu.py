"""GPU tests of the torch.library operators (miniengineao_b200/torch_ops.py) on the H100: torch.library.opcheck; the eager operator bit for
bit against AmbientOcclusion.render / render_batch on the same inputs (every depth kind, both Z directions, L = 1 and 6, strided views,
per-layer and orthographic projections, a high-quality mask, hierarchy depth 2, stereo, both camera forms); torch.compile with
fullgraph=True against eager; the graph trees of mode="reduce-overhead" and a torch.cuda.graph capture replaying a camera that moves on
every call; the kernels an eager call runs (torch.profiler); an invalid camera in the tensor; and the warm-up and generation guards."""
import numpy as np
import pytest

import harness
from gpu_harness import torch_cuda  # noqa: F401  (the fixture)
from miniengineao_b200 import AmbientOcclusion, Camera

pytestmark = pytest.mark.gpu

W, H = 200, 120


@pytest.fixture(scope="module")
def T(torch_cuda):
    from miniengineao_b200 import torch_ops
    yield torch_ops
    torch_ops.release_contexts()


# ---- inputs and the reference ---------------------------------------------------------------------------------------------------------
def _depth(torch, kind, L, seed, reversed_z=True, strided=False):
    """A depth tensor [H, W] (L = 1) or [L, H, W] of `kind`; strided: a corner of a wider, taller tensor (row and layer pitches)."""
    if kind == "linear_f32":
        a = harness.contrasting_layers(W, H, L, seed=seed)
    else:
        a = harness.frames(W, H, L, seed=seed, reversed_z=reversed_z)
        if kind != "raw_f32":
            a = np.stack([harness.ingest(r, "d16" if kind == "d16" else "d24s8")[0] for r in a])
            a = a.view(np.int16) if kind == "d16" else a.view(np.int32)
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    if kind == "d16":
        t = t.view(torch.uint16)
    if strided:
        big = torch.zeros((L, H + 5, W + 24), dtype=t.dtype, device="cuda")
        big[:, 3:3 + H, 8:8 + W] = t
        t = big[:, 3:3 + H, 8:8 + W]
    return t if L > 1 else t[0]


def _cameras(L, i):
    """The cameras of call i: Camera objects (for the reference) and their (near, far, tan_half_fov_h) rows, which move with i."""
    cams = [Camera(W, H, nearClipPlane=0.1 + 0.02 * ((i + l) % 5), farClipPlane=300.0 - 7.0 * ((i + 2 * l) % 9),
                   fieldOfView=40.0 + 1.5 * ((i + 3 * l) % 13)) for l in range(L)]
    return cams, [[c.nearClipPlane, c.farClipPlane, float(np.float32(1.0 / c.projection00))] for c in cams]


def _reference(torch, L, *, reversed_z=True, projection=None, device_rows=None, host=None, params=None, variants=None, depth=4,
               stereo=False):
    """An AmbientOcclusion outside the operator's cache, configured like the call: device_rows -> a bound tensor of those cameras;
    host -> the Camera of every layer.  projection: "orthographic" or a per-layer list, whose layers all read the host camera's
    tan_half_fov_h (the half-width on the orthographic ones), as a `camera` row means."""
    host = host or Camera(W // 2 if stereo else W, H)
    cam = Camera(host.pixelWidth, H, nearClipPlane=host.nearClipPlane, farClipPlane=host.farClipPlane, fieldOfView=host.fieldOfView,
                 usesReversedZBuffer=reversed_z, stereoEnabled=stereo, orthographic=projection == "orthographic")
    ao = AmbientOcclusion(cam, device=0)
    for k, v in (params or {}).items():
        setattr(ao, harness.PARAMS[k], v)
    v = variants or {}
    ao.sampleExhaustively, ao.highQualityMask = v.get("sample_exhaustively", False), v.get("high_quality_mask", 0)
    ao.hierarchyDepth, ao.layers = depth, L
    if isinstance(projection, list):
        from miniengineao_b200.torch_ops import _HostCamera
        near, far, tan = _host_row(cam)
        ao.perLayerProjection = True
        ao.layerCameras = [_HostCamera(cam.pixelWidth, H, near, far, tan, reversed_z, stereo) for _ in projection]
        for c, p in zip(ao.layerCameras, projection):
            c.orthographic = p == "orthographic"
    if device_rows is not None:
        ao.deviceCameras = torch.tensor(device_rows, dtype=torch.float32, device="cuda")
    return ao


def _host_row(cam, projection=None):
    """The `camera` argument that means `cam`: tan_half_fov_h = 1 / projection00 (the orthographic half-width when orthographic)."""
    if projection == "orthographic":
        cam = Camera(cam.pixelWidth, cam.pixelHeight, nearClipPlane=cam.nearClipPlane, farClipPlane=cam.farClipPlane, orthographic=True)
    return [cam.nearClipPlane, cam.farClipPlane, float(np.float32(1.0 / cam.projection00))]


def _cpu(t):
    return t.cpu().numpy() if not isinstance(t, (list, tuple)) else np.stack([x.cpu().numpy() for x in t])


CASES = {
    "raw_f32_L1_host": dict(kind="raw_f32", L=1),
    "raw_f32_L1_device": dict(kind="raw_f32", L=1, device=True),
    "raw_f32_L6_device_forward_z": dict(kind="raw_f32", L=6, device=True, reversed_z=False),
    "linear_f32_L6_host": dict(kind="linear_f32", L=6),
    "linear_f32_L1_device": dict(kind="linear_f32", L=1, device=True),
    "d16_L1_host_forward_z": dict(kind="d16", L=1, reversed_z=False),
    "d16_L6_device": dict(kind="d16", L=6, device=True),
    "d24s8_int32_L6_host": dict(kind="d24s8", L=6),
    "d24s8_uint32_L1_device": dict(kind="d24s8", L=1, device=True, uint32=True),
    "strided_L1_host": dict(kind="raw_f32", L=1, strided=True),
    "strided_L6_device": dict(kind="d16", L=6, device=True, strided=True),
    "mixed_projections_L6_host": dict(kind="raw_f32", L=6, projection=["perspective", "orthographic"] * 3),
    "mixed_projections_L6_device": dict(kind="raw_f32", L=6, device=True, projection=["orthographic"] * 3 + ["perspective"] * 3),
    "orthographic_L1_host": dict(kind="raw_f32", L=1, projection="orthographic"),
    "hq5_L6_device": dict(kind="raw_f32", L=6, device=True, variants=dict(high_quality_mask=5)),
    "hq10_exhaustive_L1_host": dict(kind="raw_f32", L=1, variants=dict(high_quality_mask=10, sample_exhaustively=True)),
    "depth2_L1_device": dict(kind="raw_f32", L=1, device=True, depth=2),
    "depth2_L6_host_params": dict(kind="raw_f32", L=6, depth=2, params=dict(intensity=1.3, thickness_modifier=2.0, blur_tolerance=-3.0)),
    "stereo_L1_host": dict(kind="raw_f32", L=1, stereo=True),
}


def _call_args(torch, cfg, rows, host_cam):
    kw = dict(kind=cfg["kind"], reversed_z=cfg.get("reversed_z", True), hierarchy_depth=cfg.get("depth", 4),
              single_pass_stereo=cfg.get("stereo", False), **cfg.get("params", {}), **cfg.get("variants", {}))
    if "projection" in cfg:
        kw["projection"] = cfg["projection"]
    if cfg.get("device"):
        kw["cameras"] = torch.tensor(rows, dtype=torch.float32, device="cuda")
    else:
        kw["camera"] = _host_row(host_cam, cfg.get("projection") if isinstance(cfg.get("projection"), str) else None)
    return kw


@pytest.mark.parametrize("case", list(CASES))
def test_eager_operator_equals_render(torch_cuda, T, case):
    torch = torch_cuda
    cfg = CASES[case]
    L = cfg["L"]
    host_cam, rows = Camera(W // 2 if cfg.get("stereo") else W, H, nearClipPlane=0.2, farClipPlane=250.0, fieldOfView=50.0), None
    if cfg.get("device"):
        rows = _cameras(L, 0)[1]
    ref = _reference(torch, L, reversed_z=cfg.get("reversed_z", True), projection=cfg.get("projection"), device_rows=rows,
                     host=host_cam, params=cfg.get("params"), variants=cfg.get("variants"), depth=cfg.get("depth", 4),
                     stereo=cfg.get("stereo", False))
    kw = _call_args(torch, cfg, rows, host_cam)
    for seed in (1, 2):
        d = _depth(torch, cfg["kind"], L, seed, reversed_z=cfg.get("reversed_z", True), strided=cfg.get("strided", False))
        if cfg.get("uint32"):
            d = d.view(torch.uint32)
        got = T.ambient_occlusion(d, **kw)
        assert got.shape == d.shape and got.dtype == torch.uint8 and got.is_contiguous()
        if cfg.get("stereo"):
            ref.OnPreRender()
        want = ref.render(d, linear=cfg["kind"] == "linear_f32")
        assert harness.n_diff(_cpu(got), _cpu(want)) == 0, f"{case}: seed {seed}"
        # the batch operator on the same layers, against render_batch
        if L > 1 and not isinstance(cfg.get("projection"), list) and not cfg.get("stereo"):
            layers = [d[l] for l in range(L)]
            got_b = T.ambient_occlusion_batch(layers, **kw)
            assert harness.n_diff(_cpu(got_b), _cpu(want)) == 0, f"{case}: batch, seed {seed}"
            ref_b = _reference(torch, L, reversed_z=cfg.get("reversed_z", True), projection=cfg.get("projection"), device_rows=rows,
                               host=host_cam, params=cfg.get("params"), variants=cfg.get("variants"), depth=cfg.get("depth", 4))
            assert harness.n_diff(_cpu(got_b), _cpu(ref_b.render_batch(layers, linear=cfg["kind"] == "linear_f32"))) == 0, case
            ref_b.close()
    ref.close()


def test_opcheck(torch_cuda, T):
    torch = torch_cuda
    d = _depth(torch, "raw_f32", 2, seed=3)
    cams = torch.tensor(_cameras(2, 0)[1], dtype=torch.float32, device="cuda")
    torch.library.opcheck(torch.ops.meao.ambient_occlusion.default, (d, cams, None, "raw_f32"))
    torch.library.opcheck(torch.ops.meao.ambient_occlusion.default, (d[0], None, [0.3, 100.0, 0.8], "raw_f32"), {"intensity": 1.2})
    torch.library.opcheck(torch.ops.meao.ambient_occlusion_batch.default, ([d[0], d[1]], cams, None, "raw_f32"))


def test_compile_fullgraph_equals_eager(torch_cuda, T):
    torch = torch_cuda
    from torch._dynamo.utils import counters
    torch._dynamo.reset()
    counters.clear()

    def frame(depth, cams):
        return T.ambient_occlusion(depth, cams, hierarchy_depth=3, intensity=1.2)

    def batch(a, b):
        return T.ambient_occlusion_batch([a, b], camera=[0.25, 400.0, 0.9], kind="d16")

    cf, cb = torch.compile(frame, fullgraph=True), torch.compile(batch, fullgraph=True)
    for i in range(3):
        d = _depth(torch, "raw_f32", 6, seed=i)
        cams = torch.tensor(_cameras(6, i)[1], dtype=torch.float32, device="cuda")
        assert torch.equal(cf(d, cams), frame(d, cams)), i
        a, b = _depth(torch, "d16", 2, seed=i, strided=True)
        assert all(torch.equal(x, y) for x, y in zip(cb(a, b), batch(a, b))), i
    assert not counters["graph_break"], dict(counters["graph_break"])
    assert counters["stats"]["unique_graphs"] == 2, dict(counters["stats"])
    torch._dynamo.reset()


@pytest.mark.parametrize("L", [1, 6])
def test_reduce_overhead_follows_moving_cameras(torch_cuda, T, L):
    """The graph trees record the frame once: calls 3..20 replay it, with new cameras every call, and match a fresh context rendering
    each camera; no recompilation, no cudagraph skip, no graph instantiation of the operator's context, no generation change."""
    torch = torch_cuda
    from torch._dynamo.utils import counters
    torch._dynamo.reset()
    counters.clear()
    T.release_contexts()
    depth = _depth(torch, "raw_f32", L, seed=5)
    torch._dynamo.mark_static_address(depth)

    @torch.compile(mode="reduce-overhead", fullgraph=True)
    def frame(d, cams):
        return T.ambient_occlusion(d, cams)

    fresh = _reference(torch, L, device_rows=_cameras(L, 0)[1])
    ctx = inst = launches = None
    for i in range(20):
        rows = _cameras(L, i)[1]
        torch.compiler.cudagraph_mark_step_begin()
        got = frame(depth, torch.tensor(rows, dtype=torch.float32, device="cuda")).cpu().numpy()
        if i == 1:          # warmed up and recorded
            (key, ctx), = T.contexts().items()
            inst, launches = ctx.reservation()["graph_instantiations"], ctx.launch_count
        if i >= 2:
            fresh.deviceCameras.copy_(torch.tensor(rows, dtype=torch.float32))
            want = fresh.render(depth).cpu().numpy()
            assert harness.n_diff(got, want) == 0, f"call {i + 1}"
    assert ctx.reservation()["graph_instantiations"] == inst
    assert ctx.launch_count == launches, "the operator ran during the replays"
    assert T._CONTEXTS[key].generation == ctx._lib.meao_frame_generation(ctx._ctx)
    assert counters["stats"]["unique_graphs"] == 1 and not counters["graph_break"], (dict(counters["stats"]), dict(counters["graph_break"]))
    assert counters["inductor"]["cudagraph_skips"] == 0
    fresh.close()
    torch._dynamo.reset()


def test_torch_cuda_graph_follows_moving_cameras(torch_cuda, T):
    torch = torch_cuda
    L = 3
    depth = _depth(torch, "d24s8", L, seed=7, strided=True)
    cams = torch.tensor(_cameras(L, 0)[1], dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        T.ambient_occlusion(depth, cams, kind="d24s8")             # the warm-up settles the context
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = T.ambient_occlusion(depth, cams, kind="d24s8")
    fresh = _reference(torch, L, device_rows=_cameras(L, 0)[1])
    for i in range(1, 9):
        rows = torch.tensor(_cameras(L, i)[1], dtype=torch.float32)
        cams.copy_(rows)
        g.replay()
        fresh.deviceCameras.copy_(rows)
        assert harness.n_diff(out.cpu().numpy(), fresh.render(depth).cpu().numpy()) == 0, f"replay {i}"
    fresh.close()


@pytest.mark.parametrize("device_cameras", [False, True])
def test_profiler_kernel_count(torch_cuda, T, device_cameras):
    """An eager call runs meao_kernels_per_frame kernels (the camera stage included), and with a cameras tensor one copy besides."""
    torch = torch_cuda
    L = 2
    d = _depth(torch, "raw_f32", L, seed=9)
    kw = dict(cameras=torch.tensor(_cameras(L, 0)[1], dtype=torch.float32, device="cuda")) if device_cameras else \
        dict(camera=[0.3, 90.0, 0.7])
    T.ambient_occlusion(d, intensity=0.9, **kw)
    torch.cuda.synchronize()
    ao = next(a for k, a in T.contexts().items() if k[4] == W and k[6][4] == np.float32(0.9) and (k[-1] == "device") == device_cameras)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        T.ambient_occlusion(d, intensity=0.9, **kw)
        torch.cuda.synchronize()
    dev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    names = [e.name for e in dev]
    copies = [n for n in names if "memcpy" in n.lower() or "copy" in n.lower()]
    kernels = [n for n in names if n not in copies]
    assert len(kernels) == ao.kernels_per_frame, names
    assert len(copies) == (1 if device_cameras else 0), names


def test_invalid_camera_in_the_tensor(torch_cuda, T):
    torch = torch_cuda
    L = 6
    d = _depth(torch, "raw_f32", L, seed=11)
    rows = _cameras(L, 3)[1]
    bad = [list(r) for r in rows]
    bad[2][1] = bad[2][0] * 0.5                                    # far below near: invalid, field 2
    T.ambient_occlusion(d, torch.tensor(rows, dtype=torch.float32, device="cuda"), intensity=0.7)     # a settled context first
    got = T.ambient_occlusion(d, torch.tensor(bad, dtype=torch.float32, device="cuda"), intensity=0.7).cpu().numpy()
    torch.cuda.synchronize()
    ao = next(a for k, a in T.contexts().items() if k[6][4] == np.float32(0.7))
    frames, layer, field = ao.deviceCameraStatus()
    assert frames == 1 and layer == 2 and field == 2, (frames, layer, field)
    want = _reference(torch, L, device_rows=rows, params=dict(intensity=0.7)).render(d).cpu().numpy()
    for l in range(L):
        if l != 2:
            assert harness.n_diff(got[l], want[l]) == 0, f"layer {l}"


def test_warm_up_and_generation_guards(torch_cuda, T):
    torch = torch_cuda
    d = _depth(torch, "raw_f32", 1, seed=13)
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="call the operator once eagerly"):
        with torch.cuda.graph(g):
            T.ambient_occlusion(d, camera=[0.3, 100.0, 0.61])      # a key never seen eagerly
    del g
    T.ambient_occlusion(d, camera=[0.3, 100.0, 0.61])
    (ao,) = [a for k, a in T.contexts().items() if k[-1] == tuple(T._f32(x) for x in (0.3, 100.0, 0.61))]
    ao.intensity = 1.5                                             # what the operator never does: a new value on a cached context
    with pytest.raises(RuntimeError, match="changed under its recorded frames"):
        T.ambient_occlusion(d, camera=[0.3, 100.0, 0.61])
