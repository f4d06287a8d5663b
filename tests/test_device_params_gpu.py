"""GPU tests of device parameters (meao_bind_device_params) on the H100: with (thickness_modifier, intensity) in a CUDA float32 tensor and
host parameters that differ from them, every layer's AO and debug buffers must equal, bit for bit, the same frame on a context whose host
parameters are the tensor's -- through pointer frames of every depth kind and Z direction, L = 1 (the layered renders with one layer) and
L = 3, the variants, stereo, host frames and MEAO_FLAG_NO_GRAPH, orthographic and mixed projection tables, device cameras bound as well,
CUDA arrays and _at viewports, pitched views, a layer-viewport table, both batches, the plugin event, both reservations, every hierarchy
depth and the stage calls.  A torch.cuda.graph captured once follows the tensor at every replay without moving meao_frame_generation or
instantiating a graph.  An invalid block is counted by the status and leaves the AO at the last valid values.  The torch operator under
torch.compile(mode="reduce-overhead") follows a changing render_params tensor with one compile."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import _native as N
from test_device_cameras_gpu import LINEAR, cam_tensor, cameras, check, depth_of, same_buffers, to_tensor

pytestmark = pytest.mark.gpu

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
DEV = (2.3, 0.6)            # the device block (thickness_modifier, intensity)
OTHER = dict(thickness_modifier=0.8, intensity=1.4)     # the bound contexts' host values: they must not show


def host_context(cams, params=DEV, table=None, **kw):
    """A context whose host cameras are `cams` and whose host (thickness_modifier, intensity) are `params`."""
    L = len(cams)
    ao = harness.context(cams[0], device=0, layers=L, layer_cameras=cams if L > 1 else None, thickness_modifier=params[0],
                         intensity=params[1], **kw)
    if table is not None and L > 1:
        ao.perLayerProjection = True
    return ao


def bound_context(torch, cams, params=DEV, table=None, **kw):
    """A context with the host cameras `cams`, host parameters OTHER and a device parameter buffer holding `params`."""
    ao = host_context(cams, (OTHER["thickness_modifier"], OTHER["intensity"]), table, **kw)
    ao.deviceParams = torch.tensor(params, dtype=torch.float32, device="cuda")
    return ao


def _pair(torch, W, H, L, kind="f32", rz=True, seed=0, **kw):
    cams = cameras(W, H, L, rz)
    d = depth_of(W, H, kind, rz, L, seed=seed)
    return cams, (d if L > 1 else d[0]), bound_context(torch, cams, **kw), host_context(cams, **kw)


@pytest.mark.parametrize("L", [1, 3])
@pytest.mark.parametrize("reversed_z", [True, False])
@pytest.mark.parametrize("kind", list(LINEAR))
def test_pointer_frames(torch_cuda, kind, reversed_z, L):
    cams, d, ao, ref = _pair(torch_cuda, 161, 93, L, kind, reversed_z, seed=3)
    got = ao.render(to_tensor(torch_cuda, d), linear=LINEAR[kind]).cpu().numpy()
    want = ref.render(to_tensor(torch_cuda, d), linear=LINEAR[kind]).cpu().numpy()
    check(torch_cuda, ao, ref, got, want, f"{kind} rz={reversed_z} L={L}")
    assert ao.deviceParamStatus() == (0, 0)
    ao.close(); ref.close()


@pytest.mark.parametrize("params", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True),
                                    dict(high_quality_mask=5, sample_exhaustively=True, use_graph=False)])
@pytest.mark.parametrize("L", [1, 3])
def test_variants_host_frames_and_no_graph(torch_cuda, params, L):
    cams, d, ao, ref = _pair(torch_cuda, 333, 187, L, seed=5, **params)
    kw = {k: v for k, v in params.items() if k != "use_graph"}
    check(torch_cuda, ao, ref, ao.render(to_tensor(torch_cuda, d)).cpu().numpy(), ref.render(to_tensor(torch_cuda, d)).cpu().numpy(),
          f"{params} L={L}", **kw)
    check(torch_cuda, ao, ref, ao.render_host(d), ref.render_host(d), f"host {params} L={L}", **kw)
    ao.close(); ref.close()


@pytest.mark.parametrize("L", [1, 2])
def test_stereo(torch_cuda, L):
    torch = torch_cuda
    W, H = 256, 96
    d = depth_of(W, H, "f32", True, L, seed=2)
    d = d if L > 1 else d[0]
    outs = []
    for bound in (True, False):
        params = OTHER if bound else dict(thickness_modifier=DEV[0], intensity=DEV[1])
        a = harness.context(W, H, device=0, stereo=True, layers=L, **params)
        if bound:
            a.deviceParams = torch.tensor(DEV, dtype=torch.float32, device="cuda")
        outs.append((a, a.render(to_tensor(torch, d)).cpu().numpy()))
    check(torch, outs[0][0], outs[1][0], outs[0][1], outs[1][1], f"stereo L={L}")


@pytest.mark.parametrize("table", [[O], [O, O], [P, O, O], [O, P, O, P, O, P]])
@pytest.mark.parametrize("device_cameras", [False, True])
def test_orthographic_mixed_and_device_cameras(torch_cuda, table, device_cameras):
    torch = torch_cuda
    W, H = 128, 80
    L = len(table)
    cams = cameras(W, H, L, table=table)
    for kind in ("f32", "d16", "linear"):
        d = depth_of(W, H, kind, True, L, seed=L)
        d = d if L > 1 else d[0]
        ao, ref = bound_context(torch, cams, table=table), host_context(cams, table=table)
        if device_cameras:
            ao.deviceCameras = cam_tensor(torch, cams)
        got = ao.render(to_tensor(torch, d), linear=LINEAR[kind]).cpu().numpy()
        want = ref.render(to_tensor(torch, d), linear=LINEAR[kind]).cpu().numpy()
        check(torch, ao, ref, got, want, f"{table} {kind} cams={device_cameras}")
        ao.close(); ref.close()


@pytest.mark.parametrize("L", [1, 3])
def test_perspective_with_device_cameras(torch_cuda, L):
    torch = torch_cuda
    cams, d, ao, ref = _pair(torch, 200, 120, L, seed=8, high_quality_mask=3)
    ao.deviceCameras = cam_tensor(torch, cams)
    check(torch, ao, ref, ao.render(to_tensor(torch, d)).cpu().numpy(), ref.render(to_tensor(torch, d)).cpu().numpy(), f"cams L={L}",
          high_quality_mask=3)
    assert ao.deviceCameraStatus() == (0, 0, 0) and ao.deviceParamStatus() == (0, 0)


def test_arrays_pitched_viewports_batches_and_events(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 96, 64, 3
    cams, d, ao, ref = _pair(torch, W, H, L, seed=9)
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
    outs = []
    for a in (ao, ref):
        bigd = torch.full((L + 1, H + 3, W + 37), 0.5, dtype=torch.float32, device="cuda")
        bigd[1:, 1:H + 1, 5:W + 5] = torch.from_numpy(d).cuda()
        out_big = torch.full((L, H + 2, W + 19), 7, dtype=torch.uint8, device="cuda")
        a.render(bigd[1:, 1:H + 1, 5:W + 5], out_big[:, 1:H + 1, 3:W + 3])
        outs.append(out_big.cpu().numpy())
    check(torch, ao, ref, outs[0], outs[1], "pitched")
    views = [(0, 0, l, 0, 0, l) for l in range(L)]
    for a in (ao, ref):
        a.layerViewports = views
        a._out = a.render(to_tensor(torch, d)).cpu().numpy()
        a.layerViewports = None
    check(torch, ao, ref, ao._out, ref._out, "viewport table")
    for a in (ao, ref):
        a._out = [o.cpu().numpy() for o in a.render_batch([to_tensor(torch, d[l]) for l in range(L)])]
    check(torch, ao, ref, ao._out, ref._out, "batch")
    for a in (ao, ref):
        deps = [Array(rt, W, H, np.float32) for _ in range(L)]
        aos = [Array(rt, W, H, np.uint8) for _ in range(L)]
        for l in range(L):
            deps[l].fill(d[l])
        a.render_arrays_batch([x.handle for x in deps], [x.handle for x in aos])
        torch.cuda.synchronize()
        a._out = np.stack([x.read() for x in aos])
        for x in deps + aos:
            a.release_array(x.handle)
            x.free()
    check(torch, ao, ref, ao._out, ref._out, "array batch")
    lib = N.lib()
    dt = to_tensor(torch, d)
    res = []
    for i, a in enumerate((ao, ref)):
        o = torch.zeros((L, H, W), dtype=torch.uint8, device="cuda")
        assert lib.meao_bind_event(a._ctx, 80 + i, C.c_void_p(dt.data_ptr()), N.MEAO_DEPTH_RAW_F32, C.c_void_p(o.data_ptr()), None) == 0
        lib.meao_get_render_event_func()(80 + i)
        torch.cuda.synchronize()
        res.append(o.cpu().numpy())
        assert lib.meao_bind_event(a._ctx, 80 + i, None, 0, None, None) == 0
    check(torch, ao, ref, res[0], res[1], "event")


@pytest.mark.parametrize("depth", [1, 2, 3, 4])
def test_hierarchy_depths_and_reservations(torch_cuda, depth):
    """Every hierarchy depth, inside a size reservation and a layer reservation, at two sizes and two layer counts."""
    torch = torch_cuda
    W, H = 160, 96
    for L, size in ((2, (W, H)), (3, (W - 32, H - 16)), (1, (W, H))):
        cams = cameras(size[0], size[1], L)
        d = depth_of(size[0], size[1], "f32", True, L, seed=depth + L)
        d = d if L > 1 else d[0]
        ao, ref = bound_context(torch, cams, high_quality_mask=1), host_context(cams, high_quality_mask=1)
        for a in (ao, ref):
            a.hierarchyDepth = depth
            a.maxResolution = (W, H)
            a.maxLayers = 4
        check(torch, ao, ref, ao.render(to_tensor(torch, d)).cpu().numpy(), ref.render(to_tensor(torch, d)).cpu().numpy(),
              f"depth {depth} L={L} {size}", high_quality_mask=1)
        ao.close(); ref.close()


@pytest.mark.parametrize("L", [1, 3])
def test_stage_calls(torch_cuda, L):
    """meao_stage_downsample derives the parameters; the later stage calls read them."""
    cams, d, ao, ref = _pair(torch_cuda, 128, 72, L, seed=11, high_quality_mask=2)
    lib = N.lib()
    n0 = lib.meao_launch_count(ao._ctx)
    for a in (ao, ref):
        a.stage_downsample(to_tensor(torch_cuda, d))
        for k in (1, 2, 3, 4):
            a.stage_render(k)
        a.stage_render_wide(2)
        for lo in (4, 3, 2, 1):
            a.stage_upsample(lo)
    torch_cuda.cuda.synchronize()
    assert lib.meao_launch_count(ao._ctx) - n0 == 11          # the parameter stage, the prepare, five renders, four upsamples
    same_buffers(ao, ref, harness.buffer_ids(2), f"stages L={L}")


def _host_frame(torch, cams, depth, params, kind, **kw):
    ref = host_context(cams, params, **kw)
    out = ref.render(depth, linear=kind == "linear").cpu().numpy()
    ref.close()
    return out


def test_torch_graph_follows_the_parameter_tensor(torch_cuda):
    """One capture; every replay equals a fresh host-parameter frame of the values written into the tensor on the stream between
    replays.  Neither the generation nor the instantiation count moves."""
    torch = torch_cuda
    W, H, L = 192, 108, 2
    cams = cameras(W, H, L)
    d = depth_of(W, H, "d24s8", True, L, seed=4)
    depth = to_tensor(torch, d)
    ao = bound_context(torch, cams, high_quality_mask=2)
    prm = ao.deviceParams
    out = torch.empty((L, H, W), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ao.render(depth, out, stream=s)         # one settling frame: binds the tensor and plans
    s.synchronize()
    lib = N.lib()
    gen, inst = lib.meao_frame_generation(ao._ctx), ao.reservation()["graph_instantiations"]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ao.render(depth, out, stream=s)
    # a fade: intensity 0 .. 1.5, thickness 0.5 .. 4, a subnormal and a huge thickness
    seq = [(1.0, 0.0), (0.5, 0.25), (1.0, 0.5), (2.0, 1.0), (4.0, 1.5), (1e-40, 0.7), (3e38, 1.2), (float("inf"), 0.9)]
    for tm, inten in seq:
        with torch.cuda.stream(s):
            prm.copy_(torch.tensor([tm, inten], dtype=torch.float32), non_blocking=False)
            g.replay()
        s.synchronize()
        want = _host_frame(torch, cams, depth, (tm, inten), "d24s8", high_quality_mask=2)
        assert np.array_equal(out.cpu().numpy(), want), (tm, inten)
    assert lib.meao_frame_generation(ao._ctx) == gen
    assert ao.reservation()["graph_instantiations"] == inst
    assert ao.deviceParamStatus() == (0, 0)
    ao.close()


def test_context_graph_follows_the_buffer_without_instantiation(torch_cuda):
    torch = torch_cuda
    cams, d, ao, _ = _pair(torch, 160, 90, 1, seed=6)
    depth = to_tensor(torch, d)
    ao.render(depth)
    torch.cuda.synchronize()
    inst, gen = ao.reservation()["graph_instantiations"], N.lib().meao_frame_generation(ao._ctx)
    for tm, inten in ((0.7, 1.3), (5.0, 0.2), (1.0, 1.0)):
        ao.deviceParams.copy_(torch.tensor([tm, inten]))
        got = ao.render(depth).cpu().numpy()
        assert np.array_equal(got, _host_frame(torch, cams, depth, (tm, inten), "f32")), (tm, inten)
    assert ao.reservation()["graph_instantiations"] == inst and N.lib().meao_frame_generation(ao._ctx) == gen


@pytest.mark.parametrize("bad", [0.0, -1.0, float("nan"), -float("inf")])
def test_invalid_block_keeps_the_last_valid_values(torch_cuda, bad):
    torch = torch_cuda
    cams, d, ao, _ = _pair(torch, 144, 80, 3, seed=12)
    depth = to_tensor(torch, d)
    # before any valid block: the host values at bind time
    ao.deviceParams.copy_(torch.tensor([bad, 0.3]))
    got = ao.render(depth).cpu().numpy()
    assert np.array_equal(got, _host_frame(torch, cams, depth, (OTHER["thickness_modifier"], OTHER["intensity"]), "f32"))
    assert ao.deviceParamStatus() == (1, 1)
    ao.deviceParams.copy_(torch.tensor([1.7, 0.8]))
    valid = ao.render(depth).cpu().numpy()
    assert np.array_equal(valid, _host_frame(torch, cams, depth, (1.7, 0.8), "f32"))
    ao.deviceParams.copy_(torch.tensor([bad, 0.1]))
    for _ in range(2):
        assert np.array_equal(ao.render(depth).cpu().numpy(), valid)
    torch.cuda.synchronize()
    assert ao.deviceParamStatus() == (3, 1)
    ao.close()


def test_host_changes_while_bound_and_unbind(torch_cuda):
    """A host thickness / intensity change while bound moves nothing and does not show; after the unbind the host values apply."""
    torch = torch_cuda
    cams, d, ao, _ = _pair(torch, 128, 64, 2, seed=13)
    depth = to_tensor(torch, d)
    first = ao.render(depth).cpu().numpy()
    gen = N.lib().meao_frame_generation(ao._ctx)
    ao.intensity, ao.thicknessModifier = 0.2, 3.0
    assert np.array_equal(ao.render(depth).cpu().numpy(), first)
    assert N.lib().meao_frame_generation(ao._ctx) == gen
    ao.deviceParams = None
    assert np.array_equal(ao.render(depth).cpu().numpy(), _host_frame(torch, cams, depth, (3.0, 0.2), "f32"))
    ao.close()


def test_profile_names_the_parameter_stage(torch_cuda):
    torch = torch_cuda
    cams, d, ao, _ = _pair(torch, 128, 72, 1, seed=1)
    out = torch.empty((72, 128), dtype=torch.uint8, device="cuda")
    names = [n for n, _ in ao.profile_frame(to_tensor(torch, d), out)]
    assert names[0] == "render_params" and names[1] == "prepare_depth", names
    assert len(names) == N.lib().meao_kernels_per_frame(ao._ctx)
    ao.deviceCameras = cam_tensor(torch, cams)
    names = [n for n, _ in ao.profile_frame(to_tensor(torch, d), out)]
    assert names[:3] == ["camera_tables", "render_params", "prepare_depth"], names
    ao.close()


def test_the_status_counts_stage_launches(torch_cuda):
    """A frame launches the stage once; a profiled frame launches it profile_repeats times, and each launch that meets an invalid block
    counts (include/meao.h meao_device_param_status)."""
    torch = torch_cuda
    cams, d, ao, _ = _pair(torch, 128, 72, 1, seed=2)
    depth = to_tensor(torch, d)
    ao.deviceParams.copy_(torch.tensor([-1.0, 0.5]))
    ao.render(depth)
    torch.cuda.synchronize()
    assert ao.deviceParamStatus() == (1, 1)
    out = torch.empty((72, 128), dtype=torch.uint8, device="cuda")
    ao.profile_frame(depth, out, repeats=3)
    assert ao.deviceParamStatus() == (4, 1)
    ao.close()


# ---- the torch operator ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def T(torch_cuda):
    from miniengineao_b200 import torch_ops
    yield torch_ops
    torch_ops.release_contexts()


def _op_depth(torch, L, seed):
    return to_tensor(torch, depth_of(160, 96, "f32", True, L, seed=seed))


def test_opcheck(torch_cuda, T):
    torch = torch_cuda
    d = _op_depth(torch, 2, 1)
    rp = torch.tensor(DEV, dtype=torch.float32, device="cuda")
    torch.library.opcheck(torch.ops.meao.ambient_occlusion.default, (d, None, [0.3, 100.0, 0.8], "raw_f32"), {"render_params": rp})
    torch.library.opcheck(torch.ops.meao.ambient_occlusion_batch.default, ([d[0], d[1]], None, [0.3, 100.0, 0.8], "raw_f32"),
                          {"render_params": rp})
    for bad in (rp.double(), rp[:1], rp.cpu(), torch.zeros((1, 2), device="cuda")):
        with pytest.raises(ValueError, match="render_params"):
            T.ambient_occlusion(d, camera=[0.3, 100.0, 0.8], render_params=bad)


@pytest.mark.parametrize("batch", [False, True])
def test_operator_equals_render(torch_cuda, T, batch):
    torch = torch_cuda
    d = _op_depth(torch, 3, 2)
    cam = [0.3, 100.0, 0.8]
    for tm, inten in ((2.0, 0.5), (0.6, 1.3)):
        rp = torch.tensor([tm, inten], dtype=torch.float32, device="cuda")
        if batch:
            got = np.stack([o.cpu().numpy() for o in T.ambient_occlusion_batch(list(d), camera=cam, render_params=rp)])
            fixed = np.stack([o.cpu().numpy() for o in T.ambient_occlusion_batch(list(d), camera=cam, thickness_modifier=tm, intensity=inten)])
        else:
            got = T.ambient_occlusion(d, camera=cam, render_params=rp).cpu().numpy()
            fixed = T.ambient_occlusion(d, camera=cam, thickness_modifier=tm, intensity=inten).cpu().numpy()
        assert np.array_equal(got, fixed), (tm, inten)
    keys = [k for k in T.contexts() if k[0] == ("batch" if batch else "frame") and k[2] == 3 and k[6][3] == "device"]
    assert len(keys) == 1, keys                   # one context serves every value


def test_reduce_overhead_follows_render_params(torch_cuda, T):
    """One compile: the graph trees record the frame once and every later call replays it with new render_params, bit-identical to
    AmbientOcclusion.render with those host values; no recompilation, no cudagraph skip, no instantiation, no generation change."""
    torch = torch_cuda
    from torch._dynamo.utils import counters
    torch._dynamo.reset()
    counters.clear()
    T.release_contexts()
    L = 2
    depth = _op_depth(torch, L, 5)
    torch._dynamo.mark_static_address(depth)
    cam = [0.3, 100.0, 0.8]

    @torch.compile(mode="reduce-overhead", fullgraph=True)
    def frame(d, rp):
        return T.ambient_occlusion(d, camera=cam, render_params=rp)

    ctx = inst = launches = None
    for i in range(12):
        tm, inten = 0.5 + 0.3 * i, 1.5 - 0.12 * i
        torch.compiler.cudagraph_mark_step_begin()
        got = frame(depth, torch.tensor([tm, inten], dtype=torch.float32, device="cuda")).cpu().numpy()
        if i == 1:
            (key, ctx), = T.contexts().items()
            inst, launches = ctx.reservation()["graph_instantiations"], ctx.launch_count
        if i >= 2:
            ref = T._HostCamera(160, 96, 0.3, 100.0, 0.8, True, False)
            fresh = harness.context(ref, device=0, layers=L, thickness_modifier=tm, intensity=inten)
            want = fresh.render(depth).cpu().numpy()
            fresh.close()
            assert np.array_equal(got, want), f"call {i + 1}"
    assert ctx.reservation()["graph_instantiations"] == inst
    assert ctx.launch_count == launches, "the operator ran during the replays"
    assert T._CONTEXTS[key].generation == ctx._lib.meao_frame_generation(ctx._ctx)
    assert counters["stats"]["unique_graphs"] == 1 and not counters["graph_break"], (dict(counters["stats"]), dict(counters["graph_break"]))
    assert counters["inductor"]["cudagraph_skips"] == 0
    torch._dynamo.reset()
