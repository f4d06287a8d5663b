"""GPU tests of live frame constants on the H100: a change of MeaoParams or of a camera takes effect at the next frame issued, with no
device synchronise, no graph instantiation and no array release.  Every frame must equal a fresh context given that frame's inputs
(the AO and every debug buffer, bit for bit) and, every few frames and on the hostile ones, the oracle.  The no-wait checks put half a
second of work in front of the frames (the backlog of test_dynamic_resolution_gpu.py) and assert that it is still running once the
last frame has been issued; a control in the same test shows that a structural change does wait."""
import ctypes as C

import numpy as np
import pytest

import harness
import hostile_cases as HC
from gpu_harness import SLEEP_CYCLES, Array, backlog, fresh_frame, native_bands, rt, torch_cuda  # noqa: F401  (the fixtures)

pytestmark = pytest.mark.gpu

# frame -> (hostile camera, hostile parameters): far/near at both extremes, fields of view at both extremes, upsample tolerances and
# noise filter strengths on both sides of upsample_fast_div_ok, thickness and intensity far outside their ranges
HOSTILE = {5: ("far_near_1e7", dict(upsample_tolerance=-16.56)), 9: ("tan_half_fov_1em6", dict(upsample_tolerance=-16.55)),
           13: ("far_near_1p2m20", dict(noise_filter_tolerance=15.66)), 17: ("tan_half_fov_1e6", dict(noise_filter_tolerance=15.65)),
           21: ("far_near_overflows", dict(thickness_modifier=1e-6, intensity=100.0, upsample_tolerance=20.0))}
N_FRAMES = 24


def _inputs(i, W, H, n=N_FRAMES):
    """Frame i of an animation: the field of view sweeps 30 -> 90 degrees, near / far, intensity, thickness and the tolerances move
    every frame; the frames of HOSTILE pass through the hostile cameras and parameters."""
    t = i / (n - 1)
    cam = dict(fieldOfView=30.0 + 60.0 * t, nearClipPlane=0.05 + 0.5 * t, farClipPlane=80.0 + 900.0 * t)
    params = dict(intensity=0.4 + 1.5 * t, thicknessModifier=1.0 + 6.0 * t, blurTolerance=-7.0 + 5.0 * t, upsampleTolerance=-11.5 + 9.0 * t,
                  noiseFilterTolerance=-7.5 + 7.0 * t)
    if i in HOSTILE:
        name, hp = HOSTILE[i]
        near, far, tan = HC.CAMERAS[name]
        cam.update(nearClipPlane=near, farClipPlane=far)
        if tan is not None:
            cam["fieldOfView"] = HC.fov_for_tan_half_h(tan, W, H)
        params.update({harness.PARAMS[k]: v for k, v in hp.items()})
    return cam, params


def _apply(ao, cam, params, cameras=None):
    for c in cameras or [ao.camera]:
        for k, v in cam.items():
            setattr(c, k, v)
    for k, v in params.items():
        setattr(ao, k, v)


def _fresh(torch, W, H, depth, cam, params, layers=1, table=None):
    """The AO and every debug buffer of a fresh context given these inputs in one go."""
    from miniengineao_b200 import Camera
    f = harness.context(W, H, device=0, layers=layers)
    _apply(f, cam, params)
    if table is not None:
        f.layerCameras = [Camera(W, H, **c) for c in table]
    return fresh_frame(torch, f, depth)


def _res(ao):
    return ao.reservation()


@pytest.mark.parametrize("W,H", [(1000, 563), (1920, 1080)])
def test_animated_camera_and_parameters(torch_cuda, W, H):
    torch = torch_cuda
    ao = harness.context(W, H, device=0)
    dd = torch.empty((H, W), device="cuda")                             # one depth and one AO buffer: one graph for every frame
    out = torch.empty((H, W), dtype=torch.uint8, device="cuda")
    r1 = None
    for i in range(N_FRAMES):
        cam, params = _inputs(i, W, H)
        _apply(ao, cam, params)
        d = harness.corridor_depth(W, H, frame=i)
        dd.copy_(torch.from_numpy(d))
        got = ao.render(dd, out).cpu().numpy()
        ref, ref_bufs = _fresh(torch, W, H, d, cam, params)
        assert harness.n_diff(got, ref) == 0, f"frame {i}: AO differs from a fresh context"
        for bid in harness.buffer_ids():
            assert harness.n_diff(ao.debug_buffer(bid), ref_bufs[bid]) == 0, f"frame {i}: buffer {bid} differs from a fresh context"
        if i % 4 == 0 or i in HOSTILE:
            orc = harness.oracle(W, H, camera=ao.camera, threads=8, **{harness.PROPERTIES[k]: v for k, v in params.items()})
            oref = orc.run(d)
            assert harness.n_diff(got, oref) == 0, f"frame {i}: AO differs from the oracle"
            harness.compare_buffers(ao.debug_buffer, orc, f"frame {i}", harness.buffer_ids())
        r = _res(ao)
        if r1 is None:
            r1 = r
        assert (r["graph_instantiations"], r["graphs_held"], r["arena_allocations"]) == \
               (r1["graph_instantiations"], r1["graphs_held"], r1["arena_allocations"]), f"frame {i}: {r} after frame 0: {r1}"
    assert r1["graph_instantiations"] == 1
    ao.close()


def test_camera_and_intensity_changes_do_not_wait(torch_cuda):
    torch = torch_cuda
    W, H = 1920, 1080
    s = torch.cuda.Stream()
    ao = harness.context(W, H, device=0)
    d = torch.from_numpy(harness.corridor_depth(W, H)).cuda()
    outs = [torch.empty((H, W), dtype=torch.uint8, device="cuda") for _ in range(5)]
    for o in outs:                                                      # every output's graph: captured before the backlog
        ao.render(d, o, stream=s)
    torch.cuda.synchronize()
    inst = _res(ao)["graph_instantiations"]
    e = backlog(torch, s, ao, d, outs[0])
    frames = []
    for i in range(1, 5):
        cam, params = dict(fieldOfView=40.0 + 10.0 * i, nearClipPlane=0.1 * i), dict(intensity=0.5 + 0.3 * i)
        _apply(ao, cam, params)
        ao.render(d, outs[i], stream=s)
        frames.append((cam, params, outs[i]))
    assert not e.query(), "a camera or parameter change waited for the GPU"
    torch.cuda.synchronize()
    assert _res(ao)["graph_instantiations"] == inst
    dn = harness.corridor_depth(W, H)
    for cam, params, out in frames:
        assert harness.n_diff(out.cpu().numpy(), _fresh(torch, W, H, dn, cam, params)[0]) == 0, (cam, params)
    # the control: a structural input (MeaoVariants) under the same backlog does drain the GPU -- the test observes what it claims
    e = backlog(torch, s, ao, d, outs[0])
    ao.sampleExhaustively = True
    ao.render(d, outs[1], stream=s)
    assert e.query(), "a variant change is expected to re-plan with a device synchronise"
    torch.cuda.synchronize()
    ao.close()


def _sleep(torch, s):
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    e = torch.cuda.Event()
    e.record(s)
    return e


def _step_inputs(i):
    return dict(fieldOfView=35.0 + 11.0 * i, nearClipPlane=0.1 + 0.07 * i, farClipPlane=60.0 + 300.0 * i), dict(intensity=0.6 + 0.25 * i,
                                                                                                              blurTolerance=-5.0 + 0.5 * i)


def test_pitched_and_no_graph_frames(torch_cuda):
    torch = torch_cuda
    W, H = 1000, 563
    s = torch.cuda.Stream()
    rtd = torch.zeros((H + 7, W + 24), device="cuda")
    d = harness.corridor_depth(W, H)
    rtd[3:3 + H, 5:5 + W].copy_(torch.from_numpy(d))
    for use_graph in (True, False):
        ao = harness.context(W, H, device=0, use_graph=use_graph)
        big = [torch.zeros((H + 3, W + 40), dtype=torch.uint8, device="cuda") for _ in range(4)]
        for b in big:
            ao.render(rtd[3:3 + H, 5:5 + W], b[:H, 8:8 + W], stream=s)
        torch.cuda.synchronize()
        inst = _res(ao)["graph_instantiations"]
        e = _sleep(torch, s)
        steps = []
        for i in range(1, 4):
            cam, params = _step_inputs(i)
            _apply(ao, cam, params)
            ao.render(rtd[3:3 + H, 5:5 + W], big[i][:H, 8:8 + W], stream=s)
            steps.append((cam, params, big[i]))
        assert not e.query(), f"use_graph={use_graph}: a constants change waited for the GPU"
        torch.cuda.synchronize()
        assert _res(ao)["graph_instantiations"] == inst
        for cam, params, b in steps:
            assert harness.n_diff(b[:H, 8:8 + W].cpu().numpy(), _fresh(torch, W, H, d, cam, params)[0]) == 0, (use_graph, cam, params)
        ao.close()


def test_array_frames_keep_their_arrays(torch_cuda, rt):
    torch = torch_cuda
    W, H = 777, 431
    s = torch.cuda.Stream()
    ao = harness.context(W, H, device=0)
    d = harness.corridor_depth(W, H)
    da = Array(rt, W, H, np.float32)
    da.fill(d)
    aas = [Array(rt, W, H, np.uint8) for _ in range(4)]
    ao.render_arrays(da.handle, aas[0].handle, stream=s)
    for a in aas[1:]:                                                   # every AO array's graph: captured before the backlog
        ao.render_arrays(da.handle, a.handle, stream=s)
    torch.cuda.synchronize()
    inst = _res(ao)["graph_instantiations"]
    e = _sleep(torch, s)
    steps = []
    for i, a in enumerate(aas):
        cam, params = _step_inputs(i + 1)
        _apply(ao, cam, params)
        ao.render_arrays(da.handle, a.handle, stream=s)
        steps.append((cam, params, a))
    assert not e.query(), "a constants change on an array frame waited for the GPU"
    torch.cuda.synchronize()
    assert _res(ao)["graph_instantiations"] == inst, "a constants change released the arrays' graphs"
    for cam, params, a in steps:
        assert harness.n_diff(a.read()[0], _fresh(torch, W, H, d, cam, params)[0]) == 0, (cam, params)
    for a in [da] + aas:
        ao.release_array(a.handle)
        a.free()
    ao.close()


def test_plugin_event_bound_once(torch_cuda):
    from miniengineao_b200 import _native as N
    torch = torch_cuda
    W, H = 1280, 720
    s = torch.cuda.Stream()
    ao = harness.context(W, H, device=0)
    ao.LateUpdate()
    d = harness.corridor_depth(W, H)
    dd = torch.from_numpy(d).cuda()
    out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    lib = N.lib()
    assert lib.meao_bind_event(ao._ctx, 91, C.c_void_p(dd.data_ptr()), 0, C.c_void_p(out.data_ptr()), C.c_void_p(s.cuda_stream)) == 0
    lib.meao_render_event(91)
    torch.cuda.synchronize()
    for i in range(1, 4):
        cam, params = _step_inputs(i)
        _apply(ao, cam, params)
        ao.LateUpdate()                                                 # the host's per-frame update, then the render thread's event
        e = _sleep(torch, s)
        lib.meao_render_event(91)
        assert not e.query(), "a constants change waited for the GPU"
        torch.cuda.synchronize()
        assert harness.n_diff(out.cpu().numpy(), _fresh(torch, W, H, d, cam, params)[0]) == 0, (cam, params)
    assert _res(ao)["graph_instantiations"] == 1
    lib.meao_bind_event(ao._ctx, 91, None, 0, None, None)
    ao.close()


def test_host_async_slots_and_stage_api(torch_cuda):
    torch = torch_cuda
    W, H = 960, 540
    ao = harness.context(W, H, device=0)
    lib = ao._lib
    d = harness.corridor_depth(W, H)
    dpin = torch.from_numpy(d).pin_memory()
    outs = [torch.zeros((H, W), dtype=torch.uint8).pin_memory() for _ in range(6)]
    ao.LateUpdate()
    assert lib.meao_render_host_async(ao._ctx, dpin.data_ptr(), 0, outs[0].data_ptr(), 0) == 0
    assert lib.meao_host_wait(ao._ctx, 0) == 0
    s = torch.cuda.Stream()
    e = _sleep(torch, s)                                               # a device synchronise would wait for it
    steps = []
    for i in range(1, 6):                                              # render_host_async, both slots, new constants every frame
        cam, params = _step_inputs(i)
        _apply(ao, cam, params)
        ao.LateUpdate()
        if i >= 3:
            assert lib.meao_host_wait(ao._ctx, i & 1) == 0
        assert lib.meao_render_host_async(ao._ctx, dpin.data_ptr(), 0, outs[i].data_ptr(), i & 1) == 0
        steps.append((cam, params, outs[i]))
    assert not e.query(), "render_host_async waited for the device after a constants change"
    assert lib.meao_host_wait(ao._ctx, 0) == 0 and lib.meao_host_wait(ao._ctx, 1) == 0
    torch.cuda.synchronize()
    for cam, params, o in steps:
        assert harness.n_diff(o.numpy(), _fresh(torch, W, H, d, cam, params)[0]) == 0, (cam, params)
    # the stage API on a stream behind a backlog: each stage call takes the constants of now
    dd = torch.from_numpy(d).cuda()
    for i in range(6, 8):
        cam, params = _step_inputs(i)
        _apply(ao, cam, params)
        e = _sleep(torch, s)
        with torch.cuda.stream(s):
            ao.stage_downsample(dd)
            for k in range(1, 5):
                ao.stage_render(k)
            for lo in range(4, 0, -1):
                ao.stage_upsample(lo)
        assert not e.query(), "the stage API waited for the GPU after a constants change"
        torch.cuda.synchronize()
        _, ref_bufs = _fresh(torch, W, H, d, cam, params)
        for bid in harness.buffer_ids():
            assert harness.n_diff(ao.debug_buffer(bid), ref_bufs[bid]) == 0, f"stage API step {i}: buffer {bid}"
    ao.close()


def test_layered_tables_change_every_frame_back_to_back(torch_cuda):
    """Six layers, each with its own camera, and a new table every frame; the frames are enqueued back to back behind a backlog, so
    every frame must read its own stream-ordered tables."""
    from miniengineao_b200 import Camera
    torch = torch_cuda
    W, H, L = 640, 360, 6

    def table(i):
        return [dict(fieldOfView=30.0 + 9.0 * l + 3.0 * i, nearClipPlane=0.05 + 0.1 * l + 0.02 * i, farClipPlane=50.0 + 200.0 * l + 17.0 * i)
                for l in range(L)]

    ao = harness.context(W, H, device=0, layers=L)
    ao.layerCameras = [Camera(W, H, **c) for c in table(0)]
    d = harness.corridor_depth(W, H, L=L)
    dd = torch.from_numpy(d).cuda()
    s = torch.cuda.Stream()
    outs = [torch.empty((L, H, W), dtype=torch.uint8, device="cuda") for _ in range(6)]
    for o in outs:
        ao.render(dd, o, stream=s)
    torch.cuda.synchronize()
    inst = _res(ao)["graph_instantiations"]
    e = _sleep(torch, s)
    frames = []
    for i, o in enumerate(outs):
        t = table(i + 1)
        ao.layerCameras = [Camera(W, H, **c) for c in t]
        ao.intensity = 0.5 + 0.2 * i
        frames.append((t, ao.intensity, ao.render(dd, o, stream=s)))
    assert not e.query(), "a layer-camera table change waited for the GPU"
    torch.cuda.synchronize()
    assert _res(ao)["graph_instantiations"] == inst
    for t, intensity, out in frames:
        ref, _ = _fresh(torch, W, H, d, {}, dict(intensity=intensity), layers=L, table=t)
        assert harness.n_diff(out.cpu().numpy(), ref) == 0, "a back-to-back frame read another frame's camera table"
    ao.close()


def test_reserved_context_with_an_aspect_following_camera(torch_cuda):
    """The default Camera's projection follows its pixel aspect, so every resize below is a camera change as well."""
    torch = torch_cuda
    M = (1920, 1080)
    ao = harness.context(*M, device=0, max_resolution=M)
    sizes = [(1920, 1080), (1601, 901), (1000, 563), (1777, 999), (1280, 720)]
    walk = sizes[1:] + sizes[:1] + sizes[2:]
    depths = {sz: torch.from_numpy(harness.corridor_depth(*sz)).cuda() for sz in sizes}
    outs = [torch.empty((sz[1], sz[0]), dtype=torch.uint8, device="cuda") for sz in walk]
    for sz, o in zip(walk, outs):                                      # the first capture of every size and output
        ao.camera.pixelWidth, ao.camera.pixelHeight = sz
        ao.render(depths[sz], o)
    torch.cuda.synchronize()
    r0 = _res(ao)
    s = torch.cuda.Stream()
    e = _sleep(torch, s)
    frames = []
    for i, (sz, o) in enumerate(zip(walk, outs)):
        ao.camera.pixelWidth, ao.camera.pixelHeight = sz
        ao.intensity = 0.7 + 0.1 * i
        frames.append((sz, ao.intensity, ao.render(depths[sz], o, stream=s)))
    assert not e.query(), "a resize with a camera change waited for the GPU"
    torch.cuda.synchronize()
    r1 = _res(ao)
    assert r1["arena_allocations"] == r0["arena_allocations"] and r1["graph_instantiations"] == r0["graph_instantiations"], (r0, r1)
    for sz, intensity, out in frames:
        ref, _ = _fresh(torch, *sz, depths[sz].cpu().numpy(), {}, dict(intensity=intensity))
        assert harness.n_diff(out.cpu().numpy(), ref) == 0, sz
    ao.close()


def test_row_bands_follow_the_camera(torch_cuda):
    """Two connected bands in one process (as the native-exchange tests run them): the camera changes between steps, the bands stay
    connected and the union of the bands equals the whole frame of a fresh context every step."""
    torch = torch_cuda
    W, H, bands = 1920, 1080, 2
    cuts, ctxs, streams = native_bands(torch, W, H, bands)
    d = harness.corridor_depth(W, H)
    bufs = [torch.from_numpy(np.ascontiguousarray(d[cuts[i]:cuts[i + 1]])).cuda() for i in range(bands)]
    outs = [torch.zeros((cuts[i + 1] - cuts[i], W), dtype=torch.uint8, device="cuda") for i in range(bands)]
    for step in range(4):
        cam, params = _step_inputs(step)
        for a in ctxs:
            _apply(a, cam, params)
            a.LateUpdate()
        for i, a in enumerate(ctxs):
            a.band_step(bufs[i], outs[i], stream=streams[i])
        torch.cuda.synchronize()
        assert [a.band_status()["error"] for a in ctxs] == [0] * bands, "a neighbour exchange timed out"
        assert [a.band_status()["epoch"] for a in ctxs] == [step + 2] * bands, "a constants change reset the band's epoch"
        got = np.concatenate([o.cpu().numpy() for o in outs], axis=0)
        assert harness.n_diff(got, _fresh(torch, W, H, d, cam, params)[0]) == 0, f"step {step}: the bands differ from the whole frame"
    assert all(_res(a)["graph_instantiations"] == 1 for a in ctxs)
    for a in ctxs:
        a.close()
