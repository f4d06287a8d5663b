"""GPU tests of frames recorded into the caller's CUDA graph on the H100: a call on a stream that is being captured records its kernels
into that capture (torch.cuda.graph, or cudaStreamBeginCapture in any mode).  Each capture follows one warm-up frame outside it.  Every
replay must give the bytes of the oracle and of an eager frame of a fresh context; a refused call must leave the caller's capture valid;
meao_frame_generation must tell a host when its graph no longer describes the context."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, native_bands, rt, runtime, torch_cuda  # noqa: F401  (the fixtures)

pytestmark = pytest.mark.gpu

REPLAYS = 8
TORCH_DTYPE = {"f32": "float32", "d16": "int16", "d24s8": "int32"}        # d16 / d24s8: the bits, viewed as uint16 / int32 codes


def _depth(kind, W, H, L, seed):
    """(depth [L, H, W] in the ingest format of `kind`, the float32 the oracle sees)."""
    raw = harness.frames(W, H, L, seed=seed)
    pairs = [harness.ingest(r, kind) for r in raw]
    codes = np.stack([p[0] for p in pairs])
    if kind == "d16":
        codes = codes.view(np.int16)
    elif kind == "d24s8":
        codes = codes.view(np.int32)
    return codes, np.stack([p[1] for p in pairs])


def _as_input(torch, t, kind):
    return t.view(torch.uint16) if kind == "d16" else t


def _oracle(ao, seen, cams=None, **variants):
    """The oracle's AO of `seen` [L, H, W] with the context's (or each layer's) camera."""
    L, H, W = seen.shape
    p = {k: getattr(ao, v) for k, v in harness.PARAMS.items()}
    return np.stack([harness.oracle(W, H, camera=(cams[l] if cams else ao.camera), threads=8, **p, **variants).run(seen[l])
                     for l in range(L)])


def _warm_up(torch, fn):
    """torch's documented warm-up before torch.cuda.graph: the calls once, on a side stream."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()


def _layer_cameras(W, H, L):
    from miniengineao_b200 import Camera
    return [Camera(W, H, fieldOfView=35.0 + 9.0 * l, nearClipPlane=0.05 + 0.1 * l, farClipPlane=60.0 + 150.0 * l) for l in range(L)]


CASES = {
    "tight": dict(),
    "pitched": dict(pitched=True),
    "layered6_cameras": dict(layers=6),
    "d16": dict(kind="d16"),
    "d24s8": dict(kind="d24s8"),
    "hq15": dict(variants=dict(high_quality_mask=15)),
    "single_scale": dict(variants=dict(single_scale=True)),
    "exhaustive": dict(variants=dict(sample_exhaustively=True)),
    "no_graph": dict(use_graph=False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_torch_graph_of_a_frame(torch_cuda, case):
    torch = torch_cuda
    cfg = CASES[case]
    kind, L, variants = cfg.get("kind", "f32"), cfg.get("layers", 1), cfg.get("variants", {})
    W, H = (256, 144) if L > 1 else (400, 232)
    cams = _layer_cameras(W, H, L) if L > 1 else None
    kw = dict(device=0, layers=L, layer_cameras=cams, use_graph=cfg.get("use_graph", True), intensity=1.1, **variants)
    ao, fresh = harness.context(W, H, **kw), harness.context(W, H, **kw)
    shape = (L, H, W) if L > 1 else (H, W)
    dt = getattr(torch, TORCH_DTYPE[kind])
    if cfg.get("pitched"):
        backing = torch.zeros((H + 7, W + 24), dtype=dt, device="cuda")
        out_backing = torch.zeros((H + 3, W + 40), dtype=torch.uint8, device="cuda")
        static, out = backing[3:3 + H, 5:5 + W], out_backing[:H, 8:8 + W]
    else:
        static, out = torch.zeros(shape, dtype=dt, device="cuda"), torch.empty(shape, dtype=torch.uint8, device="cuda")
    inp = _as_input(torch, static, kind)
    _warm_up(torch, lambda: ao.render(inp, out))
    launches, inst = ao.launch_count, ao.reservation()["graph_instantiations"]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ao.render(inp, out)
    assert ao.launch_count - launches == ao.kernels_per_frame, "a recorded frame counts its kernels once"
    assert ao.reservation()["graph_instantiations"] == inst, "the context instantiated a graph during the caller's capture"
    gen = ao.frame_generation
    for i in range(REPLAYS):
        d, seen = _depth(kind, W, H, L, seed=i + 1)
        d = d.reshape(shape)
        static.copy_(torch.from_numpy(d))
        g.replay()
        got = out.cpu().numpy().reshape(L, H, W)
        assert harness.n_diff(got, _oracle(ao, seen, cams, **variants)) == 0, f"{case}: replay {i} differs from the oracle"
        eager = fresh.render(_as_input(torch, torch.from_numpy(d).cuda(), kind)).cpu().numpy().reshape(L, H, W)
        assert harness.n_diff(got, eager) == 0, f"{case}: replay {i} differs from an eager frame of a fresh context"
    assert ao.launch_count - launches == ao.kernels_per_frame, "replays are invisible to the library"
    assert ao.frame_generation == gen
    for a in (ao, fresh):
        a.close()


@pytest.mark.parametrize("shape,kind", [("2d", "f32"), ("layered", "d16")])
def test_torch_graph_of_an_array_frame(torch_cuda, rt, shape, kind):
    torch = torch_cuda
    W, H = 320, 184
    L = 3 if shape == "layered" else 1
    ao, fresh = harness.context(W, H, device=0, layers=L), harness.context(W, H, device=0, layers=L)
    da = Array(rt, W, H, np.float32 if kind == "f32" else np.uint16, shape=shape, layers=L)
    aa = Array(rt, W, H, np.uint8, shape=shape, layers=L)
    da.fill(_depth(kind, W, H, L, seed=0)[0].view(np.uint16 if kind == "d16" else np.float32))
    ak = "raw_f32" if kind == "f32" else "d16"
    _warm_up(torch, lambda: ao.render_arrays(da.handle, aa.handle, kind=ak))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ao.render_arrays(da.handle, aa.handle, kind=ak)
    for i in range(REPLAYS):
        d, seen = _depth(kind, W, H, L, seed=i + 1)
        da.fill(d.view(np.uint16 if kind == "d16" else np.float32))
        g.replay()
        torch.cuda.synchronize()
        got = aa.read()
        assert harness.n_diff(got, _oracle(ao, seen)) == 0, f"replay {i} differs from the oracle"
        eager = fresh.render(_as_input(torch, torch.from_numpy(d.reshape((L, H, W) if L > 1 else (H, W))).cuda(), kind))
        assert harness.n_diff(got, eager.cpu().numpy().reshape(L, H, W)) == 0, f"replay {i} differs from a fresh context"
    del g
    torch.cuda.synchronize()
    for a in (da, aa):
        ao.release_array(a.handle)
        a.free()
    ao.close()
    fresh.close()


def test_one_graph_two_contexts_a_torch_op_and_a_composite(torch_cuda):
    """depth -> (a torch op) -> AO of two contexts -> both composited into one colour target, captured as ONE torch graph; every
    replay equals the same sequence run eagerly on fresh contexts."""
    torch = torch_cuda
    W, H = 480, 272

    def contexts():
        return harness.context(W, H, device=0, intensity=1.1), harness.context(W, H, device=0, intensity=0.6, high_quality_mask=8)

    def sequence(a, b, inp, oa, ob, color):
        d = torch.flip(inp, dims=[1]).contiguous()
        a.render(d, oa)
        b.render(d, ob)
        a.composite_framebuffer(oa, color)
        b.composite_framebuffer(ob, color)

    a, b = contexts()
    inp = torch.zeros((H, W), device="cuda")
    oa, ob = torch.empty((H, W), dtype=torch.uint8, device="cuda"), torch.empty((H, W), dtype=torch.uint8, device="cuda")
    color0 = torch.randint(0, 256, (H, W, 4), dtype=torch.uint8, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    color = color0.clone()
    _warm_up(torch, lambda: sequence(a, b, inp, oa, ob, color))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sequence(a, b, inp, oa, ob, color)
    ea, eb = contexts()
    for i in range(4):
        d = torch.from_numpy(harness.frames(W, H, 1, seed=i + 2)[0]).cuda()
        inp.copy_(d)
        color.copy_(color0)
        g.replay()
        got = (oa.cpu().numpy(), ob.cpu().numpy(), color.cpu().numpy())
        ra, rb, rc = torch.empty_like(oa), torch.empty_like(ob), color0.clone()
        sequence(ea, eb, d, ra, rb, rc)
        ref = (ra.cpu().numpy(), rb.cpu().numpy(), rc.cpu().numpy())
        for name, x, y in zip(("AO a", "AO b", "colour"), got, ref):
            assert np.array_equal(x, y), f"replay {i}: {name} differs from the eager sequence"
    for x in (a, b, ea, eb):
        x.close()


CAPTURE_MODES = {"global": 0, "thread_local": 1, "relaxed": 2}


def _typed_runtime():
    r = runtime()
    P = C.c_void_p
    r.cudaStreamCreateWithFlags.argtypes = [C.POINTER(P), C.c_uint]
    r.cudaStreamBeginCapture.argtypes = [P, C.c_int]
    r.cudaStreamEndCapture.argtypes = [P, C.POINTER(P)]
    r.cudaGraphGetNodes.argtypes = [P, C.POINTER(P), C.POINTER(C.c_size_t)]
    r.cudaGraphNodeGetType.argtypes = [P, C.POINTER(C.c_int)]
    r.cudaGraphInstantiate.argtypes = [C.POINTER(P), P, C.c_ulonglong]
    r.cudaGraphLaunch.argtypes = [P, P]
    for f in ("cudaStreamSynchronize", "cudaGraphExecDestroy", "cudaGraphDestroy", "cudaStreamDestroy"):
        getattr(r, f).argtypes = [P]
    return r


@pytest.mark.parametrize("mode", list(CAPTURE_MODES))
def test_raw_capture_holds_the_frames_kernels(torch_cuda, mode):
    """An engine's own cudaStreamBeginCapture: two frames recorded into it are 2 x meao_kernels_per_frame kernel nodes, and the
    instantiated graph renders what the oracle does."""
    torch = torch_cuda
    from miniengineao_b200 import _native as N
    r, lib = _typed_runtime(), N.lib()
    W, H = 400, 232
    ao = harness.context(W, H, device=0, high_quality_mask=5)
    d, _ = _depth("f32", W, H, 1, seed=4)
    dd = torch.from_numpy(d[0]).cuda()
    outs = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(2)]
    ao.render(dd, outs[0])
    torch.cuda.synchronize()
    outs[0].zero_()
    torch.cuda.synchronize()
    s, graph, exe = C.c_void_p(), C.c_void_p(), C.c_void_p()
    assert r.cudaStreamCreateWithFlags(C.byref(s), 1) == 0
    assert r.cudaStreamBeginCapture(s, CAPTURE_MODES[mode]) == 0
    for o in outs:
        assert lib.meao_render(ao._ctx, C.c_void_p(dd.data_ptr()), 0, C.c_void_p(o.data_ptr()), s) == 0, lib.meao_last_error(ao._ctx)
    assert r.cudaStreamEndCapture(s, C.byref(graph)) == 0
    n = C.c_size_t(0)
    assert r.cudaGraphGetNodes(graph, None, C.byref(n)) == 0
    nodes = (C.c_void_p * n.value)()
    assert r.cudaGraphGetNodes(graph, nodes, C.byref(n)) == 0
    types = []
    for i in range(n.value):
        t = C.c_int()
        assert r.cudaGraphNodeGetType(C.c_void_p(nodes[i]), C.byref(t)) == 0
        types.append(t.value)
    assert types.count(0) == 2 * ao.kernels_per_frame, f"{mode}: node types {types}"           # 0: cudaGraphNodeTypeKernel
    assert r.cudaGraphInstantiate(C.byref(exe), graph, 0) == 0
    assert r.cudaGraphLaunch(exe, s) == 0 and r.cudaStreamSynchronize(s) == 0
    ref = harness.oracle(W, H, camera=ao.camera, threads=8, high_quality_mask=5).run(d[0])
    for o in outs:
        assert harness.n_diff(o.cpu().numpy(), ref) == 0, mode
    for f, h in (("cudaGraphExecDestroy", exe), ("cudaGraphDestroy", graph), ("cudaStreamDestroy", s)):
        assert getattr(r, f)(h) == 0
    ao.close()


def test_refusals_leave_the_capture_valid(torch_cuda, rt):
    """A variant change, a camera change and a never-used array inside the capture are refused with MEAO_ERR_INVALID, profiling is
    refused with MEAO_ERR_UNSUPPORTED, and the capture still ends and replays the frames that were recorded."""
    torch = torch_cuda
    from miniengineao_b200 import MeaoError
    from miniengineao_b200 import _native as N
    W, H = 320, 184
    ao, cv, cc, ca = (harness.context(W, H, device=0) for _ in range(4))
    d, seen = _depth("f32", W, H, 1, seed=5)
    dd = torch.from_numpy(d[0]).cuda()
    out, scratch = torch.empty((H, W), dtype=torch.uint8, device="cuda"), torch.empty((H, W), dtype=torch.uint8, device="cuda")
    da, aa, never = Array(rt, W, H, np.float32), Array(rt, W, H, np.uint8), Array(rt, W, H, np.uint8)
    da.fill(d[0])

    def warm():
        for x in (ao, cv, cc):
            x.render(dd, scratch)
        ca.render_arrays(da.handle, aa.handle)
    _warm_up(torch, warm)
    g = torch.cuda.CUDAGraph()
    errors = {}
    with torch.cuda.graph(g):
        ao.render(dd, out)
        cv.sampleExhaustively = True
        cc.camera.fieldOfView = 75.0
        for name, call in (("variant", lambda: cv.render(dd, scratch)), ("camera", lambda: cc.render(dd, scratch)),
                           ("array", lambda: ca.render_arrays(da.handle, never.handle))):
            with pytest.raises(MeaoError) as e:
                call()
            errors[name] = (e.value.code, str(e.value))
        ms = (C.c_float * 16)()
        errors["profile"] = (N.lib().meao_profile_frame(ao._ctx, C.c_void_p(dd.data_ptr()), 0, C.c_void_p(scratch.data_ptr()), ms, None, 16),
                             N.lib().meao_last_error(ao._ctx).decode())
    for name in ("variant", "camera", "array"):
        assert errors[name][0] == N.MEAO_ERR_INVALID and "outside the capture" in errors[name][1], (name, errors[name])
    assert errors["profile"][0] == N.MEAO_ERR_UNSUPPORTED, errors["profile"]
    out.zero_()
    g.replay()
    assert harness.n_diff(out.cpu().numpy(), _oracle(ao, seen)[0]) == 0, "the capture holds the frame recorded before the refusals"
    # outside the capture the refused calls go through, as the message says
    cv.render(dd, scratch)
    cc.render(dd, scratch)
    ca.render_arrays(da.handle, never.handle)
    torch.cuda.synchronize()
    del g
    for a in (da, aa, never):
        ca.release_array(a.handle)
        a.free()
    for x in (ao, cv, cc, ca):
        x.close()


def test_generation_tells_when_to_capture_again(torch_cuda):
    torch = torch_cuda
    W, H = 400, 232
    ao = harness.context(W, H, device=0)
    d, seen = _depth("f32", W, H, 1, seed=6)
    dd = torch.from_numpy(d[0]).cuda()
    out = torch.empty((H, W), dtype=torch.uint8, device="cuda")

    def capture():
        _warm_up(torch, lambda: ao.render(dd, out))
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ao.render(dd, out)
        return g, ao.frame_generation

    g1, gen1 = capture()
    ref1 = _oracle(ao, seen)[0]
    for _ in range(3):
        out.zero_()
        g1.replay()
        assert harness.n_diff(out.cpu().numpy(), ref1) == 0
    ao.intensity = ao.intensity                                         # setters that change nothing
    ao.camera.fieldOfView = ao.camera.fieldOfView
    ao.LateUpdate()
    assert ao.frame_generation == gen1
    ao.camera.fieldOfView = 75.0                                        # a camera change outside the graph
    ao.LateUpdate()
    assert ao.frame_generation != gen1
    g2, gen2 = capture()
    ref2 = _oracle(ao, seen)[0]
    assert harness.n_diff(ref1, ref2) > 0, "the new camera changes the AO"
    out.zero_()
    g2.replay()
    assert harness.n_diff(out.cpu().numpy(), ref2) == 0, "the re-capture renders the new camera"
    assert ao.frame_generation == gen2
    del g1, g2
    ao.close()


def test_row_band_steps_in_their_own_graphs(torch_cuda):
    """Two connected row bands on one device, each meao_band_step recorded into its own torch graph and the graphs replayed in lock
    step: the union of the bands equals the oracle's whole frame every time."""
    torch = torch_cuda
    W, H, bands = 1280, 720, 2
    cuts, ctxs, streams = native_bands(torch, W, H, bands)
    bufs = [torch.zeros((cuts[i + 1] - cuts[i], W), device="cuda") for i in range(bands)]
    outs = [torch.zeros((cuts[i + 1] - cuts[i], W), dtype=torch.uint8, device="cuda") for i in range(bands)]
    for i, a in enumerate(ctxs):                                        # the warm-up step, on every band
        a.band_step(bufs[i], outs[i], stream=streams[i])
    torch.cuda.synchronize()
    graphs = []
    for i, a in enumerate(ctxs):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=streams[i]):
            a.band_step(bufs[i], outs[i])
        graphs.append(g)
    for frame in range(4):
        depth = harness.frames(W, H, 1, seed=frame + 7)[0]
        for i in range(bands):
            bufs[i].copy_(torch.from_numpy(np.ascontiguousarray(depth[cuts[i]:cuts[i + 1]])))
        torch.cuda.synchronize()
        for i, g in enumerate(graphs):
            with torch.cuda.stream(streams[i]):
                g.replay()
        torch.cuda.synchronize()
        assert [a.band_status()["error"] for a in ctxs] == [0] * bands, "a neighbour exchange timed out"
        got = np.concatenate([o.cpu().numpy() for o in outs], axis=0)
        ref = harness.oracle(W, H, camera=ctxs[0].camera, threads=8).run(depth)
        assert harness.n_diff(got, ref) == 0, f"frame {frame}: the bands differ from the oracle's whole frame"
    del graphs
    torch.cuda.synchronize()
    for a in ctxs:
        a.close()
