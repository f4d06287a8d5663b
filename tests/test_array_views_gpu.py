"""GPU tests of CUDA-array viewports (meao_render_arrays_at, meao_bind_event_arrays_at) on the H100: the frame read from a W x H
rectangle of a larger depth array and written into one of a larger AO array.  Inside the AO viewport the bytes must be the oracle's
and meao_render's on a tight copy of the depth; outside it every byte keeps its sentinel, and poisoned depth texels outside the depth
viewport change nothing.  Also: a reserved context walking many sizes inside one max-size array pair, by call and by a plugin event
bound once; two split-screen contexts sharing one array pair; a viewport frame recorded into torch.cuda.graph; every refusal."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, rt, torch_cuda  # noqa: F401  (the fixtures)

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
KINDS = {"raw_f32": np.float32, "linear_f32": np.float32, "d16": np.uint16}


def _poisoned(shape, dtype):
    """NaN, +inf, -inf and 0 in turn (float32), 0 and 65535 (D16 codes)"""
    vals = np.array([np.nan, np.inf, -np.inf, 0.0], np.float32) if np.dtype(dtype) == np.float32 else np.array([0, 65535], np.uint16)
    return np.resize(vals, int(np.prod(shape))).reshape(shape)


def _depth(kind, W, H, L, seed=0):
    """(the depth in the array's format, the float32 the oracle sees) of L layers"""
    raw = harness.frames(W, H, L, seed=seed)
    if kind == "d16":
        return harness.ingest(raw, "d16")
    if kind == "linear_f32":
        from miniengineao_b200 import synth
        lin = np.stack([synth.random_depth(W, H, seed=seed + i) for i in range(L)]).astype(np.float32)
        return lin, lin
    return raw, raw


def _embed(depth, ext, origin):
    """the whole host image of a depth array of extent ext = (w, h): poison, with `depth` at origin"""
    L, H, W = depth.shape
    (w, h), (x, y) = ext, origin
    full = _poisoned((L, h, w), depth.dtype)
    full[:, y:y + H, x:x + W] = depth
    return full


def _check_ao(got, ref, origin, tag):
    """got: the whole AO array [L, h, w]; ref: [L, H, W] expected inside the viewport at origin; sentinel everywhere else"""
    L, H, W = ref.shape
    x, y = origin
    assert harness.n_diff(got[:, y:y + H, x:x + W], ref) == 0, f"{tag}: the viewport differs"
    outside = np.ones(got.shape, bool)
    outside[:, y:y + H, x:x + W] = False
    assert (got[outside] == SENTINEL).all(), f"{tag}: a byte outside the viewport changed"


def _ext(shape, w, h):
    """an array extent of at least w x h; square for a cube map, whose faces are"""
    return (max(w, h),) * 2 if shape == "cube" else (w, h)


def _release(ao, *arrays):
    for a in arrays:
        ao.release_array(a.handle)
        a.free()


# ---- 1. parity -------------------------------------------------------------------------------------------------------------------
CASES = [(83, 61, 1, "2d"), (130, 70, 2, "layered"), (61, 61, 6, "cube")]


@pytest.mark.parametrize("hq", [0, 1])
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("W,H,L,shape", CASES)
def test_viewport_parity(torch_cuda, rt, W, H, L, shape, kind, hq):
    torch = torch_cuda
    depth, as_float = _depth(kind, W, H, L, seed=W + L)
    linear = kind == "linear_f32"
    dext, dorg, aext, aorg = _ext(shape, W + 37, H + 19), (29, 11), _ext(shape, W + 9, H + 40), (5, 33)
    ao = harness.context(W, H, device=0, layers=L, high_quality_mask=hq)
    tight = ao.render(torch.from_numpy(np.ascontiguousarray(depth if L > 1 else depth[0])).cuda(), linear=linear).cpu().numpy()
    tight = tight.reshape(L, H, W)
    da, aa = Array(rt, *dext, depth.dtype, shape, L), Array(rt, *aext, np.uint8, shape, L)
    try:
        da.fill(_embed(depth, dext, dorg))
        aa.fill(np.full((aa.layers, aext[1], aext[0]), SENTINEL, np.uint8))
        before = ao.launch_count
        ao.render_arrays(da.handle, aa.handle, kind=kind, depth_origin=dorg, ao_origin=aorg)
        assert ao.launch_count - before == ao.kernels_per_frame
        torch.cuda.synchronize()
        got = aa.read()
        tag = f"{W}x{H} L={L} {kind} hq={hq}"
        _check_ao(got, tight, aorg, tag + " vs meao_render")
        ref = np.stack([harness.oracle(W, H, linear=linear, threads=8, high_quality_mask=hq).run(as_float[l]) for l in range(L)])
        _check_ao(got, ref, aorg, tag + " vs the oracle")
        assert np.array_equal(ao.debug_buffer(17).reshape(L, H, W), ref)         # id 17 regenerated as after an array frame
    finally:
        _release(ao, da, aa)
        ao.close()


# ---- 2. dynamic resolution inside one max-size pair -----------------------------------------------------------------------------
MAX = (1024, 576)
SCHEDULE = [(1024, 576), (777, 431), (1, 1), (333, 97), (1024, 576), (513, 288), (777, 431), (64, 64), (1000, 575), (333, 97)]


def _drs_camera(W, H):
    """a camera whose projection does not follow its pixel size (an engine's dynamic resolution): a size change is no re-plan"""
    from miniengineao_b200 import Camera

    class DrsCamera(Camera):
        @property
        def projection00(self) -> float:
            return Camera(*MAX, fieldOfView=self.fieldOfView).projection00

    return DrsCamera(W, H)


def test_dynamic_resolution_in_one_max_size_pair(torch_cuda, rt):
    """Every size of the schedule, by meao_render_arrays_at at a centred origin and by an event bound once at (0, 0); one arena,
    no release, every frame the oracle's."""
    torch = torch_cuda
    ao = harness.context(_drs_camera(*MAX), device=0, max_resolution=MAX)
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    da, aa = Array(rt, *MAX, np.float32), Array(rt, *MAX, np.uint8)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    try:
        assert lib.meao_bind_event_arrays_at(ctx, 91, C.c_void_p(da.handle), 0, 0, 0, C.c_void_p(aa.handle), 0, 0, stream) == 0
        allocs = None
        for i, (W, H) in enumerate(SCHEDULE):
            ao.camera.pixelWidth, ao.camera.pixelHeight = W, H
            depth = harness.frames(W, H, 1, seed=i)
            ref = harness.oracle(W, H, camera=ao.camera, threads=8).run(depth[0])[None]
            for by_event in (False, True):
                org = (0, 0) if by_event else ((MAX[0] - W) // 2, (MAX[1] - H) // 3)
                da.fill(_embed(depth, MAX, org))
                aa.fill(np.full((1, MAX[1], MAX[0]), SENTINEL, np.uint8))
                before = ao.launch_count
                if by_event:
                    ao.LateUpdate()
                    lib.meao_get_render_event_func()(91)
                else:
                    ao.render_arrays(da.handle, aa.handle, depth_origin=org, ao_origin=org)
                assert ao.launch_count - before == ao.kernels_per_frame, (W, H, by_event, lib.meao_last_error(ctx))
                torch.cuda.synchronize()
                _check_ao(aa.read(), ref, org, f"{W}x{H} {'event' if by_event else 'call'}")
            allocs = allocs if allocs is not None else ao.reservation()["arena_allocations"]
        r = ao.reservation()
        assert r["arena_allocations"] == allocs == 1, r
        assert lib.meao_bind_event_arrays_at(ctx, 91, None, 0, 0, 0, None, 0, 0, None) == 0
    finally:
        _release(ao, da, aa)
        ao.close()


# ---- 3. split screen -----------------------------------------------------------------------------------------------------------
def test_split_screen_two_contexts_one_array_pair(torch_cuda, rt):
    torch = torch_cuda
    w, H = 481, 270
    W = 2 * w + 3                                   # three columns between the halves that neither player owns
    halves = {"left": (0, harness.frames(w, H, 1, seed=3)), "right": (w + 3, harness.frames(w, H, 1, seed=8))}
    ctxs = {k: harness.context(w, H, device=0, intensity=1.1 if k == "left" else 0.9) for k in halves}
    full = _poisoned((1, H, W), np.float32)
    for x, d in halves.values():
        full[:, :, x:x + w] = d
    da, aa = Array(rt, W, H, np.float32), Array(rt, W, H, np.uint8)
    s = torch.cuda.Stream()
    try:
        da.fill(full)
        aa.fill(np.full((1, H, W), SENTINEL, np.uint8))
        refs = {}
        for k, (x, d) in halves.items():
            refs[k] = ctxs[k].render(torch.from_numpy(d[0]).cuda()).cpu().numpy()[None]
            assert np.array_equal(refs[k][0], harness.oracle(w, H, threads=8, intensity=1.1 if k == "left" else 0.9).run(d[0]))
        ctxs["left"].render_arrays(da.handle, aa.handle, depth_origin=(0, 0), ao_origin=(0, 0), stream=s)
        torch.cuda.synchronize()
        _check_ao(aa.read(), refs["left"], (0, 0), "the left player alone")
        ctxs["right"].render_arrays(da.handle, aa.handle, depth_origin=(w + 3, 0), ao_origin=(w + 3, 0), stream=s)
        ctxs["left"].render_arrays(da.handle, aa.handle, depth_origin=(0, 0), ao_origin=(0, 0), stream=s)
        torch.cuda.synchronize()
        got = aa.read()
        assert harness.n_diff(got[:, :, :w], refs["left"]) == 0 and harness.n_diff(got[:, :, w + 3:], refs["right"]) == 0
        assert (got[:, :, w:w + 3] == SENTINEL).all()
    finally:
        for k, a in ctxs.items():
            a.release_array(da.handle)
            a.release_array(aa.handle)
            a.close()
        da.free()
        aa.free()


# ---- 4. capture ----------------------------------------------------------------------------------------------------------------
def test_torch_graph_of_a_viewport_frame(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 320, 184, 2
    ext, dorg, aorg = (400, 260), (17, 40), (80, 3)
    ao = harness.context(W, H, device=0, layers=L)
    da, aa = Array(rt, *ext, np.float32, "layered", L), Array(rt, *ext, np.uint8, "layered", L)
    try:
        depth, _ = _depth("raw_f32", W, H, L, seed=0)
        da.fill(_embed(depth, ext, dorg))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ao.render_arrays(da.handle, aa.handle, depth_origin=dorg, ao_origin=aorg)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        gen = ao.frame_generation
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ao.render_arrays(da.handle, aa.handle, depth_origin=dorg, ao_origin=aorg)
        assert ao.frame_generation == gen                    # origins are arguments, not plan inputs
        for i in range(3):
            depth, _ = _depth("raw_f32", W, H, L, seed=i + 1)
            da.fill(_embed(depth, ext, dorg))
            aa.fill(np.full((L, ext[1], ext[0]), SENTINEL, np.uint8))
            g.replay()
            torch.cuda.synchronize()
            ref = np.stack([harness.oracle(W, H, threads=8).run(depth[l]) for l in range(L)])
            _check_ao(aa.read(), ref, aorg, f"replay {i}")
        del g
        torch.cuda.synchronize()
    finally:
        _release(ao, da, aa)
        ao.close()


# ---- 5. refusals ---------------------------------------------------------------------------------------------------------------
def test_refusals_launch_nothing(torch_cuda, rt):
    from miniengineao_b200 import _native as N
    W, H = 160, 96
    ext = (200, 120)
    ao = harness.context(W, H, device=0)
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    da, aa = Array(rt, *ext, np.float32), Array(rt, *ext, np.uint8)
    d, a = C.c_void_p(da.handle), C.c_void_p(aa.handle)
    cases = [  # (tag, depth origin, kind, AO origin, status, field named)
        ("negative depth_x", (-1, 0), 0, (0, 0), N.MEAO_ERR_INVALID, b"depth_x"),
        ("negative depth_y", (0, -1), 0, (0, 0), N.MEAO_ERR_INVALID, b"depth_y"),
        ("negative ao_x", (0, 0), 0, (-1, 0), N.MEAO_ERR_INVALID, b"ao_x"),
        ("negative ao_y", (0, 0), 0, (0, -1), N.MEAO_ERR_INVALID, b"ao_y"),
        ("depth width overflow", (41, 0), 0, (0, 0), N.MEAO_ERR_INVALID, b"depth_x"),
        ("depth height overflow", (0, 25), 0, (0, 0), N.MEAO_ERR_INVALID, b"depth_y"),
        ("AO width overflow", (0, 0), 0, (41, 0), N.MEAO_ERR_INVALID, b"ao_x"),
        ("AO height overflow", (0, 0), 0, (0, 25), N.MEAO_ERR_INVALID, b"ao_y"),
        ("D24S8", (0, 0), 3, (0, 0), N.MEAO_ERR_UNSUPPORTED, b"D24S8"),
    ]
    try:
        for tag, (dx, dy), kind, (ax, ay), want, text in cases:
            before = ao.launch_count
            rc = lib.meao_render_arrays_at(ctx, d, dx, dy, kind, a, ax, ay, None)
            assert rc == want and text in lib.meao_last_error(ctx), (tag, rc, lib.meao_last_error(ctx))
            assert ao.launch_count == before, tag
            rc = lib.meao_bind_event_arrays_at(ctx, 5, d, dx, dy, kind, a, ax, ay, None)
            assert rc == want and text in lib.meao_last_error(ctx), (tag, "bind", rc)
        # the viewport that just fits renders; the plain entry point still wants W x H arrays
        assert lib.meao_render_arrays_at(ctx, d, 40, 24, 0, a, 40, 24, None) == 0
        assert lib.meao_render_arrays(ctx, d, 0, a, None) == N.MEAO_ERR_INVALID and b"extent" in lib.meao_last_error(ctx)
        # a row band
        ao.set_row_band(0, 48, -1, 96)
        before = ao.launch_count
        assert lib.meao_render_arrays_at(ctx, d, 0, 0, 0, a, 0, 0, None) == N.MEAO_ERR_UNSUPPORTED
        assert b"row band" in lib.meao_last_error(ctx) and ao.launch_count == before
        ao.set_row_band(0, H, -1, -1)
    finally:
        _release(ao, da, aa)
        ao.close()


def test_bound_event_refuses_a_viewport_that_stopped_fitting(torch_cuda, rt):
    torch = torch_cuda
    M = (200, 120)
    ao = harness.context(_drs_camera(160, 96), device=0, max_resolution=M)
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    da, aa = Array(rt, *M, np.float32), Array(rt, *M, np.uint8)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    try:
        assert lib.meao_bind_event_arrays_at(ctx, 92, C.c_void_p(da.handle), 40, 24, 0, C.c_void_p(aa.handle), 40, 24, stream) == 0
        for W, H, fits in ((160, 96, True), (180, 100, False), (160, 97, False), (150, 90, True)):
            ao.camera.pixelWidth, ao.camera.pixelHeight = W, H
            ao.LateUpdate()
            depth = harness.frames(W, H, 1, seed=W)
            da.fill(_embed(depth, M, (40, 24)) if fits else _poisoned((1, M[1], M[0]), np.float32))
            aa.fill(np.full((1, M[1], M[0]), SENTINEL, np.uint8))
            before = ao.launch_count
            lib.meao_get_render_event_func()(92)
            torch.cuda.synchronize()
            if fits:
                assert ao.launch_count - before == ao.kernels_per_frame, (W, H)
                _check_ao(aa.read(), harness.oracle(W, H, camera=ao.camera, threads=8).run(depth[0])[None], (40, 24), f"{W}x{H}")
            else:
                assert ao.launch_count == before, (W, H)
                assert b"overflows" in lib.meao_last_error(ctx), lib.meao_last_error(ctx)
                assert (aa.read() == SENTINEL).all()
        lib.meao_bind_event_arrays_at(ctx, 92, None, 0, 0, 0, None, 0, 0, None)
    finally:
        _release(ao, da, aa)
        ao.close()
