"""GPU tests of dynamic resolution (meao_reserve) on the H100: a reserved context walks a schedule of ragged sizes inside one arena and
must give, at every size, the AO and every debug buffer of a fresh context of that size and of the oracle -- after a hostile max-size
frame has left NaNs and infinities in the arena -- while a size change allocates nothing, synchronises nothing and keeps the graphs of
the other sizes.  Also: stream-ordered camera tables under a backlog, the real host flows (a plugin event bound once to max-size
pitched targets, Python views, layered frames, CUDA arrays, host buffers, the stage API) and the bound on executable graphs."""
import ctypes as C

import numpy as np
import pytest

import hostile_cases as HC
from test_arrays_gpu import Array, rt, torch_cuda  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

MAX = (3840, 2160)
SCHEDULE = [(3840, 2160), (3456, 1944), (2881, 1621), (1, 1), (17, 9), (1920, 1080), (3840, 2160), (2881, 1621)]
SLEEP_CYCLES = 1 << 30          # about half a second of one spinning thread at the H100's clock: a backlog the host cannot outrun


def _camera(W, H, **kw):
    """A camera whose projection does not follow its pixel size, as under an engine's dynamic resolution, which scales the viewport
    and keeps the projection: a size change then changes no plan input, and the context never re-plans."""
    from miniengineao_b200 import Camera

    class DrsCamera(Camera):
        @property
        def projection00(self) -> float:
            return Camera(*MAX, fieldOfView=self.fieldOfView).projection00

    return DrsCamera(W, H, **kw)


def _ao(W, H, max_res=None, layers=1, cams=None, use_graph=True):
    from miniengineao_b200 import AmbientOcclusion
    ao = AmbientOcclusion(_camera(W, H), device=0, use_graph=use_graph)
    ao.maxResolution = max_res
    ao.layers = layers
    ao.layerCameras = cams
    return ao


def _size(ao, W, H):
    ao.camera.pixelWidth, ao.camera.pixelHeight = W, H
    if ao.layerCameras:
        for c in ao.layerCameras:
            c.pixelWidth, c.pixelHeight = W, H


def _depth(W, H, frame=0, L=1):
    from miniengineao_b200 import synth
    d = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=frame + l)).astype(np.float32) for l in range(L)])
    return d if L > 1 else d[0]


def _oracle(cam, depth):
    from oracle.oracle import Oracle
    H, W = depth.shape
    orc = Oracle(W, H, threads=8, **HC.oracle_camera_kw(cam))
    return orc, orc.run(depth)


def _fresh(torch, W, H, depth, layers=1, cams=None):
    f = _ao(W, H, layers=layers, cams=cams)
    ao = f.render(torch.from_numpy(np.ascontiguousarray(depth)).cuda()).cpu().numpy()
    bufs = {bid: f.debug_buffer(bid) for bid in HC.buffer_ids()}
    f.close()
    return ao, bufs


def _res(ao):
    return ao.reservation()


def test_parity_over_a_drs_schedule_after_a_hostile_frame(torch_cuda):
    torch = torch_cuda
    ao = _ao(*MAX, max_res=MAX)
    hostile = HC.hostile_raw(*MAX, ao.zbuffer_params(), True, seed=5)
    ao.render(torch.from_numpy(hostile).cuda())                         # stale NaNs, infinities and subnormals everywhere
    allocs = _res(ao)["arena_allocations"]
    for i, (W, H) in enumerate(SCHEDULE):
        _size(ao, W, H)
        d = _depth(W, H, frame=i)
        got = ao.render(torch.from_numpy(d).cuda()).cpu().numpy()
        ref_ao, ref_bufs = _fresh(torch, W, H, d)
        assert HC.n_diff(got, ref_ao) == 0, f"{W}x{H}: AO differs from a fresh context"
        for bid in HC.buffer_ids():
            assert HC.n_diff(ao.debug_buffer(bid), ref_bufs[bid]) == 0, f"{W}x{H}: buffer {bid} differs from a fresh context"
        orc, ref = _oracle(ao.camera, d)
        assert HC.n_diff(got, ref) == 0, f"{W}x{H}: AO differs from the oracle"
        HC.compare_buffers(ao.debug_buffer, orc, f"{W}x{H}", HC.buffer_ids())
    assert _res(ao)["arena_allocations"] == allocs
    ao.close()


def _backlog(torch, s, ao, d, out, n=50):
    """A spinning kernel, then n frames at the current size into `out`, then an event E, all on stream s: E completes half a second
    from now."""
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    for _ in range(n):
        ao.render(d, out, stream=s)
    e = torch.cuda.Event()
    e.record(s)
    return e


def test_resize_does_not_synchronise(torch_cuda):
    torch = torch_cuda
    s = torch.cuda.Stream()
    A, B, NEW = MAX, (2881, 1621), (1921, 1081)
    dev = {sz: torch.from_numpy(_depth(*sz)).cuda() for sz in (A, B, NEW)}
    out = {sz: torch.empty((sz[1], sz[0]), dtype=torch.uint8, device="cuda") for sz in (A, B, NEW)}
    ao = _ao(*A, max_res=MAX)
    for sz in (A, B, A):
        _size(ao, *sz)
        ao.render(dev[sz], out[sz], stream=s)
    torch.cuda.synchronize()
    r0 = _res(ao)
    # a cached size: a plain replay
    e = _backlog(torch, s, ao, dev[A], out[A])
    _size(ao, *B)
    ao.render(dev[B], out[B], stream=s)
    assert not e.query(), "a resize to a cached size waited for the GPU"
    torch.cuda.synchronize()
    r1 = _res(ao)
    assert r1["graph_instantiations"] == r0["graph_instantiations"] and r1["arena_allocations"] == r0["arena_allocations"]
    # a size never seen: planned, tables written in stream order, graph captured -- still no wait
    _size(ao, *A)
    e = _backlog(torch, s, ao, dev[A], out[A])
    _size(ao, *NEW)
    ao.render(dev[NEW], out[NEW], stream=s)
    assert not e.query(), "a resize to a new size waited for the GPU"
    torch.cuda.synchronize()
    r2 = _res(ao)
    assert r2["arena_allocations"] == r0["arena_allocations"] and r2["graph_instantiations"] == r1["graph_instantiations"] + 1
    ao.close()
    # the same steps on an unreserved context DO wait: the test observes what it claims
    u = _ao(*A)
    u.render(dev[A], out[A], stream=s)
    torch.cuda.synchronize()
    e = _backlog(torch, s, u, dev[A], out[A])
    _size(u, *B)
    u.render(dev[B], out[B], stream=s)
    assert e.query(), "an unreserved resize is expected to drain the GPU"
    torch.cuda.synchronize()
    u.close()


def test_stream_ordered_tables_with_layer_cameras(torch_cuda):
    """Frames at sizes that recycle camera table slots, enqueued behind a backlog on one stream with no host synchronise."""
    torch = torch_cuda
    L, M = 2, (1280, 720)
    cams = [_camera(*M, nearClipPlane=0.1, farClipPlane=50.0, fieldOfView=40.0), _camera(*M, nearClipPlane=1.0, farClipPlane=1000.0, fieldOfView=90.0)]
    ao = _ao(*M, max_res=M, layers=L, cams=cams)
    sizes = [(1280 - 37 * i, 720 - 23 * i) for i in range(8)]           # fills every slot
    for sz in sizes:
        _size(ao, *sz)
        ao.render(torch.from_numpy(_depth(*sz, L=L)).cuda())
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
    order = [sizes[0], (999, 555), sizes[1], (999, 555), sizes[0], (1, 1), (401, 233)]    # A, C(new), B(evicted), C, A, ...
    outs = []
    for i, sz in enumerate(order):
        _size(ao, *sz)
        d = _depth(*sz, frame=i, L=L)
        dev = torch.from_numpy(d).cuda()                                # kept alive until stream s has read it
        outs.append((sz, d, dev, ao.render(dev, stream=s)))
    torch.cuda.synchronize()
    for sz, d, _, out in outs:
        fresh_cams = [_camera(*sz, nearClipPlane=c.nearClipPlane, farClipPlane=c.farClipPlane, fieldOfView=c.fieldOfView) for c in cams]
        ref, _ = _fresh(torch, *sz, d, layers=L, cams=fresh_cams)
        assert HC.n_diff(out.cpu().numpy(), ref) == 0, f"{sz}: a stream-ordered frame differs from a fresh context"
    ao.close()


def _event_fn():
    from miniengineao_b200 import _native as N
    return N.lib().meao_render_event


@pytest.mark.parametrize("layers", [1, 2, 6])
def test_event_bound_once_to_max_size_pitched_targets(torch_cuda, layers):
    torch = torch_cuda
    M = (1920, 1080)
    rtd = torch.full((layers, M[1], M[0]), float("nan"), device="cuda")
    rta = torch.zeros((layers, M[1], M[0]), dtype=torch.uint8, device="cuda")
    ao = _ao(*M, max_res=M, layers=layers)
    ao.LateUpdate()
    lib = ao._lib
    rp, lp = M[0] * 4, M[0] * M[1] * 4
    s = torch.cuda.current_stream()
    assert lib.meao_bind_event_pitched(ao._ctx, 77, C.c_void_p(rtd.data_ptr()), rp, lp, 0, C.c_void_p(rta.data_ptr()), M[0], M[0] * M[1],
                                       C.c_void_p(s.cuda_stream)) == 0
    allocs = _res(ao)["arena_allocations"]
    for i, (W, H) in enumerate([(1920, 1080), (1537, 865), (999, 17), (1920, 1080), (1537, 865)]):
        _size(ao, W, H)
        ao.LateUpdate()
        d = _depth(W, H, frame=i, L=layers).reshape(layers, H, W)
        rtd[:, :H, :W].copy_(torch.from_numpy(d))
        _event_fn()(77)
        ref, _ = _fresh(torch, W, H, d if layers > 1 else d[0], layers=layers)
        got = rta[:, :H, :W].cpu().numpy()
        assert HC.n_diff(got.reshape(ref.shape), ref) == 0, f"event frame at {W}x{H} differs"
    assert _res(ao)["arena_allocations"] == allocs
    lib.meao_bind_event(ao._ctx, 77, None, 0, None, None)
    ao.close()


def test_python_views_of_a_max_size_target(torch_cuda):
    torch = torch_cuda
    M = (1600, 900)
    rtd = torch.zeros((M[1], M[0]), device="cuda")
    out = torch.full((M[1], M[0]), 0xA5, dtype=torch.uint8, device="cuda")
    ao = _ao(*M, max_res=M)
    for i, (W, H) in enumerate([(1600, 900), (1201, 677), (1600, 900), (641, 361)]):
        _size(ao, W, H)
        d = _depth(W, H, frame=i)
        rtd[:H, :W].copy_(torch.from_numpy(d))
        ao.render(rtd[:H, :W], out[:H, :W])
        ref, _ = _fresh(torch, W, H, d)
        assert HC.n_diff(out[:H, :W].cpu().numpy(), ref) == 0, (W, H)
    assert int((out[:, 1600:] != 0xA5).sum()) == 0
    ao.close()


def test_array_frames_alternating_between_two_sizes(torch_cuda, rt):
    torch = torch_cuda
    M = (1024, 768)
    ao = _ao(*M, max_res=M)
    pairs = {sz: (Array(rt, *sz, np.float32), Array(rt, *sz, np.uint8)) for sz in ((1024, 768), (777, 431))}
    for i, sz in enumerate([(1024, 768), (777, 431), (1024, 768), (777, 431)]):
        _size(ao, *sz)
        d = _depth(*sz, frame=i)
        da, aa = pairs[sz]
        da.fill(d)
        ao.render_arrays(da.handle, aa.handle)
        torch.cuda.synchronize()
        ref, _ = _fresh(torch, *sz, d)
        assert HC.n_diff(aa.read()[0], ref) == 0, sz
    for da, aa in pairs.values():
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()
    ao.close()


def test_host_buffers_and_stage_api_across_size_changes(torch_cuda):
    torch = torch_cuda
    M = (960, 540)
    ao = _ao(*M, max_res=M)
    lib = ao._lib
    sizes = [(960, 540), (733, 411), (960, 540), (505, 301)]
    depths = [_depth(*sz, frame=i) for i, sz in enumerate(sizes)]
    outs = [np.empty((sz[1], sz[0]), np.uint8) for sz in sizes]
    for i, sz in enumerate(sizes):                                      # render_host_async, both slots, a size change per frame
        _size(ao, *sz)
        ao.LateUpdate()
        if i >= 2:
            assert lib.meao_host_wait(ao._ctx, i & 1) == 0
        assert lib.meao_render_host_async(ao._ctx, depths[i].ctypes.data, 0, outs[i].ctypes.data, i & 1) == 0
    assert lib.meao_host_wait(ao._ctx, 0) == 0 and lib.meao_host_wait(ao._ctx, 1) == 0
    for sz, d, o in zip(sizes, depths, outs):
        assert HC.n_diff(o, _fresh(torch, *sz, d)[0]) == 0, sz
    _size(ao, 612, 333)                                                 # render_host at a new size
    d = _depth(612, 333, frame=9)
    assert HC.n_diff(ao.render_host(d), _fresh(torch, 612, 333, d)[0]) == 0
    _size(ao, 555, 222)                                                 # the stage API at a new size
    d = _depth(555, 222, frame=10)
    ao.stage_downsample(torch.from_numpy(d).cuda())
    for k in range(1, 5):
        ao.stage_render(k)
    for lo in range(4, 0, -1):
        ao.stage_upsample(lo)
    torch.cuda.synchronize()
    orc, ref = _oracle(ao.camera, d)
    HC.compare_buffers(ao.debug_buffer, orc, "stage API at 555x222", HC.buffer_ids())
    ao.close()


def test_graphs_stay_bounded_over_200_distinct_sizes(torch_cuda):
    from miniengineao_b200 import _native as N
    torch = torch_cuda
    M = (1024, 576)
    ao = _ao(*M, max_res=M)
    ao.LateUpdate()
    allocs = _res(ao)["arena_allocations"]
    held = []
    for i in range(200):
        W, H = 1024 - 4 * i - (i % 3), 576 - 2 * i - (i % 5)
        _size(ao, W, H)
        d = _depth(W, H, frame=i)
        got = ao.render(torch.from_numpy(d).cuda())
        held.append(_res(ao)["graphs_held"])
        if i % 40 == 7:
            _, ref = _oracle(ao.camera, d)
            assert HC.n_diff(got.cpu().numpy(), ref) == 0, (W, H)
    r = _res(ao)
    assert max(held) <= N.MEAO_MAX_GRAPHS_HELD, max(held)
    assert r["arena_allocations"] == allocs
    ao.close()


def test_param_change_on_a_reserved_context_keeps_the_arena(torch_cuda):
    from oracle.oracle import Oracle
    torch = torch_cuda
    M = (1280, 720)
    ao = _ao(*M, max_res=M)
    for i, sz in enumerate([(1280, 720), (1001, 555)]):
        _size(ao, *sz)
        ao.render(torch.from_numpy(_depth(*sz, frame=i)).cuda())
    allocs = _res(ao)["arena_allocations"]
    ao.intensity, ao.blurTolerance = 1.6, -3.0
    for i, sz in enumerate([(1280, 720), (1001, 555), (700, 400)]):
        _size(ao, *sz)
        d = _depth(*sz, frame=5 + i)
        got = ao.render(torch.from_numpy(d).cuda()).cpu().numpy()
        ref = Oracle(sz[0], sz[1], threads=8, intensity=1.6, blur_tolerance=-3.0, **HC.oracle_camera_kw(ao.camera)).run(d)
        assert HC.n_diff(got, ref) == 0, sz
    assert _res(ao)["arena_allocations"] == allocs
    ao.close()
