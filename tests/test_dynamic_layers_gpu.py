"""GPU tests of dynamic view counts (meao_reserve_layers) on the H100: a context with a layer reservation walks a schedule of view
counts, mixed with sizes inside a size reservation, in one arena -- after a hostile frame at the maximum size and layer count has left
NaNs and infinities there -- and every layer must equal a fresh context of that layer count and the oracle, in every frame form
(pointers, pitched views, layered CUDA arrays, both batch calls).  A layer change allocates nothing, synchronises nothing and keeps the
graphs of the other (W, H, L); split-screen players join and leave through the viewport table on shared arrays; refusals launch
nothing; MEAO_FLAG_NO_GRAPH, torch.cuda.graph capture and meao_release_array follow the changing count."""
import ctypes as C

import numpy as np
import pytest

import harness
import hostile_cases as HC
from gpu_harness import Array, backlog, fresh_frame, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import Camera, MeaoError
from miniengineao_b200 import _native as N

pytestmark = pytest.mark.gpu

MAXR, LMAX = (1280, 720), 6
# (L, W, H): counts up and down, sizes inside the size reservation, and returns to (W, H, L) planned before.  LateUpdate sets the count
# before the size, so a step that changes both also plans the (new L, old size) it passes through; with those, the schedule plans 8
# triples, as many as MEAO_SIZE_SLOTS keeps, so the returns find their plans and graphs parked.
SCHEDULE = [(4, 1280, 720), (1, 1280, 720), (2, 961, 541), (6, 961, 541), (3, 961, 541), (4, 1280, 720), (1, 1280, 720)]


def _cams(W, H, L):
    return [Camera(W, H, fieldOfView=35.0 + 9.0 * l, nearClipPlane=0.05 + 0.1 * l, farClipPlane=60.0 + 150.0 * l) for l in range(L)]


def _reserved(W, H, L, *, max_layers=LMAX, max_resolution=MAXR, **kw):
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=_cams(W, H, L) if L > 1 else None, max_resolution=max_resolution, **kw)
    ao.maxLayers = max_layers
    return ao


def _switch(ao, L, W, H, cams=True):
    """The host's per-frame inputs for L views of W x H: the camera's size, the count, one camera per view."""
    ao.camera.pixelWidth, ao.camera.pixelHeight = W, H
    ao.layers = L
    ao.layerCameras = _cams(W, H, L) if cams and L > 1 else None


def _depth(W, H, L, seed):
    return harness.frames(W, H, L, seed=seed)                             # [L, H, W] raw f32


def _oracle(ao, depth):
    """The oracle's AO of every layer of `depth` with that layer's camera."""
    cams = ao.layerCameras or [ao.camera] * len(depth)
    return np.stack([harness.oracle(depth.shape[2], depth.shape[1], camera=cams[l], threads=8).run(depth[l]) for l in range(len(depth))])


def _shaped(x, L):
    return x if L > 1 else x[0]


def _res(ao):
    return ao.reservation()


def _hostile(torch, ao):
    ao.LateUpdate()
    d = np.stack([HC.hostile_raw(*MAXR, ao.zbuffer_params(), True, seed=l) for l in range(ao.layers)])
    ao.render(torch.from_numpy(_shaped(d, ao.layers)).cuda())
    torch.cuda.synchronize()


def test_parity_over_a_view_count_schedule_after_a_hostile_frame(torch_cuda):
    torch = torch_cuda
    ao = _reserved(*MAXR, LMAX)
    _hostile(torch, ao)
    r0 = _res(ao)
    targets = {}                                                            # one depth and AO target per (W, H, L), as a host keeps them
    for i, (L, W, H) in enumerate(SCHEDULE):
        _switch(ao, L, W, H)
        d = _depth(W, H, L, seed=i)
        revisit = (L, W, H) in targets
        if not revisit:
            shape = _shaped(d, L).shape
            targets[(L, W, H)] = (torch.empty(shape, dtype=torch.float32, device="cuda"), torch.empty(shape, dtype=torch.uint8, device="cuda"))
        dd, oo = targets[(L, W, H)]
        dd.copy_(torch.from_numpy(_shaped(d, L)))
        inst = _res(ao)["graph_instantiations"]
        got = ao.render(dd, oo).cpu().numpy().reshape(L, H, W)
        if revisit:
            assert _res(ao)["graph_instantiations"] == inst, f"L={L} {W}x{H}: a revisited (W, H, L) instantiated a graph"
        bufs = {bid: ao.debug_buffer(bid) for bid in harness.buffer_ids()}
        fresh = harness.context(W, H, device=0, layers=L, layer_cameras=_cams(W, H, L) if L > 1 else None)
        ref_ao, ref_bufs = fresh_frame(torch, fresh, _shaped(d, L))
        assert harness.n_diff(got, ref_ao.reshape(L, H, W)) == 0, f"L={L} {W}x{H}: AO differs from a fresh context"
        for bid in harness.buffer_ids():
            assert harness.n_diff(bufs[bid], ref_bufs[bid]) == 0, f"L={L} {W}x{H}: buffer {bid} differs from a fresh context"
        assert harness.n_diff(got, _oracle(ao, d)) == 0, f"L={L} {W}x{H}: AO differs from the oracle"
    assert _res(ao)["arena_allocations"] == r0["arena_allocations"]
    ao.close()


FORM_SCHEDULE = [(3, 961, 541), (1, 1280, 720), (5, 640, 360), (2, 961, 541), (3, 961, 541)]


@pytest.mark.parametrize("form", ["pitched", "arrays", "batch", "arrays_batch"])
def test_every_frame_form_follows_the_count(torch_cuda, rt, form):
    torch = torch_cuda
    ao = _reserved(*MAXR, LMAX)
    _hostile(torch, ao)
    allocs = _res(ao)["arena_allocations"]
    big_d = torch.zeros((LMAX, MAXR[1] + 3, MAXR[0] + 40), dtype=torch.float32, device="cuda")
    big_a = torch.zeros((LMAX, MAXR[1] + 5, MAXR[0] + 72), dtype=torch.uint8, device="cuda")
    pool_d = [Array(rt, *MAXR, np.float32) for _ in range(LMAX)]               # max-size targets: the frame at their top-left corner
    pool_a = [Array(rt, *MAXR, np.uint8) for _ in range(LMAX)]
    for i, (L, W, H) in enumerate(FORM_SCHEDULE):
        _switch(ao, L, W, H)
        d = _depth(W, H, L, seed=10 + i)
        if form == "pitched":
            big_d[:L, :H, :W] = torch.from_numpy(d).cuda()
            dv, av = (big_d[:L, :H, :W], big_a[:L, :H, :W]) if L > 1 else (big_d[0, :H, :W], big_a[0, :H, :W])
            ao.render(dv, av)
            got = av.cpu().numpy().reshape(L, H, W)
        elif form == "arrays":
            shape = "layered" if L > 1 else "2d"
            da, aa = Array(rt, W, H, np.float32, shape=shape, layers=L), Array(rt, W, H, np.uint8, shape=shape, layers=L)
            da.fill(d)
            ao.render_arrays(da.handle, aa.handle)
            got = aa.read()
            for a in (da, aa):
                ao.release_array(a.handle)
                a.free()
        elif form == "batch":
            outs = ao.render_batch([torch.from_numpy(d[l]).cuda() for l in range(L)])
            got = np.stack([o.cpu().numpy() for o in outs])
        else:
            for l in range(L):
                full = np.zeros((MAXR[1], MAXR[0]), np.float32)
                full[:H, :W] = d[l]
                pool_d[l].fill(full)
            ao.render_arrays_batch([a.handle for a in pool_d[:L]], [a.handle for a in pool_a[:L]])
            got = np.stack([pool_a[l].read()[0, :H, :W] for l in range(L)])
        assert harness.n_diff(got, _oracle(ao, d)) == 0, f"{form} L={L} {W}x{H}: AO differs from the oracle"
    assert _res(ao)["arena_allocations"] == allocs
    for a in pool_d + pool_a:
        ao.release_array(a.handle)
        a.free()
    ao.close()


def test_split_screen_players_join_and_leave(torch_cuda, rt):
    """Up to four players in the quadrants of one shared depth and one shared AO array: each join or leave is set_layers, the
    players' cameras and their viewports; every player's rectangle equals the oracle with its camera, and the counts seen before
    replay their graphs."""
    torch = torch_cuda
    W, H = 480, 270
    ao = harness.context(W, H, device=0, max_resolution=(W, H))
    ao.maxLayers = 4
    da, aa = Array(rt, 2 * W, 2 * H, np.float32), Array(rt, 2 * W, 2 * H, np.uint8)
    full = np.concatenate([np.concatenate(list(q), axis=1) for q in _depth(W, H, 4, seed=3).reshape(2, 2, H, W)], axis=0)
    da.fill(full)
    quads = [(0, 0), (W, 0), (0, H), (W, H)]
    seen, allocs = set(), None
    for n in (1, 2, 3, 4, 2, 1):
        ao.layers = n
        ao.layerCameras = _cams(W, H, n)
        ao.layerViewports = [(x, y, 0, x, y, 0) for (x, y) in quads[:n]]
        inst = _res(ao)["graph_instantiations"]
        ao.render_arrays(da.handle, aa.handle)
        r = _res(ao)
        allocs = allocs if allocs is not None else r["arena_allocations"]
        assert r["arena_allocations"] == allocs, f"{n} players: a join or leave allocated"
        if n in seen:
            assert r["graph_instantiations"] == inst, f"{n} players again: a graph was instantiated"
        seen.add(n)
        got = aa.read()[0]
        for p, (x, y) in enumerate(quads[:n]):
            ref = harness.oracle(W, H, camera=ao.layerCameras[p], threads=8).run(full[y:y + H, x:x + W])
            assert harness.n_diff(got[y:y + H, x:x + W], ref) == 0, f"{n} players: player {p} differs from the oracle"
    for a in (da, aa):
        ao.release_array(a.handle)
        a.free()
    ao.close()


def test_layer_changes_and_viewport_tables_do_not_synchronise(torch_cuda):
    torch = torch_cuda
    s = torch.cuda.Stream()
    W, H = 960, 540
    dev = {L: torch.from_numpy(_shaped(_depth(W, H, L, seed=L), L)).cuda() for L in (1, 2, 3, 4)}
    out = {L: torch.empty(dev[L].shape, dtype=torch.uint8, device="cuda") for L in dev}
    ao = harness.context(W, H, device=0, layers=4)
    ao.maxLayers = 4
    for L in (4, 2, 4):
        ao.layers = L
        ao.render(dev[L], out[L], stream=s)
    torch.cuda.synchronize()
    r0 = _res(ao)
    e = backlog(torch, s, ao, dev[4], out[4])
    ao.layers = 2                                                           # a planned count: a plain replay
    ao.render(dev[2], out[2], stream=s)
    assert not e.query(), "a change to a planned layer count waited for the GPU"
    ao.layers = 3                                                           # a new count: planned on the host, tables in stream order
    ao.render(dev[3], out[3], stream=s)
    assert not e.query(), "a change to a new layer count waited for the GPU"
    ao.layerViewports = [(0, 0, l, 0, 0, l) for l in range(3)]              # a table where there was none
    ao.render(dev[3], out[3], stream=s)
    assert not e.query(), "setting a viewport table waited for the GPU"
    ao.layerViewports = None                                                # and cleared again
    ao.render(dev[3], out[3], stream=s)
    assert not e.query(), "clearing a viewport table waited for the GPU"
    ao.layers = 1
    ao.render(dev[1], out[1], stream=s)
    assert not e.query(), "a change to one layer waited for the GPU"
    torch.cuda.synchronize()
    r1 = _res(ao)
    assert r1["arena_allocations"] == r0["arena_allocations"]
    ref = _oracle(ao, _depth(W, H, 1, seed=1))
    assert harness.n_diff(out[1].cpu().numpy(), ref[0]) == 0
    ao.layers = 3
    ref3 = _oracle(ao, _depth(W, H, 3, seed=3))
    assert harness.n_diff(out[3].cpu().numpy(), ref3) == 0
    ao.close()
    # the same change on a context without a layer reservation does wait: the test observes what it claims
    u = harness.context(W, H, device=0, layers=4)
    u.render(dev[4], out[4], stream=s)
    torch.cuda.synchronize()
    e = backlog(torch, s, u, dev[4], out[4])
    u.layers = 2
    u.render(dev[2], out[2], stream=s)
    assert e.query(), "an unreserved layer change is expected to drain the GPU"
    torch.cuda.synchronize()
    u.close()


def test_refusals_launch_nothing(torch_cuda):
    torch = torch_cuda
    lib = N.lib()
    W, H = 320, 180
    ao = harness.context(W, H, device=0, layers=2)
    ao.maxLayers = 2
    d = torch.from_numpy(_depth(W, H, 2, seed=1)).cuda()
    ao.render(d)
    torch.cuda.synchronize()
    n, g, r = ao.launch_count, lib.meao_frame_generation(ao._ctx), _res(ao)
    assert lib.meao_set_layers(ao._ctx, 3) == N.MEAO_ERR_INVALID
    assert "layer reservation 2" in lib.meao_last_error(ao._ctx).decode()
    assert lib.meao_reserve_layers(ao._ctx, 1) == N.MEAO_ERR_INVALID
    with pytest.raises(MeaoError):
        ao.render_batch([d[0]])                                             # one tensor for two layers
    assert lib.meao_set_row_band(ao._ctx, 0, 96, -1, H) == N.MEAO_ERR_UNSUPPORTED
    assert ao.launch_count == n and lib.meao_frame_generation(ao._ctx) == g
    assert _res(ao)["arena_allocations"] == r["arena_allocations"] and _res(ao)["graph_instantiations"] == r["graph_instantiations"]
    ao.layers = 3
    with pytest.raises(ValueError):                                         # the host refuses a count above maxLayers itself
        ao.render(d)
    ao.close()


def test_no_graph_frames_follow_the_count(torch_cuda):
    torch = torch_cuda
    ao = _reserved(*MAXR, LMAX, use_graph=False)
    _hostile(torch, ao)
    for i, (L, W, H) in enumerate([(2, 961, 541), (1, 1280, 720), (5, 640, 360), (2, 961, 541)]):
        _switch(ao, L, W, H)
        d = _depth(W, H, L, seed=20 + i)
        got = ao.render(torch.from_numpy(_shaped(d, L)).cuda()).cpu().numpy().reshape(L, H, W)
        assert harness.n_diff(got, _oracle(ao, d)) == 0, f"no graph L={L} {W}x{H}"
    assert _res(ao)["graph_instantiations"] == 0
    ao.close()


def test_torch_graph_capture_after_one_settling_frame(torch_cuda):
    torch = torch_cuda
    W, H = 640, 360
    ao = harness.context(W, H, device=0, layers=4)
    ao.maxLayers = 4
    dev = {L: torch.from_numpy(_depth(W, H, L, seed=L)).cuda() for L in (2, 3, 4)}
    out = {L: torch.empty(dev[L].shape, dtype=torch.uint8, device="cuda") for L in dev}
    ao.render(dev[4], out[4])
    ao.layers = 2
    ao.layerCameras = _cams(W, H, 2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ao.render(dev[2], out[2])                                           # the settling frame: tables of the new count written
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    ao.layers, ao.layerCameras = 3, None                                    # a new (size, L) inside the capture: refused
    with torch.cuda.graph(g):
        out[3].zero_()                                                      # the capture holds this op and nothing of the context
        with pytest.raises(MeaoError) as e:
            ao.render(dev[3], out[3])
        ao.layers = 2
        ao.layerCameras = _cams(W, H, 2)
        with pytest.raises(MeaoError):
            ao.render(dev[2], out[2])                                       # the cleared camera table is not written yet either
    assert e.value.code == N.MEAO_ERR_INVALID and "issue one frame outside the capture first" in str(e.value)
    del g
    with torch.cuda.stream(s):
        ao.render(dev[2], out[2])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ao.render(dev[2], out[2])
    out[2].zero_()
    g.replay()
    torch.cuda.synchronize()
    assert harness.n_diff(out[2].cpu().numpy(), _oracle(ao, _depth(W, H, 2, seed=2))) == 0
    del g
    ao.close()


def test_release_array_named_by_graphs_of_several_counts(torch_cuda, rt):
    torch = torch_cuda
    W, H = 320, 184
    ao = harness.context(W, H, device=0, layers=2)
    ao.maxLayers = 3
    d = _depth(W, H, 3, seed=4)
    da = [Array(rt, W, H, np.float32) for _ in range(3)]
    aa = [Array(rt, W, H, np.uint8) for _ in range(3)]
    for l in range(3):
        da[l].fill(d[l])
    for L in (2, 3):
        ao.layers = L
        ao.render_arrays_batch([a.handle for a in da[:L]], [a.handle for a in aa[:L]])
    torch.cuda.synchronize()
    held = _res(ao)["graphs_held"]
    g = ao.frame_generation
    ao.release_array(aa[1].handle)                                          # named by the graphs of both counts
    assert _res(ao)["graphs_held"] == held - 2 and ao.frame_generation != g
    ao.layers = 2
    ao.render_arrays_batch([a.handle for a in da[:2]], [a.handle for a in aa[:2]])
    got = np.stack([aa[l].read()[0] for l in range(2)])
    assert harness.n_diff(got, _oracle(ao, d[:2])) == 0
    for a in da + aa:
        ao.release_array(a.handle)
        a.free()
    ao.close()
