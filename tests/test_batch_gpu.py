"""GPU tests of batches (meao_render_batch / meao_render_arrays_batch) on the H100: one layered frame whose layer l reads and writes
tensors or CUDA arrays of its own.  Every layer's AO (and, where checked, every debug buffer) must equal, bit for bit, the single-layer
frame of that layer's depth with that layer's camera, which the other GPU tests check against the oracle; a few cases check the
oracle directly.  Oversized arrays keep a poison pattern outside W x H.  Also: count = 1 against meao_render_arrays, a reserved
context walking sizes under fixed maximum-size targets, every refusal (layer and field named, nothing launched), the graph cache
(replay without instantiation, more rotating lists than the cache holds, meao_release_array of one entry), the plugin event,
MEAO_FLAG_NO_GRAPH and a torch.cuda.graph capture that replays its own list after the host issued another."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

pytestmark = pytest.mark.gpu

POISON = 0xA7
CAMS = [(0.3, 100.0, 60.0), (0.1, 1000.0, 90.0), (0.5, 50.0, 40.0), (0.2, 300.0, 75.0)]


def _cams(W, H, L, reversed_z=True):
    return [Camera(W, H, nearClipPlane=n, farClipPlane=f, fieldOfView=v, usesReversedZBuffer=reversed_z) for n, f, v in
            (CAMS[l % len(CAMS)] for l in range(L))]


class _Singles:
    """Single-layer reference frames, one context per distinct camera: (AO [H, W], {id: debug buffer}) of a layer's depth."""

    def __init__(self, torch, W, H, debug=True, **kw):
        self.torch, self.W, self.H, self.debug, self.kw, self.ctx = torch, W, H, debug, kw, {}

    def __call__(self, cam, depth, linear=False):
        key = (cam.nearClipPlane, cam.farClipPlane, cam.fieldOfView, cam.usesReversedZBuffer)
        if key not in self.ctx:
            self.ctx[key] = harness.context(Camera(self.W, self.H, nearClipPlane=key[0], farClipPlane=key[1], fieldOfView=key[2],
                                                   usesReversedZBuffer=key[3]), device=0, **self.kw)
        one = self.ctx[key]
        out = one.render(self.torch.from_numpy(np.ascontiguousarray(depth)).cuda(), linear=linear).cpu().numpy()
        bufs = {b: one.debug_buffer(b) for b in harness.buffer_ids(self.kw.get("high_quality_mask", 0), self.kw.get("single_scale", False))} \
            if self.debug else {}
        return out, bufs

    def close(self):
        for c in self.ctx.values():
            c.close()


def _check(ao, got, refs, tag, debug_layers=()):
    for l, g in enumerate(got):
        assert harness.n_diff(g, refs[l][0]) == 0, f"{tag}: layer {l}'s AO"
    for l in debug_layers:
        for b, ref in refs[l][1].items():
            mine = ao.debug_buffer(b)
            mine = mine[l] if mine.ndim > np.ndim(ref) else mine         # a single-layer context has no layer axis
            assert np.array_equal(mine.view(np.uint8), np.asarray(ref).view(np.uint8)), f"{tag}: layer {l} debug buffer {b}"


def _tensors(torch, depth, seed):
    """Separate CUDA allocations for the layers of `depth` [L, H, W]: layer l % 3 == 1 is the corner of a wider tensor (an odd row
    pitch), l % 3 == 2 starts one element into its allocation (a base that is not 16-byte aligned); the AO outputs likewise, with
    poisoned margins.  Returns (depth views, AO views, AO backing tensors)."""
    L, H, W = depth.shape
    ds, outs, backs = [], [], []
    for l in range(L):
        # built on the host: torch has few CUDA operators for uint16 / uint32
        if l % 3 == 1:
            big = np.zeros((H, W + 3), depth.dtype)
            big[:, :W] = depth[l]
            d = torch.from_numpy(big).cuda()[:, :W]
        elif l % 3 == 2:
            flat = np.zeros(H * W + 1, depth.dtype)
            flat[1:] = depth[l].reshape(-1)
            d = torch.from_numpy(flat).cuda()[1:].view(H, W)
        else:
            d = torch.from_numpy(np.ascontiguousarray(depth[l])).cuda()
        ds.append(d)
        back = torch.full((H + 1, W + 5), POISON, dtype=torch.uint8, device="cuda")
        o = back[:H, :W] if l % 3 != 2 else back.view(-1)[3:3 + H * (W + 5)].view(H, W + 5)[:, :W]
        outs.append(o)
        backs.append((back, o))
    return ds, outs, backs


def _outside_kept(backs):
    for back, o in backs:
        m = np.ones(back.shape, bool).reshape(-1)
        base = (o.data_ptr() - back.data_ptr())
        rows, W, pitch = o.shape[0], o.shape[1], o.stride(0)
        for y in range(rows):
            m[base + y * pitch: base + y * pitch + W] = False
        assert (back.cpu().numpy().reshape(-1)[m] == POISON).all(), "a byte outside an AO view changed"


# ---- 1. pointers and arrays at several layer counts --------------------------------------------------------------------------
SIZES = {1: (517, 301), 2: (966, 541), 6: (333, 187), 64: (130, 71)}


@pytest.mark.parametrize("L", [1, 2, 6, 64])
def test_pointer_batch_layers_match_single_layer_frames(torch_cuda, L):
    torch = torch_cuda
    W, H = SIZES[L]
    cams = _cams(W, H, L)
    depth = harness.frames(W, H, L, seed=L)
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams)
    singles = _Singles(torch, W, H, debug=L <= 6)
    try:
        ds, outs, backs = _tensors(torch, depth, L)
        ao.render_batch(ds, outs)
        torch.cuda.synchronize()
        refs = [singles(cams[l], depth[l]) for l in range(L)]
        _check(ao, [o.cpu().numpy() for o in outs], refs, f"pointers L={L}", debug_layers=range(L) if L <= 6 else ())
        _outside_kept(backs)
        if L == 2:
            for l in range(L):
                assert np.array_equal(refs[l][0], harness.oracle(W, H, camera=cams[l], threads=8).run(depth[l])), f"layer {l} vs oracle"
    finally:
        singles.close()
        ao.close()


@pytest.mark.parametrize("kind", ["raw_f32", "linear_f32", "d16", "d24s8"])
def test_pointer_batch_every_depth_format_and_premin(torch_cuda, kind):
    torch = torch_cuda
    W, H, L = 203, 117, 3
    cams = _cams(W, H, L)
    if kind == "linear_f32":
        depth = harness.contrasting_layers(W, H, L, seed=5)
    elif kind == "raw_f32":
        depth = harness.frames(W, H, L, seed=5)
    else:
        depth = harness.ingest(harness.frames(W, H, L, seed=5), kind)[0]
    kw = dict(high_quality_mask=0b0011)                 # premin on the final level
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams, **kw)
    singles = _Singles(torch, W, H, **kw)
    try:
        ds, outs, _ = _tensors(torch, depth, 0)
        ao.render_batch(ds, outs, linear=kind == "linear_f32")
        torch.cuda.synchronize()
        refs = [singles(cams[l], depth[l], linear=kind == "linear_f32") for l in range(L)]
        _check(ao, [o.cpu().numpy() for o in outs], refs, kind, debug_layers=range(L))
    finally:
        singles.close()
        ao.close()


def _arrays(rt, depth, ext, kind_dt, shapes, poison=True):
    """One depth and one AO array per layer, each of extent ext[l] (>= W x H), the depth at the top-left corner; shapes[l]: "2d" or
    a "layered" array of depth 1.  Outside W x H the depth holds NaN-free garbage and the AO the poison byte."""
    L, H, W = depth.shape
    da, aa = [], []
    rng = np.random.default_rng(7)
    for l in range(L):
        w, h = ext[l]
        img = (rng.random((h, w)) * (60000 if kind_dt == np.uint16 else 0.9)).astype(kind_dt)
        img[:H, :W] = depth[l]
        d = Array(rt, w, h, kind_dt, shape=shapes[l])
        d.fill(img[None])
        a = Array(rt, w, h, np.uint8, shape=shapes[(l + 1) % L])
        a.fill(np.full((1, h, w), POISON, np.uint8))
        da.append(d)
        aa.append(a)
    return da, aa


@pytest.mark.parametrize("L", [1, 2, 6, 64])
def test_array_batch_layers_match_single_layer_frames(torch_cuda, rt, L):
    torch = torch_cuda
    W, H = SIZES[L]
    cams = _cams(W, H, L)
    d16 = L % 2 == 0
    raw = harness.frames(W, H, L, seed=L + 1)
    depth = harness.ingest(raw, "d16")[0] if d16 else raw
    ext = [(W + (l % 3) * 7, H + (l % 2) * 5) for l in range(L)]          # some exact, some larger than W x H
    shapes = ["2d" if l % 2 == 0 else "layered" for l in range(L)]
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams)
    singles = _Singles(torch, W, H, debug=L <= 6)
    da, aa = _arrays(rt, depth, ext, np.uint16 if d16 else np.float32, shapes)
    try:
        ao.render_arrays_batch([d.handle for d in da], [a.handle for a in aa], kind="d16" if d16 else "raw_f32")
        torch.cuda.synchronize()
        got = [a.read()[0] for a in aa]
        refs = [singles(cams[l], depth[l]) for l in range(L)]
        _check(ao, [g[:H, :W] for g in got], refs, f"arrays L={L}", debug_layers=range(L) if L <= 6 else ())
        for l, g in enumerate(got):
            assert (g[H:] == POISON).all() and (g[:, W:] == POISON).all(), f"layer {l}: a texel outside W x H changed"
        if L == 2:
            for l in range(L):
                orc = harness.oracle(W, H, camera=cams[l], threads=8).run(harness.ingest(raw, "d16")[1][l])
                assert np.array_equal(refs[l][0], orc), f"layer {l} vs oracle"
    finally:
        for x in da + aa:
            ao.release_array(x.handle)
            x.free()
        singles.close()
        ao.close()


def test_array_batch_premin_forward_z(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 250, 141, 3
    cams = _cams(W, H, L, reversed_z=False)
    depth = harness.frames(W, H, L, seed=3, reversed_z=False)
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams, high_quality_mask=0b1111, reversed_z=False)
    singles = _Singles(torch, W, H, high_quality_mask=0b1111)
    da, aa = _arrays(rt, depth, [(W, H)] * L, np.float32, ["2d"] * L)
    try:
        ao.render_arrays_batch([d.handle for d in da], [a.handle for a in aa])
        torch.cuda.synchronize()
        refs = [singles(cams[l], depth[l]) for l in range(L)]
        _check(ao, [a.read()[0] for a in aa], refs, "arrays premin forward Z", debug_layers=range(L))
    finally:
        for x in da + aa:
            ao.release_array(x.handle)
            x.free()
        singles.close()
        ao.close()


def test_count_one_equals_render_arrays(torch_cuda, rt):
    torch = torch_cuda
    W, H = 401, 233
    depth = harness.frames(W, H, 1, seed=9)
    one, batch = harness.context(W, H, device=0), harness.context(W, H, device=0)
    da, (a1, a2) = Array(rt, W, H, np.float32), (Array(rt, W, H, np.uint8), Array(rt, W, H, np.uint8))
    da.fill(depth)
    try:
        one.render_arrays(da.handle, a1.handle)
        batch.render_arrays_batch([da.handle], [a2.handle])
        torch.cuda.synchronize()
        assert np.array_equal(a1.read(), a2.read())
        for b in harness.buffer_ids():
            assert np.array_equal(one.debug_buffer(b).view(np.uint8), batch.debug_buffer(b).view(np.uint8)), f"debug buffer {b}"
    finally:
        for c in (one, batch):
            for x in (da, a1, a2):
                c.release_array(x.handle)
            c.close()
        for x in (da, a1, a2):
            x.free()


def test_reserved_context_walks_sizes_under_fixed_targets(torch_cuda, rt):
    torch = torch_cuda
    MW, MH, L = 640, 360, 3
    cams = _cams(MW, MH, L)
    ao = harness.context(MW, MH, device=0, layers=L, layer_cameras=cams, max_resolution=(MW, MH))
    da = [Array(rt, MW, MH, np.float32) for _ in range(L)]
    aa = [Array(rt, MW, MH, np.uint8) for _ in range(L)]
    tensors = [torch.full((MH, MW), 0.5, dtype=torch.float32, device="cuda") for _ in range(L)]
    touts = [torch.full((MH, MW), POISON, dtype=torch.uint8, device="cuda") for _ in range(L)]
    try:
        for i, (W, H) in enumerate([(MW, MH), (401, 233), (MW, MH), (257, 129), (401, 233)]):
            for c in [ao.camera] + cams:
                c.pixelWidth, c.pixelHeight = W, H
            depth = harness.frames(W, H, L, seed=i)
            for l in range(L):
                img = np.zeros((MH, MW), np.float32)
                img[:H, :W] = depth[l]
                da[l].fill(img[None])
                aa[l].fill(np.full((1, MH, MW), POISON, np.uint8))
                tensors[l][:H, :W] = torch.from_numpy(depth[l]).cuda()
            ao.render_arrays_batch([d.handle for d in da], [a.handle for a in aa])
            ao.render_batch([t[:H, :W] for t in tensors], [o[:H, :W] for o in touts])
            torch.cuda.synchronize()
            singles = _Singles(torch, W, H, debug=False)
            try:
                refs = [singles(_cams(W, H, L)[l], depth[l]) for l in range(L)]
            finally:
                singles.close()
            for l in range(L):
                g = aa[l].read()[0]
                assert np.array_equal(g[:H, :W], refs[l][0]), f"{W}x{H} array layer {l}"
                assert (g[H:] == POISON).all() and (g[:, W:] == POISON).all(), f"{W}x{H} array layer {l}: outside W x H"
                assert np.array_equal(touts[l][:H, :W].cpu().numpy(), refs[l][0]), f"{W}x{H} pointer layer {l}"
    finally:
        for x in da + aa:
            ao.release_array(x.handle)
            x.free()
        ao.close()


# ---- 2. refusals -------------------------------------------------------------------------------------------------------------------
def test_refusals_name_layer_and_field_and_launch_nothing(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 160, 96, 3
    ao = harness.context(W, H, device=0, layers=L)
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    da = [Array(rt, W, H, np.float32) for _ in range(L)]
    aa = [Array(rt, W, H, np.uint8) for _ in range(L)]
    small = Array(rt, W - 1, H, np.uint8)
    cube = Array(rt, W, W, np.uint8, shape="cube")
    P = lambda xs: (C.c_void_p * len(xs))(*xs)             # noqa: E731
    I64 = lambda xs: (C.c_int64 * len(xs))(*xs)            # noqa: E731
    d = [x.handle for x in da]
    a = [x.handle for x in aa]
    dt = [torch.zeros((H, W), dtype=torch.float32, device="cuda") for _ in range(L)]
    ot = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(L)]
    dp, op = [t.data_ptr() for t in dt], [t.data_ptr() for t in ot]
    z = [0] * L
    try:
        def refused(rc, want, *texts):
            err = lib.meao_last_error(ctx)
            assert rc == want and all(t in err for t in texts), (rc, err)

        before = ao.launch_count
        refused(lib.meao_render_arrays_batch(ctx, P(d[:2]), 0, P(a[:2]), 2, None), N.MEAO_ERR_INVALID, b"count 2", b"layer count 3")
        refused(lib.meao_render_arrays_batch(ctx, None, 0, P(a), L, None), N.MEAO_ERR_INVALID, b"depth_arrays")
        refused(lib.meao_render_arrays_batch(ctx, P(d[:1] + [None] + d[2:]), 0, P(a), L, None), N.MEAO_ERR_INVALID, b"layer 1",
                b"depth_arrays[1]")
        refused(lib.meao_render_arrays_batch(ctx, P(d), 0, P(a[:2] + [a[0]]), L, None), N.MEAO_ERR_INVALID, b"layer 2", b"ao_arrays[2]",
                b"layer 0")
        refused(lib.meao_render_arrays_batch(ctx, P(d), 0, P(a[:1] + [small.handle] + a[2:]), L, None), N.MEAO_ERR_INVALID, b"layer 1",
                b"ao_arrays[1]", b"smaller")
        refused(lib.meao_render_arrays_batch(ctx, P(d), 0, P(a[:2] + [cube.handle]), L, None), N.MEAO_ERR_INVALID, b"layer 2",
                b"ao_arrays[2]")
        refused(lib.meao_render_arrays_batch(ctx, P(a), 0, P(a), L, None), N.MEAO_ERR_INVALID, b"layer 0", b"depth_array")
        refused(lib.meao_render_arrays_batch(ctx, P(d), 3, P(a), L, None), N.MEAO_ERR_UNSUPPORTED, b"D24S8")
        refused(lib.meao_bind_event_arrays_batch(ctx, 95, P(d), 0, P(a[:2] + [a[1]]), L, None), N.MEAO_ERR_INVALID, b"layer 2")
        # pointers
        refused(lib.meao_render_batch(ctx, P(dp), None, 0, P(op), I64(z), L, None), N.MEAO_ERR_INVALID, b"depth_row_pitch")
        refused(lib.meao_render_batch(ctx, P(dp), I64(z), 0, P(op[:2] + [None]), I64(z), L, None), N.MEAO_ERR_INVALID, b"layer 2", b"ao[2]")
        refused(lib.meao_render_batch(ctx, P(dp), I64([0, 4 * W - 4, 0]), 0, P(op), I64(z), L, None), N.MEAO_ERR_INVALID, b"layer 1",
                b"depth_row_pitch[1]")
        refused(lib.meao_render_batch(ctx, P(dp), I64([0, 0, 4 * W + 2]), 0, P(op), I64(z), L, None), N.MEAO_ERR_INVALID, b"layer 2",
                b"depth_row_pitch[2]")
        refused(lib.meao_render_batch(ctx, P(dp), I64(z), 0, P(op), I64([0, W - 1, 0]), L, None), N.MEAO_ERR_INVALID, b"layer 1",
                b"ao_row_pitch[1]")
        refused(lib.meao_render_batch(ctx, P(dp[:1] + [dp[1] + 2] + dp[2:]), I64(z), 0, P(op), I64(z), L, None), N.MEAO_ERR_INVALID,
                b"layer 1", b"depth[1]", b"aligned")
        refused(lib.meao_render_batch(ctx, P(dp), I64(z), 0, P(op[:2] + [op[1] + W * H - 1]), I64(z), L, None), N.MEAO_ERR_INVALID,
                b"ao[", b"AO extent")
        refused(lib.meao_render_batch(ctx, P(dp), I64(z), 0, P(op[:2] + [dp[0] + 8]), I64(z), L, None), N.MEAO_ERR_INVALID, b"layer 2",
                b"ao[2]", b"depth extent", b"depth[0]")
        assert ao.launch_count == before
        # depth entries may repeat, and AO views that touch without overlapping are fine
        assert lib.meao_render_batch(ctx, P([dp[0]] * L), I64(z), 0, P(op), I64(z), L, None) == 0, lib.meao_last_error(ctx)
        torch.cuda.synchronize()
        assert ao.launch_count - before == ao.kernels_per_frame
        # a layer-viewport table is refused
        ao.layerViewports = [(0, 0, 0, 0, 0, 0), (0, 0, 1, 0, 0, 1), (0, 0, 2, 0, 0, 2)]
        ao.LateUpdate()
        before = ao.launch_count
        refused(lib.meao_render_batch(ctx, P(dp), I64(z), 0, P(op), I64(z), L, None), N.MEAO_ERR_INVALID, b"meao_set_layer_viewports")
        refused(lib.meao_render_arrays_batch(ctx, P(d), 0, P(a), L, None), N.MEAO_ERR_INVALID, b"meao_set_layer_viewports")
        assert ao.launch_count == before
    finally:
        for x in da + aa + [small, cube]:
            ao.release_array(x.handle)
            x.free()
        ao.close()


def test_refusals_of_the_combinations_and_the_bound(torch_cuda):
    torch = torch_cuda
    P = lambda xs: (C.c_void_p * len(xs))(*xs)             # noqa: E731
    I64 = lambda xs: (C.c_int64 * len(xs))(*xs)            # noqa: E731
    W, H = 256, 256
    # an orthographic projection and a row band: MEAO_ERR_UNSUPPORTED
    ortho = harness.context(Camera(W, H, orthographic=True), device=0)
    band = harness.context(W, H, device=0)
    big = harness.context(16, 16, device=0, layers=257)
    d = torch.zeros((H, W), dtype=torch.float32, device="cuda")
    o = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    try:
        ortho.LateUpdate()
        before = ortho.launch_count
        rc = ortho._lib.meao_render_batch(ortho._ctx, P([d.data_ptr()]), I64([0]), 0, P([o.data_ptr()]), I64([0]), 1, None)
        assert rc == N.MEAO_ERR_UNSUPPORTED and b"orthographic" in ortho._lib.meao_last_error(ortho._ctx)
        assert ortho.launch_count == before
        band.LateUpdate()
        band.set_row_band(0, 128, -1, 256)
        rc = band._lib.meao_render_batch(band._ctx, P([d.data_ptr()]), I64([0]), 0, P([o.data_ptr()]), I64([0]), 1, None)
        assert rc == N.MEAO_ERR_UNSUPPORTED and b"row band" in band._lib.meao_last_error(band._ctx)
        big.LateUpdate()
        n = 257
        rc = big._lib.meao_render_batch(big._ctx, P([d.data_ptr()] * n), I64([0] * n), 0, P([o.data_ptr()] * n), I64([0] * n), n, None)
        assert rc == N.MEAO_ERR_INVALID and b"MEAO_MAX_BATCH" in big._lib.meao_last_error(big._ctx)
        assert big.launch_count == 0
    finally:
        for c in (ortho, band, big):
            c.close()


# ---- 3. graphs, release, event, NO_GRAPH, capture ----------------------------------------------------------------------------------
def test_graph_cache_replays_and_rotates_lists(torch_cuda):
    torch = torch_cuda
    W, H, L = 96, 64, 2
    cams = _cams(W, H, L)
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams)
    depth = harness.frames(W, H, L, seed=2)
    singles = _Singles(torch, W, H, debug=False)
    try:
        refs = [singles(cams[l], depth[l])[0] for l in range(L)]
        ds = [torch.from_numpy(depth[l]).cuda() for l in range(L)]
        outs = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(L)]
        ao.render_batch(ds, outs)
        inst = ao.reservation()["graph_instantiations"]
        for _ in range(3):
            ao.render_batch(ds, outs)
        assert ao.reservation()["graph_instantiations"] == inst, "a repeated list instantiated a graph"
        # more rotating lists (of distinct AO tensors) than the cache holds
        pool = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(2 * N.MEAO_MAX_GRAPHS_HELD + 8)]
        for i in range(0, len(pool) - 1, 2):
            ao.render_batch(ds, [pool[i], pool[i + 1]])
            assert ao.reservation()["graphs_held"] <= N.MEAO_MAX_GRAPHS_HELD
        torch.cuda.synchronize()
        for i in (0, len(pool) - 4, len(pool) - 2):
            for l in range(L):
                assert np.array_equal(pool[i + l].cpu().numpy(), refs[l]), f"list {i // 2} layer {l}"
        # swapping the two layers' outputs is another list: each layer still writes its own entry
        ao.render_batch(ds, outs[::-1])
        torch.cuda.synchronize()
        assert np.array_equal(outs[1].cpu().numpy(), refs[0]) and np.array_equal(outs[0].cpu().numpy(), refs[1])
    finally:
        singles.close()
        ao.close()


def test_release_array_drops_exactly_the_graphs_and_bindings_that_name_it(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 128, 72, 2
    ao = harness.context(W, H, device=0, layers=L)
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    depth = harness.frames(W, H, L, seed=4)
    da, aa = _arrays(rt, depth, [(W, H)] * L, np.float32, ["2d"] * L)
    ab = [Array(rt, W, H, np.uint8) for _ in range(L)]
    P = lambda xs: (C.c_void_p * len(xs))(*xs)             # noqa: E731
    d, a, b = [x.handle for x in da], [x.handle for x in aa], [x.handle for x in ab]
    try:
        ao.render_arrays_batch(d, a)
        ao.render_arrays_batch(d, b)
        assert lib.meao_bind_event_arrays_batch(ctx, 96, P(d), 0, P(a), L, None) == 0
        assert lib.meao_bind_event_arrays_batch(ctx, 97, P(d), 0, P(b), L, None) == 0
        torch.cuda.synchronize()
        held = ao.reservation()["graphs_held"]
        gen = ao.frame_generation
        ao.release_array(a[1])
        assert ao.reservation()["graphs_held"] == held - 1
        assert ao.frame_generation != gen
        before = ao.launch_count
        lib.meao_get_render_event_func()(96)                # unbound by the release: renders nothing
        assert ao.launch_count == before
        inst = ao.reservation()["graph_instantiations"]
        lib.meao_get_render_event_func()(97)                # still bound, its graph still cached
        ao.render_arrays_batch(d, b)
        torch.cuda.synchronize()
        assert ao.launch_count - before == 2 * ao.kernels_per_frame
        assert ao.reservation()["graph_instantiations"] == inst
        lib.meao_bind_event_arrays_batch(ctx, 97, None, 0, None, 0, None)
    finally:
        for x in da + aa + ab:
            ao.release_array(x.handle)
            x.free()
        ao.close()


def test_event_no_graph_and_torch_capture(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 200, 120, 3
    cams = _cams(W, H, L)
    depth = harness.frames(W, H, L, seed=6)
    singles = _Singles(torch, W, H, debug=False)
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams)
    flat = harness.context(W, H, device=0, layers=L, layer_cameras=cams, use_graph=False)
    da, aa = _arrays(rt, depth, [(W + 3, H)] * L, np.float32, ["2d", "layered", "2d"])
    P = lambda xs: (C.c_void_p * len(xs))(*xs)             # noqa: E731
    try:
        refs = [singles(cams[l], depth[l])[0] for l in range(L)]
        # the plugin event
        lib, ctx = ao._lib, ao._ctx
        ao.LateUpdate()
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.meao_bind_event_arrays_batch(ctx, 98, P([x.handle for x in da]), 0, P([x.handle for x in aa]), L, stream) == 0
        before = ao.launch_count
        lib.meao_get_render_event_func()(98)
        torch.cuda.synchronize()
        assert ao.launch_count - before == ao.kernels_per_frame, lib.meao_last_error(ctx)
        for l in range(L):
            assert np.array_equal(aa[l].read()[0][:, :W], refs[l]), f"event layer {l}"
        lib.meao_bind_event_arrays_batch(ctx, 98, None, 0, None, 0, None)
        # MEAO_FLAG_NO_GRAPH
        outs = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(L)]
        flat.render_batch([torch.from_numpy(depth[l]).cuda() for l in range(L)], outs)
        torch.cuda.synchronize()
        for l in range(L):
            assert np.array_equal(outs[l].cpu().numpy(), refs[l]), f"NO_GRAPH layer {l}"
        # a capture of one list replays that list after the host issued another
        ds = [torch.from_numpy(depth[l]).cuda() for l in range(L)]
        rec = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(L)]
        other = [torch.zeros((H, W), dtype=torch.uint8, device="cuda") for _ in range(L)]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ao.render_batch(ds, rec)                        # the settling frame
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        gen = ao.frame_generation
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ao.render_batch(ds, rec)
        assert ao.frame_generation == gen
        ao.render_batch(ds[::-1], other)                    # another list outside the capture
        torch.cuda.synchronize()
        for l in range(L):      # layer l reads the other list's depth with its own camera
            assert np.array_equal(other[l].cpu().numpy(), singles(cams[l], depth[L - 1 - l])[0]), f"other list layer {l}"
        for i in range(2):
            nd = harness.frames(W, H, L, seed=20 + i)
            for l in range(L):
                ds[l].copy_(torch.from_numpy(nd[l]))
                rec[l].fill_(POISON)
            g.replay()
            torch.cuda.synchronize()
            for l in range(L):
                assert np.array_equal(rec[l].cpu().numpy(), singles(cams[l], nd[l])[0]), f"replay {i} layer {l}"
        del g
        torch.cuda.synchronize()
    finally:
        for x in da + aa:
            ao.release_array(x.handle)
            x.free()
        singles.close()
        flat.close()
        ao.close()
