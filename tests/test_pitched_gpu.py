"""GPU tests of pitched frames (meao_render_pitched, meao_bind_event_pitched) on the H100: the depth and the AO are views inside larger
device allocations, each with its own byte row and layer pitch.  Every frame must give the bytes of meao_render on a tight copy and of
the oracle, through graph replay (including re-targeted graphs), MEAO_FLAG_NO_GRAPH, the plugin event and the debug buffer; bytes
outside the depth view are 0xff (NaN as f32) and never read, bytes outside the AO view hold a sentinel that survives on the device, and
every documented refusal launches nothing."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import torch_cuda  # noqa: F401  (the fixture)
from harness import SENTINEL, View

pytestmark = pytest.mark.gpu

KINDS = {"f32": 0, "linear": 1, "d16": 2, "d24s8": 3}


class DevView:
    """A View's backing allocation copied to the device; ptr is the view's first element there."""

    def __init__(self, torch, v: View):
        self.v = v
        self.dev = torch.from_numpy(v.back.copy()).cuda()

    @property
    def ptr(self):
        return self.dev.data_ptr() + self.v.base

    def fetch(self):
        self.v.back[...] = self.dev.cpu().numpy()
        return self.v


def _depth(kind, W, H, L, seed=0, rz=True):
    """(depth [L, H, W] in the ingest format of `kind`, the float32 the oracle sees)."""
    if kind == "linear":
        from miniengineao_b200 import synth
        lin = np.stack([synth.random_depth(W, H, seed=seed + i) for i in range(L)]).astype(np.float32)
        return lin, lin
    raw = harness.frames(W, H, L, seed=seed, reversed_z=rz)
    pairs = [harness.ingest(r, kind) for r in raw]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def _up(x, a):
    return (x + a - 1) // a * a


def _views(torch, depth, drow=None, dlayer=None, dbase=0, arow=None, alayer=None, abase=0, rows=None):
    L, H, W = depth.shape
    es = depth.dtype.itemsize
    drow = drow or W * es
    dlayer = dlayer or H * drow
    arow = arow or W
    alayer = alayer or H * arow
    dv = View(depth.shape, depth.dtype, drow, dlayer, dbase)
    dv.arr[...] = depth
    av = View((L, rows or H, W), np.uint8, arow, alayer, abase, fill=SENTINEL)
    return DevView(torch, dv), DevView(torch, av)


def _render_pitched(lib, ao, d: DevView, a: DevView, kind, stream=None):
    return lib.meao_render_pitched(ao._ctx, C.c_void_p(d.ptr), d.v.row, d.v.layer, KINDS[kind], C.c_void_p(a.ptr), a.v.row, a.v.layer,
                                   stream)


def _tight(torch, ao, depth, kind):
    """meao_render on a tight copy: [L, H, W] uint8."""
    from miniengineao_b200 import _native as N
    t = torch.from_numpy(np.ascontiguousarray(depth).view(np.uint8)).cuda()
    out = torch.empty(depth.shape, dtype=torch.uint8, device="cuda")
    N.check(ao._ctx, N.lib().meao_render(ao._ctx, t.data_ptr(), KINDS[kind], out.data_ptr(), None))
    return out.cpu().numpy()


def _check_frame(torch, ao, depth, seen, kind, d: DevView, a: DevView, oracle=True, **params):
    from miniengineao_b200 import _native as N
    lib = N.lib()
    ao.LateUpdate()
    before = ao.launch_count
    assert _render_pitched(lib, ao, d, a, kind) == 0, lib.meao_last_error(ao._ctx)
    assert ao.launch_count - before == ao.kernels_per_frame
    torch.cuda.synchronize()
    v = a.fetch()
    assert (v.outside() == SENTINEL).all(), "a byte outside the AO view was written"
    got = np.array(v.arr)
    tight = _tight(torch, ao, depth, kind)
    assert np.array_equal(got, tight), "pitched frame differs from meao_render on a tight copy"
    if oracle:
        L, H, W = depth.shape
        for l in range(L):
            ref = harness.oracle(W, H, linear=(kind == "linear"), threads=8, **params).run(seen[l])
            assert np.array_equal(got[l], ref), f"layer {l} differs from the oracle"
    return got


@pytest.mark.parametrize("W,H,kind,pitch", [(1, 1, "f32", 256), (3, 5, "d16", 256), (161, 93, "d24s8", 768), (250, 131, "f32", 1028),
                                            (1366, 768, "f32", 5632), (1366, 768, "d16", 2816), (1920, 1080, "linear", 8192),
                                            (3840, 2160, "f32", 15360 + 256)])
def test_pitched_equals_tight_and_oracle(torch_cuda, W, H, kind, pitch):
    """Padded rows: 256-byte multiples (D3D12 footprints: 1366 x 4 B rows are 5632 bytes apart), and a row pitch off the 16-byte grid."""
    rz = (W + H) % 2 == 0
    depth, seen = _depth(kind, W, H, 1, seed=W % 7, rz=rz)
    ao = harness.context(W, H, device=0, layers=1, reversed_z=rz, intensity=1.1)
    d, a = _views(torch_cuda, depth, drow=pitch, arow=_up(W, 256) + (3 if W == 250 else 0))
    _check_frame(torch_cuda, ao, depth, seen, kind, d, a, reversed_z=rz, intensity=1.1)


def test_sub_rectangle_and_no_graph(torch_cuda):
    """A viewport at x0 = 1 inside an atlas (depth 4 bytes, AO 1 byte past an aligned address), with and without graphs."""
    W, H = 640, 360
    depth, seen = _depth("f32", W, H, 1, seed=3)
    for use_graph in (True, False):
        ao = harness.context(W, H, device=0, layers=1, use_graph=use_graph)
        d, a = _views(torch_cuda, depth, drow=4096, dbase=4, arow=1024, abase=1)
        _check_frame(torch_cuda, ao, depth, seen, "f32", d, a)


@pytest.mark.parametrize("L", [2, 6])
def test_layered_dynamic_resolution_corner(torch_cuda, L):
    """[L, Hmax, Wmax][:, :H, :W]: the layer pitch is the max-size image; premin on level 1."""
    W, H, Wmax, Hmax = 600, 330, 800, 450
    depth, seen = _depth("f32", W, H, L, seed=L)
    ao = harness.context(W, H, device=0, layers=L, high_quality_mask=1)
    d, a = _views(torch_cuda, depth, drow=Wmax * 4, dlayer=Hmax * Wmax * 4, arow=Wmax, alayer=Hmax * Wmax)
    _check_frame(torch_cuda, ao, depth, seen, "f32", d, a, high_quality_mask=1)


def test_layered_1080p_d16_odd_layer_pitch(torch_cuda):
    W, H = 1920, 1080
    depth, seen = _depth("d16", W, H, 2, seed=9)
    ao = harness.context(W, H, device=0, layers=2)
    d, a = _views(torch_cuda, depth, drow=4096, dlayer=4096 * H + 2, arow=2048, alayer=2048 * H + 4)
    _check_frame(torch_cuda, ao, depth, seen, "d16", d, a, oracle=False)


def test_row_band_contexts(torch_cuda):
    """A band context that needs no halo renders its rows from a pitched band view; an interior band is refused as by meao_render."""
    from miniengineao_b200 import _native as N
    lib = N.lib()
    W, H = 320, 240
    depth, seen = _depth("f32", W, H, 1, seed=5)
    ao = harness.context(W, H, device=0, layers=1)
    ao.LateUpdate()
    ao.set_row_band(0, H, -1, -1)
    d, a = _views(torch_cuda, depth, drow=2048, arow=512)
    _check_frame(torch_cuda, ao, depth, seen, "f32", d, a)
    big = harness.context(1280, 1088, device=0, layers=1)
    big.LateUpdate()
    big.set_row_band(0, 544, -1, 1088)
    dep, _ = _depth("f32", 1280, 544, 1)
    d, a = _views(torch_cuda, dep, drow=8192, arow=2048)
    before = big.launch_count
    assert _render_pitched(lib, big, d, a, "f32") == N.MEAO_ERR_INVALID
    assert b"interior row band" in lib.meao_last_error(big._ctx)
    assert big.launch_count == before


def test_graph_key_holds_the_pitches(torch_cuda):
    """Tight, then pitched at the SAME two pointers with another pitch, then tight again: each frame is right (no stale replay).  Then
    more pitch combinations than the graph cache holds (64), so least recently used graphs are re-targeted; the last frame is right."""
    from miniengineao_b200 import _native as N
    lib = N.lib()
    torch = torch_cuda
    W, H = 128, 96
    depth, seen = _depth("f32", W, H, 1, seed=7)
    ref = harness.oracle(W, H, threads=8).run(seen[0])
    ao = harness.context(W, H, device=0, layers=1)
    ao.LateUpdate()
    maxp = W * 4 + 16 * 80
    dbuf = torch.full(((H - 1) * maxp // 4 + W + 64,), float("nan"), dtype=torch.float32, device="cuda")
    abuf = torch.full(((H - 1) * (W + 80) + W + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    dflat = torch.from_numpy(depth[0]).cuda()

    def frame(drow, arow):
        dbuf.fill_(float("nan")); abuf.fill_(SENTINEL)
        torch.as_strided(dbuf, (H, W), (drow // 4, 1)).copy_(dflat)
        rc = lib.meao_render_pitched(ao._ctx, C.c_void_p(dbuf.data_ptr()), drow, H * drow, 0, C.c_void_p(abuf.data_ptr()), arow, H * arow, None)
        assert rc == 0, lib.meao_last_error(ao._ctx)
        got = torch.as_strided(abuf, (H, W), (arow, 1)).cpu().numpy()
        assert np.array_equal(got, ref), (drow, arow)

    frame(W * 4, W)
    frame(W * 4 + 64, W + 16)
    frame(W * 4, W)
    for i in range(70):
        frame(W * 4 + 16 * (i + 1), W + (i % 9))
    frame(W * 4 + 16 * 5, W + 4)            # the rotation's fifth combination (i = 4), re-targeted away since


def test_event_binding_and_debug_buffer(torch_cuda):
    from miniengineao_b200 import _native as N
    lib = N.lib()
    W, H = 300, 170
    depth, seen = _depth("f32", W, H, 1, seed=60)
    ref = harness.oracle(W, H, threads=8).run(seen[0])
    ao = harness.context(W, H, device=0, layers=1)
    ao.LateUpdate()
    d, a = _views(torch_cuda, depth, drow=2048, arow=512)
    stream = C.c_void_p(torch_cuda.cuda.current_stream().cuda_stream)
    assert lib.meao_bind_event_pitched(ao._ctx, 91, C.c_void_p(d.ptr), 2048, 2048 * H, 0, C.c_void_p(a.ptr), 512, 512 * H, stream) == 0
    before = ao.launch_count
    lib.meao_get_render_event_func()(91)
    assert ao.launch_count - before == ao.kernels_per_frame
    torch_cuda.cuda.synchronize()
    v = a.fetch()
    assert np.array_equal(v.arr[0], ref)
    assert (v.outside() == SENTINEL).all()
    assert np.array_equal(ao.debug_buffer(17), ref)                      # meao_get_buffer(17) after a pitched frame
    # a refused view is refused at binding time and leaves nothing bound
    assert lib.meao_bind_event_pitched(ao._ctx, 92, C.c_void_p(d.ptr), 4, 0, 0, C.c_void_p(a.ptr), 512, 0, stream) == N.MEAO_ERR_INVALID
    before = ao.launch_count
    lib.meao_get_render_event_func()(92)
    assert ao.launch_count == before
    assert lib.meao_bind_event_pitched(ao._ctx, 91, None, 0, 0, 0, None, 0, 0, None) == 0      # unbind
    lib.meao_get_render_event_func()(91)
    assert ao.launch_count == before


def test_refusals_launch_nothing(torch_cuda):
    from miniengineao_b200 import _native as N
    lib = N.lib()
    torch = torch_cuda
    W, H = 160, 96
    ao = harness.context(W, H, device=0, layers=1)
    ao.LateUpdate()
    buf = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    dp, ap = p, p + (1 << 21)
    I32 = 2 ** 31 - 1
    cases = [  # (tag, depth, drow, dlayer, kind, ao, arow, alayer, text)
        ("NULL depth", None, 640, 0, 0, ap, W, 0, b"NULL"),
        ("NULL AO", dp, 640, 0, 0, None, W, 0, b"NULL"),
        ("bad kind", dp, 640, 0, 9, ap, W, 0, b"kind"),
        ("depth row below width", dp, 636, 0, 0, ap, W, 0, b"depth_row_pitch"),
        ("depth row not a multiple of the element", dp, 642, 0, 0, ap, W, 0, b"depth_row_pitch"),
        ("D16 row not a multiple of 2", dp, 321, 0, 2, ap, W, 0, b"depth_row_pitch"),
        ("AO row below width", dp, 640, 0, 0, ap, W - 1, 0, b"ao_row_pitch"),
        ("depth pointer misaligned", dp + 2, 640, 0, 0, ap, W, 0, b"aligned"),
        ("D16 pointer misaligned", dp + 1, 320, 0, 2, ap, W, 0, b"aligned"),
        ("negative depth row", dp, -640, 0, 0, ap, W, 0, b"depth_row_pitch"),
        ("negative depth layer", dp, 640, -1, 0, ap, W, 0, b"depth_layer_pitch"),
        ("negative AO row", dp, 640, 0, 0, ap, -W, 0, b"ao_row_pitch"),
        ("negative AO layer", dp, 640, 0, 0, ap, W, -5, b"ao_layer_pitch"),
        ("depth row above INT32_MAX", dp, I32 + 1, 0, 0, ap, W, 0, b"INT32_MAX"),
        ("AO row above INT32_MAX", dp, 640, 0, 0, ap, I32 + 1, 0, b"INT32_MAX"),
        ("views intersect", dp, 640, 0, 0, dp + 640 * 95, W, 0, b"intersect"),
        ("views interleave", dp, 1280, 0, 0, dp + 640, 1280, 0, b"intersect"),
    ]

    def check(ctx_ao, tag, d, drow, dlayer, kind, o, arow, alayer, text):
        before = ctx_ao.launch_count
        rc = lib.meao_render_pitched(ctx_ao._ctx, C.c_void_p(d), drow, dlayer, kind, C.c_void_p(o), arow, alayer, None)
        assert rc == N.MEAO_ERR_INVALID, (tag, rc)
        assert text in lib.meao_last_error(ctx_ao._ctx), (tag, lib.meao_last_error(ctx_ao._ctx))
        assert ctx_ao.launch_count == before, tag
        if d or o:
            rc = lib.meao_bind_event_pitched(ctx_ao._ctx, 5, C.c_void_p(d), drow, dlayer, kind, C.c_void_p(o), arow, alayer, None)
            assert rc == N.MEAO_ERR_INVALID, (tag, "bind", rc)

    for c in cases:
        check(ao, *c)
    # layered: overlapping layers are refused; with one layer the layer pitches are unused (0 is fine)
    lay = harness.context(W, H, device=0, layers=2)
    lay.LateUpdate()
    check(lay, "depth layers overlap", dp, 640, 640 * (H - 1) + 636, 0, ap, W, W * H, b"depth_layer_pitch")
    check(lay, "depth layer pitch between two elements", dp, 640, 640 * H + 2, 0, ap, W, W * H, b"depth_layer_pitch")
    check(lay, "D24S8 layer pitch between two elements", dp, 640, 640 * H + 6, 3, ap, W, W * H, b"depth_layer_pitch")
    check(lay, "AO layers overlap", dp, 640, 640 * H, 0, ap, W, W * (H - 1) + W - 1, b"ao_layer_pitch")
    depth, seen = _depth("f32", W, H, 1, seed=70)
    d, a = _views(torch, depth, drow=640, dlayer=0, arow=W, alayer=0)
    d.v.layer = a.v.layer = 0
    _check_frame(torch, ao, depth, seen, "f32", d, a)


def test_python_render_accepts_corner_views(torch_cuda):
    """render() on rt[:h, :w] (and rt[:, :h, :w]) views of max-size targets, for the depth and for out."""
    torch = torch_cuda
    W, H, Wmax, Hmax = 333, 200, 512, 256
    depth, seen = _depth("f32", W, H, 2, seed=2)
    for L in (1, 2):
        ao = harness.context(W, H, device=0, layers=L)
        rt = torch.full((L, Hmax, Wmax), float("nan"), dtype=torch.float32, device="cuda")
        rt[:, :H, :W] = torch.from_numpy(depth[:L]).cuda()
        out_rt = torch.full((L, Hmax, Wmax), SENTINEL, dtype=torch.uint8, device="cuda")
        dview, oview = (rt[0, :H, :W], out_rt[0, :H, :W]) if L == 1 else (rt[:, :H, :W], out_rt[:, :H, :W])
        r = ao.render(dview, oview)
        assert r.data_ptr() == oview.data_ptr()
        got = out_rt.cpu().numpy()
        for l in range(L):
            assert np.array_equal(got[l, :H, :W], harness.oracle(W, H, threads=8).run(seen[l])), (L, l)
        mask = np.ones(got.shape, bool)
        mask[:, :H, :W] = False
        assert (got[mask] == SENTINEL).all()
        fresh = ao.render(dview)                      # strided depth, a new tight out
        assert np.array_equal(fresh.cpu().numpy().reshape(L, H, W), got[:, :H, :W])
    with pytest.raises(ValueError):
        ao.render(torch.as_strided(rt, (2, H, W), (Hmax * Wmax, Wmax, 2)))      # last stride 2: not a row of pixels


def test_python_render_one_pixel_wide_transposed_tensor(torch_cuda):
    """torch.empty(1, H).t(): shape (H, 1), strides (1, H) -- contiguous for torch, so render() takes it as a W = 1 image."""
    torch = torch_cuda
    H = 48
    depth, seen = _depth("f32", 1, H, 1, seed=4)
    ao = harness.context(1, H, device=0, layers=1)
    d = torch.empty(1, H, dtype=torch.float32, device="cuda")
    d.copy_(torch.from_numpy(np.ascontiguousarray(depth[0].T)))
    d = d.t()                                                                 # (H, 1), strides (1, H)
    assert d.shape == (H, 1) and d.stride() == (1, H)
    out = torch.empty(1, H, dtype=torch.uint8, device="cuda").t()
    ao.render(d, out)
    assert np.array_equal(out.cpu().numpy(), harness.oracle(1, H, threads=8).run(seen[0]))
