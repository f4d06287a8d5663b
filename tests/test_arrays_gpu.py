"""GPU tests of CUDA-array frames (meao_render_arrays, meao_bind_event_arrays, meao_release_array) on the H100: the depth read from and
the AO written into real CUDA arrays -- 2-D, layered and cube-map -- must give the bytes of meao_render on the same depth and of the
oracle, through graph replay, the plugin event and the debug buffers; every documented refusal launches nothing.

The arrays are made with the CUDA runtime through ctypes (libcudart.so.12, loaded after torch so the process has one dynamic runtime)."""
import ctypes as C

import numpy as np
import pytest

from test_layers_gpu import _ctx, _frames, _oracle  # noqa: E402  (tests/ is on sys.path via conftest)

pytestmark = pytest.mark.gpu

LAYERED, SURFACE_LOAD_STORE, CUBEMAP = 0x01, 0x02, 0x04
KIND_UNSIGNED, KIND_FLOAT, KIND_UNORM8, KIND_UNORM16 = 1, 2, 5, 8
H2D, D2H = 1, 2


class ChannelDesc(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("z", C.c_int), ("w", C.c_int), ("f", C.c_int)]


class Extent(C.Structure):
    _fields_ = [("width", C.c_size_t), ("height", C.c_size_t), ("depth", C.c_size_t)]


class Pos(C.Structure):
    _fields_ = [("x", C.c_size_t), ("y", C.c_size_t), ("z", C.c_size_t)]


class PitchedPtr(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("pitch", C.c_size_t), ("xsize", C.c_size_t), ("ysize", C.c_size_t)]


class Memcpy3DParms(C.Structure):
    _fields_ = [("srcArray", C.c_void_p), ("srcPos", Pos), ("srcPtr", PitchedPtr), ("dstArray", C.c_void_p), ("dstPos", Pos),
                ("dstPtr", PitchedPtr), ("extent", Extent), ("kind", C.c_int)]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a GPU")
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def rt(torch_cuda):
    r = C.CDLL("libcudart.so.12")
    r.cudaMallocArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(ChannelDesc), C.c_size_t, C.c_size_t, C.c_uint]
    r.cudaMalloc3DArray.argtypes = [C.POINTER(C.c_void_p), C.POINTER(ChannelDesc), Extent, C.c_uint]
    r.cudaFreeArray.argtypes = [C.c_void_p]
    r.cudaMemcpy3D.argtypes = [C.POINTER(Memcpy3DParms)]
    r.cudaMemcpy2DToArray.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int]
    r.cudaMemcpy2DFromArray.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int]
    return r


class Array:
    """A W x H CUDA array of `layers` layers: shape "2d" (layers 1), "layered" or "cube" (6), one channel of dtype."""
    DT = {np.dtype(np.float32): (32, KIND_FLOAT), np.dtype(np.uint16): (16, KIND_UNSIGNED), np.dtype(np.uint8): (8, KIND_UNSIGNED)}

    def __init__(self, rt, W, H, dtype, shape="2d", layers=1, flags=SURFACE_LOAD_STORE, kind=None, extra_flags=0):
        self.rt, self.W, self.H, self.dtype, self.shape = rt, W, H, np.dtype(dtype), shape
        self.layers = 6 if shape == "cube" else layers
        bits, k = self.DT[self.dtype]
        desc = ChannelDesc(bits, 0, 0, 0, k if kind is None else kind)
        h = C.c_void_p()
        if shape == "2d":
            rc = rt.cudaMallocArray(C.byref(h), C.byref(desc), W, H, flags | extra_flags)
        else:
            f = flags | extra_flags | (CUBEMAP if shape == "cube" else LAYERED)
            rc = rt.cudaMalloc3DArray(C.byref(h), C.byref(desc), Extent(W, H, self.layers), f)
        assert rc == 0, f"array allocation failed ({rc})"
        self.handle = h.value

    def _copy(self, host, to_array):
        if self.shape == "2d":
            wb = self.W * self.dtype.itemsize
            if to_array:
                rc = self.rt.cudaMemcpy2DToArray(C.c_void_p(self.handle), 0, 0, C.c_void_p(host.ctypes.data), wb, wb, self.H, H2D)
            else:
                rc = self.rt.cudaMemcpy2DFromArray(C.c_void_p(host.ctypes.data), wb, C.c_void_p(self.handle), 0, 0, wb, self.H, D2H)
        else:
            p = Memcpy3DParms()
            hp = PitchedPtr(host.ctypes.data, self.W * self.dtype.itemsize, self.W, self.H)
            if to_array:
                p.srcPtr, p.dstArray, p.kind = hp, self.handle, H2D
            else:
                p.srcArray, p.dstPtr, p.kind = self.handle, hp, D2H
            p.extent = Extent(self.W, self.H, self.layers)
            rc = self.rt.cudaMemcpy3D(C.byref(p))
        assert rc == 0, f"array copy failed ({rc})"

    def fill(self, img):
        self._copy(np.ascontiguousarray(img.reshape(self.layers, self.H, self.W), dtype=self.dtype), True)

    def read(self):
        out = np.empty((self.layers, self.H, self.W), self.dtype)
        self._copy(out, False)
        return out

    def free(self):
        if self.handle:
            assert self.rt.cudaFreeArray(C.c_void_p(self.handle)) == 0
            self.handle = None


def _pointer_frame(torch, ao, depth, linear=False):
    d = torch.from_numpy(np.ascontiguousarray(depth if ao.layers > 1 else depth[0])).cuda()
    return ao.render(d, linear=linear).cpu().numpy().reshape(depth.shape)


def _stacked_buffers(ao, ids):
    return {bid: ao.debug_buffer(bid).copy() for bid in ids}


def _depth_for(kind, W, H, L, seed=0, reversed_z=True):
    raw = _frames(W, H, L, seed=seed, reversed_z=reversed_z)
    if kind == "d16":
        codes = np.clip(np.rint(raw.astype(np.float64) * 65535), 0, 65535).astype(np.uint32)
        return codes.astype(np.uint16), (codes.astype(np.float32) * np.float32(1.0 / 65535)).astype(np.float32)
    if kind == "linear_f32":
        from miniengineao_b200 import synth
        lin = np.stack([synth.random_depth(W, H, seed=seed + i) for i in range(L)]).astype(np.float32)
        return lin, lin
    return raw, raw


def _render_and_compare(torch, rt, W, H, L=1, *, kind="raw_f32", depth_shape=None, ao_shape=None, seed=0, oracle=True,
                        buffers=True, **kw):
    depth_shape = depth_shape or ("2d" if L == 1 else "layered")
    ao_shape = ao_shape or depth_shape
    rz = kw.get("reversed_z", True)
    depth, as_float = _depth_for(kind, W, H, L, seed=seed, reversed_z=rz)
    ao = _ctx(W, H, L, **kw)
    linear = kind == "linear_f32"
    ptr = _pointer_frame(torch, ao, depth, linear=linear)
    mask = kw.get("high_quality_mask", 0)
    ids = [1, 2, 3, 4, 5, 10, 17] if kw.get("single_scale") else list(range(1, 18)) + [17 + k for k in range(1, 5) if (mask >> (k - 1)) & 1]
    ptr_bufs = _stacked_buffers(ao, ids) if buffers else None
    da = Array(rt, W, H, depth.dtype, depth_shape, L)
    aa = Array(rt, W, H, np.uint8, ao_shape, L)
    try:
        da.fill(depth)
        aa.fill(np.full((L, H, W), 0x5A, np.uint8))
        if kw.get("stereo"):
            ao.OnPreRender()                        # the next frame is again one draw of both eyes
        ao.render_arrays(da.handle, aa.handle, kind=kind)
        torch.cuda.synchronize()
        got = aa.read()
        assert np.array_equal(got, ptr), f"{W}x{H} L={L} {kind} {kw}: array frame != pointer frame"
        if buffers:
            arr_bufs = _stacked_buffers(ao, ids)
            for bid in ids:
                assert np.array_equal(arr_bufs[bid].view(np.uint8), ptr_bufs[bid].view(np.uint8)), f"buffer {bid} differs"
            assert np.array_equal(arr_bufs[17].reshape(L, H, W), got)             # meao_get_buffer(17) regenerates the AO
        if oracle:
            for l in range(L):
                okw = {k: v for k, v in kw.items() if k != "stereo"}
                ref = _oracle(W, H, stereo=kw.get("stereo", False), linear=linear, ao=ao, **okw).run(as_float[l])
                assert np.array_equal(got[l], ref), f"{W}x{H} {kind} {kw}: layer {l} differs from the oracle"
    finally:
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()
    return ao


@pytest.mark.parametrize("W,H,kind,kw", [
    (1, 1, "raw_f32", {}), (7, 5, "raw_f32", {}), (161, 93, "raw_f32", {}), (161, 93, "raw_f32", dict(reversed_z=False)),
    (161, 93, "linear_f32", {}), (161, 93, "d16", {}), (1920, 1080, "raw_f32", {}), (1920, 1080, "d16", dict(reversed_z=False)),
])
def test_parity_2d(torch_cuda, rt, W, H, kind, kw):
    _render_and_compare(torch_cuda, rt, W, H, kind=kind, **kw)


def test_parity_4k(torch_cuda, rt):
    _render_and_compare(torch_cuda, rt, 3840, 2160, buffers=False)


@pytest.mark.parametrize("kw", [dict(high_quality_mask=1), dict(high_quality_mask=15), dict(sample_exhaustively=True),
                                dict(single_scale=True), dict(stereo=True)])
def test_variants(torch_cuda, rt, kw):
    _render_and_compare(torch_cuda, rt, 322, 203, **kw)


@pytest.mark.parametrize("L,kind", [(2, "raw_f32"), (3, "d16")])
def test_layered_arrays(torch_cuda, rt, L, kind):
    _render_and_compare(torch_cuda, rt, 322, 203, L, kind=kind, intensity=1.1)


@pytest.mark.parametrize("W", [96, 512])
def test_cube_maps(torch_cuda, rt, W):
    _render_and_compare(torch_cuda, rt, W, W, 6, depth_shape="cube", high_quality_mask=1 if W == 96 else 0)


def test_mixed_shapes_and_normalised_formats(torch_cuda, rt):
    """Cube-map depth into a layered AO array; a 2-D depth into a layered AO array of depth 1; unorm channel kinds are accepted."""
    _render_and_compare(torch_cuda, rt, 64, 64, 6, depth_shape="cube", ao_shape="layered", buffers=False)
    _render_and_compare(torch_cuda, rt, 65, 33, 1, depth_shape="2d", ao_shape="layered", buffers=False)
    W, H = 90, 50
    depth, as_float = _depth_for("d16", W, H, 1, seed=4)
    ao = _ctx(W, H, 1)
    da = Array(rt, W, H, np.uint16, kind=KIND_UNORM16)
    aa = Array(rt, W, H, np.uint8, kind=KIND_UNORM8)
    try:
        da.fill(depth)
        ao.render_arrays(da.handle, aa.handle, kind="d16")
        torch_cuda.cuda.synchronize()
        assert np.array_equal(aa.read()[0], _oracle(W, H).run(as_float[0]))
    finally:
        ao.release_array(da.handle); ao.release_array(aa.handle)
        da.free(); aa.free()


def _replay_check(torch, rt, stream=None):
    W, H, L = 400, 240, 2
    ao = _ctx(W, H, L)
    pairs = []
    for i in range(2):
        da, aa = Array(rt, W, H, np.float32, "layered", L), Array(rt, W, H, np.uint8, "layered", L)
        pairs.append((da, aa))
    dptr = torch.empty((L, H, W), dtype=torch.float32, device="cuda")
    optr = torch.empty((L, H, W), dtype=torch.uint8, device="cuda")
    kpf = ao.kernels_per_frame
    try:
        for f in range(3):
            for i, (da, aa) in enumerate(pairs):
                depth = _frames(W, H, L, seed=30 + 2 * f + i)
                refs = [_oracle(W, H).run(depth[l]) for l in range(L)]
                da.fill(depth)
                before = ao.launch_count
                ao.render_arrays(da.handle, aa.handle, stream=stream)
                assert ao.launch_count - before == kpf
                dptr.copy_(torch.from_numpy(depth))
                before = ao.launch_count
                ao.render(dptr, optr, stream=stream)
                assert ao.launch_count - before == kpf
                torch.cuda.synchronize()
                got, ptr = aa.read(), optr.cpu().numpy()
                for l in range(L):
                    assert np.array_equal(got[l], refs[l]), (f, i, l)
                    assert np.array_equal(ptr[l], refs[l]), (f, i, l)
    finally:
        for da, aa in pairs:
            ao.release_array(da.handle); ao.release_array(aa.handle)
            da.free(); aa.free()


def test_replay_alternating_pointers_and_two_array_pairs(torch_cuda, rt):
    _replay_check(torch_cuda, rt)


def test_replay_on_a_non_default_stream(torch_cuda, rt):
    s = torch_cuda.cuda.Stream()
    with torch_cuda.cuda.stream(s):
        _replay_check(torch_cuda, rt, stream=s)


def test_release_then_free_and_reallocate(torch_cuda, rt):
    """After meao_release_array an array may be freed; a new one of the same shape (possibly the same handle) renders correctly."""
    W, H = 256, 144
    ao = _ctx(W, H, 1)
    for round_ in range(3):
        depth = _frames(W, H, 1, seed=50 + round_)
        da, aa = Array(rt, W, H, np.float32), Array(rt, W, H, np.uint8)
        try:
            da.fill(depth)
            ao.render_arrays(da.handle, aa.handle)
            ao.render_arrays(da.handle, aa.handle)          # replay
            torch_cuda.cuda.synchronize()
            assert np.array_equal(aa.read()[0], _oracle(W, H).run(depth[0])), round_
        finally:
            ao.release_array(da.handle)
            ao.release_array(aa.handle)
            da.free(); aa.free()
    ao.release_array(12345)                                 # never used: nothing to do


def test_event_path_and_debug_buffer(torch_cuda, rt):
    from miniengineao_b200 import _native as N
    W, H = 300, 170
    ao = _ctx(W, H, 1)
    ao.LateUpdate()
    depth = _frames(W, H, 1, seed=60)
    ref = _oracle(W, H).run(depth[0])
    da, aa = Array(rt, W, H, np.float32), Array(rt, W, H, np.uint8)
    lib, ctx = N.lib(), ao._ctx
    try:
        da.fill(depth)
        stream = C.c_void_p(torch_cuda.cuda.current_stream().cuda_stream)
        assert lib.meao_bind_event_arrays(ctx, 77, C.c_void_p(da.handle), 0, C.c_void_p(aa.handle), stream) == 0
        before = ao.launch_count
        lib.meao_get_render_event_func()(77)
        assert ao.launch_count - before == ao.kernels_per_frame
        torch_cuda.cuda.synchronize()
        assert np.array_equal(aa.read()[0], ref)
        assert np.array_equal(ao.debug_buffer(17), ref)                     # meao_get_buffer(17) after an array frame
        assert np.array_equal(ao.debug_view(17).cpu().numpy(), ref)         # meao_debug_view(17) too
        assert lib.meao_bind_event_arrays(ctx, 77, None, 0, None, None) == 0
        before = ao.launch_count
        lib.meao_get_render_event_func()(77)                                 # unbound: nothing
        assert ao.launch_count == before
        assert lib.meao_bind_event_arrays(ctx, 78, C.c_void_p(da.handle), 0, C.c_void_p(aa.handle), stream) == 0
        ao.release_array(da.handle)                                          # removes the binding that names it
        lib.meao_get_render_event_func()(78)
        assert ao.launch_count == before
    finally:
        ao.release_array(da.handle); ao.release_array(aa.handle)
        da.free(); aa.free()


def test_refusals_launch_nothing(torch_cuda, rt):
    from miniengineao_b200 import _native as N
    W, H = 160, 96
    ao = _ctx(W, H, 1)
    ao.LateUpdate()
    lib, ctx = N.lib(), ao._ctx
    made = []

    def arr(*a, **k):
        x = Array(rt, *a, **k)
        made.append(x)
        return x

    good_d, good_o = arr(W, H, np.float32), arr(W, H, np.uint8)
    depth = _frames(W, H, 1, seed=70)
    good_d.fill(depth)
    cases = [
        ("extent", arr(W + 1, H, np.float32), good_o, 0, N.MEAO_ERR_INVALID, b"extent"),
        ("channel format", arr(W, H, np.uint16), good_o, 0, N.MEAO_ERR_INVALID, b"channel"),
        ("AO channel format", good_d, arr(W, H, np.uint16), 0, N.MEAO_ERR_INVALID, b"ao_array"),
        ("no SurfaceLoadStore", arr(W, H, np.float32, flags=0), good_o, 0, N.MEAO_ERR_INVALID, b"SurfaceLoadStore"),
        ("layer count", arr(W, H, np.float32, "layered", 2), good_o, 0, N.MEAO_ERR_INVALID, b"layer count"),
        ("cube map with L != 6", arr(64, 64, np.float32, "cube"), good_o, 0, N.MEAO_ERR_INVALID, b"extent"),
        ("D24S8", good_d, good_o, 3, N.MEAO_ERR_UNSUPPORTED, b"D24S8"),
        ("NULL depth", None, good_o, 0, N.MEAO_ERR_INVALID, b"NULL"),
        ("NULL AO", good_d, None, 0, N.MEAO_ERR_INVALID, b"NULL"),
        ("bad kind", good_d, good_o, 9, N.MEAO_ERR_INVALID, b"kind"),
    ]
    try:
        for tag, d, o, kind, want, text in cases:
            before = ao.launch_count
            rc = lib.meao_render_arrays(ctx, C.c_void_p(d.handle if d else None), kind, C.c_void_p(o.handle if o else None), None)
            assert rc == want, (tag, rc, lib.meao_last_error(ctx))
            assert text in lib.meao_last_error(ctx), (tag, lib.meao_last_error(ctx))
            assert ao.launch_count == before, tag
            rc = lib.meao_bind_event_arrays(ctx, 5, C.c_void_p(d.handle if d else None), kind, C.c_void_p(o.handle if o else None), None)
            assert rc == want, (tag, "bind", rc)
        # a square context: a cube map needs 6 layers, a cube-map array is refused as such
        sq = _ctx(64, 64, 6)
        sq.LateUpdate()
        cube_d, cube_o = arr(64, 64, np.float32, "cube"), arr(64, 64, np.uint8, "cube")
        cube_arr = arr(64, 64, np.float32, "cube", extra_flags=LAYERED, layers=6)
        sqctx = sq._ctx
        before = sq.launch_count
        assert lib.meao_render_arrays(sqctx, C.c_void_p(cube_arr.handle), 0, C.c_void_p(cube_o.handle), None) == N.MEAO_ERR_UNSUPPORTED
        assert b"cube-map arrays" in lib.meao_last_error(sqctx)
        sq.layers = 2
        sq.LateUpdate()
        assert lib.meao_render_arrays(sqctx, C.c_void_p(cube_d.handle), 0, C.c_void_p(cube_o.handle), None) == N.MEAO_ERR_INVALID
        assert b"layer count" in lib.meao_last_error(sqctx)
        assert sq.launch_count == before
        # a row band
        ao.set_row_band(0, 48, -1, 96)
        before = ao.launch_count
        assert lib.meao_render_arrays(ctx, C.c_void_p(good_d.handle), 0, C.c_void_p(good_o.handle), None) == N.MEAO_ERR_UNSUPPORTED
        assert b"row band" in lib.meao_last_error(ctx)
        assert ao.launch_count == before
        ao.set_row_band(0, H, -1, -1)
        # the context still renders correctly
        ao.render_arrays(good_d.handle, good_o.handle)
        torch_cuda.cuda.synchronize()
        assert np.array_equal(good_o.read()[0], _oracle(W, H).run(depth[0]))
        sq.release_array(cube_d.handle); sq.release_array(cube_o.handle); sq.release_array(cube_arr.handle)
    finally:
        for x in made:
            ao.release_array(x.handle)
            x.free()
