"""GPU tests of CUDA-array frames (meao_render_arrays, meao_bind_event_arrays, meao_release_array) on the H100: the depth read from and
the AO written into real CUDA arrays -- 2-D, layered and cube-map -- must give the bytes of meao_render on the same depth and of the
oracle, through graph replay, the plugin event and the debug buffers; every documented refusal launches nothing.

The arrays are made with the CUDA runtime through ctypes (libcudart.so.12, loaded after torch so the process has one dynamic runtime)."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import KIND_UNORM8, KIND_UNORM16, LAYERED, Array, rt, torch_cuda  # noqa: F401  (the fixtures)

pytestmark = pytest.mark.gpu


def _pointer_frame(torch, ao, depth, linear=False):
    d = torch.from_numpy(np.ascontiguousarray(depth if ao.layers > 1 else depth[0])).cuda()
    return ao.render(d, linear=linear).cpu().numpy().reshape(depth.shape)


def _stacked_buffers(ao, ids):
    return {bid: ao.debug_buffer(bid).copy() for bid in ids}


def _depth_for(kind, W, H, L, seed=0, reversed_z=True):
    raw = harness.frames(W, H, L, seed=seed, reversed_z=reversed_z)
    if kind == "d16":
        return harness.ingest(raw, "d16")
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
    ao = harness.context(W, H, device=0, layers=L, **kw)
    linear = kind == "linear_f32"
    ptr = _pointer_frame(torch, ao, depth, linear=linear)
    ids = harness.buffer_ids(kw.get("high_quality_mask", 0), kw.get("single_scale", False))
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
                if kw.get("stereo"):
                    okw["tan_half_fov_h_"] = 1.0 / ao.camera.projection00
                ref = harness.oracle(W, H, stereo=kw.get("stereo", False), linear=linear, threads=8, **okw).run(as_float[l])
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
    ao = harness.context(W, H, device=0, layers=1)
    da = Array(rt, W, H, np.uint16, kind=KIND_UNORM16)
    aa = Array(rt, W, H, np.uint8, kind=KIND_UNORM8)
    try:
        da.fill(depth)
        ao.render_arrays(da.handle, aa.handle, kind="d16")
        torch_cuda.cuda.synchronize()
        assert np.array_equal(aa.read()[0], harness.oracle(W, H, threads=8).run(as_float[0]))
    finally:
        ao.release_array(da.handle); ao.release_array(aa.handle)
        da.free(); aa.free()


def _replay_check(torch, rt, stream=None):
    W, H, L = 400, 240, 2
    ao = harness.context(W, H, device=0, layers=L)
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
                depth = harness.frames(W, H, L, seed=30 + 2 * f + i)
                refs = [harness.oracle(W, H, threads=8).run(depth[l]) for l in range(L)]
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
    ao = harness.context(W, H, device=0, layers=1)
    for round_ in range(3):
        depth = harness.frames(W, H, 1, seed=50 + round_)
        da, aa = Array(rt, W, H, np.float32), Array(rt, W, H, np.uint8)
        try:
            da.fill(depth)
            ao.render_arrays(da.handle, aa.handle)
            ao.render_arrays(da.handle, aa.handle)          # replay
            torch_cuda.cuda.synchronize()
            assert np.array_equal(aa.read()[0], harness.oracle(W, H, threads=8).run(depth[0])), round_
        finally:
            ao.release_array(da.handle)
            ao.release_array(aa.handle)
            da.free(); aa.free()
    ao.release_array(12345)                                 # never used: nothing to do


def test_event_path_and_debug_buffer(torch_cuda, rt):
    from miniengineao_b200 import _native as N
    W, H = 300, 170
    ao = harness.context(W, H, device=0, layers=1)
    ao.LateUpdate()
    depth = harness.frames(W, H, 1, seed=60)
    ref = harness.oracle(W, H, threads=8).run(depth[0])
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
    ao = harness.context(W, H, device=0, layers=1)
    ao.LateUpdate()
    lib, ctx = N.lib(), ao._ctx
    made = []

    def arr(*a, **k):
        x = Array(rt, *a, **k)
        made.append(x)
        return x

    good_d, good_o = arr(W, H, np.float32), arr(W, H, np.uint8)
    depth = harness.frames(W, H, 1, seed=70)
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
        sq = harness.context(64, 64, device=0, layers=6)
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
        assert np.array_equal(good_o.read()[0], harness.oracle(W, H, threads=8).run(depth[0]))
        sq.release_array(cube_d.handle); sq.release_array(cube_o.handle); sq.release_array(cube_arr.handle)
    finally:
        for x in made:
            ao.release_array(x.handle)
            x.free()
