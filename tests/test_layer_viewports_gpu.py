"""GPU tests of layer viewports (meao_set_layer_viewports) on the H100: one layered frame whose layers live at their own rectangles of
shared CUDA arrays or pitched buffers -- two 960 x 1080 split-screen halves of a 1080p target, four 1920 x 1080 quadrants of a 4K one --
each with its own camera.  Every layer's AO and every debug buffer must equal, bit for bit, the single-layer frame of that rectangle
with that layer's camera (meao_render_arrays_at / meao_render_pitched on a fresh context), which the other GPU tests check against
the oracle; every AO byte outside the rectangles keeps its sentinel.  Also: MEAO_FLAG_NO_GRAPH, a table change inside a reservation
without a graph instantiation, a torch.cuda.graph capture after one settling frame, a bound plugin event, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import Array, rt, torch_cuda  # noqa: F401  (the fixtures)
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
CAMS = [(0.3, 100.0, 60.0), (0.1, 1000.0, 90.0), (0.5, 50.0, 40.0), (0.2, 300.0, 75.0)]


def _cams(W, H, L, reversed_z=True):
    return [Camera(W, H, nearClipPlane=n, farClipPlane=f, fieldOfView=v, usesReversedZBuffer=reversed_z) for n, f, v in CAMS[:L]]


def _depth(kind, W, H, L, seed, reversed_z=True):
    if kind == "linear_f32":
        return harness.contrasting_layers(W, H, L, seed=seed)
    raw = harness.frames(W, H, L, seed=seed, reversed_z=reversed_z)
    return harness.ingest(raw, kind)[0] if kind in ("d16", "d24s8") else raw


KINDS = {"raw_f32": N.MEAO_DEPTH_RAW_F32, "linear_f32": N.MEAO_DEPTH_LINEAR_F32, "d16": N.MEAO_DEPTH_RAW_D16_UNORM,
         "d24s8": N.MEAO_DEPTH_RAW_D24S8}


def _table_ctx(W, H, table, cams, use_graph=True, **kw):
    ao = harness.context(W, H, device=0, layers=len(table), layer_cameras=cams, use_graph=use_graph, **kw)
    ao.layerViewports = table
    ao.LateUpdate()
    return ao


def _single_array_frame(cam, darr, dorg, kind, W, H, rt, **kw):
    """The single-layer meao_render_arrays_at frame of one rectangle with one camera: (AO [H, W], {id: debug buffer})"""
    one = harness.context(cam, device=0, **kw)
    aa = Array(rt, W, H, np.uint8)
    try:
        one.render_arrays(darr.handle, aa.handle, kind=kind, depth_origin=dorg, ao_origin=(0, 0))
        out = aa.read()[0]
        bufs = {b: one.debug_buffer(b) for b in harness.buffer_ids(kw.get("high_quality_mask", 0))}
    finally:
        one.release_array(darr.handle)
        one.release_array(aa.handle)
        aa.free()
        one.close()
    return out, bufs


def _check_layers(ao, got, table, refs, W, H, tag, debug=True):
    """got: the whole AO image [h, w] of slice 0; refs: per layer (AO, debug buffers)"""
    written = np.zeros(got.shape, bool)
    for l, (_, _, _, ax, ay, _) in enumerate(table):
        assert harness.n_diff(got[ay:ay + H, ax:ax + W], refs[l][0]) == 0, f"{tag}: layer {l}'s AO"
        written[ay:ay + H, ax:ax + W] = True
    assert (got[~written] == SENTINEL).all(), f"{tag}: a byte outside the rectangles changed"
    if debug:
        for b, ref in refs[0][1].items():
            mine = ao.debug_buffer(b)
            for l in range(len(table)):
                assert np.array_equal(mine[l], refs[l][1][b]), f"{tag}: layer {l} debug buffer {b}"


def _array_case(torch, rt, W, H, table, ext, kind, tag, reversed_z=True, **kw):
    """A table frame into one 2-D depth array and one 2-D AO array of extent ext = (w, h); checked layer by layer."""
    L = len(table)
    cams = _cams(W, H, L, reversed_z)
    depth = _depth(kind, W, H, L, seed=W + L, reversed_z=reversed_z)
    full = np.zeros((1, ext[1], ext[0]), depth.dtype)
    for l, (dx, dy, _, _, _, _) in enumerate(table):
        full[0, dy:dy + H, dx:dx + W] = depth[l]
    da, aa = Array(rt, *ext, depth.dtype), Array(rt, *ext, np.uint8)
    ao = _table_ctx(W, H, table, cams, reversed_z=reversed_z, **kw)
    try:
        da.fill(full)
        aa.fill(np.full((1, ext[1], ext[0]), SENTINEL, np.uint8))
        before = ao.launch_count
        ao.render_arrays(da.handle, aa.handle, kind=kind)
        assert ao.launch_count - before == ao.kernels_per_frame
        torch.cuda.synchronize()
        got = aa.read()[0]
        refs = [_single_array_frame(cams[l], da, table[l][:2], kind, W, H, rt, **kw) for l in range(L)]
        _check_layers(ao, got, table, refs, W, H, tag)
    finally:
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()
        ao.close()


# ---- 1. parity at real sizes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["raw_f32", "d16"])
def test_two_players_1080p_arrays(torch_cuda, rt, kind):
    W, H = 960, 1080
    _array_case(torch_cuda, rt, W, H, [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)], (2 * W, H), kind, f"2p {kind}", high_quality_mask=1)


def test_four_quadrants_of_4k_arrays(torch_cuda, rt):
    W, H = 1920, 1080
    table = [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0), (0, H, 0, 0, H, 0), (W, H, 0, W, H, 0)]
    _array_case(torch_cuda, rt, W, H, table, (2 * W, 2 * H), "raw_f32", "4p 4K")


def _pitched_case(torch, W, H, table, row, kind, tag, use_graph=True, reversed_z=True, hq=0):
    """A table frame into one torch depth image and one AO image of rows `row` elements (a single slice), against meao_render_pitched
    on the rectangle of each layer with its camera."""
    L = len(table)
    cams = _cams(W, H, L, reversed_z)
    depth = _depth(kind, W, H, L, seed=7 + W, reversed_z=reversed_z)
    rows = max(ay + H for *_, ay, _ in table)
    full = np.zeros((rows, row), depth.dtype)
    for l, (dx, dy, _, _, _, _) in enumerate(table):
        full[dy:dy + H, dx:dx + W] = depth[l]
    d = torch.from_numpy(full.view({np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32}.get(depth.dtype, depth.dtype))).cuda()
    out = torch.full((rows, row), SENTINEL, dtype=torch.uint8, device="cuda")
    es = depth.itemsize
    k = KINDS[kind]
    ao = _table_ctx(W, H, table, cams, use_graph=use_graph, reversed_z=reversed_z, high_quality_mask=hq)
    try:
        ao._check(ao._lib.meao_render_pitched(ao._ctx, C.c_void_p(d.data_ptr()), row * es, row * es * rows, k, C.c_void_p(out.data_ptr()),
                                              row, row * rows, ao._stream()))
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        refs = []
        for l, (dx, dy, _, ax, ay, _) in enumerate(table):
            one = harness.context(cams[l], device=0, high_quality_mask=hq)
            one.LateUpdate()
            o1 = torch.full((H, W), SENTINEL, dtype=torch.uint8, device="cuda")
            base = d.data_ptr() + (dy * row + dx) * es
            one._check(one._lib.meao_render_pitched(one._ctx, C.c_void_p(base), row * es, row * es * H, k, C.c_void_p(o1.data_ptr()), W, W * H,
                                                    one._stream()))
            torch.cuda.synchronize()
            refs.append((o1.cpu().numpy(), {b: one.debug_buffer(b) for b in harness.buffer_ids(hq)}))
            one.close()
        _check_layers(ao, got, table, refs, W, H, tag)
    finally:
        ao.close()


def test_pitched_side_by_side_halves_1080p(torch_cuda):
    W, H = 960, 1080
    _pitched_case(torch_cuda, W, H, [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)], 2 * W, "raw_f32", "pitched 2p")


def test_pitched_misaligned_right_eye_d16(torch_cuda):
    """The right eye starts 957 elements into each row: its base misses the vector alignment of the depth loads and AO stores"""
    W, H = 957, 540
    _pitched_case(torch_cuda, W, H, [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)], 1920, "d16", "pitched misaligned")


def test_no_graph_flag(torch_cuda):
    W, H = 320, 184
    table = [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0), (0, H, 0, 0, H, 0), (W, H, 0, W + 3, H, 0)]
    _pitched_case(torch_cuda, W, H, table, 2 * W + 16, "raw_f32", "no graph", use_graph=False)


# every slot of the four table units' kernel tables on the hardware: the prepare forms of every depth format in both Z directions, the
# plain and premin final level of every format (tests/test_layer_viewports_emulated.py proves by the launch ledger that these cases
# launch all 20 kernels)
SLOT_CASES = [("arrays", "linear_f32", True, 0), ("arrays", "raw_f32", True, 1), ("arrays", "raw_f32", False, 0),
              ("arrays", "d16", True, 0), ("arrays", "d16", False, 1),
              ("pitched", "linear_f32", True, 0), ("pitched", "raw_f32", True, 1), ("pitched", "raw_f32", False, 0),
              ("pitched", "d16", True, 0), ("pitched", "d16", False, 1), ("pitched", "d24s8", True, 1), ("pitched", "d24s8", False, 0)]


@pytest.mark.parametrize("io,kind,reversed_z,hq", SLOT_CASES)
def test_slot_matrix(torch_cuda, rt, io, kind, reversed_z, hq):
    W, H = 200, 120
    table = [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)]
    tag = f"{io} {kind} rz={reversed_z} hq={hq}"
    if io == "arrays":
        _array_case(torch_cuda, rt, W, H, table, (2 * W, H), kind, tag, reversed_z=reversed_z, high_quality_mask=hq)
    else:
        _pitched_case(torch_cuda, W, H, table, 2 * W, kind, tag, reversed_z=reversed_z, hq=hq)


# ---- 2. the host-buffer calls keep the tight layout ----------------------------------------------------------------------------
@pytest.mark.parametrize("table", [[(0, 0, 0, 0, 0, 0), (64, 0, 0, 64, 0, 0)], [(0, 0, 1, 0, 0, 1), (0, 0, 0, 0, 0, 0)]],
                         ids=["side_by_side", "swapped_slices"])
def test_render_host_ignores_the_table(torch_cuda, table):
    """meao_render_host (and its async form) stages tight L x W x H buffers: with a table set it renders exactly what it renders
    without one -- no refusal for rectangles beyond the tight rows, no reordering of the layers"""
    W, H, L = 64, 48, 2
    cams = _cams(W, H, L)
    depth = _depth("raw_f32", W, H, L, seed=31)
    plain = harness.context(W, H, device=0, layers=L, layer_cameras=cams)
    ref = plain.render_host(depth)
    plain.close()
    ao = _table_ctx(W, H, table, cams)
    try:
        assert np.array_equal(ao.render_host(depth), ref)
        outs = [np.zeros((L, H, W), np.uint8) for _ in range(3)]
        ao.render_host_batch([depth] * 3, outs)
        assert all(np.array_equal(o, ref) for o in outs)
        if table[1][0] == W:        # and the table still governs the device frames of the same context
            d = torch_cuda.from_numpy(np.ascontiguousarray(np.concatenate(list(depth), axis=1))).cuda()
            out = torch_cuda.zeros((H, 2 * W), dtype=torch_cuda.uint8, device="cuda")
            assert ao._lib.meao_render_pitched(ao._ctx, C.c_void_p(d.data_ptr()), 8 * W, 8 * W * H, 0, C.c_void_p(out.data_ptr()), 2 * W,
                                               2 * W * H, ao._stream()) == 0
            torch_cuda.cuda.synchronize()
            got = out.cpu().numpy()
            assert np.array_equal(got[:, :W], ref[0]) and np.array_equal(got[:, W:], ref[1])
    finally:
        ao.close()


def test_pitched_slice_fit_is_exact(torch_cuda):
    """A layer pitch that holds every rectangle exactly renders, even where the rectangle furthest right and the one furthest down are
    different layers; one element (one byte) less is refused, naming the layer whose rectangle overflows"""
    torch = torch_cuda
    W, H, L = 64, 32, 2
    row = 2 * W                                       # elements (depth) and bytes (AO)
    table = [(W, 0, 0, W, 0, 0), (0, 8, 1, 0, 8, 1)]  # layer 0: right, top; layer 1: left, lower, slice 1
    dlp = (8 + H - 1) * row * 4 + W * 4               # layer 1's last byte in its slice (layer 0's ends before: row (H - 1))
    alp = (8 + H - 1) * row + W
    ao = _table_ctx(W, H, table, _cams(W, H, L))
    d = torch.zeros(2 * dlp // 4, dtype=torch.float32, device="cuda")
    a = torch.zeros(2 * alp, dtype=torch.uint8, device="cuda")
    lib, ctx = ao._lib, ao._ctx
    try:
        def frame(dl, al):
            return lib.meao_render_pitched(ctx, C.c_void_p(d.data_ptr()), row * 4, dl, 0, C.c_void_p(a.data_ptr()), row, al, None)
        before = ao.launch_count
        assert frame(dlp - 4, alp) == N.MEAO_ERR_INVALID
        err = lib.meao_last_error(ctx)
        assert b"layer 1" in err and b"depth_layer_pitch" in err, err
        assert frame(dlp, alp - 1) == N.MEAO_ERR_INVALID
        err = lib.meao_last_error(ctx)
        assert b"layer 1" in err and b"ao_layer_pitch" in err, err
        assert ao.launch_count == before
        assert frame(dlp, alp) == 0, lib.meao_last_error(ctx)
        torch.cuda.synchronize()
        assert ao.launch_count - before == ao.kernels_per_frame
    finally:
        ao.close()


# ---- 3. a table change inside a reservation, a capture, an event ------------------------------------------------------------------
def _split_arrays(rt, W, H, L, seed):
    """2-D depth and AO arrays of L side-by-side W x H views, the depth filled; (depth array, AO array, depth [L, H, W])"""
    depth = _depth("raw_f32", W, H, L, seed)
    full = np.concatenate(list(depth), axis=1)[None]
    da, aa = Array(rt, L * W, H, np.float32), Array(rt, L * W, H, np.uint8)
    da.fill(full)
    aa.fill(np.full((1, H, L * W), SENTINEL, np.uint8))
    return da, aa, depth


def _oracle_split(W, H, cams, depth, order):
    """the expected AO image: layer l's oracle AO (its camera, its depth) at column block order[l]"""
    out = np.empty((H, len(order) * W), np.uint8)
    for l, blk in enumerate(order):
        out[:, blk * W:(blk + 1) * W] = harness.oracle(W, H, camera=cams[l], threads=8).run(depth[l])
    return out


def test_table_change_inside_a_reservation_instantiates_nothing(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 480, 270, 2
    cams = _cams(W, H, L)
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams, max_resolution=(960, 540))
    straight = [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)]
    swapped = [(0, 0, 0, W, 0, 0), (W, 0, 0, 0, 0, 0)]        # each player's AO into the other half
    ao.layerViewports = straight
    da, aa, depth = _split_arrays(rt, W, H, L, seed=11)
    try:
        ao.render_arrays(da.handle, aa.handle)
        torch.cuda.synchronize()
        assert np.array_equal(aa.read()[0], _oracle_split(W, H, cams, depth, [0, 1]))
        inst, gen = ao.reservation()["graph_instantiations"], ao.frame_generation
        ao.layerViewports = swapped
        assert ao.LateUpdate(), "a changed table is a change"
        assert ao.frame_generation != gen
        ao.render_arrays(da.handle, aa.handle)
        torch.cuda.synchronize()
        assert np.array_equal(aa.read()[0], _oracle_split(W, H, cams, depth, [1, 0]))
        assert ao.reservation()["graph_instantiations"] == inst, "a table change instantiated a graph"
        # a smaller size under the same table: the rectangles are re-checked and keep their origins
        ao.camera.pixelWidth, ao.camera.pixelHeight = 400, 200
        for c in cams:
            c.pixelWidth, c.pixelHeight = 400, 200
        aa.fill(np.full((1, H, L * W), SENTINEL, np.uint8))
        ao.render_arrays(da.handle, aa.handle)
        torch.cuda.synchronize()
        got = aa.read()[0]
        assert (got[200:] == SENTINEL).all() and (got[:, 400:W] == SENTINEL).all() and (got[:, W + 400:] == SENTINEL).all()
    finally:
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()
        ao.close()


def test_torch_graph_capture_after_one_settling_frame(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 320, 184, 2
    cams = _cams(W, H, L)
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams)
    ao.layerViewports = [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)]
    da, aa, depth = _split_arrays(rt, W, H, L, seed=0)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ao.render_arrays(da.handle, aa.handle)          # the settling frame: tables written, surfaces made
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        gen = ao.frame_generation
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ao.render_arrays(da.handle, aa.handle)
        assert ao.frame_generation == gen
        for i in range(3):
            depth = _depth("raw_f32", W, H, L, seed=i + 1)
            da.fill(np.concatenate(list(depth), axis=1)[None])
            aa.fill(np.full((1, H, L * W), SENTINEL, np.uint8))
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(aa.read()[0], _oracle_split(W, H, cams, depth, [0, 1])), f"replay {i}"
        del g
        torch.cuda.synchronize()
    finally:
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()
        ao.close()


def test_bound_event_renders_with_the_table(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 256, 144, 2
    cams = _cams(W, H, L)
    ao = harness.context(W, H, device=0, layers=L, layer_cameras=cams)
    ao.layerViewports = [(W, 0, 0, 0, 0, 0), (0, 0, 0, W, 0, 0)]     # each player reads the other half
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    da, aa, depth = _split_arrays(rt, W, H, L, seed=21)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    try:
        assert lib.meao_bind_event_arrays(ctx, 93, C.c_void_p(da.handle), 0, C.c_void_p(aa.handle), stream) == 0
        before = ao.launch_count
        lib.meao_get_render_event_func()(93)
        torch.cuda.synchronize()
        assert ao.launch_count - before == ao.kernels_per_frame, lib.meao_last_error(ctx)
        assert np.array_equal(aa.read()[0], _oracle_split(W, H, cams, depth[::-1], [0, 1]))
        lib.meao_bind_event_arrays(ctx, 93, None, 0, None, None)
    finally:
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()
        ao.close()


# ---- 4. refusals ------------------------------------------------------------------------------------------------------------------
def test_refusals_name_layer_and_field_and_launch_nothing(torch_cuda, rt):
    torch = torch_cuda
    W, H, L = 160, 96, 2
    ao = harness.context(W, H, device=0, layers=L)
    ao.layerViewports = [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)]
    ao.LateUpdate()
    lib, ctx = ao._lib, ao._ctx
    da, aa = Array(rt, 2 * W, H, np.float32), Array(rt, 2 * W, H, np.uint8)
    small = Array(rt, 2 * W - 1, H, np.uint8)
    d, a = C.c_void_p(da.handle), C.c_void_p(aa.handle)
    vt = lambda rows: (N.MeaoLayerViewport * len(rows))(*[N.MeaoLayerViewport(*r) for r in rows])   # noqa: E731
    try:
        def refused(rc, want, *texts):
            err = lib.meao_last_error(ctx)
            assert rc == want and all(t in err for t in texts), (rc, err)

        before = ao.launch_count
        refused(lib.meao_render_arrays(ctx, d, 0, C.c_void_p(small.handle), None), N.MEAO_ERR_INVALID, b"layer 1", b"ao_x", b"width")
        refused(lib.meao_render_arrays_at(ctx, d, 0, 0, 0, a, 0, 0, None), N.MEAO_ERR_INVALID, b"meao_render_arrays_at")
        refused(lib.meao_bind_event_arrays_at(ctx, 94, d, 0, 0, 0, a, 0, 0, None), N.MEAO_ERR_INVALID, b"meao_render_arrays_at")
        assert lib.meao_set_layer_viewports(ctx, vt([(0, 0, 0, 0, 0, 0), (W, 1, 0, W, 0, 0)]), 2) == 1
        refused(lib.meao_render_arrays(ctx, d, 0, a, None), N.MEAO_ERR_INVALID, b"layer 1", b"depth_y", b"height")
        assert lib.meao_set_layer_viewports(ctx, vt([(0, 0, 0, 0, 0, 0), (W, 0, 1, W, 0, 0)]), 2) == 1
        refused(lib.meao_render_arrays(ctx, d, 0, a, None), N.MEAO_ERR_INVALID, b"layer 1", b"depth_slice")
        assert lib.meao_set_layer_viewports(ctx, vt([(0, 0, 0, 0, 0, 0), (W, 0, 0, W - 1, 0, 0)]), 2) == 1
        refused(lib.meao_render_arrays(ctx, d, 0, a, None), N.MEAO_ERR_INVALID, b"layer 1", b"layer 0", b"shares texels")
        # a pitched AO whose rows are one byte short for the right player
        dt = torch.zeros((H, 2 * W), dtype=torch.float32, device="cuda")
        ot = torch.zeros((H, 2 * W), dtype=torch.uint8, device="cuda")
        assert lib.meao_set_layer_viewports(ctx, vt([(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)]), 2) == 1
        refused(lib.meao_render_pitched(ctx, C.c_void_p(dt.data_ptr()), 8 * W, 8 * W * H, 0, C.c_void_p(ot.data_ptr()), 2 * W - 1, 2 * W * H,
                                        None), N.MEAO_ERR_INVALID, b"layer 1", b"ao_x", b"ao_row_pitch")
        assert ao.launch_count == before
        # the same table at pitches that fit renders
        assert lib.meao_render_pitched(ctx, C.c_void_p(dt.data_ptr()), 8 * W, 8 * W * H, 0, C.c_void_p(ot.data_ptr()), 2 * W, 2 * W * H,
                                       None) == 0
        torch.cuda.synchronize()
        assert ao.launch_count - before == ao.kernels_per_frame
    finally:
        for x in (da, aa, small):
            ao.release_array(x.handle)
            x.free()
        ao.close()
