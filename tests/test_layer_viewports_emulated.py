"""CPU tests of layer viewports (meao_set_layer_viewports): each layer of a layered CUDA-array frame at its own rectangle and array
layer of the caller's depth and AO arrays -- split-screen players in one 2-D texture, cube faces into a 2-D atlas.

The table kernels (build.py VIEW_SOURCES) run in the fiber emulator (tests/emu/frame_layer_views.cpp, linked against the emulator the
other CPU tests use).  Every array case compares each layer's AO rectangle with the single-layer viewport frame (meao_render_arrays_at,
tests/emu/frame_views.cpp) of that rectangle and that layer's camera, checks that every AO byte outside the rectangles keeps its
sentinel, and that the frame makes exactly one surface access per depth texel and per AO byte of its rectangles.  The pointer cases
(meao_render_pitched) compare each layer with the single-layer fused frame of a tight copy, in every depth format, with one layer
whose base misses the vector alignment.  Also here: the
plan-only contract of the table (set, get, clear, refusals, the layer-count reset, meao_frame_generation)."""
import ctypes as C

import numpy as np
import pytest

from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

import harness
from emu import emu, layer_views, views  # noqa: E402  (tests/ is on sys.path via conftest)
from emu.emu import Frame  # noqa: E402

SENTINEL = 0xA5
# (near, far, vertical field of view): every layer its own camera
CAMS = [(0.3, 100.0, 60.0), (0.1, 1000.0, 90.0), (0.5, 50.0, 40.0), (0.2, 300.0, 75.0), (1.0, 80.0, 50.0), (0.05, 20.0, 100.0)]


def _cameras(W, H, L, reversed_z=True):
    return [Camera(W, H, nearClipPlane=n, farClipPlane=f, fieldOfView=v, usesReversedZBuffer=reversed_z) for n, f, v in CAMS[:L]]


def _poisoned(shape, dtype):
    """Poison in every texel no layer reads: NaN, +inf, -inf, 0 (float32); 0 and 65535 (D16 codes)"""
    n = int(np.prod(shape))
    vals = np.array([np.nan, np.inf, -np.inf, 0.0], np.float32) if np.dtype(dtype) == np.float32 else np.array([0, 65535], np.uint16)
    return np.resize(vals, n).reshape(shape)


def _layer_depth(W, H, L, kind, seed, reversed_z=True):
    """(the layers' depth in the format of `kind` [L, H, W], linear?)"""
    lin = harness.contrasting_layers(W, H, L, seed=seed)
    if kind == "linear_f32":
        return lin, True
    r = harness.raw(lin, reversed_z=reversed_z)
    if kind in ("d16", "d24s8"):
        return harness.ingest(r, kind)[0], False
    return r, False


def _table_frame(W, H, table, kind, *, depth_shape, depth_ext, ao_shape, ao_ext, seed=0, reversed_z=True, **kw):
    """One table frame of len(table) layers.  depth_ext / ao_ext: (slices, height, width) of the arrays.  Checks every layer against
    its single-layer viewport frame, the sentinel outside the AO rectangles and the surface-access count; returns the AO array."""
    L = len(table)
    depth, linear = _layer_depth(W, H, L, kind, seed, reversed_z)
    darr = _poisoned(depth_ext, depth.dtype)
    aarr = np.full(ao_ext, SENTINEL, np.uint8)
    written = np.zeros(ao_ext, bool)
    for l, (dx, dy, ds, ax, ay, as_) in enumerate(table):
        darr[ds, dy:dy + H, dx:dx + W] = depth[l]
        written[as_, ay:ay + H, ax:ax + W] = True
    cams = _cameras(W, H, L, reversed_z)
    f = Frame(harness.context(W, H, layers=L, layer_cameras=cams, reversed_z=reversed_z, **kw), linear=linear)
    n0 = f.surface_accesses()
    layer_views.run_arrays_views(f, darr, aarr, table, depth_shape, ao_shape)
    assert f.surface_accesses() - n0 == 2 * L * W * H, "a surface access outside the rectangles, or one missing"
    tag = f"{W}x{H} L={L} {kind} {depth_shape}->{ao_shape} {kw}"
    assert (aarr[~written] == SENTINEL).all(), f"{tag}: a store outside the AO rectangles"
    for l, (dx, dy, ds, ax, ay, as_) in enumerate(table):
        one = Frame(harness.context(cams[l], **kw), linear=linear)
        ref = np.full((1, H, W), SENTINEL, np.uint8)
        mine = np.ascontiguousarray(darr[ds:ds + 1, dy:dy + H, dx:dx + W])     # what the rectangle holds (layers may share one)
        views.run_arrays_at(one, mine, (0, 0), ref, (0, 0), "2d")
        assert np.array_equal(aarr[as_, ay:ay + H, ax:ax + W], ref[0]), f"{tag}: layer {l} differs from its single-layer frame"
    return aarr


@pytest.mark.parametrize("hq", [0, 1])
@pytest.mark.parametrize("kind", ["raw_f32", "linear_f32", "d16"])
def test_two_players_side_by_side_in_one_2d_array(kind, hq):
    """Split-screen: two 83 x 61 views side by side in one 166 x 61 depth texture and one AO texture; high_quality_mask bit 0 selects
    the premin final level."""
    W, H = 83, 61
    _table_frame(W, H, [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)], kind, depth_shape="2d", depth_ext=(1, H, 2 * W), ao_shape="2d",
                 ao_ext=(1, H, 2 * W), seed=1, high_quality_mask=hq)


def test_four_quadrants_with_a_border_and_other_origins_in_the_ao():
    """Four players in the quadrants of a depth texture with a 3-texel border, their AO in another arrangement of a larger target"""
    W, H = 70, 45
    b = 3
    table = [(b, b, 0, 0, H, 0), (b + W, b, 0, W, H, 0), (b, b + H, 0, 0, 0, 0), (b + W, b + H, 0, W + 9, 0, 0)]
    _table_frame(W, H, table, "raw_f32", depth_shape="2d", depth_ext=(1, 2 * H + 2 * b, 2 * W + 2 * b), ao_shape="2d",
                 ao_ext=(1, 2 * H + 5, 2 * W + 9), seed=2, intensity=1.1)


@pytest.mark.parametrize("kind", ["raw_f32", "d16"])
def test_cube_faces_into_a_3x2_atlas(kind):
    """The six faces of a cube-map depth into the cells of one 2-D AO atlas"""
    W = 61
    table = [(0, 0, face, (face % 3) * W, (face // 3) * W, 0) for face in range(6)]
    _table_frame(W, W, table, kind, depth_shape="cube", depth_ext=(6, W, W), ao_shape="2d", ao_ext=(1, 2 * W, 3 * W), seed=3)


def test_layers_swap_slices_and_share_a_depth_rectangle():
    """Slices in another order than the layers; two layers read the same depth rectangle (reads may overlap) and write different AO
    slices -- their AO then differs only by camera"""
    W, H = 64, 40
    table = [(5, 2, 1, 0, 0, 2), (5, 2, 1, 1, 1, 0), (0, 0, 0, 3, 0, 1)]
    _table_frame(W, H, table, "raw_f32", depth_shape="layered", depth_ext=(2, H + 2, W + 5), ao_shape="layered", ao_ext=(3, H + 1, W + 3),
                 seed=4)


# ---- pointer frames (meao_render_pitched) ---------------------------------------------------------------------------------------
def _pitched_frame(W, H, table, kind, *, depth_row, depth_slice, ao_row, ao_slice, slices, seed=0, reversed_z=True, **kw):
    """One fused pointer frame with a table: the depth in a flat buffer of `slices` slices of depth_slice elements (rows depth_row
    elements apart), the AO likewise in bytes.  Every layer's rectangle must equal the single-layer fused frame of a tight copy with
    that layer's camera, and every AO byte outside the rectangles keeps its sentinel."""
    L = len(table)
    depth, linear = _layer_depth(W, H, L, kind, seed, reversed_z)
    es = depth.itemsize
    dbuf = _poisoned((slices * depth_slice,), np.float32 if depth.dtype == np.float32 else np.uint16).astype(depth.dtype)
    dbuf = emu._aligned(dbuf)
    abuf = emu._aligned(np.full(slices * ao_slice, SENTINEL, np.uint8))
    written = np.zeros(abuf.shape, bool)
    for l, (dx, dy, ds, ax, ay, as_) in enumerate(table):
        for r in range(H):
            o = ds * depth_slice + (dy + r) * depth_row + dx
            dbuf[o:o + W] = depth[l, r]
            o = as_ * ao_slice + (ay + r) * ao_row + ax
            written[o:o + W] = True
    cams = _cameras(W, H, L, reversed_z)
    f = Frame(harness.context(W, H, layers=L, layer_cameras=cams, reversed_z=reversed_z, **kw), linear=linear)
    layer_views.run_pitched_views(f, dbuf, (depth_row * es, depth_slice * es), abuf, (ao_row, ao_slice), table)
    tag = f"{W}x{H} L={L} {kind} pitched {kw}"
    assert (abuf[~written] == SENTINEL).all(), f"{tag}: a store outside the AO rectangles"
    for l, (dx, dy, ds, ax, ay, as_) in enumerate(table):
        one = Frame(harness.context(cams[l], **kw), linear=linear)
        one.run_fused(np.ascontiguousarray(depth[l]))
        got = np.stack([abuf[as_ * ao_slice + (ay + r) * ao_row + ax:][:W] for r in range(H)])
        assert np.array_equal(got, one.buffer(17)), f"{tag}: layer {l} differs from its single-layer frame"


@pytest.mark.parametrize("kind", ["raw_f32", "linear_f32", "d16", "d24s8"])
def test_pitched_side_by_side_pair_with_a_misaligned_right_half(kind):
    """Side-by-side stereo in one linear buffer: the right eye starts 83 elements into each row, so its base misses the 16-byte
    alignment of the vector loads and the 8-byte one of the vector stores -- its pixels take the element-wise path, the left eye's do not"""
    W, H = 83, 61
    drow, arow = 176, 176          # rows 16-byte aligned in every format: the left eye takes the vector paths
    _pitched_frame(W, H, [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)], kind, depth_row=drow, depth_slice=drow * H, ao_row=arow,
                   ao_slice=arow * H, slices=1, seed=5)


@pytest.mark.parametrize("hq", [0, 1])
def test_pitched_quadrants_and_slices(hq):
    """Four players: two in the top half of slice 0, one in slice 1, one at an odd offset in slice 0's bottom half; the AO in slices
    of another arrangement"""
    W, H = 64, 36
    drow, arow = 2 * W + 16, 2 * W + 8
    dsl, asl = drow * (2 * H + 1), arow * (2 * H + 3)
    table = [(0, 0, 0, 0, 0, 1), (W, 0, 0, W, 0, 1), (3, 1, 1, 1, H + 2, 0), (W + 1, H, 0, 0, 0, 0)]
    _pitched_frame(W, H, table, "raw_f32", depth_row=drow, depth_slice=dsl, ao_row=arow, ao_slice=asl, slices=2, seed=6,
                   high_quality_mask=hq)


# ---- every kernel of the table units, by the launch ledger -----------------------------------------------------------------------
# (io, depth kind, reversed Z, high_quality_mask): together they select every slot of the four units' tables -- the five prepare forms
# of an array, the seven of a pointer (D24S8 too), both Z directions, and the plain and premin final level of every depth format
SLOT_CASES = [("arrays", "linear_f32", True, 0), ("arrays", "raw_f32", True, 1), ("arrays", "raw_f32", False, 0),
              ("arrays", "d16", True, 0), ("arrays", "d16", False, 1),
              ("pitched", "linear_f32", True, 0), ("pitched", "raw_f32", True, 1), ("pitched", "raw_f32", False, 0),
              ("pitched", "d16", True, 0), ("pitched", "d16", False, 1), ("pitched", "d24s8", True, 1), ("pitched", "d24s8", False, 0)]


def _slot_case(io, kind, reversed_z, hq):
    W, H = 40, 24
    table = [(0, 0, 0, 0, 0, 0), (W, 0, 0, W, 0, 0)]
    if io == "arrays":
        _table_frame(W, H, table, kind, depth_shape="2d", depth_ext=(1, H, 2 * W), ao_shape="2d", ao_ext=(1, H, 2 * W), seed=7,
                     reversed_z=reversed_z, high_quality_mask=hq)
    else:
        _pitched_frame(W, H, table, kind, depth_row=2 * W, depth_slice=2 * W * H, ao_row=2 * W, ao_slice=2 * W * H, slices=1, seed=7,
                       reversed_z=reversed_z, high_quality_mask=hq)


@pytest.mark.parametrize("io,kind,reversed_z,hq", SLOT_CASES)
def test_slot_case_matches_the_single_layer_frames(io, kind, reversed_z, hq):
    _slot_case(io, kind, reversed_z, hq)


def test_the_slot_cases_launch_every_table_kernel():
    """The launch ledger of the cases above holds every kernel the table units build, and nothing else of theirs"""
    built = layer_views.kernels()
    assert len(built) == 20, sorted(built)
    ran = set()
    for c in SLOT_CASES:
        emu.ledger_reset()
        _slot_case(*c)
        ran |= layer_views.launched()
    assert ran == built, sorted(built - ran)


# ---- the table on plan-only contexts ---------------------------------------------------------------------------------------
def _plan(L, W=320, H=180):
    a = harness.context(W, H, layers=L)
    a.LateUpdate()
    return a


def _vt(rows):
    return (N.MeaoLayerViewport * len(rows))(*[N.MeaoLayerViewport(*r) for r in rows])


def _get(a):
    cap = int(a.layers)
    out = (N.MeaoLayerViewport * cap)()
    n = N.lib().meao_get_layer_viewports(a._ctx, out, cap)
    return n, [tuple(getattr(v, f) for f, _ in N.MeaoLayerViewport._fields_) for v in out[:max(n, 0)]]


def test_set_get_clear_and_generation():
    a, nl = _plan(2), N.lib()
    rows = [(0, 0, 0, 0, 0, 0), (320, 0, 0, 320, 0, 0)]
    g0 = nl.meao_frame_generation(a._ctx)
    assert nl.meao_set_layer_viewports(a._ctx, _vt(rows), 2) == 1
    g1 = nl.meao_frame_generation(a._ctx)
    assert g1 > g0
    assert _get(a) == (2, rows)
    assert nl.meao_set_layer_viewports(a._ctx, _vt(rows), 2) == 0, "the same table again"
    assert nl.meao_frame_generation(a._ctx) == g1
    moved = [(0, 0, 0, 0, 0, 0), (320, 0, 0, 330, 0, 0)]
    assert nl.meao_set_layer_viewports(a._ctx, _vt(moved), 2) == 1
    g2 = nl.meao_frame_generation(a._ctx)
    assert g2 > g1 and _get(a) == (2, moved)
    small = (N.MeaoLayerViewport * 1)()
    assert nl.meao_get_layer_viewports(a._ctx, small, 1) == N.MEAO_ERR_INVALID, "a capacity below the entry count"
    assert nl.meao_set_layer_viewports(a._ctx, None, 0) == 1
    assert nl.meao_frame_generation(a._ctx) > g2 and _get(a) == (0, [])
    assert nl.meao_set_layer_viewports(a._ctx, None, 0) == 0, "clearing no table"


@pytest.mark.parametrize("field", range(6))
def test_a_negative_coordinate_names_layer_and_field_and_keeps_the_table(field):
    a, nl = _plan(3), N.lib()
    good = [(0, 0, 0, 0, 0, 0), (10, 0, 0, 10, 0, 0), (0, 7, 1, 0, 7, 1)]
    assert nl.meao_set_layer_viewports(a._ctx, _vt(good), 3) == 1
    g = nl.meao_frame_generation(a._ctx)
    bad = [list(r) for r in good]
    bad[2][field] = -1
    assert nl.meao_set_layer_viewports(a._ctx, _vt([tuple(r) for r in bad]), 3) == N.MEAO_ERR_INVALID
    name = [f for f, _ in N.MeaoLayerViewport._fields_][field]
    err = nl.meao_last_error(a._ctx).decode()
    assert "layer 2" in err and name in err, err
    assert _get(a) == (3, good) and nl.meao_frame_generation(a._ctx) == g


def test_count_and_null_refusals():
    a, nl = _plan(2), N.lib()
    assert nl.meao_set_layer_viewports(a._ctx, _vt([(0,) * 6] * 3), 3) == N.MEAO_ERR_INVALID
    assert "3" in nl.meao_last_error(a._ctx).decode() and "2 layers" in nl.meao_last_error(a._ctx).decode()
    assert nl.meao_set_layer_viewports(a._ctx, None, 2) == N.MEAO_ERR_INVALID
    assert _get(a) == (0, [])


def test_a_layer_count_change_clears_the_table():
    a, nl = _plan(2), N.lib()
    assert nl.meao_set_layer_viewports(a._ctx, _vt([(0,) * 6, (320, 0, 0, 320, 0, 0)]), 2) == 1
    assert nl.meao_set_layers(a._ctx, 4) == 1
    assert _get(a) == (0, [])
    assert nl.meao_set_layers(a._ctx, 4) == 0


def test_python_property_hands_the_table_over():
    a = harness.context(320, 180, layers=2)
    a.layerViewports = [(0, 0, 0, 0, 0, 0), (320, 0, 0, 320, 0, 0)]
    assert a.LateUpdate()
    assert _get(a) == (2, [(0, 0, 0, 0, 0, 0), (320, 0, 0, 320, 0, 0)])
    assert not a.LateUpdate(), "the same table every frame is no change"
    a.layerViewports = [(0, 0, 0, 0, 0, 0)]
    with pytest.raises(ValueError):
        a.LateUpdate()
    a.layerViewports = None
    a.LateUpdate()
    assert _get(a) == (0, [])
