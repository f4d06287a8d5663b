"""CPU tests of per-layer projections (meao_set_layer_projections) on plan-only contexts: the setter's and the getter's semantics, return
values and generation; the clearing by a layer change, inside a layer reservation as host bookkeeping; every restriction an orthographic
layer carries, in both orders; each layer's constants against a single-layer context of that projection and camera; uniform tables
against the context projection; and the Python component's opt-in."""
import ctypes as C

import pytest

import harness
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
CAM = (0.5, 80.0, 6.0, 1)


def _create(layers=1, W=160, H=90, cam=CAM, proj=P):
    lib = N.lib()
    h = C.c_void_p()
    assert lib.meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
    assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*cam))) == 0
    if proj != P:
        assert lib.meao_set_projection(h, proj) == 1
    if layers != 1:
        assert lib.meao_set_layers(h, layers) == 1
    if W:
        assert lib.meao_resize(h, W, H) == 1
    return h


def _set(h, table):
    if table is None:
        return N.lib().meao_set_layer_projections(h, None, 0)
    return N.lib().meao_set_layer_projections(h, (C.c_int32 * len(table))(*table), len(table))


def _get(h, capacity=64):
    out = (C.c_int32 * capacity)()
    n = N.lib().meao_get_layer_projections(h, out, capacity)
    assert n >= 0
    return list(out[:n])


def _set_cams(h, cams):
    return N.lib().meao_set_layer_cameras(h, (N.MeaoCamera * len(cams))(*[N.MeaoCamera(*c) for c in cams]), len(cams))


def _error(h):
    return N.lib().meao_last_error(h).decode()


def _fresh_constants(L, **kw):
    """Every constant getter of a fresh plan-only context of L layers."""
    f = _create(L, **kw)
    try:
        return harness.plan_constants(f, L)
    finally:
        N.lib().meao_destroy(f)


def _reservation(h):
    r = N.MeaoReservation()
    assert N.lib().meao_reservation(h, C.byref(r)) == 0
    return r


def test_setter_and_getter():
    lib = N.lib()
    assert lib.meao_set_layer_projections(None, None, 0) == N.MEAO_ERR_INVALID
    assert lib.meao_get_layer_projections(None, None, 0) == N.MEAO_ERR_INVALID
    h = _create(4)
    assert _get(h) == []
    assert _set(h, None) == 0                               # nothing to clear
    g = lib.meao_frame_generation(h)
    assert _set(h, [P, O, P, O]) == 1
    assert lib.meao_frame_generation(h) == g + 1
    assert _get(h) == [P, O, P, O]
    assert _set(h, [P, O, P, O]) == 0 and lib.meao_frame_generation(h) == g + 1
    assert _set(h, [O, O, P, O]) == 1 and lib.meao_frame_generation(h) == g + 2
    small = (C.c_int32 * 3)()
    assert lib.meao_get_layer_projections(h, small, 3) == N.MEAO_ERR_INVALID       # does not fit
    assert lib.meao_get_layer_projections(h, None, 4) == N.MEAO_ERR_INVALID
    # refusals name the layer and the field, and change nothing
    for table, what in (([P, O, 2, O], "layer 2: projection 2"), ([-1, O, P, O], "layer 0: projection -1"),
                        ([P, O, P], "count 3"), ([P] * 5, "count 5")):
        assert _set(h, table) == N.MEAO_ERR_INVALID, table
        assert what in _error(h), (table, _error(h))
        assert _get(h) == [O, O, P, O] and lib.meao_frame_generation(h) == g + 2
    assert lib.meao_set_layer_projections(h, None, 4) == N.MEAO_ERR_INVALID
    assert "NULL" in _error(h)
    # the context's projection is still recorded under a table, and takes effect when the table goes
    assert lib.meao_set_projection(h, O) == 1
    assert lib.meao_get_projection(h) == O and _get(h) == [O, O, P, O]
    assert _set(h, None) == 1 and lib.meao_frame_generation(h) == g + 4
    assert _get(h) == [] and _set(h, None) == 0
    lib.meao_destroy(h)


def test_single_layer_table():
    h, ref = _create(1), _create(1, proj=O)
    assert _set(h, [O]) == 1
    assert harness.plan_constants(h, 1) == harness.plan_constants(ref, 1)
    N.lib().meao_destroy(h)
    N.lib().meao_destroy(ref)


def test_layer_change_clears_the_table():
    lib = N.lib()
    h = _create(3)
    assert _set(h, [O, P, O]) == 1
    g = lib.meao_frame_generation(h)
    assert lib.meao_set_layers(h, 2) == 1
    assert _get(h) == [] and lib.meao_frame_generation(h) > g
    assert harness.plan_constants(h, 2) == _fresh_constants(2)
    lib.meao_destroy(h)


def test_layer_change_inside_a_reservation_is_bookkeeping():
    lib = N.lib()
    h = _create(4)
    assert lib.meao_reserve_layers(h, 8) == 1
    r0 = _reservation(h)
    assert _set(h, [P, O, O, P]) == 1
    for L in (2, 4, 3, 4):
        g = lib.meao_frame_generation(h)
        assert lib.meao_set_layers(h, L) == 1
        assert _get(h) == [] and lib.meao_frame_generation(h) > g
        r = _reservation(h)
        assert (r.arena_allocations, r.arena_bytes, r.graph_instantiations) == (r0.arena_allocations, r0.arena_bytes, r0.graph_instantiations)
        # the revisited (W, H, 4) plans with the context's projection again, not with the table it was planned under
        assert harness.plan_constants(h, L) == _fresh_constants(L), L
        if L == 3:
            assert _set(h, [O, P, O]) == 1
            assert harness.plan_constants(h, 3) == _mixed_reference(3, [O, P, O])
    lib.meao_destroy(h)


def test_orthographic_layer_restrictions_both_orders():
    lib = N.lib()
    views = (N.MeaoLayerViewport * 2)(N.MeaoLayerViewport(0, 0, 0, 0, 0, 0), N.MeaoLayerViewport(0, 0, 1, 0, 0, 1))
    # a table with an orthographic layer refuses a viewport table ...
    h = _create(2, W=128, H=64)
    assert _set(h, [P, O]) == 1
    g = lib.meao_frame_generation(h)
    assert lib.meao_set_layer_viewports(h, views, 2) == N.MEAO_ERR_UNSUPPORTED
    assert "orthographic layer" in _error(h)
    assert lib.meao_get_layer_viewports(h, None, 0) == 0 and lib.meao_frame_generation(h) == g
    # ... an all-perspective table does not, and a viewport table refuses an orthographic layer
    assert _set(h, [P, P]) == 1
    assert lib.meao_set_layer_viewports(h, views, 2) == 1
    g = lib.meao_frame_generation(h)
    assert _set(h, [O, P]) == N.MEAO_ERR_UNSUPPORTED
    assert "layer 0: projection" in _error(h) and "layer-viewport" in _error(h)
    assert _get(h) == [P, P] and lib.meao_frame_generation(h) == g
    lib.meao_destroy(h)
    # row bands: a single-layer table with its orthographic layer refuses a band, and a band refuses the table
    h = _create(1, W=128, H=64)
    assert _set(h, [O]) == 1
    assert lib.meao_set_row_band(h, 0, 32, -1, 64) == N.MEAO_ERR_UNSUPPORTED
    assert "orthographic layer" in _error(h)
    assert lib.meao_halo_bytes(h, 1) == N.MEAO_ERR_UNSUPPORTED
    assert _set(h, [P]) == 1
    assert lib.meao_set_row_band(h, 0, 32, -1, 64) >= 0
    assert _set(h, [O]) == N.MEAO_ERR_UNSUPPORTED
    assert "row band" in _error(h)
    assert _get(h) == [P]
    lib.meao_destroy(h)
    # the context-level refusals stay as they are: an orthographic context refuses a viewport table whatever the table says
    h = _create(2, W=128, H=64, proj=O)
    assert _set(h, [P, P]) == 1
    assert lib.meao_set_layer_viewports(h, views, 2) == N.MEAO_ERR_UNSUPPORTED
    assert "orthographic projection" in _error(h)
    lib.meao_destroy(h)


def _mixed_reference(L, table, cams=None):
    """What a mixed context's every constant getter must return: each layer's from a single-layer context of its projection and camera,
    with the layer-0 getters from layer 0's."""
    lib = N.lib()
    cams = cams or [CAM] * L
    per = []
    for l in range(L):
        s = _create(1, cam=cams[l], proj=table[l])
        per.append(s)
    parts = []
    for k in range(1, 5):
        for getter, n in ((lib.meao_render_constants, 28), (lib.meao_render_constants_wide, 28), (lib.meao_upsample_constants, 8)):
            out = (C.c_float * n)()
            assert getter(per[0], k, out) == 0
            parts.append(bytes(out))
        for l in range(L):
            for wide in (0, 1):
                out = (C.c_float * 28)()
                assert lib.meao_render_constants_layer(per[l], 0, k, wide, out) == 0
                parts.append(bytes(out))
    out = (C.c_float * 4)()
    assert lib.meao_zbuffer_params(per[0], out) == 0
    parts.append(bytes(out))
    for l in range(L):
        assert lib.meao_zbuffer_params_layer(per[l], 0, out) == 0
        parts.append(bytes(out))
    for s in per:
        lib.meao_destroy(s)
    return b"".join(parts)


@pytest.mark.parametrize("reversed_z", [1, 0])
@pytest.mark.parametrize("table", [[P, O], [O, P, O, O], [O, P] * 3])
@pytest.mark.parametrize("layer_cams", [False, True])
def test_each_layer_has_its_projections_constants(reversed_z, table, layer_cams):
    L = len(table)
    cams = [(0.3 + 0.1 * l, 60.0 + 25 * l, 0.8 + 0.5 * l, reversed_z) for l in range(L)] if layer_cams else [CAM[:3] + (reversed_z,)] * L
    h = _create(L, cam=cams[0])
    if layer_cams:
        assert _set_cams(h, cams) == 1
    assert _set(h, table) == 1
    assert harness.plan_constants(h, L) == _mixed_reference(L, table, cams)
    N.lib().meao_destroy(h)


@pytest.mark.parametrize("proj", [P, O])
@pytest.mark.parametrize("variants", [(0, 0, 0, 0), (0, 1, 15, 0), (1, 0, 5, 0), (0, 0, 0, 1)])
def test_uniform_table_plans_like_the_context_projection(proj, variants):
    L = 3
    h = _create(L, proj=P if proj == O else O)        # the context's projection is the other one: the table alone decides
    ref = _create(L, proj=proj)
    for c in (h, ref):
        N.lib().meao_set_variants(c, C.byref(N.MeaoVariants(*variants)))
    assert _set(h, [proj] * L) == 1
    assert harness.plan_constants(h, L) == harness.plan_constants(ref, L)
    assert N.lib().meao_kernels_per_frame(h) == N.lib().meao_kernels_per_frame(ref)
    N.lib().meao_destroy(h)
    N.lib().meao_destroy(ref)


def test_python_per_layer_projection():
    cam = Camera(160, 90)
    ao = harness.context(cam)
    ao.layers = 2
    ao.layerCameras = [cam, Camera(160, 90, orthographic=True, orthographicSize=3.0)]
    with pytest.raises(ValueError, match="orthographic"):         # the default keeps the check
        ao.LateUpdate()
    ao.perLayerProjection = True
    ao.LateUpdate()
    assert _get(ao._ctx) == [P, O]
    assert ao._lib.meao_get_projection(ao._ctx) == P
    ao.layerCameras = None
    ao.LateUpdate()
    assert _get(ao._ctx) == []
    # a viewport table after an orthographic layer: the table is cleared first, so the change goes through
    ao.layerCameras = [cam, cam]
    ao.layerViewports = [(0, 0, 0, 0, 0, 0), (0, 0, 1, 0, 0, 1)]
    ao.LateUpdate()
    assert _get(ao._ctx) == [P, P]
    ao.close()
