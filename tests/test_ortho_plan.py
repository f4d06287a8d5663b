"""CPU tests of orthographic cameras (meao_set_projection): the orthographic oracle's render restatement against meao_oracle.c, what
the projection means on the oracle (depth-shift and scale invariance, a tilted plane), the committed orthographic fixture, the planner's constants, and the setter on
plan-only contexts (return values, re-plan, refusals, frame constants)."""
import ctypes as C

import numpy as np
import pytest

import harness
import ortho_oracle as OO
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N
from oracle import direct_formulation as D


def _ctx(W=160, H=90, cam=(0.5, 80.0, 6.0, 1), proj=N.MEAO_PROJECTION_ORTHOGRAPHIC):
    lib = N.lib()
    h = C.c_void_p()
    assert lib.meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
    assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*cam))) == 0
    if proj != N.MEAO_PROJECTION_PERSPECTIVE:
        assert lib.meao_set_projection(h, proj) == 1
    assert lib.meao_resize(h, W, H) == 1
    return lib, h


@pytest.mark.parametrize("reversed_z", [True, False])
@pytest.mark.parametrize("variant", [{}, dict(sample_exhaustively=True), dict(high_quality_mask=15, sample_exhaustively=True)])
def test_render_restatement_equals_thread_group_oracle(reversed_z, variant):
    """With the perspective formulas the numpy render core reproduces meao_oracle.c's Occlusion / HighQuality codes bit for bit."""
    W, H = 161, 93
    o = harness.oracle(W, H, reversed_z=reversed_z, threads=4, **variant)
    o.run(harness.raw_with_sky(W, H, seed=1, reversed_z=reversed_z))
    dims = D.level_dims(W, H)
    for k in range(1, 5):
        sw, sh = dims[k + 2]
        rc = o.render_constants(k)
        pad = OO.F(1e5) if reversed_z else OO.F(OO.F(1) / OO.F(o.zbuffer_params()[1]))
        codes = OO.render_core(OO.interleaved_tap(o.buffer(1 + k), sw, sh, pad if k <= 2 else 0), dims[k][::-1], rc["inv_thickness"],
                               rc["sample_weight"], rc["reject_fadeoff"], rc["intensity"], variant.get("sample_exhaustively", False), True)
        assert (codes == o.codes(9 + k)).all(), k
        if (variant.get("high_quality_mask", 0) >> (k - 1)) & 1:
            rw = o.render_constants(k, wide=True)
            codes = OO.render_core(OO.wide_tap(o.buffer(1 + k)), dims[k][::-1], rw["inv_thickness"], rw["sample_weight"],
                                   rw["reject_fadeoff"], rw["intensity"], variant.get("sample_exhaustively", False), True)
            assert (codes == o.codes(17 + k)).all(), ("wide", k)


@pytest.mark.parametrize("reversed_z", [True, False])
@pytest.mark.parametrize("stereo", [False, True])
def test_pinned_constants(reversed_z, stereo):
    W, H = 333, 187
    cam = (0.25, 96.0, 7.5, int(reversed_z))
    lib, h = _ctx(W, H, cam)
    if stereo:
        assert lib.meao_set_variants(h, C.byref(N.MeaoVariants(1, 0, 0, 0))) == 1
    orc = OO.OrthoOracle(W, H, near=cam[0], far=cam[1], tan_half_fov_h_=cam[2], reversed_z=reversed_z, single_pass_stereo=stereo)
    zb = (C.c_float * 4)()
    assert lib.meao_zbuffer_params(h, zb) == 0
    assert np.array(zb[:], np.float32).tobytes() == orc.zbuffer_params().tobytes()
    r = np.float32(cam[0]) / np.float32(cam[1])
    assert zb[0] == (np.float32(r - 1) if reversed_z else np.float32(1 - r)) and zb[1] == (1.0 if reversed_z else r)
    for k in range(1, 5):
        for wide in (False, True):
            out = (C.c_float * 28)()
            fn = lib.meao_render_constants_wide if wide else lib.meao_render_constants
            assert fn(h, k, out) == 0
            assert np.array(out[:12], np.float32).tobytes() == orc.inv_thickness(k, wide).tobytes(), (k, wide)
    lib.meao_destroy(h)


def test_setter_plan_only():
    lib, h = _ctx(proj=N.MEAO_PROJECTION_PERSPECTIVE)
    g0 = lib.meao_frame_generation(h)
    assert lib.meao_get_projection(h) == N.MEAO_PROJECTION_PERSPECTIVE
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_ORTHOGRAPHIC) == 1
    assert lib.meao_frame_generation(h) == g0 + 1
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_ORTHOGRAPHIC) == 0
    assert lib.meao_frame_generation(h) == g0 + 1
    for bad in (2, -1, 1 << 20):
        assert lib.meao_set_projection(h, bad) == N.MEAO_ERR_INVALID
        assert b"projection" in lib.meao_last_error(h)
        assert lib.meao_get_projection(h) == N.MEAO_PROJECTION_ORTHOGRAPHIC
    assert lib.meao_frame_generation(h) == g0 + 1
    # the planner follows the projection both ways
    zb = (C.c_float * 4)()
    lib.meao_zbuffer_params(h, zb)
    assert abs(zb[0] - (0.5 / 80.0 - 1)) < 1e-6 and zb[1] == 1.0
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_PERSPECTIVE) == 1
    lib.meao_zbuffer_params(h, zb)
    assert zb[0] == np.float32(np.float32(80.0) / np.float32(0.5)) - 1
    assert lib.meao_get_projection(None) == N.MEAO_ERR_INVALID
    lib.meao_destroy(h)


def test_half_width_is_a_frame_constant():
    lib, h = _ctx()
    out = (C.c_float * 28)()
    lib.meao_render_constants(h, 1, out)
    it0 = out[0]
    g = lib.meao_frame_generation(h)
    assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(0.5, 80.0, 3.0, 1))) == 0
    lib.meao_render_constants(h, 1, out)
    assert out[0] == pytest.approx(2 * it0, rel=1e-6)         # half the half-width: twice it_i, at once
    assert lib.meao_frame_generation(h) == g + 1
    assert lib.meao_get_projection(h) == N.MEAO_PROJECTION_ORTHOGRAPHIC
    lib.meao_destroy(h)


def test_refusals_both_orders():
    lib, h = _ctx(W=128, H=64)
    assert lib.meao_set_layers(h, 2) == 1
    views = (N.MeaoLayerViewport * 2)(N.MeaoLayerViewport(0, 0, 0, 0, 0, 0), N.MeaoLayerViewport(0, 0, 1, 0, 0, 1))
    assert lib.meao_set_layer_viewports(h, views, 2) == N.MEAO_ERR_UNSUPPORTED
    assert b"orthographic" in lib.meao_last_error(h)
    assert lib.meao_get_layer_viewports(h, None, 0) == 0
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_PERSPECTIVE) == 1
    assert lib.meao_set_layer_viewports(h, views, 2) == 1
    g = lib.meao_frame_generation(h)
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_ORTHOGRAPHIC) == N.MEAO_ERR_UNSUPPORTED
    assert b"layer-viewport" in lib.meao_last_error(h)
    assert lib.meao_get_projection(h) == N.MEAO_PROJECTION_PERSPECTIVE and lib.meao_frame_generation(h) == g
    lib.meao_destroy(h)
    # row bands: refused under the projection, and the projection refused with a band
    lib, h = _ctx(W=128, H=64)
    assert lib.meao_set_row_band(h, 0, 32, -1, 64) == N.MEAO_ERR_UNSUPPORTED
    assert b"orthographic" in lib.meao_last_error(h)
    assert lib.meao_halo_bytes(h, 1) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_PERSPECTIVE) == 1
    assert lib.meao_set_row_band(h, 0, 32, -1, 64) >= 0
    assert lib.meao_set_projection(h, N.MEAO_PROJECTION_ORTHOGRAPHIC) == N.MEAO_ERR_UNSUPPORTED
    assert b"row band" in lib.meao_last_error(h)
    assert lib.meao_get_projection(h) == N.MEAO_PROJECTION_PERSPECTIVE
    lib.meao_destroy(h)


def test_python_camera_projection():
    cam = Camera(160, 90, orthographic=True, orthographicSize=4.0)
    assert cam.projection00 == pytest.approx(1.0 / (160 / 90 * 4.0))
    ao = harness.context(cam)
    ao.LateUpdate()
    assert ao._lib.meao_get_projection(ao._ctx) == N.MEAO_PROJECTION_ORTHOGRAPHIC
    ao.layers = 2
    ao.layerCameras = [cam, Camera(160, 90)]
    with pytest.raises(ValueError, match="orthographic"):
        ao.LateUpdate()
    ao.layerCameras = None
    cam.orthographic = False
    ao.LateUpdate()
    assert ao._lib.meao_get_projection(ao._ctx) == N.MEAO_PROJECTION_PERSPECTIVE


# ---- what the projection means, on the oracle -----------------------------------------------------------------------------------------
def _occ(o, linear_depth, **kw):
    o.run(linear_depth)
    return [o.codes(bid).astype(int) for bid in (10, 11, 12, 13)]


def test_depth_shift_invariance():
    """A scene and the same scene moved back by a constant: the same AO under the orthographic projection, not under perspective."""
    W, H = 192, 108
    rng = np.random.default_rng(3)
    step = np.float32(2.0 ** -10)
    base = np.float32(0.25) + step * np.round(rng.uniform(0, 60, (H // 4, W // 4))).astype(np.float32)
    scene = np.kron(base, np.ones((4, 4), np.float32)).astype(np.float32)
    shifted = (scene + np.float32(0.125)).astype(np.float32)
    for a in (scene, shifted):
        assert (D._f16r(a) == a).all()                           # exact in f16: the atlas stores the same geometry
    ortho = [OO.OrthoOracle(W, H, near=0.5, far=100.0, tan_half_fov_h_=0.02, linear=True) for _ in range(2)]
    oa, ob = _occ(ortho[0], scene), _occ(ortho[1], shifted)
    for k in range(4):
        assert np.abs(oa[k] - ob[k]).max() <= 1, k
    persp = [harness.oracle(W, H, linear=True, near=0.5, far=100.0, tan_half_fov_h_=0.02) for _ in range(2)]
    pa, pb = _occ(persp[0], scene), _occ(persp[1], shifted)
    assert max(np.abs(pa[k] - pb[k]).max() for k in range(4)) > 8


def test_scale_invariance():
    """Scaling near, far, the half-width and the scene by a power of two changes no bit."""
    W, H = 150, 90
    raw = harness.raw_with_sky(W, H, seed=4, reversed_z=True)
    outs = []
    for s in (1.0, 4.0, 0.125):
        o = OO.OrthoOracle(W, H, near=0.5 * s, far=60.0 * s, tan_half_fov_h_=3.0 * s, reversed_z=True)
        o.run(raw)
        outs.append([o.codes(b).copy() for b in range(10, 18)])
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert (a == b).all()



def test_tilted_plane_is_unoccluded():
    """A plane tilted in both directions, exact in f16, gives Occlusion1..3 codes within one code of 255 away from its borders (the
    render's reach, 16 level pixels); Occlusion4 of this frame is all border."""
    W, H = 512, 320
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    plane = (0.25 + 2.0 ** -12 * (x + y)).astype(np.float32)
    assert (D._f16r(plane) == plane).all()
    for hw in (6.25, 12.5):                   # world slopes of about 35 and 20 degrees along each axis
        o = OO.OrthoOracle(W, H, near=0.5, far=100.0, tan_half_fov_h_=hw, linear=True)
        o.run(plane)
        for bid in (10, 11, 12):
            inner = o.codes(bid)[17:-17, 17:-17]
            assert inner.size and inner.min() >= 254, (hw, bid, int(inner.min()))


def test_golden_fixture_is_the_oracles():
    """tests/golden/ortho/*.npz still equal what the orthographic oracle computes (make_golden_ortho.py)."""
    import glob
    import os
    paths = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ortho", "*.npz")))
    assert paths
    for path in paths:
        g = np.load(path)
        H, W = g["depth"].shape
        near, far, size, rz = (float(v) for v in g["camera"])
        cam = Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=bool(rz), orthographic=True, orthographicSize=size)
        o = OO.OrthoOracle(W, H, near=near, far=far, tan_half_fov_h_=1.0 / cam.projection00, reversed_z=bool(rz),
                           intensity=float(g["params"][4]))
        assert np.array_equal(o.run(g["depth"]), g["ao"])
        for key in g.files:
            if key.startswith("buf"):
                bid = int(key[3:])
                ref = g[key]
                mine = o.codes(bid) if bid >= 10 else o.buffer(bid).astype(ref.dtype)
                assert np.array_equal(mine.view(np.uint8), ref.view(np.uint8)), key
