"""CPU tests of per-layer cameras (meao_set_layer_cameras): every layer of a layered frame with its own near plane, far plane and field
of view.

The layered kernel sources run in the fiber emulator (tests/emu/frame_driver.cpp), with each layer's
constants read from a plan-only libmeao context through the per-layer getters.  Layer l must be bit-identical to the oracle run on that
layer alone with camera l -- the AO and every buffer.  Also here: the plan-only contract of meao_set_layer_cameras (return values,
refusals, the per-layer getters against single-layer contexts) and the Python property."""
import ctypes as C

import numpy as np
import pytest

from miniengineao_b200 import AmbientOcclusion, Camera, MeaoError
from miniengineao_b200 import _native as N
from oracle.oracle import Oracle

from emu.emu import Frame
from test_layers_emulated import _raw, contrasting_layers


# visibly different cameras: near 0.1 / 0.3 / 1.0, far 50 / 100 / 1000, vertical FOV 40 / 60 / 90 degrees
CAMS = [(0.1, 50.0, 40.0), (0.3, 100.0, 60.0), (1.0, 1000.0, 90.0)]
PARAMS = {"noise_filter_tolerance": "noiseFilterTolerance", "blur_tolerance": "blurTolerance", "upsample_tolerance": "upsampleTolerance",
          "thickness_modifier": "thicknessModifier", "intensity": "intensity", "sample_exhaustively": "sampleExhaustively",
          "high_quality_mask": "highQualityMask"}


def cameras(W, H, n, reversed_z=True):
    return [Camera(W, H, nearClipPlane=CAMS[i % 3][0], farClipPlane=CAMS[i % 3][1], fieldOfView=CAMS[i % 3][2], usesReversedZBuffer=reversed_z)
            for i in range(n)]


def _plan(W, H, cams, single_scale=False, **kw):
    p = AmbientOcclusion(Camera(W, H, usesReversedZBuffer=kw.get("reversed_z", True)), device=-1)
    for py, cs in PARAMS.items():
        if py in kw:
            setattr(p, cs, kw[py])
    p.singleScale = single_scale
    p.layers = len(cams)
    p.layerCameras = cams
    return p


def _aligned(nbytes):
    raw = np.zeros(nbytes + 128, np.uint8)
    off = (-raw.ctypes.data) % 64
    return raw[off:off + nbytes]


def _oracle(W, H, cam, **kw):
    return Oracle(W, H, threads=4, near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00,
                  reversed_z=cam.usesReversedZBuffer, **kw)


def _compare(f, W, H, depth, cams, *, linear=False, single_scale=False, oracle_depth=None, ao_of=None, **kw):
    okw = {k: v for k, v in kw.items() if k != "reversed_z"}
    if linear:
        okw["depth_is_linear"] = True
    if single_scale:
        okw["single_scale"] = True
    mask = kw.get("high_quality_mask", 0)
    ids = [1, 2, 3, 4, 5, 10, 17] if single_scale else list(range(1, 18)) + [17 + k for k in range(1, 5) if (mask >> (k - 1)) & 1]
    for l, cam in enumerate(cams):
        orc = _oracle(W, H, cam, **okw)
        ref = orc.run(depth[l] if oracle_depth is None else oracle_depth[l])
        if ao_of is not None:
            assert np.array_equal(ao_of(l), ref), (W, H, l, "caller's AO view")
        bad = []
        for bid in ids:
            got, want = f.buffer(bid, l), orc.buffer(bid)
            if got.dtype == np.uint8:
                n = int((got != orc.codes(bid)).sum())
            elif got.dtype == np.float16:
                with np.errstate(over="ignore"):
                    n = int((got.view(np.uint16) != want.astype(np.float16).view(np.uint16)).sum())
            else:
                n = int((got.view(np.uint32) != want.view(np.uint32)).sum())
            if n:
                bad.append((bid, n, got.size))
        assert not bad, f"{W}x{H} {kw} layer {l}: mismatching buffers (id, #diff, size): {bad}"


def _run(W, H, depth, *, use_tma=True, linear=False, single_scale=False, fused=True, oracle_depth=None, **kw):
    cams = cameras(W, H, depth.shape[0], kw.get("reversed_z", True))
    f = Frame(_plan(W, H, cams, single_scale=single_scale, **kw), linear=linear, use_tma=use_tma)
    (f.run_fused if fused else f.run)(depth)
    _compare(f, W, H, depth, cams, linear=linear, single_scale=single_scale, oracle_depth=oracle_depth, **kw)
    return f


# ---- kernels in the emulator against the oracle, layer by layer ---------------------------------------------------------------
@pytest.mark.parametrize("use_tma", [True, False])
@pytest.mark.parametrize("W,H", [(161, 93), (37, 300)])
def test_ragged_layers_take_their_own_camera(W, H, use_tma):
    f = _run(W, H, _raw(contrasting_layers(W, H, 3, seed=W)), use_tma=use_tma, intensity=1.1)
    if not use_tma:
        assert f.tma_loads_in_run == 0


def test_interior_tiles_take_the_tma_path_with_layer_cameras():
    W, H = 640, 360
    f = _run(W, H, _raw(contrasting_layers(W, H, 3, seed=3)), intensity=1.1, high_quality_mask=0b0011)
    assert f.tma_loads_in_run > 300, f.tma_loads_in_run


def test_forward_z_pads_each_layer_with_its_own_linearize0():
    """reversed_z = False: the atlas padding value Linearize(0) = near / far differs per layer."""
    W, H = 130, 70
    _run(W, H, _raw(contrasting_layers(W, H, 3, seed=5), reversed_z=False), reversed_z=False, intensity=1.2)


@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True)])
def test_layer_cameras_with_variants(kw):
    W, H = 130, 70
    _run(W, H, _raw(contrasting_layers(W, H, 3, seed=7)), intensity=1.2, **kw)


def test_prepare_then_layered_upsample_pair():
    """The pair prepare_depth -> LinearDepth -> layered upsample (stage API, array frames) with per-layer cameras."""
    W, H = 161, 93
    _run(W, H, _raw(contrasting_layers(W, H, 3, seed=11)), fused=False, high_quality_mask=15)


def test_linear_and_native_ingest():
    W, H = 250, 131
    lin = contrasting_layers(W, H, 3, seed=9)
    _run(W, H, lin, linear=True)
    raw = _raw(lin).astype(np.float64)
    for bits, dt in ((16, np.uint16), (24, np.uint32)):
        full = (1 << bits) - 1
        codes = np.clip(np.rint(raw * full), 0, full).astype(np.uint32)
        as_float = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
        words = codes.astype(np.uint16) if bits == 16 else (codes | (np.uint32(0xA5) << np.uint32(24)))
        _run(W, H, words.astype(dt), oracle_depth=as_float)


def test_pitched_layered_corner():
    """The fused final level reading a layered depth corner of a larger buffer and writing into a padded AO view."""
    W, H, L = 150, 77, 3
    depth = _raw(contrasting_layers(W, H, L, seed=13))
    dr, dl = 176, 176 * 90                     # element pitches of the depth view
    big = _aligned(dl * L * 4).view(np.float32)
    big[:] = np.nan
    for l in range(L):
        for y in range(H):
            big[l * dl + y * dr: l * dl + y * dr + W] = depth[l, y]
    ar, al = 192, 192 * 80 + 64
    ao = _aligned(al * L)
    ao[:] = 0xA7
    cams = cameras(W, H, L)
    f = Frame(_plan(W, H, cams))
    f.run_fused(big, depth_row=dr, depth_layer=dl, ao=ao, ao_row=ar, ao_layer=al)
    view = lambda l: np.stack([ao[l * al + y * ar: l * al + y * ar + W] for y in range(H)])
    _compare(f, W, H, depth, cams, ao_of=view)


# ---- plan-only contract ----------------------------------------------------------------------------------------------------------
def _mc(cam):
    return N.MeaoCamera(cam.nearClipPlane, cam.farClipPlane, 1.0 / cam.projection00, int(cam.usesReversedZBuffer))


def _table(cams):
    return (N.MeaoCamera * len(cams))(*[_mc(c) for c in cams])


def _getters(ctx, layer=None):
    nl = N.lib()
    out = []
    for k in range(1, 5):
        for wide in (0, 1):
            b = (C.c_float * 28)()
            if layer is None:
                N.check(ctx, (nl.meao_render_constants_wide if wide else nl.meao_render_constants)(ctx, k, b))
            else:
                N.check(ctx, nl.meao_render_constants_layer(ctx, layer, k, wide, b))
            out.append(np.frombuffer(b, np.float32).copy())
    z = (C.c_float * 4)()
    N.check(ctx, nl.meao_zbuffer_params(ctx, z) if layer is None else nl.meao_zbuffer_params_layer(ctx, layer, z))
    out.append(np.frombuffer(z, np.float32).copy())
    return np.concatenate(out)


@pytest.mark.parametrize("rz", [True, False])
def test_per_layer_getters_equal_single_layer_contexts(rz):
    W, H = 1920, 1080
    cams = cameras(W, H, 5, reversed_z=rz)
    a = AmbientOcclusion(Camera(W, H, usesReversedZBuffer=rz), device=-1)
    a.layers = 5
    a.layerCameras = cams
    a.highQualityMask = 15
    a.LateUpdate()
    for l, cam in enumerate(cams):
        s = AmbientOcclusion(cam, device=-1)
        s.highQualityMask = 15
        s.LateUpdate()
        assert _getters(a._ctx, l).view(np.uint32).tolist() == _getters(s._ctx).view(np.uint32).tolist(), l
    assert _getters(a._ctx).view(np.uint32).tolist() == _getters(a._ctx, 0).view(np.uint32).tolist()    # the old getters: layer 0
    for bad in (-1, 5):
        assert N.lib().meao_zbuffer_params_layer(a._ctx, bad, (C.c_float * 4)()) == N.MEAO_ERR_INVALID
        assert N.lib().meao_render_constants_layer(a._ctx, bad, 1, 0, (C.c_float * 28)()) == N.MEAO_ERR_INVALID


def test_set_layer_cameras_return_values_and_refusals():
    nl = N.lib()
    a = AmbientOcclusion(Camera(640, 360), device=-1)
    a.layers = 3
    a.LateUpdate()
    ctx = a._ctx
    cams = cameras(640, 360, 3)
    t = _table(cams)
    assert nl.meao_get_layer_cameras(ctx, None, 0) == 0
    assert nl.meao_set_layer_cameras(ctx, t, 3) == 1
    assert nl.meao_set_layer_cameras(ctx, _table(cams), 3) == 0          # the same table again: no re-plan
    got = (N.MeaoCamera * 3)()
    assert nl.meao_get_layer_cameras(ctx, got, 3) == 3
    assert bytes(got) == bytes(t)
    assert nl.meao_get_layer_cameras(ctx, got, 2) == N.MEAO_ERR_INVALID
    before = _getters(ctx, 2)

    def refused(table, count, *words):
        assert nl.meao_set_layer_cameras(ctx, table, count) == N.MEAO_ERR_INVALID
        msg = nl.meao_last_error(ctx).decode()
        for w in words:
            assert w in msg, msg
        g = (N.MeaoCamera * 3)()
        assert nl.meao_get_layer_cameras(ctx, g, 3) == 3 and bytes(g) == bytes(t)      # the previous table stays
        assert _getters(ctx, 2).view(np.uint32).tolist() == before.view(np.uint32).tolist()

    refused(_table(cams[:2]), 2, "count 2", "3 layers")
    refused(None, 3, "NULL")
    for field, value, word in (("near_clip", 0.0, "near_clip"), ("far_clip", 0.05, "far_clip"), ("tan_half_fov_h", -1.0, "tan_half_fov_h"),
                               ("near_clip", float("nan"), "near_clip"), ("reversed_z", 0, "reversed_z")):
        bad = _table(cams)
        setattr(bad[2], field, value)
        refused(bad, 3, "layer 2", word)
    # meao_set_camera records the shared camera but does not re-plan while a table is set
    assert nl.meao_set_camera(ctx, C.byref(_mc(Camera(640, 360, nearClipPlane=2.0)))) == 0
    assert _getters(ctx, 2).view(np.uint32).tolist() == before.view(np.uint32).tolist()
    # clearing: every layer takes the shared camera again
    assert nl.meao_set_layer_cameras(ctx, None, 0) == 1
    assert nl.meao_set_layer_cameras(ctx, None, 0) == 0
    assert nl.meao_get_layer_cameras(ctx, None, 0) == 0
    s = AmbientOcclusion(Camera(640, 360, nearClipPlane=2.0), device=-1)
    s.LateUpdate()
    for l in range(3):
        assert _getters(ctx, l).view(np.uint32).tolist() == _getters(s._ctx).view(np.uint32).tolist()
    assert nl.meao_set_layer_cameras(None, t, 3) == N.MEAO_ERR_INVALID


def test_set_layers_clears_the_table_and_one_layer_is_set_camera():
    nl = N.lib()
    a = AmbientOcclusion(Camera(320, 180), device=-1)
    a.layers = 2
    a.LateUpdate()
    ctx = a._ctx
    assert nl.meao_set_layer_cameras(ctx, _table(cameras(320, 180, 2)), 2) == 1
    assert nl.meao_set_layers(ctx, 2) == 0 and nl.meao_get_layer_cameras(ctx, None, 0) == N.MEAO_ERR_INVALID   # kept (2 entries)
    assert nl.meao_set_layers(ctx, 1) == 1
    assert nl.meao_get_layer_cameras(ctx, None, 0) == 0
    cam = cameras(320, 180, 3)[2]
    assert nl.meao_set_layer_cameras(ctx, _table([cam]), 1) == 1
    s = AmbientOcclusion(cam, device=-1)
    s.LateUpdate()
    assert _getters(ctx).view(np.uint32).tolist() == _getters(s._ctx).view(np.uint32).tolist()


def test_python_layer_cameras_property():
    a = AmbientOcclusion(Camera(320, 180), device=-1)
    a.layers = 3
    a.LateUpdate()
    a.layerCameras = cameras(320, 180, 3)
    assert a.LateUpdate() is True
    assert a.LateUpdate() is False                                      # the same table every frame: no re-plan
    g = (N.MeaoCamera * 3)()
    assert N.lib().meao_get_layer_cameras(a._ctx, g, 3) == 3
    assert [round(x.near_clip, 6) for x in g] == [0.1, 0.3, 1.0]
    for bad in (Camera(321, 180), Camera(320, 181), Camera(320, 180, usesReversedZBuffer=False)):
        a.layerCameras = cameras(320, 180, 2) + [bad]
        with pytest.raises(ValueError):
            a.LateUpdate()
    a.layerCameras = cameras(320, 180, 2)
    with pytest.raises(ValueError):
        a.LateUpdate()
    a.layerCameras = None
    assert a.LateUpdate() is True
    assert N.lib().meao_get_layer_cameras(a._ctx, None, 0) == 0
    a.layerCameras = cameras(320, 180, 3)
    a.LateUpdate()
    a.layers = 2                                                        # set_layers clears the table; the property re-applies it
    a.layerCameras = cameras(320, 180, 2)
    assert a.LateUpdate() is True
    assert N.lib().meao_get_layer_cameras(a._ctx, (N.MeaoCamera * 2)(), 2) == 2
