"""CPU tests of the kernels' fast-path guards at the edges of the input domain (the case table is tests/hostile_cases.py).

The kernel sources run in the fiber emulator, whose MUFU.RCP flushes subnormal operands and results like rcp.approx.ftz.f32, so a
guard that lets a zero, subnormal, infinite or out-of-range operand into a fast path gives wrong bits here too.  Hostile depth --
signed zeros, negatives, subnormals, the 2^-60 / 2^60 edges, the f16 overflow band, infinities, NaNs of every sign and payload, raw
depths where the linearisation's denominator crosses zero, the D16 / D24 sentinels -- goes through every frame form the emulator
has (whole frame with and without TMA, the fused final upsample, layered, per-layer cameras, pitched views, CUDA arrays, the
variants), with extreme cameras and tolerances.  Every buffer must equal the oracle's: unorm8 codes exactly, f16 / f32 bit for bit
except that two NaNs match.  Also here: the second restatement of the oracle (oracle/direct_formulation.py) on the same frames."""
import numpy as np
import pytest

from miniengineao_b200 import AmbientOcclusion, Camera
from oracle import direct_formulation as DF
from oracle.oracle import Oracle

import hostile_cases as HC
from emu.emu import Frame
from test_fused_lin_emulated import fused_frame
from test_pitched_emulated import SENTINEL, View

PARAMS = {"noise_filter_tolerance": "noiseFilterTolerance", "blur_tolerance": "blurTolerance", "upsample_tolerance": "upsampleTolerance",
          "thickness_modifier": "thicknessModifier", "intensity": "intensity"}
W0, H0 = 203, 97            # ragged: no level is a multiple of 4, 16 or 64, W % 8 == 3


def _plan(cam, layers=1, *, high_quality_mask=0, sample_exhaustively=False, single_scale=False, layer_cameras=None, **params):
    p = AmbientOcclusion(cam, device=-1)
    for py, cs in PARAMS.items():
        if py in params:
            setattr(p, cs, params[py])
    p.highQualityMask, p.sampleExhaustively, p.singleScale, p.layers = high_quality_mask, sample_exhaustively, single_scale, layers
    p.layerCameras = layer_cameras
    return p


def _oracle(W, H, cam, *, linear=False, stereo=False, **kw):
    okw = HC.oracle_camera_kw(cam)
    if stereo:
        okw["single_pass_stereo"] = True
    return Oracle(W, H, threads=4, depth_is_linear=linear, **okw, **kw)


def _check(get, W, H, cam, seen, tag, *, linear=False, high_quality_mask=0, single_scale=False, stereo=False, **kw):
    """get(bid) -> the kernel's buffer of this layer; seen: the float32 depth the oracle reads."""
    orc = _oracle(W, H, cam, linear=linear, stereo=stereo, high_quality_mask=high_quality_mask, single_scale=single_scale, **kw)
    orc.run(seen)
    HC.compare_buffers(get, orc, tag, HC.buffer_ids(high_quality_mask, single_scale))


def _whole(cam, depth, seen, tag, *, linear=False, use_tma=True, **kw):
    f = Frame(_plan(cam, **kw), linear=linear, use_tma=use_tma)
    f.run(depth)
    _check(f.buffer, cam.pixelWidth, cam.pixelHeight, cam, seen, tag, linear=linear, **kw)


def _zb(cam):
    return _plan(cam).zbuffer_params()


# ---- depth values through the whole frame ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_tma", [True, False])
@pytest.mark.parametrize("W,H", [(W0, H0), (136, 72)])
def test_linear_ingest_hostile_values(W, H, use_tma):
    cam = Camera(W, H)
    d = HC.hostile_linear(W, H, seed=W)
    _whole(cam, d, d, f"linear {W}x{H} tma={use_tma}", linear=True, use_tma=use_tma)


@pytest.mark.parametrize("use_tma", [True, False])
@pytest.mark.parametrize("rz", [True, False])
def test_raw_ingest_hostile_values(rz, use_tma):
    cam = Camera(W0, H0, usesReversedZBuffer=rz)
    d = HC.hostile_raw(W0, H0, _zb(cam), rz, seed=3)
    _whole(cam, d, d, f"raw rz={rz} tma={use_tma}", use_tma=use_tma)


@pytest.mark.parametrize("value", [0.0, -0.0, -0.5, 1e-40, 2.0 ** -61, 1e30, 7e4, np.inf, np.nan])
def test_solid_hostile_linear_frame(value):
    """The whole frame one hostile value: every tile of every level, every group of every guard, is out of range."""
    W, H = 70, 37
    cam = Camera(W, H)
    d = np.full((H, W), value, np.float32)
    _whole(cam, d, d, f"solid {value!r}", linear=True)


@pytest.mark.parametrize("rz", [True, False])
@pytest.mark.parametrize("bits", [16, 24])
def test_unorm_sentinel_codes(bits, rz):
    """Codes 0 and 2^n - 1 (sky / far plane) of D16 and D24S8, stencil bytes 0x00 and 0xFF."""
    cam = Camera(W0, H0, usesReversedZBuffer=rz)
    codes, seen = HC.hostile_unorm(W0, H0, bits, rz, seed=bits)
    _whole(cam, codes, seen, f"D{bits} rz={rz}")


# ---- the fused final upsample (what a tight frame runs on the GPU) ---------------------------------------------------------------
@pytest.mark.parametrize("kind", ["linear", "raw_rz", "raw", "d16", "d24s8"])
def test_fused_frame_hostile(kind):
    rz = kind != "raw"
    cam = Camera(W0, H0, usesReversedZBuffer=rz)
    if kind == "linear":
        depth = seen = HC.hostile_linear(W0, H0, seed=7)
    elif kind.startswith("raw"):
        depth = seen = HC.hostile_raw(W0, H0, _zb(cam), rz, seed=7)
    else:
        depth, seen = HC.hostile_unorm(W0, H0, 16 if kind == "d16" else 24, rz, seed=7)
    f = fused_frame(_plan(cam), linear=kind == "linear")
    f.run_fused(depth)
    _check(f.buffer, W0, H0, cam, seen, f"fused {kind}", linear=kind == "linear")


# ---- cameras ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rz", [True, False])
@pytest.mark.parametrize("name", sorted(HC.CAMERAS))
def test_extreme_camera(name, rz):
    W, H = 136, 72
    cam = HC.camera(name, W, H, rz)
    d = HC.hostile_raw(W, H, _zb(cam), rz, seed=11)
    _whole(cam, d, d, f"camera {name} rz={rz}")


@pytest.mark.parametrize("name", sorted(HC.CAMERAS))
def test_extreme_camera_as_one_layer_of_a_batch(name):
    """A 3-layer per-layer-camera batch: the hostile camera in the middle, ordinary cameras either side, hostile depth in every layer."""
    W, H = 136, 72
    cams = [Camera(W, H, nearClipPlane=0.1, farClipPlane=50.0), HC.camera(name, W, H, True), Camera(W, H, nearClipPlane=1.0, farClipPlane=1000.0)]
    depth = np.stack([HC.hostile_raw(W, H, _zb(c), True, seed=20 + l) for l, c in enumerate(cams)])
    f = Frame(_plan(Camera(W, H), 3, layer_cameras=cams))
    f.run_fused(depth)
    for l, c in enumerate(cams):
        _check(lambda bid: f.buffer(bid, l), W, H, c, depth[l], f"batch {name} layer {l}")


# ---- parameters ---------------------------------------------------------------------------------------------------------------
def test_parameter_table_straddles_the_proven_final_division_range():
    sides = [HC.fast_div_sides(_plan(Camera(W0, H0), **p)) for p in HC.PARAMS]
    assert True in set.union(*sides) and False in set.union(*sides)
    by = {tuple(p.items()): s for p, s in zip(HC.PARAMS, sides)}
    assert by[(("upsample_tolerance", -16.55),)] == {True} and by[(("upsample_tolerance", -16.56),)] == {False}
    assert by[(("upsample_tolerance", 0.0),)] == {True} and by[(("upsample_tolerance", 20.0),)] == {False}
    assert by[(("noise_filter_tolerance", 15.65),)] == {True} and by[(("noise_filter_tolerance", 15.66),)] == {False}


@pytest.mark.parametrize("params", HC.PARAMS, ids=lambda p: "-".join(f"{k}={v}" for k, v in p.items()))
def test_extreme_parameters(params):
    cam = Camera(W0, H0)
    d = HC.hostile_raw(W0, H0, _zb(cam), True, seed=13)
    _whole(cam, d, d, str(params), **params)


# ---- variants, layered, pitched and array frames ----------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True), dict(stereo=True)],
                         ids=["hq15", "exhaustive", "single_scale", "stereo"])
def test_variants_hostile(kw):
    kw = dict(kw)
    stereo = kw.pop("stereo", False)
    W, H = 2 * 68 if stereo else W0, H0
    cam = Camera(W // 2 if stereo else W, H, stereoEnabled=stereo)
    p = _plan(cam, **kw)
    if stereo:
        p.OnPreRender()                     # one draw for both eyes
    d = HC.hostile_linear(W, H, seed=17)
    f = Frame(p, linear=True)
    f.run(d)
    _check(f.buffer, W, H, cam, d, str(kw), linear=True, stereo=stereo, **kw)


@pytest.mark.parametrize("use_tma", [True, False])
def test_layered_frame_hostile(use_tma):
    """L = 3 with different hostile content per layer: linear-ingest values, the raw values, a solid NaN block."""
    W, H = 136, 72
    cam = Camera(W, H)
    d = np.stack([HC.hostile_raw(W, H, _zb(cam), True, seed=30), HC.salt(HC.hostile_raw(W, H, _zb(cam), True, seed=31), HC.LINEAR, 31),
                  HC.hostile_raw(W, H, _zb(cam), True, seed=32)])
    d[2, 16:64, 32:96] = np.nan
    f = Frame(_plan(cam, 3), use_tma=use_tma)
    f.run(d)
    for l in range(3):
        _check(lambda bid: f.buffer(bid, l), W, H, cam, d[l], f"layered layer {l}")


@pytest.mark.parametrize("linear", [False, True])
def test_pitched_view_hostile(linear):
    """Depth and AO as views with padded rows (a D3D12 footprint): the fused frame on hostile depth."""
    W, H = W0, H0
    cam = Camera(W, H)
    d = HC.hostile_linear(W, H, seed=40) if linear else HC.hostile_raw(W, H, _zb(cam), True, seed=40)
    f = fused_frame(_plan(cam), linear=linear)
    dv = View((1, H, W), np.float32, 1024, 1024 * H)
    dv.arr[...] = d
    av = View((1, H, W), np.uint8, 256, 256 * H, fill=SENTINEL)
    f.run_pitched(dv, av)
    assert (av.outside() == SENTINEL).all()
    _check(lambda bid: av.arr[0] if bid == 17 else f.buffer(bid), W, H, cam, d, f"pitched linear={linear}", linear=linear)


@pytest.mark.parametrize("kind", ["raw_f32", "d16"])
def test_array_frame_hostile(kind):
    W, H = 136, 72
    cam = Camera(W, H)
    if kind == "d16":
        depth, seen = HC.hostile_unorm(W, H, 16, True, seed=50)
    else:
        depth = seen = HC.hostile_raw(W, H, _zb(cam), True, seed=50)
    f = Frame(_plan(cam))
    ao = f.run_arrays(depth[None])
    _check(lambda bid: ao[0] if bid == 17 else f.buffer(bid, 0), W, H, cam, seen, f"array {kind}")


# ---- the oracle's second restatement on the same frames ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["linear", "raw_rz", "raw"])
def test_direct_formulation_agrees_on_hostile_frames(kind):
    """oracle/direct_formulation.py against the thread-group oracle (no-FMA build) on hostile frames, with the same NaN rule: pins the
    HLSL NaN / saturate / min / max semantics of the oracle from a second restatement."""
    W, H = 136, 72
    rz = kind != "raw"
    cam = Camera(W, H, usesReversedZBuffer=rz)
    linear = kind == "linear"
    d = HC.hostile_linear(W, H, seed=60) if linear else HC.hostile_raw(W, H, _zb(cam), rz, seed=60)
    o = Oracle(W, H, variant="nofma", reversed_z=rz, depth_is_linear=linear)
    ao = o.run(d)
    rc = {k: o.render_constants(k) for k in range(1, 5)}
    uc = {k: o.upsample_constants(k) for k in range(1, 5)}
    with np.errstate(all="ignore"):
        r = DF.run(d, rc, uc, o.zbuffer_params(), reversed_z=rz, linear=linear, return_all=True)
        assert HC.n_diff(np.asarray(r["linear"], np.float32).astype(np.float16), o.buffer(1)) == 0, "LinearDepth"
    dims = DF.level_dims(W, H)
    for k in range(1, 5):
        assert HC.n_diff(np.asarray(r["low"][k], np.float32), o.buffer(1 + k)) == 0, f"LowDepth{k}"
        tv = DF.tiled_view(r["low"][k], dims[k + 2][0], dims[k + 2][1], r["pad12"] if k <= 2 else np.float32(0))
        assert HC.n_diff(np.asarray(tv, np.float32), o.buffer(5 + k)) == 0, f"TiledDepth{k}"
        assert np.array_equal(r["occ"][k], o.codes(9 + k)), f"Occlusion{k}"
    for k in range(1, 4):
        assert np.array_equal(r["comb"][k], o.codes(13 + k)), f"Combined{k}"
    assert np.array_equal(r["comb"][0], ao)
