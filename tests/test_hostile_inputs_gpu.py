"""GPU tests of the kernels' fast-path guards at the edges of the input domain, on the H100 (the case table is tests/hostile_cases.py).

The hardware MUFU.RCP flushes subnormals and is only an approximation outside the guarded range, so these are the runs in which a
guard that admits a bad operand shows: hostile depth (signed zeros, negatives, subnormals, the 2^-60 / 2^60 edges, the f16 overflow
band, infinities, NaNs, raw depths where the linearisation's denominator crosses zero, the D16 / D24 sentinels) at every lane of the
grouped guards, with extreme cameras and tolerances, through every public entry point: render (tight, so the fused final upsample),
render_host, a pitched view, a layered frame, render_arrays, the variants, a 2-band row split with hostile rows on the seam, and a 4K
frame.  Every buffer must equal the oracle's: unorm8 codes exactly, f16 / f32 bit for bit except that two NaNs match."""
import numpy as np
import pytest

import harness
import hostile_cases as HC
from gpu_harness import Array, rt, torch_cuda  # noqa: F401  (the fixtures)

pytestmark = pytest.mark.gpu

W0, H0 = 643, 363           # ragged: W % 8 == 3, no level a multiple of 4, 16 or 64


def _check(ao, cam, seen, tag, *, layer=None, got_ao=None, linear=False, high_quality_mask=0, single_scale=False, **kw):
    """Every buffer of `ao` (layer `layer` of a layered context) against the oracle run on `seen`, the float32 depth it reads."""
    H, W = seen.shape
    orc = harness.oracle(W, H, camera=cam, linear=linear, stereo=cam.stereoEnabled, threads=8, high_quality_mask=high_quality_mask,
                         single_scale=single_scale, **kw)
    ref = orc.run(seen)
    if got_ao is not None:
        assert harness.n_diff(got_ao, ref, nan_equal=True) == 0, f"{tag}: AO differs from the oracle"
    get = (lambda bid: ao.debug_buffer(bid)) if layer is None else (lambda bid: ao.debug_buffer(bid)[layer])
    harness.compare_buffers(get, orc, tag, harness.buffer_ids(high_quality_mask, single_scale), nan_equal=True)


def _render(torch, ao, depth, linear=False):
    return ao.render(torch.from_numpy(np.ascontiguousarray(depth)).cuda(), linear=linear).cpu().numpy()


def _zb(cam):
    return harness.context(cam).zbuffer_params()


def _depth(kind, cam, seed):
    """(depth in the ingest format, float32 the oracle sees, linear?)"""
    W, H, rz = cam.pixelWidth, cam.pixelHeight, cam.usesReversedZBuffer
    if kind == "linear":
        d = HC.hostile_linear(W, H, seed=seed)
        return d, d, True
    if kind == "raw":
        d = HC.hostile_raw(W, H, _zb(cam), rz, seed=seed)
        return d, d, False
    codes, seen = HC.hostile_unorm(W, H, 16 if kind == "d16" else 24, rz, seed=seed)
    return codes, seen, False


# ---- render (tight: the fused final upsample) and render_host ------------------------------------------------------------------------
@pytest.mark.parametrize("kind,rz", [("linear", True)] + [(k, rz) for k in ("raw", "d16", "d24s8") for rz in (True, False)])
def test_render_hostile(torch_cuda, kind, rz):
    from miniengineao_b200 import Camera
    cam = Camera(W0, H0, usesReversedZBuffer=rz)
    depth, seen, linear = _depth(kind, cam, seed=1)
    ao = harness.context(cam, device=0)
    got = _render(torch_cuda, ao, depth, linear)
    _check(ao, cam, seen, f"render {kind} rz={rz}", got_ao=got, linear=linear)


@pytest.mark.parametrize("value", [0.0, -0.5, 1e-40, 1e30, np.inf, np.nan])
def test_solid_hostile_linear_frame(torch_cuda, value):
    from miniengineao_b200 import Camera
    W, H = 1100, 600                    # a solid block that fills whole level-4 render tiles
    cam = Camera(W, H)
    d = HC.hostile_linear(W, H, seed=2)
    d[:576, :1088] = value
    ao = harness.context(cam, device=0)
    got = _render(torch_cuda, ao, d, True)
    _check(ao, cam, d, f"solid {value!r}", got_ao=got, linear=True)


def test_render_host_hostile(torch_cuda):
    from miniengineao_b200 import Camera
    cam = Camera(321, 203)
    d = HC.hostile_raw(321, 203, _zb(cam), True, seed=3)
    ao = harness.context(cam, device=0)
    got = ao.render_host(d)
    _check(ao, cam, d, "render_host", got_ao=got)


def test_4k_hostile(torch_cuda):
    from miniengineao_b200 import Camera
    cam = Camera(3840, 2160)
    d = HC.hostile_linear(3840, 2160, seed=4)
    ao = harness.context(cam, device=0)
    got = _render(torch_cuda, ao, d, True)
    _check(ao, cam, d, "4K linear", got_ao=got, linear=True)


# ---- pitched view, layered frame, CUDA arrays ------------------------------------------------------------------------------------
def test_pitched_view_hostile(torch_cuda):
    from miniengineao_b200 import Camera
    torch = torch_cuda
    cam = Camera(W0, H0)
    d = HC.hostile_raw(W0, H0, _zb(cam), True, seed=5)
    rt = torch.full((H0 + 37, 1024), float("nan"), dtype=torch.float32, device="cuda")
    rt[:H0, :W0] = torch.from_numpy(d).cuda()
    out = torch.full((H0 + 5, 768), 0xA5, dtype=torch.uint8, device="cuda")
    ao = harness.context(cam, device=0)
    ao.render(rt[:H0, :W0], out[:H0, :W0])
    o = out.cpu().numpy()
    assert (o[:, W0:] == 0xA5).all() and (o[H0:] == 0xA5).all(), "a store outside the AO view"
    _check(ao, cam, d, "pitched", got_ao=o[:H0, :W0])


def test_layered_frame_hostile(torch_cuda):
    """L = 3 with different hostile content per layer: raw values, linear-ingest values salted into raw depth, a NaN block."""
    from miniengineao_b200 import Camera
    cam = Camera(W0, H0)
    zb = _zb(cam)
    d = np.stack([HC.hostile_raw(W0, H0, zb, True, seed=6), HC.salt(HC.hostile_raw(W0, H0, zb, True, seed=7), HC.LINEAR, 7),
                  HC.hostile_raw(W0, H0, zb, True, seed=8)])
    d[2, 64:256, 128:512] = np.nan
    ao = harness.context(cam, device=0, layers=3)
    got = _render(torch_cuda, ao, d)
    for l in range(3):
        _check(ao, cam, d[l], f"layered layer {l}", layer=l, got_ao=got[l])


@pytest.mark.parametrize("kind", ["raw_f32", "d16"])
def test_render_arrays_hostile(torch_cuda, rt, kind):
    from miniengineao_b200 import Camera
    W, H = 321, 203
    cam = Camera(W, H)
    depth, seen, _ = _depth("raw" if kind == "raw_f32" else "d16", cam, seed=9)
    ao = harness.context(cam, device=0)
    da, aa = Array(rt, W, H, depth.dtype), Array(rt, W, H, np.uint8)
    try:
        da.fill(depth)
        aa.fill(np.full((1, H, W), 0x5A, np.uint8))
        ao.render_arrays(da.handle, aa.handle, kind=kind)
        torch_cuda.cuda.synchronize()
        got = aa.read()[0]
        _check(ao, cam, seen, f"arrays {kind}", got_ao=got)
    finally:
        ao.release_array(da.handle)
        ao.release_array(aa.handle)
        da.free()
        aa.free()


# ---- variants and a row split -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(sample_exhaustively=True), dict(single_scale=True), dict(stereo=True)],
                         ids=["hq15", "exhaustive", "single_scale", "stereo"])
def test_variants_hostile(torch_cuda, kw):
    from miniengineao_b200 import Camera
    kw = dict(kw)
    stereo = kw.pop("stereo", False)
    W, H = (2 * 322, H0) if stereo else (W0, H0)
    cam = Camera(W // 2 if stereo else W, H, stereoEnabled=stereo)
    d = HC.hostile_linear(W, H, seed=10)
    ao = harness.context(cam, device=0, stereo=cam.stereoEnabled, **kw)
    got = _render(torch_cuda, ao, d, True)
    _check(ao, cam, d, f"{kw} stereo={stereo}", got_ao=got, linear=True, **kw)


def test_two_band_row_split_with_hostile_rows_on_the_seam(torch_cuda):
    from miniengineao_b200 import Camera
    torch = torch_cuda
    W, H = 1280, 720
    cam = Camera(W, H)
    cut = 16 * (((H + 15) // 16) // 2)
    d = HC.hostile_raw(W, H, _zb(cam), True, seed=11)
    d[cut - 3:cut + 3] = HC.salt(d[cut - 3:cut + 3], HC.raw_values(_zb(cam)), 11)
    ref = harness.oracle(W, H, threads=8).run(d)
    cuts = [0, cut, H]
    ctxs = []
    for i in range(2):
        a = harness.context(W, H, device=0)
        a.set_row_band(cuts[i], cuts[i + 1], cuts[i - 1] if i > 0 else -1, cuts[i + 2] if i + 2 <= 2 else -1)
        ctxs.append(a)
    for i, a in enumerate(ctxs):
        a.band_prepare(torch.from_numpy(d[cuts[i]:cuts[i + 1]].copy()).cuda())
    torch.cuda.synchronize()
    for i, side, j in ((0, 1, 1), (1, 0, 0)):
        nbytes = ctxs[i].halo_bytes(side)
        buf = torch.empty(max(nbytes, 4), dtype=torch.uint8, device="cuda")
        ctxs[i].halo_pack(side, buf)
        ctxs[i].synchronize()
        ctxs[j].halo_unpack(1 - side, buf)
        ctxs[j].synchronize()
    got = np.zeros((H, W), np.uint8)
    for i, a in enumerate(ctxs):
        o = torch.empty((cuts[i + 1] - cuts[i], W), dtype=torch.uint8, device="cuda")
        a.band_finish(o)
        a.synchronize()
        got[cuts[i]:cuts[i + 1]] = o.cpu().numpy()
    assert harness.n_diff(got, ref, nan_equal=True) == 0


# ---- cameras and parameters -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rz", [True, False])
@pytest.mark.parametrize("name", sorted(HC.CAMERAS))
def test_extreme_camera(torch_cuda, name, rz):
    cam = HC.camera(name, W0, H0, rz)
    d = HC.hostile_raw(W0, H0, _zb(cam), rz, seed=12)
    ao = harness.context(cam, device=0)
    got = _render(torch_cuda, ao, d)
    _check(ao, cam, d, f"camera {name} rz={rz}", got_ao=got)


@pytest.mark.parametrize("name", sorted(HC.CAMERAS))
def test_extreme_camera_as_one_layer_of_a_batch(torch_cuda, name):
    from miniengineao_b200 import Camera
    cams = [Camera(W0, H0, nearClipPlane=0.1, farClipPlane=50.0), HC.camera(name, W0, H0, True),
            Camera(W0, H0, nearClipPlane=1.0, farClipPlane=1000.0)]
    d = np.stack([HC.hostile_raw(W0, H0, _zb(c), True, seed=13 + l) for l, c in enumerate(cams)])
    ao = harness.context(Camera(W0, H0), device=0, layers=3, layer_cameras=cams)
    got = _render(torch_cuda, ao, d)
    for l, c in enumerate(cams):
        _check(ao, c, d[l], f"batch {name} layer {l}", layer=l, got_ao=got[l])


@pytest.mark.parametrize("params", HC.PARAMS, ids=lambda p: "-".join(f"{k}={v}" for k, v in p.items()))
def test_extreme_parameters(torch_cuda, params):
    from miniengineao_b200 import Camera
    cam = Camera(W0, H0)
    d = HC.hostile_raw(W0, H0, _zb(cam), True, seed=14)
    ao = harness.context(cam, device=0, **params)
    got = _render(torch_cuda, ao, d)
    _check(ao, cam, d, str(params), got_ao=got, **params)
