"""CPU tests of the orthographic kernels (build.py ORTHO_SOURCES) in the emulator (tests/emu/ortho.py): a case matrix of whole frames --
stage and fused pointer frames and CUDA arrays, one layer and three layers with per-layer cameras, every depth kind and Z direction,
exhaustive sampling, the high-quality levels and every render tile height -- each bit-exact to the orthographic oracle on every buffer
(ids 1-21) and launching exactly the orthographic kernels its fields name; together the cases launch every orthographic kernel built.
Hostile depth and extreme cameras (tests/hostile_cases.py) under the projection are held to the oracle the same way."""
import itertools

import numpy as np
import pytest

import harness
import hostile_cases as HC
from emu import emu, ortho
from miniengineao_b200 import Camera
from ortho_oracle import OrthoOracle

IN = {"f32": 0, "d16": 1, "d24s8": 2}
KIND_CODE = {"f32": 0, "linear": 1, "d16": 2, "d24s8": 3}           # MEAO_DEPTH_*
TILE_H = (32, 16, 8)
LAYER_CAMS = ((0.5, 80.0, 6.0), (1.0, 300.0, 25.0), (0.1, 20.0, 2.0))


def ortho_camera(W, H, rz, near, far, size):
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True, orthographicSize=size)


def _b(v):
    return "true" if v else "false"


def expected(c) -> set:
    """The orthographic kernels case `c` launches, written from its fields: the raw prepare (linear ingest keeps the perspective
    kernel), the render of every level (wide ones for the hq levels) at the forced tile height, and the fused final upsample of raw
    depth (premin when level 1 is a high-quality level)."""
    lay = "_layered" if c["L"] > 1 else ""
    out = set()
    raw = c["kind"] != "linear"
    if raw:
        if c["form"] == "arrays":
            out.add(f"prepare_depth_array_ortho_kernel<true, {_b(c['rz'])}, {IN[c['kind']]}>")
        else:
            base = "prepare_depth_low_ortho" if c["form"] == "fused" else "prepare_depth_ortho"
            out.add(f"{base}{lay}_kernel<true, {_b(c['rz'])}, {IN[c['kind']]}>")
    th = TILE_H[c["tile"]]
    for k in range(1, 5):
        out.add(f"render_ao_ortho{lay}_kernel<0, {_b(c['exh'])}, {th}>")
        if (c["hq"] >> (k - 1)) & 1:
            out.add(f"render_ao_ortho{lay}_kernel<1, {_b(c['exh'])}, {th}>")
    if raw and c["form"] == "fused":
        pre = "premin_" if c["hq"] & 1 else ""
        out.add(f"blur_upsample_{pre}lin_ortho{lay}_kernel<{IN[c['kind']]}, false, true>")
    return out


def _cases():
    cases = []
    kinds = list(itertools.product(("f32", "d16", "d24s8", "linear"), (True, False)))
    for L in (1, 3):
        for form, exh, hq in (("fused", False, 0), ("stage", True, 15), ("fused", False, 1)):
            for i, (kind, rz) in enumerate(kinds):
                cases.append(dict(form=form, L=L, kind=kind, rz=rz, exh=exh, hq=hq, tile=i % 3))
        for i, (kind, rz) in enumerate(itertools.product(("f32", "d16", "linear"), (True, False))):
            cases.append(dict(form="arrays", L=L, kind=kind, rz=rz, exh=i % 2 == 1, hq=2 if i < 3 else 0, tile=i % 3))
    return cases


CASES = _cases()


def _depth(W, H, L, kind, rz, seed):
    if kind == "linear":
        d = harness.contrasting_layers(W, H, L, seed=seed)
        return d, d
    r = harness.frames(W, H, L, seed=seed, reversed_z=rz)
    return harness.ingest(r, kind)


def _oracle(cam, c, seen):
    orc = OrthoOracle(cam.pixelWidth, cam.pixelHeight, near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00,
                      reversed_z=cam.usesReversedZBuffer, linear=c["kind"] == "linear", sample_exhaustively=c["exh"],
                      high_quality_mask=c["hq"])
    orc.run(seen)
    return orc


@pytest.fixture(scope="module")
def launched_all():
    return set()


@pytest.mark.parametrize("c", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_case_matrix(c, launched_all):
    W, H = (300, 136) if c["L"] == 1 else (150, 70)
    cams = [ortho_camera(W, H, c["rz"], *LAYER_CAMS[l]) for l in range(c["L"])]
    plan = harness.context(cams[0], layers=c["L"], layer_cameras=cams if c["L"] > 1 else None, sample_exhaustively=c["exh"],
                           high_quality_mask=c["hq"])
    f = ortho.frame(plan, linear=c["kind"] == "linear")
    d, seen = _depth(W, H, c["L"], c["kind"], c["rz"], seed=c["tile"] + 3 * c["L"])
    emu.ledger_reset()
    if c["form"] == "arrays":
        ao = ortho.run_arrays(f, d, "layered" if c["L"] > 1 else "2d", ren_tile=c["tile"])
    else:
        ortho.run(f, d if c["L"] > 1 else d[0], fused=c["form"] == "fused", ren_tile=c["tile"])
    got = ortho.launched()
    assert got == expected(c), (sorted(got ^ expected(c)))
    launched_all |= got
    kind = KIND_CODE[c["kind"]]
    ids = [b for b in harness.buffer_ids(c["hq"]) if not (c["form"] == "arrays" and b == 17)]     # an array frame's AO is the array
    for l, cam in enumerate(cams):
        orc = _oracle(cam, c, seen[l])
        harness.compare_buffers(lambda bid: ortho.buffer(f, bid, l, kind), orc, f"{c} layer {l}", ids)
        if c["form"] == "arrays":
            assert (ao[l] == orc.codes(17)).all(), l


def test_cases_launch_every_orthographic_kernel(launched_all):
    if len(launched_all) < len(expected_union()):
        pytest.skip("the case matrix did not run in this session")
    assert launched_all == ortho.kernels()
    assert len(ortho.kernels()) == 64


def expected_union():
    u = set()
    for c in CASES:
        u |= expected(c)
    return u


def test_matrix_names_every_kernel_built():
    assert expected_union() == ortho.kernels()


def test_emulator_units_match_libmeao_tables():
    assert ortho.kernel_units() == {"prepare_depth_ortho.cu": 12, "prepare_depth_ortho_layered.cu": 12, "prepare_depth_array_ortho.cu": 4,
                                    "render_ao_ortho.cu": 12, "render_ao_ortho_layered.cu": 12, "blur_upsample_lin_ortho.cu": 12}


# ---- hostile depth and extreme cameras ------------------------------------------------------------------------------------------------
W0, H0 = 203, 97
# name -> (near, far, half-width): hostile_cases.CAMERAS' planes, their tan_half_fov_h as the half-width (5 for the default camera),
# and a half-width small enough that it_i of the coarse levels overflows to inf
ORTHO_CAMERAS = {name: (n, f, 5.0 if t is None else t) for name, (n, f, t) in HC.CAMERAS.items()}
ORTHO_CAMERAS["it_overflows"] = (1.0, 1e30, 1e-10)


def _hostile_cam(name, rz):
    near, far, t = ORTHO_CAMERAS[name]
    return ortho_camera(W0, H0, rz, near, far, t / (W0 / H0))


def _hostile_check(f, cam, seen, tag, linear=False, dtype=np.float32, **kw):
    orc = OrthoOracle(W0, H0, near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00,
                      reversed_z=cam.usesReversedZBuffer, linear=linear, **kw)
    orc.run(seen)
    kind = 1 if linear else {np.dtype(np.uint16): 2, np.dtype(np.uint32): 3}.get(np.dtype(dtype), 0)
    harness.compare_buffers(lambda bid: ortho.buffer(f, bid, 0, kind), orc, tag, harness.buffer_ids(kw.get("high_quality_mask", 0)),
                            nan_equal=True)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("rz", [True, False])
@pytest.mark.parametrize("name", list(ORTHO_CAMERAS))
def test_hostile_raw_depth_extreme_cameras(name, rz, fused):
    cam = _hostile_cam(name, rz)
    plan = harness.context(cam, high_quality_mask=9)
    f = ortho.frame(plan)
    d = HC.hostile_raw(W0, H0, plan.zbuffer_params(), rz, seed=5)
    ortho.run(f, d, fused=fused)
    _hostile_check(f, cam, d, f"raw {name} rz={rz} fused={fused}", high_quality_mask=9)


@pytest.mark.parametrize("bits", [16, 24])
@pytest.mark.parametrize("rz", [True, False])
def test_hostile_unorm_depth(bits, rz):
    cam = _hostile_cam("far_near_1e7", rz)
    f = ortho.frame(harness.context(cam))
    codes, seen = HC.hostile_unorm(W0, H0, bits, rz, seed=bits)
    ortho.run(f, codes, fused=True)
    _hostile_check(f, cam, seen, f"unorm{bits} rz={rz}", dtype=codes.dtype)


@pytest.mark.parametrize("name", ["tan_half_fov_1em6", "tan_half_fov_1e6", "it_overflows"])
def test_hostile_linear_depth(name):
    cam = _hostile_cam(name, True)
    f = ortho.frame(harness.context(cam, sample_exhaustively=True), linear=True)
    d = HC.hostile_linear(W0, H0, seed=2)
    ortho.run(f, d, fused=True)
    _hostile_check(f, cam, d, f"linear {name}", linear=True, sample_exhaustively=True)


def test_it_overflows_camera_reaches_inf():
    cam = _hostile_cam("it_overflows", True)
    orc = OrthoOracle(W0, H0, near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00)
    assert np.isinf(orc.inv_thickness(4)).any()
