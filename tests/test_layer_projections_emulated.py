"""CPU tests of the per-layer projection kernels (build.py MIXED_SOURCES) in the emulator (tests/emu/mixed.py): a case matrix of whole
layered frames whose layers mix both projections -- stage and fused pointer frames and CUDA arrays, tables [P, O] and [O, P, O, O] with
per-layer cameras, every depth kind and Z direction, plain and premin final upsamples, exhaustive sampling, the high-quality levels and
every render tile height -- each layer bit-exact on every buffer (ids 1-21) to the perspective oracle or the orthographic oracle
(tests/ortho_oracle.py), by its projection, and each case launching exactly the mixed kernels its fields name; together the cases launch
every mixed kernel built.  Hostile depth and the extreme cameras of tests/hostile_cases.py on a mixed table are held to the oracles the
same way."""
import ctypes as C
import itertools

import numpy as np
import pytest

import harness
import hostile_cases as HC
from emu import emu, mixed
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N
from ortho_oracle import OrthoOracle

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
IN = {"f32": 0, "d16": 1, "d24s8": 2}
KIND_CODE = {"f32": 0, "linear": 1, "d16": 2, "d24s8": 3}           # MEAO_DEPTH_*
TILE_H = (32, 16, 8)
TABLES = {2: [P, O], 4: [O, P, O, O]}
# (near, far, size): the orthographic half-height (orthographicSize), or the perspective vertical field of view in degrees
LAYER_CAMS = ((0.5, 80.0, 6.0), (1.0, 300.0, 55.0), (0.1, 20.0, 2.0), (0.3, 150.0, 9.0))


def camera(W, H, proj, rz, near, far, size):
    if proj == O:
        return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True, orthographicSize=size)
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, fieldOfView=size)


def plan_context(cams, table, **kw):
    plan = harness.context(cams[0], layers=len(cams), layer_cameras=cams, **kw)
    plan.perLayerProjection = True
    plan.LateUpdate()
    return plan


def oracle(cam, linear, **kw):
    """The oracle of one layer: the orthographic one for an orthographic camera, else the perspective one."""
    if cam.orthographic:
        return OrthoOracle(cam.pixelWidth, cam.pixelHeight, near=cam.nearClipPlane, far=cam.farClipPlane,
                           tan_half_fov_h_=1.0 / cam.projection00, reversed_z=cam.usesReversedZBuffer, linear=linear, **kw)
    return harness.oracle(cam.pixelWidth, cam.pixelHeight, camera=cam, linear=linear, **kw)


def _b(v):
    return "true" if v else "false"


def expected(c) -> set:
    """The mixed kernels case `c` launches, written from its fields: the raw prepare (linear ingest keeps the perspective kernel), the
    render of every level (wide ones for the hq levels) at the forced tile height, and the fused final upsample of raw depth (premin when
    level 1 is a high-quality level)."""
    out = set()
    raw = c["kind"] != "linear"
    if raw:
        if c["form"] == "arrays":
            out.add(f"prepare_depth_array_mixed_kernel<true, {_b(c['rz'])}, {IN[c['kind']]}>")
        else:
            base = "prepare_depth_low_mixed_layered" if c["form"] == "fused" else "prepare_depth_mixed_layered"
            out.add(f"{base}_kernel<true, {_b(c['rz'])}, {IN[c['kind']]}>")
    th = TILE_H[c["tile"]]
    for k in range(1, 5):
        out.add(f"render_ao_mixed_layered_kernel<0, {_b(c['exh'])}, {th}>")
        if (c["hq"] >> (k - 1)) & 1:
            out.add(f"render_ao_mixed_layered_kernel<1, {_b(c['exh'])}, {th}>")
    if raw and c["form"] == "fused":
        pre = "premin_" if c["hq"] & 1 else ""
        out.add(f"blur_upsample_{pre}lin_mixed_kernel<{IN[c['kind']]}, false, true>")
    return out


def _cases():
    cases = []
    kinds = list(itertools.product(("f32", "d16", "d24s8", "linear"), (True, False)))
    for L in (2, 4):
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


@pytest.fixture(scope="module")
def launched_all():
    return set()


@pytest.mark.parametrize("c", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_case_matrix(c, launched_all):
    W, H = (150, 70) if c["L"] == 2 else (120, 56)
    table = TABLES[c["L"]]
    cams = [camera(W, H, table[l], c["rz"], *LAYER_CAMS[l]) for l in range(c["L"])]
    plan = plan_context(cams, table, sample_exhaustively=c["exh"], high_quality_mask=c["hq"])
    f = mixed.frame(plan, table, linear=c["kind"] == "linear")
    assert mixed.is_mixed(f)
    d, seen = _depth(W, H, c["L"], c["kind"], c["rz"], seed=c["tile"] + 3 * c["L"])
    emu.ledger_reset()
    if c["form"] == "arrays":
        ao = mixed.run_arrays(f, d, "layered", ren_tile=c["tile"])
    else:
        mixed.run(f, d, fused=c["form"] == "fused", ren_tile=c["tile"])
    got = mixed.launched()
    assert got == expected(c), (sorted(got ^ expected(c)))
    launched_all |= got
    kind = KIND_CODE[c["kind"]]
    ids = [b for b in harness.buffer_ids(c["hq"]) if not (c["form"] == "arrays" and b == 17)]     # an array frame's AO is the array
    for l, cam in enumerate(cams):
        orc = oracle(cam, c["kind"] == "linear", sample_exhaustively=c["exh"], high_quality_mask=c["hq"])
        orc.run(seen[l])
        harness.compare_buffers(lambda bid: mixed.buffer(f, bid, l, kind), orc, f"{c} layer {l} ({'O' if cam.orthographic else 'P'})", ids)
        if c["form"] == "arrays":
            assert (ao[l] == orc.codes(17)).all(), l


def expected_union():
    u = set()
    for c in CASES:
        u |= expected(c)
    return u


def test_cases_launch_every_mixed_kernel(launched_all):
    if len(launched_all) < len(expected_union()):
        pytest.skip("the case matrix did not run in this session")
    assert launched_all == mixed.kernels()
    assert len(mixed.kernels()) == 34


def test_matrix_names_every_kernel_built():
    assert expected_union() == mixed.kernels()


def test_emulator_units_match_libmeao_tables():
    assert mixed.kernel_units() == {"prepare_depth_mixed_layered.cu": 12, "prepare_depth_array_mixed.cu": 4, "render_ao_mixed_layered.cu": 12,
                                    "blur_upsample_lin_mixed.cu": 6}


def test_uniform_tables_are_not_mixed():
    W, H = 64, 40
    for table in ([P, P], [O, O]):
        cams = [camera(W, H, p, True, *LAYER_CAMS[l]) for l, p in enumerate(table)]
        f = mixed.frame(plan_context(cams, table), table)
        assert not mixed.is_mixed(f)


# ---- hostile depth and extreme cameras ------------------------------------------------------------------------------------------------
W0, H0 = 203, 97
HOSTILE = dict(HC.CAMERAS)
HOSTILE["it_overflows"] = (1.0, 1e30, 1e-10)        # the orthographic half-width that sends it_i of the coarse levels to inf


def _hostile_cams(name, rz):
    """[perspective, orthographic] cameras of hostile camera `name`: its planes, and its tan_half_fov_h (5 when it has none) as the
    perspective layer's tan of the half field of view and as the orthographic layer's half-width."""
    near, far, t = HOSTILE[name]
    t = 5.0 if t is None else t
    aspect = W0 / H0
    p = Camera(W0, H0, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, fieldOfView=HC.fov_for_tan_half_h(t, W0, H0))
    o = Camera(W0, H0, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True, orthographicSize=t / aspect)
    return [p, o]


def _zb(plan, l):
    out = (C.c_float * 4)()
    assert N.lib().meao_zbuffer_params_layer(plan._ctx, l, out) == 0
    return np.array(out[:], np.float32)


def _hostile_check(f, cams, seen, tag, kind, linear=False, **kw):
    for l, cam in enumerate(cams):
        orc = oracle(cam, linear, **kw)
        orc.run(seen[l])
        harness.compare_buffers(lambda bid: mixed.buffer(f, bid, l, kind), orc, f"{tag} layer {l}", harness.buffer_ids(kw.get("high_quality_mask", 0)),
                                nan_equal=True)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("rz", [True, False])
@pytest.mark.parametrize("name", list(HOSTILE))
def test_hostile_raw_depth_extreme_cameras(name, rz, fused):
    cams = _hostile_cams(name, rz)
    plan = plan_context(cams, [P, O], high_quality_mask=9)
    f = mixed.frame(plan, [P, O])
    d = np.stack([HC.hostile_raw(W0, H0, _zb(plan, l), rz, seed=5 + l) for l in range(2)])
    mixed.run(f, d, fused=fused)
    _hostile_check(f, cams, d, f"raw {name} rz={rz} fused={fused}", 0, high_quality_mask=9)


@pytest.mark.parametrize("bits", [16, 24])
@pytest.mark.parametrize("rz", [True, False])
def test_hostile_unorm_depth(bits, rz):
    cams = _hostile_cams("far_near_1e7", rz)
    f = mixed.frame(plan_context(cams, [P, O]), [P, O])
    pairs = [HC.hostile_unorm(W0, H0, bits, rz, seed=bits + l) for l in range(2)]
    codes, seen = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    mixed.run(f, codes, fused=True)
    _hostile_check(f, cams, seen, f"unorm{bits} rz={rz}", 2 if bits == 16 else 3)


@pytest.mark.parametrize("name", ["tan_half_fov_1em6", "tan_half_fov_1e6", "it_overflows"])
def test_hostile_linear_depth(name):
    cams = _hostile_cams(name, True)
    f = mixed.frame(plan_context(cams, [P, O], sample_exhaustively=True), [P, O], linear=True)
    d = np.stack([HC.hostile_linear(W0, H0, seed=2 + l) for l in range(2)])
    mixed.run(f, d, fused=True)
    _hostile_check(f, cams, d, f"linear {name}", 1, linear=True, sample_exhaustively=True)
