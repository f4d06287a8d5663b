"""CPU tests of the per-layer projection kernels (build.py MIXED_SOURCES) in the emulator (tests/emu/mixed.py): which tables are mixed,
and hostile depth and the extreme cameras of tests/hostile_cases.py on a mixed table, each layer held on every buffer to the
perspective oracle or the orthographic oracle (tests/ortho_oracle.py), by its projection.  The case matrix that launches every mixed
kernel is tests/unit_matrix.py's, run by test_unit_matrix_emulated.py."""
import ctypes as C

import numpy as np
import pytest

import harness
import hostile_cases as HC
import unit_matrix as um
from emu import emu, mixed
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N
from ortho_oracle import OrthoOracle

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
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


def test_matrix_names_every_kernel_built():
    assert set().union(*(um.expected_kernels(c) for c in um.CASES if c.unit == "mixed")) == mixed.kernels()


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
