"""CPU tests of the orthographic kernels (build.py ORTHO_SOURCES) in the emulator (tests/emu/ortho.py): hostile depth and extreme cameras
(tests/hostile_cases.py) under the projection, held to the orthographic oracle on every buffer.  The case matrix that launches every
orthographic kernel is tests/unit_matrix.py's, run by test_unit_matrix_emulated.py."""
import numpy as np
import pytest

import harness
import hostile_cases as HC
import unit_matrix as um
from emu import emu, ortho
from miniengineao_b200 import Camera
from ortho_oracle import OrthoOracle


def ortho_camera(W, H, rz, near, far, size):
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True, orthographicSize=size)


def test_matrix_names_every_kernel_built():
    assert set().union(*(um.expected_kernels(c) for c in um.CASES if c.unit == "ortho")) == ortho.kernels()


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
