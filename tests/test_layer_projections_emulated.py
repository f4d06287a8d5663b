"""CPU tests of the per-layer projection kernels (build.py MIXED_SOURCES) in the emulator (tests/emu/mixed.py): which tables are mixed.
The case matrix that launches every mixed kernel, on ordinary and on hostile depth (tests/hostile_cases.py) under extreme cameras and
tolerances, each layer held on every buffer to the oracle of its projection, is tests/unit_matrix.py's, run by
test_unit_matrix_emulated.py."""
import harness
import unit_matrix as um
from emu import mixed
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

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
