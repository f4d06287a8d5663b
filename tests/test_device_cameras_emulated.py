"""CPU tests of the device-camera kernel (build.py CAMERA_SOURCES) in the emulator (tests/emu/device_cameras.py).

- The tables it derives from a camera buffer are, byte for byte, camera_tables() of a plan whose host cameras are the buffer's, taken
  from a plan-only libmeao context through the per-layer getters.  The cases are random cameras and the extreme cameras of
  tests/hostile_cases.py, plus cameras whose products are subnormal and whose orthographic it_i overflows to inf.  They cover both Z
  directions, perspective, orthographic and mixed tables, single-pass stereo, exhaustive sampling, odd sizes and L = 1, 3 and 6.
- An invalid entry leaves its layer's rows as they were, sets the status words, and every other layer is exact.
- Whole bound frames at L = 1 (the layered kernels with one layer) and L = 3 are bit-exact to the oracle of the buffer's cameras on
  every buffer, ids 1-21, while the plan's host cameras are other ones."""
import itertools

import numpy as np
import pytest

import harness
import hostile_cases as HC
from emu import device_cameras as DC
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
TABLES = {1: [[P], [O]], 3: [[P, P, P], [O, O, O], [P, O, P]], 6: [[O, P, P, O, P, O]]}


def camera(W, H, near, far, tan, proj, rz, stereo=False):
    """A Camera with tan_half_fov_h (perspective) or half-width (orthographic) `tan`."""
    if proj == O:
        return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, orthographic=True, orthographicSize=tan * H / W,
                      stereoEnabled=stereo)
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=rz, fieldOfView=HC.fov_for_tan_half_h(tan, W, H),
                  stereoEnabled=stereo)


def rows(cams) -> np.ndarray:
    """The device buffer of `cams`: what meao_set_camera is handed, as float32."""
    return np.array([(c.nearClipPlane, c.farClipPlane, 1.0 / c.projection00) for c in cams], np.float32)


def plan_of(cams, table, *, stereo=False, **kw):
    """A plan-only context whose host cameras are `cams` and whose layers have the projections `table`."""
    L = len(cams)
    plan = harness.context(cams[0], layers=L, layer_cameras=cams if L > 1 else None, **kw)
    plan.perLayerProjection = L > 1
    if stereo:
        plan.OnPreRender()
    return plan


def frame_of(cams, table, *, stereo=False, linear=False, **kw):
    return DC.frame(plan_of(cams, table, stereo=stereo, **kw), table, stereo=stereo, linear=linear)


def same_bytes(a, b) -> bool:
    return a.tobytes() == b.tobytes()


def check_tables(cams, table, stereo=False, **kw):
    """Host cameras `cams` against the same cameras in the buffer: derived tables == camera_tables() byte for byte."""
    f = frame_of(cams, table, stereo=stereo, **kw)
    want_zb, want_ren = DC.expected(f)
    DC.clobber(f)
    status = DC.new_status()
    DC.derive(f, rows(cams), status)
    zb, ren = DC.tables(f)
    for l in range(len(cams)):
        assert same_bytes(zb[l], want_zb[l]), ("LayerZ", l, zb[l], want_zb[l])
        for r in range(8):
            assert same_bytes(ren[r, l], want_ren[r, l]), ("LayerRender", l, r, ren[r, l], want_ren[r, l])
    assert list(status) == [0] * DC.STATUS_WORDS


def random_cams(rng, W, H, table, rz, stereo):
    out = []
    for p in table:
        near = float(10 ** rng.uniform(-3, 1))
        far = near * float(10 ** rng.uniform(0.01, 6))
        tan = float(10 ** rng.uniform(-2, 1.5))
        out.append(camera(W, H, near, far, tan, p, rz, stereo))
    return out


def _cases():
    out = []
    for (L, tables), rz, stereo, exh in itertools.product(TABLES.items(), (True, False), (False, True), (False, True)):
        for table in tables:
            out.append((table, rz, stereo, exh))
    return out


@pytest.mark.parametrize("size", [(97, 61), (160, 90)])
@pytest.mark.parametrize("table,rz,stereo,exh", _cases())
def test_random_cameras_derive_the_host_planners_bytes(table, rz, stereo, exh, size):
    W, H = size
    rng = np.random.default_rng(hash((tuple(table), rz, stereo, exh, W)) & 0xFFFF)
    for _ in range(3):
        check_tables(random_cams(rng, W, H, table, rz, stereo), table, stereo=stereo, sample_exhaustively=exh)


# (near, far, tan_half_fov_h): tests/hostile_cases.py's extreme cameras, and cameras whose products go subnormal or overflow
EXTREME = [(n, f, 1.0 if t is None else t) for n, f, t in HC.CAMERAS.values()] + [
    (1e-38, 1e3, 1.0),          # an orthographic n / f of 1e-41: subnormal, then 1 - subnormal
    (0.3, 100.0, 3e-38),        # (2 t) 10: 6e-37, then / src_w: subnormal ThicknessMultipliers
    (1e-3, 3e38, 1e-6),         # orthographic it_i = (far / ThicknessMultiplier) / SampleThickness overflows to inf
    (0.5, 1e30, 1e-30),         # and 1 / ThicknessMultiplier overflows under perspective
]


@pytest.mark.parametrize("rz", [True, False])
@pytest.mark.parametrize("table", [[P], [O], [O, P, O]])
@pytest.mark.parametrize("cam", EXTREME, ids=[f"{n:g}-{f:g}-{t:g}" for n, f, t in EXTREME])
def test_extreme_cameras_derive_the_host_planners_bytes(cam, table, rz):
    W, H = 97, 61
    check_tables([camera(W, H, *cam, p, rz) for p in table], table)
    check_tables([camera(W, H, *cam, p, rz, stereo=True) for p in table], table, stereo=True, sample_exhaustively=True)


def test_an_orthographic_it_i_overflows_to_inf():
    """The overflow case above does reach inf in the tables, and the kernel writes the same inf."""
    W, H = 97, 61
    cams = [camera(W, H, 1e-3, 3e38, 1e-6, O, True)]
    f = frame_of(cams, [O])
    _, ren = DC.expected(f)
    assert np.isinf(ren[:, 0, 0]).any()
    check_tables(cams, [O])


@pytest.mark.parametrize("bad,field", [((0.0, 50.0, 1.0), 1), ((float("nan"), 50.0, 1.0), 1), ((2.0, 2.0, 1.0), 2),
                                       ((2.0, float("nan"), 1.0), 2), ((0.5, 50.0, 0.0), 3), ((0.5, 50.0, float("nan")), 3)])
def test_an_invalid_entry_sets_the_status_and_leaves_every_other_layer_exact(bad, field):
    W, H = 97, 61
    table = [P, O, P]
    cams = [camera(W, H, 0.2 + 0.1 * l, 60.0 + 30 * l, 0.7 + 0.2 * l, p, True) for l, p in enumerate(table)]
    f = frame_of(cams, table)
    want_zb, want_ren = DC.expected(f)
    DC.clobber(f, 0x5A)
    status = DC.new_status()
    buf = rows(cams)
    buf[1] = bad
    DC.derive(f, buf, status)
    zb, ren = DC.tables(f)
    for l in (0, 2):
        assert same_bytes(zb[l], want_zb[l]) and same_bytes(ren[:, l], want_ren[:, l]), l
    assert (zb[1].view(np.uint8) == 0x5A).all() and (ren[:, 1].view(np.uint8) == 0x5A).all(), "an invalid layer's rows were written"
    assert list(status) == [1, 1, field, 0, 0, 0]
    buf[0] = bad
    DC.derive(f, buf, status)
    assert list(status) == [2, 0, field, 0, 0, 0]            # the lowest invalid layer of the latest frame; frames counted
    DC.derive(f, rows(cams), status)
    zb, ren = DC.tables(f)
    assert same_bytes(zb, want_zb) and same_bytes(ren, want_ren)
    assert list(status) == [2, 0, field, 0, 0, 0]


def test_the_unit_table_lists_every_kernel():
    assert DC.kernel_unit() == ("camera_tables.cu", 2)


FRAMES = [  # (layers, table, reversed_z, depth kind, fused, variants)
    (1, [P], True, "f32", True, {}),
    (1, [P], False, "d16", True, dict(high_quality_mask=15, sample_exhaustively=True)),
    (1, [O], True, "f32", True, {}),
    (3, [P, P, P], False, "f32", True, {}),
    (3, [P, P, P], True, "linear", False, dict(high_quality_mask=5)),
    (3, [O, P, O], False, "d24s8", True, {}),
]


@pytest.mark.parametrize("L,table,rz,kind,fused,variants", FRAMES)
def test_bound_frames_are_bit_exact_to_the_oracles(L, table, rz, kind, fused, variants):
    W, H = 97, 61
    cams = [camera(W, H, 0.2 + 0.15 * l, 60.0 + 40.0 * l, 0.6 + 0.25 * l, p, rz) for l, p in enumerate(table)]
    host = [camera(W, H, 1.0, 500.0, 2.0, p, rz) for p in table]       # the plan's host cameras: never read by a bound frame
    linear = kind == "linear"
    f = frame_of(host, table, linear=linear, **variants)
    lin = harness.contrasting_layers(W, H, L, seed=L) if linear else harness.frames(W, H, L, seed=L, reversed_z=rz)
    depth, as_float = harness.ingest(lin, kind)
    status = DC.new_status()
    DC.run(f, rows(cams), status, depth if L > 1 else depth[0], fused=fused)
    assert list(status) == [0] * DC.STATUS_WORDS
    code = {"f32": N.MEAO_DEPTH_RAW_F32, "linear": N.MEAO_DEPTH_LINEAR_F32, "d16": N.MEAO_DEPTH_RAW_D16_UNORM, "d24s8": N.MEAO_DEPTH_RAW_D24S8}[kind]
    ids = harness.buffer_ids(variants.get("high_quality_mask", 0))
    for l, cam in enumerate(cams):
        if cam.orthographic:
            from ortho_oracle import OrthoOracle
            orc = OrthoOracle(W, H, near=cam.nearClipPlane, far=cam.farClipPlane, tan_half_fov_h_=1.0 / cam.projection00,
                              reversed_z=rz, linear=linear, **variants)
        else:
            orc = harness.oracle(W, H, camera=cam, linear=linear, **variants)
        orc.run(as_float[l])
        harness.compare_buffers(lambda bid: DC.buffer(f, bid, l, code), orc, f"L={L} {table} rz={rz} {kind} layer {l}", ids)
