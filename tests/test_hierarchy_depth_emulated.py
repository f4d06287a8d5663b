"""Frames of every hierarchy depth (include/meao.h meao_set_hierarchy_depth) in the CPU emulator: pointer frames fused and unfused, layered
frames, CUDA arrays, batches, orthographic and [P, O] mixed frames and a bound device camera buffer, in both Z directions, with exhaustive
sampling and high-quality masks whose bits reach above the depth.  Every buffer the frame writes must equal each layer's oracle of that
depth bit for bit, and the launch ledger must hold exactly the launches of the frame schedule."""
import numpy as np
import pytest

import depth_oracle as DO
import harness
from emu import batch, emu, mixed, ortho
from emu.depth import set_levels
from emu import device_cameras as DC
from emu.emu import Frame
from miniengineao_b200 import Camera
from miniengineao_b200 import _native as N

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
DEPTHS = [1, 2, 3, 4]


def launches() -> int:
    return sum(e[0] for e in emu._ledger().values())


def check(cams, depth, get, n, tag, ao=None, linear=False, skip=(), **kw):
    """Each layer against the oracle of its camera at depth n: ao[l] when the AO is the caller's, and every written buffer but `skip`."""
    for l, cam in enumerate(cams):
        orc = DO.for_camera(cam, n, linear=linear, **kw)
        ref = orc.run(depth[l])
        if ao is not None:
            assert np.array_equal(ao[l], ref), f"{tag} layer {l}: AO"
        ids = [b for b in DO.written_ids(n, kw.get("high_quality_mask", 0)) if b not in skip]
        harness.compare_buffers(lambda bid: get(bid, l), orc, f"{tag} layer {l}", ids)


def perspective_plan(cam, n, layers=1, cams=None, **kw):
    plan = harness.context(cam, layers=layers, layer_cameras=cams, **kw)
    plan.hierarchyDepth = n
    plan.LateUpdate()
    return plan


def camera(W, H, l=0, reversed_z=True, ortho_=False):
    near, far = 0.2 + 0.15 * l, 60.0 + 40.0 * l
    if ortho_:
        return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, orthographic=True, orthographicSize=3.0 + 2.5 * l)
    return Camera(W, H, nearClipPlane=near, farClipPlane=far, usesReversedZBuffer=reversed_z, fieldOfView=50.0 + 7.0 * l)


# ---- perspective pointer frames, layered frames and CUDA arrays ---------------------------------------------------------------------
@pytest.mark.parametrize("n", DEPTHS)
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("reversed_z,kw", [(True, dict()), (False, dict(high_quality_mask=0b1011)), (True, dict(high_quality_mask=15, sample_exhaustively=True))],
                         ids=["plain", "hq11-stdz", "hq15-exh"])
def test_pointer_frames(n, fused, reversed_z, kw):
    W, H = 131, 77
    cam = camera(W, H, reversed_z=reversed_z)
    plan = perspective_plan(cam, n, **kw)
    d = harness.frames(W, H, 1, seed=n, reversed_z=reversed_z)
    f = set_levels(harness.fused_frame(plan) if fused else Frame(plan), n)
    emu.ledger_reset()
    if fused:
        f.run_fused(d[0])
    else:
        f.run(d[0])
    assert launches() == plan.kernels_per_frame
    names = emu.kernel_ledger()
    assert sum(v[0] for k, v in names.items() if k.startswith("blur_upsample")) == n
    assert sum(v[0] for k, v in names.items() if k.startswith("render_ao")) == n + bin(kw.get("high_quality_mask", 0) & ((1 << n) - 1)).count("1")
    check([cam], d, lambda bid, l: f.buffer(bid, l), n, f"n={n} fused={fused}", **kw)


@pytest.mark.parametrize("n", DEPTHS)
def test_layered_and_array_frames(n):
    W, H, L = 96, 70, 3
    cams = [camera(W, H, l) for l in range(L)]
    kw = dict(high_quality_mask=0b0110)
    plan = perspective_plan(cams[0], n, layers=L, cams=cams, **kw)
    d = harness.frames(W, H, L, seed=7 + n)
    f = set_levels(harness.fused_frame(plan), n)
    emu.ledger_reset()
    f.run_fused(d)
    assert launches() == plan.kernels_per_frame
    check(cams, d, lambda bid, l: f.buffer(bid, l), n, f"layered n={n}", **kw)
    f = set_levels(Frame(plan), n)
    emu.ledger_reset()
    ao = f.run_arrays(d, "layered")
    assert launches() == plan.kernels_per_frame
    check(cams, d, lambda bid, l: f.buffer(bid, l), n, f"arrays n={n}", ao=ao, **kw)


@pytest.mark.parametrize("n", DEPTHS)
def test_batch_of_arrays(n):
    W, H, L = 88, 52, 2
    cams = [camera(W, H, l) for l in range(L)]
    plan = perspective_plan(cams[0], n, layers=L, cams=cams, high_quality_mask=1)
    d = harness.frames(W, H, L, seed=3 + n)
    f = set_levels(Frame(plan), n)
    aos = [np.zeros((H, W), np.uint8) for _ in range(L)]
    emu.ledger_reset()
    batch.run_arrays_batch(f, [np.ascontiguousarray(x) for x in d], aos)
    assert launches() == 1 + plan.kernels_per_frame         # batch.run_arrays_batch's own prepare notes the depth kind first
    # a batch stores its AO into each layer's own array only, never into the context's AO buffer (id 17)
    check(cams, d, lambda bid, l: f.buffer(bid, l), n, f"batch n={n}", ao=np.stack(aos), skip=(17,), high_quality_mask=1)


# ---- orthographic and mixed frames --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", DEPTHS)
@pytest.mark.parametrize("reversed_z", [True, False])
def test_orthographic_frames(n, reversed_z):
    W, H = 120, 66
    cam = camera(W, H, reversed_z=reversed_z, ortho_=True)
    kw = dict(high_quality_mask=0b1100)
    plan = perspective_plan(cam, n, **kw)
    d = harness.frames(W, H, 1, seed=11 + n, reversed_z=reversed_z)
    f = set_levels(ortho.frame(plan), n)
    emu.ledger_reset()
    ortho.run(f, d[0], fused=True)
    assert launches() == plan.kernels_per_frame
    check([cam], d, lambda bid, l: ortho.buffer(f, bid, l, 0), n, f"ortho n={n}", ao=f.buffer(17)[None], **kw)


@pytest.mark.parametrize("n", DEPTHS)
def test_mixed_frames(n):
    W, H = 104, 60
    table = [P, O]
    cams = [camera(W, H, l, ortho_=p == O) for l, p in enumerate(table)]
    kw = dict(high_quality_mask=0b0011, sample_exhaustively=True)
    plan = harness.context(cams[0], layers=2, layer_cameras=cams, **kw)
    plan.perLayerProjection = True
    plan.hierarchyDepth = n
    plan.LateUpdate()
    d = harness.frames(W, H, 2, seed=5 + n)
    f = set_levels(mixed.frame(plan, table), n)
    assert mixed.is_mixed(f)
    emu.ledger_reset()
    mixed.run(f, d, fused=True)
    assert launches() == plan.kernels_per_frame
    ao = np.stack([f.buffer(17, l) for l in range(2)])
    check(cams, d, lambda bid, l: mixed.buffer(f, bid, l, 0), n, f"mixed n={n}", ao=ao, **kw)


# ---- a bound device camera buffer ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", DEPTHS)
@pytest.mark.parametrize("reversed_z", [True, False])
def test_device_cameras(n, reversed_z):
    W, H, L = 100, 64, 2
    cams = [camera(W, H, l, reversed_z=reversed_z) for l in range(L)]
    host = [Camera(W, H, nearClipPlane=1.0, farClipPlane=500.0, usesReversedZBuffer=reversed_z, fieldOfView=70.0) for _ in range(L)]
    kw = dict(high_quality_mask=0b1001, sample_exhaustively=True)
    plan = harness.context(host[0], layers=L, layer_cameras=host, **kw)
    plan.perLayerProjection = True
    plan.hierarchyDepth = n
    plan.LateUpdate()
    f = set_levels(DC.frame(plan, [P] * L), n)
    d = harness.frames(W, H, L, seed=13 + n, reversed_z=reversed_z)
    rows = np.array([(k.nearClipPlane, k.farClipPlane, 1.0 / k.projection00) for k in cams], np.float32)
    status = DC.new_status()
    emu.ledger_reset()
    DC.run(f, rows, status, d, fused=True)
    assert list(status) == [0] * DC.STATUS_WORDS
    assert launches() == 1 + plan.kernels_per_frame == 2 + 2 * n + bin(0b1001 & ((1 << n) - 1)).count("1")     # the camera stage first
    ao = np.stack([f.buffer(17, l) for l in range(L)])
    check(cams, d, lambda bid, l: DC.buffer(f, bid, l, 0), n, f"device cameras n={n}", ao=ao, **kw)
