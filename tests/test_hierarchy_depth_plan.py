"""The hierarchy depth (include/meao.h meao_set_hierarchy_depth) on plan-only contexts: validation, return values, the frame generation,
the re-plan inside reservations, the frame schedule of every depth x high_quality_mask x device-camera binding (launches, branches,
waits, PDL classes), meao_kernels_per_frame, meao_algorithmic_bytes, the stage-API refusals, single_scale as depth 1 and the Python
property."""
import ctypes as C
import itertools

import pytest

import harness
from miniengineao_b200 import AmbientOcclusion, Camera
from miniengineao_b200 import _native as N

from emu import emu
from emu.depth import schedule  # noqa: E402  (tests/ is on sys.path via conftest)


def plan(W=320, H=180, **kw):
    return harness.context(W, H, **kw)


def depth_of(ao):
    return ao._lib.meao_get_hierarchy_depth(ao._ctx)


def set_depth(ao, n):
    return ao._lib.meao_set_hierarchy_depth(ao._ctx, n)


def last_error(ao):
    return ao._lib.meao_last_error(ao._ctx).decode()


def generation(ao):
    """meao_frame_generation without applying the Python properties (AmbientOcclusion.frame_generation applies hierarchyDepth)."""
    return ao._lib.meao_frame_generation(ao._ctx)


# ---- the setter ------------------------------------------------------------------------------------------------------------------
def test_default_is_four_and_returns_follow_changes():
    ao = plan()
    ao.LateUpdate()
    assert depth_of(ao) == 4
    assert set_depth(ao, 4) == 0
    for n in (3, 1, 2, 4):
        assert set_depth(ao, n) == 1 and depth_of(ao) == n
        assert set_depth(ao, n) == 0


@pytest.mark.parametrize("bad", [0, 5, -1, 1 << 20, -(1 << 31)])
def test_out_of_range_is_refused_and_changes_nothing(bad):
    ao = plan()
    ao.LateUpdate()
    assert set_depth(ao, 2) == 1
    g = generation(ao)
    assert set_depth(ao, bad) == N.MEAO_ERR_INVALID
    assert "hierarchy depth" in last_error(ao) and str(bad) in last_error(ao)
    assert depth_of(ao) == 2 and generation(ao) == g
    assert ao._lib.meao_get_hierarchy_depth(None) == N.MEAO_ERR_INVALID
    assert ao._lib.meao_set_hierarchy_depth(None, 2) == N.MEAO_ERR_INVALID


def test_a_change_moves_the_frame_generation():
    ao = plan()
    ao.LateUpdate()
    g = generation(ao)
    assert set_depth(ao, 3) == 1 and generation(ao) > g
    g = generation(ao)
    assert set_depth(ao, 3) == 0 and generation(ao) == g


def test_a_change_inside_reservations_keeps_the_reservation():
    """As for a variants change, the reservation and the arena layout stay; the allocation count and the graphs are checked on the
    H100."""
    ao = plan(640, 360, max_resolution=(640, 360))
    ao.maxLayers = 4
    ao.LateUpdate()
    ao.camera.pixelWidth, ao.camera.pixelHeight = 320, 180
    ao.LateUpdate()
    before = ao.reservation()
    g = ao.frame_generation
    ao.hierarchyDepth = 2
    assert ao.LateUpdate()
    after = ao.reservation()
    assert (after["width"], after["height"], after["arena_bytes"]) == (before["width"], before["height"], before["arena_bytes"]) == (640, 360, before["arena_bytes"])
    assert ao._lib.meao_layer_reservation(ao._ctx) == 4
    assert ao.frame_generation > g


# ---- the schedule ----------------------------------------------------------------------------------------------------------------
def expected(n, mask, cams):
    """The schedule of depth n by the rules of frame_record.h frame_schedule, written out."""
    rows = []
    if cams:
        rows.append(("camera", 0, 0, None, "never"))
    prep = len(rows)
    rows.append(("prepare", 0, 0, None, "never"))
    last = {0: prep}
    for k in range(1, n + 1):
        last[k - 1] = len(rows)
        rows.append(("render", k, k - 1, None if k == 1 else prep, ">=1" if k == 1 else "never"))
    for k in range(1, n + 1):
        if (mask >> (k - 1)) & 1:
            last[k - 1] = len(rows)
            rows.append(("render_wide", k, k - 1, None, ">=1"))
    for lo in range(n, 2, -1):
        wait = last[lo - 2]
        last[n - 1] = len(rows)
        rows.append(("upsample", lo, n - 1, wait, ">=2"))
    if n >= 2:
        rows.append(("upsample", 2, 0, last[n - 1], ">=2"))
    rows.append(("upsample", 1, 0, None, ">=1"))
    return rows


ALL = list(itertools.product((1, 2, 3, 4), range(16), (False, True)))


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_schedule_of_every_depth_mask_and_binding(n):
    for mask, cams in itertools.product(range(16), (False, True)):
        got = schedule((0, 0, mask, 0), levels=n, device_cameras=cams)
        assert [r[:5] for r in got] == expected(n, mask, cams), (n, mask, cams)


def test_depth_four_is_the_parents_schedule():
    for mask, cams in itertools.product(range(16), (False, True)):
        got = schedule((0, 0, mask, 0), levels=4, device_cameras=cams)
        assert [r for r in got if r[0] != "camera"][0][0] == "prepare"
        if not cams:
            assert got == emu.schedule((0, 0, mask, 0))


def test_schedule_is_a_dag_whose_upsamples_wait_for_what_they_read():
    """Every launch after the one it reads: a render after the prepare, an upsample of lo level lo after Occlusion<lo - 1>, after the
    renders of level lo (its LoResAO1 at the top, and HighQuality<lo>) and after the upsample that wrote Combined<lo>.  Waits name an
    earlier launch on another branch, every forked branch joins back, and the branches' first launches carry no PDL."""
    for n, mask, cams in ALL:
        s = schedule((0, 0, mask, 0), levels=n, device_cameras=cams)
        pred = {i: set() for i in range(len(s))}
        for i, r in enumerate(s):
            on_branch = [j for j in range(i) if s[j][2] == r[2]]
            if on_branch:
                pred[i].add(on_branch[-1])
            if r[3] is not None:
                assert 0 <= r[3] < i and s[r[3]][2] != r[2], (n, mask, i)
                pred[i].add(r[3])
            if not on_branch:
                assert r[4] == "never", (n, mask, i)

        def before(i):
            out, todo = set(), [i]
            while todo:
                for p in pred[todo.pop()]:
                    if p not in out:
                        out.add(p)
                        todo.append(p)
            return out

        idx = {(r[0], r[1]): i for i, r in enumerate(s)}
        for i, r in enumerate(s):
            b = before(i)
            if r[0] in ("render", "render_wide"):
                assert idx[("prepare", 0)] in b
            if r[0] == "upsample":
                lo = r[1]
                if lo >= 2:
                    assert idx[("render", lo - 1)] in b, (n, mask, i)
                    if (mask >> (lo - 2)) & 1 and lo - 1 <= n:
                        assert idx[("render_wide", lo - 1)] in b, (n, mask, i)
                assert idx[("render", lo)] in b
                if (mask >> (lo - 1)) & 1:
                    assert idx[("render_wide", lo)] in b
                if lo < n:
                    assert idx[("upsample", lo + 1)] in b
        for br in (1, 2, 3):
            on_b = [i for i, r in enumerate(s) if r[2] == br]
            if on_b:
                assert s[on_b[0]][3] is not None and any(r[3] == on_b[-1] for r in s), (n, mask, br)
        assert s[-1][:3] == ("upsample", 1, 0)
        assert [r[5] for r in s if r[0] == "upsample"] == [f"blur_upsample L{lo}->L{lo - 1}" for lo in range(n, 0, -1)]


def test_single_scale_is_depth_one():
    for levels in (1, 2, 3, 4):
        assert schedule((0, 0, 0, 1), levels=levels) == schedule((0, 0, 0, 0), levels=1) == emu.schedule((0, 0, 0, 1))


def test_depth_one_with_a_high_quality_level_one():
    assert [r[:2] for r in schedule((0, 0, 1, 0), levels=1)] == [("prepare", 0), ("render", 1), ("render_wide", 1), ("upsample", 1)]


# ---- counts ---------------------------------------------------------------------------------------------------------------------
def test_kernels_per_frame_follow_the_schedule():
    ao = AmbientOcclusion(Camera(64, 64), device=-1)
    lib = N.lib()
    for n, mask in itertools.product((1, 2, 3, 4), range(16)):
        assert lib.meao_set_variants(ao._ctx, C.byref(N.MeaoVariants(0, 0, mask, 0))) >= 0
        assert set_depth(ao, n) >= 0
        want = 1 + n + bin(mask & ((1 << n) - 1)).count("1") + n
        assert ao.kernels_per_frame == want == len(schedule((0, 0, mask, 0), levels=n)), (n, mask)
    assert lib.meao_set_variants(ao._ctx, C.byref(N.MeaoVariants(0, 0, 0, 0))) >= 0
    assert set_depth(ao, 4) >= 0 and ao.kernels_per_frame == 9


def test_kernels_per_frame_with_a_device_camera_buffer():
    ao = AmbientOcclusion(Camera(64, 64), device=-1)
    lib = N.lib()
    assert lib.meao_bind_device_cameras(ao._ctx, C.c_void_p(4096), 1) == 1      # plan-only: the binding is recorded
    for n in (1, 2, 3, 4):
        set_depth(ao, n)
        assert ao.kernels_per_frame == 2 + 2 * n


def test_algorithmic_bytes_count_the_launched_levels():
    W, H = 1920, 1080
    full = plan(W, H)
    full.LateUpdate()
    px = lambda l: ((W + (1 << l) - 1) >> l) * ((H + (1 << l) - 1) >> l)  # noqa: E731
    ren = {k: 32 * px(k + 2) + px(k) for k in range(1, 5)}
    ups = {lo: 5 * px(lo) + (2 if lo == 1 else 5) * px(lo - 1) + px(lo - 1) for lo in range(1, 5)}
    assert full.algorithmic_bytes(3) == sum(ren.values()) and full.algorithmic_bytes(4) == sum(ups.values())
    for n in (1, 2, 3, 4):
        ao = plan(W, H)
        ao.hierarchyDepth = n
        ao.LateUpdate()
        assert ao.algorithmic_bytes(1) == full.algorithmic_bytes(1) and ao.algorithmic_bytes(2) == full.algorithmic_bytes(2)
        assert ao.algorithmic_bytes(3) == sum(ren[k] for k in range(1, n + 1))
        assert ao.algorithmic_bytes(4) == sum(ups[k] for k in range(1, n + 1))
        assert ao.algorithmic_bytes(5) == full.algorithmic_bytes(5)
        assert ao.algorithmic_bytes(0) == sum(ao.algorithmic_bytes(s) for s in (1, 2, 3, 4))


# ---- single_scale and the variants ------------------------------------------------------------------------------------------------
def test_single_scale_keeps_its_refusal_and_depth_one_takes_mask_bit_zero():
    ao = plan()
    lib = N.lib()
    assert set_depth(ao, 1) == 1
    assert lib.meao_set_variants(ao._ctx, C.byref(N.MeaoVariants(0, 0, 1, 1))) == N.MEAO_ERR_INVALID
    assert lib.meao_set_variants(ao._ctx, C.byref(N.MeaoVariants(0, 0, 1, 0))) == 1
    assert ao.kernels_per_frame == 4
    # bits above the depth are kept, whichever setter comes first
    assert lib.meao_set_variants(ao._ctx, C.byref(N.MeaoVariants(0, 0, 15, 0))) == 1
    assert ao.kernels_per_frame == 4
    assert set_depth(ao, 3) == 1 and ao.kernels_per_frame == 1 + 3 + 3 + 3
    v = N.MeaoVariants()
    assert lib.meao_get_variants(ao._ctx, C.byref(v)) == 0 and v.high_quality_mask == 15


def test_single_scale_sets_depth_one_in_effect_but_not_as_set():
    ao = plan(single_scale=True)
    ao.LateUpdate()
    assert depth_of(ao) == 4 and ao.kernels_per_frame == 3
    assert set_depth(ao, 2) == 1 and ao.kernels_per_frame == 3


def test_constants_do_not_depend_on_the_depth():
    ref = plan()
    ref.LateUpdate()
    want = harness.plan_constants(ref._ctx, 1)
    for n in (1, 2, 3):
        ao = plan()
        ao.hierarchyDepth = n
        ao.LateUpdate()
        assert harness.plan_constants(ao._ctx, 1) == want


# ---- the stage API ------------------------------------------------------------------------------------------------------------------
def test_stage_upsample_above_the_depth_is_refused_on_plan_only_contexts():
    """A plan-only context refuses every stage call for want of a device; the level check itself is covered on the H100."""
    ao = plan()
    ao.hierarchyDepth = 2
    ao.LateUpdate()
    assert ao._lib.meao_stage_upsample(ao._ctx, 3, None, None) == N.MEAO_ERR_CUDA


# ---- the Python property ------------------------------------------------------------------------------------------------------------
def test_python_property_is_applied_with_the_structural_inputs():
    ao = plan()
    assert ao.hierarchyDepth == 4
    assert ao.LateUpdate() in (True, False)
    assert ao.LateUpdate() is False
    ao.hierarchyDepth = 3
    assert ao.LateUpdate() is True and depth_of(ao) == 3
    assert ao.LateUpdate() is False
    ao.hierarchyDepth = 7
    with pytest.raises(N.MeaoError):
        ao.LateUpdate()
    assert depth_of(ao) == 3
