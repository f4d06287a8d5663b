"""The frame schedule (csrc/frame_record.h frame_schedule): which kernels a frame launches, in what order, on which stream, after which
other launch and with which programmatic-dependent-launch class.  libmeao's graph recorder, its serial recorder, meao_kernels_per_frame
and the emulator all walk this one list; these tests pin it on the CPU through the emulator's export."""
import ctypes as C
import itertools

import pytest

from miniengineao_b200 import AmbientOcclusion, Camera
from miniengineao_b200 import _native as N

from emu.emu import schedule  # noqa: E402  (tests/ is on sys.path via conftest)


def _valid_variants():
    for sps, exh, mask, single in itertools.product((0, 1), (0, 1), range(16), (0, 1)):
        if not (single and mask):                           # single_scale excludes the high-quality passes
            yield (sps, exh, mask, single)


# (stage, level, branch, wait, PDL class): branch 0 is the caller's stream, 1..3 the forked ones; wait is the index of the launch
# waited for.  Read off the frame DAG libmeao recorded before the schedule existed.
DEFAULT = [
    ("prepare", 0, 0, None, "never"),
    ("render", 1, 0, None, ">=1"),
    ("render", 2, 1, 0, "never"),
    ("render", 3, 2, 0, "never"),
    ("render", 4, 3, 0, "never"),
    ("upsample", 4, 3, 3, ">=2"),                           # after render 3, the last launch on branch 2
    ("upsample", 3, 3, 2, ">=2"),                           # after render 2, the last launch on branch 1
    ("upsample", 2, 0, 6, ">=2"),                           # after upsample 3
    ("upsample", 1, 0, None, ">=1"),
]
HQ15 = [
    ("prepare", 0, 0, None, "never"),
    ("render", 1, 0, None, ">=1"),
    ("render", 2, 1, 0, "never"),
    ("render", 3, 2, 0, "never"),
    ("render", 4, 3, 0, "never"),
    ("render_wide", 1, 0, None, ">=1"),
    ("render_wide", 2, 1, None, ">=1"),
    ("render_wide", 3, 2, None, ">=1"),
    ("render_wide", 4, 3, None, ">=1"),
    ("upsample", 4, 3, 7, ">=2"),                           # after wide render 3, the last launch on branch 2
    ("upsample", 3, 3, 6, ">=2"),                           # after wide render 2, the last launch on branch 1
    ("upsample", 2, 0, 10, ">=2"),
    ("upsample", 1, 0, None, ">=1"),
]
SINGLE_SCALE = [
    ("prepare", 0, 0, None, "never"),
    ("render", 1, 0, None, ">=1"),
    ("upsample", 1, 0, None, ">=1"),
]


@pytest.mark.parametrize("variants,want", [((0, 0, 0, 0), DEFAULT), ((0, 0, 15, 0), HQ15), ((0, 0, 0, 1), SINGLE_SCALE)],
                         ids=["default", "hq15", "single_scale"])
def test_schedule_tables(variants, want):
    assert [r[:5] for r in schedule(variants)] == want


def test_schedule_length_is_kernels_per_frame():
    """meao_kernels_per_frame of a plan-only context counts the schedule of the variants as set."""
    ao = AmbientOcclusion(Camera(64, 64), device=-1)
    for v in _valid_variants():
        assert N.lib().meao_set_variants(ao._ctx, C.byref(N.MeaoVariants(*v))) >= 0, v
        assert len(schedule(v)) == ao.kernels_per_frame, v


def test_waits_name_an_earlier_launch_on_another_branch():
    for v in _valid_variants():
        s = schedule(v)
        for i, (_, _, branch, wait, _, _) in enumerate(s):
            if wait is not None:
                assert 0 <= wait < i and s[wait][2] != branch, (v, i)
        for b in (1, 2, 3):
            on_b = [i for i, r in enumerate(s) if r[2] == b]
            if on_b:
                assert s[on_b[0]][3] is not None, (v, b)                    # a forked branch starts after a launch it waits for
                assert any(r[3] == on_b[-1] for r in s), (v, b)              # and its last launch is waited for: it joins back
        assert s[-1][:3] == ("upsample", 1, 0), v


def _parent_profile_names(mask, single):
    """The names meao_profile_frame reported before the schedule: prepare, render 1..k, wide renders, upsamples k..1."""
    kmax = 1 if single else 4
    return (["prepare_depth"] + [f"render_ao L{k}" for k in range(1, kmax + 1)]
            + [f"render_ao_wide L{k}" for k in range(1, kmax + 1) if (mask >> (k - 1)) & 1]
            + [f"blur_upsample L{lo}->L{lo - 1}" for lo in range(kmax, 0, -1)])


def test_names_are_the_profile_names():
    """bench.py, scripts/tune.sh and scripts/pick_best.sh key on these strings."""
    for v in _valid_variants():
        assert [r[5] for r in schedule(v)] == _parent_profile_names(v[2], v[3]), v
