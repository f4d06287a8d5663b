"""CPU tests of live frame constants on plan-only contexts: MeaoParams and the cameras change between frames without a re-plan, on
a reserved context whose resizes cycle through every size slot and evict from them.  After every step each constant getter (every
level, wide and narrow, every layer) must be bit-identical to a fresh context given the same inputs in one go -- for the current size
and for a parked size swapped back in, which must never keep the constants it was parked with.  Also: the setters' return values, that
a refused input changes nothing, and that a change of the Z direction is refused inside a layer table or re-plans."""
import ctypes as C
import math
import random

import pytest

import harness
import hostile_cases as HC
from miniengineao_b200 import _native as N

MAX = (3840, 2160)
# ten sizes for eight slots: a walk through them evicts, and comes back to sizes parked several constant changes ago
SIZES = [(3840, 2160), (1920, 1080), (1000, 563), (2881, 1621), (17, 9), (1, 1), (641, 359), (3457, 1945), (64, 16), (1001, 999)]
PARAM_FIELDS = ("noise_filter_tolerance", "blur_tolerance", "upsample_tolerance", "thickness_modifier", "intensity", "debug")


def _params(**kw):
    p = N.MeaoParams()
    N.lib().meao_default_params(C.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _key(p):
    return tuple(getattr(p, f) for f in PARAM_FIELDS)


def _cams(cams):
    return (N.MeaoCamera * len(cams))(*[N.MeaoCamera(*c) for c in cams])


class State:
    """The inputs a context has been given, to build a fresh context from in one go."""

    def __init__(self, layers, variants):
        self.layers, self.variants = layers, variants
        self.params = _params()
        self.camera = (0.3, 1000.0, 1.0, 1)
        self.table = None
        self.size = None

    def fresh(self, size=None):
        lib = N.lib()
        h = C.c_void_p()
        assert lib.meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
        assert lib.meao_set_params(h, C.byref(self.params)) >= 0
        assert lib.meao_set_variants(h, C.byref(N.MeaoVariants(*self.variants))) >= 0
        assert lib.meao_set_layers(h, self.layers) >= 0
        assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*self.camera))) == 0
        if self.table:
            assert lib.meao_set_layer_cameras(h, _cams(self.table), self.layers) == 1
        assert lib.meao_resize(h, *(size or self.size)) == 1
        return h


def _check_fresh(h, st, tag, size=None):
    lib = N.lib()
    f = st.fresh(size)
    try:
        assert harness.plan_constants(h, st.layers) == harness.plan_constants(f, st.layers), tag
    finally:
        lib.meao_destroy(f)


def _random_camera(rng, z):
    fov = rng.uniform(30.0, 90.0)
    near = rng.choice([0.01, 0.1, 0.3, 1.0]) * rng.uniform(0.5, 2.0)
    return (near, near * rng.uniform(10.0, 1e5), math.tan(math.radians(fov) / 2) * 16 / 9, z)


def _hostile_camera(name, z):
    near, far, t = HC.CAMERAS[name]
    return (near, far, t if t is not None else math.tan(math.radians(30.0)) * 16 / 9, z)


SETUPS = {"single": (1, (0, 0, 0, 0)), "layers3_stereo_exhaustive_premin": (3, (1, 1, 15, 0)), "single_scale": (1, (0, 0, 0, 1))}


@pytest.mark.parametrize("setup", sorted(SETUPS))
def test_constants_follow_every_change_across_reserved_resizes(setup):
    layers, variants = SETUPS[setup]
    lib = N.lib()
    st = State(layers, variants)
    st.size = SIZES[0]
    h = st.fresh()
    assert lib.meao_reserve(h, *MAX) == 1
    rng = random.Random(11)
    hostile_params = list(HC.PARAMS)
    hostile_cams = sorted(HC.CAMERAS)
    sides = set()
    walk = 0
    try:
        for step in range(120):
            z = st.camera[3] if not st.table else st.table[0][3]
            action = ("resize", "params", "camera", "table")[step % 4] if step % 9 else "repeat"
            if action == "resize":
                walk += rng.choice([1, 1, 3, 7])
                size = SIZES[walk % len(SIZES)]
                rc = lib.meao_resize(h, *size)
                assert rc == (0 if size == st.size else 1)
                st.size = size
            elif action == "params":
                if (step // 4) % 2 == 0 and hostile_params:
                    kw = hostile_params.pop()
                else:
                    kw = dict(intensity=rng.uniform(0.0, 2.0), thickness_modifier=rng.uniform(1.0, 10.0), blur_tolerance=rng.uniform(-8, -1),
                              upsample_tolerance=rng.uniform(-12, -1), noise_filter_tolerance=rng.uniform(-8, 0), debug=rng.randrange(18))
                p = _params(**kw)
                expect = 1 if _key(p) != _key(st.params) else 0
                assert lib.meao_set_params(h, C.byref(p)) == expect, "1 = a value changed"
                st.params = p
            elif action == "camera":
                cam = _hostile_camera(hostile_cams.pop(), z) if (step // 4) % 2 == 0 and hostile_cams else _random_camera(rng, z)
                assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*cam))) == 0
                st.camera = cam
            elif action == "table":
                if step % 5 == 0 and st.table:
                    assert lib.meao_set_layer_cameras(h, None, 0) == 1          # cleared: back to the shared camera
                    st.table = None
                else:
                    table = [_random_camera(rng, z) for _ in range(layers)]
                    assert lib.meao_set_layer_cameras(h, _cams(table), layers) == 1
                    st.table = table
            else:                                                               # the same inputs again: nothing changed
                assert lib.meao_set_params(h, C.byref(st.params)) == 0
                assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*st.camera))) == 0
                if st.table:
                    assert lib.meao_set_layer_cameras(h, _cams(st.table), layers) == 0
                else:
                    assert lib.meao_set_layer_cameras(h, None, 0) == 0
            _check_fresh(h, st, f"step {step} ({action}) at {st.size}")
            for lo in range(1, 5):
                out = (C.c_float * 8)()
                assert lib.meao_upsample_constants(h, lo, out) == 0
                sides.add(HC.fast_div_ok(float(out[7]), float(out[4])))
        assert not hostile_params and not hostile_cams
        assert sides == {True, False}, "the parameters crossed both sides of upsample_fast_div_ok"
        # every size the walk left parked, swapped back in: the constants of now, not those it was parked with
        for size in SIZES:
            assert lib.meao_resize(h, *size) >= 0
            st.size = size
            _check_fresh(h, st, f"return to {size}")
    finally:
        lib.meao_destroy(h)


def test_refused_inputs_change_nothing():
    lib = N.lib()
    st = State(3, (0, 0, 0, 0))
    st.size = (1280, 720)
    h = st.fresh()
    assert lib.meao_reserve(h, 1920, 1080) == 1
    table = [(0.1, 50.0, 0.5, 1), (1.0, 1000.0, 1.2, 1), (0.3, 80.0, 0.8, 1)]
    assert lib.meao_set_layer_cameras(h, _cams(table), 3) == 1
    st.table = table
    assert lib.meao_resize(h, 999, 555) == 1
    st.size = (999, 555)

    def snapshot():
        p, got = N.MeaoParams(), (N.MeaoCamera * 3)()
        assert lib.meao_get_params(h, C.byref(p)) == 0
        assert lib.meao_get_layer_cameras(h, got, 3) == 3
        return harness.plan_constants(h, 3), _key(p), bytes(got)

    before = snapshot()
    refusals = [
        lambda: lib.meao_set_params(h, C.byref(_params(thickness_modifier=0.0, intensity=1.7))),
        lambda: lib.meao_set_params(h, C.byref(_params(thickness_modifier=-1.0))),
        lambda: lib.meao_set_camera(h, C.byref(N.MeaoCamera(0.0, 10.0, 1.0, 1))),
        lambda: lib.meao_set_camera(h, C.byref(N.MeaoCamera(1.0, 1.0, 1.0, 1))),
        lambda: lib.meao_set_camera(h, C.byref(N.MeaoCamera(0.3, 10.0, 0.0, 1))),
        lambda: lib.meao_set_layer_cameras(h, _cams([table[0], (0.0, 1.0, 1.0, 1), table[2]]), 3),
        lambda: lib.meao_set_layer_cameras(h, _cams([table[0], table[1], (0.3, 0.2, 1.0, 1)]), 3),
        lambda: lib.meao_set_layer_cameras(h, _cams(table[:2]), 2),
        lambda: lib.meao_set_layer_cameras(h, None, 3),
        lambda: lib.meao_set_layer_cameras(h, _cams([table[0], (0.1, 50.0, 0.5, 0), table[2]]), 3),    # two Z directions
    ]
    for i, call in enumerate(refusals):
        assert call() == N.MEAO_ERR_INVALID, i
        assert snapshot() == before, i
    _check_fresh(h, st, "after the refusals")
    lib.meao_destroy(h)


def test_a_z_direction_change_replans():
    """reversed_z selects kernel instantiations: a change of it is refused inside one table and re-plans otherwise, at the current size
    and at every parked one."""
    lib = N.lib()
    st = State(2, (0, 0, 0, 0))
    st.size = (1920, 1080)
    h = st.fresh()
    assert lib.meao_reserve(h, *MAX) == 1
    parked = [(1920, 1080), (1000, 563), (17, 9)]
    for size in parked:
        assert lib.meao_resize(h, *size) >= 0
    st.size = parked[-1]
    st.camera = (0.3, 1000.0, 0.7, 0)                                           # the shared camera flips to standard Z
    assert lib.meao_set_camera(h, C.byref(N.MeaoCamera(*st.camera))) == 0
    _check_fresh(h, st, "shared camera, standard Z")
    table = [(0.1, 50.0, 0.5, 1), (1.0, 1000.0, 1.2, 1)]                        # a table back to reversed Z
    assert lib.meao_set_layer_cameras(h, _cams(table), 2) == 1
    st.table = table
    _check_fresh(h, st, "table, reversed Z")
    assert lib.meao_set_layer_cameras(h, _cams([table[0], (1.0, 1000.0, 1.2, 0)]), 2) == N.MEAO_ERR_INVALID
    assert "reversed_z" in lib.meao_last_error(h).decode()
    _check_fresh(h, st, "after the refused table")
    assert lib.meao_set_layer_cameras(h, None, 0) == 1                          # cleared: the shared camera's standard Z again
    st.table = None
    _check_fresh(h, st, "cleared, standard Z")
    for size in parked:
        assert lib.meao_resize(h, *size) >= 0
        st.size = size
        _check_fresh(h, st, f"parked {size} after the Z changes")
    lib.meao_destroy(h)
