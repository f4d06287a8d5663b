"""CPU tests of dynamic view counts (meao_reserve_layers) on plan-only contexts: the setter's validation and return values, the
generation, the combinations with a size reservation and their refusals, the exclusion of row bands, and that after any walk of layer
counts and sizes every constant getter is bit-identical to a fresh context of that (W, H, L), with the camera and viewport tables a
layer change clears.  A seeded walk of a few hundred set_layers / resize / table calls checks every return value and the generation."""
import ctypes as C
import random

import pytest

import harness
from miniengineao_b200 import _native as N

MAX = (1920, 1080)


def _create(layers=1):
    h = C.c_void_p()
    assert N.lib().meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
    if layers != 1:
        assert N.lib().meao_set_layers(h, layers) == 1
    return h


def _reservation(h):
    r = N.MeaoReservation()
    assert N.lib().meao_reservation(h, C.byref(r)) == 0
    return r


def _error(h):
    return N.lib().meao_last_error(h).decode()


def _cams(rng, n, z=1):
    return [(rng.choice([0.05, 0.3, 1.0]), rng.choice([100.0, 3000.0]), rng.choice([0.5, 1.0, 1.7]), z) for _ in range(n)]


def _set_cams(h, cams):
    return N.lib().meao_set_layer_cameras(h, (N.MeaoCamera * len(cams))(*[N.MeaoCamera(*c) for c in cams]), len(cams))


def _set_views(h, views):
    return N.lib().meao_set_layer_viewports(h, (N.MeaoLayerViewport * len(views))(*[N.MeaoLayerViewport(*v) for v in views]), len(views))


def _fresh_constants(W, H, L, cams=None):
    f = _create(L)
    try:
        assert N.lib().meao_resize(f, W, H) == 1
        if cams:
            assert _set_cams(f, cams) == 1
        return harness.plan_constants(f, L)
    finally:
        N.lib().meao_destroy(f)


def test_setter_validation_and_return_values():
    lib = N.lib()
    assert lib.meao_reserve_layers(None, 4) == N.MEAO_ERR_INVALID
    assert lib.meao_layer_reservation(None) == N.MEAO_ERR_INVALID
    h = _create(3)
    try:
        assert lib.meao_layer_reservation(h) == 0
        g = lib.meao_frame_generation(h)
        for bad in (-1, 65536, 1 << 30):
            assert lib.meao_reserve_layers(h, bad) == N.MEAO_ERR_INVALID
            assert "max_layers" in _error(h)
        assert lib.meao_reserve_layers(h, 2) == N.MEAO_ERR_INVALID            # below the current count
        assert "max_layers 2 is below the current layer count 3" in _error(h)
        assert lib.meao_layer_reservation(h) == 0 and lib.meao_frame_generation(h) == g
        assert lib.meao_reserve_layers(h, 8) == 1 and lib.meao_layer_reservation(h) == 8
        assert lib.meao_frame_generation(h) != g
        g = lib.meao_frame_generation(h)
        assert lib.meao_reserve_layers(h, 8) == 0 and lib.meao_frame_generation(h) == g
        assert lib.meao_reserve_layers(h, 65535) == 1 and lib.meao_reserve_layers(h, 3) == 1
        assert lib.meao_set_layers(h, 4) == N.MEAO_ERR_INVALID                 # above the reservation
        assert "layers 4 lies above the layer reservation 3" in _error(h)
        assert lib.meao_set_layers(h, 1) == 1 and lib.meao_set_layers(h, 1) == 0 and lib.meao_set_layers(h, 3) == 1
        assert lib.meao_set_layers(h, 0) == N.MEAO_ERR_INVALID
        assert lib.meao_reserve_layers(h, 0) == 1 and lib.meao_layer_reservation(h) == 0
        assert lib.meao_reserve_layers(h, 0) == 0
        assert lib.meao_set_layers(h, 7) == 1                                  # no reservation: any count again
    finally:
        lib.meao_destroy(h)


def test_arena_bytes_follow_both_reservations():
    """arena_bytes is the layout of (the size reservation or the current size) x max_layers -- what an unreserved context of that
    size and count allocates -- and arena_bytes_needed the current (W, H, L)'s."""
    lib = N.lib()
    h, big = _create(2), _create(6)
    try:
        assert lib.meao_resize(h, 640, 360) == 1 and lib.meao_resize(big, 640, 360) == 1
        needed = _reservation(h).arena_bytes
        assert lib.meao_reserve_layers(h, 6) == 1
        r = _reservation(h)
        assert r.arena_bytes == _reservation(big).arena_bytes and r.arena_bytes_needed == needed
        assert lib.meao_reserve(h, *MAX) == 1 and lib.meao_resize(big, *MAX) == 1
        r = _reservation(h)
        assert r.arena_bytes == _reservation(big).arena_bytes and r.arena_bytes_needed == needed
        for L in (1, 5, 6, 3):
            assert lib.meao_set_layers(h, L) == 1
            f = _create(L)
            assert lib.meao_resize(f, 640, 360) == 1
            assert _reservation(h).arena_bytes_needed == _reservation(f).arena_bytes <= r.arena_bytes
            lib.meao_destroy(f)
    finally:
        lib.meao_destroy(h)
        lib.meao_destroy(big)


def test_with_a_size_reservation_and_its_refusals():
    lib = N.lib()
    h = _create()
    try:
        assert lib.meao_reserve(h, *MAX) == 1 and lib.meao_reserve_layers(h, 4) == 1
        assert lib.meao_resize(h, 1280, 720) == 1
        assert lib.meao_resize(h, MAX[0] + 1, 720) == N.MEAO_ERR_INVALID and "outside the reservation" in _error(h)
        assert lib.meao_set_layers(h, 5) == N.MEAO_ERR_INVALID and "layer reservation 4" in _error(h)
        assert lib.meao_set_layers(h, 4) == 1
        assert lib.meao_reserve_layers(h, 3) == N.MEAO_ERR_INVALID and "below the current layer count 4" in _error(h)
        assert lib.meao_reserve(h, 1000, 720) == N.MEAO_ERR_INVALID and "width" in _error(h)
        assert lib.meao_layer_reservation(h) == 4 and _reservation(h).width == MAX[0]
        # clearing the size reservation keeps the layer reservation, and the other way round
        assert lib.meao_reserve(h, 0, 0) == 1 and lib.meao_layer_reservation(h) == 4
        assert lib.meao_set_layers(h, 2) == 1 and lib.meao_resize(h, 640, 360) == 1
        assert harness.plan_constants(h, 2) == _fresh_constants(640, 360, 2)
        assert lib.meao_reserve(h, *MAX) == 1 and lib.meao_reserve_layers(h, 0) == 1 and _reservation(h).width == MAX[0]
        assert lib.meao_set_layers(h, 9) == 1
    finally:
        lib.meao_destroy(h)


def test_row_bands_and_layer_reservations_exclude_each_other():
    lib = N.lib()
    h = _create()
    try:
        assert lib.meao_resize(h, 640, 352) == 1
        assert lib.meao_set_row_band(h, 0, 176, -1, 352) == 0
        g = lib.meao_frame_generation(h)
        assert lib.meao_reserve_layers(h, 4) == N.MEAO_ERR_UNSUPPORTED and "row band" in _error(h)
        assert lib.meao_layer_reservation(h) == 0 and lib.meao_frame_generation(h) == g
        assert lib.meao_set_row_band(h, 0, 352, -1, -1) == 0                 # back to the whole frame
        assert lib.meao_reserve_layers(h, 4) == 1
        g = lib.meao_frame_generation(h)
        assert lib.meao_set_row_band(h, 0, 176, -1, 352) == N.MEAO_ERR_UNSUPPORTED
        assert "reserves 4 layers, meao_reserve_layers" in _error(h) and lib.meao_frame_generation(h) == g
        rows = (C.c_int32 * 5)()
        assert lib.meao_halo_rows(h, 0, 1, rows) == N.MEAO_ERR_UNSUPPORTED
    finally:
        lib.meao_destroy(h)


def test_set_layers_before_the_first_resize():
    lib = N.lib()
    h = _create()
    try:
        assert lib.meao_reserve_layers(h, 6) == 1 and lib.meao_set_layers(h, 5) == 1
        assert lib.meao_resize(h, 321, 123) == 1
        assert harness.plan_constants(h, 5) == _fresh_constants(321, 123, 5)
    finally:
        lib.meao_destroy(h)


def test_slots_are_keyed_by_size_and_layer_count():
    """More distinct (W, H, L) than MEAO_SIZE_SLOTS, revisited in turn, with per-layer cameras set after each layer change: every
    getter equals a fresh context of that (W, H, L) with those cameras, and a parked (W, H, L) never answers for another count."""
    lib = N.lib()
    rng = random.Random(5)
    h = _create()
    triples = [(w, hh, L) for (w, hh) in [(1920, 1080), (641, 359), (17, 9)] for L in (1, 2, 4, 7)]
    try:
        assert lib.meao_reserve(h, *MAX) == 1 and lib.meao_reserve_layers(h, 7) == 1
        for i in range(40):
            w, hh, L = triples[(i * 5) % len(triples)] if i < 24 else rng.choice(triples)
            lib.meao_resize(h, w, hh)
            lib.meao_set_layers(h, L)
            cams = _cams(rng, L) if L > 1 and rng.random() < 0.6 else None
            if cams:
                assert _set_cams(h, cams) == 1
            else:
                assert lib.meao_set_layer_cameras(h, None, 0) >= 0
            assert harness.plan_constants(h, L) == _fresh_constants(w, hh, L, cams), (i, w, hh, L)
    finally:
        lib.meao_destroy(h)


def test_a_layer_change_clears_both_tables():
    lib = N.lib()
    rng = random.Random(3)
    h = _create()
    try:
        assert lib.meao_reserve_layers(h, 4) == 1 and lib.meao_resize(h, 320, 180) == 1 and lib.meao_set_layers(h, 3) == 1
        assert _set_cams(h, _cams(rng, 3)) == 1 and _set_views(h, [(0, 0, l, 0, 0, l) for l in range(3)]) == 1
        assert lib.meao_set_layers(h, 2) == 1
        assert lib.meao_get_layer_cameras(h, None, 0) == 0 and lib.meao_get_layer_viewports(h, None, 0) == 0
        assert harness.plan_constants(h, 2) == _fresh_constants(320, 180, 2)
        # a table whose Z direction differs from the shared camera's: clearing it is a structural change, and still no refusal
        cams = _cams(rng, 2, z=0)
        assert _set_cams(h, cams) == 1 and lib.meao_set_layers(h, 3) == 1
        assert harness.plan_constants(h, 3) == _fresh_constants(320, 180, 3)
    finally:
        lib.meao_destroy(h)


class Walk:
    """One plan-only context under both reservations; mirrors the inputs that decide each call's return value."""

    SIZES = [(1920, 1080), (1280, 720), (641, 359), (17, 9), (1000, 563)]

    def __init__(self, seed):
        self.lib, self.h, self.rng = N.lib(), _create(), random.Random(seed)
        self.max_layers = self.rng.choice([3, 6, 8])
        assert self.lib.meao_reserve(self.h, *MAX) == 1 and self.lib.meao_reserve_layers(self.h, self.max_layers) == 1
        self.layers, self.size, self.cams, self.views = 1, None, None, None
        self.gen = self.lib.meao_frame_generation(self.h)
        self.changes = self.noops = self.refusals = 0

    def expect(self, rc, want, tag):
        assert rc == want, f"{tag}: returned {rc}, expected {want} ({_error(self.h)})"
        g = self.lib.meao_frame_generation(self.h)
        assert (g != self.gen) == (rc == 1), f"{tag}: generation {self.gen} -> {g} after a call that returned {rc}"
        self.gen = g
        self.changes += rc == 1
        self.noops += rc == 0
        self.refusals += rc < 0

    def step(self, i):
        lib, h, rng = self.lib, self.h, self.rng
        action = rng.choice(["layers", "layers", "layers", "resize", "cams", "views", "constants"])
        tag = f"step {i} ({action})"
        if action == "layers":
            n = rng.choice(list(range(1, self.max_layers + 1)) + [self.layers, self.max_layers + 1, 0])
            want = N.MEAO_ERR_INVALID if not 1 <= n <= self.max_layers else int(n != self.layers)
            self.expect(lib.meao_set_layers(h, n), want, tag)
            if want == 1:
                self.layers, self.cams, self.views = n, None, None
        elif action == "resize":
            size = rng.choice(self.SIZES + [(MAX[0] + 1, 9)] + ([self.size] if self.size else []))
            want = N.MEAO_ERR_INVALID if size[0] > MAX[0] else int(size != self.size)
            self.expect(lib.meao_resize(h, *size), want, tag)
            if want == 1:
                self.size = size
        elif action == "cams":
            r = rng.random()
            if r < 0.25:
                self.expect(lib.meao_set_layer_cameras(h, None, 0), int(self.cams is not None), tag)
                self.cams = None
            elif r < 0.4:
                self.expect(_set_cams(h, _cams(rng, self.layers + 1)), N.MEAO_ERR_INVALID, tag)
            elif r < 0.55 and self.cams:
                self.expect(_set_cams(h, self.cams), 0, tag)
            else:
                cams = _cams(rng, self.layers)
                self.expect(_set_cams(h, cams), int(cams != self.cams), tag)
                self.cams = cams
        elif action == "views":
            r = rng.random()
            if r < 0.3:
                self.expect(lib.meao_set_layer_viewports(h, None, 0), int(self.views is not None), tag)
                self.views = None
            elif r < 0.4:
                self.expect(_set_views(h, [(0, 0, 0, -1, 0, 0)] * self.layers), N.MEAO_ERR_INVALID, tag)
            elif r < 0.55 and self.views:
                self.expect(_set_views(h, self.views), 0, tag)
            else:
                views = [(rng.randrange(4), 0, l, rng.randrange(4), 0, l) for l in range(self.layers)]
                self.expect(_set_views(h, views), int(views != self.views), tag)
                self.views = views
        elif self.size:
            assert harness.plan_constants(h, self.layers) == _fresh_constants(*self.size, self.layers, self.cams), tag
            self.expect(0, 0, tag)
        assert _reservation(h).arena_allocations == 0                           # plan-only: nothing is ever allocated


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_scripted_walk_return_values_and_generation(seed):
    w = Walk(seed)
    try:
        for i in range(300):
            w.step(i)
        assert w.changes > 80 and w.noops > 20 and w.refusals > 20, (w.changes, w.noops, w.refusals)
    finally:
        w.lib.meao_destroy(w.h)
