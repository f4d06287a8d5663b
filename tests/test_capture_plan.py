"""CPU tests of meao_frame_generation on plan-only contexts.  A frame recorded into a caller's CUDA graph replays with everything it was
recorded with, so the generation must change at every call that changed something a frame depends on -- a frame constant, a size, a
structural input, a reservation, a row band -- and at no other: not at a setter given the value it already has, not at a refused call,
not at a getter or a frame.  A long scripted walk mixes all of them on several setups."""
import ctypes as C
import random

import pytest

import harness
from miniengineao_b200 import _native as N

SIZES = [(1920, 1080), (1280, 720), (641, 359), (17, 9), (3840, 2160), (1000, 563)]
RESERVATIONS = [(0, 0), (1920, 1080), (3840, 2160), (4000, 2200)]


def _create():
    h = C.c_void_p()
    assert N.lib().meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
    return h


def _cam(rng, z=1):
    near = rng.choice([0.05, 0.3, 1.0])
    return (near, near * rng.choice([100.0, 3000.0]), rng.choice([0.5, 1.0, 1.7]), z)


class Walk:
    """Drives one plan-only context and mirrors the inputs that decide whether a call changes anything."""

    def __init__(self, seed):
        self.lib, self.h, self.rng = N.lib(), _create(), random.Random(seed)
        self.layers, self.camera, self.table, self.size, self.res = 1, (0.3, 1000.0, 1.0, 1), None, None, (0, 0)
        self.params = N.MeaoParams()
        self.lib.meao_default_params(C.byref(self.params))
        self.gen = self.generation()
        self.changes = self.noops = self.refusals = 0

    def generation(self):
        g = self.lib.meao_frame_generation(self.h)
        assert g >= 0
        return g

    def expect(self, changed, tag):
        g = self.generation()
        if changed:
            assert g != self.gen, f"{tag}: a call that changed something left the generation at {g}"
            self.changes += 1
        else:
            assert g == self.gen, f"{tag}: a call that changed nothing moved the generation {self.gen} -> {g}"
        self.gen = g

    def step(self, i):
        lib, h, rng = self.lib, self.h, self.rng
        action = rng.choice(["params", "params", "camera", "camera", "table", "variants", "layers", "resize", "resize", "reserve",
                             "getters", "frame"])
        tag = f"step {i} ({action})"
        if action == "params":
            p = N.MeaoParams()
            C.memmove(C.byref(p), C.byref(self.params), C.sizeof(p))
            r = rng.random()
            if r < 0.3:
                pass                                                            # the same block again
            elif r < 0.4:
                p.ambient_only = 1 - p.ambient_only                             # not a frame constant (CheckPropertiesChanged)
            elif r < 0.5:
                p.thickness_modifier = rng.choice([0.0, -2.0])                  # refused
                p.intensity = 1.9
            else:
                p.intensity, p.blur_tolerance = rng.choice([0.5, 1.0, 1.5]), rng.choice([-4.6, -3.0])
            rc = lib.meao_set_params(h, C.byref(p))
            if rc >= 0:
                self.params = p
            self.count(rc)
            self.expect(rc == 1, tag)
        elif action == "camera":
            z = self.table[0][3] if self.table else self.camera[3]
            r = rng.random()
            if r < 0.3:
                cam = self.camera
            elif r < 0.45:
                cam = (0.0, 10.0, 1.0, z) if rng.random() < 0.5 else (2.0, 1.0, 1.0, z)       # refused
            elif r < 0.55:
                cam = self.camera[:3] + (1 - self.camera[3],)                   # the Z direction: a structural change
            else:
                cam = _cam(rng, self.camera[3])
            rc = lib.meao_set_camera(h, C.byref(N.MeaoCamera(*cam)))
            if rc < 0:
                self.refusals += 1
                self.expect(False, tag)
                return
            changed = cam != self.camera and self.table is None               # under a table the shared camera waits for the clear
            self.camera = cam
            self.noops += not changed
            self.expect(changed, tag)
        elif action == "table":
            z = self.table[0][3] if self.table else self.camera[3]
            r = rng.random()
            if r < 0.25:
                rc = lib.meao_set_layer_cameras(h, None, 0)
                if rc == 1:
                    self.table = None
            elif r < 0.4 and self.table:
                t = self.table
                rc = lib.meao_set_layer_cameras(h, (N.MeaoCamera * len(t))(*[N.MeaoCamera(*c) for c in t]), len(t))
            elif r < 0.55:
                n = self.layers + 1                                             # refused: one camera per layer
                t = [_cam(rng, z) for _ in range(n)]
                rc = lib.meao_set_layer_cameras(h, (N.MeaoCamera * n)(*[N.MeaoCamera(*c) for c in t]), n)
                assert rc == N.MEAO_ERR_INVALID
            else:
                t = [_cam(rng, z) for _ in range(self.layers)]
                rc = lib.meao_set_layer_cameras(h, (N.MeaoCamera * len(t))(*[N.MeaoCamera(*c) for c in t]), len(t))
                if rc == 1:
                    self.table = t
            self.count(rc)
            self.expect(rc == 1, tag)
        elif action == "variants":
            r = rng.random()
            if r < 0.2:
                v = (0, 0, 3, 1)                                                # refused: single_scale excludes the high-quality mask
            elif r < 0.3:
                v = (0, 0, 16, 0)                                               # refused: mask out of range
            else:
                v = (0, rng.randrange(2), rng.choice([0, 0, 8, 15]), 0)
            rc = lib.meao_set_variants(h, C.byref(N.MeaoVariants(*v)))
            self.count(rc)
            self.expect(rc == 1, tag)
        elif action == "layers":
            n = rng.choice([1, 1, 2, 6, 0])                                     # 0: refused
            rc = lib.meao_set_layers(h, n)
            if rc == 1:
                self.layers, self.table = n, None                               # a new layer count clears the table
            self.count(rc)
            self.expect(rc == 1, tag)
        elif action == "resize":
            r = rng.random()
            if r < 0.15:
                size = (0, 5) if rng.random() < 0.5 else (40000, 10)            # refused: bounds
            elif r < 0.3 and self.res != (0, 0):
                size = (self.res[0] + 16, self.res[1])                          # refused: outside the reservation
            elif r < 0.45 and self.size:
                size = self.size
            else:
                fits = [s for s in SIZES if self.res == (0, 0) or (s[0] <= self.res[0] and s[1] <= self.res[1])]
                size = rng.choice(fits or [self.res])
            rc = lib.meao_resize(h, *size)
            if rc >= 0:
                self.size = size
            self.count(rc)
            self.expect(rc == 1, tag)
        elif action == "reserve":
            res = rng.choice(RESERVATIONS + [self.res, (8, 8)])                 # (8, 8): refused once the size is larger
            rc = lib.meao_reserve(h, *res)
            if rc >= 0:
                self.res = res
            self.count(rc)
            self.expect(rc == 1, tag)
        elif action == "getters":
            if self.size:
                harness.plan_constants(h, self.layers)                          # re-plans on the host: nothing a frame depends on changes
                rows = (C.c_int32 * 30)()
                assert lib.meao_band_rows(h, rows) == 0
            r = N.MeaoReservation()
            assert lib.meao_reservation(h, C.byref(r)) == 0
            lib.meao_kernels_per_frame(h)
            self.expect(False, tag)
        else:                                                                   # frames fail on a plan-only context and change nothing
            assert lib.meao_render(h, None, 0, None, None) < 0
            assert lib.meao_synchronize(h) == 0
            self.expect(False, tag)

    def count(self, rc):
        if rc < 0:
            self.refusals += 1
        elif rc == 0:
            self.noops += 1


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generation_changes_exactly_at_the_calls_that_change_something(seed):
    w = Walk(seed)
    try:
        for i in range(600):
            w.step(i)
        assert w.changes > 100 and w.noops > 60 and w.refusals > 40, (w.changes, w.noops, w.refusals)
    finally:
        w.lib.meao_destroy(w.h)


def test_generation_follows_the_plan_constants():
    """Whenever a constant getter's answer moves, the generation has moved with it (a frame recorded before would replay stale ones)."""
    w = Walk(7)
    try:
        before, gen = None, None
        for i in range(300):
            w.step(i)
            if w.size is None:
                continue
            now = harness.plan_constants(w.h, w.layers) + bytes(str((w.size, w.layers)), "ascii")
            g = w.generation()
            if before is not None and now != before:
                assert g != gen, f"step {i}: the plan changed and the generation did not"
            before, gen = now, g
    finally:
        w.lib.meao_destroy(w.h)


def test_row_band_calls():
    lib = N.lib()
    a = harness.context(1920, 1088)
    a.LateUpdate()
    g = a.frame_generation
    a.set_row_band(0, 544, -1, 1088)
    assert a.frame_generation != g, "a new row band"
    g = a.frame_generation
    with pytest.raises(N.MeaoError):
        a.set_row_band(272, 544, 0, 816)                                        # refused: the halo reaches past the band above
    with pytest.raises(N.MeaoError):
        a.set_row_band(100, 544, 0, 816)                                        # refused: not 16-row aligned
    assert a.frame_generation == g
    a.halo_rows(1, True), a.band_rows(), a.halo_bytes(1)
    assert a.frame_generation == g
    assert lib.meao_band_connect(a._ctx, 1, None) == N.MEAO_ERR_CUDA              # plan-only: refused before anything changes
    assert a.frame_generation == g


def test_the_host_mirror_applies_pending_properties_first():
    a = harness.context(640, 360)
    g = a.frame_generation
    assert a.frame_generation == g, "reading it twice"
    a.intensity = 1.5
    assert a.frame_generation != g, "a changed property is applied before the generation is read"
    g = a.frame_generation
    a.camera.fieldOfView = 70.0
    assert a.frame_generation != g
    g = a.frame_generation
    a.LateUpdate()
    assert a.frame_generation == g, "LateUpdate with unchanged properties changes nothing"
    assert N.lib().meao_frame_generation(None) == N.MEAO_ERR_INVALID
