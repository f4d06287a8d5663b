"""CPU tests of dynamic resolution (meao_reserve) on plan-only contexts: after any sequence of resizes inside a reservation the
host-side plan -- every constant getter, per layer with per-layer cameras -- is bit-identical to a fresh context of that size; the
layout of every size fits the reserved arena; and the refusals leave the context as it was."""
import ctypes as C

import numpy as np
import pytest

from miniengineao_b200 import AmbientOcclusion, Camera
from miniengineao_b200 import _native as N

MAX = (3840, 2160)
# ragged sizes: 1x1, odd, not multiples of 4 / 16 / 64, the reservation itself, and more distinct sizes than the context keeps planned
SCHEDULE = [(3840, 2160), (3456, 1944), (2881, 1621), (1, 1), (17, 9), (1920, 1080), (3840, 2160), (2881, 1621), (63, 15), (1, 2160),
            (3840, 1), (129, 65), (1000, 999), (641, 359), (17, 9), (3457, 1945), (64, 16), (2881, 1621), (3, 5), (3840, 2160)]


def _new(layers=1, cams=None, variants=None, params=None):
    lib = N.lib()
    h = C.c_void_p()
    assert lib.meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
    if params:
        p = N.MeaoParams()
        lib.meao_default_params(C.byref(p))
        for k, v in params.items():
            setattr(p, k, v)
        assert lib.meao_set_params(h, C.byref(p)) >= 0
    if variants:
        assert lib.meao_set_variants(h, C.byref(N.MeaoVariants(*variants))) >= 0
    assert lib.meao_set_layers(h, layers) >= 0
    if cams:
        arr = (N.MeaoCamera * len(cams))(*[N.MeaoCamera(*c) for c in cams])
        assert lib.meao_set_layer_cameras(h, arr, len(cams)) >= 0
    return h


def _constants(h, layers):
    """Every constant getter of the plan, as one byte string."""
    lib = N.lib()
    parts = []
    for k in range(1, 5):
        for getter, n in ((lib.meao_render_constants, 28), (lib.meao_render_constants_wide, 28), (lib.meao_upsample_constants, 8)):
            out = (C.c_float * n)()
            assert getter(h, k, out) == 0
            parts.append(bytes(out))
        for l in range(layers):
            for wide in (0, 1):
                out = (C.c_float * 28)()
                assert lib.meao_render_constants_layer(h, l, k, wide, out) == 0
                parts.append(bytes(out))
    out = (C.c_float * 4)()
    assert lib.meao_zbuffer_params(h, out) == 0
    parts.append(bytes(out))
    for l in range(layers):
        assert lib.meao_zbuffer_params_layer(h, l, out) == 0
        parts.append(bytes(out))
    return b"".join(parts)


def _reservation(h):
    r = N.MeaoReservation()
    assert N.lib().meao_reservation(h, C.byref(r)) == 0
    return r


CAMS3 = [(0.3, 1000.0, 1.0, 1), (0.05, 20.0, 0.4142, 1), (2.0, 1e6, 1.7, 1)]
SETUPS = {
    "single": dict(layers=1),
    "layer_cameras": dict(layers=3, cams=CAMS3),
    "stereo_exhaustive_premin": dict(layers=2, variants=(1, 1, 15, 0)),
    "single_scale": dict(layers=1, variants=(0, 0, 0, 1), params=dict(upsample_tolerance=-3.0, blur_tolerance=-2.0)),
}


@pytest.mark.parametrize("setup", sorted(SETUPS))
def test_constants_after_resizes_match_a_fresh_context(setup):
    kw = SETUPS[setup]
    lib = N.lib()
    h = _new(**kw)
    assert lib.meao_reserve(h, *MAX) == 1
    try:
        for w, hh in SCHEDULE:
            lib.meao_resize(h, w, hh)
            f = _new(**kw)
            try:
                assert lib.meao_resize(f, w, hh) == 1
                assert _constants(h, kw["layers"]) == _constants(f, kw["layers"]), (w, hh)
            finally:
                lib.meao_destroy(f)
    finally:
        lib.meao_destroy(h)


def test_param_change_between_resizes_replans_every_size():
    """A plan input that changes while other sizes are parked: a later return to a parked size gets the new inputs."""
    lib = N.lib()
    h = _new(layers=3, cams=CAMS3)
    assert lib.meao_reserve(h, *MAX) == 1
    for w, hh in SCHEDULE[:6]:
        assert lib.meao_resize(h, w, hh) == 1
        _constants(h, 3)
    p = N.MeaoParams()
    lib.meao_default_params(C.byref(p))
    p.intensity, p.blur_tolerance = 1.7, -3.0
    assert lib.meao_set_params(h, C.byref(p)) == 1
    cams = (N.MeaoCamera * 3)(*[N.MeaoCamera(*c) for c in reversed(CAMS3)])
    assert lib.meao_set_layer_cameras(h, cams, 3) == 1
    for w, hh in reversed(SCHEDULE[:6]):
        lib.meao_resize(h, w, hh)
        f = _new(layers=3, cams=list(reversed(CAMS3)), params=dict(intensity=1.7, blur_tolerance=-3.0))
        assert lib.meao_resize(f, w, hh) == 1
        assert _constants(h, 3) == _constants(f, 3), (w, hh)
        lib.meao_destroy(f)
    lib.meao_destroy(h)


@pytest.mark.parametrize("layers", [1, 2, 6])
@pytest.mark.parametrize("wmax,hmax", [(3840, 2160), (1921, 1079), (257, 129), (64, 64), (1, 1)])
def test_every_size_fits_the_reserved_arena(layers, wmax, hmax):
    lib = N.lib()
    h = _new(layers=layers)
    assert lib.meao_reserve(h, wmax, hmax) == 1
    ref = _new(layers=layers)
    assert lib.meao_resize(ref, wmax, hmax) == 1
    full = _reservation(ref).arena_bytes
    lib.meao_destroy(ref)
    assert full > 0
    ws = sorted({1, 2, 3, 4, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 1000, 1919, 2881} | {wmax, max(1, wmax - 1)})
    hs = sorted({1, 2, 3, 8, 9, 31, 33, 100, 1079, 1621} | {hmax, max(1, hmax - 1)})
    for w in [x for x in ws if x <= wmax]:
        for hh in [y for y in hs if y <= hmax]:
            assert lib.meao_resize(h, w, hh) >= 0
            r = _reservation(h)
            assert (r.width, r.height) == (wmax, hmax)
            assert r.arena_bytes == full, "a reservation allocates what an unreserved context of the maximum size does"
            assert 0 < r.arena_bytes_needed <= r.arena_bytes, (w, hh)
            if w == wmax and hh == hmax:
                assert r.arena_bytes_needed == full
    lib.meao_destroy(h)


def _size(h):
    d = N.MeaoBufferDesc()
    assert N.lib().meao_buffer_desc(h, 17, C.byref(d)) == 0
    return d.width, d.height


def _err(h):
    return N.lib().meao_last_error(h).decode()


def test_return_values_and_clearing():
    lib = N.lib()
    h = _new()
    assert lib.meao_reserve(h, 0, 0) == 0                     # nothing reserved: the same (empty) reservation again
    assert lib.meao_reserve(h, 1920, 1080) == 1               # before the first resize: recorded
    assert lib.meao_reserve(h, 1920, 1080) == 0
    assert lib.meao_resize(h, 1280, 720) == 1
    assert lib.meao_resize(h, 1280, 720) == 0
    assert lib.meao_resize(h, 1920, 1080) == 1
    assert lib.meao_resize(h, 1280, 720) == 1                 # back to a parked size: still a change of size
    assert lib.meao_reserve(h, 2560, 1440) == 1
    assert _size(h) == (1280, 720)
    assert lib.meao_reserve(h, 0, 0) == 1                     # cleared: the arena is for the current size again
    r = _reservation(h)
    assert (r.width, r.height) == (0, 0) and r.arena_bytes == r.arena_bytes_needed
    assert lib.meao_resize(h, 2560, 1440) == 1                # no reservation: any size
    assert lib.meao_reserve(h, 0, 0) == 0
    lib.meao_destroy(h)


def test_refusals_change_nothing():
    lib = N.lib()
    h = _new(layers=2, cams=CAMS3[:2])
    assert lib.meao_reserve(h, 1920, 1080) == 1
    assert lib.meao_resize(h, 1001, 601) == 1
    before = (_size(h), _constants(h, 2), bytes(_reservation(h)))

    def unchanged():
        assert (_size(h), _constants(h, 2), bytes(_reservation(h))) == before

    for w, hh in ((1921, 1080), (1920, 1081), (4000, 3000)):
        assert lib.meao_resize(h, w, hh) == N.MEAO_ERR_INVALID
        assert "reservation" in _err(h)
        unchanged()
    assert lib.meao_reserve(h, 1000, 1080) == N.MEAO_ERR_INVALID
    assert "width" in _err(h)
    unchanged()
    assert lib.meao_reserve(h, 1920, 600) == N.MEAO_ERR_INVALID
    assert "height" in _err(h)
    unchanged()
    for w, hh in ((-1, 100), (100, -1), (0, 100), (100, 0), (32769, 100), (100, 32769)):
        assert lib.meao_reserve(h, w, hh) == N.MEAO_ERR_INVALID
        unchanged()
    lib.meao_destroy(h)


def test_row_bands_and_reservations_exclude_each_other():
    lib = N.lib()
    # band first, then a reservation
    h = _new()
    assert lib.meao_resize(h, 640, 480) == 1
    assert lib.meao_set_row_band(h, 0, 240, -1, 480) == 0
    assert lib.meao_reserve(h, 1280, 720) == N.MEAO_ERR_UNSUPPORTED
    assert "row band" in _err(h)
    assert _reservation(h).width == 0
    lib.meao_destroy(h)
    # a reservation first, then every band / halo / exchange entry point
    h = _new()
    assert lib.meao_reserve(h, 1280, 720) == 1
    assert lib.meao_resize(h, 640, 480) == 1
    rows = (C.c_int32 * 8)()
    calls = [
        lambda: lib.meao_set_row_band(h, 0, 240, -1, 480),
        lambda: lib.meao_halo_bytes(h, 1),
        lambda: lib.meao_halo_recv_bytes(h, 1),
        lambda: lib.meao_halo_rows(h, 1, 1, rows),
        lambda: lib.meao_halo_pack(h, 1, None, None),
        lambda: lib.meao_halo_unpack(h, 1, None, None),
        lambda: lib.meao_render_band_prepare(h, None, 0, None),
        lambda: lib.meao_render_band_finish(h, None, None),
        lambda: lib.meao_band_phase_a(h, None, 0, None, None, None),
        lambda: lib.meao_band_phase_b(h, None, None, None, None),
        lambda: lib.meao_band_export(h, None),
        lambda: lib.meao_band_connect(h, 1, None),
        lambda: lib.meao_band_step(h, None, 0, None, None),
        lambda: lib.meao_band_step_host(h, None, 0, None),
    ]
    for call in calls:
        assert call() == N.MEAO_ERR_UNSUPPORTED
        assert "meao_reserve" in _err(h)
    assert _size(h) == (640, 480)
    lib.meao_destroy(h)


def test_set_layers_keeps_the_reservation():
    lib = N.lib()
    h = _new()
    assert lib.meao_reserve(h, 1920, 1080) == 1
    assert lib.meao_resize(h, 999, 555) == 1
    assert lib.meao_set_layers(h, 6) == 1
    r = _reservation(h)
    f = _new(layers=6)
    assert lib.meao_resize(f, 1920, 1080) == 1
    assert (r.width, r.height, r.arena_bytes) == (1920, 1080, _reservation(f).arena_bytes)
    assert _size(h) == (999, 555)
    lib.meao_destroy(f)
    lib.meao_destroy(h)


@pytest.mark.parametrize("stereo", [False, True])
def test_python_max_resolution(stereo):
    cam = Camera(1280, 720, stereoEnabled=stereo)
    ao = AmbientOcclusion(cam, device=-1)
    ao.maxResolution = (1920, 1080)
    if stereo:
        ao.OnPreRender()                                      # one draw for both eyes: single-pass stereo
    assert ao.LateUpdate() is True
    r = ao.reservation()
    assert (r["width"], r["height"]) == ((3840 if stereo else 1920), 1080)
    assert ao._width == (2560 if stereo else 1280)
    # a size change inside the reservation, then a reservation below the current size: the host resizes first
    cam.pixelWidth, cam.pixelHeight = 1600, 900
    if stereo:
        ao.OnPreRender()
    ao.LateUpdate()
    assert ao.reservation()["width"] == (3840 if stereo else 1920)
    ao.maxResolution = (1600, 900)
    if stereo:
        ao.OnPreRender()
    ao.LateUpdate()
    assert (ao.reservation()["width"], ao.reservation()["height"]) == ((3200 if stereo else 1600), 900)
    cam.pixelWidth, cam.pixelHeight = 1280, 720               # a reservation below the current size: the host resizes first
    ao.maxResolution = (1280, 720)
    if stereo:
        ao.OnPreRender()
    ao.LateUpdate()
    assert (ao.reservation()["width"], ao.reservation()["height"]) == ((2560 if stereo else 1280), 720)
    ao.maxResolution = None
    if stereo:
        ao.OnPreRender()
    ao.LateUpdate()
    assert ao.reservation()["width"] == 0
    ao.close()
