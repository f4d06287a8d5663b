"""CPU tests of dynamic resolution (meao_reserve): frames of smaller, ragged sizes run inside ONE arena laid out for the largest size,
at the offsets and pitches of arena_layout (csrc/arena_layout.h, shared with meao_api.cu), through the host-compiled kernel sources
(tests/emu/drs_driver.cpp).  The arena first holds stale data -- the buffers of a hostile frame at the maximum size, or an 0xFF
poison (NaN in every f16 / f32) -- where a fresh context's arena holds zeros; any kernel that read a byte its frame did not write
(pitch padding, rows beyond the frame) would change bits.  AO and every debug buffer of every layer must equal the oracle's, for single
and layered frames, with and without the fused final level, and for the premin and single-scale variants."""
import ctypes as C

import numpy as np
import pytest

import hostile_cases as HC
from emu import build_drs_emu  # noqa: E402  (tests/ is on sys.path via conftest)
from emu.layered_emu import _aligned
from miniengineao_b200 import _native as N
from oracle.oracle import Oracle
from test_layers_emulated import _compare_layer, _plan, _raw, contrasting_layers

MAX = (330, 190)
SIZES = [(1, 1), (33, 17), (97, 61), (329, 189), (257, 131), (64, 32)]

_lib = None


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(build_drs_emu.build())
        l.demu_create.restype = C.c_void_p
        l.demu_create.argtypes = [C.c_int, C.c_int, C.c_int]
        l.demu_destroy.argtypes = [C.c_void_p]
        l.demu_arena_bytes.restype = C.c_size_t
        l.demu_arena_bytes.argtypes = [C.c_void_p]
        l.demu_fill.argtypes = [C.c_void_p, C.c_int]
        l.demu_resize.argtypes = [C.c_void_p, C.c_int, C.c_int]
        l.lemu_set_constants.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float] + [C.c_int] * 6
        l.lemu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        l.femu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        l.lemu_get_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        _lib = l
    return _lib


class Frame:
    """The frames of one reserved arena: resize() places the buffers of a size and loads its plan, run() renders one frame."""

    def __init__(self, layers, fused, **kw):
        self.L, self.fused, self.kw = layers, fused, kw
        self.h = lib().demu_create(*MAX, layers)

    def close(self):
        lib().demu_destroy(self.h)

    def resize(self, W, H):
        assert lib().demu_resize(self.h, W, H) == 0
        self.W, self.H = W, H
        self.plan = p = _plan(W, H, self.L, **self.kw)
        p.LateUpdate()
        nl = N.lib()
        rc, rcw, uc, zb = (C.c_float * 112)(), (C.c_float * 112)(), (C.c_float * 32)(), (C.c_float * 4)()
        for k in range(1, 5):
            nl.meao_render_constants(p._ctx, k, C.cast(C.byref(rc, 112 * (k - 1)), C.POINTER(C.c_float)))
            nl.meao_render_constants_wide(p._ctx, k, C.cast(C.byref(rcw, 112 * (k - 1)), C.POINTER(C.c_float)))
            nl.meao_upsample_constants(p._ctx, k, C.cast(C.byref(uc, 32 * (k - 1)), C.POINTER(C.c_float)))
        nl.meao_zbuffer_params(p._ctx, zb)
        self.zb = np.array(zb[:])
        lib().lemu_set_constants(self.h, rc, rcw, uc, zb, 1e5, 1, 1, int(p.highQualityMask), int(p.sampleExhaustively), int(p.singleScale), 1)

    def run(self, depth):
        d = _aligned(np.ascontiguousarray(depth, np.float32))
        if self.fused:
            lib().femu_run(self.h, d.ctypes.data, 0, 0, 0)
        else:
            lib().lemu_run(self.h, d.ctypes.data, 0)

    def buffer(self, bid, layer):
        d = self.plan.buffer_desc(bid)
        dt = {1: np.uint8, 2: np.float16, 4: np.float32}[d.elem_bytes]
        out = np.zeros((d.slices, d.height, d.width) if d.slices > 1 else (d.height, d.width), dt)
        assert lib().lemu_get_buffer(self.h, bid, layer, out.ctypes.data) == 0
        return out


def test_layout_is_the_librarys():
    """The arena the driver allocates is the one meao_reserve reports for the same reservation and layer count."""
    for L in (1, 3):
        h = lib().demu_create(*MAX, L)
        p = _plan(64, 32, L)
        p.maxResolution = MAX
        p.LateUpdate()
        assert lib().demu_arena_bytes(h) == p.reservation()["arena_bytes"]
        assert lib().demu_resize(h, MAX[0] + 1, MAX[1]) == -1
        lib().demu_destroy(h)


CASES = {
    "single_fused": dict(layers=1, fused=True),
    "single_full": dict(layers=1, fused=False),
    "layered_fused": dict(layers=3, fused=True),
    "layered_full": dict(layers=3, fused=False),
    "premin_fused": dict(layers=1, fused=True, high_quality_mask=1),
    "premin_layered_full": dict(layers=2, fused=False, high_quality_mask=15),
    "single_scale_fused": dict(layers=1, fused=True, single_scale=True),
    "single_scale_layered_full": dict(layers=3, fused=False, single_scale=True),
}


@pytest.mark.parametrize("stale", ["max_frame", "poison"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_smaller_frames_in_a_stale_arena_match_the_oracle(case, stale):
    kw = dict(CASES[case])
    L, fused = kw.pop("layers"), kw.pop("fused")
    f = Frame(L, fused, intensity=1.1, **kw)
    try:
        if stale == "max_frame":
            f.resize(*MAX)
            hostile = np.stack([HC.hostile_raw(*MAX, f.zb, True, seed=l) for l in range(L)])
            f.run(hostile)
        else:
            f.resize(*MAX)
            lib().demu_fill(f.h, 0xFF)
        ids = [1, 2, 3, 4, 5, 10, 17] if kw.get("single_scale") else None
        for i, (W, H) in enumerate(SIZES):
            f.resize(W, H)
            depth = _raw(contrasting_layers(W, H, L, seed=i))
            f.run(depth)
            for l in range(L):
                orc = Oracle(W, H, threads=4, intensity=1.1, **kw)
                ref = orc.run(depth[l])
                assert np.array_equal(f.buffer(17, l), ref), (case, stale, W, H, l)
                _compare_layer(f, l, orc, f"{case} {stale} {W}x{H}", kw.get("high_quality_mask", 0), ids)
    finally:
        f.close()
