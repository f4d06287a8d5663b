"""CPU tests of dynamic view counts (meao_reserve_layers): frames of L = 1, 3, 2, 5 and 1 layers, at sizes inside a size reservation,
run inside ONE arena laid out for the largest size and the reserved layer count, at the offsets arena_layout gives under a layer
reservation (csrc/arena_layout.h with table_layers = Lmax, what meao_api.cu's place_size uses), through the host-compiled kernel
sources.  The arena first holds the buffers of a hostile frame at the maximum size and layer count, where a fresh context's arena holds
zeros; a kernel that read a byte its frame did not write, or a layer image or camera table placed outside its own bytes, would change
bits.  Every layer, with its own camera, must equal the oracle on every buffer id, fused and unfused."""
import ctypes as C
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import harness
import hostile_cases as HC
from emu import build_emu
from emu.emu import Frame, lib as emu_lib
from miniengineao_b200 import Camera

MAX = (200, 120)
LMAX = 6
# (W, H, L): the view count moves up and down inside the reservation, with sizes inside the size reservation
SCHEDULE = [(200, 120, 1), (97, 61, 3), (33, 17, 2), (161, 89, 5), (200, 120, 1), (64, 32, 3)]

SRC = os.path.join(build_emu.HERE, "frame_layers.cpp")
LIB = os.path.join(build_emu.HERE, "libmeao_emu_layers.so")
_lib = None


def layers_lib():
    """tests/emu/frame_layers.cpp, linked against libmeao_emu.so (one instance of the emulator), built through a private temporary
    directory and an atomic rename like the other emulator libraries."""
    global _lib
    if _lib is None:
        emu_lib()
        base = build_emu.LIB
        deps = [base, SRC] + [os.path.join(build_emu.CSRC, f) for f in os.listdir(build_emu.CSRC)]
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
            tmp = tempfile.mkdtemp(prefix="meao_emu_layers_")
            try:
                obj, out = os.path.join(tmp, "frame_layers.o"), os.path.join(tmp, "lib.so")
                p = subprocess.run(["g++"] + build_emu.FLAGS + ["-c", SRC, "-o", obj], capture_output=True, text=True)
                if p.returncode:
                    sys.stderr.write(p.stdout + p.stderr)
                    raise RuntimeError("emulator build failed: frame_layers.cpp")
                subprocess.check_call(["g++", "-shared", "-o", out, obj, "-L", build_emu.HERE, "-l:" + os.path.basename(base),
                                       "-Wl,-rpath,$ORIGIN"])
                staged = f"{LIB}.tmp{os.getpid()}"
                shutil.copyfile(out, staged)
                os.replace(staged, LIB)
            finally:
                shutil.rmtree(tmp, ignore_errors=True)
        l = C.CDLL(LIB)
        l.frame_place_layers.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_longlong]
        l.frame_layers_layout.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_longlong)]
        _lib = l
    return _lib


def layout(W, H, L, Lmax):
    out = (C.c_longlong * 5)()
    layers_lib().frame_layers_layout(W, H, L, Lmax, out)
    return tuple(out)


class _PlaceLayers:
    """The emulator library with frame_resize replaced by the placement of a layer-reserved context: the frame's layer count, the
    tables laid out for LMAX, and its camera tables in the next of the MEAO_SIZE_SLOTS slots."""

    def __init__(self, frame, base):
        self._frame, self._base, self.slot = frame, base, -1

    def __getattr__(self, name):
        return getattr(self._base, name)

    def frame_resize(self, h, W, H):
        self.slot = (self.slot + 1) % 8
        return layers_lib().frame_place_layers(h, W, H, self._frame.layers, LMAX, self.slot, self._frame.arena_bytes())


def _cams(W, H, L, seed):
    rng = np.random.default_rng(seed)
    return [Camera(W, H, nearClipPlane=float(rng.choice([0.05, 0.3, 1.0])), farClipPlane=float(rng.choice([50.0, 1000.0, 3e4])),
                   fieldOfView=float(rng.choice([40.0, 60.0, 90.0]))) for _ in range(L)]


def _plan(W, H, L, seed, **kw):
    cams = _cams(W, H, L, seed) if L > 1 else None
    return harness.context(W, H, layers=L, layer_cameras=cams, intensity=1.1, **kw), cams


def test_layout_tables_do_not_move_and_every_frame_fits():
    """Under a layer reservation the tile counters, the camera-table slots and the viewport table sit at offsets no (W, H, L) moves,
    and every (W, H, L <= Lmax) fits the arena of (Wmax, Hmax, Lmax); without one (table_layers = L) the offsets do move with L."""
    full = layout(*MAX, LMAX, LMAX)
    for W, H in [(1, 1), (33, 17), MAX, (200, 1), (1, 120)]:
        for L in range(1, LMAX + 1):
            a = layout(W, H, L, LMAX)
            assert a[:4] == full[:4] and a[4] <= full[4], (W, H, L)
    assert layout(*MAX, 2, 2)[1:4] != full[1:4]


def test_arena_is_the_librarys():
    """The arena the driver allocates is the one meao_reservation reports for the same size and layer reservations."""
    p = harness.context(64, 32, layers=2)
    p.maxResolution, p.maxLayers = MAX, LMAX
    p.LateUpdate()
    f = Frame(harness.context(*MAX, layers=LMAX), max_size=MAX)
    r = p.reservation()
    assert f.arena_bytes() == r["arena_bytes"] == layout(*MAX, LMAX, LMAX)[4]
    assert r["arena_bytes_needed"] == layout(64, 32, 2, 2)[4]


CASES = {
    "fused": dict(fused=True),
    "full": dict(fused=False),
    "premin_fused": dict(fused=True, high_quality_mask=15),
    "single_scale_full": dict(fused=False, single_scale=True),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_changing_view_counts_in_one_stale_arena_match_the_oracle(case):
    kw = dict(CASES[case])
    fused = kw.pop("fused")
    f = Frame(_plan(*MAX, LMAX, 99, **kw)[0], max_size=MAX)
    run = (lambda fr, d: fr.run_fused(d)) if fused else (lambda fr, d: fr.run(d))
    f.fill()
    run(f, np.stack([HC.hostile_raw(*MAX, f.zb, True, seed=l) for l in range(LMAX)]).astype(np.float32))
    f._lib = _PlaceLayers(f, f._lib)
    ids = harness.buffer_ids(kw.get("high_quality_mask", 0), kw.get("single_scale", False))
    for i, (W, H, L) in enumerate(SCHEDULE):
        plan, cams = _plan(W, H, L, i, **kw)
        f.layers = L
        f.load(plan)
        depth = harness.raw(harness.contrasting_layers(W, H, L, seed=i)).astype(np.float32)
        run(f, depth)
        for l in range(L):
            orc = harness.oracle(W, H, camera=cams[l] if cams else None, intensity=1.1, **kw)
            ref = orc.run(depth[l])
            assert np.array_equal(f.buffer(17, l), ref), (case, W, H, L, l)
            harness.compare_buffers(lambda bid: f.buffer(bid, l), orc, f"{case} {W}x{H}x{L} layer {l}", ids)
