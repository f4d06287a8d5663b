"""CPU tests of the device-parameter units (build.py PARAM_SOURCES) in the emulator (tests/emu/device_params.py).

- The slot the parameter stage derives from {thickness_modifier, intensity} is, byte for byte, the reject_fadeoff and intensity of a
  plan-only libmeao context given the same MeaoParams (meao_render_constants), for random, subnormal, huge and infinite thickness and any
  intensity (NaN included).  An invalid thickness (0, -0, negative, -inf, NaN) leaves the slot as it was and counts in the status words.
- Whole frames through the render twins at L = 1 (a twin with one layer) and L = 2 / 3 equal, on every buffer (ids 1-21), the same frame
  of a plan whose HOST parameters are the buffer's, launched without the binding -- perspective, orthographic and mixed projections,
  checker and exhaustive sampling, narrow and wide renders at every tile height, single-pass stereo, with and without device cameras --
  while the bound plan's host parameters are other ones.  Each frame launches exactly the parameter stage and the expected twins, and the
  frames name all 37 kernels of the units.
- An invalid block reproduces the frame of the last valid one."""
import itertools
import math

import ctypes as C
import numpy as np
import pytest

import harness
from emu import batch, emu, layer_views, mixed, ortho
from emu import device_cameras as DC
from emu import device_params as DP
from miniengineao_b200 import _native as N
from test_device_cameras_emulated import camera, plan_of, rows

P, O = N.MEAO_PROJECTION_PERSPECTIVE, N.MEAO_PROJECTION_ORTHOGRAPHIC
DEV = (2.3, 0.6)                    # the device block
HOST = dict(thickness_modifier=0.8, intensity=1.4)     # the bound plan's host values: never read by a bound frame
FAMILY = {"persp": "render_ao_params_layered_kernel", "ortho": "render_ao_ortho_params_layered_kernel",
          "mixed": "render_ao_mixed_params_layered_kernel"}
TILE_H = (32, 16, 8)                # MEAO_REN_TILE 0 / 1 / 2


# ---- the parameter stage ----------------------------------------------------------------------------------------------------------
def host_derived(tm: float, intensity: float) -> np.ndarray:
    """reject_fadeoff and intensity of a plan-only context given (tm, intensity): out[26], out[27] of meao_render_constants."""
    lib = N.lib()
    h = C.c_void_p()
    assert lib.meao_create(C.byref(N.MeaoDeviceCfg(-1, 0)), C.byref(h)) == 0
    p = N.MeaoParams()
    lib.meao_default_params(C.byref(p))
    p.thickness_modifier, p.intensity = tm, intensity
    assert lib.meao_set_params(h, C.byref(p)) >= 0
    assert lib.meao_resize(h, 64, 40) == 1
    out = (C.c_float * 28)()
    assert lib.meao_render_constants(h, 1, out) == 0
    lib.meao_destroy(h)
    return np.array([out[26], out[27]], np.float32)


def _f32(x):
    return float(np.float32(x))


def _valid_blocks():
    rng = np.random.default_rng(7)
    tms = [_f32(10 ** rng.uniform(-6, 6)) for _ in range(24)]
    tms += [1e-40, 1.4e-45, 1.17549435e-38, 5e-39, 3e38, 3.4028235e38, math.inf, 1.0, 0.5, 3.0]     # subnormal, huge, inf
    ins = [_f32(rng.uniform(-2, 3)) for _ in range(len(tms))]
    ins[:6] = [0.0, -0.0, 1e30, -1e-42, math.inf, math.nan]
    return list(zip(tms, ins))


@pytest.mark.parametrize("tm,intensity", _valid_blocks())
def test_the_slot_is_the_host_planners_bytes(tm, intensity):
    slot = DP.new_slot(-7.0, 7.0)
    DP.derive([tm, intensity], slot)
    assert slot[:2].tobytes() == host_derived(tm, intensity).tobytes(), (tm, intensity, slot[:2], host_derived(tm, intensity))
    assert DP.status(slot) == [0, 0]


@pytest.mark.parametrize("bad", [0.0, -0.0, -1.0, -1e-40, -math.inf, math.nan])
def test_an_invalid_block_leaves_the_slot_and_counts(bad):
    slot = DP.new_slot(-0.25, 1.5)
    before = slot[:2].tobytes()
    DP.derive([bad, 0.3], slot)
    assert slot[:2].tobytes() == before and DP.status(slot) == [1, 1]
    DP.derive([bad, 0.9], slot)
    assert slot[:2].tobytes() == before and DP.status(slot) == [2, 1]
    DP.derive([4.0, 0.9], slot)
    assert slot[:2].tobytes() == host_derived(4.0, 0.9).tobytes() and DP.status(slot) == [2, 1]


def test_the_unit_tables_list_every_kernel():
    assert DP.kernel_units() == {"render_params.cu": 1, "render_ao_params_layered.cu": 12, "render_ao_ortho_params_layered.cu": 12,
                                 "render_ao_mixed_params_layered.cu": 12}
    assert len(DP.kernels()) == 37


def test_the_librarys_kernels_have_distinct_offsets():
    """The ledger keys a kernel by its offset in its own library (emu.unit_ledger): none of this library's may share one."""
    mine = set(DP._kernel_symbols())
    others = set(emu._kernel_symbols()).union(*(set(m._kernel_symbols()) for m in (ortho, mixed, batch, layer_views, DC)))
    assert mine and not mine & others


# ---- whole frames -----------------------------------------------------------------------------------------------------------------
def _cases():
    """(family, table, tile, exhaustive, device cameras, stereo): every family at every tile height, checker and exhaustive, all with
    wide renders (high_quality_mask 15); L alternates between 1 and 3 (mixed: 2 and 3), device cameras on half of them."""
    out = []
    for i, (fam, tile, exh) in enumerate(itertools.product(FAMILY, range(3), (False, True))):
        L = (1 if i % 2 else 3) if fam != "mixed" else (2 if i % 2 else 3)
        proj = {"persp": P, "ortho": O}.get(fam)
        table = [proj] * L if proj is not None else [P, O, P][:L]
        out.append((fam, table, tile, exh, i % 3 == 0, False))
    out += [("persp", [P], 1, False, False, True), ("persp", [P, P, P], 0, True, True, True), ("mixed", [O, P], 2, False, True, True)]
    return out


def _id(c):
    fam, table, tile, exh, cams, stereo = c
    return f"{fam}-L{len(table)}-t{TILE_H[tile]}-{'exh' if exh else 'chk'}{'-cams' if cams else ''}{'-stereo' if stereo else ''}"


def expected_kernels(c) -> set:
    fam, _, tile, exh, _, _ = c
    return {"render_params_kernel"} | {f"{FAMILY[fam]}<{m}, {'true' if exh else 'false'}, {TILE_H[tile]}>" for m in (0, 1)}


def _frame(cams, table, params, stereo, exh):
    plan = plan_of(cams, table, stereo=stereo, sample_exhaustively=exh, high_quality_mask=15, **params)
    return DC.frame(plan, table, stereo=stereo)


def _depth(f, rz, seed):
    lin = harness.frames(f.W, f.H, f.layers, seed=seed, reversed_z=rz)
    d, _ = harness.ingest(lin, "f32")
    return d if f.layers > 1 else d[0]


def _buffers(f, cams_bound):
    out = {}
    for l in range(f.layers):
        for bid in harness.buffer_ids(15):
            out[(bid, l)] = DC.buffer(f, bid, l, N.MEAO_DEPTH_RAW_F32) if cams_bound else f.buffer(bid, l)
    return out


def _same(a, b, tag):
    for k in a:
        x, y = a[k], b[k]
        view = {1: np.uint8, 2: np.uint16, 4: np.uint32}[x.dtype.itemsize]
        assert np.array_equal(x.view(view), y.view(view)), f"{tag}: buffer {k[0]} layer {k[1]}"


@pytest.mark.parametrize("case", _cases(), ids=_id)
def test_bound_frames_equal_host_parameter_frames(case):
    fam, table, tile, exh, with_cams, stereo = case
    W, H, rz = 64, 40, fam != "ortho"
    cams = [camera(W, H, 0.2 + 0.15 * l, 60.0 + 40.0 * l, 0.6 + 0.25 * l, p, rz, stereo) for l, p in enumerate(table)]
    host = [camera(W, H, 1.0, 500.0, 2.0, p, rz, stereo) for p in table]
    # the reference: host parameters DEV, no parameter binding; the bound frame: host parameters HOST, the buffer DEV
    ref = _frame(cams if not with_cams else host, table, dict(thickness_modifier=DEV[0], intensity=DEV[1]), stereo, exh)
    f = _frame(cams if not with_cams else host, table, HOST, stereo, exh)
    depth = _depth(f, rz, seed=len(table) + tile)
    cam_kw = lambda: dict(cams=rows(cams), cam_status=DC.new_status()) if with_cams else {}     # noqa: E731
    DP.run(ref, depth, ren_tile=tile, **cam_kw())
    slot = DP.new_slot(-1 / np.float32(HOST["thickness_modifier"]), HOST["intensity"])
    emu.ledger_reset()
    DP.run(f, depth, params=DEV, slot=slot, ren_tile=tile, **cam_kw())
    got = DP.ledger()
    assert set(got) == expected_kernels(case), sorted(set(got) ^ expected_kernels(case))
    assert got["render_params_kernel"][0] == 1
    assert sorted(v[0] for k, v in got.items() if k != "render_params_kernel") == [4, 4]      # levels 1-4, narrow and wide
    assert DP.status(slot) == [0, 0]
    _same(_buffers(f, with_cams), _buffers(ref, with_cams), _id(case))


def test_the_frames_name_every_kernel():
    named = set().union(*(expected_kernels(c) for c in _cases()))
    assert named == DP.kernels() and len(named) == 37, sorted(DP.kernels() - named)


@pytest.mark.parametrize("bad", [0.0, math.nan])
def test_an_invalid_block_reproduces_the_last_valid_frame(bad):
    W, H = 64, 40
    table = [P, O, P]
    cams = [camera(W, H, 0.3 + 0.1 * l, 80.0, 0.7, p, True) for l, p in enumerate(table)]
    f = _frame(cams, table, HOST, False, False)
    depth = _depth(f, True, seed=5)
    slot = DP.new_slot(-1 / np.float32(HOST["thickness_modifier"]), HOST["intensity"])
    DP.run(f, depth, params=(1.7, 0.8), slot=slot)
    valid = _buffers(f, False)
    f2 = _frame(cams, table, HOST, False, False)
    DP.run(f2, depth, params=(bad, 0.2), slot=slot)          # the same context slot: it still holds the valid block's values
    assert DP.status(slot) == [1, 1]
    _same(_buffers(f2, False), valid, f"invalid {bad}")
    # before any valid block the slot holds the host values written at bind time
    f3, f4 = _frame(cams, table, HOST, False, False), _frame(cams, table, HOST, False, False)
    slot = DP.new_slot(-1 / np.float32(HOST["thickness_modifier"]), HOST["intensity"])
    DP.run(f3, depth, params=(bad, 0.2), slot=slot)
    DP.run(f4, depth)
    _same(_buffers(f3, False), _buffers(f4, False), f"invalid {bad} at bind")
