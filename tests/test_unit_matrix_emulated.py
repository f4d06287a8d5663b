"""Every kernel of the satellite units (orthographic, mixed projections, batches, layer viewports, device camera tables), run in the CPU
emulator as the instantiation its slot stands for (tests/unit_matrix.py).

Each case resets the emulator's launch ledger, runs its frames, and must have launched exactly the units' kernels
unit_matrix.expected_kernels names.  Every frame must equal the oracle of each layer's camera bit for bit: the AO and every
intermediate, ids 1-21.  In the TMA-fed cases every render and upsample kernel the case launched must have issued TMA box loads, so
the interior tiles ran too.  In the tile-loop cases (MEAO_UPS_PERSIST_MIN_WAVES tiny) the final upsample's grid must be the one wave
of the persistent loop, not one CTA per tile: the emulator runs its CTAs in turn, so the first walks every tile of every layer and the
last re-arms the counters for the next of the three frames.  The matrix as a whole names all 140 kernels of the five units, feeds
every render and upsample kernel among them TMA boxes and runs every final upsample kernel through the tile loop.

The hostile cases run the same way on the depth of tests/hostile_cases.py, with the NaN rule documented there for the float buffers.
A case with tolerance overrides first checks that its plan lands on the side of upsample_fast_div_ok it was chosen for.  Their share
of the matrix must reach all 140 kernels, meet both sides of fast_div_ok in every unit's final upsample, and run hostile depth through
the tile loop of every unit and target form that has one."""
import numpy as np
import pytest

import harness
import hostile_cases as HC
import unit_matrix as um  # noqa: E402  (tests/ is on sys.path via conftest)
from emu import batch, emu, layer_views, mixed, ortho
from emu import device_cameras as DC
from emu.emu import Frame

LIBS = {"ortho": ortho, "mixed": mixed, "batch": batch, "views": layer_views, "camera": DC}
WAVE = 132 * 5          # the persistent upsample grid: one wave of MEAO_UPS_MINB CTAs on each of a plan-only context's 132 SMs
POISON = 0x5C


def _ledger() -> dict:
    """{kernel: (launches, TMA box loads, CTAs)} of every library's kernels since the last reset."""
    out = {}
    for m in LIBS.values():
        out.update(m.ledger())
    return out


def _render_plan(c):
    cams = c.cameras()
    plan = harness.context(cams[0], layers=c.layers, layer_cameras=cams if c.layers > 1 else None, sample_exhaustively=c.exhaustive,
                           high_quality_mask=c.hq, **dict(c.params))
    if c.unit == "mixed" or (c.unit == "camera" and c.layers > 1):
        plan.perLayerProjection = True
        plan.LateUpdate()
    return plan, cams


def _check_layers(c, cams, seen, get, ao=None, tag=""):
    """Each layer against its oracle: the debug buffers through get(bid, layer), and ao[l] when the AO is the caller's."""
    for l, cam in enumerate(cams):
        orc = um.oracle(c, cam)
        ref = orc.run(seen[l])
        if ao is not None:
            assert np.array_equal(ao[l], ref), f"{tag} layer {l}: the AO differs from the oracle"
        harness.compare_buffers(lambda bid: get(bid, l), orc, f"{tag} layer {l} ({'O' if cam.orthographic else 'P'})", c.buffer_ids(),
                                nan_equal=c.hostile)


def _check_fast_div_side(c, plan):
    """A tolerance case tests nothing unless its plan's final upsample levels fall on the side of fast_div_ok it was chosen for."""
    if c.fast_div_side is not None:
        assert HC.fast_div_sides(plan) == {c.fast_div_side}, f"{c.id}: the plan is not on the {c.fast_div_side} side of fast_div_ok"


# ---- orthographic, mixed and bound-camera frames ------------------------------------------------------------------------------------
def _render_unit(c):
    plan, cams = _render_plan(c)
    mod = LIBS[c.unit]
    if c.unit == "ortho":
        f = ortho.frame(plan, linear=c.linear)
    elif c.unit == "mixed":
        f = mixed.frame(plan, list(c.table), linear=c.linear)
        assert mixed.is_mixed(f)
    else:
        host = [type(cam)(cam.pixelWidth, cam.pixelHeight, nearClipPlane=1.0, farClipPlane=500.0, usesReversedZBuffer=c.reversed_z,
                          **(dict(orthographic=True, orthographicSize=2.0) if cam.orthographic else dict(fieldOfView=70.0))) for cam in cams]
        plan = harness.context(host[0], layers=c.layers, layer_cameras=host, high_quality_mask=c.hq, sample_exhaustively=c.exhaustive,
                               **dict(c.params))
        plan.perLayerProjection = True
        f = DC.frame(plan, list(c.table), linear=c.linear)
    _check_fast_div_side(c, plan)
    emu.ledger_reset()
    for n in range(c.frames):
        d, seen = um.depth(c, n)
        tag = f"{c.id} frame {n}"
        ao = None
        if c.unit == "camera":
            status = DC.new_status()
            rows = np.array([(k.nearClipPlane, k.farClipPlane, 1.0 / k.projection00) for k in cams], np.float32)
            DC.run(f, rows, status, d, fused=c.form == "fused", ren_tile=c.tile)
            assert list(status) == [0] * DC.STATUS_WORDS
        elif c.form == "arrays":
            ao = mod.run_arrays(f, d, "layered" if c.layers > 1 else "2d", ren_tile=c.tile)
        else:
            mod.run(f, d if c.layers > 1 else d[0], fused=c.form == "fused", ren_tile=c.tile)
        _check_layers(c, cams, seen, lambda bid, l: mod.buffer(f, bid, l, um.KIND_CODE[c.kind]), ao, tag)


# ---- batches ------------------------------------------------------------------------------------------------------------------------
def _batch_arrays_frame(c, f, cams, n):
    W, H = c.size
    depth, seen = um.depth(c, n)
    fill = np.float32(np.nan) if depth.dtype == np.float32 else 0
    ds, aos, dsh, ash = [], [], [], []
    for l, (ext, dshape, ashape) in enumerate(um.batch_array_layout(c)):
        d = np.full(ext, fill, depth.dtype)
        if depth.dtype == np.float32 and ext != (H, W):
            d[H:] = np.inf
        d[:H, :W] = depth[l]
        ds.append(d)
        aos.append(np.full(ext, POISON, np.uint8))
        dsh.append(dshape)
        ash.append(ashape)
    n0 = f.surface_accesses()
    batch.run_arrays_batch(f, ds, aos, dsh, ash)
    assert f.surface_accesses() - n0 == 2 * c.layers * W * H, "a surface access outside W x H, or one missing"
    for l, a in enumerate(aos):
        assert (a[H:] == POISON).all() and (a[:, W:] == POISON).all(), f"{c.id}: layer {l} stored outside W x H"
    return seen, [a[:H, :W] for a in aos]


def _batch_pointers_frame(c, f, cams, n):
    W, H = c.size
    depth, seen = um.depth(c, n)
    es = depth.itemsize
    ds, abufs, aviews, layout = [], [], [], um.batch_pointer_layout(c)
    for l, (drow, doff, arow, aoff) in enumerate(layout):
        buf = np.zeros(H * drow + doff, depth.dtype)
        for r in range(H):
            buf[doff + r * drow:][:W] = depth[l, r]
        ds.append(emu._aligned(buf)[doff:])
        a = emu._aligned(np.full(H * arow + aoff + 7, POISON, np.uint8))
        abufs.append(a)
        aviews.append(a[aoff:])
    batch.run_pointers_batch(f, ds, [d * es for d, _, _, _ in layout], aviews, [a for _, _, a, _ in layout])
    ao = []
    for l, (_, _, arow, aoff) in enumerate(layout):
        written = np.zeros(abufs[l].shape, bool)
        for r in range(H):
            written[aoff + r * arow:][:W] = True
        assert (abufs[l][~written] == POISON).all(), f"{c.id}: layer {l} stored outside its view"
        ao.append(np.stack([aviews[l][r * arow:][:W] for r in range(H)]))
    return seen, ao


# ---- layer viewports ----------------------------------------------------------------------------------------------------------------
def _poisoned(shape, dtype):
    """NaN, +inf, -inf, 0 (float32) or 0, 65535 (D16 codes) in every texel no layer reads."""
    n = int(np.prod(shape))
    vals = np.array([np.nan, np.inf, -np.inf, 0.0], np.float32) if np.dtype(dtype) == np.float32 else np.array([0, 65535], np.uint16)
    return np.resize(vals, n).reshape(shape).astype(dtype)


def _views_arrays_frame(c, f, cams, n):
    W, H = c.size
    depth, seen = um.depth(c, n)
    table, dshape, dext, ashape, aext = um.view_arrays_layout(c)
    darr = _poisoned(dext, depth.dtype)
    aarr = np.full(aext, POISON, np.uint8)
    written = np.zeros(aext, bool)
    for l, (dx, dy, dsl, ax, ay, asl) in enumerate(table):
        darr[dsl, dy:dy + H, dx:dx + W] = depth[l]
        written[asl, ay:ay + H, ax:ax + W] = True
    n0 = f.surface_accesses()
    layer_views.run_arrays_views(f, darr, aarr, table, dshape, ashape)
    assert f.surface_accesses() - n0 == 2 * c.layers * W * H, "a surface access outside the rectangles, or one missing"
    assert (aarr[~written] == POISON).all(), f"{c.id}: a store outside the AO rectangles"
    return seen, [aarr[asl, ay:ay + H, ax:ax + W] for _, _, _, ax, ay, asl in table]


def _views_pitched_frame(c, f, cams, n):
    W, H = c.size
    depth, seen = um.depth(c, n)
    es = depth.itemsize
    table, drow, dsl, arow, asl, slices = um.view_pitched_layout(c)
    dbuf = emu._aligned(_poisoned((slices * dsl,), depth.dtype))
    abuf = emu._aligned(np.full(slices * asl, POISON, np.uint8))
    written = np.zeros(abuf.shape, bool)
    for l, (dx, dy, ds, ax, ay, as_) in enumerate(table):
        for r in range(H):
            o = ds * dsl + (dy + r) * drow + dx
            dbuf[o:o + W] = depth[l, r]
            o = as_ * asl + (ay + r) * arow + ax
            written[o:o + W] = True
    layer_views.run_pitched_views(f, dbuf, (drow * es, dsl * es), abuf, (arow, asl), table)
    assert (abuf[~written] == POISON).all(), f"{c.id}: a store outside the AO rectangles"
    return seen, [np.stack([abuf[as_ * asl + (ay + r) * arow + ax:][:W] for r in range(H)]) for _, _, _, ax, ay, as_ in table]


TARGET_FRAMES = {("batch", "arrays"): _batch_arrays_frame, ("batch", "pointers"): _batch_pointers_frame,
                 ("views", "arrays"): _views_arrays_frame, ("views", "pitched"): _views_pitched_frame}


def _target_unit(c):
    W, H = c.size
    cams = c.cameras()
    plan = harness.context(W, H, layers=c.layers, layer_cameras=cams, reversed_z=c.reversed_z, high_quality_mask=c.hq, **dict(c.params))
    _check_fast_div_side(c, plan)
    f = Frame(plan, linear=c.linear)
    emu.ledger_reset()
    for n in range(c.frames):
        seen, ao = TARGET_FRAMES[(c.unit, c.form)](c, f, cams, n)
        _check_layers(c, cams, seen, lambda bid, l: f.buffer(bid, l), ao, f"{c.id} frame {n}")


@pytest.mark.parametrize("case", um.CASES, ids=lambda c: c.id)
def test_case_launches_its_kernels_and_matches_the_oracle(case, monkeypatch):
    c = case
    if c.persist:
        monkeypatch.setenv("MEAO_UPS_PERSIST_MIN_WAVES", "0.0001")
    (_target_unit if c.unit in ("batch", "views") else _render_unit)(c)
    ledger = _ledger()
    want = um.expected_kernels(c)
    assert set(ledger) == want, f"{c.id}: launched {sorted(set(ledger) - want)} unexpectedly, never launched {sorted(want - set(ledger))}"
    if c.tma_fed:
        base = {k: v for k, v in emu.kernel_ledger().items() if not k.startswith("0x")}
        everything = {**{k: v[:2] for k, v in ledger.items()}, **base}
        untouched = [k for k, (_, tma) in everything.items() if k.startswith(("render_ao", "blur_upsample")) and tma == 0]
        assert not untouched, f"{c.id}: no TMA box loads in {untouched}"
    if any(k.startswith("blur_upsample") for k in want):
        launches, _, ctas = ledger[um.upsample_kernel(c)]
        assert launches == c.frames, f"{c.id}: {launches} final upsamples in {c.frames} frames"
        grid = WAVE if c.persist else um.loop_tiles(c)         # the tile loop's one wave, or one CTA per tile
        assert ctas == launches * grid, f"{c.id}: final upsample grids of {ctas // launches} CTAs, {grid} expected"


# ---- the matrix as a whole ----------------------------------------------------------------------------------------------------------
def _named() -> set:
    return set().union(*(um.expected_kernels(c) for c in um.CASES))


def test_the_matrix_names_every_kernel_of_the_five_units():
    built = set().union(*(m.kernels() for m in LIBS.values()))
    named = _named()
    assert named == built, f"never launched: {sorted(built - named)}; not built: {sorted(named - built)}"
    assert {u: len(m.kernels()) for u, m in LIBS.items()} == {"ortho": 64, "mixed": 34, "batch": 20, "views": 20, "camera": 2}
    assert len(built) == 140


def test_every_render_and_upsample_kernel_is_launched_by_a_tma_fed_case():
    fed = set().union(*(um.expected_kernels(c) for c in um.CASES if c.tma_fed))
    need = {k for k in _named() if k.startswith(("render_ao", "blur_upsample"))}
    assert len(need) == 70 and need <= fed, sorted(need - fed)


def test_every_final_upsample_kernel_runs_the_tile_loop():
    looped = {um.upsample_kernel(c) for c in um.CASES if c.persist}
    need = {k for k in _named() if k.startswith("blur_upsample")}
    assert len(need) == 34 and looped == need, sorted(need - looped)
    for c in um.CASES:
        if c.persist:
            assert um.loop_tiles(c) != WAVE and (c.layers >= 2 or c.unit == "ortho"), c.id


def test_the_libraries_kernels_have_distinct_offsets():
    """The ledger keys a kernel by its offset in its own library: no two libraries may have a kernel at the same offset, or a launch
    would be credited to both."""
    tables = [set(m._kernel_symbols()) for m in LIBS.values()] + [set(emu._kernel_symbols())]
    assert sum(map(len, tables)) == len(set().union(*tables))


# ---- the hostile cases as a whole ---------------------------------------------------------------------------------------------------
def test_the_hostile_cases_name_every_kernel_of_the_five_units():
    hostile = set().union(*(um.expected_kernels(c) for c in um.CASES if c.hostile))
    assert hostile == _named() and len(hostile) == 140, sorted(_named() - hostile)


def test_every_units_final_upsample_meets_both_sides_of_fast_div_ok():
    sides = {}
    for c in um.CASES:
        if c.unit != "camera" and any(k.startswith("blur_upsample") for k in um.expected_kernels(c)):
            plan = harness.context(*c.size, reversed_z=c.reversed_z, high_quality_mask=c.hq, **dict(c.params))
            got = HC.fast_div_sides(plan)
            assert c.fast_div_side is None or got == {c.fast_div_side}, c.id
            sides.setdefault(c.unit, set()).update(got)
            if c.fast_div_side is not None:
                sides.setdefault((c.unit, "premin"), set()).update(got if c.hq & 1 else ())
    for u in ("ortho", "mixed", "batch", "views"):
        assert sides[u] == {True, False}, f"{u}: the final upsample meets only the {sides[u]} side of fast_div_ok"
        assert sides[(u, "premin")] == {True, False}, f"{u}: no premin tolerance case on each side of fast_div_ok"


def test_every_unit_and_target_form_with_a_tile_loop_has_a_hostile_loop_case():
    loops = {(c.unit, c.form) for c in um.CASES if c.persist}
    hostile = {(c.unit, c.form, c.kind) for c in um.CASES if c.persist and c.hostile}
    for unit, form in loops:
        assert {(unit, form, k) for k in ("f32", "d16")} <= hostile, f"{unit} {form}: no hostile tile-loop case in f32 and in D16"
