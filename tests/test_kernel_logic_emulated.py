"""CPU tests of the CUDA KERNEL SOURCES: miniengineao_b200/csrc/*.cu compiled by g++ for the host (tests/emu, -DMEAO_EMULATE,
one fiber per CUDA thread, fibers switch at __syncthreads) and run against the oracle, bit for bit, without a GPU.

What this proves: the kernels' logic -- tiling, aprons, border / padding handling, operation order, packed-lane bookkeeping,
the variants' plumbing -- is the reference's arithmetic.  What it cannot prove: anything about the real
hardware path (TMA boxes, MUFU.RCP + refinement, memory model); that is what tests/test_parity_gpu.py does on the H100.
TMA box loads are emulated as synchronous copies with zero fill, so interior tiles run the same TMA branch as on the GPU
(use_tma=True, the default) and the gather branch can be forced everywhere (use_tma=False = MEAO_DISABLE_TMA=1).
The emulator is test infrastructure: libmeao.so never contains it and still has no CPU path (test_abi.py).
"""
import numpy as np
import pytest

from miniengineao_b200 import synth
from oracle import oracle as O

import harness
from emu.emu import Frame, composite, composite_debug  # noqa: E402  (tests/ is on sys.path via conftest)


def _run(W, H, seed=1, depth=None, use_tma=True, **kw):
    okw = {k: v for k, v in kw.items()}
    orc = harness.oracle(W, H, **okw)
    if depth is None:
        depth = synth.lin01_to_raw(synth.random_depth(W, H, seed=seed), reversed_z=kw.get("reversed_z", True))
    ref = orc.run(depth)
    f = Frame(harness.context(W, H, **kw), use_tma=use_tma)
    n0 = f.tma_box_loads()
    got = f.run(depth)
    f.tma_loads_in_run = f.tma_box_loads() - n0
    assert int((got != ref).sum()) == 0, (W, H, kw)
    harness.compare_buffers(f.buffer, orc, f"{W}x{H} {kw}", harness.buffer_ids(kw.get("high_quality_mask", 0)))
    return f, orc


@pytest.mark.parametrize("W,H", [(256, 256), (64, 64), (16, 16), (1, 1), (3, 5), (130, 70), (250, 131), (321, 203), (37, 300), (300, 37)])
def test_reference_path_all_buffers(W, H):
    _run(W, H, seed=W * 7 + H, intensity=1.1)


@pytest.mark.parametrize("kw", [
    dict(intensity=0.0), dict(intensity=2.0), dict(thickness_modifier=10.0), dict(blur_tolerance=-1.0), dict(blur_tolerance=-8.0),
    dict(upsample_tolerance=-1.0), dict(upsample_tolerance=-6.0, noise_filter_tolerance=-8.0), dict(reversed_z=False),
    dict(noise_filter_tolerance=-3.0, blur_tolerance=-3.0, upsample_tolerance=-4.0, thickness_modifier=4.0, intensity=0.7),
])
def test_parameter_sweep(kw):
    _run(194, 110, seed=11, **kw)


@pytest.mark.parametrize("kw", [
    dict(sample_exhaustively=True), dict(high_quality_mask=15), dict(high_quality_mask=0b0110, sample_exhaustively=True, intensity=1.3),
    dict(high_quality_mask=0b1001, reversed_z=False),
])
@pytest.mark.parametrize("W,H", [(130, 70), (201, 155)])
def test_shader_variants(W, H, kw):
    _run(W, H, seed=5, **kw)


def test_sky_pixels_take_the_ieee_fallbacks():
    """Raw depth 0 -> 1e5 -> inf in f16 -> NaN in the sampler; grouped range tests must fall back for the whole group."""
    W, H = 200, 120
    depth = synth.lin01_to_raw(synth.random_depth(W, H, seed=5))
    depth[20:60, 30:90] = 0.0
    depth[::17, ::13] = 0.0
    _run(W, H, depth=depth)
    _run(W, H, depth=depth, high_quality_mask=15, sample_exhaustively=True)


@pytest.mark.parametrize("use_tma", [True, False])
def test_corridor_640x360(use_tma):
    """Large enough for interior tiles at levels 1-2 of the render and 0-1 of the upsample (the TMA branch)."""
    f, _ = _run(640, 360, depth=synth.lin01_to_raw(synth.corridor(640, 360)), intensity=1.1, use_tma=use_tma)
    # interior tiles: render L1 3 x 4 + L2 1 x 1, upsample L1->L0 8 x 9 (two boxes each) + L2->L1 3 x 3 ...
    assert (f.tma_loads_in_run > 100) if use_tma else (f.tma_loads_in_run == 0), f.tma_loads_in_run


@pytest.mark.parametrize("use_tma", [True, False])
def test_variants_with_interior_tiles(use_tma):
    """Wide render (80 x 48 box), premin upsample (second AO box) and exhaustive sampling on TMA-fed tiles; sky patch inside."""
    W, H = 768, 400
    depth = synth.lin01_to_raw(synth.random_depth(W, H, seed=13))
    depth[150:230, 300:500] = 0.0
    f, _ = _run(W, H, depth=depth, use_tma=use_tma, high_quality_mask=15, sample_exhaustively=True, intensity=1.2)
    assert (f.tma_loads_in_run > 200) if use_tma else (f.tma_loads_in_run == 0), f.tma_loads_in_run


def test_unaligned_tma_start_is_refused():
    """DESIGN.md 2.4: on the GPU a box whose start coordinate is not 16-byte aligned raises 'illegal instruction'; the emulated
    TMA refuses the same thing, so a tile-origin change that breaks the rule fails here before it reaches the GPU."""
    import ctypes as C
    import subprocess
    import sys
    code = ("import sys; sys.path.insert(0, 'tests'); import ctypes as C; from emu.emu import lib; l = lib();"
            "l.emu_selfcheck_unaligned_tma.restype = C.c_int; l.emu_selfcheck_unaligned_tma()")
    import os
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode != 0 and "16-byte aligned" in r.stderr, (r.returncode, r.stderr[-300:])


def test_linear_and_native_depth_ingest():
    W, H = 250, 131
    lin = synth.random_depth(W, H, seed=9)
    orc = harness.oracle(W, H, linear=True, threads=1)
    ref = orc.run(lin)
    f = Frame(harness.context(W, H), linear=True)
    assert np.array_equal(f.run(lin), ref)
    harness.compare_buffers(f.buffer, orc, "linear ingest", harness.buffer_ids())
    raw = synth.lin01_to_raw(lin)
    assert np.rint(raw.astype(np.float64) * 65535).min() >= 1           # no code 0: the frame has no sky
    for kind in ("d16", "d24s8"):
        words, as_float = harness.ingest(raw, kind)
        orc = harness.oracle(W, H, threads=1)
        ref = orc.run(as_float)
        f = Frame(harness.context(W, H))
        assert np.array_equal(f.run(words), ref), kind
        harness.compare_buffers(f.buffer, orc, kind, harness.buffer_ids())


def test_debug_views():
    W, H = 130, 70
    f, orc = _run(W, H, seed=4, high_quality_mask=0b0101)
    for bid in harness.buffer_ids(high_quality_mask=0b0101):
        assert np.array_equal(f.debug_view(bid), orc.debug_view(bid)), bid


def test_composite_passes():
    rng = np.random.default_rng(0)
    ao = rng.integers(0, 256, size=(45, 67), dtype=np.uint8)
    c8 = rng.integers(0, 256, size=(45, 67, 4), dtype=np.uint8)
    c16 = (rng.uniform(0, 4, size=(45, 67, 4)) ** 3).astype(np.float16)
    for col in (c8, c16):
        assert np.array_equal(composite(ao, col, rgb=True, alpha=True, one_minus=False).view(np.uint8), O.composite_framebuffer(ao, col).view(np.uint8))
        g0, g3 = O.composite_gbuffer(ao, c8, col)
        assert np.array_equal(composite(ao, c8, rgb=False, alpha=True, one_minus=True), g0)
        assert np.array_equal(composite(ao, col, rgb=True, alpha=False, one_minus=True).view(np.uint8), g3.view(np.uint8))


def test_debug_composite_pass3():
    """Blit.shader pass 3 (AO.cs:826-829): target = view.rrrr, on sizes that are and are not multiples of the 4-pixel step."""
    rng = np.random.default_rng(1)
    for shape in ((45, 67), (1, 1), (3, 5), (64, 64)):
        v = rng.integers(0, 256, size=shape, dtype=np.uint8)
        for like in (np.zeros(1, np.uint8), np.zeros(1, np.float16)):
            assert np.array_equal(composite_debug(v, like).view(np.uint8), O.composite_debug(v, like).view(np.uint8)), (shape, like.dtype)


def test_odd_size_and_premin_sky_frames():
    """An odd-sized frame at intensity 1.2, and a frame with a sky patch and the premin upsample on every level."""
    _run(161, 93, seed=21, intensity=1.2)
    depth = synth.lin01_to_raw(synth.random_depth(120, 80, seed=2))
    depth[10:30, 15:60] = 0.0
    _run(120, 80, depth=depth, high_quality_mask=15)


# ---- round 2: render tile-height variants, single-scale plan, native neighbour exchange ---------------------------------------
@pytest.mark.parametrize("tile", [0, 1, 2])
@pytest.mark.parametrize("use_tma", [True, False])
def test_render_tile_height_variants(tile, use_tma):
    """render_ao_kernel<MODE, EXH, TH> for TH = 32 / 16 / 8 (kernels.h kRenderTileHs): the coarse levels take the small tiles on the
    GPU (meao_api.cu render_tile_variant); every variant must give the same bits on interior (TMA) and border (gather) tiles."""
    W, H = 700, 420
    depth = synth.lin01_to_raw(synth.random_depth(W, H, seed=31))
    depth[100:140, 200:330] = 0.0
    orc = harness.oracle(W, H, intensity=1.1, high_quality_mask=0b0011)
    ref = orc.run(depth)
    f = Frame(harness.context(W, H, intensity=1.1, high_quality_mask=0b0011), use_tma=use_tma, render_tile=tile)
    n0 = f.tma_box_loads()
    assert np.array_equal(f.run(depth), ref)
    harness.compare_buffers(f.buffer, orc, f"tile variant {tile}", harness.buffer_ids(0b0011))
    assert (f.tma_box_loads() - n0 > 50) if use_tma else (f.tma_box_loads() == n0)


@pytest.mark.parametrize("W,H", [(256, 256), (130, 70), (321, 203), (3, 5)])
def test_single_scale_plan(W, H):
    """BASELINE.json configs[0]: Downsample -> Render level 1 -> final-style Upsample on Occlusion1 (MeaoVariants.single_scale)."""
    lin = synth.flat_sphere(W, H) if (W, H) == (256, 256) else synth.random_depth(W, H, seed=W)
    depth = synth.lin01_to_raw(lin)
    orc = harness.oracle(W, H, intensity=1.1, single_scale=True)
    ref = orc.run(depth)
    plan = harness.context(W, H, intensity=1.1)
    plan.singleScale = True
    f = Frame(plan)
    assert np.array_equal(f.run(depth), ref)
    for bid in (1, 2, 3, 4, 5, 10, 17):
        got = f.buffer(bid)
        want = orc.codes(bid) if got.dtype == np.uint8 else orc.buffer(bid)
        with np.errstate(over="ignore"):
            assert np.array_equal(got, want.astype(got.dtype)), bid
    assert plan.kernels_per_frame == 3


@pytest.mark.parametrize("W,H,nb,single_scale", [(200, 528, 2, False), (130, 1296, 3, False), (200, 528, 2, True)],
                         ids=["200-528-2", "130-1296-3", "200-528-2-single_scale"])
def test_native_exchange_kernel_bands_equal_whole_frame(W, H, nb, single_scale):
    """band_exchange_kernel (peer stores + epoch flags): each band pushes its border rows of LowDepth1..4 straight into the
    neighbours' buffers (NaN-poisoned beforehand); the union of the bands must equal the whole-frame oracle bit for bit.
    The fiber emulator runs one grid at a time, so the flags a CONCURRENT neighbour would have raised are preset for the band
    that runs first; every later band finds them raised by the kernels that already ran.  single_scale: phase b is render 1 and
    the final-style upsample, as in libmeao's frame schedule."""
    depth = synth.lin01_to_raw(synth.random_depth(W, H, seed=3))
    okw = dict(intensity=1.1, single_scale=single_scale)
    ref = harness.oracle(W, H, **okw).run(depth)
    for frame_no in (1, 2):                                      # two epochs through the same flags
        cuts, frames = (harness.band_frames(W, H, nb, intensity=1.1, single_scale=single_scale)) if frame_no == 1 else (cuts, frames)
        d = depth if frame_no == 1 else depth[:, ::-1].copy()
        want = ref if frame_no == 1 else harness.oracle(W, H, **okw).run(d)
        for i, f in enumerate(frames):
            if frame_no == 2:
                f.poison_low()
        for i, f in enumerate(frames):
            f.band_phase_a(d[cuts[i]:cuts[i + 1]])
        for i, f in enumerate(frames):
            up = frames[i - 1] if i > 0 else None
            down = frames[i + 1] if i + 1 < nb else None
            fl = f.flags()
            # what the not-yet-run neighbour below WOULD have written by now: its announce (ack) and its rows (ready)
            f.flags(set_ready_ack=(fl["ready"][0], frame_no if down is not None else 0, fl["ack"][0], frame_no if down is not None else 0))
            assert f.exchange(up, down) == 0
            after = f.flags()
            assert after["epoch"] == frame_no + 1 and after["done"] == 0 and after["error"] == 0 and after["host_error"] == 0
        for i, f in enumerate(frames):
            if i + 1 < nb:                                       # the rows really came from the neighbour, not from the preset flags
                assert frames[i + 1].flags()["ready"][0] == frame_no and frames[i + 1].flags()["ack"][0] == frame_no
            got = f.band_phase_b()
            assert np.array_equal(got, want[cuts[i]:cuts[i + 1]]), (frame_no, i)


def test_native_exchange_times_out_instead_of_hanging():
    """A neighbour that never arrives: the kernel gives up after the time-out, sets the sticky error (1 = no ack, 2 = no rows),
    mirrors it to the host word, and later exchanges return immediately."""
    cuts, frames = harness.band_frames(200, 528, 2, intensity=1.1)
    depth = synth.lin01_to_raw(synth.random_depth(200, 528, seed=3))
    a, b = frames
    a.band_phase_a(depth[cuts[0]:cuts[1]])
    assert a.exchange(None, b, timeout_polls=50) == 1            # b never announced: no ack
    st = a.flags()
    assert st["error"] == 1 and st["host_error"] == 1 and st["epoch"] == 2 and st["done"] == 0
    # nothing was written into the neighbour (its LowDepth rows are still poisoned), but it was told we are at epoch 1
    assert b.flags()["ack"][0] == 1 and b.flags()["ready"][0] == 1
    assert np.isnan(b.buffer(2)).all()
    b.band_phase_a(depth[cuts[1]:cuts[2]])
    b.flags(set_ready_ack=(0, 0, 1, 0))                          # ack from a, but a's rows "never arrive"
    assert b.exchange(a, None, timeout_polls=50) == 2
    assert b.flags()["host_error"] == 2


def test_tolerances_outside_the_proven_range_take_the_ieee_path():
    """fast_div_ok = 0 (upsample tolerance 10^-17 < 2^-55): the whole upsample runs upsample8_slow."""
    _run(161, 93, seed=21, upsample_tolerance=-17.0, noise_filter_tolerance=-8.0, intensity=1.2)


@pytest.mark.parametrize("use_tma", [True, False])
def test_persistent_tile_loop_forced_on_every_level(use_tma, monkeypatch):
    """The tile loop of blur_upsample (atomic tile cursor, next tile's boxes staged into the other buffer pair, per-barrier wait parity,
    double-buffered lo_depth, counters re-armed by the last CTA) is used on the GPU only when a launch has >= 2 tiles per CTA slot;
    MEAO_UPS_PERSIST_MIN_WAVES forces it everywhere.  In the fiber emulator the first CTA then walks ALL tiles of a level, interior
    and border tiles mixed, and the second frame must find the counters re-armed."""
    monkeypatch.setenv("MEAO_UPS_PERSIST_MIN_WAVES", "0.0001")
    W, H = 640, 360
    depth = synth.lin01_to_raw(synth.corridor(W, H))
    depth[100:130, 200:300] = 0.0                                   # sky: the out-of-line IEEE path inside the loop
    orc = harness.oracle(W, H, intensity=1.1, high_quality_mask=0b0101)
    ref = orc.run(depth)
    f = Frame(harness.context(W, H, intensity=1.1, high_quality_mask=0b0101), use_tma=use_tma)
    for frame in range(2):
        assert np.array_equal(f.run(depth), ref), frame
    harness.compare_buffers(f.buffer, orc, "tile loop", harness.buffer_ids(0b0101))
