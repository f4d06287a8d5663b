"""CPU tests of CUDA-array viewports (meao_render_arrays_at): the frame read from a W x H rectangle of a larger depth array and written
into one of a larger AO array, at any origin inside each.

The array kernel sources run in the fiber emulator (tests/emu/frame_views.cpp frame_run_arrays_at, linked against the emulator the
other CPU tests use) on emulated arrays whose extent is the whole array, so a texel outside the array is dropped rather than aliased.  Each case checks that the AO inside the AO viewport is
bit-identical to the oracle run on the cropped depth, that every AO byte outside it keeps its sentinel, that the depth texels outside
the depth viewport (NaN, +-inf and 0 in a float array; 0 and 65535 in a D16 one) change nothing, and that the frame makes exactly one
surface access per depth texel and per AO byte of its viewports.  Also here: the launch ledger of a viewport frame, the register
budget of the seven array kernels, and the plan-only contract of the two new entry points."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from miniengineao_b200 import _native as N

import harness
from emu import emu, views  # noqa: E402  (tests/ is on sys.path via conftest)
from emu.emu import Frame  # noqa: E402

SENTINEL = 0xA5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _poisoned(shape, dtype):
    """An array of `shape` whose every texel is poison: NaN, +inf, -inf and 0 in turn (float32), 0 and 65535 (D16 codes)."""
    n = int(np.prod(shape))
    if np.dtype(dtype) == np.float32:
        vals = np.array([np.nan, np.inf, -np.inf, 0.0], np.float32)
    else:
        vals = np.array([0, 65535], np.uint16)
    return np.resize(vals, n).reshape(shape)


def _case_depth(W, H, L, kind, seed):
    """(the frame's depth in the array's format, the float32 the oracle sees, linear?) of L layers"""
    lin = harness.contrasting_layers(W, H, L, seed=seed)
    if kind == "linear_f32":
        return lin, lin, True
    r = harness.raw(lin)
    if kind == "d16":
        codes, as_float = harness.ingest(r, "d16")
        return codes, as_float, False
    return r, r, False


def _viewport_frame(W, H, L, kind, *, shape, ao_shape=None, depth_ext, depth_origin, ao_ext, ao_origin, seed=0, **kw):
    """One viewport frame; returns the Frame and the whole AO array after it."""
    depth, as_float, linear = _case_depth(W, H, L, kind, seed)
    (dw, dh), (dx, dy), (aw, ah), (ax, ay) = depth_ext, depth_origin, ao_ext, ao_origin
    assert dx + W <= dw and dy + H <= dh and ax + W <= aw and ay + H <= ah
    darr = _poisoned((L, dh, dw), depth.dtype)
    darr[:, dy:dy + H, dx:dx + W] = depth
    aarr = np.full((L, ah, aw), SENTINEL, np.uint8)
    f = Frame(harness.context(W, H, layers=L, **kw), linear=linear)
    n0 = f.surface_accesses()
    views.run_arrays_at(f, darr, (dx, dy), aarr, (ax, ay), shape, ao_shape)
    assert f.surface_accesses() - n0 == 2 * L * W * H, "a surface access outside the viewports, or one missing"
    tag = f"{W}x{H} L={L} {kind} {shape} depth {depth_ext}@{depth_origin} ao {ao_ext}@{ao_origin} {kw}"
    outside = np.ones(aarr.shape, bool)
    outside[:, ay:ay + H, ax:ax + W] = False
    assert (aarr[outside] == SENTINEL).all(), f"{tag}: a store outside the AO viewport"
    for l in range(L):
        ref = harness.oracle(W, H, linear=linear, **kw).run(as_float[l])
        assert np.array_equal(aarr[l, ay:ay + H, ax:ax + W], ref), f"{tag}: layer {l} differs from the oracle"
    return f, aarr


def _ext(shape, w, h):
    """an array extent of at least w x h; square for a cube map, whose faces are"""
    return (max(w, h),) * 2 if shape == "cube" else (w, h)


# (W, H, layers, shape): ragged widths, one, two and six (cube-map) layers
CASES = [(83, 61, 1, "2d"), (130, 70, 2, "layered"), (61, 61, 6, "cube")]


@pytest.mark.parametrize("hq", [0, 1])
@pytest.mark.parametrize("kind", ["raw_f32", "linear_f32", "d16"])
@pytest.mark.parametrize("W,H,L,shape", CASES)
def test_viewport_matches_the_oracle_of_the_cropped_depth(W, H, L, shape, kind, hq):
    """Non-zero origins in arrays larger than the frame, of different extents for the depth and the AO; high_quality_mask bit 0
    selects the premin final level."""
    _viewport_frame(W, H, L, kind, shape=shape, depth_ext=_ext(shape, W + 37, H + 19), depth_origin=(29, 11),
                    ao_ext=_ext(shape, W + 9, H + 40), ao_origin=(5, 33), seed=W + L, high_quality_mask=hq)


@pytest.mark.parametrize("W,H,L,shape", CASES)
def test_exact_depth_copy_into_a_max_size_ao_target(W, H, L, shape):
    """The depth at (0, 0) of an array of exactly W x H, the AO into the bottom-right corner of a larger one."""
    _viewport_frame(W, H, L, "raw_f32", shape=shape, depth_ext=(W, H), depth_origin=(0, 0), ao_ext=_ext(shape, W + 24, H + 16),
                    ao_origin=(24, 16), intensity=1.1)


def test_viewports_flush_against_every_edge():
    """Viewports touching the far right and bottom edges of the depth array, and the top-left corner of the AO array."""
    W, H = 83, 61
    _viewport_frame(W, H, 1, "d16", shape="2d", depth_ext=(W + 13, H + 7), depth_origin=(13, 7), ao_ext=(W + 13, H + 7),
                    ao_origin=(0, 0))


def test_mixed_shapes_cube_depth_into_a_layered_ao():
    W = 50
    _viewport_frame(W, W, 6, "raw_f32", shape="cube", ao_shape="layered", depth_ext=(W + 6, W + 6), depth_origin=(3, 6),
                    ao_ext=(W + 30, W + 2), ao_origin=(30, 1), high_quality_mask=1)


def test_viewport_at_zero_origins_is_the_array_frame():
    """At (0, 0) in arrays of exactly W x H a viewport frame is the array frame, byte for byte."""
    W, H, L = 130, 70, 2
    depth, _, _ = _case_depth(W, H, L, "raw_f32", seed=4)
    f = Frame(harness.context(W, H, layers=L))
    ref = f.run_arrays(depth, "layered")
    ao = np.full((L, H, W), SENTINEL, np.uint8)
    views.run_arrays_at(f, np.ascontiguousarray(depth), (0, 0), ao, (0, 0), "layered")
    assert np.array_equal(ao, ref)


@pytest.mark.parametrize("hq", [0, 1])
def test_kernel_ledger_equals_the_array_frames(hq):
    """A viewport frame launches the kernels of an array frame of the same case, as often, with as many TMA box loads."""
    W, H, L = 640, 360, 2
    depth, _, _ = _case_depth(W, H, L, "raw_f32", seed=7)
    f = Frame(harness.context(W, H, layers=L, high_quality_mask=hq))
    emu.ledger_reset()
    f.run_arrays(depth, "layered")
    plain = emu.kernel_ledger()
    darr = _poisoned((L, H + 40, W + 64), np.float32)
    darr[:, 40:, 64:] = depth
    ao = np.full((L, H + 8, W + 8), SENTINEL, np.uint8)
    emu.ledger_reset()
    views.run_arrays_at(f, darr, (64, 40), ao, (8, 8), "layered")
    assert emu.kernel_ledger() == plain
    assert any(k.startswith("prepare_depth_array_kernel") for k in plain) and any("_array_kernel" in k and "upsample" in k for k in plain)


# ---- the register budget of the seven array kernels (DESIGN.md 2.7) ---------------------------------------------------------------
# kernel name -> (instantiations, most registers, most spill-store bytes): the counts of the array kernels before viewports, where the
# premin twin spilled 12 bytes
BUDGET = {"prepare_depth_array_kernel": (5, 40, 0), "blur_upsample_array_kernel": (1, 48, 0), "blur_upsample_premin_array_kernel": (1, 48, 12)}


def test_array_kernels_keep_their_register_budget(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    seen = {}
    for tu in ("prepare_depth_array.cu", "blur_upsample_array.cu"):
        p = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false", "-Xptxas", "-v", "-cubin",
                            "-o", str(tmp_path / (tu + ".cubin")), os.path.join(ROOT, "miniengineao_b200", "csrc", tu)],
                           capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-2000:]
        cur = None
        for line in (p.stdout + p.stderr).splitlines():
            m = re.search(r"Compiling entry function '\w*?(%s)I" % "|".join(BUDGET), line)
            if m:
                cur = m.group(1)
                seen.setdefault(cur, []).append([None, None])
                continue
            if re.search(r"Function properties for \w*upsample8_slow", line):
                cur = None                  # the out-of-line slow path's own figures
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and cur:
                seen[cur][-1][1] = int(m.group(1))
            m = re.search(r"Used (\d+) registers", line)
            if m and cur:
                seen[cur][-1][0] = int(m.group(1))
    assert set(seen) == set(BUDGET)
    for name, (n, regs, spill) in BUDGET.items():
        assert len(seen[name]) == n, (name, seen[name])
        assert all(r <= regs and s <= spill for r, s in seen[name]), (name, seen[name])


# ---- plan-only contract ------------------------------------------------------------------------------------------------------
def test_viewport_entry_points_on_a_plan_only_context():
    from miniengineao_b200 import AmbientOcclusion, Camera
    lib = N.lib()
    a = AmbientOcclusion(Camera(64, 48), device=-1)
    a.LateUpdate()
    ctx = a._ctx
    fake = C.c_void_p(0x1000)
    assert lib.meao_render_arrays_at(ctx, fake, 0, 0, 0, fake, 8, 8, None) == N.MEAO_ERR_CUDA
    assert b"plan-only" in lib.meao_last_error(ctx)
    assert lib.meao_bind_event_arrays_at(ctx, 7, fake, 0, 0, 0, fake, 8, 8, None) == N.MEAO_ERR_CUDA
    assert lib.meao_bind_event_arrays_at(ctx, 7, None, 0, 0, 0, None, 0, 0, None) == N.MEAO_OK       # unbinding needs no device
    assert lib.meao_render_arrays_at(None, fake, 0, 0, 0, fake, 0, 0, None) == N.MEAO_ERR_INVALID
    assert lib.meao_bind_event_arrays_at(None, 7, fake, 0, 0, 0, fake, 0, 0, None) == N.MEAO_ERR_INVALID
    with pytest.raises(ValueError):
        a.render_arrays(1, 2, kind="d24", depth_origin=(0, 0))
