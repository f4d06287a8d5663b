"""CPU tests of layered frames (meao_set_layers): L same-size views stacked at a stride of one image, one launch per stage.

The layered kernel sources (csrc/*_layered.cu) run in the fiber emulator (tests/emu/layered_emu.py) and every layer must be bit-identical to the
oracle run on that layer alone -- all 17 buffers and the AO.  Neighbouring layers are chosen to contrast (a corridor, constant
depth, a frame with a sky patch, random depth) at sizes where no level is a multiple of 4, 16 or 64, so a read across a layer
boundary changes bits.  Also here: the packed-contraction audit of the layered translation units and the plan-only contract of
meao_set_layers (return values, refusals, algorithmic bytes, the Python shape checks)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from miniengineao_b200 import AmbientOcclusion, Camera, MeaoError, synth
from miniengineao_b200 import _native as N
from oracle.oracle import Oracle

from emu.layered_emu import LayeredFrame  # noqa: E402  (tests/ is on sys.path via conftest)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "miniengineao_b200", "csrc")

PARAMS = {"noise_filter_tolerance": "noiseFilterTolerance", "blur_tolerance": "blurTolerance", "upsample_tolerance": "upsampleTolerance",
          "thickness_modifier": "thicknessModifier", "intensity": "intensity", "sample_exhaustively": "sampleExhaustively",
          "high_quality_mask": "highQualityMask"}


def _plan(W, H, layers=1, single_scale=False, **kw):
    p = AmbientOcclusion(Camera(W, H, usesReversedZBuffer=kw.get("reversed_z", True)), device=-1)
    for py, cs in PARAMS.items():
        if py in kw:
            setattr(p, cs, kw[py])
    p.singleScale = single_scale
    p.layers = layers
    return p


def contrasting_layers(W, H, n, seed=0):
    """Linear depth in [0, 1) of n layers that differ sharply at every boundary; layer 2 carries a sky patch (raw depth 0)."""
    out = []
    for i in range(n):
        kind = i % 4
        if kind == 0:
            lin = synth.corridor(W, H, frame=i)
        elif kind == 1:
            lin = np.full((H, W), 0.37, np.float32)
        elif kind == 2:
            lin = synth.random_depth(W, H, seed=seed + 17 * i, lo=0.05, hi=0.6)
        else:
            lin = synth.random_depth(W, H, seed=seed + 31 * i)
        out.append(lin.astype(np.float32))
    return np.stack(out)


def _raw(lin, reversed_z=True):
    raw = np.stack([synth.lin01_to_raw(l, reversed_z=reversed_z) for l in lin])
    if len(raw) > 2:
        H, W = raw.shape[1:]
        raw[2, H // 4: H // 2, W // 5: W // 2] = 0.0          # sky: raw 0 -> 1e5 -> inf in f16 -> NaN paths
    return raw


def _compare_layer(f, layer, orc, tag, mask=0, ids=None):
    bad = []
    for bid in ids or (list(range(1, 18)) + [17 + k for k in range(1, 5) if (mask >> (k - 1)) & 1]):
        got, ref = f.buffer(bid, layer), orc.buffer(bid)
        if got.dtype == np.uint8:
            n = int((got != orc.codes(bid)).sum())
        elif got.dtype == np.float16:
            with np.errstate(over="ignore"):
                n = int((got.view(np.uint16) != ref.astype(np.float16).view(np.uint16)).sum())
        else:
            n = int((got.view(np.uint32) != ref.view(np.uint32)).sum())
        if n:
            bad.append((bid, n, got.size))
    assert not bad, f"{tag} layer {layer}: mismatching buffers (id, #diff, size): {bad}"


def _run_layers(W, H, depth, *, use_tma=True, linear=False, single_scale=False, oracle_depth=None, **kw):
    """depth: [L, H, W] in the ingest format; oracle_depth: the float32 the oracle sees per layer (default: depth itself)."""
    L = depth.shape[0]
    f = LayeredFrame(_plan(W, H, L, single_scale=single_scale, **kw), linear=linear, use_tma=use_tma)
    n0 = f.tma_box_loads()
    f.run(depth)
    f.tma_loads_in_run = f.tma_box_loads() - n0
    okw = dict(kw)
    if linear:
        okw["depth_is_linear"] = True
    if single_scale:
        okw["single_scale"] = True
    ids = [1, 2, 3, 4, 5, 10, 17] if single_scale else None
    for l in range(L):
        orc = Oracle(W, H, threads=4, **okw)
        ref = orc.run(depth[l] if oracle_depth is None else oracle_depth[l])
        assert np.array_equal(f.buffer(17, l), ref), (W, H, l, kw)
        _compare_layer(f, l, orc, f"{W}x{H} {kw}", kw.get("high_quality_mask", 0), ids)
    return f


@pytest.mark.parametrize("use_tma", [True, False])
@pytest.mark.parametrize("W,H", [(161, 93), (37, 300), (250, 131)])
def test_ragged_layers_equal_single_layer_oracle(W, H, use_tma):
    depth = _raw(contrasting_layers(W, H, 3, seed=W))
    f = _run_layers(W, H, depth, use_tma=use_tma, intensity=1.1)
    if not use_tma:
        assert f.tma_loads_in_run == 0


def test_layered_interior_tiles_take_the_tma_path():
    """Big enough for interior (TMA-fed) tiles in every layer: the boxes are fetched at the layer's row offset of the stacked map."""
    W, H = 640, 360
    depth = _raw(contrasting_layers(W, H, 3, seed=3))
    f = _run_layers(W, H, depth, intensity=1.1, high_quality_mask=0b0011)
    assert f.tma_loads_in_run > 300, f.tma_loads_in_run


@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(sample_exhaustively=True, reversed_z=False), dict(single_scale=True)])
def test_layered_variants(kw):
    W, H = 130, 70
    rz = kw.get("reversed_z", True)
    depth = _raw(contrasting_layers(W, H, 3, seed=7), reversed_z=rz)
    _run_layers(W, H, depth, intensity=1.2, **kw)


def test_layered_linear_and_native_ingest():
    W, H = 250, 131
    lin = contrasting_layers(W, H, 3, seed=9)
    _run_layers(W, H, lin, linear=True)
    raw = _raw(lin).astype(np.float64)
    for bits, dt in ((16, np.uint16), (24, np.uint32)):
        full = (1 << bits) - 1
        codes = np.clip(np.rint(raw * full), 0, full).astype(np.uint32)
        as_float = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
        words = codes.astype(np.uint16) if bits == 16 else (codes | (np.uint32(0xA5) << np.uint32(24)))
        _run_layers(W, H, words.astype(dt), oracle_depth=as_float)


def test_layered_vector_alignment_widths():
    """W % 8 == 0 keeps the 128-bit input loads in every layer (the layer stride W x H keeps the 16-byte alignment); W % 4 == 0
    with D16 input takes the per-element path.  Both must equal the oracle."""
    for W, H, dt in ((136, 40, np.uint16), (132, 44, np.uint16), (132, 44, np.float32)):
        raw = _raw(contrasting_layers(W, H, 3, seed=W)).astype(np.float64)
        if dt == np.uint16:
            codes = np.clip(np.rint(raw * 65535), 0, 65535).astype(np.uint32)
            as_float = (codes.astype(np.float32) * np.float32(1.0 / 65535)).astype(np.float32)
            _run_layers(W, H, codes.astype(np.uint16), oracle_depth=as_float)
        else:
            _run_layers(W, H, raw.astype(np.float32))


# ---- packed-contraction audit of the layered translation units (the method of test_no_packed_contraction.py) ---------------
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false"]
EXPECTED = {"prepare_depth_layered.cu": 0, "render_ao_layered.cu": 0, "blur_upsample_layered.cu": 12}   # the same surpluses as the single-image TUs


@pytest.mark.parametrize("tu", sorted(EXPECTED))
def test_layered_units_have_only_the_audited_contractions(tu, tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else shutil.which("nvcc")
    if not nvcc or not shutil.which("cuobjdump"):
        pytest.skip("nvcc / cuobjdump not available")
    src = os.path.join(CSRC, tu)
    ptx, cubin = os.path.join(str(tmp_path), "k.ptx"), os.path.join(str(tmp_path), "k.cubin")
    subprocess.check_call([nvcc] + FLAGS + ["-ptx", "-o", ptx, src], stderr=subprocess.DEVNULL)
    subprocess.check_call([nvcc] + FLAGS + ["-cubin", "-o", cubin, src], stderr=subprocess.DEVNULL)
    p = open(ptx).read()
    s = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True).stdout
    assert "f32x2" not in p, tu
    assert not re.search(r"\b(FFMA2|FMUL2|FADD2)\b", s), tu
    n_mul = len(re.findall(r"\bmul\.rn\.f32\b", p))
    n_fmul = len(re.findall(r"\bFMUL\b", s))
    assert n_mul > 0, tu
    assert n_fmul - n_mul == EXPECTED[tu], (tu, n_mul, n_fmul)


# ---- plan-only contract ------------------------------------------------------------------------------------------------------
def test_set_layers_return_values_and_limits():
    lib = N.lib()
    a = AmbientOcclusion(Camera(640, 360), device=-1)
    a.LateUpdate()
    ctx = a._ctx
    assert lib.meao_set_layers(ctx, 1) == 0
    assert lib.meao_set_layers(ctx, 3) == 1
    assert lib.meao_set_layers(ctx, 3) == 0
    for bad in (0, -1, 65536, 1 << 30):
        assert lib.meao_set_layers(ctx, bad) == N.MEAO_ERR_INVALID
        assert b"layers" in lib.meao_last_error(ctx)
    assert lib.meao_set_layers(ctx, 65535) == 1            # the largest grid z dimension
    assert lib.meao_set_layers(ctx, 1) == 1
    assert lib.meao_set_layers(None, 2) == N.MEAO_ERR_INVALID
    # before the first resize the value is simply kept
    b = AmbientOcclusion(Camera(64, 64), device=-1)
    assert lib.meao_set_layers(b._ctx, 2) == 1


def test_python_layers_property_is_a_plan_input():
    a = AmbientOcclusion(Camera(320, 180), device=-1)
    a.LateUpdate()
    a.set_row_band(0, 96, -1, 180)
    a.layers = 2
    assert a.LateUpdate() is True
    assert a._band is None and a.band_rows()["produce"][0] == (0, 180)      # like a resize: back to the whole frame
    assert a.LateUpdate() is False
    assert a.kernels_per_frame == 9                                         # one layered launch is one kernel


def test_bands_and_halos_are_refused_with_layers():
    lib = N.lib()
    a = AmbientOcclusion(Camera(640, 720), device=-1)
    a.layers = 3
    a.LateUpdate()
    with pytest.raises(MeaoError) as e:
        a.set_row_band(0, 368, -1, 720)
    assert e.value.code == N.MEAO_ERR_UNSUPPORTED and "single-layer" in str(e.value)
    ctx = a._ctx
    assert lib.meao_halo_bytes(ctx, 0) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_halo_recv_bytes(ctx, 1) == N.MEAO_ERR_UNSUPPORTED
    assert lib.meao_halo_rows(ctx, 0, 1, (C.c_int32 * 8)()) == N.MEAO_ERR_UNSUPPORTED
    for rc in (lib.meao_halo_pack(ctx, 0, None, None), lib.meao_halo_unpack(ctx, 0, None, None),
               lib.meao_render_band_prepare(ctx, None, 0, None), lib.meao_render_band_finish(ctx, None, None),
               lib.meao_band_phase_a(ctx, None, 0, None, None, None), lib.meao_band_phase_b(ctx, None, None, None, None),
               lib.meao_band_export(ctx, C.byref(N.MeaoPeerHandle())), lib.meao_band_connect(ctx, 0, None),
               lib.meao_band_step(ctx, None, 0, None, None), lib.meao_band_step_host(ctx, None, 0, None)):
        assert rc == N.MEAO_ERR_UNSUPPORTED
        assert b"layers" in lib.meao_last_error(ctx)
    a.layers = 1
    a.LateUpdate()
    a.set_row_band(0, 368, -1, 720)                                         # single layer again: bands work
    assert a.halo_bytes(1) > 0


def test_algorithmic_bytes_scale_by_layers():
    a = AmbientOcclusion(Camera(1920, 1080), device=-1)
    one = [a.algorithmic_bytes(s) for s in range(6)]
    for L in (2, 6):
        a.layers = L
        assert [a.algorithmic_bytes(s) for s in range(6)] == [L * v for v in one]


def test_python_shape_checks_take_a_layer_axis():
    a = AmbientOcclusion(Camera(64, 48), device=-1)
    a.layers = 3
    with pytest.raises(ValueError):
        a.render_host(np.zeros((48, 64), np.float32))                       # a single image is not a 3-layer frame
    with pytest.raises(MeaoError) as e:
        a.render_host(np.zeros((3, 48, 64), np.float32))                    # the right shape reaches the library (no device here)
    assert e.value.code == N.MEAO_ERR_CUDA
    with pytest.raises(ValueError):
        a.render_host_batch([np.zeros((48, 64), np.float32)], [np.zeros((48, 64), np.uint8)])
    d = a.buffer_desc(6)
    assert a._buffer_shape(d) == (3, 16, d.height, d.width)
    assert a._buffer_shape(a.buffer_desc(2)) == (3, 24, 32)
    a.layers = 1
    assert a._frame_shape() == (48, 64) and a._buffer_shape(a.buffer_desc(2)) == (24, 32)
