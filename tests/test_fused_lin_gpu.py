"""The fused final upsample on the H100: a whole frame runs prepare_depth in its low-only form (LowDepth1..4 from the even depth
rows, no LinearDepth) and the final blur_upsample reads the raw depth, linearises it and writes LinearDepth itself
(csrc/blur_upsample_lin.cu).  Checked here: oracle parity of every buffer over the depth kinds, Z directions, variants and sizes up
to 4K; that LinearDepth is still produced by every frame (a NaN-poisoned buffer is fully overwritten); and that the fused frame
equals the split forms that keep prepare_depth -> LinearDepth -> blur_upsample (stage API, band prepare / finish).
meao_band_step (the fused form on a row band) is checked against the oracle by test_parity_gpu.py's native-exchange tests."""
import numpy as np
import pytest

import harness
from gpu_harness import torch_cuda  # noqa: F401  (the fixture)

pytestmark = pytest.mark.gpu


def _depth(kind, W, H, seed, reversed_z=True):
    """(device tensor, what the oracle sees) for one depth kind; sky patches so that the grouped range test falls back."""
    import torch
    from miniengineao_b200 import synth
    lin = synth.random_depth(W, H, seed=seed)
    raw = synth.lin01_to_raw(lin, reversed_z=reversed_z) if kind != "linear" else lin.astype(np.float32)
    raw = raw.astype(np.float32)
    sky = np.float32(0.0 if reversed_z else 1.0)
    raw[: max(1, H // 7), : max(1, W // 5)] = sky
    words, as_float = harness.ingest(raw, kind, stencil=0x5A)
    if kind in ("f32", "linear"):
        return torch.from_numpy(raw).cuda(), raw
    if kind == "d16":
        return torch.from_numpy(words.view(np.int16)).cuda().view(torch.uint16), as_float
    return torch.from_numpy(words.view(np.int32)).cuda(), as_float


SIZES = [(1, 1), (3, 5), (161, 93), (250, 131), (37, 1000), (644, 362), (1920, 1080)]


@pytest.mark.parametrize("kind", ["f32", "d16", "d24s8", "linear"])
@pytest.mark.parametrize("W,H", SIZES)
def test_fused_frame_matches_oracle(torch_cuda, kind, W, H):
    reversed_z = (W + H) % 2 == 0
    ao, orc = harness.context_and_oracle(W, H, intensity=1.1, reversed_z=reversed_z)
    d, seen = _depth(kind, W, H, seed=W * 3 + H, reversed_z=reversed_z)
    if kind == "linear":
        orc = harness.oracle(W, H, threads=8, intensity=1.1, reversed_z=reversed_z, linear=True)
    ref = orc.run(seen)
    got = ao.render(d, linear=(kind == "linear")).cpu().numpy()
    assert np.array_equal(got, ref)
    harness.compare_buffers(ao.debug_buffer, orc, f"{kind} {W}x{H}", harness.buffer_ids())


@pytest.mark.parametrize("variant", [dict(high_quality_mask=15), dict(high_quality_mask=1), dict(single_scale=True)])
@pytest.mark.parametrize("W,H", [(250, 131), (1283, 721)])
def test_fused_variants_match_oracle(torch_cuda, variant, W, H):
    ao, orc = harness.context_and_oracle(W, H, intensity=1.1, **{k: v for k, v in variant.items() if k != "single_scale"})
    if variant.get("single_scale"):
        ao.singleScale = True
        orc = harness.oracle(W, H, threads=8, intensity=1.1, single_scale=True)
    d, seen = _depth("f32", W, H, seed=5)
    ref = orc.run(seen)
    assert np.array_equal(ao.render(d).cpu().numpy(), ref)
    if not variant.get("single_scale"):
        harness.compare_buffers(ao.debug_buffer, orc, str(variant), harness.buffer_ids(variant.get("high_quality_mask", 0)))


def test_fused_4k_matches_oracle(torch_cuda):
    from miniengineao_b200 import synth
    W, H = 3840, 2160
    depth = synth.lin01_to_raw(synth.corridor(W, H))
    ao = harness.context(W, H, device=0, intensity=1.1, high_quality_mask=15)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    ref = harness.oracle(W, H, threads=16, intensity=1.1, high_quality_mask=15).run(depth)
    assert np.array_equal(got, ref)


def test_linear_depth_is_written_by_every_frame(torch_cuda):
    """LinearDepth poisoned with NaN before a frame: after it, every element equals the oracle's (the low-only prepare_depth does not
    write it; the fused final upsample writes each pixel once, partial rows included)."""
    W, H = 331, 187
    ao, orc = harness.context_and_oracle(W, H, intensity=1.1)
    d, seen = _depth("f32", W, H, seed=11)
    ref = orc.run(seen)
    ao.render(d)
    torch_cuda.cuda.synchronize()
    ao.set_debug_buffer(1, np.full((H, W), np.nan, np.float16))
    assert np.isnan(ao.debug_buffer(1).astype(np.float32)).all()
    got = ao.render(d).cpu().numpy()
    assert np.array_equal(got, ref)
    lin = ao.debug_buffer(1)
    assert np.array_equal(lin.view(np.uint16), orc.buffer(1).astype(np.float16).view(np.uint16))


def test_host_batch_matches_oracle(torch_cuda):
    """meao_render_host_async: the staged depth is now read by the last kernel of the frame too."""
    W, H = 500, 284
    ao, orc = harness.context_and_oracle(W, H, intensity=1.1)
    ds = [_depth("f32", W, H, seed=40 + i)[1] for i in range(4)]
    outs = [np.zeros((H, W), np.uint8) for _ in ds]
    ao.render_host_batch(ds, outs)
    for i, (dd, o) in enumerate(zip(ds, outs)):
        assert np.array_equal(o, orc.run(dd)), i


def test_fused_equals_stage_api_and_band_split(torch_cuda):
    """The same depth through the fused frame, the stage API and one whole-frame band's prepare / finish (both of which keep
    prepare_depth -> LinearDepth -> blur_upsample): identical AO and LinearDepth."""
    from miniengineao_b200 import AmbientOcclusion, Camera
    torch = torch_cuda
    W, H = 720, 404
    d, _ = _depth("f32", W, H, seed=3)
    fused = AmbientOcclusion(Camera(W, H), device=0)
    ref = fused.render(d).cpu().numpy()
    ref_lin = fused.debug_buffer(1).view(np.uint16)

    st = AmbientOcclusion(Camera(W, H), device=0)
    st.stage_downsample(d)
    for k in range(1, 5):
        st.stage_render(k)
    for lo in range(4, 0, -1):
        st.stage_upsample(lo)
    st.synchronize()
    assert np.array_equal(st.debug_buffer(17), ref)
    assert np.array_equal(st.debug_buffer(1).view(np.uint16), ref_lin)

    band = AmbientOcclusion(Camera(W, H), device=0)
    band.set_row_band(0, H)
    band.band_prepare(d)
    out = torch.empty((H, W), dtype=torch.uint8, device="cuda")
    band.band_finish(out)
    band.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)
    assert np.array_equal(band.debug_buffer(1).view(np.uint16), ref_lin)
