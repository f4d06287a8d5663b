"""GPU tests of layered frames (meao_set_layers): every layer of one layered frame must be bit-identical to the oracle run on that
layer alone, on the H100, through every public path (graph replay, direct launches, host buffers, stage buffers, debug views,
composites)."""
import ctypes as C

import numpy as np
import pytest

import harness
from gpu_harness import torch_cuda  # noqa: F401  (the fixture)

pytestmark = pytest.mark.gpu


def _check_layers(ao, got, refs, tag):
    for l, ref in enumerate(refs):
        n = int((got[l] != ref).sum())
        assert n == 0, f"{tag}: layer {l} differs from the oracle in {n} pixels"


def _oracles(ao, W, H, L, stereo=False, linear=False, **kw):
    """L oracles with the context's variants; under stereo with the field of view of ao's eye camera."""
    if stereo:
        kw["tan_half_fov_h_"] = 1.0 / ao.camera.projection00
    return [harness.oracle(W, H, stereo=stereo, linear=linear, threads=8, **kw) for _ in range(L)]


def _refs(W, H, depth, **kw):
    return [orc.run(depth[l]) for l, orc in enumerate(_oracles(None, W, H, depth.shape[0], **kw))]


def _compare_buffers(ao, W, H, depth, tag, **kw):
    """All debug buffers of every layer (stacked form of meao_get_buffer) against the single-layer oracle."""
    ids = harness.buffer_ids(kw.get("high_quality_mask", 0), kw.get("single_scale", False))
    got = {bid: ao.debug_buffer(bid) for bid in ids}
    for l, orc in enumerate(_oracles(ao, W, H, depth.shape[0], **kw)):
        orc.run(depth[l])
        harness.compare_buffers(lambda bid: got[bid][l], orc, f"{tag} layer {l}", ids)


@pytest.mark.parametrize("L", [2, 6])
def test_1080p_distinct_frames(torch_cuda, L):
    from miniengineao_b200 import synth
    W, H = 1920, 1080
    depth = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    ao = harness.context(W, H, device=0, layers=L)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    assert got.shape == (L, H, W)
    _check_layers(ao, got, _refs(W, H, depth), f"1080p L={L}")


def test_4k_two_layers(torch_cuda):
    W, H = 3840, 2160
    depth = harness.frames(W, H, 2, seed=3)
    ao = harness.context(W, H, device=0, layers=2)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    _check_layers(ao, got, _refs(W, H, depth), "4K L=2")


def test_ragged_1001x563_all_buffers(torch_cuda):
    W, H = 1001, 563
    depth = harness.frames(W, H, 3, seed=1)
    ao = harness.context(W, H, device=0, layers=3, intensity=1.1)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    _check_layers(ao, got, _refs(W, H, depth, intensity=1.1), "1001x563")
    _compare_buffers(ao, W, H, depth, "1001x563", intensity=1.1)


@pytest.mark.parametrize("W,H,L", [(640, 360, 1), (640, 360, 4), (1280, 720, 2), (1280, 720, 3), (1920, 1080, 1), (160, 90, 9)])
def test_both_sides_of_the_tile_rules(torch_cuda, W, H, L):
    """The persistent upsample loop (>= 2 tiles per CTA slot, counted over all layers) and the render tile height (CTAs of all
    layers) switch at different layer counts; every side must give the single-layer bits."""
    depth = harness.frames(W, H, L, seed=L)
    ao = harness.context(W, H, device=0, layers=L)
    d = torch_cuda.from_numpy(depth if L > 1 else depth[0]).cuda()       # a single-layer context takes [H, W]
    got = ao.render(d).cpu().numpy().reshape(L, H, W)
    _check_layers(ao, got, _refs(W, H, depth), f"{W}x{H} L={L}")


@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(sample_exhaustively=True, reversed_z=False), dict(single_scale=True),
                                dict(stereo=True), dict(high_quality_mask=0b0101, sample_exhaustively=True, intensity=1.3)])
def test_variants_three_layers(torch_cuda, kw):
    W, H = 322, 203
    depth = harness.frames(W, H, 3, seed=5, reversed_z=kw.get("reversed_z", True))
    ao = harness.context(W, H, device=0, layers=3, **kw)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    _check_layers(ao, got, [orc.run(depth[l]) for l, orc in enumerate(_oracles(ao, W, H, 3, **kw))], str(kw))
    _compare_buffers(ao, W, H, depth, str(kw), **kw)


def test_native_and_linear_ingest_three_layers(torch_cuda):
    from miniengineao_b200 import synth
    W, H = 322, 203
    lin = np.stack([synth.random_depth(W, H, seed=40 + i) for i in range(3)]).astype(np.float32)
    ao = harness.context(W, H, device=0, layers=3)
    got = ao.render(torch_cuda.from_numpy(lin).cuda(), linear=True).cpu().numpy()
    _check_layers(ao, got, _refs(W, H, lin, linear=True), "linear")
    raw = np.stack([synth.lin01_to_raw(l) for l in lin])
    for kind in ("d16", "d24s8"):
        words, as_float = harness.ingest(raw, kind, stencil=0x5A)
        words = words if kind == "d16" else words.view(np.int32)                  # D24S8 as int32 words
        got = ao.render(torch_cuda.from_numpy(np.ascontiguousarray(words)).cuda()).cpu().numpy()
        _check_layers(ao, got, _refs(W, H, as_float), kind)


def test_graph_replay_three_frames_and_launch_count(torch_cuda):
    W, H, L = 640, 360, 3
    ao = harness.context(W, H, device=0, layers=L)
    d = torch_cuda.empty((L, H, W), dtype=torch_cuda.float32, device="cuda")
    out = torch_cuda.empty((L, H, W), dtype=torch_cuda.uint8, device="cuda")
    for f in range(3):
        depth = harness.frames(W, H, L, seed=10 + f)
        d.copy_(torch_cuda.from_numpy(depth))
        before = ao.launch_count
        ao.render(d, out)
        assert ao.launch_count - before == ao.kernels_per_frame == 9
        _check_layers(ao, out.cpu().numpy(), _refs(W, H, depth), f"replay {f}")


def test_no_graph_flag(torch_cuda):
    W, H, L = 400, 240, 2
    depth = harness.frames(W, H, L, seed=2)
    ao = harness.context(W, H, device=0, layers=L, use_graph=False)
    before = ao.launch_count
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    assert ao.launch_count - before == 9
    _check_layers(ao, got, _refs(W, H, depth), "NO_GRAPH")


def test_host_paths(torch_cuda):
    from miniengineao_b200 import _native as N
    W, H, L = 330, 190, 3
    ao = harness.context(W, H, device=0, layers=L)
    depth = harness.frames(W, H, L, seed=4)
    refs = _refs(W, H, depth)
    _check_layers(ao, ao.render_host(depth), refs, "render_host")
    lib = N.lib()
    n = L * W * H
    pin_d = [lib.meao_host_alloc(n * 4) for _ in range(3)]
    pin_o = [lib.meao_host_alloc(n) for _ in range(3)]
    try:
        ds = [np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), (L, H, W)) for p in pin_d]
        os_ = [np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), (L, H, W)) for p in pin_o]
        frames = [harness.frames(W, H, L, seed=20 + i) for i in range(3)]
        for i in range(3):
            ds[i][...] = frames[i]
        ao.render_host_batch(ds, os_)            # render_host_async over both staging slots
        for i in range(3):
            _check_layers(ao, os_[i], _refs(W, H, frames[i]), f"async {i}")
    finally:
        for p in pin_d + pin_o:
            lib.meao_host_free(p)


def test_stacked_buffers_debug_view_and_composite(torch_cuda):
    from oracle import oracle as O
    W, H, L = 258, 146, 2
    ao = harness.context(W, H, device=0, layers=L)
    depth = harness.frames(W, H, L, seed=6)
    out = ao.render(torch_cuda.from_numpy(depth).cuda())
    torch_cuda.cuda.synchronize()
    orcs = []
    for l in range(L):
        o = harness.oracle(W, H, threads=8)
        o.run(depth[l])
        orcs.append(o)
    for bid in (1, 3, 6, 11, 17):
        view = ao.debug_view(bid).cpu().numpy()
        assert view.shape == (L, H, W)
        for l in range(L):
            assert np.array_equal(view[l], orcs[l].debug_view(bid)), (bid, l)
    # set_buffer in stacked form: overwrite Occlusion2 of both layers, re-run the upsample chain through the stage entry points
    occ2 = ao.debug_buffer(11)
    assert occ2.shape[0] == L
    new = np.ascontiguousarray(occ2[::-1])                       # swap the layers
    ao.set_debug_buffer(11, new)
    assert np.array_equal(ao.debug_buffer(11), new)
    ao.set_debug_buffer(11, occ2)
    # composite over L x W x H pixels
    rng = np.random.default_rng(0)
    color = rng.integers(0, 256, size=(L, H, W, 4), dtype=np.uint8)
    col = torch_cuda.from_numpy(color).cuda()
    ao.composite_framebuffer(out, col)
    got = col.cpu().numpy()
    aoc = out.cpu().numpy()
    for l in range(L):
        assert np.array_equal(got[l], O.composite_framebuffer(aoc[l], color[l])), l


def test_switching_layers_back_to_one_equals_a_fresh_context(torch_cuda):
    W, H = 500, 280
    depth3 = harness.frames(W, H, 3, seed=8)
    ao = harness.context(W, H, device=0, layers=3)
    ao.render(torch_cuda.from_numpy(depth3).cuda())
    ao.layers = 1
    d1 = torch_cuda.from_numpy(depth3[1]).cuda()
    got = ao.render(d1).cpu().numpy()
    assert got.shape == (H, W)
    fresh = harness.context(W, H, device=0, layers=1).render(d1).cpu().numpy()
    assert np.array_equal(got, fresh)
    assert np.array_equal(got, harness.oracle(W, H, threads=8).run(depth3[1]))


def test_band_entry_points_refuse_layers(torch_cuda):
    from miniengineao_b200 import MeaoError
    from miniengineao_b200 import _native as N
    ao = harness.context(640, 720, device=0, layers=2)
    ao.LateUpdate()
    with pytest.raises(MeaoError) as e:
        ao.set_row_band(0, 368, -1, 720)
    assert e.value.code == N.MEAO_ERR_UNSUPPORTED
    lib, ctx = N.lib(), ao._ctx
    d = torch_cuda.zeros((2, 720, 640), device="cuda")
    o = torch_cuda.zeros((2, 720, 640), dtype=torch_cuda.uint8, device="cuda")
    buf = torch_cuda.zeros(1 << 20, device="cuda")
    for rc in (lib.meao_halo_bytes(ctx, 1), lib.meao_halo_recv_bytes(ctx, 1), lib.meao_halo_rows(ctx, 1, 1, (C.c_int32 * 8)()),
               lib.meao_halo_pack(ctx, 1, buf.data_ptr(), None), lib.meao_halo_unpack(ctx, 1, buf.data_ptr(), None),
               lib.meao_render_band_prepare(ctx, d.data_ptr(), 0, None), lib.meao_render_band_finish(ctx, o.data_ptr(), None),
               lib.meao_band_phase_a(ctx, d.data_ptr(), 0, None, None, None), lib.meao_band_phase_b(ctx, None, None, o.data_ptr(), None),
               lib.meao_band_export(ctx, C.byref(N.MeaoPeerHandle())), lib.meao_band_connect(ctx, 1, None),
               lib.meao_band_step(ctx, d.data_ptr(), 0, o.data_ptr(), None)):
        assert rc == N.MEAO_ERR_UNSUPPORTED
        assert b"single-layer" in lib.meao_last_error(ctx)
    hd = np.zeros((2, 720, 640), np.float32)
    ho = np.zeros((2, 720, 640), np.uint8)
    assert lib.meao_band_step_host(ctx, hd.ctypes.data, 0, ho.ctypes.data) == N.MEAO_ERR_UNSUPPORTED
