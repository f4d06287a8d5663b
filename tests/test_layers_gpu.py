"""GPU tests of layered frames (meao_set_layers): every layer of one layered frame must be bit-identical to the oracle run on that
layer alone, on the H100, through every public path (graph replay, direct launches, host buffers, stage buffers, debug views,
composites)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a GPU")
    return torch


def _ctx(W, H, layers, *, use_graph=True, stereo=False, **params):
    from miniengineao_b200 import AmbientOcclusion, Camera
    cam = Camera(W // 2 if stereo else W, H, stereoEnabled=stereo, usesReversedZBuffer=params.get("reversed_z", True))
    ao = AmbientOcclusion(cam, device=0, use_graph=use_graph)
    ao.sampleExhaustively = bool(params.get("sample_exhaustively", False))
    ao.highQualityMask = int(params.get("high_quality_mask", 0))
    ao.singleScale = bool(params.get("single_scale", False))
    if "intensity" in params:
        ao.intensity = params["intensity"]
    ao.layers = layers
    if stereo:
        ao.OnPreRender()
    return ao


def _oracle(W, H, stereo=False, linear=False, ao=None, **params):
    from oracle.oracle import Oracle
    okw = {k: params[k] for k in ("sample_exhaustively", "high_quality_mask", "single_scale", "intensity", "reversed_z") if k in params}
    if stereo:
        okw["single_pass_stereo"] = True
        okw["tan_half_fov_h_"] = 1.0 / ao.camera.projection00
    if linear:
        okw["depth_is_linear"] = True
    return Oracle(W, H, threads=8, **okw)


def _frames(W, H, L, seed=0, reversed_z=True):
    """L contrasting raw-depth layers: corridors of distinct frames, constant depth, a sky patch, random depth."""
    from miniengineao_b200 import synth
    out = []
    for i in range(L):
        k = (i + seed) % 4
        if k == 0:
            lin = synth.corridor(W, H, frame=i + seed)
        elif k == 1:
            lin = np.full((H, W), 0.37, np.float32)
        else:
            lin = synth.random_depth(W, H, seed=seed * 13 + i)
        raw = synth.lin01_to_raw(lin, reversed_z=reversed_z).astype(np.float32)
        if k == 2:
            raw[H // 4: H // 2, W // 5: W // 2] = 0.0
        out.append(raw)
    return np.stack(out)


def _check_layers(ao, got, refs, tag):
    for l, ref in enumerate(refs):
        n = int((got[l] != ref).sum())
        assert n == 0, f"{tag}: layer {l} differs from the oracle in {n} pixels"


def _refs(W, H, depth, **kw):
    out = []
    for l in range(depth.shape[0]):
        orc = _oracle(W, H, **kw)
        out.append(orc.run(depth[l]))
    return out


def _compare_buffers(ao, W, H, depth, tag, oracle_depth=None, **kw):
    """All debug buffers of every layer (stacked form of meao_get_buffer) against the single-layer oracle."""
    L = depth.shape[0]
    mask = kw.get("high_quality_mask", 0)
    ids = [1, 2, 3, 4, 5, 10, 17] if kw.get("single_scale") else list(range(1, 18)) + [17 + k for k in range(1, 5) if (mask >> (k - 1)) & 1]
    got = {bid: ao.debug_buffer(bid) for bid in ids}
    for l in range(L):
        orc = _oracle(W, H, ao=ao, **kw)
        orc.run(depth[l] if oracle_depth is None else oracle_depth[l])
        bad = []
        for bid in ids:
            g = got[bid][l]
            if g.dtype == np.uint8:
                n = int((g != orc.codes(bid)).sum())
            elif g.dtype == np.float16:
                with np.errstate(over="ignore"):
                    n = int((g.view(np.uint16) != orc.buffer(bid).astype(np.float16).view(np.uint16)).sum())
            else:
                n = int((g.view(np.uint32) != orc.buffer(bid).view(np.uint32)).sum())
            if n:
                bad.append((bid, n))
        assert not bad, f"{tag} layer {l}: (id, #diff) {bad}"


@pytest.mark.parametrize("L", [2, 6])
def test_1080p_distinct_frames(torch_cuda, L):
    from miniengineao_b200 import synth
    W, H = 1920, 1080
    depth = np.stack([synth.lin01_to_raw(synth.corridor(W, H, frame=i)).astype(np.float32) for i in range(L)])
    ao = _ctx(W, H, L)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    assert got.shape == (L, H, W)
    _check_layers(ao, got, _refs(W, H, depth), f"1080p L={L}")


def test_4k_two_layers(torch_cuda):
    W, H = 3840, 2160
    depth = _frames(W, H, 2, seed=3)
    ao = _ctx(W, H, 2)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    _check_layers(ao, got, _refs(W, H, depth), "4K L=2")


def test_ragged_1001x563_all_buffers(torch_cuda):
    W, H = 1001, 563
    depth = _frames(W, H, 3, seed=1)
    ao = _ctx(W, H, 3, intensity=1.1)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    _check_layers(ao, got, _refs(W, H, depth, intensity=1.1), "1001x563")
    _compare_buffers(ao, W, H, depth, "1001x563", intensity=1.1)


@pytest.mark.parametrize("W,H,L", [(640, 360, 1), (640, 360, 4), (1280, 720, 2), (1280, 720, 3), (1920, 1080, 1), (160, 90, 9)])
def test_both_sides_of_the_tile_rules(torch_cuda, W, H, L):
    """The persistent upsample loop (>= 2 tiles per CTA slot, counted over all layers) and the render tile height (CTAs of all
    layers) switch at different layer counts; every side must give the single-layer bits."""
    depth = _frames(W, H, L, seed=L)
    ao = _ctx(W, H, L)
    d = torch_cuda.from_numpy(depth if L > 1 else depth[0]).cuda()       # a single-layer context takes [H, W]
    got = ao.render(d).cpu().numpy().reshape(L, H, W)
    _check_layers(ao, got, _refs(W, H, depth), f"{W}x{H} L={L}")


@pytest.mark.parametrize("kw", [dict(high_quality_mask=15), dict(sample_exhaustively=True, reversed_z=False), dict(single_scale=True),
                                dict(stereo=True), dict(high_quality_mask=0b0101, sample_exhaustively=True, intensity=1.3)])
def test_variants_three_layers(torch_cuda, kw):
    W, H = 322, 203
    depth = _frames(W, H, 3, seed=5, reversed_z=kw.get("reversed_z", True))
    ao = _ctx(W, H, 3, **kw)
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    okw = dict(kw)
    _check_layers(ao, got, [(_oracle(W, H, ao=ao, **okw).run(depth[l])) for l in range(3)], str(kw))
    _compare_buffers(ao, W, H, depth, str(kw), **okw)


def test_native_and_linear_ingest_three_layers(torch_cuda):
    from miniengineao_b200 import synth
    W, H = 322, 203
    lin = np.stack([synth.random_depth(W, H, seed=40 + i) for i in range(3)]).astype(np.float32)
    ao = _ctx(W, H, 3)
    got = ao.render(torch_cuda.from_numpy(lin).cuda(), linear=True).cpu().numpy()
    _check_layers(ao, got, [_oracle(W, H, linear=True).run(lin[l]) for l in range(3)], "linear")
    raw = np.stack([synth.lin01_to_raw(l) for l in lin]).astype(np.float64)
    for bits in (16, 24):
        full = (1 << bits) - 1
        codes = np.clip(np.rint(raw * full), 0, full).astype(np.uint32)
        as_float = (codes.astype(np.float32) * np.float32(1.0 / full)).astype(np.float32)
        words = codes.astype(np.uint16) if bits == 16 else (codes | (np.uint32(0x5A) << np.uint32(24))).view(np.int32)   # D24S8 as int32 words
        got = ao.render(torch_cuda.from_numpy(np.ascontiguousarray(words)).cuda()).cpu().numpy()
        _check_layers(ao, got, _refs(W, H, as_float), f"D{bits}")


def test_graph_replay_three_frames_and_launch_count(torch_cuda):
    W, H, L = 640, 360, 3
    ao = _ctx(W, H, L)
    d = torch_cuda.empty((L, H, W), dtype=torch_cuda.float32, device="cuda")
    out = torch_cuda.empty((L, H, W), dtype=torch_cuda.uint8, device="cuda")
    for f in range(3):
        depth = _frames(W, H, L, seed=10 + f)
        d.copy_(torch_cuda.from_numpy(depth))
        before = ao.launch_count
        ao.render(d, out)
        assert ao.launch_count - before == ao.kernels_per_frame == 9
        _check_layers(ao, out.cpu().numpy(), _refs(W, H, depth), f"replay {f}")


def test_no_graph_flag(torch_cuda):
    W, H, L = 400, 240, 2
    depth = _frames(W, H, L, seed=2)
    ao = _ctx(W, H, L, use_graph=False)
    before = ao.launch_count
    got = ao.render(torch_cuda.from_numpy(depth).cuda()).cpu().numpy()
    assert ao.launch_count - before == 9
    _check_layers(ao, got, _refs(W, H, depth), "NO_GRAPH")


def test_host_paths(torch_cuda):
    from miniengineao_b200 import _native as N
    W, H, L = 330, 190, 3
    ao = _ctx(W, H, L)
    depth = _frames(W, H, L, seed=4)
    refs = _refs(W, H, depth)
    _check_layers(ao, ao.render_host(depth), refs, "render_host")
    lib = N.lib()
    n = L * W * H
    pin_d = [lib.meao_host_alloc(n * 4) for _ in range(3)]
    pin_o = [lib.meao_host_alloc(n) for _ in range(3)]
    try:
        ds = [np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), (L, H, W)) for p in pin_d]
        os_ = [np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), (L, H, W)) for p in pin_o]
        frames = [_frames(W, H, L, seed=20 + i) for i in range(3)]
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
    ao = _ctx(W, H, L)
    depth = _frames(W, H, L, seed=6)
    out = ao.render(torch_cuda.from_numpy(depth).cuda())
    torch_cuda.cuda.synchronize()
    orcs = []
    for l in range(L):
        o = _oracle(W, H)
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
    depth3 = _frames(W, H, 3, seed=8)
    ao = _ctx(W, H, 3)
    ao.render(torch_cuda.from_numpy(depth3).cuda())
    ao.layers = 1
    d1 = torch_cuda.from_numpy(depth3[1]).cuda()
    got = ao.render(d1).cpu().numpy()
    assert got.shape == (H, W)
    fresh = _ctx(W, H, 1).render(d1).cpu().numpy()
    assert np.array_equal(got, fresh)
    assert np.array_equal(got, _oracle(W, H).run(depth3[1]))


def test_band_entry_points_refuse_layers(torch_cuda):
    from miniengineao_b200 import MeaoError
    from miniengineao_b200 import _native as N
    ao = _ctx(640, 720, 2)
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
