"""GPU tests of the frame schedule's launch counts (csrc/frame_record.h frame_schedule): every way of issuing a frame -- the captured
graph and its replays, MEAO_FLAG_NO_GRAPH, band_prepare + band_finish -- launches meao_kernels_per_frame kernels, and a replayed graph
counts exactly the launches its capture recorded."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

VARIANTS = [dict(), dict(high_quality_mask=15), dict(single_scale=True)]
IDS = ["default", "hq15", "single_scale"]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a GPU")
    return torch


def _ctx(W, H, *, use_graph=True, high_quality_mask=0, single_scale=False):
    from miniengineao_b200 import AmbientOcclusion, Camera
    ao = AmbientOcclusion(Camera(W, H), device=0, use_graph=use_graph)
    ao.highQualityMask, ao.singleScale, ao.intensity = high_quality_mask, single_scale, 1.1
    ao.LateUpdate()
    return ao


def _depth(torch, W, H):
    from miniengineao_b200 import synth
    return torch.from_numpy(synth.lin01_to_raw(synth.random_depth(W, H, seed=7))).cuda()


def _oracle(W, H, depth, **kw):
    from oracle.oracle import Oracle
    return Oracle(W, H, threads=8, intensity=1.1, **kw).run(depth.cpu().numpy())


@pytest.mark.parametrize("kw", VARIANTS, ids=IDS)
def test_every_frame_form_launches_kernels_per_frame(torch_cuda, kw):
    torch = torch_cuda
    W, H = 320, 184
    d = _depth(torch, W, H)
    ref = _oracle(W, H, d, **kw)
    kpf = 3 if kw.get("single_scale") else 9 + bin(kw.get("high_quality_mask", 0)).count("1")
    for use_graph in (True, False):
        ao = _ctx(W, H, use_graph=use_graph, **kw)
        assert ao.kernels_per_frame == kpf
        out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
        for _ in range(2):                                  # with a graph: the capture, then a replay
            before = ao.launch_count
            ao.render(d, out)
            assert ao.launch_count - before == kpf, (use_graph, kw)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), ref), (use_graph, kw)
        # the stage API's band pair on a whole-frame context: the full prepare_depth, then the rest of the schedule
        out.zero_()
        before = ao.launch_count
        ao.band_prepare(d)
        ao.band_finish(out)
        assert ao.launch_count - before == kpf, (use_graph, kw)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), ref), (use_graph, kw)


def test_band_phases_count_the_launches_they_captured(torch_cuda):
    """A halo buffer for a side without a neighbour: its rows are empty, so no halo kernel is recorded and a replay counts none."""
    torch = torch_cuda
    W, H = 320, 184
    d = _depth(torch, W, H)
    ref = _oracle(W, H, d)
    ao = _ctx(W, H)
    assert ao.halo_bytes(0) == 0 and ao.halo_recv_bytes(0) == 0
    spare = torch.zeros(16, dtype=torch.uint8, device="cuda")
    out = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    for _ in range(2):
        before = ao.launch_count
        ao.band_phase_a(d, spare, None)
        assert ao.launch_count - before == 1
        before = ao.launch_count
        ao.band_phase_b(spare, None, out)
        assert ao.launch_count - before == ao.kernels_per_frame - 1
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), ref)
