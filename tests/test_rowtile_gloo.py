"""world_size-2 (and 3) gloo test of the row-band path on CPU (no GPU): the host-side logic of the
multi-GPU mode -- partition, the C planner's halo row ranges, pack/unpack layout and the neighbour
exchange over torch.distributed -- with the ORACLE standing in for the kernels.

Each rank sees only its band of the raw depth, produces LowDepth1..4 for its own rows, exchanges exactly the
rows meao_halo_rows names, then POISONS (NaN) every LowDepth row the planner says it does not need.  If the
planner's ranges were too small anywhere, NaNs would reach the band's output rows; the band rows must equal
the single-process full-frame result bit for bit."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, W, H, q, mask=0):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from miniengineao_b200 import AmbientOcclusion, Camera, rowtile, synth
    from oracle.oracle import Oracle

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        lin = synth.random_depth(W, H, seed=77)
        depth = synth.lin01_to_raw(lin)
        ref = Oracle(W, H, intensity=1.1, high_quality_mask=mask).run(depth)

        cuts = rowtile.partition(H, world)
        r0, r1 = cuts[rank], cuts[rank + 1]
        plan = AmbientOcclusion(Camera(W, H), device=-1)        # planning-only context: no GPU needed
        plan.intensity = 1.1
        plan.highQualityMask = mask
        prev0, next1 = rowtile.neighbours(cuts, rank)
        plan.set_row_band(r0, r1, prev0, next1)
        rows = plan.band_rows()

        # this rank only has its band of the depth buffer
        mine = np.full((H, W), 0.5, np.float32)
        mine[r0:r1] = depth[r0:r1]
        o = Oracle(W, H, intensity=1.1, high_quality_mask=mask)
        o.downsample(mine)
        low = {k: o.buffer(1 + k) for k in range(1, 5)}
        for k in range(1, 5):                                   # forget everything this band does not own
            olo, ohi = rows["own_low"][k]
            low[k][:olo] = np.nan
            low[k][ohi:] = np.nan

        send = [torch.from_numpy(rowtile.pack_rows(low, plan.halo_rows(side, True))) for side in (0, 1)]
        recv = [torch.empty(plan.halo_recv_bytes(side) // 4, dtype=torch.float32) for side in (0, 1)]
        assert [t.numel() * 4 for t in send] == [plan.halo_bytes(0), plan.halo_bytes(1)]
        rowtile.exchange(send[0], send[1], recv[0], recv[1], rank, world)
        for side in (0, 1):
            rowtile.unpack_rows(low, plan.halo_rows(side, False), recv[side].numpy())

        for k in range(1, 5):                                   # the planner claims only these rows are read
            nlo, nhi = rows["need_low"][k]
            assert not np.isnan(low[k][nlo:nhi]).any(), f"level {k}: needed rows still missing after the exchange"
        # the oracle's render reads the deinterleaved atlases: rebuild them from the exchanged LowDepth rows
        # exactly as Downsample1/2 would have written them (padding: Linearize(0) = 1e5 for k <= 2, 0 for k >= 3)
        from oracle import direct_formulation as DF
        for k in range(1, 5):
            sw, sh = o.level_dims(k + 2)
            with np.errstate(over="ignore", invalid="ignore"):
                o.set_buffer(5 + k, DF.tiled_view(low[k], sw, sh, np.float32(1e5) if k <= 2 else np.float32(0)))
        for k in range(1, 5):
            o.render(k)
        for k in range(1, 5):                                   # Render.compute kernel "main" reads LowDepth<k> itself (+-8 rows, clamped)
            if (mask >> (k - 1)) & 1:
                for kk in range(1, 5):
                    nlo, nhi = rows["need_low"][kk]
                    chk = o.buffer(1 + kk)
                    chk[:nlo] = np.nan
                    chk[nhi:] = np.nan                              # poison what the planner says is never read
                o.render_wide(k)
        for lo_level in range(4, 0, -1):
            o.upsample(lo_level)
        got = o.ao_u8()[r0:r1]
        q.put((rank, int((got != ref[r0:r1]).sum()), int(send[0].numel() + send[1].numel())))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,W,H,mask", [(2, 192, 1088, 0), (3, 128, 1584, 0), (2, 192, 1088, 15)])
def test_row_bands_over_gloo_match_full_frame(world, W, H, mask):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, W, H, q, mask)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    results = sorted(q.get(timeout=5) for _ in range(world))
    assert [r[0] for r in results] == list(range(world))
    assert all(r[1] == 0 for r in results), results          # band rows identical to the full-frame oracle
    assert all(r[2] > 0 for r in results)                    # and something was actually exchanged


def test_partition_is_16_row_aligned_and_balanced():
    from miniengineao_b200 import rowtile
    for H, world in ((4320, 8), (4320, 4), (4320, 2), (2160, 4), (1080, 2)):
        cuts = rowtile.partition(H, world)
        assert cuts[0] == 0 and cuts[-1] == H and len(cuts) == world + 1
        assert all(c % 16 == 0 for c in cuts[:-1])
        sizes = [b - a for a, b in zip(cuts[:-1], cuts[1:])]
        assert max(sizes) - min(sizes) <= 16 + (H % 16)
    assert rowtile.neighbours([0, 544, 1088], 0) == (-1, 1088)
    assert rowtile.neighbours([0, 544, 1088], 1) == (0, -1)


def _worker_emulated(rank, world, port, W, H, q, mask):
    """Same protocol as RowTiledAO.step, but with the HOST-COMPILED kernel sources (tests/emu) as the compute of each rank:
    prepare_depth on the band -> halo_copy pack -> gloo exchange -> halo_copy unpack -> render / upsample on the band's rows."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from miniengineao_b200 import AmbientOcclusion, Camera, rowtile, synth
    from oracle.oracle import Oracle
    from emu.emu import Frame

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        depth = synth.lin01_to_raw(synth.random_depth(W, H, seed=99))
        ref = Oracle(W, H, intensity=1.1, high_quality_mask=mask).run(depth)
        cuts = rowtile.partition(H, world)
        r0, r1 = cuts[rank], cuts[rank + 1]
        plan = AmbientOcclusion(Camera(W, H), device=-1)
        plan.intensity, plan.highQualityMask = 1.1, mask
        plan.set_row_band(r0, r1, *rowtile.neighbours(cuts, rank))
        f = Frame(plan)
        f.use_plan_band()                                   # also poisons every LowDepth texel with NaN
        f.band_phase_a(depth[r0:r1])                        # this rank only ever sees its band of the depth buffer
        send = [torch.from_numpy(f.halo_pack(side).copy()) for side in (0, 1)]
        recv = [torch.empty(plan.halo_recv_bytes(side) // 4, dtype=torch.float32) for side in (0, 1)]
        rowtile.exchange(send[0], send[1], recv[0], recv[1], rank, world)
        for side in (0, 1):
            f.halo_unpack(side, recv[side].numpy())
        got = f.band_phase_b()
        q.put((rank, int((got != ref[r0:r1]).sum()), int(send[0].numel() + send[1].numel())))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,W,H,mask", [(2, 192, 1088, 0), (3, 160, 1600, 0b1010)])
def test_row_bands_with_emulated_kernels_over_gloo(world, W, H, mask):
    """The multi-GPU band path end to end on CPU: the C planner's ranges, the REAL kernels' row-range logic (host build),
    the halo pack / unpack kernel and the neighbour exchange; every LowDepth row a band neither owns nor receives is NaN."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_emulated, args=(r, world, port, W, H, q, mask)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    results = sorted(q.get(timeout=5) for _ in range(world))
    assert all(r[1] == 0 for r in results), results
    assert all(r[2] > 0 for r in results)
