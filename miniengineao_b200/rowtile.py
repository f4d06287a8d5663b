"""Row-band partition of ONE frame over several GPUs (BASELINE.json configs[3]; a capability the reference
does not have -- SURVEY.md 8e).

One process per GPU.  Rank r owns output rows [cuts[r], cuts[r+1]) (16-row aligned) and only ever sees that
band of the raw depth.

mode "native" (default on GPUs): the exchange lives INSIDE libmeao (include/meao.h "native neighbour exchange"): the
ranks swap arena handles once (meao_band_export -> all_gather -> meao_band_connect: cudaIpc peer mappings), after which a
step is ONE CUDA graph per band -- prepare_depth -> band_exchange_kernel (peer stores over NVLink + epoch flags) ->
render x4 + upsample x4 -- with no Python, no NCCL call and no staging copy between the phases.

mode "p2p" (the CPU / gloo tests, and the fallback when peer mappings are unavailable).  Per frame:

    phase A  (one CUDA graph)  prepare_depth on the own rows (LinearDepth + LowDepth1..4)
                               + pack of the border rows of LowDepth1..4 each neighbour needs (<= ~0.6 MB per side at 8K)
    exchange                   ONE send + ONE recv per neighbour (torch.distributed P2P: NCCL on GPUs, gloo in the CPU tests)
    phase B  (one CUDA graph)  unpack into the same global-coordinate buffers + render x4 + upsample x4 on exactly
                               the rows the band needs

The exchange is neighbour-only; no all-reduce / all-gather is ever needed.  The row ranges come from the C
planner (meao_band_rows / meao_halo_rows), so this module contains no geometry of its own.
"""
from __future__ import annotations

import numpy as np


def partition(height: int, world: int) -> list[int]:
    """Band boundaries: world contiguous bands of 16-row blocks, as even as possible."""
    blocks = (height + 15) // 16
    cuts = [min(height, 16 * ((blocks * i) // world)) for i in range(world)] + [height]
    for a, b in zip(cuts[:-1], cuts[1:]):
        if b <= a:
            raise ValueError(f"{world} bands do not fit into {height} rows")
    return cuts


def neighbours(cuts: list[int], rank: int) -> tuple[int, int]:
    """(prev_row0, next_row1) for meao_set_row_band; -1 where there is no neighbour."""
    world = len(cuts) - 1
    return (cuts[rank - 1] if rank > 0 else -1, cuts[rank + 2] if rank + 1 < world else -1)


def exchange(send_up, send_down, recv_up, recv_down, rank: int, world: int, group=None) -> None:
    """One message per direction per neighbour.  Tensors may be CUDA (NCCL) or CPU (gloo); empty ones are skipped."""
    import torch.distributed as dist
    ops = []
    if rank > 0:
        if send_up is not None and send_up.numel():
            ops.append(dist.P2POp(dist.isend, send_up, rank - 1, group))
        if recv_up is not None and recv_up.numel():
            ops.append(dist.P2POp(dist.irecv, recv_up, rank - 1, group))
    if rank + 1 < world:
        if send_down is not None and send_down.numel():
            ops.append(dist.P2POp(dist.isend, send_down, rank + 1, group))
        if recv_down is not None and recv_down.numel():
            ops.append(dist.P2POp(dist.irecv, recv_down, rank + 1, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()


class RowTiledAO:
    """GPU driver of one band (one per rank)."""

    def __init__(self, camera, rank: int, world: int, device: int, mode: str = "native", group=None, **params):
        import torch
        from .ambient_occlusion import AmbientOcclusion
        self.rank, self.world, self.mode, self.group = rank, world, mode, group
        self.cuts = partition(camera.pixelHeight, world)
        self.row0, self.row1 = self.cuts[rank], self.cuts[rank + 1]
        self.ao = AmbientOcclusion(camera, device=device)
        for k, v in params.items():
            setattr(self.ao, k, v)
        prev0, next1 = neighbours(self.cuts, rank)
        self.ao.set_row_band(self.row0, self.row1, prev0, next1)
        dev = torch.device("cuda", device)
        mk = lambda n: torch.empty(max(int(n), 0), dtype=torch.uint8, device=dev)  # noqa: E731
        self.send = [mk(self.ao.halo_bytes(0)), mk(self.ao.halo_bytes(1))]
        self.recv = [mk(self.ao.halo_recv_bytes(0)), mk(self.ao.halo_recv_bytes(1))]
        self.width = camera.pixelWidth
        if mode == "native" and world > 1:
            self._connect_native(dev)

    def _connect_native(self, dev) -> None:
        """Swap the arena handles with every rank (one all_gather of 128 bytes) and map the two neighbours' arenas."""
        import torch
        import torch.distributed as dist
        mine = torch.frombuffer(bytearray(self.ao.band_export()), dtype=torch.uint8)
        backend = dist.get_backend(self.group)
        mine = mine.to(dev) if backend == "nccl" else mine
        allh = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(allh, mine, group=self.group)
        handles = [bytes(h.cpu().numpy().tobytes()) for h in allh]
        err = None
        try:
            if self.rank > 0:
                self.ao.band_connect(0, handles[self.rank - 1])
            if self.rank + 1 < self.world:
                self.ao.band_connect(1, handles[self.rank + 1])
        except Exception as e:              # no peer access / IPC on this box
            err = e
        # the decision must be COLLECTIVE: a rank that fell back while its neighbours stepped natively would leave them spinning
        ok = torch.tensor([0 if err else 1], dtype=torch.int32, device=dev if backend == "nccl" else "cpu")
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)       # also: nobody steps before every mapping exists
        if int(ok.item()) == 0:
            for side in (0, 1):
                try:
                    self.ao.band_connect(side, None)
                except Exception:
                    pass
            raise RuntimeError(f"native neighbour exchange unavailable on at least one rank ({err if err else 'another rank failed'})")

    @property
    def rows(self) -> int:
        return self.row1 - self.row0

    def step(self, depth_band, out_band, stream=None) -> None:
        """depth_band: CUDA f32 [rows, W]; out_band: CUDA u8 [rows, W].  Everything is enqueued on `stream`
        (default: torch's current stream), the P2P included, so steps can be issued back to back."""
        ao = self.ao
        if self.mode == "native":
            ao.band_step(depth_band, out_band, stream=stream)                        # ONE graph, exchange kernel inside
            return
        import torch
        ao.band_phase_a(depth_band, self.send[0], self.send[1], stream=stream)       # graph: prepare_depth + pack
        # NCCL enqueues the P2P on torch's CURRENT stream: make `stream` current so pack -> send and recv -> unpack are ordered
        with torch.cuda.stream(stream) if stream is not None else _null_ctx():
            exchange(self.send[0], self.send[1], self.recv[0], self.recv[1], self.rank, self.world, self.group)
        ao.band_phase_b(self.recv[0], self.recv[1], out_band, stream=stream)         # graph: unpack + 8 kernels (DAG)


class _null_ctx:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


def pack_rows(low: dict[int, np.ndarray], rows: list[tuple[int, int]]) -> np.ndarray:
    """The message meao_halo_pack sends: rows[k - 1] of level k, level 1 first, rows tightly packed."""
    parts = [low[k + 1][lo:hi].reshape(-1) for k, (lo, hi) in enumerate(rows) if hi > lo]
    return np.concatenate(parts).astype(np.float32) if parts else np.zeros(0, np.float32)


def unpack_rows(low: dict[int, np.ndarray], rows: list[tuple[int, int]], buf: np.ndarray) -> None:
    off = 0
    for k, (lo, hi) in enumerate(rows):
        if hi <= lo:
            continue
        w = low[k + 1].shape[1]
        n = (hi - lo) * w
        low[k + 1][lo:hi] = buf[off:off + n].reshape(hi - lo, w)
        off += n
