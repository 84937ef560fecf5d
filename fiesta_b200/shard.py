"""Multi-GPU driver for the x-slab sharded UpdateESDF (one process per GPU, torch.distributed for the plumbing).

Every rank integrates every frame identically (ray casting / UpdateOccupancy are replicated); only the distance-field
relaxation is partitioned: rank r relaxes the tile columns of its x-slab and the 2-voxel ghost layers on the internal faces
(dirs_ reaches 2 voxels, FIESTA include/parameters.h:66-68) travel between neighbouring ranks after every local
relaxation -- over NVLink with NCCL on GPUs (gloo in the CPU protocol test) -- until no rank sees a changed ghost record.
A ghost x-layer is Gy*Pz contiguous records, so layers are exchanged exactly as they lie in HBM (no packing kernel).
"""
import torch
import torch.distributed as dist


class HaloBuffers:
    """Four exchange buffers of `layer_words` 32-bit words on `device`."""

    def __init__(self, layer_words, device):
        mk = lambda: torch.zeros(int(layer_words), dtype=torch.int32, device=device)
        self.send_lo, self.send_hi, self.recv_lo, self.recv_hi = mk(), mk(), mk(), mk()


def exchange(bufs, rank, world):
    """send_lo -> rank-1 (arrives as its recv_hi), send_hi -> rank+1 (arrives as its recv_lo)."""
    ops = []
    if rank > 0:
        ops.append(dist.P2POp(dist.isend, bufs.send_lo, rank - 1))
        ops.append(dist.P2POp(dist.irecv, bufs.recv_lo, rank - 1))
    if rank + 1 < world:
        ops.append(dist.P2POp(dist.isend, bufs.send_hi, rank + 1))
        ops.append(dist.P2POp(dist.irecv, bufs.recv_hi, rank + 1))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()


def sharded_update_esdf(m, bufs, rank, world, ptr=lambda t: t.data_ptr(), max_rounds=10000):
    """m: a map with UpdateESDF(), shard_pack(lo, hi), shard_ingest(lo, hi) -> changed ghost records and
    shard_relax() -> changed slab records (fiesta_b200.ESDFMap after set_shard, or the mock of the CPU protocol test).
    Returns the number of exchange rounds."""
    m.UpdateESDF()
    rounds = 0
    while True:
        rounds += 1
        m.shard_pack(ptr(bufs.send_lo) if rank > 0 else 0, ptr(bufs.send_hi) if rank + 1 < world else 0)
        exchange(bufs, rank, world)
        changed = m.shard_ingest(ptr(bufs.recv_lo) if rank > 0 else 0, ptr(bufs.recv_hi) if rank + 1 < world else 0)
        if changed:
            changed += m.shard_relax()
        t = torch.tensor([changed], dtype=torch.int64, device=bufs.send_lo.device)
        dist.all_reduce(t)
        if int(t.item()) == 0 or rounds >= max_rounds:
            return rounds
