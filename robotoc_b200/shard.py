"""Multi-GPU sharding of the OCP batch (SURVEY.md 8e).

OCP instances are independent (no coupling between batch elements anywhere in OCPSolver::updateSolution,
robotoc/src/solver/ocp_solver.cpp:111-145), so the batch is split into contiguous blocks, one per rank / GPU;
there is no data-path collective inside an iteration.  The only exchange is ONE all-gather of the Newton step
(direction records) so that every rank sees the whole step (north_star: "a single NCCL all-gather of the converged
step").  torch.distributed is plumbing: NCCL over NVLink on GPUs, gloo in the CPU tests.
"""
from typing import Tuple


def shard_range(batch: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous block [lo, hi) of a global batch owned by `rank`; sizes differ by at most one."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("[shard_range] invalid argument: need 0 <= rank < world")
    if batch < 0:
        raise ValueError("[shard_range] invalid argument: batch must be non-negative")
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def allgather_step(local, global_batch=None, out=None, group=None):
    """All-gather the per-rank tensor [b_local, ...] into [global_batch, ...] (rank-major, i.e. shard_range order).
    Shard sizes follow from (global_batch, world) -- no size exchange, no host sync.  Equal shards: one
    all_gather_into_tensor straight into `out` (NCCL, in place); ragged shards (global_batch % world != 0) are padded to the
    largest shard first."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    if global_batch is None:
        global_batch = local.shape[0] * world
    sizes = [shard_range(global_batch, world, r)[1] - shard_range(global_batch, world, r)[0] for r in range(world)]
    if sizes[dist.get_rank(group)] != local.shape[0]:
        raise ValueError("[allgather_step] invalid argument: local shard size does not match shard_range")
    if out is None:
        out = torch.empty((global_batch,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    if len(set(sizes)) == 1:
        dist.all_gather_into_tensor(out.view(-1), local.contiguous().view(-1), group=group)
    else:
        mx = max(sizes)
        pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        pad[:local.shape[0]].copy_(local)
        buf = torch.empty((world * mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(buf.view(-1), pad.view(-1), group=group)
        off = 0
        for r, n in enumerate(sizes):
            out[off:off + n].copy_(buf[r * mx:r * mx + n])
            off += n
    return out
