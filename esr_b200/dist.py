"""Multi-GPU plumbing: one process per GPU, torch.distributed (NCCL on the GPUs, gloo in CPU tests).

The hot path shards by batch (independent sequences, no BatchNorm; SURVEY.md 8e): inference, encoding and
redistribution need NO collective; ranks only meet to agree on timings.  Training adds exactly one exchange --
the all-reduce of the 1 813 120-element gradient -- for which `flat_allreduce_` is the bucket primitive."""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """(rank, world, local_rank); initialises the default process group when WORLD_SIZE > 1."""
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        dist.init_process_group(backend or ("nccl" if torch.cuda.is_available() else "gloo"))
    return rank, world, local


def shard_range(n, world, rank):
    """Contiguous [lo, hi) slice of n independent units for `rank`: sizes differ by at most one, earlier ranks larger
    (same split as torch.utils.data.DistributedSampler without padding)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def max_over_ranks(value, device="cpu"):
    """Timing reduction: every rank reports the slowest rank's value."""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def flat_allreduce_(tensors, average=True):
    """One all-reduce over a single flat bucket holding all `tensors` (gradients + logging scalars), in place."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return tensors
    flat = torch.cat([t.reshape(-1) for t in tensors])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    if average:
        flat /= dist.get_world_size()
    off = 0
    for t in tensors:
        t.copy_(flat[off:off + t.numel()].view_as(t))
        off += t.numel()
    return tensors
