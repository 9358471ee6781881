"""Multi-GPU plumbing: one process per GPU, torch.distributed (NCCL on the GPUs, gloo in CPU tests).

Inference shards scenes across ranks with NO data-path collective (scenes are independent, SURVEY.md §8e);
the only exchange on the hot path is the codebook-EMA statistics of the training step, which the reference
issues as two blocking all-reduces inside the quantizer forward (viewformer/models/utils_th.py:50-52) and which
are packed into ONE all-reduce here.
"""
import torch
import torch.distributed as dist


def shard_range(n_items, rank, world):
    """Contiguous, balanced [lo, hi) of ``n_items`` scenes for ``rank`` (first n % world ranks get one extra)."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def allreduce_ema_stats(counts, embed_sum, group=None):
    """SUM-all-reduce of (counts [K], embed_sum [D,K]) as one packed [K + D*K] buffer; returns new tensors."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return counts, embed_sum
    k = counts.numel()
    packed = torch.cat([counts.reshape(-1), embed_sum.reshape(-1)])
    dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
    return packed[:k].reshape(counts.shape).contiguous(), packed[k:].reshape(embed_sum.shape).contiguous()


def max_over_ranks(value, device):
    """max of a python float over all ranks (bench timing: device time, max over ranks)."""
    t = torch.tensor([float(value)], device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)
