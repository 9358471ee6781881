"""Multi-GPU plumbing: one process per GPU, torch.distributed (NCCL on the GPUs, gloo in CPU tests).

Inference shards scenes across ranks with NO data-path collective (scenes are independent, SURVEY.md §8e).  The training steps exchange
two things: the codebook-EMA statistics, which the reference issues as two blocking all-reduces inside the quantizer forward
(viewformer/models/utils_th.py:50-52) and which are packed into ONE all-reduce here, and the gradients, through ``GradExchange``: one
flat buffer in backward-completion order, all-reduced bucket by bucket while the backward pass is still running.
"""
import math

import torch
import torch.distributed as dist

from . import _lib as L


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


class GradExchange:
    """The trainers' parameters, gradients and optimizer moments in flat fp32 buffers, and the data-parallel gradient exchange over them.

    ``entries``: (name, shape) pairs in the order the backward pass completes them.  Each name gets 16-byte aligned views ``p[name]`` /
    ``g[name]`` / ``m[name]`` / ``v[name]`` at ``offs[name]`` of ``flat_p`` / ``flat_g`` / ``flat_m`` / ``flat_v``.  A bucket is a contiguous range
    (start, end, name of its last parameter) of the flat gradient, closed after the parameter that pushes it past ``bucket_bytes``; the
    last one closes at the end.  Once the backward pass has signalled every gradient of a bucket (``ready``), the bucket is divided by
    the running step's gradient-seed scale and its asynchronous SUM all-reduce starts, so the transfers ride under the rest of the
    backward pass.

    Gradient accumulation: ``reset(seed_scale, micro_batches=N)`` opens a window of N backward passes that all add into ``flat_g``, which
    is zeroed only there.  ``next_micro_batch()`` arms each further pass.  In passes 1 .. N-1 a completed bucket is only counted; in pass N
    it is unscaled and exchanged as above (DDP's ``no_sync``), so a window costs one exchange whatever N is.  ``flush()`` exchanges the
    buckets of a window that ends early."""

    def __init__(self, entries, device, bucket_bytes, group=None):
        self.group = group
        self.order, self.offs, n = [name for name, _ in entries], {}, 0
        sizes = {name: math.prod(shape) for name, shape in entries}
        for name in self.order:
            self.offs[name] = n
            n += (sizes[name] + 3) // 4 * 4                  # 16-byte aligned views
        self.flat_p = torch.zeros((n,), dtype=torch.float32, device=device)
        self.flat_g, self.flat_m, self.flat_v = torch.zeros_like(self.flat_p), torch.zeros_like(self.flat_p), torch.zeros_like(self.flat_p)
        self.p, self.g, self.m, self.v = {}, {}, {}, {}
        for name, shape in entries:
            o = self.offs[name]
            for views, flat in ((self.p, self.flat_p), (self.g, self.flat_g), (self.m, self.flat_m), (self.v, self.flat_v)):
                views[name] = flat[o:o + sizes[name]].view(shape)
        self.buckets, self._bucket_of, self._bucket_size, start, count = [], {}, [], 0, 0
        for i, name in enumerate(self.order):
            self._bucket_of[name] = len(self.buckets)
            count += 1
            end = self.offs[name] + (sizes[name] + 3) // 4 * 4
            if (end - start) * 4 >= bucket_bytes or i == len(self.order) - 1:
                self.buckets.append((start, end, name))
                self._bucket_size.append(count)
                start, count = end, 0
        self.launched = []                                   # buckets in the order their exchange started; cleared in place every step
        self.reset()

    def world(self):
        return dist.get_world_size(self.group) if (dist.is_available() and dist.is_initialized()) else 1

    def reset(self, seed_scale=1.0, micro_batches=1):
        """Open a window of ``micro_batches`` backward passes and arm the first: zero the gradient, no bucket signalled yet.  Every pass of
        the window runs on seeds times ``seed_scale`` (a power of two), so the one division at the end is exact."""
        if int(micro_batches) < 1:
            raise ValueError(f"micro_batches must be >= 1, got {micro_batches}")
        self.flat_g.zero_()
        self.seed_scale = seed_scale
        self.micro_batches, self.micro = int(micro_batches), 1     # passes in the window; the running pass (1-based)
        self.handles, self._left = [], list(self._bucket_size)
        self.launched.clear()

    def next_micro_batch(self):
        """Arm the next backward pass of the open window; the previous pass must have signalled every bucket."""
        self.check_complete()
        if self.micro >= self.micro_batches:
            raise RuntimeError(f"the accumulation window of {self.micro_batches} micro-batches is complete")
        self.micro += 1
        self._left = list(self._bucket_size)

    def ready(self, *names):
        """The backward pass has finished the gradients of ``names``.  In the window's last pass: unscale and start the all-reduce of every
        bucket this completes."""
        for name in names:
            b = self._bucket_of[name]
            self._left[b] -= 1
            if self._left[b] == 0:
                if self.micro == self.micro_batches:
                    self._exchange(b)
            elif self._left[b] < 0:
                raise RuntimeError(f"gradient of {name} signalled twice")

    def _exchange(self, b):
        self.launched.append(b)
        s, e, _ = self.buckets[b]
        if self.seed_scale != 1.0:                           # divide the seed scale back out (exact: a power of two)
            L.lincomb3(1.0 / self.seed_scale, self.flat_g[s:e], out=self.flat_g[s:e])
        if self.world() > 1:
            self.handles.append(dist.all_reduce(self.flat_g[s:e], op=dist.ReduceOp.SUM, group=self.group, async_op=True))

    def flush(self):
        """End the window after the running pass even if it is not the last planned one (an optimizer step on a partial window): unscale
        and exchange every bucket.  Nothing to do in the window's last pass: its own ``ready`` calls exchange the buckets."""
        if self.micro == self.micro_batches:
            return
        self.check_complete()
        for b in range(len(self.buckets)):
            self._exchange(b)
        self.micro_batches = self.micro

    def check_complete(self):
        """End of the backward pass: every bucket must have been signalled."""
        if any(self._left):
            raise RuntimeError("backward pass left gradient buckets incomplete: " + str([self.buckets[i][2] for i, n in enumerate(self._left) if n]))

    def wait(self):
        """Wait for the all-reduces of the step: flat_g then holds the gradient summed over ranks."""
        for h in self.handles:
            h.wait()
        self.handles = []


def max_over_ranks(value, device):
    """max of a python float over all ranks (bench timing: device time, max over ranks)."""
    t = torch.tensor([float(value)], device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)
