"""Gradient accumulation in the shared gradient exchange (dist.GradExchange), world_size 2 over gloo on the CPU: a window of N micro-batches
adds into one flat gradient and exchanges it once — no all-reduce before the window's last backward pass, every bucket reduced exactly once,
and the result bit for bit the plain all-reduce of the locally summed gradient.  Driven as each trainer builds the exchange
(VQGANTrainer._flatten, MIGTTrainer._build); the kernels are not involved."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from viewformer_b200.dist import GradExchange


def _codebook_exchange():
    from types import SimpleNamespace
    from viewformer_b200.train import VQGANTrainer, _P
    g = torch.Generator().manual_seed(5)
    shapes = [(3, 3, 7, 5), (5,), (33, 17), (17,), (1,), (64, 9), (9,), (1023,), (2, 2)]
    params = [_P(f"p{i}", torch.randn(s, generator=g), lambda v: None, "conv") for i, s in enumerate(shapes)]
    tr = VQGANTrainer.__new__(VQGANTrainer)
    tr.model = SimpleNamespace(device=torch.device("cpu"), _refresh_decode_table=lambda: None)
    tr.params, tr.bucket_bytes, tr.group = params, 4096, None
    tr._flatten()
    return tr.ex


def _transformer_exchange():
    from viewformer_b200 import MIGT
    from viewformer_b200.config import MIGTConfig
    from viewformer_b200.train_migt import MIGTTrainer
    from oracle import synth
    cfg = MIGTConfig(n_layer=2, n_head=4, d_model=64, sequence_size=4, n_embeddings=32, token_image_size=4)
    mt = MIGTTrainer.__new__(MIGTTrainer)
    mt.model, mt.cfg, mt.device, mt.bucket_bytes, mt.group = MIGT(cfg, precision="fp32"), cfg, torch.device("cpu"), 32 << 10, None
    mt._build(synth.make_migt_state_dict(cfg, 3))
    return mt.ex


def _window(ex, rank, n, group_size, seed, check):
    """One window of ``n`` backward passes with seed scale 1: each pass adds a random gradient per tensor and signals the names in groups
    of ``group_size``, in backward order.  Returns the locally summed gradient, accumulated in the same order."""
    local = torch.zeros_like(ex.flat_g)
    ex.reset(1.0, micro_batches=n)
    for mb in range(n):
        if mb:
            ex.next_micro_batch()
        gr = torch.Generator().manual_seed(seed + 100 * mb + rank)
        names = ex.order
        for i in range(0, len(names), group_size):
            for name in names[i:i + group_size]:
                t = torch.randn(ex.g[name].shape, generator=gr)
                ex.g[name].add_(t)                              # what every gradient kernel does: add into the flat buffer
                o = ex.offs[name]
                local[o:o + t.numel()] += t.reshape(-1)
            ex.ready(*names[i:i + group_size])
            if mb < n - 1:
                check(not ex.launched and not ex.handles, f"an exchange started in micro-batch {mb + 1} of {n}")
        ex.check_complete()
    check(sorted(ex.launched) == list(range(len(ex.buckets))) and len(ex.handles) == len(ex.buckets),
          f"buckets exchanged {sorted(ex.launched)}, expected each of {len(ex.buckets)} once")
    return local


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ok, why = True, []

    def check(cond, msg):
        nonlocal ok
        if not cond:
            ok = False
            why.append(msg)

    for tag, ex, group_size in (("codebook", _codebook_exchange(), 2), ("transformer", _transformer_exchange(), 3)):
        check(len(ex.buckets) >= 3, f"{tag}: expected several buckets")
        for window in range(2):                                 # two windows: the per-window bookkeeping must reset
            local = _window(ex, rank, 3, group_size, 1000 * window, check)
            want = local.clone()
            dist.all_reduce(want)
            ex.flush()                                          # a complete window: nothing left to exchange
            check(len(ex.handles) == len(ex.buckets), f"{tag}: flush() after the last micro-batch exchanged again")
            ex.wait()
            check(torch.equal(ex.flat_g, want), f"{tag} window {window}: accumulated exchange != all-reduce of the local sum")
        # a fourth micro-batch in a window of three, and a gradient signalled twice within one micro-batch, are refused
        try:
            ex.next_micro_batch()
            check(False, f"{tag}: a micro-batch past the window's end must raise")
        except RuntimeError:
            pass
        ex.reset(1.0, micro_batches=2)
        ex.ready(*ex.order)
        try:
            ex.ready(ex.order[0])
            check(False, f"{tag}: a gradient signalled twice in one micro-batch must raise")
        except RuntimeError:
            pass
        # a partial window (2 of 3 micro-batches) closed by flush(): every bucket exchanged once
        local = torch.zeros_like(ex.flat_g)
        ex.reset(1.0, micro_batches=3)
        for mb in range(2):
            if mb:
                ex.next_micro_batch()
            gr = torch.Generator().manual_seed(7 + 10 * mb + rank)
            for name in ex.order:
                t = torch.randn(ex.g[name].shape, generator=gr)
                ex.g[name].add_(t)
                o = ex.offs[name]
                local[o:o + t.numel()] += t.reshape(-1)
                ex.ready(name)
        check(not ex.launched, f"{tag}: partial window exchanged before flush()")
        ex.flush()
        check(sorted(ex.launched) == list(range(len(ex.buckets))), f"{tag}: flush() did not exchange every bucket once")
        ex.wait()
        dist.all_reduce(local)
        check(torch.equal(ex.flat_g, local), f"{tag}: flushed partial window != all-reduce of the local sum")
    q.put((rank, ok, "; ".join(why)))
    dist.destroy_process_group()


def test_accumulation_window_exchanges_once_and_equals_a_plain_allreduce():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True, ""), (1, True, "")], res


def test_window_of_one_keeps_the_single_step_sequence():
    """N = 1: reset() then ready() exchanges each bucket the moment it completes, as before accumulation existed; flush() has nothing
    to do."""
    ex = GradExchange([("a", (5,)), ("b", (7,)), ("c", (3,))], torch.device("cpu"), bucket_bytes=16)
    ex.reset()
    ex.ready("a")
    assert ex.launched == [0]
    ex.ready("b", "c")
    ex.flush()
    assert ex.launched == [0, 1, 2]
    with pytest.raises(RuntimeError, match="complete"):
        ex.next_micro_batch()
    with pytest.raises(ValueError):
        ex.reset(1.0, micro_batches=0)
