"""world_size-2 gloo tests (CPU) of the multi-GPU host logic: scene sharding, the packed EMA all-reduce, and the bucketed gradient
exchange shared by the two trainers (driven on CPU tensors with each trainer's real parameter list)."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from viewformer_b200.dist import shard_range, allreduce_ema_stats, max_over_ranks


def test_shard_range_partitions_exactly():
    for n in (0, 1, 7, 64, 65):
        for world in (1, 2, 3, 8):
            spans = [shard_range(n, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g = torch.Generator().manual_seed(100 + rank)
    counts = torch.randint(0, 5, (32,), generator=g).float()
    esum = torch.randn((8, 32), generator=g)
    # reference pattern: two all-reduces (utils_th.py:50-52)
    c2, e2 = counts.clone(), esum.clone()
    dist.all_reduce(c2)
    dist.all_reduce(e2)
    c1, e1 = allreduce_ema_stats(counts, esum)
    ok = torch.equal(c1, c2) and torch.allclose(e1, e2, atol=0, rtol=0)
    ok = ok and c1.shape == counts.shape and e1.shape == esum.shape
    ok = ok and max_over_ranks(float(rank + 1), "cpu") == float(world)
    lo, hi = shard_range(7, rank, world)
    tot = torch.tensor([hi - lo])
    dist.all_reduce(tot)
    ok = ok and int(tot) == 7
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_packed_ema_allreduce_equals_reference_two_call_pattern():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


# ---------------------------------------------------------------------------------------- gradient buckets of the two trainers
def _bucket_worker(rank, world, port, q):
    """Drives the shared gradient exchange (dist.GradExchange) as each trainer builds it (VQGANTrainer._flatten, MIGTTrainer._build) on
    CPU tensors over gloo: the kernels are not involved, only the host logic of the exchange — flat buffer layout in backward order,
    bucket boundaries, an async all-reduce launched the moment a bucket's last gradient is signalled, SUM semantics
    (train_codebook_th.py:39-41 DDP; migt.py:471-476 MirroredStrategy)."""
    from types import SimpleNamespace
    from viewformer_b200.train import VQGANTrainer, _P
    from viewformer_b200.train_migt import MIGTTrainer
    from viewformer_b200 import MIGT
    from viewformer_b200.config import MIGTConfig
    from oracle import synth
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ok, why = True, []

    def check(cond, msg):
        nonlocal ok
        if not cond:
            ok = False
            why.append(msg)

    # ---- codebook trainer: 9 tensors of odd sizes (padding to 16-byte views), 4 KiB buckets
    g = torch.Generator().manual_seed(5)
    shapes = [(3, 3, 7, 5), (5,), (33, 17), (17,), (1,), (64, 9), (9,), (1023,), (2, 2)]
    homes = {}
    params = [_P(f"p{i}", torch.randn(s, generator=g), (lambda v, i=i: homes.__setitem__(i, v)), "conv") for i, s in enumerate(shapes)]
    originals = [p.tensor.clone() for p in params]
    tr = VQGANTrainer.__new__(VQGANTrainer)
    tr.model = SimpleNamespace(device=torch.device("cpu"), _refresh_decode_table=lambda: None)
    tr.params, tr.bucket_bytes, tr.group = params, 4096, None
    tr._flatten()
    ex = tr.ex
    check(len(tr.buckets) >= 3, f"expected several buckets, got {tr.buckets}")
    check(tr.buckets[0][0] == 0 and tr.buckets[-1][1] == ex.flat_g.numel() and all(a[1] == b[0] for a, b in zip(tr.buckets, tr.buckets[1:])),
          "buckets do not partition the flat gradient")
    check(ex.order == [f"p{i}" for i in reversed(range(len(shapes)))], "flat buffer is not in backward order")
    check(all(torch.equal(homes[i], originals[i]) and homes[i].data_ptr() == params[i].tensor.data_ptr() == ex.p[f"p{i}"].data_ptr()
              for i in range(len(shapes))), "parameters were not re-homed into the flat buffer")
    check(all(ex.offs[p.name] % 4 == 0 for p in params), "views are not 16-byte aligned")
    for step in range(2):                                            # two steps: the per-step bookkeeping must reset
        ex.reset()
        gr = torch.Generator().manual_seed(1000 * step + rank)
        for name in ex.order:                                        # "backward": gradients complete in flat-buffer order
            ex.g[name].copy_(torch.randn(ex.g[name].shape, generator=gr))
        want = ex.flat_g.clone()
        dist.all_reduce(want)                                        # what one big all-reduce after backward would give
        ex.flat_g.zero_()
        gr = torch.Generator().manual_seed(1000 * step + rank)
        seen = 0
        for name in ex.order:
            ex.g[name].copy_(torch.randn(ex.g[name].shape, generator=gr))
            ex.ready(name)
            check(len(ex.handles) == len(ex.launched) >= seen, "handle bookkeeping")
            seen = len(ex.launched)
        check(not any(ex._left) and ex.launched == list(range(len(tr.buckets))), "buckets not launched in completion order")
        ex.check_complete()
        ex.wait()
        check(not ex.handles, "wait() leaves handles behind")
        check(torch.equal(ex.flat_g, want), f"codebook trainer: bucketed exchange != plain all-reduce (step {step})")
    try:
        ex.ready(ex.order[0])
        check(False, "a gradient signalled twice must raise")
    except RuntimeError:
        pass

    # ---- transformer trainer: the real parameter list of a 2-layer MIGT, 32 KiB buckets
    cfg = MIGTConfig(n_layer=2, n_head=4, d_model=64, sequence_size=4, n_embeddings=32, token_image_size=4)
    model = MIGT(cfg, precision="fp32")
    sd = synth.make_migt_state_dict(cfg, 3)
    mt = MIGTTrainer.__new__(MIGTTrainer)
    mt.model, mt.cfg, mt.device, mt.bucket_bytes, mt.group = model, cfg, torch.device("cpu"), 32 << 10, None
    mt._build(sd)
    ex = mt.ex
    names = list(model.param_shapes().keys())
    check(sorted(ex.order) == sorted(names) and ex.order[-1] == "wte.weight" and ex.order[0].split(".")[0] in ("pose_loss_weighting_criterion", "pose_classifier", "ln_f"),
          "transformer flat buffer is not in backward-completion order")
    check(len(ex.buckets) >= 3 and ex.buckets[0][0] == 0 and ex.buckets[-1][1] == ex.flat_g.numel()
          and all(a[1] == b[0] for a, b in zip(ex.buckets, ex.buckets[1:])), "transformer buckets do not partition the flat gradient")
    check(all(torch.equal(mt.p[k], sd[k].float()) for k in names), "transformer parameters not copied into the flat buffer")
    check(all(mt.decay[k] == ("bias" not in k) for k in names), "weight-decay mask")
    ex.reset()
    gr = torch.Generator().manual_seed(77 + rank)
    for k in ex.order:
        mt.g[k].copy_(torch.randn(mt.g[k].shape, generator=gr))
    want = ex.flat_g.clone()
    dist.all_reduce(want)
    i = 0
    while i < len(ex.order):                                         # the step signals groups of names at once (e.g. weight + bias)
        ex.ready(*ex.order[i:i + 3])
        i += 3
    check(not any(ex._left) and sorted(ex.launched) == list(range(len(ex.buckets))), "transformer buckets incomplete")
    ex.wait()
    check(torch.equal(ex.flat_g, want), "transformer trainer: bucketed exchange != plain all-reduce")
    q.put((rank, ok, "; ".join(why)))
    dist.destroy_process_group()


def test_shared_gradient_exchange_of_both_trainers_equals_a_plain_allreduce():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_bucket_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True, ""), (1, True, "")], res
