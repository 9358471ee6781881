"""Stopping and continuing both trainers (GPU): what is restored equals what was saved bit for bit — flat weights, Adam moments, counters,
loss scale, EMA buffers, and the operand copies derived from them — through the on-disk containers (Lightning-layout pickle for the
codebook, TF object-graph checkpoint with slot variables for the transformer); a resumed run continues as the uninterrupted one does;
fine-tuning offsets the schedule and nothing else.

A training step is not bit-reproducible on every path (several backward kernels accumulate with atomicAdd), so "resumed == uninterrupted"
is held to what two uninterrupted runs themselves achieve: bitwise if they agree bitwise, else within 4x their largest difference (weights:
element-wise max-abs; reported losses: absolute).  Where the operands are rounded to bf16, a last-bit difference in a master weight can flip
a rounding, and run-to-run differences are then a few rare jumps rather than a noise floor — two runs say little about a third.  There the
bar does not go below 5 % of the distance a weights-only restore (zero moments, counters at 0) ends up at: the resumed run has to sit at
least 20x closer to the uninterrupted one than that restore does, and that restore has to miss the bar."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import synth
from oracle.make_golden import SMALL_VQ, vq_images, keras_adamw_reference
from viewformer_b200.config import MIGTConfig, VQGANConfig

pytestmark = pytest.mark.gpu

VQ_CFG = {"fp32": dict(SMALL_VQ, perceptual_weight=0.0),
          "bf16": dict(ch=128, ch_mult=[1, 2], attn_resolutions=[16], image_size=32, n_embed=256, perceptual_weight=0.0)}
LOC_SCHEDULE = "warmup(cosine(1,0.25,40),4)"
MIGT_CFG = {"fp32": dict(n_layer=2, n_head=4, d_model=128, sequence_size=4, n_loss_skip=1, dropout=0.1, weight_decay=0.01, total_steps=50,
                         learning_rate=1e-3, label_smoothing=0.05, localization_weight=LOC_SCHEDULE, image_generation_weight=0.8, pose_multiplier=1.0),
            "bf16": dict(n_layer=2, n_head=4, d_model=256, token_image_size=8, n_loss_skip=1, dropout=0.1, weight_decay=0.01, total_steps=50,
                         learning_rate=1e-3, label_smoothing=0.05, localization_weight=LOC_SCHEDULE, image_generation_weight=0.8, pose_multiplier=1.0)}
WARMUP = 3


# ----------------------------------------------------------------------------------------------- the bar
def _compare_runs(tag, first, second, resumed, weights_only):
    """Each run: (flat weights after step 5, [loss of step 4, loss of step 5]).  ``first`` / ``second``: two uninterrupted runs."""
    def dist(a, b):
        return float((a[0] - b[0]).abs().max()), max(abs(x - y) for x, y in zip(a[1], b[1]))

    bitwise = torch.equal(first[0], second[0]) and first[1] == second[1]
    dw, dl = dist(first, second)
    ww, wl = dist(weights_only, first)
    bar_w, bar_l = max(4 * dw, 0.05 * ww), max(4 * dl, 0.05 * wl)

    def meets(run):
        if bitwise:
            return torch.equal(run[0], first[0]) and run[1] == first[1]
        w, l = dist(run, first)
        return w <= bar_w and l <= bar_l

    rw, rl = dist(resumed, first)
    print(f"[resume {tag}] two uninterrupted runs {'agree bitwise' if bitwise else f'differ by {dw:.2e} (weights) / {dl:.2e} (losses)'}; resumed run: "
          f"{rw:.2e} / {rl:.2e}; weights-only restore: {ww:.2e} / {wl:.2e}")
    assert meets(resumed), (tag, bitwise, (dw, dl), (rw, rl))
    assert not meets(weights_only), (tag, bitwise, (dw, dl), (ww, wl))


# ----------------------------------------------------------------------------------------------- codebook
def _vq_trainer(precision, quantizer, seed=5):
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    cfg = VQGANConfig(**VQ_CFG[precision])
    sd = synth.make_vqgan_state_dict(cfg, seed)
    if quantizer == "commit":                       # Quantize has no EMA buffers
        sd = {k: v for k, v in sd.items() if not k.startswith("quantize.") or k == "quantize.embeddings"}
    return VQGANTrainer(VQGAN(cfg, precision="fp32", quantizer=quantizer).load_state_dict(sd), precision=precision)


def _vq_batches(precision, n=5):
    return [vq_images(3, VQ_CFG[precision]["image_size"], 2000 + i) for i in range(n)]


def _vq_tail(tr, batches):
    losses = [float(tr.training_step(x)) for x in batches]
    torch.cuda.synchronize()
    return tr.flat_p.clone(), losses[-2:]


def _assert_vq_state_equal(a, b):
    assert torch.equal(a.flat_p, b.flat_p) and torch.equal(a.flat_m, b.flat_m) and torch.equal(a.flat_v, b.flat_v)
    assert (a.step_count, a.lr, tuple(a.betas), a.eps) == (b.step_count, b.lr, tuple(b.betas), b.eps)
    qa, qb = a.model._w["q"], b.model._w["q"]
    for k in ("emb", "et") + (("cs", "dw") if a.model.quantizer == "ema" else ()):
        assert torch.equal(qa[k], qb[k]), k
    if a.model.quantizer == "ema":
        assert qa["counter"] == qb["counter"]
    # |e|^2 is formed with fused multiply-adds by the EMA kernel and with separate multiplies and adds when a codebook is loaded: the two
    # may differ in the last bit.  The lookup settles every near-tie in fp64 from the codebook itself, so the codes do not depend on it.
    assert torch.allclose(qa["esq"], qb["esq"], rtol=1e-6, atol=0)
    assert torch.equal(a.model._w["pq_table"], b.model._w["pq_table"])
    if a.bf16:
        copies = lambda t: [w for cw, _ in t._convs if id(cw) in t._wb16 for w in t._wb16[id(cw)] if w is not None]
        assert len(copies(a)) == len(copies(b)) > 0 and all(torch.equal(x, y) for x, y in zip(copies(a), copies(b)))


@pytest.mark.parametrize("precision,quantizer", [("fp32", "ema"), ("fp32", "commit"), ("bf16", "ema"), ("bf16", "commit")])
def test_vqgan_resume_from_checkpoint(tmp_path, precision, quantizer):
    from viewformer_b200 import VQGAN
    from viewformer_b200.registry import load_model
    batches = _vq_batches(precision)
    first, second = _vq_tail(_vq_trainer(precision, quantizer), batches), _vq_tail(_vq_trainer(precision, quantizer), batches)
    saver = _vq_trainer(precision, quantizer)
    for x in batches[:3]:
        saver.training_step(x)
    path = str(tmp_path / "run" / "last.ckpt")
    saver.save_checkpoint(path, epoch=2)
    ckpt = torch.load(path, map_location="cpu")
    assert ckpt["global_step"] == 3 and ckpt["epoch"] == 2 and set(ckpt["state_dict"]) == set(saver.model.expected_keys())
    assert len(ckpt["optimizer_states"][0]["state"]) == len(saver.params) + sum(1 for p in saver.params if p.part)       # q and k count apiece
    # a fresh model + trainer from the config alone (other initial weights: a restore that does nothing cannot pass)
    cfg = VQGANConfig(**VQ_CFG[precision])
    model = VQGAN(cfg, precision="fp32", quantizer=quantizer, train_precision=precision).init_weights(seed=1)
    resumed = model.configure_optimizers(resume_from_checkpoint=path)
    assert resumed.precision == precision
    _assert_vq_state_equal(saver, resumed)
    xq = vq_images(2, cfg.image_size, 7)
    for got, want in zip(model.encode(xq)[::2], saver.model.encode(xq)[::2]):             # quantized rows and codes, no step taken in between
        assert torch.equal(got, want)
    if quantizer == "ema":                          # the plain loader reads the same file and ignores everything but state_dict
        assert torch.equal(load_model(os.path.dirname(path), precision="fp32").encode(xq)[2], saver.model.encode(xq)[2])
    # weights only: the same weights and EMA buffers, Adam from zero
    plain = _vq_trainer(precision, quantizer, seed=1)
    only = str(tmp_path / "weights" / "last.ckpt")
    os.makedirs(os.path.dirname(only))
    torch.save(dict(state_dict=ckpt["state_dict"]), only)
    with pytest.warns(UserWarning, match="no optimizer state"):
        plain.load_checkpoint(only)
    assert torch.equal(plain.flat_p, saver.flat_p) and plain.step_count == 0 and not bool(plain.flat_m.any())
    _compare_runs(f"vqgan {precision} {quantizer}", first, second, _vq_tail(resumed, batches[3:]), _vq_tail(plain, batches[3:]))


def test_vqgan_mismatched_state_is_refused_before_anything_is_written():
    tr = _vq_trainer("fp32", "ema")
    tr.training_step(_vq_batches("fp32", 1)[0])
    before = [t.clone() for t in (tr.flat_p, tr.flat_m, tr.flat_v)]
    state, sd = tr.optimizer_state(), tr.export_state_dict()
    name = "decoder.conv_in.weight"
    bad = copy.copy(state)
    bad["exp_avg_sq"] = dict(state["exp_avg_sq"], **{name: state["exp_avg_sq"][name][:, :-1]})
    with pytest.raises(RuntimeError, match=name):
        tr.load_optimizer_state(bad)
    short = copy.copy(state)
    short["exp_avg_sq"] = {k: v for k, v in state["exp_avg_sq"].items() if k != "encoder.mid.attn_1.k.bias"}
    with pytest.raises(RuntimeError, match="attn_1.k.bias"):
        tr.load_optimizer_state(short)
    with pytest.raises(RuntimeError, match=name):
        tr.load_state_dict(dict(sd, **{name: sd[name][:, :, :2]}))
    with pytest.raises(RuntimeError, match="unexpected"):
        tr.load_state_dict(dict(sd, extra=torch.zeros(1)))
    with pytest.raises(RuntimeError, match="ema_dw_hidden"):
        tr.load_state_dict({k: v for k, v in sd.items() if k != "quantize.ema_dw_hidden"})
    assert all(torch.equal(a, b) for a, b in zip(before, (tr.flat_p, tr.flat_m, tr.flat_v))) and tr.step_count == 1
    tr.load_optimizer_state(short, strict=False)                                        # non-strict: what is there is loaded
    assert all(torch.equal(a, b) for a, b in zip(before, (tr.flat_p, tr.flat_m, tr.flat_v)))


def test_vqgan_full_size_checkpoint_round_trip(tmp_path):
    """VQGANConfig defaults (346 state tensors, 342 of them trained): one step, save, restore into a fresh trainer."""
    import time
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    cfg = VQGANConfig(perceptual_weight=0.0)
    saver = VQGANTrainer(VQGAN(cfg, precision="fp32").load_state_dict(synth.make_vqgan_state_dict(cfg, 5)))
    saver.training_step(vq_images(2, cfg.image_size, 3000))
    path = str(tmp_path / "last.ckpt")
    t0 = time.time()
    saver.save_checkpoint(path)
    t1 = time.time()
    resumed = VQGAN(cfg, precision="fp32").init_weights(seed=1).configure_optimizers(resume_from_checkpoint=path)
    print(f"[resume vqgan full size] {os.path.getsize(path) / 2**20:.0f} MiB written in {t1 - t0:.1f} s, restored in {time.time() - t1:.1f} s")
    ckpt = torch.load(path, map_location="cpu")
    assert len(ckpt["state_dict"]) == 346 and len(ckpt["optimizer_states"][0]["state"]) == 342
    _assert_vq_state_equal(saver, resumed)


# ----------------------------------------------------------------------------------------------- transformer
def _migt(size, init_seed=None, **compile_kw):
    """(model, trainer) of MIGT_CFG[size] trained in that precision unless ``compile_kw`` says otherwise: synthetic weights, or —
    ``init_seed`` — a model built from the config alone."""
    from viewformer_b200 import MIGT
    cfg = MIGTConfig(**MIGT_CFG[size])
    model = MIGT(cfg, precision="fp32")
    model = model.init_weights(init_seed) if init_seed is not None else model.load_state_dict(synth.make_migt_state_dict(cfg, 9))
    return model, model.compile(**dict(dict(precision=size, warmup_steps=WARMUP, seed=4, bucket_bytes=1 << 18), **compile_kw))


def _migt_batches(precision, n=5):
    from oracle import migt_oracle as mo
    cfg = MIGTConfig(**MIGT_CFG[precision])
    return [(mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(2, 4, seed=60 + i))[0]),
             synth.make_codes(2, 4, n_embed=cfg.n_embeddings, side=cfg.token_image_size, seed=50 + i)) for i in range(n)]


def _migt_tail(model, batches):
    outs = [model.train_step(b) for b in batches]
    torch.cuda.synchronize()
    return model._trainer.flat_p.clone(), [o["loss"] for o in outs[-2:]], outs


def _assert_migt_state_equal(a, b):
    assert torch.equal(a.flat_p, b.flat_p) and torch.equal(a.flat_m, b.flat_m) and torch.equal(a.flat_v, b.flat_v)
    scalars = lambda t: (t.iterations, t.train_counter, t.schedule_offset, t.loss_scale, t.loss_scale_counter, t.seed, t.precision)
    assert scalars(a) == scalars(b)
    if a.bf16:
        assert sorted(a._w16) == sorted(b._w16) and len(a._w16) > 0
        assert all(torch.equal(x, y) for k in a._w16 for x, y in zip(a._w16[k], b._w16[k]))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_migt_resume_from_checkpoint(tmp_path, precision):
    from viewformer_b200 import tf_checkpoint as tfc
    from viewformer_b200.schedules import parse
    batches = _migt_batches(precision)
    first, second = _migt_tail(_migt(precision)[0], batches), _migt_tail(_migt(precision)[0], batches)
    smodel, saver = _migt(precision)
    for b in batches[:3]:
        smodel.train_step(b)
    prefix = str(tmp_path / "run" / "model")
    smodel.save_weights(prefix, include_optimizer=True)
    ck = tfc.Checkpoint(prefix)
    owner = "optimizer/base_optimizer" if precision == "bf16" else "optimizer"
    assert int(ck.tensor(ck.resolve(owner + "/iter"))) == 3 and ck.slot("ln_f/gamma", "m", owner) and ck.slot("wpe", "v", owner)
    rmodel, resumed = _migt(precision, init_seed=1, seed=0)                   # config alone; the dropout seed too comes from the file
    rmodel.load_weights(prefix).expect_partial()
    _assert_migt_state_equal(saver, resumed)
    assert rmodel._train_counter == 3 and resumed.iterations == 3
    inputs = dict(input_ids=batches[4][1], poses=batches[4][0])
    assert torch.equal(rmodel(inputs)["logits"], smodel(inputs)["logits"])     # inference with the restored weights, no step taken in between
    # weights only: a file without optimizer entries leaves the compiled optimizer as it is
    weights = str(tmp_path / "weights" / "model")
    smodel.save_weights(weights)
    pmodel, plain = _migt(precision, init_seed=1)
    pmodel.load_weights(weights)
    assert torch.equal(plain.flat_p, saver.flat_p) and plain.iterations == 0 and not bool(plain.flat_m.any())
    r = _migt_tail(rmodel, batches[3:])
    # dropout masks and the schedules carry on: step 4 runs at the rate, localisation weight and loss scale of step 4, not of step 1
    sched = parse(LOC_SCHEDULE).with_total_steps(50)
    assert r[2][0]["learning_rate"] == first[2][3]["learning_rate"] == 1e-3 and first[2][0]["learning_rate"] == 0.0
    assert resumed.loc_weight == float(sched(5)) != float(sched(2)) and resumed.iterations == 5
    if precision == "bf16":
        assert r[2][0]["loss_scale"] == first[2][3]["loss_scale"]
    _compare_runs(f"migt {precision}", first[:2], second[:2], r[:2], _migt_tail(pmodel, batches[3:])[:2])


def test_migt_loss_scale_state_survives(tmp_path):
    """A halved loss scale and its good-step counter come back; state of the other precision loads with the scale at its default."""
    model, tr = _migt("bf16")
    batches = _migt_batches("bf16", 2)
    model.train_step(batches[0])
    tr.forward_backward(*batches[1])
    tr.flat_g[0] = float("inf")                      # a host-side write: the finiteness check sees an overflowed gradient
    assert not tr.optimizer_step()
    model.train_step(batches[1])
    assert (tr.loss_scale, tr.loss_scale_counter, tr.iterations) == (2.0 ** 14, 1, 3)
    prefix = str(tmp_path / "model")
    model.save_weights(prefix, include_optimizer=True)
    rmodel, resumed = _migt("bf16", init_seed=1)
    rmodel.load_weights(prefix)
    assert (resumed.loss_scale, resumed.loss_scale_counter, resumed.iterations) == (2.0 ** 14, 1, 3)
    _assert_migt_state_equal(tr, resumed)
    _, as_fp32 = _migt("bf16", init_seed=1, precision="fp32")
    as_fp32.model.load_weights(prefix)
    assert (as_fp32.loss_scale, as_fp32.loss_scale_counter, as_fp32.iterations) == (1.0, 0, 3) and torch.equal(as_fp32.flat_m, tr.flat_m)
    back = resumed.load_optimizer_state(as_fp32.optimizer_state())
    assert (back.loss_scale, back.loss_scale_counter) == (2.0 ** 15, 0) and torch.equal(back.flat_v, tr.flat_v)


def test_migt_finetune_offsets_the_schedule_and_nothing_else(tmp_path):
    """finetune_transformer.py:72-86: new peak rate and horizon, warm-up from the restored ``iterations``; Adam's bias correction carries
    on from ``iterations`` (one tensor's update against the restated Keras AdamWeightDecay at step = iterations + 1)."""
    from viewformer_b200 import MIGT
    batches = _migt_batches("fp32")
    smodel, saver = _migt("fp32")
    for b in batches[:3]:
        smodel.train_step(b)
    prefix = str(tmp_path / "model")
    smodel.save_weights(prefix, include_optimizer=True)
    cfg = MIGTConfig(**MIGT_CFG["fp32"])
    model = MIGT(cfg, precision="fp32")
    new_lr, new_warm = 4e-4, 4
    tr = model.finetune(prefix, learning_rate=new_lr, total_steps=20, warmup_steps=new_warm, bucket_bytes=1 << 18)
    assert tr.schedule_offset == tr.iterations == 3 and tr.train_counter == 0 and model._train_counter == 0 and tr.seed == saver.seed
    assert torch.equal(tr.flat_p, saver.flat_p) and torch.equal(tr.flat_m, saver.flat_m) and torch.equal(tr.flat_v, saver.flat_v)
    assert tr.learning_rate() == 0.0 and tr.loc_weight == float(saver._loc_schedule(0)) != saver.loc_weight
    key = "h.1.mlp.c_fc.weight"
    for j in range(3):
        assert tr.learning_rate() == new_lr * j / new_warm
        tr.forward_backward(*batches[3 + j % 2])
        tr.ex.wait()
        p, m, v, g = ({key: t[key].clone()} for t in (tr.state_dict(), tr.optimizer_state()["m"], tr.optimizer_state()["v"], tr.gradients()))
        wrong = {key: p[key].clone()}
        keras_adamw_reference(p, g, {key: m[key].clone()}, {key: v[key].clone()}, tr.iterations + 1, tr.learning_rate(), cfg.weight_decay)
        keras_adamw_reference(wrong, g, m, v, tr.iterations - tr.schedule_offset + 1, tr.learning_rate(), cfg.weight_decay)
        assert tr.optimizer_step()
        got = tr.state_dict()[key]
        err, off = float((got - p[key]).abs().max()), float((got - wrong[key]).abs().max())
        print(f"[finetune step {j}] lr {new_lr * j / new_warm:.1e}: update vs AdamW at step iterations+1: {err:.2e}; at step since the offset: {off:.2e}")
        assert err <= 2e-7 and (j == 0 or off > 20 * err)
    assert (tr.iterations, tr.train_counter, tr.schedule_offset) == (6, 3, 3)
    # a file without optimizer entries: fine-tuning starts fresh, with a warning
    weights = str(tmp_path / "weights")
    smodel.save_weights(weights)
    with pytest.warns(UserWarning, match="no optimizer entries"):
        fresh = MIGT(cfg, precision="fp32").finetune(weights, learning_rate=new_lr, total_steps=20)
    assert fresh.iterations == fresh.schedule_offset == 0 and torch.equal(fresh.flat_p, saver.flat_p)


def test_migt_mismatched_state_is_refused_before_anything_is_written():
    model, tr = _migt("fp32")
    model.train_step(_migt_batches("fp32", 1)[0])
    model.train_step(_migt_batches("fp32", 1)[0])
    before = [t.clone() for t in (tr.flat_p, tr.flat_m, tr.flat_v)]
    state = tr.optimizer_state()
    bad = dict(state, v=dict(state["v"], **{"ln_f.gamma": torch.zeros(129)}))
    with pytest.raises(RuntimeError, match="ln_f.gamma"):
        tr.load_optimizer_state(bad)
    short = dict(state, m={k: v for k, v in state["m"].items() if k != "wpe.embeddings"})
    with pytest.raises(RuntimeError, match="wpe.embeddings"):
        tr.load_optimizer_state(short)
    with pytest.raises(RuntimeError, match="iterations"):
        tr.load_optimizer_state({k: v for k, v in state.items() if k != "iterations"})
    with pytest.raises(RuntimeError, match="ln_f.gamma"):
        tr.load_state_dict(dict(tr.state_dict(), **{"ln_f.gamma": torch.zeros(3)}))
    assert all(torch.equal(a, b) for a, b in zip(before, (tr.flat_p, tr.flat_m, tr.flat_v))) and tr.iterations == 2
    tr.load_optimizer_state(short, strict=False)
    assert all(torch.equal(a, b) for a, b in zip(before, (tr.flat_p, tr.flat_m, tr.flat_v)))


def test_migt_full_size_state_round_trip():
    """MIGTConfig defaults (156 tensors): one bf16 step, then the whole state into a fresh trainer, in memory (the TF container's pure-Python
    checksums make a full-size file a matter of minutes; its layout is covered at small sizes)."""
    from viewformer_b200 import MIGT
    from oracle import migt_oracle as mo
    cfg = MIGTConfig(dropout=0.1, total_steps=100, learning_rate=1e-4)
    smodel = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 13))
    saver = smodel.compile(precision="bf16", warmup_steps=1)
    batch = (mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(1, 5, seed=71))[0]), synth.make_codes(1, 5, n_embed=cfg.n_embeddings, seed=70))
    smodel.train_step(batch)
    smodel.train_step(batch)
    state = saver.optimizer_state()
    assert len(state["m"]) == len(state["v"]) == len(saver.state_dict()) == 156
    assert sum(t.numel() for t in state["m"].values()) == sum(math_prod(s) for s in smodel.param_shapes().values())
    rmodel = MIGT(cfg, precision="fp32").init_weights(1)
    resumed = rmodel.compile(precision="bf16", warmup_steps=1)
    resumed.load_state_dict(saver.state_dict()).load_optimizer_state(state)
    _assert_migt_state_equal(saver, resumed)


def math_prod(shape):
    return int(np.prod(shape)) if len(shape) else 1
