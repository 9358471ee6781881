"""Gradient accumulation in both trainers (GPU): a window of N micro-batches equals the sum of their single-micro-batch gradients (divided by
N for the codebook, as Lightning divides the loss), the one update per window equals Adam / Keras AdamWeightDecay applied in fp64 on the
host to that gradient, every gradient producer adds rather than overwrites, the window's memory peak is one micro-batch's, the bf16 loss
scaler runs once per window, and a run saved at a window boundary resumes as the uninterrupted one.

Two runs of the same step are not bit-identical (several backward kernels accumulate with atomicAdd), so gradients are compared per
tensor against the tensor's largest element; the measured differences are printed."""
import numpy as np
import pytest
import torch

from oracle import synth
from oracle.make_golden import SMALL_VQ, vq_images, keras_adamw_reference
from viewformer_b200.config import MIGTConfig, VQGANConfig

pytestmark = pytest.mark.gpu

VQ_CFG = {"fp32": dict(SMALL_VQ, perceptual_weight=0.0),
          "bf16": dict(ch=128, ch_mult=[1, 2], attn_resolutions=[16], image_size=32, n_embed=256, perceptual_weight=0.0)}
MIGT_CFG = dict(n_layer=2, n_head=4, d_model=256, token_image_size=8, n_loss_skip=1, dropout=0.1, weight_decay=0.01, total_steps=50,
                learning_rate=1e-3, label_smoothing=0.05, localization_weight="warmup(cosine(1,0.25,40),4)", image_generation_weight=0.8,
                pose_multiplier=1.0, use_dynamic_pose_loss=True)
WKEY = "pose_loss_weighting_criterion.pos_ori_weights"


def _worst(got, want, floor=0.0):
    """max over tensors of max |got - want| / max(max |want|, floor), with the tensor's name; tensors whose gradient is zero are skipped."""
    return max((float((got[k].double() - want[k].double()).abs().max() / max(float(want[k].double().abs().max()), floor)), k)
               for k in want if float(want[k].abs().max()) > 0)


def _within_rounding(got, want, noise):
    """max over tensors of max |got - want| / (4 max |noise| + 1e-4 max |want|): ``noise`` is the difference of two runs of the same
    step, so a tensor whose true gradient is zero (a conv bias feeding a GroupNorm, the attention's key bias) is held to its rounding."""
    return max((float((got[k].double() - want[k].double()).abs().max()
                      / (4 * float(noise[k].double().abs().max()) + 1e-4 * float(want[k].double().abs().max()))), k)
               for k in want if float(want[k].abs().max()) > 0)


def _norm_projection(got, want, seed=99):
    """tests/test_train_gpu.py's per-tensor measure: norm and a random projection, relative to the norm (floor 1e-4); [(error, name)]."""
    gen = torch.Generator().manual_seed(seed)
    errs = []
    for k in want:
        pr = torch.randn(tuple(want[k].shape), generator=gen, dtype=torch.float64)
        gn, rn = float(got[k].double().norm()), float(want[k].double().norm())
        gd, rd = float((got[k].double() * pr).sum()), float((want[k].double() * pr).sum())
        errs.append((max(abs(gn - rn), abs(gd - rd)) / max(rn, 1e-4), k))
    return errs


def _vq_gradients_agree(tag, got, want, precision, second=None):
    """Two runs of the codebook step held to each other.  fp32: tests/test_train_gpu.py's bars — element-wise 2e-3 of the tensor's largest
    element (floor 1e-4: conv biases that feed a GroupNorm and the attention's key biases have an exactly-zero true gradient, so both sides
    hold rounding noise there) and 3e-3 on norm and projection.  bf16: tests/test_train_bf16_gpu.py's bars on norm and projection — worst
    1e-1, median 1e-2 — or, when ``second`` (another run of what ``want`` ran) differs from ``want`` by more, 4x that difference: a
    last-bit difference upstream (the EMA statistics are summed with atomics) flips bf16 operand roundings, and those differences grow
    through the layers.  An overwritten gradient would be off by half."""
    errs = _norm_projection(got, want)
    worst, med = max(errs), float(np.median([e for e, _ in errs]))
    elem = _worst(got, want, floor=1e-4)
    bar_w, bar_m = 1e-1, 1e-2
    if second is not None:
        errs2 = _norm_projection(second, want)
        bar_w, bar_m = max(bar_w, 4 * max(errs2)[0]), max(bar_m, 4 * float(np.median([e for e, _ in errs2])))
    print(f"[{tag}] gradients: worst element {elem[0]:.2e} ({elem[1]}); norm / projection worst {worst[0]:.2e} ({worst[1]}), median {med:.2e}"
          + ("" if second is None else f"; a second run: worst {max(errs2)[0]:.2e}, median {float(np.median([e for e, _ in errs2])):.2e}"))
    if precision == "fp32":
        assert elem[0] < 2e-3 and worst[0] < 3e-3, (elem, worst)
    else:
        assert worst[0] <= bar_w and med <= bar_m, (worst, med, bar_w, bar_m)


# ----------------------------------------------------------------------------------------------- codebook
def _vq_trainer(precision, quantizer, n=1, **cfg_kw):
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    cfg = VQGANConfig(**dict(VQ_CFG[precision], **cfg_kw))
    sd = synth.make_vqgan_state_dict(cfg, 5)
    if quantizer == "commit":                       # Quantize has no EMA buffers
        sd = {k: v for k, v in sd.items() if not k.startswith("quantize.") or k == "quantize.embeddings"}
    return VQGANTrainer(VQGAN(cfg, precision="fp32", quantizer=quantizer).load_state_dict(sd), precision=precision, accumulate_grad_batches=n,
                        bucket_bytes=1 << 16)


def _adam_fp64(p, g, lr, betas, eps, clip):
    """torch.optim.Adam's first step (zero moments) in fp64, after Lightning's global-norm clip when ``clip`` > 0."""
    g = g.double()
    if clip > 0:
        g = g * min(1.0, clip / (float(g.norm()) + 1e-6))
    m, v = (1 - betas[0]) * g, (1 - betas[1]) * g * g
    return p.double() - lr * (m / (1 - betas[0])) / ((v / (1 - betas[1])).sqrt() + eps)


@pytest.mark.parametrize("precision,quantizer", [("fp32", "ema"), ("fp32", "commit"), ("bf16", "ema"), ("bf16", "commit")])
def test_vqgan_window_equals_mean_of_micro_batch_gradients(precision, quantizer):
    """accumulate_grad_batches=2 over micro-batches A, B == a trainer with N = 1 from the same state running forward_backward(A), then
    forward_backward(B) (the EMA codebook moved by A in both): gradient (g_A + g_B) / 2 at the bars between two runs
    (``_vq_gradients_agree``), the same codes and losses; no step after A, one after B, and that step equals Adam in fp64 on the window's
    gradient (clipped with the commitment quantizer: clip = half the gradient's norm)."""
    size = VQ_CFG[precision]["image_size"]
    xa, xb = vq_images(3, size, 2000), vq_images(3, size, 2001)
    one = _vq_trainer(precision, quantizer)
    la = float(one.forward_backward(xa))
    ga, codes_a = one.export_gradients(), one.last["codes"].clone()
    lb = float(one.forward_backward(xb))
    gb, codes_b = one.export_gradients(), one.last["codes"].clone()
    want = {k: (ga[k] + gb[k]) / 2 for k in ga}
    clip = 0.5 * float(torch.sqrt(sum((t.double() ** 2).sum() for t in want.values()))) if quantizer == "commit" else 0.0
    acc = _vq_trainer(precision, quantizer, n=2, gradient_clip_val=clip)
    p0 = acc.flat_p.clone()
    got_a = float(acc.training_step(xa))
    assert acc.step_count == 0 and acc.pending == 1 and torch.equal(acc.flat_p, p0) and not acc.launched
    assert torch.equal(acc.last["codes"], codes_a)
    got_b = float(acc.training_step(xb))
    torch.cuda.synchronize()
    assert acc.step_count == 1 and acc.pending == 0 and sorted(acc.launched) == list(range(len(acc.buckets)))
    assert torch.equal(acc.last["codes"], codes_b)
    # the EMA statistics of A are summed with atomics, so the codebook B is quantised against differs in the last bits between the two
    # trainers; the bf16 step's operand roundings carry that into B's loss
    bar = 1e-6 if precision == "fp32" else 1e-3
    assert abs(got_a - la) <= bar * abs(la) and abs(got_b - lb) <= bar * abs(lb), (got_a, la, got_b, lb)
    second = None
    if precision == "bf16":                         # how far two N = 1 runs of A, B land from each other
        two = _vq_trainer(precision, quantizer)
        two.forward_backward(xa)
        g2a = two.export_gradients()
        two.forward_backward(xb)
        second = {k: (g2a[k] + t) / 2 for k, t in two.export_gradients().items()}
    _vq_gradients_agree(f"vqgan window {precision} {quantizer}: vs (g_A + g_B) / 2", acc.export_gradients(), want, precision, second)
    step = _adam_fp64(p0, acc.flat_g, acc.lr, acc.betas, acc.eps, clip)
    dp = (acc.flat_p.double() - step).abs()
    bar = 4 * torch.finfo(torch.float32).eps * step.abs() + 1e-4 * acc.lr
    print(f"[vqgan window {precision} {quantizer}] post-Adam weights vs fp64 (clip {clip:.3g}): worst {float((dp / bar).max()):.2f} of the bar")
    assert bool((dp <= bar).all())


def test_vqgan_accumulation_surface():
    """configure_optimizers(accumulate_grad_batches=3): two of three micro-batches pending -> save_checkpoint refuses; optimizer_step()
    flushes the partial window (step count 1); a new window then runs to its third micro-batch."""
    from viewformer_b200 import VQGAN
    cfg = VQGANConfig(**VQ_CFG["fp32"])
    model = VQGAN(cfg, precision="fp32").load_state_dict(synth.make_vqgan_state_dict(cfg, 5))
    tr = model.configure_optimizers(accumulate_grad_batches=3)
    assert tr.accumulate_grad_batches == 3
    xs = [vq_images(2, cfg.image_size, 3000 + i) for i in range(5)]
    model.training_step(xs[0])
    model.training_step(xs[1])
    assert tr.pending == 2 and tr.step_count == 0
    with pytest.raises(RuntimeError, match="pending"):
        tr.save_checkpoint("/nonexistent/never-written.ckpt")
    p0 = tr.flat_p.clone()
    tr.optimizer_step()
    assert tr.step_count == 1 and tr.pending == 0 and not torch.equal(tr.flat_p, p0)
    for i, x in enumerate(xs[2:]):
        model.training_step(x)
        assert tr.step_count == (2 if i == 2 else 1)
    with pytest.raises(ValueError):
        model.configure_optimizers(accumulate_grad_batches=0)


# ----------------------------------------------------------------------------------------------- transformer
def _migt_trainers(precision, ns=(1, 2), **cfg_kw):
    from viewformer_b200 import MIGT
    from viewformer_b200.train_migt import MIGTTrainer
    cfg = MIGTConfig(**dict(MIGT_CFG, **cfg_kw))
    sd = synth.make_migt_state_dict(cfg, 9)
    sd[WKEY] = torch.tensor([0.3, -1.2])
    model = MIGT(cfg, precision="fp32").load_state_dict(sd)
    return cfg, [MIGTTrainer(model, precision=precision, seed=4, warmup_steps=3, bucket_bytes=1 << 18, accumulate_steps=n) for n in ns]


def _migt_batch(cfg, B, T, seed):
    from oracle import migt_oracle as mo
    return (mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=seed + 1))[0]),
            synth.make_codes(B, T, n_embed=cfg.n_embeddings, side=cfg.token_image_size, seed=seed))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_migt_window_equals_sum_of_micro_batch_gradients(precision):
    """accumulate_steps=2 over micro-batches A, B (dropout 0.1, localisation on, dynamic pose weights on) == the sum of two N = 1
    forward_backward calls at the same ``iterations`` (the same dropout masks, learning rate and localisation weight): per tensor within
    4e-6 of its largest element (test_train_migt_bf16_gpu.py's bar between two runs).  One update after B, equal to Keras
    AdamWeightDecay on that sum."""
    cfg, (one, acc) = _migt_trainers(precision)
    for t in (one, acc):
        t.iterations = 5                                  # past the warm-up: lr > 0, the localisation weight schedule moving
    ba, bb = _migt_batch(cfg, 2, 4, 40), _migt_batch(cfg, 2, 4, 50)
    la = float(one.forward_backward(*ba))
    ga = one.gradients()
    lb = float(one.forward_backward(*bb))
    gb = one.gradients()
    want = {k: ga[k] + gb[k] for k in ga}
    p0, flat0, lr, ls = acc.state_dict(), acc.flat_p.clone(), acc.learning_rate(), acc.loss_scale
    oa = acc.train_step(ba)
    assert not oa["applied"] and oa["pending"] == 1 and acc.iterations == 5 and torch.equal(acc.flat_p, flat0)
    ob = acc.train_step(bb)
    torch.cuda.synchronize()
    assert ob["applied"] and ob["pending"] == 0 and acc.iterations == 6 and oa["learning_rate"] == ob["learning_rate"] == lr
    assert abs(oa["loss"] - la) <= 1e-6 * abs(la) and abs(ob["loss"] - lb) <= 1e-6 * abs(lb)
    got = acc.gradients()
    elem = _worst(got, want)
    print(f"[migt window {precision}] gradient vs g_A + g_B: worst element {elem[0]:.2e} ({elem[1]}); dynamic pose weights "
          f"{got[WKEY].tolist()} vs {want[WKEY].tolist()}")
    assert elem[0] <= 4e-6, elem
    params = {k: v.double() for k, v in p0.items()}
    m = {k: torch.zeros_like(v) for k, v in params.items()}
    v = {k: torch.zeros_like(t) for k, t in params.items()}
    keras_adamw_reference(params, {k: got[k].double() / ls for k in got}, m, v, 6, lr, cfg.weight_decay)
    after = acc.state_dict()
    worst = max(float(((after[k].double() - params[k]).abs() / (2e-7 + 4 * torch.finfo(torch.float32).eps * params[k].abs())).max())
                for k in params)
    print(f"[migt window {precision}] post-step weights vs Keras AdamWeightDecay in fp64: worst {worst:.2f} of the bar")
    assert worst <= 1.0


# ----------------------------------------------------------------------------------------------- audit: every producer adds
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_every_gradient_producer_accumulates(precision):
    """The same micro-batch twice in one window, dropout 0: the window's gradient is twice each pass's contribution, tensor by tensor — for
    the codebook (commitment quantizer, so the codebook stays put; the seeds halved) the single-pass gradient, at the bars between two
    runs; for the transformer (dynamic pose weights on) twice it, within 4x the difference of two single-pass runs plus 1e-4 of the
    tensor's largest element.  A producer that overwrote its gradient instead of adding would be off by half."""
    # codebook
    one, acc = _vq_trainer(precision, "commit"), _vq_trainer(precision, "commit", n=2)
    x = vq_images(3, VQ_CFG[precision]["image_size"], 2000)
    one.forward_backward(x)
    want = one.export_gradients()
    acc.forward_backward(x)
    acc.forward_backward(x)
    torch.cuda.synchronize()
    assert acc.pending == 2 and sorted(acc.launched) == list(range(len(acc.buckets)))
    _vq_gradients_agree(f"accumulation audit {precision}, codebook", acc.export_gradients(), want, precision)
    # transformer
    cfg, (one, acc) = _migt_trainers(precision, dropout=0.0)
    b = _migt_batch(cfg, 2, 4, 60)
    one.forward_backward(*b)
    g1 = one.gradients()
    one.forward_backward(*b)
    want, noise = {k: 2 * t for k, t in g1.items()}, {k: 2 * (t - g1[k]) for k, t in one.gradients().items()}
    acc.forward_backward(*b)
    acc.forward_backward(*b)
    torch.cuda.synchronize()
    tf = _within_rounding(acc.gradients(), want, noise)
    print(f"[accumulation audit {precision}, transformer] worst difference / (4 x two-run difference + 1e-4 max|g|): {tf[0]:.2e} ({tf[1]})")
    assert tf[0] <= 1.0, tf


def test_vq_commit_grad_accumulate_mode():
    """vf_vq_commit_grad with accumulate=1 adds coef (count_k e_k - esum) to what the buffer holds, element for element what a plain
    fp32 add of the overwrite result gives; accumulate=0 overwrites."""
    from viewformer_b200 import _lib as L
    g = torch.Generator().manual_seed(4)
    D, K, M = 16, 64, 500
    emb, z = torch.randn((D, K), generator=g).cuda(), torch.randn((M, D), generator=g).cuda()
    idx = torch.randint(0, K, (M,), generator=g).cuda()
    counts, zsum = L.vq_ema_stats(z, idx, K)
    fresh = L.vq_commit_grad(emb, counts, zsum, 0.37, torch.full((D, K), float("nan"), device="cuda"))
    base = torch.randn((D, K), generator=g).cuda()
    acc = L.vq_commit_grad(emb, counts, zsum, 0.37, base.clone(), accumulate=True)
    assert torch.isfinite(fresh).all() and torch.equal(acc, base + fresh)


# ----------------------------------------------------------------------------------------------- memory
def _peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_window_memory_is_one_micro_batch():
    """The peak of a window of 4 x 8 images is within 64 MB of an 8-image step and well below a 32-image step (VQGANConfig defaults, bf16);
    the transformer's window of 2 x 5 scenes (fp32, T = 8) likewise against 5 and 10 scenes."""
    from viewformer_b200 import VQGAN, MIGT
    from viewformer_b200.train import VQGANTrainer
    from viewformer_b200.train_migt import MIGTTrainer
    MB = 1 << 20
    cfg = VQGANConfig(perceptual_weight=0.0)
    one = VQGANTrainer(VQGAN(cfg, precision="fp32").init_weights(0), precision="bf16")
    acc = VQGANTrainer(VQGAN(cfg, precision="fp32").init_weights(0), precision="bf16", accumulate_grad_batches=4)
    x8 = [vq_images(8, cfg.image_size, 10 + i) for i in range(4)]
    x32 = torch.cat(x8)
    one.training_step(x8[0])                                # warm-up: operand buffers of the 8-image shapes
    win = _peak(lambda: [acc.training_step(x) for x in x8])
    p8 = _peak(lambda: one.training_step(x8[0]))
    p32 = _peak(lambda: one.training_step(x32))
    assert acc.step_count == 1
    cfg_t = MIGTConfig(**dict(MIGT_CFG, use_dynamic_pose_loss=False))
    mt = MIGT(cfg_t, precision="fp32").init_weights(0)
    t1, t2 = MIGTTrainer(mt), MIGTTrainer(mt, accumulate_steps=2)
    b5 = [_migt_batch(cfg_t, 5, 8, 70 + 10 * i) for i in range(2)]
    b10 = (np.concatenate([b5[0][0], b5[1][0]]), np.concatenate([b5[0][1], b5[1][1]]))
    t1.train_step(b5[0])
    twin = _peak(lambda: [t2.train_step(b) for b in b5])
    t5 = _peak(lambda: t1.train_step(b5[0]))
    t10 = _peak(lambda: t1.train_step(b10))
    print(f"[window memory] codebook: window 4 x 8 {win / MB:.0f} MB, step of 8 {p8 / MB:.0f} MB, of 32 {p32 / MB:.0f} MB; transformer: "
          f"window 2 x 5 {twin / MB:.0f} MB, step of 5 {t5 / MB:.0f} MB, of 10 {t10 / MB:.0f} MB")
    assert win <= p8 + 64 * MB and win <= p32 - (p32 - p8) / 2
    assert twin <= t5 + 64 * MB and twin <= t10 - (t10 - t5) / 2


# ----------------------------------------------------------------------------------------------- bf16 loss scaling and state
def test_migt_bf16_loss_scale_runs_once_per_window():
    """A non-finite micro-batch (one NaN pose) in a window of 2: the whole window is skipped (weights, m, v unchanged bit for bit), the scale
    halves once, ``iterations`` advances by 1.  A window under a huge loss scale (its seeds overflow fp32) likewise.  The next finite
    window applies and counts one good step."""
    cfg, (acc,) = _migt_trainers("bf16", ns=(2,))
    acc.iterations = 5
    ba, bb = _migt_batch(cfg, 2, 4, 40), _migt_batch(cfg, 2, 4, 50)
    bad = torch.as_tensor(bb[0]).clone()
    bad[0, 1, 2] = float("nan")
    p0, m0, v0, s0 = acc.flat_p.clone(), acc.flat_m.clone(), acc.flat_v.clone(), acc.loss_scale
    acc.train_step(ba)
    out = acc.train_step((bad, bb[1]))
    assert not out["applied"] and out["pending"] == 0 and out["loss_scale"] == s0 / 2
    assert (acc.iterations, acc.loss_scale, acc.loss_scale_counter) == (6, s0 / 2, 0)
    assert torch.equal(acc.flat_p, p0) and torch.equal(acc.flat_m, m0) and torch.equal(acc.flat_v, v0)
    acc.loss_scale = 2.0 ** 140
    acc.train_step(ba)
    out = acc.train_step(bb)
    assert not out["applied"] and (acc.iterations, acc.loss_scale, acc.loss_scale_counter) == (7, 2.0 ** 139, 0)
    assert torch.equal(acc.flat_p, p0)
    acc.loss_scale = s0
    acc.train_step(ba)
    out = acc.train_step(bb)
    assert out["applied"] and (acc.iterations, acc.loss_scale, acc.loss_scale_counter) == (8, s0, 1) and not torch.equal(acc.flat_p, p0)


def test_migt_save_mid_window_refused_and_resume_at_a_boundary(tmp_path):
    """save_weights(include_optimizer=True) with a micro-batch pending raises.  A bf16 run of three windows of 2 saved after the second
    and restored into a fresh model continues as the uninterrupted run, held to tests/test_resume_gpu.py's bar."""
    from test_resume_gpu import _compare_runs, _migt, _migt_batches, _migt_tail
    batches = _migt_batches("bf16", 6)
    first, second = _migt_tail(_migt("bf16", accumulate_steps=2)[0], batches), _migt_tail(_migt("bf16", accumulate_steps=2)[0], batches)
    assert [o["applied"] for o in first[2]] == [False, True] * 3
    smodel, saver = _migt("bf16", accumulate_steps=2)
    smodel.train_step(batches[0])
    with pytest.raises(RuntimeError, match="pending"):
        smodel.save_weights(str(tmp_path / "mid" / "model"), include_optimizer=True)
    for b in batches[1:4]:
        smodel.train_step(b)
    assert saver.iterations == 2 and saver.pending == 0
    prefix = str(tmp_path / "run" / "model")
    smodel.save_weights(prefix, include_optimizer=True)
    rmodel, resumed = _migt("bf16", init_seed=1, seed=0, accumulate_steps=2)
    rmodel.load_weights(prefix).expect_partial()
    assert resumed.iterations == 2 and torch.equal(resumed.flat_m, saver.flat_m)
    weights = str(tmp_path / "weights" / "model")
    smodel.save_weights(weights)
    pmodel, _ = _migt("bf16", init_seed=1, accumulate_steps=2)
    pmodel.load_weights(weights)
    r = _migt_tail(rmodel, batches[4:])
    assert resumed.iterations == 3
    _compare_runs("migt bf16, windows of 2", first[:2], second[:2], r[:2], _migt_tail(pmodel, batches[4:])[:2])
