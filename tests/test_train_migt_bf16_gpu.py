"""bf16 transformer training step (MIGTTrainer(precision="bf16")): the fused attention forward / backward kernels against fp64 torch on the
same bf16 operands, the step against the fp32 trainer (which the reference pins, test_train_gpu.py) and the full-size reference fixture, and
the dynamic loss scaler (TF 2.4 DynamicLossScale / LossScaleOptimizer, restated in MIGTTrainer.optimizer_step).

The step bars are estimates from bf16 rounding (2^-9 relative per operand); measured values are printed."""
import os

import numpy as np
import pytest
import torch

from oracle import synth

pytestmark = pytest.mark.gpu

MEDIUM = dict(n_layer=2, d_model=256, n_head=4, token_image_size=8, n_loss_skip=1, weight_decay=0.01, total_steps=100, learning_rate=1e-3,
              label_smoothing=0.05, localization_weight="0.5", image_generation_weight=0.8, pose_multiplier=1.0)


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _cos(a, b):
    return float((a.double() * b.double()).sum() / (a.double().norm() * b.double().norm()).clamp_min(1e-300))


# ----------------------------------------------------------------------------------------------- kernels
def _attn_reference(qk, vt, dout, B, S, ns, H, d, rate, seed):
    """fp64 torch: per stream O, LSE and (autograd) dQ, dK, dV of sum_s <O_s, dO_s> with the fp32 trainer's dropout mask."""
    from viewformer_b200 import _lib as L
    dh, T = d // H, S // 64
    q = [qk[:, s * S:(s + 1) * S, :d].double().reshape(B, S, H, dh).permute(0, 2, 1, 3).clone().requires_grad_() for s in range(ns)]
    k = [qk[:, s * S:(s + 1) * S, d:].double().reshape(B, S, H, dh).permute(0, 2, 1, 3).clone().requires_grad_() for s in range(ns)]
    v = [vt[:, :, s * S:(s + 1) * S].double().reshape(B, H, dh, S).transpose(2, 3).clone().requires_grad_() for s in range(ns)]
    view = torch.arange(S, device=qk.device) // 64
    outs, lses, total = [], [], 0.0
    for s in range(ns):
        if s == 0:
            logits = q[0] @ k[0].transpose(2, 3)
            vis = view[None, :] <= view[:, None]
            vv = v[0]
        else:
            logits = torch.cat([q[s] @ k[0].transpose(2, 3), q[s] @ k[s].transpose(2, 3)], dim=3)
            vis = torch.cat([view[None, :] < view[:, None], view[None, :] == view[:, None]], dim=1)
            vv = torch.cat([v[0], v[s]], dim=2)
        logits = logits.masked_fill(~vis, float("-inf"))
        lse = torch.logsumexp(logits, dim=3)
        P = torch.exp(logits - lse[..., None])
        if rate > 0:
            P = P * L.dropout(torch.ones(P.shape, dtype=torch.float32, device=qk.device), rate, seed + s).double()
        o = P @ vv                                                                     # [B, H, S, dh]
        outs.append(o.detach().permute(0, 2, 1, 3).reshape(B * S, d))
        lses.append(lse.detach())
        total = total + (o.permute(0, 2, 1, 3).reshape(B * S, d) * dout[s].double()).sum()
    total.backward()
    grads = []
    for s in range(ns):
        f = lambda t: t.grad.permute(0, 2, 1, 3).reshape(B * S, d)
        grads.append((f(v[s]), f(q[s]), f(k[s])))                                    # v | q | k, the c_attn column order
    return outs, lses, grads


@pytest.mark.parametrize("ns", [1, 3])
@pytest.mark.parametrize("T", [4, 5])
@pytest.mark.parametrize("rate", [0.0, 0.1])
def test_fused_attention_train_kernels_vs_fp64(ns, T, rate):
    """vf_attn_multiend_train (O, LSE) and vf_attn_multiend_bwd (dQ, dK, dV per stream) against fp64 torch on the same bf16 Q, K, V and dO,
    the dropout mask taken from vf_dropout.  Bars: relative error <= 1e-2, gradient cosine >= 0.999."""
    from viewformer_b200 import _lib as L
    B, H, d = 2, 2, 128
    S = T * 64
    g = torch.Generator().manual_seed(10 * ns + T)
    qk = (torch.randn((B, ns * S, 2 * d), generator=g) * 0.5).to(torch.bfloat16).cuda()
    vt = torch.randn((B, d, ns * S), generator=g).to(torch.bfloat16).cuda()
    dout = torch.randn((ns, B * S, d), generator=g).to(torch.bfloat16).cuda()
    seed = 123457
    o16 = torch.empty((ns, B * S, d), dtype=torch.bfloat16, device="cuda")
    o32 = torch.empty((ns, B * S, d), dtype=torch.float32, device="cuda")
    lse = torch.empty((ns, B, H, S), dtype=torch.float32, device="cuda")
    for s in range(ns):
        L.attn_multiend_train(qk, vt, B, S, ns, s, H, d, 64, rate=rate, seed=seed + s, lse=lse[s], out_f32=o32[s], out=o16[s])
    dvqk = L.attn_multiend_bwd(qk, vt, dout, o32, lse, B, S, ns, H, d, 64, rate=rate, seed=seed)
    torch.cuda.synchronize()
    outs, lses, grads = _attn_reference(qk, vt, dout, B, S, ns, H, d, rate, seed)
    for s in range(ns):
        eo, el = _rel(o32[s].double(), outs[s]), _rel(lse[s].double(), lses[s])
        assert torch.equal(o16[s], o32[s].to(torch.bfloat16))
        errs = []
        for j, name in enumerate("vqk"):
            got, ref = dvqk[s][:, j * d:(j + 1) * d].double(), grads[s][j]
            e, c = _rel(got, ref), _cos(got, ref)
            errs.append(f"d{name} {e:.2e}/{c:.6f}")
            assert e <= 1e-2 and c >= 0.999, f"stream {s} d{name}: rel {e:.3e} cos {c:.6f}"
        print(f"[attn train ns={ns} T={T} rate={rate} stream {s}] O {eo:.2e} lse {el:.2e} " + " ".join(errs))
        assert eo <= 1e-2 and el <= 1e-2


@pytest.mark.parametrize("ns", [1, 3])
@pytest.mark.parametrize("T", [4, 5])
def test_fused_attention_train_forward_bits_match_inference(ns, T):
    """With no LSE output and rate 0 the training forward computes the inference kernels' bits."""
    from viewformer_b200 import _lib as L
    B, H, d = 2, 4, 256
    S = T * 64
    g = torch.Generator().manual_seed(T)
    qk = torch.randn((B, ns * S, 2 * d), generator=g).to(torch.bfloat16).cuda()
    vt = torch.randn((B, d, ns * S), generator=g).to(torch.bfloat16).cuda()
    for s in range(ns):
        got = L.attn_multiend_train(qk, vt, B, S, ns, s, H, d, 64)
        ref = L.attn_block_causal(qk, vt, B, S, H, d, 64) if ns == 1 else L.attn_block_multiend(qk, vt, B, S, ns, s, H, d, 64)
        assert torch.equal(got, ref)


def test_bf16_copy_and_weight_refresh_bit_identical():
    """vf_to_bf16 (with and without dropout) and vf_dense_weights_bf16 equal torch relayouts followed by .to(torch.bfloat16); the bf16
    dense weight gradient is within 1e-5 of sum |x||dy| of fp64 on the same bf16-rounded operands."""
    from viewformer_b200 import _lib as L
    g = torch.Generator().manual_seed(3)
    x = (torch.randn((333, 160), generator=g) * 5).cuda()
    assert torch.equal(L.to_bf16(x), x.to(torch.bfloat16))
    y, y16 = L.to_bf16(x, 0.1, 99, out_f32=True)
    ref = L.dropout(x, 0.1, 99)
    assert torch.equal(y, ref) and torch.equal(y16, ref.to(torch.bfloat16))
    ws = [torch.randn(shape, generator=g).cuda() for shape in ((256, 768), (1024, 256), (96, 200))]
    entries = [(w, torch.empty((w.shape[1], w.shape[0]), dtype=torch.bfloat16, device="cuda"),
                torch.empty(w.shape, dtype=torch.bfloat16, device="cuda")) for w in ws]
    L.dense_weights_bf16(L.dense_weights_bf16_table(entries, "cuda"))
    for w, fw, bw in entries:
        assert torch.equal(fw, w.t().contiguous().to(torch.bfloat16)) and torch.equal(bw, w.to(torch.bfloat16))
    xa, dy = torch.randn((700, 256), generator=g).cuda(), torch.randn((700, 384), generator=g).cuda()
    dw = torch.ones((256, 384), device="cuda")
    L.dense_wgrad_bf16(xa, dy, dw)
    xr, dr = xa.to(torch.bfloat16).double(), dy.to(torch.bfloat16).double()
    err = float(((dw.double() - 1.0) - xr.t() @ dr).abs().max() / (xr.abs().t() @ dr.abs()).max())
    print(f"[dense wgrad bf16] max err / sum|x||dy| {err:.2e}")
    assert err < 1e-5


# ----------------------------------------------------------------------------------------------- the step
def _trainers(cfg_kw, seed=0, **kw):
    from viewformer_b200 import MIGT
    from viewformer_b200.config import MIGTConfig
    from viewformer_b200.train_migt import MIGTTrainer
    cfg = MIGTConfig(**cfg_kw)
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    return cfg, MIGTTrainer(model, seed=seed, **kw), MIGTTrainer(model, seed=seed, precision="bf16", **kw)


def _batch(cfg, B, T, seed):
    from oracle import migt_oracle as mo
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=seed)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=seed + 1))[0])
    return cams, codes


@pytest.mark.parametrize("T", [4, 5])
@pytest.mark.parametrize("dropout", [0.0, 0.1])
def test_bf16_step_matches_fp32_trainer(T, dropout):
    """One medium-config step (2 layers, d = 256, 4 heads, localisation on): loss within 5e-3 relative of the fp32 trainer and every
    gradient tensor at cosine >= 0.99 with the loss scale divided out.  With dropout 0.1 and equal seeds this also shows that both trainers
    drop the same elements: different masks would move the loss by far more than the bar."""
    cfg, t32, t16 = _trainers(dict(MEDIUM, dropout=dropout))
    cams, codes = _batch(cfg, 2, T, 40 + T)
    l32, l16 = float(t32.forward_backward(cams, codes)), float(t16.forward_backward(cams, codes))
    torch.cuda.synchronize()
    g32, g16 = t32.gradients(), t16.gradients()
    worst = min((_cos(g16[k] / t16.loss_scale, g32[k]), k) for k in g32 if float(g32[k].norm()) > 0)
    print(f"[bf16 step T={T} dropout={dropout}] loss {l16:.6f} vs fp32 {l32:.6f} ({abs(l16 - l32) / abs(l32):.2e}); "
          f"worst gradient cosine {worst[0]:.5f} ({worst[1]})")
    assert abs(l16 - l32) <= 5e-3 * abs(l32)
    assert worst[0] >= 0.99, worst


def test_bf16_step_full_size_matches_reference(golden_dir):
    """Full size (12 layers, d = 768; B = 1, T = 5, dropout 0) against tests/golden/migt_train_full.npz: loss and CE within 5e-3, gradient
    norms and projections with the loss scale divided out: median error <= 1e-2, worst <= 1e-1."""
    from viewformer_b200 import MIGT
    from viewformer_b200.config import MIGTConfig
    from viewformer_b200.train_migt import MIGTTrainer
    g = np.load(os.path.join(golden_dir, "migt_train_full.npz"))
    cfg = MIGTConfig(dropout=0.0, label_smoothing=0.1, localization_weight="0.7", total_steps=100, learning_rate=1e-4)
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 13))
    tr = MIGTTrainer(model, precision="bf16")
    B, T = 1, 5
    from oracle import migt_oracle as mo
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=70)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=71))[0])
    loss = float(tr.forward_backward(cams, codes))
    torch.cuda.synchronize()
    ce = tr.last["ce_loss"].cpu().numpy()
    print(f"[bf16 full-size step] loss {loss:.6f} (ref {float(g['loss']):.6f}), ce {ce} (ref {g['ce']})")
    assert abs(loss - float(g["loss"])) <= 5e-3 * abs(float(g["loss"]))
    np.testing.assert_allclose(ce, g["ce"], rtol=5e-3)
    names = [str(n) for n in g["names"]]
    grads = tr.gradients()
    gen = torch.Generator().manual_seed(78)
    errs = []
    for i, n in enumerate(names):
        pr = torch.randn(tuple(grads[n].shape), generator=gen)
        gr = grads[n] / tr.loss_scale
        gn, gd = float(gr.norm()), float((gr * pr).sum())
        rn, rd = float(g["gnorm"][i]), float(g["gdot"][i])
        errs.append((max(abs(gn - rn), abs(gd - rd)) / max(rn, 1e-4), n))
    med, worst = float(np.median([e for e, _ in errs])), max(errs)
    print(f"[bf16 full-size step] gradients: median {med:.2e}, worst {worst[0]:.2e} ({worst[1]}) over {len(names)} tensors")
    assert med <= 1e-2 and worst[0] <= 1e-1, worst


# ----------------------------------------------------------------------------------------------- loss scaling
def test_loss_scale_divides_out():
    """A finite step at the initial scale 2^15: gradients / scale equal those of the same trainer run at scale 1 to 4e-6 * max|g| per tensor.
    Power-of-two scaling is exact, but the attention backward adds dQ with fp32 atomics whose order differs from run to run, so two runs
    at the same scale differ too.  Measured on an H100: 5.5e-7 to 6.6e-7 in four runs and above the first bar of 1e-6 in a fifth; the bar
    is 4e-6."""
    cfg, _, t16 = _trainers(dict(MEDIUM, dropout=0.1))
    cams, codes = _batch(cfg, 2, 4, 7)
    assert t16.loss_scale == 2.0 ** 15
    t16.forward_backward(cams, codes)
    scaled = {k: v / t16.loss_scale for k, v in t16.gradients().items()}
    t16.loss_scale = 1.0
    t16.forward_backward(cams, codes)
    plain = t16.gradients()
    worst = max(float((scaled[k] - plain[k]).abs().max() / plain[k].abs().max().clamp_min(1e-30)) for k in plain if float(plain[k].abs().max()) > 0)
    print(f"[loss scale] worst |g/2^15 - g(scale 1)| / max|g| = {worst:.2e}")
    assert worst <= 4e-6


def test_loss_scale_skips_non_finite_step_and_grows():
    """A batch with one NaN pose: no update (weights, m and v unchanged bit for bit), the scale halves, iterations still advance; the next
    finite step applies.  With the good-step counter at 1999 a finite step doubles the scale and resets the counter."""
    cfg, _, tr = _trainers(dict(MEDIUM, dropout=0.0), warmup_steps=2)
    cams, codes = _batch(cfg, 2, 4, 11)
    tr.train_step((cams, codes))                       # iteration 0 runs at lr 0: take one step so m / v are non-zero
    p0, m0, v0 = tr.flat_p.clone(), tr.flat_m.clone(), tr.flat_v.clone()
    it0, s0 = tr.iterations, tr.loss_scale
    bad = torch.as_tensor(cams).clone()
    bad[0, 1, 2] = float("nan")
    out = tr.train_step((bad, codes))
    assert torch.equal(tr.flat_p, p0) and torch.equal(tr.flat_m, m0) and torch.equal(tr.flat_v, v0)
    assert tr.loss_scale == s0 / 2 and out["loss_scale"] == s0 / 2 and tr.iterations == it0 + 1 and tr.loss_scale_counter == 0
    tr.train_step((cams, codes))
    assert not torch.equal(tr.flat_p, p0) and tr.loss_scale == s0 / 2 and tr.loss_scale_counter == 1
    tr.loss_scale_counter = 1999
    out = tr.train_step((cams, codes))
    assert tr.loss_scale == s0 and out["loss_scale"] == s0 and tr.loss_scale_counter == 0


def test_bf16_loss_curve_tracks_fp32():
    """30 medium-config steps on fixed batches: the bf16 loss stays within 5 % of the fp32 trainer's over the first 10 steps and within
    10 % on the mean of the last 10."""
    cfg, t32, t16 = _trainers(dict(MEDIUM, dropout=0.1), warmup_steps=3)
    batches = [_batch(cfg, 2, 4, 100 + i) for i in range(3)]
    c32, c16 = [], []
    for step in range(30):
        b = batches[step % 3]
        c32.append(t32.train_step(b)["loss"])
        c16.append(t16.train_step(b)["loss"])
    first = max(abs(a - b) / abs(b) for a, b in zip(c16[:10], c32[:10]))
    last = abs(np.mean(c16[-10:]) - np.mean(c32[-10:])) / abs(np.mean(c32[-10:]))
    print(f"[bf16 curve] fp32 {c32[0]:.4f} -> {c32[-1]:.4f}, bf16 {c16[0]:.4f} -> {c16[-1]:.4f}; first 10 worst {first:.2e}, last-10 mean {last:.2e}")
    assert first <= 0.05 and last <= 0.10


# ----------------------------------------------------------------------------------------------- memory and surface
def test_bf16_step_saves_the_probability_memory():
    """Full size, B = 2, T = 20: the bf16 step's peak allocation is below the fp32 step's by at least the bytes of the probability tensors
    the fp32 trainer keeps ([B, H, S, S] + 2 x [B, H, S, 2S] fp32 per layer)."""
    cfg, t32, t16 = _trainers(dict(dropout=0.1))
    B, T = 2, 20
    cams, codes = _batch(cfg, B, T, 5)
    peaks = {}
    for name, tr in (("fp32", t32), ("bf16", t16)):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        tr.forward_backward(cams, codes)
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    S, H = T * 64, cfg.n_head
    probs = cfg.n_layer * B * H * (S * S + 2 * S * 2 * S) * 4
    print(f"[memory] peak above baseline: fp32 {peaks['fp32'] / 2**30:.2f} GiB, bf16 {peaks['bf16'] / 2**30:.2f} GiB; "
          f"fp32 probabilities {probs / 2**30:.2f} GiB")
    assert peaks["fp32"] - peaks["bf16"] >= probs


def test_compile_bf16_surface_and_inference_reload():
    """model.compile(precision="bf16"); model.train_step(batch) runs, reports the loss scale, and the trained weights serve inference."""
    from viewformer_b200 import MIGT
    from viewformer_b200.config import MIGTConfig
    cfg = MIGTConfig(**dict(MEDIUM, dropout=0.1))
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    tr = model.compile(precision="bf16")
    cams, codes = _batch(cfg, 2, 4, 3)
    out = model.train_step((cams, codes))
    assert np.isfinite(out["loss"]) and out["loss_scale"] == 2.0 ** 15 and model._train_counter == 1
    m2 = MIGT(cfg, precision="bf16").load_state_dict(tr.state_dict())
    pred = m2.generate_codes(np.asarray(codes)[:, :-1], cams)
    assert pred.shape[0] == 2 and torch.isfinite(m2(dict(input_ids=codes, poses=cams))["logits"]).all()


def test_bf16_rejects_unsupported_shapes():
    from viewformer_b200 import MIGT
    from viewformer_b200.config import MIGTConfig
    from viewformer_b200.train_migt import MIGTTrainer
    cfg = MIGTConfig(**dict(MEDIUM, n_head=2))
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    with pytest.raises(NotImplementedError, match="d_model / n_head == 64"):
        MIGTTrainer(model, precision="bf16")
