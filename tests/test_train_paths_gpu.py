"""Training-step paths that the fixture comparisons do not reach, each against an independent reference:

* the fp32 transformer step with dropout (the reference recipes' default rate 0.1) against fp64 autograd through a restatement of the
  trainer's three-stream forward with the trainer's own dropout masks (the restatement itself is checked against the oracle at rate 0);
* gradient clipping: the transformer's per-tensor ``tf.clip_by_norm`` (fp32 and bf16 steps) and the codebook's global-norm clip as
  pytorch-lightning applies it, each followed by its optimizer, restated in fp64;
* the CUDA-core fallback (``VF_TRAIN_TC=0``) of both trainers against the reference fixtures, with the fixture tests' own assertions.
"""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import migt_oracle as mo
from oracle import synth
from oracle.make_golden import MIGT_TRAIN, SMALL_VQ, vq_images
from viewformer_b200.config import MIGTConfig, VQGANConfig

gpu = pytest.mark.gpu
U = 2.0 ** -24


def f32(x):
    return float(np.float32(x))


def keras_lr_t(lr, b1, b2, t):
    """lr sqrt(1 - b2^t) / (1 - b1^t) in fp32, as vf_adamw_keras evaluates it on the host (and TF 2.4's Adam for fp32 variables)."""
    one = np.float32(1.0)
    return float(np.float32(lr) * np.sqrt(one - np.float32(b2) ** np.float32(t)) / (one - np.float32(b1) ** np.float32(t)))


# ----------------------------------------------------------------------------- the transformer forward, restated
def restated_forward(sd, cfg, codes, cams, localization_weight, masks=None):
    """MIGTTrainer.forward_backward's forward pass in plain torch, in the trainer's layouts: streams [B*S, d] (rows = scene, view, token) for
    tokens + poses, MASK token + poses and tokens + LOC token; attention probabilities [B, H, S, cols], cols = S for stream 0 (block-causal)
    and 2 S for streams s > 0 (stream-0 keys of earlier views, then the stream's own view).  ``masks`` maps ("emb", s), ("attn", layer, s),
    ("attn_out", layer, s) and ("mlp", layer, s) to multiplicative dropout masks of those shapes (None: no dropout).
    Returns dict(loss [B], ce_loss [B], pose_loss [B])."""
    def drop(x, key):
        return x if masks is None else x * masks[key]

    codes = torch.as_tensor(codes)
    B, T = codes.shape[:2]
    Lt, d, H, V = cfg.token_image_size ** 2, cfg.d_model, cfg.n_head, cfg.n_embeddings
    S, dh, skip = T * Lt, d // H, cfg.n_loss_skip
    wte, wpe = sd["wte.weight"], sd["wpe.embeddings"]
    ids = codes.reshape(B * S).long()
    mult = torch.tensor([cfg.pose_multiplier] * 3 + [1.0] * 4, dtype=wte.dtype)
    pin = torch.as_tensor(cams).to(wte.dtype).reshape(B * T, 7) * mult
    pe = mo.mlp(sd, "pose_embedding", pin).repeat_interleave(Lt, 0)
    pos = wpe[:Lt].repeat(B * T, 1)
    xs = [wte[ids] + pos + pe, wte[V].expand(B * S, d) + pos + pe, wte[ids] + pos + wte[V + 1]]
    xs = [drop(x, ("emb", s)) for s, x in enumerate(xs)]
    view = torch.arange(S) // Lt
    causal, earlier, same = view[None] <= view[:, None], view[None] < view[:, None], view[None] == view[:, None]

    def heads(t):
        return t.reshape(B, S, H, dh).permute(0, 2, 1, 3)

    for li in range(cfg.n_layer):
        p = f"h.{li}."
        vqk = [mo.conv1d(sd, p + "attn.c_attn", mo.layer_norm(sd, p + "ln_1", x)) for x in xs]
        v, q, k = ([heads(t[:, i * d:(i + 1) * d]) for t in vqk] for i in range(3))
        outs = []
        for s in range(len(xs)):
            if s == 0:
                sc = torch.where(causal, q[0] @ k[0].transpose(-1, -2), -1e4)
            else:
                sc = torch.cat([torch.where(earlier, q[s] @ k[0].transpose(-1, -2), -1e4), torch.where(same, q[s] @ k[s].transpose(-1, -2), -1e4)], -1)
            P = drop(torch.softmax(sc, -1), ("attn", li, s))
            o = P[..., :S] @ v[0] + (P[..., S:] @ v[s] if s else 0)
            outs.append(o.permute(0, 2, 1, 3).reshape(B * S, d))
        ys = [x + drop(mo.conv1d(sd, p + "attn.c_proj", o), ("attn_out", li, s)) for s, (x, o) in enumerate(zip(xs, outs))]
        xs = [y + drop(mo.mlp(sd, p + "mlp", mo.layer_norm(sd, p + "ln_2", y)), ("mlp", li, s)) for s, y in enumerate(ys)]
    hn = [mo.layer_norm(sd, "ln_f", x) for x in xs]
    logits = hn[1] @ wte[:V].t()
    ls = float(cfg.label_smoothing)
    target = F.one_hot(ids, V).to(logits.dtype) * (1 - ls) + ls / V
    ce = -(target * F.log_softmax(logits, -1)).sum(-1).reshape(B, T, Lt)[:, skip:].mean((1, 2))
    raw = mo.mlp(sd, "pose_classifier", hn[2]).reshape(B, T, Lt, 7)
    y = pin.reshape(B, T, 1, 7)
    pl = ((y[..., :3] - raw[..., :3]) ** 2).mean(-1)[:, skip:].mean((1, 2))
    ol = ((y[..., 3:] - raw[..., 3:]) ** 2).mean(-1)[:, skip:].mean((1, 2))
    return dict(loss=ce * cfg.image_generation_weight + (pl + ol) * localization_weight, ce_loss=ce, pose_loss=pl + ol)


def _batch(cfg, B, T, seed):
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=seed)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=seed + 10))[0])
    return codes, cams


@pytest.mark.parametrize("T", [4, 5])
def test_restatement_matches_oracle_at_rate_0(T):
    """CPU: at dropout 0 the restatement gives oracle.migt_oracle.forward(compute_losses=True)'s loss terms and gradients.  The oracle casts the
    poses to fp32, so both run in fp32; a wrong layout, mask or stream is an O(1) difference, summation order a ~1e-6 one."""
    cfg = MIGTConfig(**MIGT_TRAIN)
    sd0 = synth.make_migt_state_dict(cfg, 9)
    codes, cams = _batch(cfg, 2, T, 50)
    lw = 0.5
    sa = {k: v.clone().requires_grad_(True) for k, v in sd0.items()}
    sb = {k: v.clone().requires_grad_(True) for k, v in sd0.items()}
    r = restated_forward(sa, cfg, codes, cams, lw)
    o = mo.forward(sb, cfg, dict(input_ids=codes, poses=cams), compute_losses=True, localization_weight=lw)
    for key in ("loss", "ce_loss", "pose_loss"):
        err = float((r[key] - o[key]).detach().abs().max() / o[key].detach().abs().max())
        print(f"[restatement T={T}] {key}: rel err {err:.2e} (bar 1e-5)")
        assert err < 1e-5, key
    r["loss"].mean().backward()
    o["loss"].mean().backward()
    worst = 0.0
    for k in sd0:
        ga = sa[k].grad if sa[k].grad is not None else torch.zeros_like(sa[k])
        gb = sb[k].grad if sb[k].grad is not None else torch.zeros_like(sb[k])
        err = float((ga - gb).abs().max() / gb.abs().max().clamp_min(1e-6))
        worst = max(worst, err)
        assert err < 1e-4, f"grad {k}: rel err {err:.2e}"
    print(f"[restatement T={T}] gradients of {len(sd0)} tensors: worst rel err {worst:.2e} (bar 1e-4)")


def _trainer_masks(L, tr, cfg, B, T):
    """The trainer's dropout masks at its current (seed, iterations): vf_dropout of ones at each site, exactly 0 or 1 / (1 - rate)."""
    Lt, d, H = cfg.token_image_size ** 2, cfg.d_model, cfg.n_head
    S, rate = T * Lt, float(cfg.dropout)

    def mask(shape, site):
        return L.dropout(torch.ones(shape, device="cuda"), rate, tr._drop_seed(site)).double().cpu()

    masks = {}
    for s in range(3):
        masks[("emb", s)] = mask((B * S, d), 10 + s)
        for li in range(cfg.n_layer):
            site = 100 + 20 * li
            masks[("attn", li, s)] = mask((B, H, S, S if s == 0 else 2 * S), site + s)
            masks[("attn_out", li, s)] = mask((B * S, d), site + 4 + s)
            masks[("mlp", li, s)] = mask((B * S, d), site + 8 + s)
    return masks


ELEMENTWISE = ["wte.weight", "wpe.embeddings", "h.0.attn.c_attn.weight", "pose_embedding.c_fc.weight", "h.0.attn.c_proj.weight",
               "h.1.attn.c_attn.bias", "h.1.mlp.c_fc.weight", "h.0.mlp.c_proj.bias", "h.0.ln_1.gamma", "h.1.ln_2.beta", "ln_f.gamma",
               "pose_classifier.c_fc.weight"]


@gpu
@pytest.mark.parametrize("T,seed", [(4, 0), (5, 3)])
def test_migt_fp32_dropout_step_matches_restated_autograd(lib, T, seed):
    """The fp32 transformer step at dropout 0.1 (3 streams) computes the gradient of its own forward pass: loss terms and the gradient of
    every tensor against fp64 autograd through the restatement with the trainer's masks, for two consecutive steps with optimizer_step
    between them (the masks follow ``iterations``) and two trainer seeds (the masks follow ``seed``).  Bars of
    test_migt_training_step_matches_oracle_autograd: 3e-3 on norm and projection, 2e-3 element-wise on a dozen tensors."""
    from viewformer_b200 import MIGT
    from viewformer_b200 import _lib as L
    from viewformer_b200.train_migt import MIGTTrainer
    cfg = MIGTConfig(**dict(MIGT_TRAIN, dropout=0.1))
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    tr = MIGTTrainer(model, warmup_steps=0, bucket_bytes=1 << 18, seed=seed)
    B = 2
    gen = torch.Generator().manual_seed(77)
    probe = {k: torch.randn(tuple(tr.p[k].shape), generator=gen) for k in tr.p}
    prev = None
    for step in range(2):
        codes, cams = _batch(cfg, B, T, 50 + step)
        masks = _trainer_masks(L, tr, cfg, B, T)
        tr.seed += 1
        other = _trainer_masks(L, tr, cfg, B, T)
        tr.seed -= 1
        for key in masks:                       # every site's mask changes with the seed and with the step
            assert not torch.equal(masks[key], other[key]), f"mask {key} does not depend on the trainer seed"
            assert prev is None or not torch.equal(masks[key], prev[key]), f"mask {key} did not change between steps"
        kept = float(sum(float((m != 0).double().mean()) for m in masks.values()) / len(masks))
        prev = masks
        sd = {k: v.double().requires_grad_(True) for k, v in tr.state_dict().items()}
        lw = tr.loc_weight
        loss = tr.forward_backward(cams, codes)
        torch.cuda.synchronize()
        r = restated_forward(sd, cfg, codes, cams.double(), lw, masks)
        ref = r["loss"].mean()
        ref.backward()
        print(f"[migt dropout T={T} seed={seed} step {step}] loss {float(loss):.6f} (fp64 restatement {float(ref.detach()):.6f}); mean keep fraction {kept:.4f}")
        assert abs(float(loss) - float(ref.detach())) < 3e-5 * abs(float(ref.detach()))
        np.testing.assert_allclose(tr.last["ce_loss"].cpu().double().numpy(), r["ce_loss"].detach().numpy(), rtol=3e-5)
        np.testing.assert_allclose(tr.last["pose_loss"].cpu().double().numpy(), r["pose_loss"].detach().numpy(), rtol=1e-4)
        grads = tr.gradients()
        worst = wfull = 0.0
        for k, gk in grads.items():
            want = sd[k].grad if sd[k].grad is not None else torch.zeros_like(sd[k])
            gk = gk.double()
            rn = float(want.norm())
            e = max(abs(float(gk.norm()) - rn), abs(float((gk * probe[k]).sum()) - float((want * probe[k]).sum()))) / max(rn, 1e-4)
            worst = max(worst, e)
            assert e < 3e-3, f"step {step} {k}: |g| {float(gk.norm()):.6e} vs {rn:.6e}"
        for k in ELEMENTWISE:
            want = sd[k].grad
            err = float((grads[k].double() - want).abs().max() / want.abs().max().clamp_min(1e-4))
            wfull = max(wfull, err)
            assert err < 2e-3, f"step {step} grad {k}: max rel err {err:.3e}"
        print(f"[migt dropout T={T} seed={seed} step {step}] gradients: worst norm/projection rel err {worst:.2e} (bar 3e-3) over {len(grads)} "
              f"tensors; worst element-wise {wfull:.2e} (bar 2e-3) over {len(ELEMENTWISE)}")
        tr.optimizer_step()


# ----------------------------------------------------------------------------- gradient clipping
MEDIUM = dict(n_layer=2, d_model=256, n_head=4, token_image_size=8, n_loss_skip=1, weight_decay=0.01, total_steps=100, learning_rate=1e-3,
              label_smoothing=0.05, localization_weight="0.5", image_generation_weight=0.8, pose_multiplier=1.0, dropout=0.0)


@gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_migt_per_tensor_clipping_then_adamw(lib, precision):
    """MIGTTrainer.optimizer_step with gradient_clip_val set to the median gradient norm (so about half the tensors are clipped) == the fp64
    restatement: tf.clip_by_norm per tensor on the unscaled gradients (bf16: tr.gradients() / tr.loss_scale), then the Keras AdamWeightDecay
    step applied to the pre-step weights and moments, with lr sqrt(1 - b2^t) / (1 - b1^t) evaluated in fp32 as the kernel and TF 2.4 do (an
    fp64 one differs by u / (1 - b2^t) = 3e-5 relative at t = 2, which measured 3.5 x the bar on the second step).  Two steps: Adam's first step is invariant to a per-tensor scale, the second is not.
    Bar per element: 1e-6 lr + 2 u |p| (the fp32 weight is rounded when the decay and the update are stored); the clip itself moves the
    second step's weights by far more, which the test also checks."""
    from viewformer_b200 import MIGT
    from viewformer_b200.train_migt import MIGTTrainer
    cfg = MIGTConfig(**MEDIUM)
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    tr = MIGTTrainer(model, warmup_steps=0, precision=precision)
    b1, b2, eps, wd = f32(0.9), f32(0.999), f32(1e-8), f32(cfg.weight_decay)
    moved = 0.0
    for step in range(2):
        codes, cams = _batch(cfg, 2, 4, 80 + step)
        tr.forward_backward(cams, codes)
        torch.cuda.synchronize()
        grads = {k: v.double() / tr.loss_scale for k, v in tr.gradients().items()}
        norms = {k: float(g.norm()) for k, g in grads.items()}
        if step == 0:
            tr.cfg.gradient_clip_val = float(np.median(list(norms.values())))
        clip = tr.cfg.gradient_clip_val
        clipped = sorted(k for k in norms if norms[k] > clip)
        print(f"[migt clip {precision} step {step}] clip {clip:.4e}: {len(clipped)} of {len(norms)} tensors clipped, e.g. {clipped[:4]}; "
              f"not clipped e.g. {sorted(set(norms) - set(clipped))[:4]}")
        assert 0 < len(clipped) < len(norms)
        lr, t = f32(tr.learning_rate()), tr.iterations + 1
        lr_t = keras_lr_t(lr, 0.9, 0.999, t)
        pre = {k: (tr.p[k].double().cpu(), tr.flat_m[tr.offs[k]:tr.offs[k] + tr.p[k].numel()].double().cpu().reshape(tr.p[k].shape),
                   tr.flat_v[tr.offs[k]:tr.offs[k] + tr.p[k].numel()].double().cpu().reshape(tr.p[k].shape)) for k in tr.order}
        assert tr.optimizer_step()
        worst = 0.0
        for k in tr.order:
            p0, m0, v0 = pre[k]

            def adamw(g):
                p = p0 - lr * wd * p0 if tr.decay[k] else p0
                m = m0 + (g - m0) * (1 - b1)
                v = v0 + (g * g - v0) * (1 - b2)
                return p - lr_t * m / (v.sqrt() + eps)

            want = adamw(grads[k] * (clip / max(norms[k], clip)))
            bar = 1e-6 * lr + 2 * U * p0.abs()
            ratio = float(((tr.p[k].double().cpu() - want).abs() / bar).max())
            worst = max(worst, ratio)
            assert ratio <= 1.0, f"step {step} {k}: error {ratio:.3e} x the bar"
            if k in clipped:
                moved = max(moved, float(((adamw(grads[k]) - want).abs() / bar).max()))
        print(f"[migt clip {precision} step {step}] weights vs fp64 clip_by_norm + AdamW: worst err/bar {worst:.3e}; the clip moves the "
              f"weights by up to {moved:.2e} x the bar")
    assert moved > 100.0


def _vq_trainer(quantizer):
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    cfg = VQGANConfig(**dict(SMALL_VQ, perceptual_weight=0.0))
    sd = synth.make_vqgan_state_dict(cfg, 5)
    if quantizer == "commit":
        sd = {k: v for k, v in sd.items() if not k.startswith("quantize.") or k == "quantize.embeddings"}
    model = VQGAN(cfg, precision="fp32", quantizer=quantizer).load_state_dict(sd)
    return cfg, VQGANTrainer(model)


@gpu
@pytest.mark.parametrize("quantizer", ["ema", "commit"])
def test_vqgan_global_norm_clipping_then_adam(lib, quantizer):
    """VQGANTrainer.optimizer_step with gradient_clip_val > 0 clips as pytorch-lightning does before the optimizer: every gradient times
    min(1, clip / (|g| + 1e-6)), |g| the global L2 norm over all parameters.  Three trainers on the same batches, two steps each:
      clip 0 and clip 10 |g| (coefficient 1): the step is bit-identical to a plain vf_adam call on the unscaled gradient (today's step);
      clip |g| / 2: torch.optim.Adam in fp64 on the clipped gradients from the pre-step weights and moments, within 1e-6 lr + 2 u |p|
      element-wise (Adam's first step is scale-invariant, so the second step is the one the clip moves)."""
    from viewformer_b200 import _lib as L
    xs = [vq_images(3, SMALL_VQ["image_size"], 2000 + s) for s in range(2)]
    for mode in ("off", "loose", "half"):
        cfg, tr = _vq_trainer(quantizer)
        moved = 0.0
        for step, x in enumerate(xs):
            tr.forward_backward(x)
            torch.cuda.synchronize()
            g = tr.flat_g.clone()
            norm = float(g.double().norm())
            if step == 0:
                tr.cfg.gradient_clip_val = {"off": 0.0, "loose": 10.0 * norm, "half": 0.5 * norm}[mode]
            clip = tr.cfg.gradient_clip_val
            p0, m0, v0 = tr.flat_p.clone(), tr.flat_m.clone(), tr.flat_v.clone()
            tr.optimizer_step()
            if mode != "half":
                L.adam(p0, g, m0, v0, lr=tr.lr, beta1=tr.betas[0], beta2=tr.betas[1], eps=tr.eps, step=tr.step_count, grad_scale=1.0)
                assert torch.equal(tr.flat_p, p0) and torch.equal(tr.flat_m, m0) and torch.equal(tr.flat_v, v0)
                print(f"[vqgan clip {quantizer} {mode} step {step}] clip {clip:.4e}, |g| {norm:.4e}: bit-identical to the unclipped vf_adam step")
                continue
            coef = min(1.0, clip / (norm + 1e-6))
            lr, b1, b2, eps, t = f32(tr.lr), f32(tr.betas[0]), f32(tr.betas[1]), f32(tr.eps), tr.step_count
            p0d, m0d, v0d = p0.double().cpu(), m0.double().cpu(), v0.double().cpu()

            def adam(gd):
                m = m0d + (gd - m0d) * (1 - b1)
                v = v0d * b2 + (1 - b2) * gd * gd
                return p0d - lr / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + eps)

            gd = g.double().cpu()
            want = adam(gd * coef)
            bar = 1e-6 * lr + 2 * U * p0d.abs()
            ratio = float(((tr.flat_p.double().cpu() - want).abs() / bar).max())
            moved = max(moved, float(((adam(gd) - want).abs() / bar).max()))
            print(f"[vqgan clip {quantizer} step {step}] clip {clip:.4e}, |g| {norm:.4e}, coefficient {coef:.4f}: weights vs fp64 Adam on the "
                  f"clipped gradient: worst err/bar {ratio:.3e}; the clip moves the weights by up to {moved:.2e} x the bar")
            assert ratio <= 1.0
        if mode == "half":
            assert moved > 100.0


# ----------------------------------------------------------------------------- the CUDA-core fallback
def _fixture_tests():
    """tests/test_train_gpu.py as a module of its own: its fixture comparisons are rerun here unchanged, with their own bars."""
    spec = importlib.util.spec_from_file_location("_train_fixture_tests", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_train_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@gpu
@pytest.mark.parametrize("fixture_test", ["test_vqgan_training_step_matches_reference", "test_vqgan_training_step_full_size_matches_reference",
                                          "test_migt_training_step_matches_oracle_autograd", "test_migt_training_step_full_size_matches_oracle_autograd"])
def test_cuda_core_fallback_matches_fixtures(lib, golden_dir, monkeypatch, fixture_test):
    """VF_TRAIN_TC=0 (read by both trainers' __init__): every conv, dense layer and weight gradient on the fp32 CUDA-core kernels — at full
    size this is the only path where vf_conv_wgrad runs at 128-512 channels on 128x128 maps and the transformer's d = 768 layers run on
    vf_simt_gemm + vf_conv_wgrad.  Reruns the fixture comparisons of tests/test_train_gpu.py with their bars; every trainer they build
    must report use_tc False."""
    from viewformer_b200.train import VQGANTrainer
    from viewformer_b200.train_migt import MIGTTrainer
    monkeypatch.setenv("VF_TRAIN_TC", "0")
    built = []
    for cls in (VQGANTrainer, MIGTTrainer):
        def init(self, *a, _orig=cls.__init__, **k):
            _orig(self, *a, **k)
            built.append(self)
        monkeypatch.setattr(cls, "__init__", init)
    getattr(_fixture_tests(), fixture_test)(golden_dir)
    assert built and all(t.use_tc is False for t in built)
    print(f"[VF_TRAIN_TC=0] {fixture_test}: passed with {len(built)} CUDA-core trainer(s)")
