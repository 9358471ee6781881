"""TEST INFRASTRUCTURE — regenerate tests/golden/migt_train_rpm_small.npz: three calls of the REAL reference's MIGT.train_step (executed
over oracle/tf_shim.py, container only) with the pose-scale augmentation on (random_pose_multiplier = 2.5, pose_multiplier = 0.3).  The
per-scene exponents u ~ U[-1, 1) the reference draws with tf.random.uniform (migt.py:349-351) are recorded by wrapping the shim's
tf.random.uniform, so the GPU trainer can be fed the same draws.

The size is migt_train_small's (2 layers, d = 128, B = 2 scenes of 4 views) with 2 heads instead of 4: 64-wide heads are what the bf16
trainer's fused attention kernels take, so both trainers run against this one file.  Localisation on, dropout 0; variant "dyn." adds
use_dynamic_pose_loss.

    python -m oracle.make_golden_rpm
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth, ref_loader, migt_oracle  # noqa: E402
from oracle.make_golden import OUT, MIGT_TRAIN, MIGT_TRAIN_WARMUP, warmup_cosine  # noqa: E402
from viewformer_b200.config import MIGTConfig  # noqa: E402

MIGT_TRAIN_RPM = dict(MIGT_TRAIN, n_head=2, pose_multiplier=0.3, random_pose_multiplier=2.5)
VARIANTS = (("", {}), ("dyn.", dict(use_dynamic_pose_loss=True)))
DYN_WEIGHTS = [0.3, -2.0]
WKEY = "pose_loss_weighting_criterion.pos_ori_weights"
KEEP = ("h.1.mlp.c_proj.bias", "h.1.ln_2.gamma", "ln_f.beta", "pose_classifier.c_proj.weight", "pose_classifier.c_proj.bias",
        "pose_embedding.c_fc.weight", "pose_embedding.c_fc.bias")                # whole tensors kept: those the pose scale reaches first
B, T, STEPS = 2, 4, 3


def batch(cfg, step):
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=150 + step)
    cams = migt_oracle.normalize_cameras(migt_oracle.to_relative_cameras(synth.make_cameras(B, T, seed=160 + step))[0])
    return cams, codes


def state_dict(cfg):
    sd = dict(synth.make_migt_state_dict(cfg, 19))
    if cfg.use_dynamic_pose_loss:
        sd[WKEY] = torch.tensor(DYN_WEIGHTS)
    return sd


def _var(model, key):
    suffix = "/" + ("pos_ori_weights" if key == WKEY else key).replace(".", "/")      # DynamicLossWeightingCriterion's own weight name
    hits = [v for v in model.variables if ("/" + v.name[:-2].replace(".", "/")).endswith(suffix)]
    assert len(hits) == 1, (key, [v.name for v in hits])
    return hits[0]


def run_reference(kw, torch_seed=0):
    """Three train_step calls of the reference model built from state_dict(cfg), under AdamWeightDecay with WarmUp(CosineDecay).  Returns
    {name: array} as stored in the fixture (without the variant prefix).  The torch generator behind the shim's tf.random.uniform is
    seeded with ``torch_seed``."""
    tf = sys.modules["tensorflow"]
    cfg = MIGTConfig(**kw)
    sd = state_dict(cfg)
    model = ref_loader.build_reference_migt({k: v for k, v in sd.items() if k != WKEY},
                                            dynamic_pose_weights=DYN_WEIGHTS if cfg.use_dynamic_pose_loss else None, **kw)
    utils = sys.modules["viewformer.models.utils"]
    opt, _ = utils.create_optimizer(cfg.learning_rate, num_train_steps=cfg.total_steps, num_warmup_steps=MIGT_TRAIN_WARMUP,
                                    weight_decay_rate=cfg.weight_decay)
    model.compile(optimizer=opt)
    names = list(sd.keys())
    gen = torch.Generator().manual_seed(77)
    probe = {k: torch.randn(sd[k].shape, generator=gen) for k in names}
    draws, outputs, grads = [], [], []
    uniform, call, apply = tf.random.uniform, model.call, opt.apply_gradients

    def recording_uniform(*a, **k):
        u = uniform(*a, **k)
        draws.append(torch.as_tensor(u).as_subclass(torch.Tensor).detach().clone())
        return u

    def recording_call(*a, **k):
        o = call(*a, **k)
        outputs.append(o)
        return o

    def recording_apply(pairs):
        pairs = list(pairs)
        grads.append({id(v): g for g, v in pairs})
        return apply(pairs)

    out = dict(names=np.array(names))
    torch.manual_seed(torch_seed)
    tf.random.uniform, model.call, opt.apply_gradients = recording_uniform, recording_call, recording_apply
    try:
        for step in range(STEPS):
            cams, codes = batch(cfg, step)
            model._train_counter.assign(step)
            n_draws = len(draws)
            model.train_step((cams, codes))
            assert len(draws) == n_draws + 1, "train_step should draw the pose multipliers once"
            u = draws[-1].to(torch.float32)
            o = outputs[-1]
            out[f"u{step}"] = u.numpy()
            out[f"r{step}"] = (torch.tensor(cfg.random_pose_multiplier, dtype=torch.float32) ** u).numpy()
            out[f"loss{step}"] = np.float32(float(torch.as_tensor(o["loss"]).as_subclass(torch.Tensor).detach().mean()))
            for key, name in (("ce_loss", "ce"), ("pose_loss", "pose"), ("pose_pos_loss", "pos"), ("pose_ori_loss", "ori")):
                out[f"{name}{step}"] = torch.as_tensor(o[key]).as_subclass(torch.Tensor).detach().numpy().copy()
            g = {k: grads[-1][id(_var(model, k))] for k in names}
            g = {k: (torch.zeros_like(sd[k]) if v is None else torch.as_tensor(v).as_subclass(torch.Tensor).detach()) for k, v in g.items()}
            out[f"gnorm{step}"] = np.array([float(g[k].norm()) for k in names])
            out[f"gdot{step}"] = np.array([float((g[k] * probe[k]).sum()) for k in names])
            for k in KEEP:
                out[f"g{step}.{k}"] = g[k].numpy().astype(np.float32)
            out[f"lr{step}"] = np.float32(warmup_cosine(step, cfg.learning_rate, MIGT_TRAIN_WARMUP, cfg.total_steps))
            w = {k: _var(model, k).detach().as_subclass(torch.Tensor) for k in names}
            out[f"pdot{step}"] = np.array([float((w[k] * probe[k]).sum()) for k in names])
            for k in KEEP + ((WKEY,) if cfg.use_dynamic_pose_loss else ()):
                out[f"p{step}.{k}"] = w[k].numpy().copy()
    finally:
        tf.random.uniform = uniform
        del model.call, opt.apply_gradients
    assert int(opt.iterations) == STEPS
    return out


def golden_migt_train_rpm():
    from oracle import tf_shim
    tf_shim.install()
    ref_loader.load_reference_migt()
    try:
        out = {}
        for prefix, extra in VARIANTS:
            rec = run_reference(dict(MIGT_TRAIN_RPM, **extra), torch_seed=len(prefix))
            out.update({prefix + k: v for k, v in rec.items()})
            print(f"rpm {prefix or 'plain'}: r", [rec[f"r{i}"].tolist() for i in range(STEPS)], "losses", [float(rec[f"loss{i}"]) for i in range(STEPS)])
    finally:
        tf_shim.uninstall()
    np.savez_compressed(os.path.join(OUT, "migt_train_rpm_small.npz"), **out)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count())
    golden_migt_train_rpm()
