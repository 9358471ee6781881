"""TEST INFRASTRUCTURE — the transformer's training forward with the pose-scale augmentation (random_pose_multiplier, models/migt.py:349-354):
``migt_oracle.forward(..., compute_losses=True)`` restated for the training call, where scene b's poses take a multiplier r_b.  Built from
migt_oracle's layers (mlp, block, layer_norm, quaternion helpers); with r = None it computes what migt_oracle.forward does
(tests/test_pose_scale_host.py holds the two equal).
"""
import torch
import torch.nn.functional as F

from oracle import migt_oracle as mo


def _per_scene(r, x):
    """r [B] shaped to broadcast over x [B, ...] (expand_pose_multiplier, migt.py:147-148)."""
    return r.to(x.dtype).reshape([-1] + [1] * (x.dim() - 1))


def pose_model_input(cfg, poses, r=None):
    """get_model_input (migt.py:139-145): xyz * pose_multiplier, then * r (two roundings), concatenated with the quaternion."""
    xyz = poses[..., :3] * cfg.pose_multiplier
    if r is not None:
        xyz = xyz * _per_scene(r, xyz)
    return torch.cat([xyz, poses[..., 3:]], -1)


def forward(sd, cfg, inputs, r=None, use_localization=True, localization_weight=1.0):
    """MIGT.call(dict(poses, input_ids), compute_losses=True) (migt.py:338-455) with the training-time per-scene pose multiplier
    ``r`` [B] (None: 1): the pose inputs of streams 0 and 1 scaled by r_b, the pose head's xyz divided by r_b before the position loss
    (QuaternionPoseRepresentation.call, :156-177).  Returns dict(logits, loss, ce_loss, [pose_prediction, pose_pos_loss, pose_ori_loss,
    pose_loss])."""
    dt = sd["wte.weight"].dtype
    poses = inputs["poses"].to(dt)
    ids = inputs["input_ids"]
    orig_shape = list(ids.shape)
    ids = ids.reshape(ids.shape[0], ids.shape[1], -1)
    B, T, L = ids.shape
    wte, wpe = sd["wte.weight"], sd["wpe.embeddings"]
    mask_tok, loc_tok = cfg.n_embeddings, cfg.n_embeddings + 1
    pose_emb = mo.mlp(sd, "pose_embedding", pose_model_input(cfg, poses, r)).unsqueeze(-2)            # [B,T,1,d], streams 0 and 1
    pos = wpe[:L][None, None]
    emb = wte[ids]
    hs = [emb + pos + pose_emb, wte[mask_tok].reshape(1, 1, 1, -1) + pos + pose_emb]
    if use_localization:
        hs.append(emb + pos + wte[loc_tok].reshape(1, 1, 1, -1))
    for i in range(cfg.n_layer):
        hs = mo.block(sd, f"h.{i}.", hs, cfg.n_head)
    hs = [mo.layer_norm(sd, "ln_f", x) for x in hs]
    logits = (hs[1] @ wte.t())[..., : cfg.n_embeddings]
    skip = cfg.n_loss_skip
    ls = float(getattr(cfg, "label_smoothing", 0.0))
    flat = logits.reshape(-1, logits.shape[-1])
    if ls > 0:
        y = F.one_hot(ids.reshape(-1).long(), flat.shape[-1]).to(flat.dtype) * (1.0 - ls) + ls / flat.shape[-1]
        ce = -(y * F.log_softmax(flat, -1)).sum(-1).reshape(B, T, L)
    else:
        ce = F.cross_entropy(flat, ids.reshape(-1).long(), reduction="none").reshape(B, T, L)
    ce = ce[:, skip:].mean((1, 2))
    out = dict(ce_loss=ce)
    loss = ce * cfg.image_generation_weight
    if use_localization:
        o = mo.mlp(sd, "pose_classifier", hs[2])
        xyz, quat = o[..., :3], o[..., 3:]
        if r is not None:
            xyz = xyz / _per_scene(r, xyz)
        out["pose_prediction"] = torch.cat([xyz / cfg.pose_multiplier, mo.quaternion_remove_sign(mo.quaternion_normalize(quat))], -1)
        y = poses.unsqueeze(-2) * torch.tensor([cfg.pose_multiplier] * 3 + [1.0] * 4, dtype=dt)
        pl = ((y[..., :3] - xyz) ** 2).mean(-1)[:, skip:].mean((1, 2))
        ol = ((y[..., 3:] - quat) ** 2).mean(-1)[:, skip:].mean((1, 2))
        wkey = "pose_loss_weighting_criterion.pos_ori_weights"
        if getattr(cfg, "use_dynamic_pose_loss", False) and wkey in sd:
            w = sd[wkey]                                          # DynamicLossWeightingCriterion.call (migt.py:116-118)
            pose_loss = (w + torch.exp(-w) * torch.stack([pl, ol], -1)).sum()
        else:
            pose_loss = pl + ol
        out.update(pose_pos_loss=pl, pose_ori_loss=ol, pose_loss=pose_loss)
        loss = loss + pose_loss * localization_weight
    out["logits"] = logits.reshape(orig_shape + [-1])
    out["loss"] = loss
    return out
