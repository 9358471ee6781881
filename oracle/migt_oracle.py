"""TEST INFRASTRUCTURE — torch-CPU restatement of the reference TensorFlow MIGT transformer.

Pinned to the reference's own SOURCE, not to TensorFlow's kernels: the reference transformer exists only in
TensorFlow/Keras (viewformer/models/migt.py) and TensorFlow cannot be installed here (no network, TF 2.4.1 has
no cp312 wheel), and the reference ships no tests or golden vectors for it.  tests/test_reference_on_shim.py
therefore executes the reference's files unmodified from /root/reference over oracle/tf_shim.py (a torch-backed
restatement of the ~70 TensorFlow leaf ops they call) and requires this restatement to reproduce MIGT.call,
MIGT.train_step (GradientTape + AdamWeightDecay under WarmUp/CosineDecay) and generate_batch_predictions of both
evaluation scripts to 1e-6; tests/golden/migt_reference_shim.npz carries outputs of that run to machines without
/root/reference.  Further cross-checks: transformers' GPT2Block / GPT2Model (tests/test_migt_oracle_vs_gpt2.py)
and the structural invariants of SURVEY.md §8(c) (tests/test_oracle_pinned.py).  What is not exercised anywhere:
TensorFlow's own floating-point evaluation order.

Follows (file:line in /root/reference):
  viewformer/models/migt.py:13-14      GELU = exact erf form, LayerNorm eps 1e-5
  viewformer/models/migt.py:17-56      SharedEmbeddings (gather / tied linear)
  viewformer/models/migt.py:59-96      MLP, Conv1D  (x @ W[in,out] + b[1,out])
  viewformer/models/migt.py:123-179    quaternion_reduce_mean, QuaternionPoseRepresentation
  viewformer/models/migt.py:182-238    BranchingAttention ((v,q,k) split order), Block (pre-LN)
  viewformer/models/migt.py:338-455    MIGT.call
  viewformer/models/branching_attention.py:5-18, 41-61, 82-126   masked attention (no 1/sqrt(d),
                                        multiplicative mask with -1e4), block-causal, multi-end
  viewformer/utils/geometry_tf.py:6-13, 44-50, 53-91              quaternion helpers
  viewformer/evaluate/evaluate_transformer.py:70-146              generate_batch_predictions
  viewformer/evaluate/evaluate_transformer_multictx.py:37-95      multi-context variant
"""
import torch
import torch.nn.functional as F

LN_EPS = 1e-5


# ----------------------------------------------------------------------------- geometry
def quaternion_multiply(q1, q2):
    w1, x1, y1, z1 = q1.unbind(-1)
    w2, x2, y2, z2 = q2.unbind(-1)
    x = x1 * w2 + y1 * z2 - z1 * y2 + w1 * x2
    y = -x1 * z2 + y1 * w2 + z1 * x2 + w1 * y2
    z = x1 * y2 - y1 * x2 + z1 * w2 + w1 * z2
    w = -x1 * x2 - y1 * y2 - z1 * z2 + w1 * w2
    return torch.stack((w, x, y, z), -1)


def quaternion_conjugate(q):
    return torch.cat((q[..., :1], -q[..., 1:]), -1)


def quaternion_rotate(point, q):
    p = torch.cat([torch.zeros_like(point[..., :1]), point], -1)
    p = quaternion_multiply(q, p)
    p = quaternion_multiply(p, quaternion_conjugate(q))
    return p[..., 1:]


def quaternion_normalize(x, epsilon=1e-12):
    # tf.linalg.l2_normalize: x * rsqrt(max(sum(x^2), eps))
    return x * torch.rsqrt(torch.clamp((x * x).sum(-1, keepdim=True), min=epsilon))


def quaternion_remove_sign(x):
    sign = 2 * (x[..., :1] >= 0).to(x.dtype) - 1
    return x * sign


def quaternion_reduce_mean(q, axis=-2):
    q = quaternion_remove_sign(quaternion_normalize(q))
    q = q.mean(axis)
    return quaternion_remove_sign(quaternion_normalize(q))


def reduce_cameras(x, axis=-2):
    """migt.py:150-154, 532-533."""
    return torch.cat((x[..., :3].mean(axis), quaternion_reduce_mean(x[..., 3:], axis)), -1)


def to_relative_cameras(cameras):
    xyz, quat = cameras[..., :3], cameras[..., 3:]
    t_xyz, t_q = xyz[..., :1, :], quat[..., :1, :]
    inv = quaternion_conjugate(t_q)
    xyz = quaternion_rotate(xyz - t_xyz, inv.expand_as(quat))
    quat = quaternion_multiply(inv.expand_as(quat), quat)
    return torch.cat((xyz, quat), -1), torch.cat((t_xyz, t_q), -1)


def from_relative_cameras(cameras, transform):
    t_xyz, t_q = transform[..., :3], transform[..., 3:]
    xyz, quat = cameras[..., :3], cameras[..., 3:]
    t_qe = t_q.expand_as(quat)
    quat = quaternion_multiply(t_qe, quat)
    xyz = quaternion_rotate(xyz, t_qe) + t_xyz
    return torch.cat((xyz, quat), -1)


def normalize_cameras(cameras):
    q = quaternion_remove_sign(quaternion_normalize(cameras[..., 3:]))
    return torch.cat((cameras[..., :3], q), -1)


# ----------------------------------------------------------------------------- layers
def conv1d(sd, p, x):
    return x @ sd[p + ".weight"] + sd[p + ".bias"]


def mlp(sd, p, x):
    return conv1d(sd, p + ".c_proj", F.gelu(conv1d(sd, p + ".c_fc", x)))


def layer_norm(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".gamma"], sd[p + ".beta"], LN_EPS)


def masked_attention(k, v, q, mask=None):
    """branching_attention.py:5-18 — no 1/sqrt(d) scaling; multiplicative mask, masked logits = -1e4."""
    w = q @ k.transpose(-1, -2)
    if mask is not None:
        w = w * mask - 1e4 * (1 - mask)
    return F.softmax(w, dim=-1) @ v


def causal_block_attention(k, v, q):
    """branching_attention.py:41-61 — q,k,v [B,H,T,L,dh]; a view attends to itself and earlier views."""
    b, h, ns, l, _ = k.shape
    nd = q.shape[-3]
    i = torch.arange(nd).repeat_interleave(l)[:, None]
    j = torch.arange(ns).repeat_interleave(l)
    m = (i >= j - ns + nd).to(k.dtype)
    a = masked_attention(k.reshape(b, h, ns * l, -1), v.reshape(b, h, ns * l, -1), q.reshape(b, h, nd * l, -1), m)
    return a.reshape(b, h, nd, l, -1)


def causal_block_multiend_attention(kset, vset, qset):
    """branching_attention.py:82-126."""
    k, v = kset[0], vset[0]
    outputs = [causal_block_attention(k, v, qset[0])]
    b, h, ns, l, _ = k.shape
    k_flat = k[:, :, :-1].reshape(b, h, (ns - 1) * l, -1)
    v_flat = v[:, :, :-1].reshape(b, h, (ns - 1) * l, -1)
    nd = qset[0].shape[-3]
    i = torch.arange(nd).repeat_interleave(l)[:, None]
    j = torch.arange(ns - 1).repeat_interleave(l)
    m = (i >= j - ns + nd + 1).to(k.dtype).reshape(1, 1, nd * l, (ns - 1) * l)
    for k_new, v_new, q in zip(kset[1:], vset[1:], qset[1:]):
        nd = q.shape[-3]
        q_flat = q.reshape(b, h, nd * l, -1)
        w_old = q_flat @ k_flat.transpose(-1, -2)
        w_old = w_old * m - 1e4 * (1 - m)
        w_new = (q @ k_new.transpose(-1, -2)).reshape(b, h, -1, l)
        w = F.softmax(torch.cat([w_old, w_new], -1), dim=-1)
        a_old = (w[..., : (ns - 1) * l] @ v_flat).reshape(b, h, nd, l, -1)
        w_n = w[..., (ns - 1) * l:].reshape(b, h, nd, l, l)
        outputs.append(a_old + torch.einsum("ijklm,ijkmv->ijklv", w_n, v_new))
    return outputs


def _split_heads(x, n_head):
    b, t, l, d = x.shape
    return x.reshape(b, t, l, n_head, d // n_head).permute(0, 3, 1, 2, 4)


def _merge_heads(x):
    b, h, t, l, dh = x.shape
    return x.permute(0, 2, 3, 1, 4).reshape(b, t, l, h * dh)


def block(sd, p, xs, n_head):
    """migt.py:230-238 + 207-217."""
    a = [layer_norm(sd, p + "ln_1", x) for x in xs]
    vs, qs, ks = [], [], []
    for y in a:
        v, q, k = conv1d(sd, p + "attn.c_attn", y).chunk(3, dim=-1)   # (v, q, k) order, migt.py:212
        vs.append(_split_heads(v, n_head)); qs.append(_split_heads(q, n_head)); ks.append(_split_heads(k, n_head))
    att = causal_block_multiend_attention(ks, vs, qs)
    att = [conv1d(sd, p + "attn.c_proj", _merge_heads(t)) for t in att]
    xs = [x + t for x, t in zip(xs, att)]
    m = [mlp(sd, p + "mlp", layer_norm(sd, p + "ln_2", x)) for x in xs]
    return [x + t for x, t in zip(xs, m)]


def pose_model_input(cfg, poses):
    """migt.py:139-145 (eval: random multiplier == 1)."""
    return torch.cat([poses[..., :3] * cfg.pose_multiplier, poses[..., 3:]], -1)


def pose_head(sd, cfg, h):
    """migt.py:156-164 (no targets)."""
    o = mlp(sd, "pose_classifier", h)
    xyz, quat = o[..., :3], o[..., 3:]
    qn = quaternion_remove_sign(quaternion_normalize(quat))
    return torch.cat([xyz / cfg.pose_multiplier, qn], -1), xyz, quat


def forward(sd, cfg, inputs, compute_losses=False, use_localization=True, localization_weight=1.0):
    """migt.py:338-455 with training=False.  Returns dict(logits, hidden_states, [pose_prediction], loss...).  Poses are cast to the
    weights' dtype (the reference's float32; float64 weights give an fp64 reference end to end)."""
    dt = sd["wte.weight"].dtype
    poses = inputs["poses"].to(dt)
    ids = inputs["input_ids"]
    orig_shape = list(ids.shape)
    ids = ids.reshape(ids.shape[0], ids.shape[1], -1)
    B, T, L = ids.shape
    loc_tokens = inputs.get("localization_tokens")
    out_poses = inputs.get("output_poses")
    wte, wpe = sd["wte.weight"], sd["wpe.embeddings"]
    mask_tok, loc_tok = cfg.n_embeddings, cfg.n_embeddings + 1

    pose_emb = mlp(sd, "pose_embedding", pose_model_input(cfg, poses)).unsqueeze(-2)   # [B,Tp,1,d]
    pos = wpe[:L][None, None]
    emb = wte[ids]
    loc_seq = T - pose_emb.shape[1]
    loc_emb = None
    out_pose_emb = None
    gen_ptr = pose_ptr = 0
    if compute_losses:
        if loc_tokens is None and use_localization:
            loc_tokens, loc_emb = ids, emb
        if out_poses is None:
            out_poses, out_pose_emb = poses, pose_emb
    if loc_tokens is not None and loc_emb is None:
        loc_emb = wte[loc_tokens.reshape(loc_tokens.shape[0], loc_tokens.shape[1], -1)]
    if out_poses is not None and out_pose_emb is None:
        out_pose_emb = mlp(sd, "pose_embedding", pose_model_input(cfg, out_poses.to(dt))).unsqueeze(-2)
    if use_localization and not compute_losses:
        lp = wte[loc_tok].reshape(1, 1, 1, -1).expand(B, loc_seq, 1, wte.shape[1])
        pose_emb = torch.cat([pose_emb, lp], 1)
    hs = [emb + pos + pose_emb]
    if out_pose_emb is not None:
        hs.append(wte[mask_tok].reshape(1, 1, 1, -1) + pos + out_pose_emb)
        gen_ptr = len(hs) - 1
    if loc_emb is not None:
        hs.append(loc_emb + pos + wte[loc_tok].reshape(1, 1, 1, -1))
        pose_ptr = len(hs) - 1
    for i in range(cfg.n_layer):
        hs = block(sd, f"h.{i}.", hs, cfg.n_head)
    hs = [layer_norm(sd, "ln_f", x) for x in hs]
    out = {"hidden_states": hs}
    logits = (hs[gen_ptr] @ wte.t())[..., : cfg.n_embeddings]
    loss = 0
    if compute_losses:
        skip = cfg.n_loss_skip
        ls = float(getattr(cfg, "label_smoothing", 0.0))
        flat = logits.reshape(-1, logits.shape[-1])
        if ls > 0:      # migt.py:99-104: one-hot * (1 - s) + s / n_classes, then softmax_cross_entropy_with_logits
            y = F.one_hot(ids.reshape(-1).long(), flat.shape[-1]).to(flat.dtype) * (1.0 - ls) + ls / flat.shape[-1]
            ce = -(y * F.log_softmax(flat, -1)).sum(-1).reshape(B, T, L)
        else:
            ce = F.cross_entropy(flat, ids.reshape(-1).long(), reduction="none").reshape(B, T, L)
        ce = ce[:, skip:].mean((1, 2))
        out["ce_loss"] = ce
        loss = loss + ce * cfg.image_generation_weight
    if use_localization:
        pred, xyz, quat = pose_head(sd, cfg, hs[pose_ptr])
        if compute_losses:
            y = poses.unsqueeze(-2) * torch.tensor([cfg.pose_multiplier] * 3 + [1.0] * 4, dtype=dt)
            pl = ((y[..., :3] - xyz) ** 2).mean(-1)[:, cfg.n_loss_skip:].mean((1, 2))
            ol = ((y[..., 3:] - quat) ** 2).mean(-1)[:, cfg.n_loss_skip:].mean((1, 2))
            wkey = "pose_loss_weighting_criterion.pos_ori_weights"
            if getattr(cfg, "use_dynamic_pose_loss", False) and wkey in sd:
                # DynamicLossWeightingCriterion.call (migt.py:116-118): reduce_sum(w + exp(-w) * stack([pos, ori], -1)) — a scalar
                w = sd[wkey]
                pose_loss = (w + torch.exp(-w) * torch.stack([pl, ol], -1)).sum()
            else:
                pose_loss = pl + ol                                   # migt.py:284
            out["pose_pos_loss"], out["pose_ori_loss"], out["pose_loss"] = pl, ol, pose_loss
            loss = loss + pose_loss * localization_weight
        out["pose_prediction"] = pred
    out["logits"] = logits.reshape(orig_shape + [-1])
    out["loss"] = loss
    return out


# ----------------------------------------------------------------------------- callers
def images_to_float(images_u8_nhwc):
    """evaluate_transformer.py:106-108 — tf.image.convert_image_dtype(uint8->f32) (x * (1/255)) then *2-1."""
    return images_u8_nhwc.to(torch.float32) * torch.tensor(1.0 / 255.0, dtype=torch.float32) * 2 - 1


def float_to_images(x):
    """evaluate_transformer.py:128-129 — clip [-1,1]; convert_image_dtype(f32->uint8) = saturate(trunc(x*255.5))."""
    x = x.clamp(-1, 1) / 2 + 0.5
    return (x * 255.5).clamp(0, 255).to(torch.uint8)


def generate_batch_predictions(forward_fn, encode_fn, decode_code_fn, cfg, images, cameras, use_localization=True):
    """evaluate_transformer.py:97-146.  images uint8 [B,T,H,W,3]; cameras f32 [B,T,7].
    encode_fn(x NCHW f32)->codes int64 [N,h,w]; decode_code_fn(codes)->NCHW f32;
    forward_fn(dict)->dict.  Layout note: the TF caller is NHWC; the torch codebook is NCHW."""
    gt_cam = cameras[:, -1]
    transform = None
    if cfg.augment_poses == "relative":
        cameras, transform = to_relative_cameras(cameras)
    cameras = normalize_cameras(cameras)
    B, T = images.shape[:2]
    x = images_to_float(images.reshape((B * T,) + tuple(images.shape[2:]))).permute(0, 3, 1, 2).contiguous()
    codes = encode_fn(x).reshape(B, T, cfg.token_image_size, cfg.token_image_size)
    ids = torch.cat([codes[:, :-1], torch.full_like(codes[:, :1], cfg.n_embeddings)], 1)
    out = forward_fn(dict(input_ids=ids, poses=cameras))
    gen_codes = out["logits"].argmax(-1)[:, -1]
    gen = float_to_images(decode_code_fn(gen_codes)).permute(0, 2, 3, 1).contiguous()
    if use_localization:
        out2 = forward_fn(dict(input_ids=codes, poses=cameras[:, :-1]))
        gen_cam = reduce_cameras(out2["pose_prediction"][:, -1:], -2)
    else:
        gen_cam = cameras[:, :1]
    if transform is not None:
        gen_cam = from_relative_cameras(gen_cam, transform)
    return dict(ground_truth_images=images[:, -1], generated_images=gen, ground_truth_cameras=gt_cam,
                generated_cameras=gen_cam[:, -1], generated_codes=gen_codes, codes=codes)


def generate_batch_predictions_multictx(forward_fn, encode_fn, decode_code_fn, cfg, images, cameras):
    """evaluate_transformer_multictx.py:37-95 (3-stream call; per-context-size predictions)."""
    gt_cam = cameras[:, -1]
    transform = None
    if cfg.augment_poses == "relative":
        cameras, transform = to_relative_cameras(cameras)
    cameras = normalize_cameras(cameras)
    B, T = images.shape[:2]
    x = images_to_float(images.reshape((B * T,) + tuple(images.shape[2:]))).permute(0, 3, 1, 2).contiguous()
    codes = encode_fn(x).reshape(B, T, cfg.token_image_size, cfg.token_image_size)
    ids = torch.cat([codes[:, :-1], torch.full_like(codes[:, :1], cfg.n_embeddings)], 1)
    ctx_cams = torch.cat([cameras[:, :-1], torch.zeros_like(cameras[:, :1])], 1)
    out = forward_fn(dict(input_ids=ids, poses=ctx_cams, localization_tokens=codes[:, -1:].repeat(1, T, 1, 1),
                          output_poses=cameras[:, -1:].repeat(1, T, 1)))
    gen_codes = out["logits"].argmax(-1)
    gen_cam = reduce_cameras(out["pose_prediction"], -2)
    gen = float_to_images(decode_code_fn(gen_codes.reshape((B * T,) + tuple(gen_codes.shape[2:])))).permute(0, 2, 3, 1)
    gen = gen.reshape((B, T) + tuple(gen.shape[1:]))
    if transform is not None:
        gen_cam = from_relative_cameras(gen_cam, transform)
    return dict(ground_truth_images=images[:, -1], generated_images=gen, ground_truth_cameras=gt_cam,
                generated_cameras=gen_cam, generated_codes=gen_codes)
