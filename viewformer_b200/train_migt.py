"""Transformer training step — MIGT.train_step (viewformer/models/migt.py:464-505) on libvf_b200 kernels, fp32 or bf16.

    forward   three streams as in ``call(compute_losses=True, training=True)`` (migt.py:338-455): tokens + poses, MASK tokens + query
              poses (image generation), tokens + LOC token (localisation); block-causal multi-end attention
              (branching_attention.py:82-126); dropout at the reference's four sites (embeddings, attention weights, attention
              output, MLP output) from a stateless hash generator
    loss      mean over the batch of  image_generation_weight * CE(stream 1 logits, tokens)[views >= n_loss_skip]
              + localization_weight * (position MSE + orientation MSE of the stream-2 pose head)
    backward  hand-written: dense layers on the exact split-fp16 tensor-core GEMM (forward, data and weight gradient; VF_TRAIN_TC=0: the
              fp32 CUDA-core kernels), attention through vf_simt_gemm (strided, batched per (scene, head)), vf_conv_wgrad for the remaining weight
              gradients, LayerNorm / GELU / softmax / embedding / loss kernels of vf_backward.cu
    update    per-tensor tf.clip_by_norm when gradient_clip_val > 0 (migt.py:486-487), AdamWeightDecay = Keras Adam preceded by the
              decoupled decay lr*wd*p for every variable whose name has no "bias" (models/utils.py:424, 507-515 — LayerNorm gamma /
              beta ARE decayed: their Keras names are ln_1/gamma ..., which match none of the exclusion patterns), learning rate
              = 2000-step linear warm-up then cosine decay to 0 (migt.py:457-462, models/utils.py:310-416; the first step runs at lr 0)
    exchange  the codebook trainer's ``dist.GradExchange``: gradients live in one flat buffer ordered by backward completion;
              contiguous buckets are all-reduced (SUM; grad_reduce="mean" divides by the world size — see the note in DESIGN.md on
              MirroredStrategy's per-replica reduce_mean) asynchronously while the rest of the backward pass runs.

precision="bf16" (the reference's 16-bit recipes: --fp16 -> mixed-precision policy + LossScaleOptimizer, train_transformer.py:102-104,
models/utils.py:432-433, migt.py:466-488): every dense GEMM that fits the tensor-core tiles (forward, data and weight gradient) takes bf16
operands in one wgmma pass; the attention runs forward in the fused multi-end kernel (vf_attn_multiend_train, which also keeps the per-row
log-sum-exp) and backward in vf_attn_multiend_bwd, which recomputes the probabilities, so no [S, S] tensor is kept or written.  Accumulation,
the residual stream, LayerNorm, GELU pre-activations, softmax statistics, losses, embeddings, gradients, the all-reduce, clipping and AdamW
stay fp32; the flat fp32 buffers remain the master copy and bf16 operand copies of the weights are rewritten after every applied step.
Dynamic loss scaling as TF 2.4's DynamicLossScale: see optimizer_step.

Parameters are kept in the reference's own layouts (Conv1D weight [in, out], bias [1, out]); ``state_dict()`` can be loaded straight
into ``viewformer_b200.MIGT`` for inference.
"""
import math
import os
from collections import OrderedDict

import torch
import torch.distributed as dist

from . import _lib as L
from . import pose_scale as PS
from .dist import GradExchange

LN_EPS = 1e-5


def warmup_cosine(step, init, warm, total_steps, offset=0):
    """create_optimizer's WarmUp(CosineDecay) (models/utils.py:310-416) at optimizer step ``step``: the schedule runs on
    ``max(step - offset, 0)`` (WarmUp.__call__, :344-358; ``offset`` is what fine-tuning sets to the restored ``iterations``)."""
    step = max(step - offset, 0)
    if warm and step < warm:
        return init * (step / float(warm))
    decay_steps = max(1, total_steps - warm)
    t = min(max(step - warm, 0), decay_steps) / float(decay_steps)
    return init * 0.5 * (1.0 + math.cos(math.pi * t))


def dense_route(precision, use_tc, k, n):
    """Kernel route of a dense layer x [m, k] W [k, n] (forward, data and weight gradient alike): "bf16" (single-pass bf16 wgmma), "split"
    (the exact split-fp16 tensor-core GEMM) or "cuda" (fp32 CUDA-core kernels).  ``use_tc``: the bf16 step, or VF_TRAIN_TC is not 0."""
    if not use_tc or k % 128 or n % 128:
        return "cuda"
    return "bf16" if precision == "bf16" else "split"


class _Dense:
    """One dense layer y = x W (+ b): views of W [k, n], b and their gradients (no b: the tied head), its route and split-fp16 copies."""

    def __init__(self, name, w, gw, b, gb, route):
        self.name, self.w, self.gw, self.b, self.gb, self.route = name, w, gw, b, gb, route
        self.split = {}                                            # split-fp16 weights per product, until the next optimizer step


class MIGTTrainer:
    LOSS_SCALE_INIT = 2.0 ** 15                                    # tf.mixed_precision DynamicLossScale defaults (TF 2.4)
    LOSS_SCALE_GROWTH_STEPS = 2000
    _seed_scale = 1.0                                              # the gradient-seed scale of the running step (see grad_seed_scale)

    def __init__(self, model, betas=(0.9, 0.999), eps=1e-8, warmup_steps=2000, bucket_bytes=64 << 20, process_group=None, seed=0,
                 grad_reduce="sum", precision="fp32", learning_rate=None, total_steps=None, accumulate_steps=1):
        """``learning_rate`` / ``total_steps``: peak rate and horizon of the learning-rate schedule when they differ from the config's (the
        optimizer a fine-tuning run builds, finetune_transformer.py:81-83); the localisation-weight schedule keeps the config's horizon.

        ``accumulate_steps`` = N: ``train_step`` adds the gradient of N micro-batches, each the mean loss of its own scenes, and applies
        one update per N calls, so every micro-batch plays one more replica of the reference's MirroredStrategy: one GPU with N = 8
        performs the update of 8 replicas.  ``grad_reduce="mean"`` divides by world size x N.  ``iterations`` (hence the learning rate,
        the localisation weight, Adam's bias correction and the dropout masks), the loss scale and its good-step counter advance once per
        window.  A new value takes effect at the next window."""
        if int(accumulate_steps) < 1:
            raise ValueError(f"accumulate_steps must be >= 1, got {accumulate_steps}")
        self.accumulate_steps = int(accumulate_steps)
        self.pending = 0                                           # micro-batches in the gradient since the last optimizer step
        cfg = model.config
        if not (math.isfinite(cfg.random_pose_multiplier) and cfg.random_pose_multiplier > 0):
            raise ValueError(f"random_pose_multiplier must be a positive number, got {cfg.random_pose_multiplier}")
        if precision not in ("fp32", "bf16"):
            raise ValueError(f"precision must be 'fp32' or 'bf16', got {precision!r}")
        self.precision, self.bf16 = precision, precision == "bf16"
        if self.bf16 and (cfg.d_model % cfg.n_head or cfg.d_model // cfg.n_head != 64 or cfg.token_image_size != 8):
            raise NotImplementedError(f"precision='bf16' needs d_model / n_head == 64 and token_image_size == 8 (the fused attention kernels), got "
                                      f"d_model={cfg.d_model} n_head={cfg.n_head} token_image_size={cfg.token_image_size}")
        # dynamic loss scaling (bf16 only): the scale multiplies the loss gradient seeds; updates are skipped on non-finite gradients
        self.loss_scale = self.LOSS_SCALE_INIT if self.bf16 else 1.0
        self.loss_scale_counter = 0
        # fp32 gradient-seed scale: None = 2^round(log2(denom)) (denom = the loss's row count), which brings the cross-entropy and pose seeds
        # (weight / denom) to about 1 so that the backward operands sit inside the split-fp16 tensor-core path's faithful range; a number =
        # that fixed power of two (1 = off).  Unlike loss_scale it is divided out of each gradient bucket as the bucket completes, so
        # flat_g, gradients(), the all-reduce, clipping and AdamW see the same values as without it.
        self.grad_seed_scale = 1.0 if self.bf16 else None
        self.model, self.cfg, self.device = model, cfg, model.device
        self.betas, self.eps, self.warmup_steps = betas, eps, warmup_steps
        self.group, self.bucket_bytes, self.seed = process_group, bucket_bytes, seed
        # "sum": what the reference does — every replica takes tf.reduce_mean of ITS loss and MirroredStrategy sums the replica
        # gradients (migt.py:471-476: "the learning rate should be scaled accordingly"); "mean" divides by the world size instead
        assert grad_reduce in ("sum", "mean")
        self.grad_reduce = grad_reduce
        self.iterations = 0                                        # optimizer.iterations (0-based: the schedule sees it BEFORE the increment)
        self.init_lr = float(cfg.learning_rate if learning_rate is None else learning_rate)
        self.total_steps = int(cfg.total_steps if total_steps is None else total_steps)
        self.schedule_offset = 0                                   # WarmUp.offset (models/utils.py:342-346): the schedule runs on iterations - offset
        self._train_counter_base = 0                               # see train_counter
        self.use_tc = self.bf16 or os.environ.get("VF_TRAIN_TC", "1") != "0"
        self.use_loc = model.use_localization
        from .schedules import parse
        self._loc_schedule = parse(cfg.localization_weight).with_total_steps(int(cfg.total_steps))
        self.dynamic_pose = bool(cfg.use_dynamic_pose_loss) and self.use_loc
        self._build(model.state_dict())
        self._build_dense()
        if self.bf16:
            self._build_bf16_weights()

    @property
    def train_counter(self):
        """The Keras model's ``_train_counter`` (migt.py:446), which the localisation-weight schedule reads: steps taken since it was last
        set.  It is kept as a distance from ``iterations``, so it advances with every step; ``finetune`` sets it to 0 while ``iterations``
        (Adam's bias correction, the dropout seed) carries on."""
        return self.iterations - self._train_counter_base

    @train_counter.setter
    def train_counter(self, value):
        self._train_counter_base = self.iterations - int(value)

    @property
    def loc_weight(self):
        """localization_weight(self._train_counter) (migt.py:446): the schedule at the number of steps taken so far."""
        return float(self._loc_schedule(self.train_counter)) if self.use_loc else 0.0

    # ------------------------------------------------------------------ parameters
    def _build(self, sd):
        names = list(self.model.param_shapes().keys())
        # backward completion order: heads, ln_f, blocks from last to first, pose embedding, wpe, wte (tied: complete only at the very end)
        n_layer = self.cfg.n_layer
        order = ([k for k in names if k.startswith("pose_loss_weighting_criterion.")] + [k for k in names if k.startswith("pose_classifier.")]
                 + [k for k in names if k.startswith("ln_f.")])
        for i in reversed(range(n_layer)):
            order += [k for k in names if k.startswith(f"h.{i}.")]
        order += [k for k in names if k.startswith("pose_embedding.")] + ["wpe.embeddings", "wte.weight"]
        assert sorted(order) == sorted(names)
        ex = self.ex = GradExchange([(k, sd[k].shape) for k in order], self.device, self.bucket_bytes, self.group)
        self.flat_p, self.flat_g, self.flat_m, self.flat_v, self.p, self.g = ex.flat_p, ex.flat_g, ex.flat_m, ex.flat_v, ex.p, ex.g
        self.order, self.offs, self.buckets, self.launched = ex.order, ex.offs, ex.buckets, ex.launched
        for k in order:
            self.p[k].copy_(sd[k].to(torch.float32))
        # AdamWeightDecay: every variable except the ones whose name contains "bias" (see the module docstring)
        self.decay = {k: ("bias" not in k) for k in order}

    def _build_dense(self):
        """One record per dense layer, in backward-completion order, with its kernel route; the tied head last."""
        self.dense = {}
        for k in self.order:
            if k.endswith(".weight") and k != "wte.weight" and self.p[k].dim() == 2:
                name, b = k[:-len(".weight")], k[:-len("weight")] + "bias"
                route = dense_route(self.precision, self.use_tc, *self.p[k].shape)
                self.dense[name] = _Dense(name, self.p[k], self.g[k], self.p[b].reshape(-1), self.g[b].reshape(-1), route)
        # the tied LM head (migt.py:417) is the bias-free layer W = wte[:V] (in V, out d), used transposed: logits are its data-gradient
        # product on ln_f's output, whose gradient is its forward product on the logits' gradient
        V = self.cfg.n_embeddings
        head = self.p["wte.weight"][:V]
        self.dense["wte"] = _Dense("wte", head, self.g["wte.weight"][:V], None, None, dense_route(self.precision, self.use_tc, *head.shape))

    def _build_bf16_weights(self):
        """bf16 operand copies of every bf16 dense layer's weights: forward [n, k] (K = k) and data gradient [k, n] (K = n); rewritten from
        the fp32 master weights by one vf_dense_weights_bf16 launch after every applied step."""
        self._w16, entries = {}, []
        for r in self.dense.values():
            if r.route == "bf16":
                k, n = r.w.shape
                fw = torch.empty((n, k), dtype=torch.bfloat16, device=self.device)
                bw = torch.empty((k, n), dtype=torch.bfloat16, device=self.device)
                self._w16[r.name] = (fw, bw)
                entries.append((r.w, fw, bw))
        self._w16_table = L.dense_weights_bf16_table(entries, self.device)
        L.dense_weights_bf16(self._w16_table)

    def state_dict(self):
        return OrderedDict((k, self.p[k].detach().cpu().clone()) for k in self.model.param_shapes().keys())

    def gradients(self):
        return OrderedDict((k, self.g[k].detach().cpu().clone()) for k in self.model.param_shapes().keys())

    # ------------------------------------------------------------------ resume: everything a step reads besides the batch
    def optimizer_state(self):
        """Host copies of what ``state_dict()`` leaves out: Adam's moments under the weights' key names and layouts, and the scalars.
        Every rank of a data-parallel run holds the same state; writing it out is rank 0's business."""
        names = list(self.model.param_shapes().keys())
        return dict(m=OrderedDict((k, self.ex.m[k].detach().cpu().clone()) for k in names),
                    v=OrderedDict((k, self.ex.v[k].detach().cpu().clone()) for k in names),
                    iterations=self.iterations, train_counter=self.train_counter, schedule_offset=self.schedule_offset,
                    loss_scale=self.loss_scale, loss_scale_counter=self.loss_scale_counter, seed=self.seed, precision=self.precision)

    def _checked(self, tensors, what, strict):
        """{name: fp32 host tensor} of ``tensors`` for this trainer's parameters; raises on a wrong shape, and (strict) on a missing or
        unknown name, before anything on the device is written."""
        shapes = self.model.param_shapes()
        missing, unknown = [k for k in shapes if k not in tensors], [k for k in tensors if k not in shapes]
        if strict and (missing or unknown):
            raise RuntimeError(f"{what}: missing keys {missing[:8]}, unexpected keys {unknown[:8]}")
        out = {k: torch.as_tensor(tensors[k]).detach().to("cpu", torch.float32) for k in shapes if k in tensors}
        bad = [(k, tuple(t.shape), tuple(shapes[k])) for k, t in out.items() if tuple(t.shape) != tuple(shapes[k])]
        if bad:
            raise RuntimeError(f"{what}: shape mismatch (name, got, expected) {bad[:8]}")
        return out

    def load_state_dict(self, state_dict, strict=True):
        """Weights (the keys of ``state_dict()``) into the fp32 master copy, then what an applied step does to the operand copies."""
        sd = self._checked(state_dict, "MIGTTrainer.load_state_dict", strict)
        for k, t in sd.items():
            self.p[k].copy_(t)
        self._weights_changed()
        return self

    def load_optimizer_state(self, state, strict=True):
        """Inverse of ``optimizer_state()``.  State saved by a trainer of the other precision loads too (the master copy is fp32 either
        way); the loss scale then starts at this precision's default."""
        m, v = self._checked(state["m"], "first moments", strict), self._checked(state["v"], "second moments", strict)
        same_scale = self.bf16 and state.get("precision") == "bf16"
        scalars = ("iterations", "train_counter", "schedule_offset", "seed", "precision") + (("loss_scale", "loss_scale_counter") if same_scale else ())
        absent = [k for k in scalars if k not in state]
        if strict and absent:
            raise RuntimeError(f"MIGTTrainer.load_optimizer_state: missing {absent}")
        for views, src in ((self.ex.m, m), (self.ex.v, v)):
            for k, t in src.items():
                views[k].copy_(t)
        self.iterations = int(state.get("iterations", self.iterations))
        self.train_counter = int(state.get("train_counter", self.iterations))
        self.schedule_offset = int(state.get("schedule_offset", self.schedule_offset))
        self.seed = int(state.get("seed", self.seed))
        if same_scale:
            self.loss_scale = float(state.get("loss_scale", self.loss_scale))
            self.loss_scale_counter = int(state.get("loss_scale_counter", self.loss_scale_counter))
        else:
            self.loss_scale, self.loss_scale_counter = (self.LOSS_SCALE_INIT if self.bf16 else 1.0), 0
        return self

    # ------------------------------------------------------------------ dense layer (Conv1D: x @ W[in,out] + b[1,out])
    # Dense layers whose sizes fit the tensor-core tiles run forward, data gradient and weight gradient on the exact split-fp16 GEMM
    # (fp32-faithful: three fp16 MMA passes, chunked accumulation — DESIGN.md 5.3); VF_TRAIN_TC=0 keeps everything on the CUDA cores.
    def _split_gemm(self, x, r, product, n, k, bias=None, residual=None):
        """x [M, k] fp32 times layer r's weights on the exact split-fp16 GEMM -> [M, n] fp32: its forward ("fw", x W) or data-gradient
        ("bw", x W^T) product."""
        out = torch.empty((x.shape[0], n), dtype=torch.float32, device=x.device)
        xs = L.split_f16x2(x)
        ws = r.split.get(product)
        if ws is None:                          # K-major weights: W^T for the forward product, W [k, n] itself for the data gradient
            ws = r.split[product] = L.split_f16x2(r.w.t().contiguous() if product == "fw" else r.w.contiguous())
        L.tc_gemm(xs, ws, out, M=x.shape[0], N=n, K=k, lda=2 * k, ldb=2 * k, ldc=n, bias=bias,
                  bias_mode=L.BIAS_N if bias is not None else L.BIAS_NONE, residual=residual, lo_a=k, lo_b=k)
        return out

    def _lin(self, x, name, residual=None):
        """The forward product x W (+ b) (+ residual) [m, n] fp32."""
        r = self.dense[name]
        k, n = r.w.shape
        if r.route == "split":
            return self._split_gemm(x, r, "fw", n, k, bias=r.b, residual=residual)
        bias_mode = L.BIAS_N if r.b is not None else L.BIAS_NONE
        out = torch.empty((x.shape[0], n), dtype=torch.float32, device=x.device)
        if r.route == "bf16":
            L.tc_gemm(x if x.dtype == torch.bfloat16 else L.to_bf16(x), self._w16[name][0], out, M=x.shape[0], N=n, K=k, lda=k, ldb=k, ldc=n,
                      bias=r.b, bias_mode=bias_mode, residual=residual)
        else:
            L.simt_gemm(x, r.w, out, M=x.shape[0], N=n, K=k, a_strides=(k, 1), b_strides=(n, 1), ldc=n, bias=r.b, bias_mode=bias_mode,
                        residual=residual)
        return out

    def _dgrad(self, dy, name, residual=None, out16=None):
        """The data-gradient product dx = dy W^T (+ residual) [m, k] fp32 (bf16 route with ``out16``: written as bf16 only)."""
        r = self.dense[name]
        k, n = r.w.shape
        m = dy.shape[0]
        if r.route == "split":
            return self._split_gemm(dy, r, "bw", k, n, residual=residual)
        dx = out16 if out16 is not None and r.route == "bf16" else torch.empty((m, k), dtype=torch.float32, device=dy.device)
        if r.route == "bf16":
            L.tc_gemm(L.to_bf16(dy), self._w16[name][1], dx, M=m, N=k, K=n, lda=n, ldb=n, ldc=k, residual=residual)
        else:
            L.simt_gemm(dy, r.w, dx, M=m, N=k, K=n, a_strides=(n, 1), b_strides=(1, n), ldc=k, residual=residual)
        return dx

    def _lin_bw(self, x, dy, name, *, need_dx=True, residual=None, last=True, out16=None):
        """Accumulates dW (and db) of x W (+ b) and returns dx = dy W^T (+ residual).  A layer applied to every stream is called once per
        stream: the weight-gradient kernels accumulate, and readiness is signalled on the ``last`` call.  bf16: ``out16`` receives dx as
        bf16 only (the attention backward's dO operand)."""
        r = self.dense[name]
        k, n = r.w.shape
        m = x.shape[0]
        if r.route == "cuda":
            L.conv_wgrad(x.reshape(1, m, 1, k), dy.reshape(1, m, 1, n), r.gw, kh=1, pad=(0, 0), so=(n, 1))
        else:
            (L.dense_wgrad_bf16 if r.route == "bf16" else L.dense_wgrad_tc)(x, dy, r.gw)
        if r.b is not None:
            L.col_sums(dy, r.gb)
        if last:
            self.ex.ready(name + ".bias", name + ".weight")
        return self._dgrad(dy, name, residual=residual, out16=out16) if need_dx else None

    def _ln(self, x, name, dtype=torch.float32):
        return L.layernorm(x, self.p[name + ".gamma"], self.p[name + ".beta"], dtype, eps=LN_EPS)

    def _ln_bw(self, x, dy, name, add=None, last=True):
        dx = L.layernorm_bwd(x, dy, self.p[name + ".gamma"], self.g[name + ".gamma"], self.g[name + ".beta"], eps=LN_EPS, add=add)
        if last:
            self.ex.ready(name + ".beta", name + ".gamma")
        return dx

    def _drop_seed(self, site):
        return (self.seed * 1000003 + self.iterations) * 4096 + site

    def _drop(self, x, site):
        rate = float(self.cfg.dropout)
        if rate <= 0.0:
            return x
        return L.dropout(x, rate, self._drop_seed(site))

    # ------------------------------------------------------------------ attention over the stream list
    def _attention_fw(self, vqk, B, S, Lt, site0):
        """vqk: per stream [B*S, 3d] = v | q | k.  Returns (outputs [B*S, d] per stream, saved probabilities)."""
        d, H = self.cfg.d_model, self.cfg.n_head
        dh = d // H
        dev = vqk[0].device
        outs, probs = [], []
        for s, t in enumerate(vqk):
            cols = S if s == 0 else 2 * S
            sc = torch.empty((B, H, S, cols), dtype=torch.float32, device=dev)
            for half, ks in ((0, 0),) if s == 0 else ((0, 0), (1, s)):
                L.simt_gemm(t, vqk[ks], sc, M=S, N=S, K=dh, a_strides=(3 * d, 1), b_strides=(1, 3 * d), ldc=cols, batch=(B, H),
                            a_bs=(S * 3 * d, dh), b_bs=(S * 3 * d, dh), c_bs=(H * S * cols, S * cols), a_off=d, b_off=2 * d, c_off=half * S)
            P = torch.empty_like(sc)
            L.softmax_rows(sc, P, rows_total=B * H * S, rows_per_batch=S, cols=cols, ld_in=cols, ld_out=cols, mask_mode=1 if s == 0 else 2, block=Lt)
            Pd = self._drop(P, site0 + s)
            o = torch.empty((B * S, d), dtype=torch.float32, device=dev)
            L.simt_gemm(Pd, vqk[0], o, M=S, N=dh, K=S, a_strides=(cols, 1), b_strides=(3 * d, 1), ldc=d, batch=(B, H), a_bs=(H * S * cols, S * cols),
                        b_bs=(S * 3 * d, dh), c_bs=(S * d, dh))
            if s > 0:
                L.simt_gemm(Pd, t, o, M=S, N=dh, K=S, a_strides=(cols, 1), b_strides=(3 * d, 1), ldc=d, batch=(B, H), a_bs=(H * S * cols, S * cols),
                            b_bs=(S * 3 * d, dh), c_bs=(S * d, dh), a_off=S, residual=o)
            outs.append(o)
            probs.append(P)
        return outs, probs

    def _attention_bw(self, vqk, probs, dos, B, S, Lt, site0):
        d, H = self.cfg.d_model, self.cfg.n_head
        dh = d // H
        dev = vqk[0].device
        dvqk = [torch.zeros_like(t) for t in vqk]
        for s, (t, P, do) in enumerate(zip(vqk, probs, dos)):
            cols = S if s == 0 else 2 * S
            Pd = self._drop(P, site0 + s)
            pb = (H * S * cols, S * cols)
            dP = torch.empty_like(P)
            for half, ks in ((0, 0),) if s == 0 else ((0, 0), (1, s)):
                # dP[:, half] = do v_ks^T ;  dv_ks += Pd[:, half]^T do
                L.simt_gemm(do, vqk[ks], dP, M=S, N=S, K=dh, a_strides=(d, 1), b_strides=(1, 3 * d), ldc=cols, batch=(B, H), a_bs=(S * d, dh),
                            b_bs=(S * 3 * d, dh), c_bs=pb, c_off=half * S)
                L.simt_gemm(Pd, do, dvqk[ks], M=S, N=dh, K=S, a_strides=(1, cols), b_strides=(d, 1), ldc=3 * d, batch=(B, H), a_bs=pb, b_bs=(S * d, dh),
                            c_bs=(S * 3 * d, dh), a_off=half * S, residual=dvqk[ks])
            dP = self._drop(dP, site0 + s)                          # same mask and scale as the forward pass
            dS = L.softmax_bwd_rows(P, dP)
            for half, ks in ((0, 0),) if s == 0 else ((0, 0), (1, s)):
                # dq_s += dS[:, half] k_ks ;  dk_ks += dS[:, half]^T q_s
                L.simt_gemm(dS, vqk[ks], dvqk[s], M=S, N=dh, K=S, a_strides=(cols, 1), b_strides=(3 * d, 1), ldc=3 * d, batch=(B, H), a_bs=pb,
                            b_bs=(S * 3 * d, dh), c_bs=(S * 3 * d, dh), a_off=half * S, b_off=2 * d, c_off=d, residual=dvqk[s])
                L.simt_gemm(dS, t, dvqk[ks], M=S, N=dh, K=S, a_strides=(1, cols), b_strides=(3 * d, 1), ldc=3 * d, batch=(B, H), a_bs=pb,
                            b_bs=(S * 3 * d, dh), c_bs=(S * 3 * d, dh), a_off=half * S, b_off=d, c_off=2 * d, residual=dvqk[ks])
        return dvqk

    def _attention_fw16(self, a16, pre, B, S, Lt, site0):
        """bf16: a16 per stream [B*S, d] (LayerNorm output) -> q|k [B, ns*S, 2d] and V^T [B, d, ns*S] from the c_attn GEMMs, then the fused
        training forward per stream.  Returns (outputs bf16 [ns, B*S, d], what the backward pass needs)."""
        d, H = self.cfg.d_model, self.cfg.n_head
        ns, dev = len(a16), a16[0].device
        w16, bias = self._w16[pre + "attn.c_attn"][0], self.dense[pre + "attn.c_attn"].b                # [3d, d]: rows v | q | k
        qk = torch.empty((B, ns * S, 2 * d), dtype=torch.bfloat16, device=dev)
        vt = torch.empty((B, d, ns * S), dtype=torch.bfloat16, device=dev)
        for s, a in enumerate(a16):
            L.tc_gemm(a, w16, qk, M=S, N=2 * d, K=d, lda=d, ldb=d, ldc=2 * d, batch=(B, 1), a_bs=(S * d, 0), c_bs=(ns * S * 2 * d, 0),
                      b_off=d * d, c_off=s * S * 2 * d, bias=bias[d:], bias_mode=L.BIAS_N)
            L.tc_gemm(w16, a, vt, M=d, N=S, K=d, lda=d, ldb=d, ldc=ns * S, batch=(B, 1), b_bs=(S * d, 0), c_bs=(d * ns * S, 0),
                      c_off=s * S, bias=bias[:d], bias_mode=L.BIAS_M)
        o16 = torch.empty((ns, B * S, d), dtype=torch.bfloat16, device=dev)
        o32 = torch.empty((ns, B * S, d), dtype=torch.float32, device=dev)
        lse = torch.empty((ns, B, H, S), dtype=torch.float32, device=dev)
        rate = float(self.cfg.dropout)
        for s in range(ns):
            L.attn_multiend_train(qk, vt, B, S, ns, s, H, d, Lt, rate=rate, seed=self._drop_seed(site0 + s), lse=lse[s], out_f32=o32[s], out=o16[s])
        return o16, (qk, vt, o32, lse)

    # ------------------------------------------------------------------ the step
    def _pose_scale(self, B, pose_scale_u):
        """(u, r) of this micro-batch's pose-scale augmentation, fp32 [B] on the host: r = c ** u (migt.py:349-354).  u: the hashed draw
        (pose_scale.pose_scale_exponents), or ``pose_scale_u`` when given.  Each scene of each micro-batch of each rank draws its own u, as each
        MirroredStrategy replica runs its own tf.random.uniform (DESIGN.md section 6)."""
        if pose_scale_u is None:
            rank = dist.get_rank(self.group) if (dist.is_available() and dist.is_initialized()) else 0
            micro = 0 if self.pending in (0, self.ex.micro_batches) else self.pending
            u = PS.pose_scale_exponents(self.seed, self.iterations, rank, micro, B)
        else:
            u = torch.as_tensor(pose_scale_u, dtype=torch.float32).reshape(B).clone()
        return u, torch.pow(torch.tensor(float(self.cfg.random_pose_multiplier), dtype=torch.float32), u)

    def forward_backward(self, poses, tokens, pose_scale_u=None):
        """One micro-batch's loss and gradient.  ``pose_scale_u`` [B]: the exponents of the pose-scale augmentation in place of the hashed
        draw (random_pose_multiplier != 1 only)."""
        cfg, dev, p, g = self.cfg, self.device, self.p, self.g
        tokens = torch.as_tensor(tokens)
        B, T = tokens.shape[:2]
        Lt, d, V = self.model.n_image_tokens, cfg.d_model, cfg.n_embeddings
        S, skip = T * Lt, cfg.n_loss_skip
        ids = tokens.reshape(B, T, Lt).to(device=dev, dtype=torch.int32).contiguous()
        poses = torch.as_tensor(poses, dtype=torch.float32).to(dev).reshape(B * T, 7).contiguous()
        # get_model_input (migt.py:139-145); with random_pose_multiplier c != 1 scene b's xyz is also scaled by r_b = c ** u_b and its
        # predicted xyz divided by r_b before the position loss (:158-160)
        if cfg.random_pose_multiplier != 1.0:
            pose_u, pose_r = self._pose_scale(B, pose_scale_u)
            scene_mult = pose_r.to(dev)
            pin = PS.pose_model_input(poses, float(cfg.pose_multiplier), T, scene_mult)
        else:
            if pose_scale_u is not None:
                raise ValueError("pose_scale_u is given but random_pose_multiplier is 1: there is no pose-scale augmentation to draw")
            scene_mult = None
            mult = torch.tensor([cfg.pose_multiplier] * 3 + [1.0] * 4, dtype=torch.float32, device=dev)
            pin = (poses * mult).contiguous()
        # ---------------- embeddings: three streams (migt.py:354-405)
        pe_h = self._lin(pin, "pose_embedding.c_fc")
        pe = self._lin(self._gelu(pe_h), "pose_embedding.c_proj")                # [B*T, d]
        wte, wpe = p["wte.weight"], p["wpe.embeddings"]
        loc_rows = wte[self.model.localization_token].reshape(1, d).expand(B * T, d).contiguous()
        xs = [L.migt_embed(ids, 0, wte, wpe, pe, B * T, Lt), L.migt_embed(None, self.model.mask_token, wte, wpe, pe, B * T, Lt)]
        if self.use_loc:
            xs.append(L.migt_embed(ids, 0, wte, wpe, loc_rows, B * T, Lt))
        ns = len(xs)
        xs = [self._drop(x, 10 + s) for s, x in enumerate(xs)]
        tape = []
        for li in range(cfg.n_layer):
            pre = f"h.{li}."
            site = 100 + li * 20
            if self.bf16:
                # outs: bf16 attention outputs (c_proj's operands); vqk: what the fused backward needs in place of the probabilities
                outs, vqk = self._attention_fw16([self._ln(x, pre + "ln_1", torch.bfloat16) for x in xs], pre, B, S, Lt, site)
                probs = None
            else:
                a = [self._ln(x, pre + "ln_1") for x in xs]
                vqk = [self._lin(t, pre + "attn.c_attn") for t in a]
                outs, probs = self._attention_fw(vqk, B, S, Lt, site)
            ys = [self._drop(self._lin(o, pre + "attn.c_proj"), site + 4 + s) for s, o in enumerate(outs)]
            ys = [L.lincomb3(1.0, x, 1.0, y) for x, y in zip(xs, ys)]
            ln2_dt = torch.bfloat16 if self.bf16 else torch.float32
            hm = [self._lin(self._ln(y, pre + "ln_2", ln2_dt), pre + "mlp.c_fc") for y in ys]
            zs = [self._drop(self._lin(self._gelu(h), pre + "mlp.c_proj"), site + 8 + s) for s, h in enumerate(hm)]
            zs = [L.lincomb3(1.0, y, 1.0, z) for y, z in zip(ys, zs)]
            tape.append((xs, vqk, probs, outs, ys, hm))
            xs = zs
        # ---------------- heads and losses (migt.py:408-452)
        hn = [self._ln(x, "ln_f") for x in xs]
        denom = float(B * (T - skip) * Lt)
        view_ok = (torch.arange(T, device=dev) >= skip).to(torch.float32).repeat_interleave(Lt).repeat(B)        # [B*S] row mask
        logits = self._dgrad(hn[1], "wte")                                                                         # tied head (:417)
        ce_rows = L.cross_entropy_rows(logits, ids.reshape(-1), float(cfg.label_smoothing))
        ce = L.row_mean(ce_rows.reshape(B, S), skip * Lt)
        loss = ce * float(cfg.image_generation_weight)
        self.last = dict(ce_loss=ce, logits=logits.reshape(B, T, Lt, V))
        if scene_mult is not None:
            self.last.update(pose_scale_u=pose_u, pose_scale=pose_r)
        dhn = [None] * ns
        if self.pending in (0, self.ex.micro_batches):                            # the first micro-batch opens the accumulation window
            self.ex.reset(float(2.0 ** round(math.log2(denom)) if self.grad_seed_scale is None else self.grad_seed_scale), self.accumulate_steps)
            self.pending = 0
        else:
            self.ex.next_micro_batch()
        self._seed_scale = self.ex.seed_scale                                      # the window's: fixed from its first micro-batch
        ls = self.loss_scale * self._seed_scale                                   # gradient seeds carry the loss scale (1 in fp32) and the seed scale
        dlog = L.cross_entropy_grad(logits, ids.reshape(-1), (view_ok * (float(cfg.image_generation_weight) * ls / denom)).contiguous(),
                                    float(cfg.label_smoothing))
        # tied LM head backward: d hn1 = dlogits wte[:V];  d wte[:V] += dlogits^T hn1 (ready with the embeddings)
        dhn[1] = self._lin(dlog, "wte")
        self._lin_bw(dlog, hn[1], "wte", need_dx=False, last=False)
        if self.use_loc:
            pc_h = self._lin(hn[2], "pose_classifier.c_fc")
            raw = self._lin(self._gelu(pc_h), "pose_classifier.c_proj")            # [B*S, 7]
            if scene_mult is None:
                pl_rows, ol_rows = L.pose_loss_rows(raw, poses, Lt, float(cfg.pose_multiplier))
            else:
                pl_rows, ol_rows = PS.pose_loss_rows_scaled(raw, poses, Lt, float(cfg.pose_multiplier), T, scene_mult)
            pl, ol = L.row_mean(pl_rows.reshape(B, S), skip * Lt), L.row_mean(ol_rows.reshape(B, S), skip * Lt)
            lw_now = self.loc_weight
            if self.dynamic_pose:
                # DynamicLossWeightingCriterion (migt.py:107-120): P = sum_b (w0 + e^-w0 pos_b) + (w1 + e^-w1 ori_b), a scalar added to every
                # scene's loss; d mean(loss) / d w = lw (B - e^-w sum_b loss_b), d / d pos_b = lw e^-w0 (B times the plain-sum case)
                wkey = "pose_loss_weighting_criterion.pos_ori_weights"
                w01 = self.p[wkey].detach().double().cpu()
                e0, e1 = math.exp(-float(w01[0])), math.exp(-float(w01[1]))
                pls, ols = float(pl.double().sum()), float(ol.double().sum())
                pose_loss = torch.full_like(pl, float(B * (w01[0] + w01[1]) + e0 * pls + e1 * ols))
                dw01 = torch.tensor([lw_now * (B - e0 * pls) * ls, lw_now * (B - e1 * ols) * ls], dtype=torch.float32).to(dev)
                L.lincomb3(1.0, self.g[wkey], 1.0, dw01, out=self.g[wkey])       # added: the window's earlier micro-batches are in g
                self.ex.ready(wkey)
                ps, os_ = e0 * B, e1 * B
            else:
                pose_loss, ps, os_ = pl + ol, 1.0, 1.0
            loss = loss + pose_loss * lw_now
            self.last.update(pose_pos_loss=pl, pose_ori_loss=ol, pose_loss=pose_loss)
            row_w = (view_ok * (lw_now * ls / denom)).contiguous()
            if scene_mult is None:
                draw = L.pose_loss_grad(raw, poses, row_w, Lt, float(cfg.pose_multiplier), ps, os_)
            else:
                draw = PS.pose_loss_grad_scaled(raw, poses, row_w, Lt, float(cfg.pose_multiplier), T, scene_mult, ps, os_)
            dg_ = self._lin_bw(self._gelu(pc_h), draw, "pose_classifier.c_proj")
            dhn[2] = self._lin_bw(hn[2], L.gelu_bwd(pc_h, dg_), "pose_classifier.c_fc")
        else:
            self.ex.ready(*[k for k in self.order if k.startswith("pose_classifier.") or k.startswith("pose_loss_weighting_criterion.")])
        # ln_f backward (shared parameters: accumulate over the streams that carry a loss)
        dxs = [torch.zeros_like(xs[0])] + [None] * (ns - 1)
        live = [s for s in range(ns) if dhn[s] is not None]
        for s in live:
            dxs[s] = self._ln_bw(xs[s], dhn[s], "ln_f", last=(s == live[-1]))
        # ---------------- blocks, last to first
        for li in reversed(range(cfg.n_layer)):
            pre = f"h.{li}."
            site = 100 + li * 20
            xin, vqk, probs, outs, ys, hm = tape[li]
            dys = []
            for s in range(ns):
                dz = self._drop(dxs[s], site + 8 + s)
                last = s == ns - 1
                dgel = self._lin_bw(self._gelu(hm[s]), dz, pre + "mlp.c_proj", last=last)
                dm = self._lin_bw(self._ln(ys[s], pre + "ln_2"), L.gelu_bwd(hm[s], dgel), pre + "mlp.c_fc", last=last)
                dys.append(self._ln_bw(ys[s], dm, pre + "ln_2", add=dxs[s], last=last))
            if self.bf16:
                qk, vt, o32, lse = vqk
                do16 = torch.empty((ns, B * S, d), dtype=torch.bfloat16, device=dev)
                for s in range(ns):
                    self._lin_bw(o32[s], self._drop(dys[s], site + 4 + s), pre + "attn.c_proj", last=s == ns - 1, out16=do16[s])
                dvqk = L.attn_multiend_bwd(qk, vt, do16, o32, lse, B, S, ns, cfg.n_head, d, Lt, rate=float(cfg.dropout), seed=self._drop_seed(site))
            else:
                dos = []
                for s in range(ns):
                    dos.append(self._lin_bw(outs[s], self._drop(dys[s], site + 4 + s), pre + "attn.c_proj", last=s == ns - 1))
                dvqk = self._attention_bw(vqk, probs, dos, B, S, Lt, site)
            new_dxs = []
            for s in range(ns):
                last = s == ns - 1
                da = self._lin_bw(self._ln(xin[s], pre + "ln_1"), dvqk[s], pre + "attn.c_attn", last=last)
                new_dxs.append(self._ln_bw(xin[s], da, pre + "ln_1", add=dys[s], last=last))
            dxs = new_dxs
        # ---------------- embeddings backward
        dxs = [self._drop(dx, 10 + s) for s, dx in enumerate(dxs)]
        dpe = torch.zeros((B * T, d), dtype=torch.float32, device=dev)
        L.migt_embed_bwd(dxs[0], ids, 0, B * T, Lt, g["wte.weight"], g["wpe.embeddings"], dpe)
        L.migt_embed_bwd(dxs[1], None, self.model.mask_token, B * T, Lt, g["wte.weight"], g["wpe.embeddings"], dpe)
        if self.use_loc:
            dloc = torch.zeros((B * T, d), dtype=torch.float32, device=dev)
            L.migt_embed_bwd(dxs[2], ids, 0, B * T, Lt, g["wte.weight"], g["wpe.embeddings"], dloc)
            L.col_sums(dloc, g["wte.weight"][self.model.localization_token])
        dh_ = self._lin_bw(self._gelu(pe_h), dpe, "pose_embedding.c_proj")
        self._lin_bw(pin, L.gelu_bwd(pe_h, dh_), "pose_embedding.c_fc", need_dx=False)
        self.ex.ready("wpe.embeddings", "wte.weight")
        self.ex.check_complete()
        self.pending += 1
        self.last["loss_per_scene"] = loss
        return loss.mean()

    def _gelu(self, x):
        return L.gelu(x)

    # ------------------------------------------------------------------ schedule + optimizer (models/utils.py:310-564)
    def learning_rate(self, step=None):
        return warmup_cosine(self.iterations if step is None else step, self.init_lr, self.warmup_steps, self.total_steps, self.schedule_offset)

    def optimizer_step(self):
        """AdamW on the all-reduced gradients; returns whether the update was applied.

        bf16: Keras LossScaleOptimizer over TF 2.4's DynamicLossScale (migt.py:466-488).  The gradients carry the loss scale; one fp64 sum of
        squares of the flat gradient decides whether all of them are finite.  Non-finite: no update (weights and moments untouched), the
        scale halves (not below 1) and the good-step counter resets, but ``iterations`` still advances, as Keras's do_not_apply_fn does, so
        the learning-rate and localisation schedules move on.  Finite: the update runs on the unscaled gradients (clipping included), and
        when the counter has reached 1999 the scale doubles (if that is finite) and the counter resets, else the counter counts up.

        Under accumulation this runs once per window, on the sum of its micro-batches' gradients: one finiteness check, one skip or
        update.  Called on a partial window, it steps on the micro-batches accumulated so far."""
        self.ex.flush()
        self.ex.wait()
        self.pending = 0
        lr = self.learning_rate()
        self.iterations += 1
        ls = self.loss_scale
        if self.bf16:
            if not math.isfinite(float(L.sumsq(self.flat_g))):
                self.loss_scale = max(ls / 2.0, 1.0)
                self.loss_scale_counter = 0
                return False
            if self.loss_scale_counter == self.LOSS_SCALE_GROWTH_STEPS - 1:
                if math.isfinite(ls * 2.0):
                    self.loss_scale = ls * 2.0
                self.loss_scale_counter = 0
            else:
                self.loss_scale_counter += 1
        wd = float(self.cfg.weight_decay)
        clip = float(self.cfg.gradient_clip_val or 0.0)
        gs = (1.0 / (self.ex.world() * self.ex.micro_batches) if self.grad_reduce == "mean" else 1.0) / ls
        for k in self.order:
            cs = 1.0
            if clip > 0:                                                  # tf.clip_by_norm: g * clip / max(|g|, clip), per tensor
                nrm = math.sqrt(float(L.sumsq(self.g[k].reshape(-1)))) * gs
                cs = clip / max(nrm, clip)
            o, n = self.offs[k], self.p[k].numel()
            L.adamw_keras(self.flat_p[o:o + n], self.flat_g[o:o + n], self.flat_m[o:o + n], self.flat_v[o:o + n], lr=lr, beta1=self.betas[0],
                          beta2=self.betas[1], eps=self.eps, weight_decay=wd if (wd > 0 and self.decay[k]) else 0.0, step=self.iterations,
                          grad_scale=gs, clip_scale=cs)
        self._weights_changed()
        return True

    def _weights_changed(self):
        """flat_p has new values: drop the split-fp16 operand copies and rewrite the bf16 ones."""
        for r in self.dense.values():
            r.split.clear()
        if self.bf16:
            L.dense_weights_bf16(self._w16_table)

    def train_step(self, batch, pose_scale_u=None):
        """(poses [B,T,7], tokens [B,T,h,w]) -> dict(loss, ce_loss, [pose losses], acc, learning_rate, applied, pending) — migt.py:464-505.
        The metrics are this micro-batch's; ``applied``: an update ran after it (False inside an accumulation window and on a skipped
        non-finite bf16 window); ``pending``: micro-batches accumulated and not yet stepped on (0 after every optimizer step).
        ``pose_scale_u``: see forward_backward."""
        poses, tokens = batch
        loss = self.forward_backward(poses, tokens, pose_scale_u=pose_scale_u)
        lr = self.learning_rate()
        applied = self.optimizer_step() if self.pending == self.ex.micro_batches else False
        out = {k: float(torch.as_tensor(v, dtype=torch.float32).mean()) for k, v in self.last.items() if k.endswith("loss")}
        out["loss"] = float(loss)
        tok = torch.as_tensor(tokens).to(self.device)
        logits = self.last["logits"]
        pred = L.argmax_rows(logits.reshape(-1, logits.shape[-1])).reshape(tok.shape[0], tok.shape[1], -1)
        skip = self.cfg.n_loss_skip
        out["acc"] = float((pred[:, skip:] == tok.reshape(tok.shape[0], tok.shape[1], -1)[:, skip:]).float().mean())
        out["learning_rate"] = lr
        out["applied"], out["pending"] = bool(applied), self.pending
        if self.bf16:
            out["loss_scale"] = self.loss_scale
        return out
