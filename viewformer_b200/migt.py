"""MIGT context-view transformer — H100-native drop-in for the reference's Keras ``MIGT``.

Surface (viewformer/models/migt.py:241-455, 532-533):
    MIGT(config).load_state_dict(sd)
    model(dict(input_ids=int[B,T,8,8], poses=f32[B,T|T-1,7] [, output_poses=f32[B,T,7]]
               [, localization_tokens=int[B,T,8,8]]), training=False)
        -> dict(logits [B,T,8,8,n_embeddings], pose_prediction [B,T,64,7] (if use_localization), ...)
    .mask_token / .localization_token / .use_localization / .config / .reduce_cameras(x, axis)
plus the inference entry points the reference spreads over evaluate/*.py:
    .generate_codes(codes_ctx, poses)                 last-view argmax codes only (evaluate_transformer.py:118-123)
    .prefill_context(...) / .query(...)               context K/V cache (exact: block-causality makes context
                                                      states independent of the query view, SURVEY.md §3.3-7)

Weight names follow the reference's layer names (``h.<i>.attn.c_attn.weight`` [in,out], ``wte.weight`` [1026,d],
``wpe.embeddings`` [256,d] ...; see INTEGRATION.md for the TF checkpoint variable map).  c_attn columns are
[v | q | k] (migt.py:207-213); attention logits are NOT scaled by 1/sqrt(dh) (branching_attention.py:7).
"""
from collections import OrderedDict

import torch

from . import _lib as L
from .config import MIGTConfig, load_config
from .ops import Precision, Linear, gemm_nt, linear

LN_EPS = 1e-5   # migt.py:14


class MIGT:
    def __init__(self, config=None, precision="bf16", device="cuda", **config_overrides):
        if config is None:
            config = MIGTConfig(**config_overrides)
        self.config = load_config(config)
        cfg = self.config
        self.prec = Precision(precision)
        self.exact = Precision("fp32")
        self.device = torch.device(device)
        self.n_image_tokens = cfg.token_image_size ** 2
        self.n_embeddings = cfg.n_embeddings
        self.token_image_size = cfg.token_image_size
        self.d_model = cfg.d_model
        self.mask_token = cfg.n_embeddings                 # migt.py:256
        self.localization_token = cfg.n_embeddings + 1     # migt.py:257
        self.use_localization = cfg.use_localization       # migt.py:268-269
        self._train_counter = 0                            # Keras Model._train_counter: optimisation steps taken (migt.py:446)
        self._codebook_model = None
        self._sd = None
        self._w = None

    # ------------------------------------------------------------------ plumbing
    @property
    def codebook_model(self):
        return self._codebook_model

    @codebook_model.setter
    def codebook_model(self, model):
        self._codebook_model = model

    def param_shapes(self):
        """Ordered {name: shape}; names follow the reference's Keras layer names (migt.py:84-87, 288-315)."""
        cfg, d = self.config, self.config.d_model
        out = OrderedDict()
        out["wte.weight"] = (cfg.n_embeddings + 2, d)
        out["wpe.embeddings"] = (256, d)
        for n, (nx, nf) in (("pose_embedding.c_fc", (7, 2 * d)), ("pose_embedding.c_proj", (2 * d, d)),
                            ("pose_classifier.c_fc", (d, 2 * d)), ("pose_classifier.c_proj", (2 * d, 7))):
            out[n + ".weight"] = (nx, nf)
            out[n + ".bias"] = (1, nf)
        for i in range(cfg.n_layer):
            p = f"h.{i}."
            for ln in ("ln_1", "ln_2"):
                out[p + ln + ".gamma"] = (d,)
                out[p + ln + ".beta"] = (d,)
            for n, (nx, nf) in (("attn.c_attn", (d, 3 * d)), ("attn.c_proj", (d, d)), ("mlp.c_fc", (d, 4 * d)), ("mlp.c_proj", (4 * d, d))):
                out[p + n + ".weight"] = (nx, nf)
                out[p + n + ".bias"] = (1, nf)
        out["ln_f.gamma"] = (d,)
        out["ln_f.beta"] = (d,)
        if cfg.use_dynamic_pose_loss:
            out["pose_loss_weighting_criterion.pos_ori_weights"] = (2,)      # DynamicLossWeightingCriterion (migt.py:107-120)
        return out

    def expected_keys(self):
        return list(self.param_shapes().keys())

    def init_weights(self, seed=0):
        """Reference initialisers: TruncatedNormal(0.02) for wte / wpe / Conv1D weights (migt.py:26,85,314),
        zero biases, LayerNorm gamma 1 / beta 0."""
        g = torch.Generator().manual_seed(int(seed))
        sd = OrderedDict()
        for k, shp in self.param_shapes().items():
            if k.endswith("gamma"):
                sd[k] = torch.ones(shp)
            elif k.endswith("pos_ori_weights"):
                sd[k] = torch.tensor([0.0, -3.0])                           # migt.py:114
            elif k.endswith("beta") or k.endswith("bias"):
                sd[k] = torch.zeros(shp)
            else:
                sd[k] = torch.nn.init.trunc_normal_(torch.empty(shp), std=0.02, a=-0.04, b=0.04, generator=g)
        return self.load_state_dict(sd)

    _keys_to_ignore_on_load_unexpected = [r"h\.\d+\.attn\.bias"]      # migt.py:242 (causal-mask buffers of older checkpoints)

    @L.on_model_device
    def load_state_dict(self, state_dict, strict=True):
        import re
        ign = [re.compile(p) for p in self._keys_to_ignore_on_load_unexpected]
        sd = OrderedDict((k, v) for k, v in state_dict.items() if not any(r.fullmatch(k) for r in ign))
        if not strict:
            shapes = self.param_shapes()
            sd = OrderedDict((k, v) for k, v in sd.items() if k in shapes)
            if self._sd is not None:
                for k in shapes:
                    sd.setdefault(k, self._sd[k])
        if strict:
            want, got = set(self.expected_keys()), set(sd.keys())
            if want - got:
                raise RuntimeError(f"Missing keys: {want - got}")
            if got - want:
                raise RuntimeError(f"Unexpected keys: {got - want}")
        self._sd = OrderedDict((k, torch.as_tensor(v).detach().to("cpu").clone()) for k, v in sd.items())
        self._build()
        return self

    def state_dict(self):
        return OrderedDict((k, v.clone()) for k, v in self._sd.items())

    # ------------------------------------------------------------------ Keras checkpoint surface (train_transformer.py:106-129)
    def load_weights(self, filepath):
        """Keras ``model.load_weights(<dir>/model)`` of a TF2 object-graph checkpoint (viewformer/utils/tensorflow.py:57-61), read by
        the pure-Python TensorBundle reader (viewformer_b200/tf_checkpoint.py).  Returns a status object with ``expect_partial()``.
        On a compiled model the weights also go to the trainer and, when the file carries optimizer entries (``save_weights(...,
        include_optimizer=True)``), so do Adam's moments, the step counters and the loss scale — as Keras restores the optimizer of a
        compiled model, which finetune_transformer.py:85 relies on."""
        from . import tf_checkpoint
        self.load_state_dict(tf_checkpoint.load_state_dict(filepath, self.expected_keys()))
        trainer = getattr(self, "_trainer", None)
        if trainer is not None:
            trainer.load_state_dict(self._sd)
            state = tf_checkpoint.load_optimizer_state(filepath, self.expected_keys())
            if state is not None:
                trainer.load_optimizer_state(state)
                self._train_counter = trainer.train_counter

        class _Status:
            def expect_partial(self):
                return self

            def assert_consumed(self):
                return self
        return _Status()

    def save_weights(self, filepath, include_optimizer=False):
        """Keras ``model.save_weights``.  ``include_optimizer=True`` (a compiled model) adds what Keras stores for a compiled model — the
        optimizer's ``iter``, the ``m`` / ``v`` slot of every variable, the schedule's ``offset``, the loss scale (bf16) — so that
        ``load_weights`` on a compiled model resumes training (tf_checkpoint.OPTIMIZER_SCALARS lists the entries)."""
        from . import tf_checkpoint
        # object paths = the reference model's attribute names (wpe at the root, pose_classifier under pose_criterion): tf_checkpoint.object_paths
        tensors, slots = {tf_checkpoint.object_paths(k)[0]: v.numpy() for k, v in self.state_dict().items()}, None
        if include_optimizer:
            if getattr(self, "_trainer", None) is None:
                raise RuntimeError("save_weights(include_optimizer=True) needs a compiled model: call compile() first")
            tr = self._trainer
            if 0 < tr.pending < tr.ex.micro_batches:
                raise RuntimeError(f"save_weights(include_optimizer=True): {tr.pending} of {tr.ex.micro_batches} micro-batches of the "
                                   "accumulation window are pending; save after the step that closes the window")
            extra, slots = tf_checkpoint.optimizer_entries(self._trainer.optimizer_state())
            tensors.update(extra)
        tf_checkpoint.write_checkpoint(filepath, tensors, slots)

    def _build(self):
        L.load(require_device=True)
        sd, prec, dev, cfg = self._sd, self.prec, self.device, self.config
        d = cfg.d_model
        f32 = lambda t: t.to(dev, torch.float32).contiguous()
        w = dict(wte=f32(sd["wte.weight"]), wpe=f32(sd["wpe.embeddings"]))
        w["lm"] = Linear(sd["wte.weight"][: cfg.n_embeddings], None, prec, dev)        # tied head, first n_embeddings rows (:417)
        # pose MLPs stay fp32 (reference: dtype='float32' islands, migt.py:136,291); pose_multiplier folded into c_fc rows 0..2
        fc = sd["pose_embedding.c_fc.weight"].clone()
        fc[:3] = fc[:3] * cfg.pose_multiplier
        w["pe_fc"] = Linear(fc.t(), sd["pose_embedding.c_fc.bias"], self.exact, dev)
        w["pe_proj"] = Linear(sd["pose_embedding.c_proj.weight"].t(), sd["pose_embedding.c_proj.bias"], self.exact, dev)
        w["pc_fc"] = Linear(sd["pose_classifier.c_fc.weight"].t(), sd["pose_classifier.c_fc.bias"], self.exact, dev)
        w["pc_proj"] = Linear(sd["pose_classifier.c_proj.weight"].t(), sd["pose_classifier.c_proj.bias"], self.exact, dev)
        layers = []
        for i in range(cfg.n_layer):
            p = f"h.{i}."
            ca_w, ca_b = sd[p + "attn.c_attn.weight"], sd[p + "attn.c_attn.bias"].reshape(-1)    # [d,3d] cols = v|q|k
            layers.append(dict(
                ln1=(f32(sd[p + "ln_1.gamma"]), f32(sd[p + "ln_1.beta"])),
                ln2=(f32(sd[p + "ln_2.gamma"]), f32(sd[p + "ln_2.beta"])),
                qk=Linear(ca_w[:, d:].t(), ca_b[d:], prec, dev),              # [2d, d]: rows 0..d-1 -> q, d..2d-1 -> k
                v=Linear(ca_w[:, :d].t(), ca_b[:d], prec, dev),               # [d, d]
                proj=Linear(sd[p + "attn.c_proj.weight"].t(), sd[p + "attn.c_proj.bias"], prec, dev),
                fc=Linear(sd[p + "mlp.c_fc.weight"].t(), sd[p + "mlp.c_fc.bias"], prec, dev),
                fc2=Linear(sd[p + "mlp.c_proj.weight"].t(), sd[p + "mlp.c_proj.bias"], prec, dev)))
        w["layers"] = layers
        w["lnf"] = (f32(sd["ln_f.gamma"]), f32(sd["ln_f.beta"]))
        self._w = w

    def _in(self, x, dtype):
        t = torch.as_tensor(x)
        if t.device != self.device or t.dtype != dtype or not t.is_contiguous():
            t = t.to(device=self.device, dtype=dtype).contiguous()
        return t

    # ------------------------------------------------------------------ embeddings
    def _pose_embed(self, poses_rows):
        """pose MLP 7 -> 2d (GELU erf) -> d in fp32 (migt.py:139-145, 291, 354)."""
        h = linear(self.exact, poses_rows, self._w["pe_fc"], torch.float32, act=L.ACT_GELU)
        return linear(self.exact, h, self._w["pe_proj"], torch.float32)

    def _embed_stream(self, ids, fixed_token, pose_rows, B, T):
        Lt = self.n_image_tokens
        return L.migt_embed(ids, fixed_token, self._w["wte"], self._w["wpe"], pose_rows, B * T, Lt)

    # ------------------------------------------------------------------ transformer body
    def _attention(self, lw, a_list, B, T, kv_out=None):
        """BranchingAttention (migt.py:211-217 -> branching_attention.py:82-126) on normalised streams ``a_list``
        (each [B*S, d] in operand dtype).  Stream 0 is block-causal over its own keys; stream s>=1 attends to
        stream-0 keys of strictly earlier views plus its own view in its own stream.  Returns per-stream
        attention outputs [B*S, d] (operand dtype) before c_proj."""
        prec, cfg = self.prec, self.config
        d, H = cfg.d_model, cfg.n_head
        dh = d // H
        Lt = self.n_image_tokens
        S = T * Lt
        dev = a_list[0].device
        ns = len(a_list)
        # q|k rows and V^T of every stream, laid side by side: keys [B, ns*S, 2d], V^T [B, d, ns*S]
        qk = torch.empty((B, ns * S, 2 * d), dtype=prec.opd, device=dev)
        vt = torch.empty((B, d, ns * S), dtype=prec.opd, device=dev)
        for s, a in enumerate(a_list):
            gemm_nt(prec, a, lw["qk"].w, qk, M=S, N=2 * d, K=d, lda=d, ldb=d, ldc=2 * d, batch=(B, 1), a_bs=(S * d, 0),
                    b_bs=(0, 0), c_bs=(ns * S * 2 * d, 0), c_off=s * S * 2 * d, bias=lw["qk"].b, bias_mode=L.BIAS_N)
            gemm_nt(prec, lw["v"].w, a, vt, M=d, N=S, K=d, lda=d, ldb=d, ldc=ns * S, batch=(B, 1), a_bs=(0, 0),
                    b_bs=(S * d, 0), c_bs=(d * ns * S, 0), c_off=s * S, bias=lw["v"].b, bias_mode=L.BIAS_M)
        if kv_out is not None:
            kv_out.append((qk, vt))                      # context K (k half of qk) and V^T of this layer: the KV cache
        if ns == 1 and prec.opd == torch.bfloat16 and dh == 64:
            # single-stream forward (the generate() hot path): one fused wgmma kernel, no S x S tensor in HBM
            return [L.attn_block_causal(qk, vt, B, S, H, d, Lt)]
        if ns > 1 and prec.opd == torch.bfloat16 and dh == 64 and Lt == 64:
            # 3-stream forward (multi-context generation, localisation): the same fused kernel with the multi-end key-tile schedule
            return [L.attn_block_multiend(qk, vt, B, S, ns, s, H, d, Lt) for s in range(ns)]
        outs = []
        for s in range(ns):
            if s == 0:
                kc, koff, mask_mode = S, 0, 1                     # keys: stream 0 only, block-causal (>=)
            else:
                kc, koff, mask_mode = 2 * S, 0, 2                 # keys: [stream 0 | stream s]
            o = torch.empty((B * S, d), dtype=prec.opd, device=dev)
            scores = torch.empty((B, H, S, kc), dtype=torch.float32, device=dev)
            p = torch.empty((B, H, S, kc), dtype=prec.opd, device=dev)
            if s == 0:
                gemm_nt(prec, qk, qk, scores, M=S, N=S, K=dh, lda=2 * d, ldb=2 * d, ldc=S, batch=(B, H),
                        a_bs=(ns * S * 2 * d, dh), b_bs=(ns * S * 2 * d, dh), c_bs=(H * S * S, S * S), a_off=0, b_off=d,
                        causal_block=Lt, causal_skip_n=True)
                L.softmax_rows(scores, p, rows_total=B * H * S, rows_per_batch=S, cols=S, ld_in=S, ld_out=S, mask_mode=1, block=Lt)
                gemm_nt(prec, p, vt, o, M=S, N=dh, K=S, lda=S, ldb=ns * S, ldc=d, batch=(B, H), a_bs=(H * S * S, S * S),
                        b_bs=(d * ns * S, dh * ns * S), c_bs=(S * d, dh), causal_block=Lt)
            else:
                # logits vs stream-0 keys -> columns [0,S); vs own-stream keys -> columns [S,2S)
                for half, key_stream in ((0, 0), (1, s)):
                    gemm_nt(prec, qk, qk, scores, M=S, N=S, K=dh, lda=2 * d, ldb=2 * d, ldc=2 * S, batch=(B, H),
                            a_bs=(ns * S * 2 * d, dh), b_bs=(ns * S * 2 * d, dh), c_bs=(H * S * 2 * S, S * 2 * S),
                            a_off=s * S * 2 * d, b_off=key_stream * S * 2 * d + d, c_off=half * S)
                L.softmax_rows(scores, p, rows_total=B * H * S, rows_per_batch=S, cols=2 * S, ld_in=2 * S, ld_out=2 * S,
                               mask_mode=2, block=Lt)
                # P[:, :S] . V0 + P[:, S:] . Vs : two accumulating passes would need beta=1; instead gather the two
                # V^T panels side by side (they already are when s == 1; otherwise copy panel s next to panel 0)
                if s == 1:
                    vcat, ldv = vt, ns * S
                else:
                    vcat = torch.empty((B, d, 2 * S), dtype=prec.opd, device=dev)
                    vcat[:, :, :S].copy_(vt[:, :, :S]); vcat[:, :, S:].copy_(vt[:, :, s * S:(s + 1) * S])
                    ldv = 2 * S
                gemm_nt(prec, p, vcat, o, M=S, N=dh, K=2 * S, lda=2 * S, ldb=ldv, ldc=d, batch=(B, H),
                        a_bs=(H * S * 2 * S, S * 2 * S), b_bs=(d * ldv, dh * ldv), c_bs=(S * d, dh))
            outs.append(o)
        return outs

    def _block(self, lw, xs, B, T, kv_out=None):
        """Block.call (migt.py:230-238): pre-LN attention + pre-LN MLP over a list of streams (shared weights)."""
        prec = self.prec
        a = [L.layernorm(x, *lw["ln1"], out_dtype=prec.opd, eps=LN_EPS) for x in xs]
        att = self._attention(lw, a, B, T, kv_out)
        xs = [linear(prec, o, lw["proj"], torch.float32, residual=x) for o, x in zip(att, xs)]
        out = []
        for x in xs:
            m = L.layernorm(x, *lw["ln2"], out_dtype=prec.opd, eps=LN_EPS)
            hmid = linear(prec, m, lw["fc"], prec.opd, act=L.ACT_GELU)
            out.append(linear(prec, hmid, lw["fc2"], torch.float32, residual=x))
        return out

    def _body(self, xs, B, T, kv_out=None):
        for lw in self._w["layers"]:
            xs = self._block(lw, xs, B, T, kv_out)
        return xs

    def _lm_logits(self, h_rows_f32):
        """ln_f -> tied-embedding logits, first n_embeddings classes (migt.py:408, 417)."""
        hn = L.layernorm(h_rows_f32, *self._w["lnf"], out_dtype=self.prec.opd, eps=LN_EPS)
        return linear(self.prec, hn, self._w["lm"], torch.float32)

    def _lm_logits_last(self, h_rows_f32, B, T):
        """Same, for the last view's rows only — read in place through the GEMM's batch stride (no gather copy)."""
        cfg, Lt, d = self.config, self.n_image_tokens, self.config.d_model
        hn = L.layernorm(h_rows_f32, *self._w["lnf"], out_dtype=self.prec.opd, eps=LN_EPS)
        logits = torch.empty((B * Lt, cfg.n_embeddings), dtype=torch.float32, device=hn.device)
        lm = self._w["lm"]
        gemm_nt(self.prec, hn, lm.w, logits, M=Lt, N=lm.n, K=d, lda=d, ldb=d, ldc=lm.n, batch=(B, 1), a_bs=(T * Lt * d, 0),
                b_bs=(0, 0), c_bs=(Lt * lm.n, 0), a_off=(T - 1) * Lt * d)
        return logits

    def _pose_head(self, h_rows_f32, return_raw=False):
        """QuaternionPoseRepresentation.call without targets (migt.py:156-164), fp32."""
        hn = L.layernorm(h_rows_f32, *self._w["lnf"], out_dtype=torch.float32, eps=LN_EPS)
        raw = linear(self.exact, linear(self.exact, hn, self._w["pc_fc"], torch.float32, act=L.ACT_GELU), self._w["pc_proj"], torch.float32)
        pred = L.pose_postprocess(raw, self.config.pose_multiplier)
        return (pred, raw) if return_raw else pred

    def _localization_weight(self, step=None):
        """``self.localization_weight(self._train_counter)`` of migt.py:268, 446: the config's schedule string evaluated at the number of
        optimisation steps taken so far (``_train_counter``; 0 for a freshly loaded model, advanced by ``train_step``)."""
        from .schedules import parse
        sched = parse(self.config.localization_weight).with_total_steps(int(self.config.total_steps))
        return float(sched(self._train_counter if step is None else step))

    def _pose_loss(self, pl, ol):
        """pose_loss_weighting_criterion (migt.py:279-284): position + orientation loss, or — use_dynamic_pose_loss — the learned
        homoscedastic weighting  sum(w + exp(-w) * [pos, ori])  over the batch (migt.py:116-118), a scalar."""
        if not self.config.use_dynamic_pose_loss:
            return pl + ol, {}
        w = self._sd["pose_loss_weighting_criterion.pos_ori_weights"].to(torch.float64)
        pl64, ol64 = pl.double().cpu(), ol.double().cpu()
        total = (w[0] + torch.exp(-w[0]) * pl64).sum() + (w[1] + torch.exp(-w[1]) * ol64).sum()
        return total.to(torch.float32).to(pl.device), dict(dynamic_loss_weight_pos=float(w[0]), dynamic_loss_weight_ori=float(w[1]))

    # ------------------------------------------------------------------ reference call surface
    @L.on_model_device
    def __call__(self, inputs, training=False, compute_losses=False, last_only=False, **kwargs):
        """MIGT.call (migt.py:338-455), inference semantics (training=False; dropout inactive).
        ``last_only=True`` computes logits for the last view only (what evaluate_transformer.py:123 consumes)."""
        if training:
            raise NotImplementedError("the training-mode forward (dropout) lives in the optimisation step: use MIGT.train_step / "
                                      "viewformer_b200.train_migt.MIGTTrainer")
        if compute_losses and last_only:
            raise ValueError("compute_losses needs the logits of every view (last_only=False)")
        if self._w is None:
            raise RuntimeError("MIGT has no weights: call load_state_dict() first")
        cfg = self.config
        ids_in = torch.as_tensor(inputs["input_ids"])
        orig_shape = list(ids_in.shape)
        B, T = orig_shape[0], orig_shape[1]
        Lt, d = self.n_image_tokens, cfg.d_model
        ids = self._in(ids_in.reshape(B, T, -1), torch.int32)
        assert ids.shape[2] == Lt, "input_ids must hold token_image_size**2 tokens per view"
        if kwargs.get("validate_ids", compute_losses):
            # the embedding gather and the cross-entropy label read are unchecked on the device: ids beyond the table
            # (or a MASK / LOC token used as a CE label) would read out of bounds -> fail here instead (one D2H sync)
            lo, hi = int(ids.min()), int(ids.max())
            limit = cfg.n_embeddings if compute_losses else cfg.n_embeddings + 2
            if lo < 0 or hi >= limit:
                raise ValueError(f"input_ids out of range [{lo}, {hi}]: " + ("cross-entropy labels must be real tokens < n_embeddings"
                                 if compute_losses else "ids must be < n_embeddings + 2"))
        poses = torch.as_tensor(inputs["poses"])
        if poses.dtype != torch.float32:
            raise AssertionError("poses must be float32")            # tf.debugging.assert_type, migt.py:346
        poses = self._in(poses, torch.float32)
        Tp = poses.shape[1]
        out_poses = inputs.get("output_poses")
        loc_tokens = inputs.get("localization_tokens")
        if compute_losses:                                       # migt.py:364-373: teacher-forced evaluation streams
            if Tp != T:
                raise AssertionError("compute_losses needs one pose per view")
            if loc_tokens is None and self.use_localization:
                loc_tokens = ids
            if out_poses is None:
                out_poses = poses
        wte = self._w["wte"]

        pose_rows = torch.empty((B, T, d), dtype=torch.float32, device=self.device)
        pe = self._pose_embed(poses.reshape(B * Tp, 7)).reshape(B, Tp, d)
        if Tp == T:
            pose_rows = pe
        else:
            if not self.use_localization:
                raise AssertionError("poses has fewer views than input_ids and the model has no localization token")
            pose_rows[:, :Tp].copy_(pe)
            pose_rows[:, Tp:].copy_(wte[self.localization_token])       # migt.py:387-390
        xs = [self._embed_stream(ids, 0, pose_rows.reshape(B * T, d), B, T)]
        gen_ptr = pose_ptr = 0
        if out_poses is not None:
            op = self._in(out_poses, torch.float32)
            ope = self._pose_embed(op.reshape(B * T, 7))
            xs.append(self._embed_stream(None, self.mask_token, ope, B, T))          # migt.py:393-396
            gen_ptr = len(xs) - 1
        if loc_tokens is not None:
            lt = self._in(torch.as_tensor(loc_tokens).reshape(B, T, -1), torch.int32)
            loc_rows = wte[self.localization_token].reshape(1, d).expand(B * T, d).contiguous()
            xs.append(self._embed_stream(lt, 0, loc_rows, B, T))                     # migt.py:398-401
            pose_ptr = len(xs) - 1
        xs = self._body(xs, B, T)

        out = {}
        if last_only:
            out["logits"] = self._lm_logits_last(xs[gen_ptr], B, T).reshape(B, 1, *orig_shape[2:], cfg.n_embeddings)
        else:
            out["logits"] = self._lm_logits(xs[gen_ptr]).reshape(orig_shape + [cfg.n_embeddings])
        loss = 0
        skip = cfg.n_loss_skip
        if compute_losses:                                       # migt.py:417-423
            ce_rows = L.cross_entropy_rows(out["logits"].reshape(B * T * Lt, cfg.n_embeddings), ids.reshape(-1),
                                           float(cfg.label_smoothing))
            out["ce_loss"] = L.row_mean(ce_rows.reshape(B, T * Lt), skip * Lt)
            loss = out["ce_loss"] * float(cfg.image_generation_weight)
        if self.use_localization:
            if compute_losses:                                   # migt.py:425-448, 165-177
                pred, raw = self._pose_head(xs[pose_ptr], return_raw=True)
                pl_rows, ol_rows = L.pose_loss_rows(raw, poses.reshape(B * T, 7).contiguous(), Lt, float(cfg.pose_multiplier))
                pl = L.row_mean(pl_rows.reshape(B, T * Lt), skip * Lt)
                ol = L.row_mean(ol_rows.reshape(B, T * Lt), skip * Lt)
                w = self._localization_weight()
                pose_loss, wc_metrics = self._pose_loss(pl, ol)
                out.update(wc_metrics)
                out["pose_pos_loss"], out["pose_ori_loss"], out["pose_loss"] = pl, ol, pose_loss
                out["localization_weight"] = w
                loss = loss + pose_loss * w
            else:
                pred = self._pose_head(xs[pose_ptr])
            out["pose_prediction"] = pred.reshape(B, T, Lt, 7)
        out["loss"] = loss
        return out

    def reduce_cameras(self, cameras, axis=-2):
        """QuaternionPoseRepresentation.reduce (migt.py:150-154, 123-129): host-side, a handful of floats."""
        from .generate import reduce_cameras
        return reduce_cameras(cameras, axis)

    # ------------------------------------------------------------------ Keras training surface (migt.py:457-505)
    def compile(self, optimizer=None, **kwargs):
        """migt.py:457-462: AdamWeightDecay + 2000-step warm-up + cosine decay; the trainer owns the flat parameter / gradient buffers.
        Keyword arguments go to MIGTTrainer.  ``precision="bf16"`` selects the reference's 16-bit recipe (--fp16): bf16 tensor-core
        operands for the dense layers and the fused attention forward and backward, fp32 master weights, and dynamic loss scaling
        (LossScaleOptimizer semantics; ``train_step`` then reports ``loss_scale``).  It needs d_model / n_head == 64 and
        token_image_size == 8.  ``precision="fp32"`` (the default) is the fp32-faithful step."""
        from .train_migt import MIGTTrainer
        self._trainer = optimizer if optimizer is not None else MIGTTrainer(self, **kwargs)
        return self._trainer

    @L.on_model_device
    def train_step(self, batch):
        """(poses [B,T,7], tokens [B,T,h,w]) -> metrics dict; one optimisation step (forward, backward, gradient exchange, AdamW).
        The model serves inference with the updated weights right away (they are re-laid-out for the inference kernels)."""
        if getattr(self, "_trainer", None) is None:
            self.compile()
        out = self._trainer.train_step(batch)
        if not out["pending"]:                          # inside an accumulation window the weights have not moved
            self.load_state_dict(self._trainer.state_dict())
        self._train_counter = self._trainer.train_counter
        return out

    def finetune(self, checkpoint, *, learning_rate, total_steps, **trainer_kwargs):
        """finetune_transformer.py:72-86: a new optimizer (new peak rate, new horizon) that takes over the moments and ``iterations`` of
        ``checkpoint`` (written with ``save_weights(..., include_optimizer=True)``) and whose warm-up and decay start at the restored
        ``iterations`` (``lr_schedule.offset.assign(optimizer.iterations)``); Adam's bias correction and the dropout seed carry on from
        ``iterations``, the localisation-weight schedule starts again at 0.  Returns the trainer."""
        import warnings
        from . import tf_checkpoint
        self.load_state_dict(tf_checkpoint.load_state_dict(checkpoint, self.expected_keys()))
        trainer = self.compile(learning_rate=learning_rate, total_steps=total_steps, **trainer_kwargs)
        state = tf_checkpoint.load_optimizer_state(checkpoint, self.expected_keys())
        if state is None:
            warnings.warn(f"{checkpoint} carries no optimizer entries: fine-tuning starts with a fresh optimizer")
        else:
            trainer.load_optimizer_state(state)
        trainer.schedule_offset = trainer.iterations
        trainer.train_counter = self._train_counter = 0
        return trainer

    # ------------------------------------------------------------------ Keras evaluation steps (migt.py:507-541)
    @L.on_model_device
    def test_step(self, batch):
        """(poses [B,T,7], tokens [B,T,h,w]) -> dict of scalars: losses of ``call(compute_losses=True)``, token accuracy and, with
        a codebook attached, the PSNR between the decoded predicted and true last views (migt.py:507-530)."""
        poses, tokens = batch
        out = self(dict(poses=poses, input_ids=tokens), compute_losses=True, training=False)
        res = {k: float(torch.as_tensor(v, dtype=torch.float32).mean()) for k, v in out.items()
               if k in ("loss", "ce_loss", "pose_loss", "pose_pos_loss", "pose_ori_loss", "localization_weight", "dynamic_loss_weight_pos",
                        "dynamic_loss_weight_ori")}                  # every output that has a Keras metric of its name (migt.py:260-283, :510-512)
        tok = self._in(torch.as_tensor(tokens), torch.int64)
        logits = out["logits"]
        pred = L.argmax_rows(logits.reshape(-1, logits.shape[-1])).reshape(tok.shape)
        skip = self.config.n_loss_skip
        res["acc"] = float((pred[:, skip:] == tok[:, skip:]).float().mean())            # _compute_accuracy, first n_loss_skip views excluded
        if "pose_prediction" in out:
            from .metrics import camera_position_error, camera_orientation_error
            pp = out["pose_prediction"][:, skip:].cpu()
            gt = torch.as_tensor(poses)[:, skip:, None].cpu()
            res["pose_pos_err"] = float(camera_position_error(pp, gt).mean())
            res["pose_ori_err"] = float(camera_orientation_error(pp, gt.expand_as(pp)).nan_to_num(0.0).mean())
        if self._codebook_model is not None:
            from .metrics import image_metrics
            gen = self._codebook_model.decode_code_u8(pred[:, -1])
            gt_img = self._codebook_model.decode_code_u8(tok[:, -1])
            res["psnr"] = float(image_metrics(gt_img, gen, self.device)["psnr"].mean())
        return res

    @L.on_model_device
    def predict_step(self, batch):
        """migt.py:535-541: decoded images of the teacher-forced argmax tokens and of the true tokens (float NHWC in [-1, 1])."""
        poses, tokens = batch
        logits = self(dict(poses=poses, input_ids=tokens), compute_losses=True, training=False)["logits"]
        side = self.token_image_size
        gen = L.argmax_rows(logits.reshape(-1, logits.shape[-1])).reshape(-1, self.config.sequence_size, side, side)
        gen = torch.where(gen < self.n_embeddings, gen, torch.zeros_like(gen))
        tok = self._in(torch.as_tensor(tokens), torch.int64)
        return {"decoded_image": self._codebook_model.decode_code_nhwc(gen.reshape(-1, side, side)), "latent_code": gen,
                "ground_truth_image": self._codebook_model.decode_code_nhwc(tok.reshape(-1, side, side))}

    # ------------------------------------------------------------------ context KV cache (BASELINE config 5)
    @L.on_model_device
    def prefill_context(self, codes_ctx, poses_ctx):
        """Run the context views once and keep every layer's K / V^T.  Exact: the transformer is block-causal over
        views, so context hidden states never depend on the query view (SURVEY.md §3.3-7, oracle invariant (ii)).
        codes_ctx int [B,Tc,8,8]; poses_ctx f32 [B,Tc,7] (already relative / normalised)."""
        if self._w is None:
            raise RuntimeError("MIGT has no weights: call load_state_dict() first")
        codes_ctx = torch.as_tensor(codes_ctx)
        B, Tc = codes_ctx.shape[0], codes_ctx.shape[1]
        d = self.config.d_model
        ids = self._in(codes_ctx.reshape(B, Tc, -1), torch.int32)
        poses = self._in(poses_ctx, torch.float32)
        pe = self._pose_embed(poses.reshape(B * Tc, 7))
        xs = [self._embed_stream(ids, 0, pe, B, Tc)]
        kv = []
        self._body(xs, B, Tc, kv_out=kv)
        cache = dict(kv=kv, B=B, Tc=Tc)
        Lt, H = self.n_image_tokens, self.config.n_head
        # the query view goes to the start of a 128-row tile: with an odd number of context views one view slot stays empty (its keys are
        # skipped by the kernel), otherwise half of the decode tile's softmax work would recompute the last context view
        pad = (Tc * Lt) % 128 // Lt if Lt == 64 else 0
        S_tot = (Tc + pad + 1) * Lt
        if self.prec.opd == torch.bfloat16 and d // H == 64 and ((Tc + pad) * Lt) % 128 == 0:
            # fused decode: keep every layer's q|k rows and V^T columns in buffers with room for ONE more view, so that a query is
            # "append the view, run the fused block-causal kernel on the last 128-row tile" — no [Nq,H,64,S] score tensor in HBM
            fq, fv = [], []
            for qk, vt in kv:
                qk_c = torch.empty((B, S_tot, 2 * d), dtype=qk.dtype, device=qk.device)
                vt_c = torch.empty((B, d, S_tot), dtype=vt.dtype, device=vt.device)
                qk_c[:, : Tc * Lt].copy_(qk)
                vt_c[:, :, : Tc * Lt].copy_(vt)
                fq.append(qk_c)
                fv.append(vt_c)
            cache["fused"] = dict(qk=fq, vt=fv, S_tot=S_tot, q_row0=(Tc + pad) * Lt, skip_view=(Tc if pad else -1),
                                  out=torch.empty((B * S_tot, d), dtype=torch.bfloat16, device=self.device))
        return cache

    def _query_block(self, lw, x, qk_c, vt_c, Nq, Bc, S_ctx):
        """One transformer block for Nq mask-token query views (64 rows each) against cached context K / V^T."""
        prec, cfg = self.prec, self.config
        d, H = cfg.d_model, cfg.n_head
        dh, Lt = d // H, self.n_image_tokens
        ld = S_ctx + Lt
        dev = x.device
        shared = Bc == 1 and Nq > 1                       # every query reads the same scene's cache (stride-0 batch)
        a = L.layernorm(x, *lw["ln1"], out_dtype=prec.opd, eps=LN_EPS)
        qk_q = linear(prec, a, lw["qk"], prec.opd)                                                   # [Nq*Lt, 2d] = q | k
        vt_q = torch.empty((Nq, d, Lt), dtype=prec.opd, device=dev)
        gemm_nt(prec, lw["v"].w, a, vt_q, M=d, N=Lt, K=d, lda=d, ldb=d, ldc=Lt, batch=(Nq, 1), a_bs=(0, 0), b_bs=(Lt * d, 0),
                c_bs=(d * Lt, 0), bias=lw["v"].b, bias_mode=L.BIAS_M)
        scores = torch.empty((Nq, H, Lt, ld), dtype=torch.float32, device=dev)
        cb = 0 if shared else S_ctx * 2 * d
        gemm_nt(prec, qk_q, qk_c, scores, M=Lt, N=S_ctx, K=dh, lda=2 * d, ldb=2 * d, ldc=ld, batch=(Nq, H), a_bs=(Lt * 2 * d, dh),
                b_bs=(cb, dh), c_bs=(H * Lt * ld, Lt * ld), b_off=d)                                 # vs cached context keys
        gemm_nt(prec, qk_q, qk_q, scores, M=Lt, N=Lt, K=dh, lda=2 * d, ldb=2 * d, ldc=ld, batch=(Nq, H), a_bs=(Lt * 2 * d, dh),
                b_bs=(Lt * 2 * d, dh), c_bs=(H * Lt * ld, Lt * ld), b_off=d, c_off=S_ctx)             # vs the view's own keys
        p = torch.empty((Nq, H, Lt, ld), dtype=prec.opd, device=dev)
        L.softmax_rows(scores, p, rows_total=Nq * H * Lt, rows_per_batch=Lt, cols=ld, ld_in=ld, ld_out=ld)   # all keys visible
        o1 = torch.empty((Nq * Lt, d), dtype=torch.float32, device=dev)
        gemm_nt(prec, p, vt_c, o1, M=Lt, N=dh, K=S_ctx, lda=ld, ldb=S_ctx, ldc=d, batch=(Nq, H), a_bs=(H * Lt * ld, Lt * ld),
                b_bs=(0 if shared else d * S_ctx, dh * S_ctx), c_bs=(Lt * d, dh))
        o = torch.empty((Nq * Lt, d), dtype=prec.opd, device=dev)
        gemm_nt(prec, p, vt_q, o, M=Lt, N=dh, K=Lt, lda=ld, ldb=Lt, ldc=d, batch=(Nq, H), a_bs=(H * Lt * ld, Lt * ld),
                b_bs=(d * Lt, dh * Lt), c_bs=(Lt * d, dh), a_off=S_ctx, residual=o1)                  # + own-view values
        x = linear(prec, o, lw["proj"], torch.float32, residual=x)
        m = L.layernorm(x, *lw["ln2"], out_dtype=prec.opd, eps=LN_EPS)
        hmid = linear(prec, m, lw["fc"], prec.opd, act=L.ACT_GELU)
        return linear(prec, hmid, lw["fc2"], torch.float32, residual=x)

    def _query_block_fused(self, lw, x, qk_c, vt_c, fz, Nq):
        """Decode step of one block on the fused kernel: the query view's q|k rows / V^T columns are written behind the cached context
        (at the start of a 128-row tile, see prefill_context) and the block-causal kernel runs on that tile only."""
        prec, cfg = self.prec, self.config
        d, H, Lt = cfg.d_model, cfg.n_head, self.n_image_tokens
        S_tot, r0, out_buf = fz["S_tot"], fz["q_row0"], fz["out"]
        a = L.layernorm(x, *lw["ln1"], out_dtype=prec.opd, eps=LN_EPS)
        gemm_nt(prec, a, lw["qk"].w, qk_c, M=Lt, N=2 * d, K=d, lda=d, ldb=d, ldc=2 * d, batch=(Nq, 1), a_bs=(Lt * d, 0), b_bs=(0, 0),
                c_bs=(S_tot * 2 * d, 0), c_off=r0 * 2 * d, bias=lw["qk"].b, bias_mode=L.BIAS_N)
        gemm_nt(prec, lw["v"].w, a, vt_c, M=d, N=Lt, K=d, lda=d, ldb=d, ldc=S_tot, batch=(Nq, 1), a_bs=(0, 0), b_bs=(Lt * d, 0),
                c_bs=(d * S_tot, 0), c_off=r0, bias=lw["v"].b, bias_mode=L.BIAS_M)
        L.attn_block_causal(qk_c, vt_c, Nq, S_tot, H, d, Lt, first_query=r0, out=out_buf, skip_view=fz["skip_view"])
        xn = torch.empty_like(x)
        gemm_nt(prec, out_buf, lw["proj"].w, xn, M=Lt, N=d, K=d, lda=d, ldb=d, ldc=d, batch=(Nq, 1), a_bs=(S_tot * d, 0), b_bs=(0, 0),
                c_bs=(Lt * d, 0), a_off=r0 * d, bias=lw["proj"].b, bias_mode=L.BIAS_N, residual=x)
        m = L.layernorm(xn, *lw["ln2"], out_dtype=prec.opd, eps=LN_EPS)
        hmid = linear(prec, m, lw["fc"], prec.opd, act=L.ACT_GELU)
        return linear(prec, hmid, lw["fc2"], torch.float32, residual=xn)

    @L.on_model_device
    def query(self, cache, query_poses, return_logits=False):
        """Novel-view codes for query poses against a prefilled context.  query_poses f32 [Nq,7]; Nq == cache batch
        (one query per scene) or cache batch == 1 (many queries share one scene, evaluate_transformer_multictx_allimg.py:141-173).
        Only the 64 mask tokens of each query view are computed: 14 GFLOP/view instead of 249 at 19 context views."""
        qp = self._in(query_poses, torch.float32).reshape(-1, 7)
        Nq, Bc, Tc = qp.shape[0], cache["B"], cache["Tc"]
        if not (Nq == Bc or Bc == 1):
            raise ValueError(f"{Nq} query poses for a cache of {Bc} scenes: need one per scene, or a single shared scene")
        Lt = self.n_image_tokens
        S_ctx = Tc * Lt
        x = self._embed_stream(None, self.mask_token, self._pose_embed(qp), Nq, 1)
        fz = cache.get("fused")
        if fz is not None and Nq == Bc:
            for lw, qk_c, vt_c in zip(self._w["layers"], fz["qk"], fz["vt"]):
                x = self._query_block_fused(lw, x, qk_c, vt_c, fz, Nq)
        else:
            for lw, (qk_c, vt_c) in zip(self._w["layers"], cache["kv"]):
                x = self._query_block(lw, x, qk_c, vt_c, Nq, Bc, S_ctx)
        logits = self._lm_logits(x)
        side = self.token_image_size
        codes = L.argmax_rows(logits).reshape(Nq, side, side)
        return (codes, logits.reshape(Nq, side, side, -1)) if return_logits else codes

    # ------------------------------------------------------------------ fast inference entry points
    @L.on_model_device
    def generate_codes(self, codes_ctx, poses):
        """Context codes [B,T-1,8,8] + poses [B,T,7] (already relative/normalised) -> argmax codes of view T
        (evaluate_transformer.py:118-123 without materialising logits of the context views)."""
        codes_ctx = torch.as_tensor(codes_ctx)
        B = codes_ctx.shape[0]
        side = self.token_image_size
        mask = torch.full((B, 1, side, side), self.mask_token, dtype=codes_ctx.dtype, device=codes_ctx.device)
        ids = torch.cat([codes_ctx.reshape(B, -1, side, side), mask], 1)
        logits = self({"input_ids": ids, "poses": poses}, last_only=True)["logits"]
        return L.argmax_rows(logits.reshape(-1, self.n_embeddings)).reshape(B, side, side)
