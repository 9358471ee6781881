"""Codebook training step — forward + backward + Adam + data-parallel gradient exchange, on libvf_b200 kernels.

Reference: viewformer/models/vqgan_th.py:395-423 (forward, _compute_loss, training_step), :443-445 (Adam, betas (0.5, 0.9)),
models/utils_th.py:32-68 (QuantizeEMA: straight-through estimator, codebook moved by EMA — not by the gradient — with the
statistics all-reduced across ranks), train/train_codebook_th.py:39-41 (DDP: gradients averaged over ranks).  fp32, as the
reference requires (vqgan_th.py:326); LPIPS is not available offline, so ``perceptual_weight`` must be 0 (SURVEY.md §8c).

    trainer = VQGANTrainer(VQGAN(cfg, precision="fp32").load_state_dict(sd))
    loss = trainer.training_step(x)        # x f32 NCHW in [-1, 1]: forward, backward, gradient all-reduce, Adam, codebook EMA
    trainer.export_state_dict()            # reference-keyed weights after the step

Data layout: every trainable tensor lives in ONE flat fp32 buffer (kernel layouts: conv [kh*kw*Cin, Cout], dense [out, in]) with a
twin flat gradient buffer ordered by backward completion (decoder.conv_out first, encoder.conv_in last), both owned by the trainers'
shared gradient exchange (``dist.GradExchange``), so that
  * the data-parallel exchange is a handful of large NCCL all-reduces over contiguous buckets, each launched (async) the moment
    the backward pass has produced its last gradient — the transfers ride under the remaining backward kernels;
  * Adam is one kernel launch over the whole model (``gradient_clip_val`` > 0: the global-norm clip the reference's Lightning trainer
    applies first, folded into Adam's gradient scale).
Activations needed by the backward pass are kept on a tape; GroupNorm+swish outputs are recomputed from the saved statistics.

Arithmetic: fp32 throughout, as the reference requires.  The 3x3 stride-1 convolutions with tensor-core-sized channel counts run
their forward pass and their data gradient on the exact split-fp16 tensor-core kernels (fp32-faithful results from three fp16 MMA passes,
DESIGN.md 5.3; ``VF_TRAIN_TC=0`` keeps everything on the CUDA cores), and their weight gradient as nine exact GEMMs over the pixel axis
(``_lib.conv_wgrad_tc``) when both channel counts are multiples of 128; strided / upsampling convs, 1x1 layers and the remaining weight
gradients use the fp32 CUDA-core kernels.  The backward pass runs on loss seeds multiplied by a power of two near the number of output
elements (``grad_seed_scale``), because the split is only fp32-faithful for operands of magnitude 2^-10 .. 2^15 and the plain seeds
(1 / numel) are far below that; the gradient buffer is unscaled bucket by bucket, so every result outside the backward pass is unscaled.

``precision="bf16"`` (BASELINE configs[3]: bf16 activations over fp32 master weights) runs every conv that a bf16-built model puts on the
tensor cores (3x3, Cin % 64 == 0, Cout % 16 == 0, Cout >= 64) as ONE bf16 wgmma pass: forward (stride-2 convs on the space-to-depth
operand), data gradient (flipped bf16 weights) and weight gradient (``_lib.conv_wgrad_bf16``, bf16 operands transposed with GroupNorm(+swish)
or the x2 upsample applied on the way).  Accumulation, conv outputs (the residual stream), GroupNorm statistics and backward, the loss, the
gradient buffers, the all-reduce, Adam and the whole quantizer block stay fp32, as do conv_in / conv_out, the 1x1 layers, the attention
blocks and the stride-2 convs' gradients.  No loss scaling: bf16 has fp32's exponent range.  The bf16 weight operands are rewritten from
the fp32 master weights by one kernel after every Adam step.
"""
import json
import math
import os
import warnings

import torch

from . import _lib as L
from .dist import GradExchange
from .ops import linear
from .vqgan import tc_conv_shape_ok


_REGISTERED = dict(top=("encoder", "decoder", "quantize", "quant_conv", "post_quant_conv"), mid=("block_1", "attn_1", "block_2"),
                   encoder=("conv_in", "down", "mid", "norm_out", "conv_out"), decoder=("conv_in", "mid", "up", "norm_out", "conv_out"),
                   level=("block", "attn", "downsample", "upsample"))


def _registration_key(name):
    """Where the reference module tree registers the module that owns ``name`` (vqgan_th.py:159-197, 249-285, 329-333): per resolution
    level all ResnetBlocks, then all AttnBlocks, then the resampling conv — not the order they run in."""
    parts = name.split(".")
    key = [_REGISTERED["top"].index(parts[0])]
    if parts[0] in ("encoder", "decoder"):
        key.append(_REGISTERED[parts[0]].index(parts[1]))
        if parts[1] in ("down", "up"):
            key += [int(parts[2]), _REGISTERED["level"].index(parts[3])] + ([int(parts[4])] if parts[3] in ("block", "attn") else [])
        elif parts[1] == "mid":
            key.append(_REGISTERED["mid"].index(parts[2]))
    return key


def trainable_names(model):
    """Reference state_dict keys of the tensors Adam updates, in the order of the reference module's ``parameters()`` (encoder, decoder,
    [Quantize's codebook,] quant_conv, post_quant_conv; QuantizeEMA holds buffers only) — the order ``torch.optim.Adam.state_dict()``
    numbers them in."""
    names = [k for k in model.param_shapes() if not (model.quantizer == "ema" and k.startswith("quantize."))]
    return sorted(names, key=_registration_key)                   # stable: a module's own tensors keep their order


def adam_state_dict(names, exp_avg, exp_avg_sq, step, lr, betas, eps):
    """``torch.optim.Adam.state_dict()`` (what a Lightning checkpoint keeps in ``optimizer_states[i]``) over the parameters ``names``:
    per-parameter state keyed by the parameter's position, one parameter group."""
    state = {i: dict(step=torch.tensor(float(step)), exp_avg=exp_avg[k], exp_avg_sq=exp_avg_sq[k]) for i, k in enumerate(names)}
    group = dict(lr=float(lr), betas=tuple(betas), eps=float(eps), weight_decay=0, amsgrad=False, maximize=False, foreach=None,
                 capturable=False, differentiable=False, fused=None, params=list(range(len(names))))
    return dict(state=state, param_groups=[group])


def read_adam_state_dict(osd, names):
    """Inverse of ``adam_state_dict``: dict(exp_avg, exp_avg_sq, step_count, lr, betas, eps).  A state written before the first step has
    no per-parameter entries: zero moments, step 0."""
    (group,) = osd["param_groups"]
    if len(group["params"]) != len(names):
        raise RuntimeError(f"optimizer state holds {len(group['params'])} parameters, the model has {len(names)}")
    states = [osd["state"].get(i) for i in group["params"]]
    if any(st is None for st in states) and any(st is not None for st in states):
        raise RuntimeError("optimizer state holds moments for some parameters only")
    steps = {int(st["step"]) for st in states if st is not None} or {0}
    if len(steps) != 1:
        raise RuntimeError(f"optimizer state holds different step counts {sorted(steps)}")
    out = dict(step_count=steps.pop(), lr=float(group["lr"]), betas=tuple(group["betas"]), eps=float(group["eps"]), exp_avg={}, exp_avg_sq={})
    for k, st in zip(names, states):
        if st is not None:
            out["exp_avg"][k], out["exp_avg_sq"][k] = st["exp_avg"], st["exp_avg_sq"]
    return out


class _P:
    """One trainable tensor: kernel-layout view into the flat parameter buffer, how to re-home it in the model, and how to export it."""

    def __init__(self, name, tensor, setter, kind, part=None, cin=None):
        self.name, self.tensor, self.setter, self.kind, self.part, self.cin = name, tensor, setter, kind, part, cin


def conv_routes(precision, use_tc, k, cin, cout, stride=1, upsample=False, out=False):
    """Kernel routes (forward, data gradient, weight gradient) of one conv: "bf16" (single-pass bf16 wgmma), "split" (the exact split-fp16
    tensor-core kernels) or "cuda" (the fp32 CUDA-core kernels).  ``use_tc``: VF_TRAIN_TC is not 0; ``upsample``: the conv runs on the x2
    map of its input; ``out``: a conv_out, whose backward pass the bf16 step runs on the fp32 step's kernels."""
    wgrad_split = "split" if use_tc and k == 3 and stride == 1 and cin % 128 == 0 and cout % 128 == 0 else "cuda"
    if precision == "fp32":
        split = "split" if use_tc and k == 3 and stride == 1 and cin % 64 == 0 and cout % 64 == 0 else "cuda"
        return split, split, wgrad_split
    fw = "bf16" if tc_conv_shape_ok(k, cin, cout) else "cuda"        # stride 2 on the space-to-depth operand, upsample on the x2 map
    if out:
        return fw, "split" if fw == "bf16" else "cuda", wgrad_split
    if fw == "cuda" or stride == 2:
        return fw, "cuda", "cuda"
    return fw, "bf16", "bf16" if cin % 128 == 0 and cout % 128 == 0 else "cuda"


class _Conv:
    """One conv of the step: where it sits, its kernel routes (``conv_routes``: ``VQGANTrainer._route_convs``), its split-fp16 weights."""

    def __init__(self, name, cw, stride, upsample, out):
        self.name, self.cw, self.stride, self.upsample, self.out = name, cw, stride, upsample, out
        self.fw = self.dgrad = self.wgrad = None
        self.split = {}                                 # split-fp16 weights per direction, until the next optimizer step


class VQGANTrainer:
    _seed_scale = 1.0                                   # the gradient-seed scale of the running step (see grad_seed_scale)

    def __init__(self, model, lr=None, betas=(0.5, 0.9), eps=1e-8, bucket_bytes=64 << 20, process_group=None, precision="fp32",
                 accumulate_grad_batches=1):
        """``precision``: "fp32" (the reference's arithmetic) or "bf16" (single-pass bf16 tensor-core convs, see the module docstring);
        either way the model is built with precision="fp32" and its fp32 weights are the master copy.

        ``accumulate_grad_batches`` = N (Lightning's option of that name, train_codebook_th.py:30,67): ``training_step`` runs forward and
        backward on its micro-batch with the loss divided by N, adding into one gradient; every N-th call exchanges that gradient once,
        clips it and runs Adam.  QuantizeEMA moves its codebook in every micro-batch, as the reference's forward does under Lightning.
        A run option: it is not saved in checkpoints, and a new value takes effect at the next window."""
        if precision not in ("fp32", "bf16"):
            raise ValueError("VQGANTrainer precision must be 'fp32' or 'bf16'")
        if int(accumulate_grad_batches) < 1:
            raise ValueError(f"accumulate_grad_batches must be >= 1, got {accumulate_grad_batches}")
        self.accumulate_grad_batches = int(accumulate_grad_batches)
        self.pending = 0                                # micro-batches in the gradient since the last optimizer step
        if model.enc_prec.name != "fp32" or model.dec_prec.name != "fp32":
            raise ValueError("VQGANTrainer runs the fp32 path (the reference asserts no mixed precision, vqgan_th.py:326): build the model "
                             "with precision='fp32'")
        if model.config.perceptual_weight != 0:
            raise NotImplementedError("LPIPS (VGG16 weights) is not available offline: set perceptual_weight=0")
        model._need_weights()
        self.model, self.cfg = model, model.config
        self.lr = float(model.learning_rate if lr is None else lr)
        self.betas, self.eps, self.step_count = betas, eps, 0
        self.group = process_group
        self.bucket_bytes = bucket_bytes
        self.use_tc = os.environ.get("VF_TRAIN_TC", "1") != "0"
        self.precision, self.bf16 = precision, precision == "bf16"
        self._collect_params()
        self._route_convs()
        self._flatten()
        self.last = {}
        # gradient-seed scale: None = 2^round(log2(numel of the reconstruction)), which brings the loss seeds (1 / numel) to about 1 so that
        # the backward operands sit inside the split-fp16 tensor-core path's faithful range; a number = that fixed power of two (1 = off)
        self.grad_seed_scale = 1.0 if self.bf16 else None
        if self.bf16:
            self._setup_bf16_weights()

    # ------------------------------------------------------------------ parameter registry
    def _collect_params(self):
        """The trainable tensors in the order of the model's layout: encoder, quantizer block, decoder; a record per conv."""
        w = self.model._w
        ps, self.convs = [], {}

        def conv(name, cw, stride=1, upsample=False, out=False):
            if not hasattr(cw, "w_kn"):
                raise RuntimeError(f"{name}: tensor-core weight layout in an fp32 model")
            self.convs[name] = _Conv(name, cw, stride, upsample, out)
            ps.append(_P(name + ".weight", cw.w_kn, lambda t, cw=cw: setattr(cw, "w_kn", t), "conv", cin=cw.cin))
            ps.append(_P(name + ".bias", cw.bias, lambda t, cw=cw: setattr(cw, "bias", t), "vec"))

        def lin(name, ln, parts=None):
            ps.append(_P(name + ".weight", ln.w, lambda t, ln=ln: setattr(ln, "w", t), "dense", parts))
            ps.append(_P(name + ".bias", ln.b, lambda t, ln=ln: setattr(ln, "b", t), "vec", parts))

        def norm(name, d, key):
            ps.append(_P(name + ".weight", d[key][0], lambda t, d=d, key=key: d.__setitem__(key, (t, d[key][1])), "vec"))
            ps.append(_P(name + ".bias", d[key][1], lambda t, d=d, key=key: d.__setitem__(key, (d[key][0], t)), "vec"))

        def stages(built):
            for st, sw in built:
                n = st.name
                if st.kind == "res":
                    norm(n + ".norm1", sw, "n1"); conv(n + ".conv1", sw["c1"]); norm(n + ".norm2", sw, "n2"); conv(n + ".conv2", sw["c2"])
                    if "sc" in sw:
                        lin(n + ".nin_shortcut", sw["sc"])
                elif st.kind == "attn":
                    norm(n + ".norm", sw, "norm")
                    lin(n + ".qk", sw["qk"], parts=(n + ".q", n + ".k"))
                    lin(n + ".v", sw["v"]); lin(n + ".proj_out", sw["proj"])
                elif st.kind == "out":
                    norm(n + ".norm_out", sw, "norm"); conv(n + ".conv_out", sw["conv"], out=True)
                else:
                    conv(n, sw, st.stride, st.upsample)

        stages(w["enc"])
        lin("quant_conv", w["quant_conv"])
        if self.model.quantizer == "commit":          # Quantize (utils_th.py:75-124): the codebook is an ordinary parameter
            q = w["q"]
            ps.append(_P("quantize.embeddings", q["emb"], lambda t, q=q: q.__setitem__("emb", t), "vec"))
        lin("post_quant_conv", w["post_quant_conv"])
        stages(w["dec"])
        self.params = ps

    def _route_convs(self):
        """Each conv's kernel routes under this trainer's precision and VF_TRAIN_TC."""
        for c in self.convs.values():
            cw = c.cw
            c.fw, c.dgrad, c.wgrad = conv_routes(self.precision, self.use_tc, cw.k, cw.cin, cw.cout, c.stride, c.upsample, c.out)

    def _flatten(self):
        """Re-home every parameter in the flat buffers of the gradient exchange, in BACKWARD order (decoder.conv_out first)."""
        order = list(reversed(self.params))
        ex = self.ex = GradExchange([(p.name, p.tensor.shape) for p in order], self.model.device, self.bucket_bytes, self.group)
        self.flat_p, self.flat_g, self.flat_m, self.flat_v, self.buckets, self.launched = ex.flat_p, ex.flat_g, ex.flat_m, ex.flat_v, ex.buckets, ex.launched
        for p in order:
            view = self.ex.p[p.name]
            view.copy_(p.tensor)
            p.setter(view)
            p.tensor = view
        self.model._refresh_decode_table()

    def _setup_bf16_weights(self):
        """bf16 operand copies of every tensor-core conv's weights: forward [Cout, 9 Cin] and (stride-1 convs) data gradient [Cin, 9 Cout],
        rewritten from the fp32 master weights in the flat buffer by one launch per step (``_refresh_bf16_weights``)."""
        dev = self.model.device
        self._wb16, entries = {}, []
        for c in [c for c in self.convs.values() if c.fw == "bf16"]:
            cw = c.cw
            fw = torch.empty((cw.cout, 9 * cw.cin), dtype=torch.bfloat16, device=dev)
            bw = torch.empty((cw.cin, 9 * cw.cout), dtype=torch.bfloat16, device=dev) if c.stride == 1 else None
            self._wb16[id(cw)] = (fw, bw)
            entries.append((cw.w_kn, fw, bw))
        self._wb16_table = L.conv_weights_bf16_table(entries, dev)
        self._refresh_bf16_weights()

    @property
    def _convs(self):
        """(weights, stride) of every conv, in registration order."""
        return [(c.cw, c.stride) for c in self.convs.values()]

    def _refresh_bf16_weights(self):
        L.conv_weights_bf16(self._wb16_table)

    # ------------------------------------------------------------------ primitive forward / backward pairs
    def _gn_apply(self, x, st, nw, swish, dtype=torch.float32):
        return L.groupnorm(x, nw[0], nw[1], swish=swish, out_dtype=dtype, stats=st)

    def _act(self, x, st, nw, swish, c):
        """GroupNorm(+swish) of x as the operand of conv ``c``: bf16 when its forward pass runs on bf16 wgmma, else fp32."""
        return self._gn_apply(x, st, nw, swish, torch.bfloat16 if c.fw == "bf16" else torch.float32)

    @staticmethod
    def _dgrad_weight(cw, flip=True):
        """The weights of the conv that computes the data gradient: [tap * Cout, Cin], taps flipped (a stride-2 conv's gather form: not)."""
        wk = cw.w_kn.reshape(cw.k, cw.k, cw.cin, cw.cout)
        return (wk.flip(0, 1) if flip else wk).permute(0, 1, 3, 2).reshape(cw.k * cw.k * cw.cout, cw.cin).contiguous()

    @classmethod
    def _split_weight(cls, c, direction):
        """Split-fp16 weights [n_out, tap * 2C] for L.tc_conv, forward ("fw") or data gradient ("bw"); cached until the next optimizer step."""
        if direction not in c.split:
            w_nk = (c.cw.w_kn if direction == "fw" else cls._dgrad_weight(c.cw)).t().contiguous()          # [n_out, 9 * C]
            c.split[direction] = L.split_f16x2(w_nk.reshape(w_nk.shape[0] * 9, -1)).reshape(w_nk.shape[0], -1)
        return c.split[direction]

    @staticmethod
    def _split_act(x):
        n, h, w, c = x.shape
        return L.split_f16x2(x.reshape(n * h * w, c)).reshape(n, h, w, 2 * c)

    @staticmethod
    def _b16(t):
        """The bf16 operand copy of an fp32 gradient: the one its producer wrote alongside (``_bf16``), else one rounding pass."""
        hit = getattr(t, "_bf16", None)
        return hit if hit is not None else L.groupnorm(t, None, None, swish=False, out_dtype=torch.bfloat16, normalize=False)

    def _conv_fw(self, c, a, residual=None):
        cw = c.cw
        if c.fw == "bf16":
            if c.stride == 2:                                   # space-to-depth operand: a stride-1 tap-table conv (as the bf16 model)
                a16 = L.groupnorm(a, None, None, swish=False, out_dtype=torch.bfloat16, normalize=False, s2d=True)
                return L.tc_conv(a16, self._wb16[id(cw)][0], cw.bias, taps=L.TAPS_S2D, coffs=L.s2d_coffs(cw.cin), cin=cw.cin)
            if c.upsample or a.dtype != torch.bfloat16:
                a = L.groupnorm(a, None, None, swish=False, out_dtype=torch.bfloat16, normalize=False, upsample=c.upsample)
            return L.tc_conv(a, self._wb16[id(cw)][0], cw.bias, residual=residual)
        if c.fw == "split":                                     # upsample: the split operand of the materialised x2 map
            a_split = (L.groupnorm(a, None, None, swish=False, out_dtype=torch.float16, normalize=False, upsample=True) if c.upsample
                       else self._split_act(a))
            return L.tc_conv(a_split, self._split_weight(c, "fw"), cw.bias, residual=residual)
        return self.model._conv(cw, a, residual=residual, stride=c.stride, upsample=c.upsample, stats=False)

    def _conv_bw(self, dy, c, x, norm=None, need_dx=True):
        """x: the conv's fp32 input before ``norm`` = (mean_rstd, (gamma, beta), swish) and the x2 upsample; dy: its output's gradient.
        Accumulates dW, db; returns dx (or None).  The bf16 weight gradient applies the norm on the way; other routes get a norm pass first."""
        G, cw = self.ex.g, c.cw
        gw = G[c.name + ".weight"]
        if c.wgrad == "bf16":
            L.conv_wgrad_bf16(x, dy, gw, norm=None if norm is None else (norm[0], norm[1][0], norm[1][1], norm[2]), upsample=c.upsample)
        else:
            a = x if norm is None else self._gn_apply(x, *norm)
            if c.wgrad == "split":                              # exact split-fp16 GEMMs over the pixel axis (K = pixels)
                if c.upsample:
                    a = L.groupnorm(a, None, None, swish=False, out_dtype=torch.float32, normalize=False, upsample=True)
                L.conv_wgrad_tc(a, dy, gw)
            else:
                L.conv_wgrad(a, dy, gw, kh=cw.k, stride=c.stride, pad=(1, 1) if cw.k == 3 and c.stride == 1 else (0, 0), upsample=c.upsample)
        L.col_sums(dy.reshape(-1, cw.cout), G[c.name + ".bias"])
        self.ex.ready(c.name + ".bias", c.name + ".weight")
        if not need_dx:
            return None
        if c.dgrad == "bf16":
            dx = L.tc_conv(self._b16(dy), self._wb16[id(cw)][1], None)
        elif c.dgrad == "split":                                # a data gradient is a conv with flipped taps and swapped channel roles
            wd = self._split_weight(c, "bw")
            dx = L.tc_conv(self._split_act(dy), wd, None)
        elif c.stride == 2:                                     # Downsample: gather form, taps not flipped
            return L.simt_conv_dgrad_s2(dy, self._dgrad_weight(cw, flip=False), (x.shape[1], x.shape[2]))
        else:
            dx = L.simt_conv(dy, self._dgrad_weight(cw), None, kh=cw.k, stride=1, pad=(1, 1) if cw.k == 3 else (0, 0))
        return L.sumpool2x2(dx) if c.upsample else dx

    def _lin_bw(self, name, ln, x_rows, dy_rows, residual=None):
        """y = x W^T + b.  Accumulates dW [out,in], db; returns dx = dy W (+ residual)."""
        G = self.ex.g
        m = x_rows.shape[0]
        L.conv_wgrad(x_rows.reshape(1, m, 1, ln.k), dy_rows.reshape(1, m, 1, ln.n), G[name + ".weight"], kh=1, pad=(0, 0), so=(1, ln.k))
        L.col_sums(dy_rows, G[name + ".bias"])
        self.ex.ready(name + ".bias", name + ".weight")
        dx = torch.empty((m, ln.k), dtype=torch.float32, device=x_rows.device)
        L.simt_gemm(dy_rows, ln.w, dx, M=m, N=ln.k, K=ln.n, a_strides=(ln.n, 1), b_strides=(ln.k, 1), ldc=ln.k, residual=residual)
        return dx

    # ------------------------------------------------------------------ blocks
    def _res_fw(self, stage, r, x, tape):
        ex = self.model.exact
        c1, c2 = self.convs[stage.name + ".conv1"], self.convs[stage.name + ".conv2"]
        st1 = L.gn_mean_rstd(x)
        h = self._conv_fw(c1, self._act(x, st1, r["n1"], True, c1))
        st2 = L.gn_mean_rstd(h)
        a2 = self._act(h, st2, r["n2"], True, c2)
        n, hh, ww, c = x.shape
        res = linear(ex, x.reshape(-1, c), r["sc"], torch.float32).reshape(n, hh, ww, -1) if "sc" in r else x
        y = self._conv_fw(c2, a2, residual=res)
        tape.append((self._res_bw, stage, r, x, st1, h, st2))
        return y

    def _res_bw(self, dy, stage, r, x, st1, h, st2):
        name, G = stage.name, self.ex.g
        da2 = self._conv_bw(dy, self.convs[name + ".conv2"], h, norm=(st2, r["n2"], True))
        dh = L.groupnorm_bwd(h, da2, st2, r["n2"][0], r["n2"][1], G[name + ".norm2.weight"], G[name + ".norm2.bias"], swish=True,
                             out_bf16=self.bf16)
        self.ex.ready(name + ".norm2.bias", name + ".norm2.weight")
        da1 = self._conv_bw(dh, self.convs[name + ".conv1"], x, norm=(st1, r["n1"], True))
        n, hh, ww, c = x.shape
        if "sc" in r:
            dres = self._lin_bw(name + ".nin_shortcut", r["sc"], x.reshape(-1, c), dy.reshape(-1, dy.shape[-1])).reshape(x.shape)
        else:
            dres = dy
        dx = L.groupnorm_bwd(x, da1, st1, r["n1"][0], r["n1"][1], G[name + ".norm1.weight"], G[name + ".norm1.bias"], swish=True, add=dres,
                             out_bf16=self.bf16)
        self.ex.ready(name + ".norm1.bias", name + ".norm1.weight")
        return dx

    def _attn_fw(self, stage, aw, x, tape):
        ex = self.model.exact
        n, hh, ww, c = x.shape
        hw = hh * ww
        st = L.gn_mean_rstd(x)
        a = self._gn_apply(x, st, aw["norm"], False).reshape(n * hw, c)
        qk = linear(ex, a, aw["qk"], torch.float32)                                   # [rows, 2c] = q | k
        v = linear(ex, a, aw["v"], torch.float32)                                     # [rows, c]
        scale = float(int(c) ** (-0.5))
        S = torch.empty((n, hw, hw), dtype=torch.float32, device=x.device)
        L.simt_gemm(qk, qk, S, M=hw, N=hw, K=c, a_strides=(2 * c, 1), b_strides=(1, 2 * c), ldc=hw, batch=(n, 1), a_bs=(hw * 2 * c, 0),
                    b_bs=(hw * 2 * c, 0), c_bs=(hw * hw, 0), b_off=c, alpha=scale)
        Pm = torch.empty_like(S)
        L.softmax_rows(S, Pm, rows_total=n * hw, rows_per_batch=hw, cols=hw, ld_in=hw, ld_out=hw)
        o = torch.empty((n * hw, c), dtype=torch.float32, device=x.device)
        L.simt_gemm(Pm, v, o, M=hw, N=c, K=hw, a_strides=(hw, 1), b_strides=(c, 1), ldc=c, batch=(n, 1), a_bs=(hw * hw, 0), b_bs=(hw * c, 0),
                    c_bs=(hw * c, 0))
        y = linear(ex, o, aw["proj"], torch.float32, residual=x.reshape(n * hw, c)).reshape(x.shape)
        tape.append((self._attn_bw, stage, aw, x, st, qk, v, Pm, o))
        return y

    def _attn_bw(self, dy, stage, aw, x, st, qk, v, Pm, o):
        name, G = stage.name, self.ex.g
        n, hh, ww, c = x.shape
        hw = hh * ww
        scale = float(int(c) ** (-0.5))
        dyr = dy.reshape(n * hw, c)
        do = self._lin_bw(name + ".proj_out", aw["proj"], o, dyr)
        dP = torch.empty_like(Pm)                                                      # dP = do v^T
        L.simt_gemm(do, v, dP, M=hw, N=hw, K=c, a_strides=(c, 1), b_strides=(1, c), ldc=hw, batch=(n, 1), a_bs=(hw * c, 0), b_bs=(hw * c, 0),
                    c_bs=(hw * hw, 0))
        dv = torch.empty_like(v)                                                       # dv = P^T do
        L.simt_gemm(Pm, do, dv, M=hw, N=c, K=hw, a_strides=(1, hw), b_strides=(c, 1), ldc=c, batch=(n, 1), a_bs=(hw * hw, 0), b_bs=(hw * c, 0),
                    c_bs=(hw * c, 0))
        dS = L.softmax_bwd_rows(Pm, dP)
        dqk = torch.empty_like(qk)
        L.simt_gemm(dS, qk, dqk, M=hw, N=c, K=hw, a_strides=(hw, 1), b_strides=(2 * c, 1), ldc=2 * c, batch=(n, 1), a_bs=(hw * hw, 0),
                    b_bs=(hw * 2 * c, 0), c_bs=(hw * 2 * c, 0), b_off=c, alpha=scale)                       # dq = scale dS k
        L.simt_gemm(dS, qk, dqk, M=hw, N=c, K=hw, a_strides=(1, hw), b_strides=(2 * c, 1), ldc=2 * c, batch=(n, 1), a_bs=(hw * hw, 0),
                    b_bs=(hw * 2 * c, 0), c_bs=(hw * 2 * c, 0), c_off=c, alpha=scale)                       # dk = scale dS^T q
        a = self._gn_apply(x, st, aw["norm"], False).reshape(n * hw, c)
        da = self._lin_bw(name + ".v", aw["v"], a, dv)
        da = self._lin_bw(name + ".qk", aw["qk"], a, dqk, residual=da)
        dx = L.groupnorm_bwd(x, da.reshape(x.shape), st, aw["norm"][0], aw["norm"][1], G[name + ".norm.weight"], G[name + ".norm.bias"],
                             swish=False, add=dy, out_bf16=self.bf16)
        self.ex.ready(name + ".norm.bias", name + ".norm.weight")
        return dx

    # ------------------------------------------------------------------ the step
    def forward_backward(self, x_nchw):
        """x f32 NCHW in [-1,1] -> loss (python float).  Leaves the gradient (summed over ranks once the exchange is waited for) in flat_g.
        One micro-batch of the accumulation window: the first one (no micro-batch pending, or the previous window complete) opens a new
        window, the others add their gradient (of the loss divided by the window's length) to the pending one."""
        model, cfg, w = self.model, self.cfg, self.model._w
        was_training = model.training
        model.training = True                                      # QuantizeEMA.forward: EMA statistics + codebook overwrite (utils_th.py:46-64)
        x = L.nchw_to_nhwc(model._in(x_nchw))
        tape = []                                                  # (backward function, its saved arguments) per stage
        hz = self._walk_fw(w["enc"], x, tape)
        n, zh, zw, zc = hz.shape
        # ---------------- quantizer (utils_th.py:32-68): z rows, nearest code, straight-through
        z = linear(model.exact, hz.reshape(-1, zc), w["quant_conv"], torch.float32)
        quant, diff, idx = model._quantize(z, want_quant=True)      # training: EMA update + packed all-reduce inside
        pq = linear(model.exact, quant, w["post_quant_conv"], torch.float32).reshape(n, zh, zw, -1)
        tape.append((self._quant_bw, hz, z, quant, idx))
        dec = self._walk_fw(w["dec"], pq, tape)
        # ---------------- loss (vqgan_th.py:400-411): mean |x - xrec| + codebook_weight * diff
        # the backward pass is linear in its seed, so it runs on seeds times a power of two s (exact in fp32: no CUDA-core result changes)
        # that keeps the split-fp16 operands of the tensor-core convs away from fp16's subnormal range; each gradient bucket is divided
        # by s when it completes, so flat_g, the all-reduce, clipping and Adam see the unscaled gradient.  Under accumulation s is the
        # window's first micro-batch's, and the seeds are divided by the window's length N (Lightning divides the loss by N)
        if self.pending in (0, self.ex.micro_batches):
            s = float(2.0 ** round(math.log2(dec.numel())) if self.grad_seed_scale is None else self.grad_seed_scale)
            self.ex.reset(s, self.accumulate_grad_batches)
            self.pending = 0
        else:
            self.ex.next_micro_batch()
        self._seed_scale = self.ex.seed_scale
        s = self._seed_scale / self.ex.micro_batches
        ddec, l1 = L.l1_grad(x, dec, s / dec.numel())
        rec = l1 / dec.numel()
        loss = rec.to(torch.float32).reshape(()) + float(cfg.codebook_weight) * diff
        self.last = dict(rec_loss=rec, quant_loss=diff, codes=idx.reshape(n, zh, zw), reconstruction=dec)
        # ---------------- backward
        dy = ddec
        for bw, *saved in reversed(tape):
            dy = bw(dy, *saved)
        model.training = was_training
        self.ex.check_complete()
        self.pending += 1
        return loss

    def _walk_fw(self, stages, h, tape):
        """Forward pass of one half's built stages (as VQGAN._walk, fp32 activations); each stage leaves its backward on the tape."""
        for st, sw in stages:
            if st.kind == "res":
                h = self._res_fw(st, sw, h, tape)
            elif st.kind == "attn":
                h = self._attn_fw(st, sw, h, tape)
            elif st.kind == "out":
                ms = L.gn_mean_rstd(h)
                a = self._gn_apply(h, ms, sw["norm"], True)
                tape.append((self._out_bw, st, sw, h, ms))
                h = self._conv_fw(self.convs[st.name + ".conv_out"], a)
            else:                                                  # the first stage's input is the image: it needs no data gradient
                c = self.convs[st.name]
                tape.append((self._conv_bw, c, h, None, bool(tape)))
                h = self._conv_fw(c, h)
        return h

    def _out_bw(self, dy, stage, sw, x, ms):
        """norm_out + swish + conv_out (conv_out's backward pass on the fp32 step's kernels in both precisions)."""
        n, G, nw = stage.name, self.ex.g, sw["norm"]
        da = self._conv_bw(dy, self.convs[n + ".conv_out"], x, norm=(ms, nw, True))
        dx = L.groupnorm_bwd(x, da, ms, nw[0], nw[1], G[n + ".norm_out.weight"], G[n + ".norm_out.bias"], swish=True, out_bf16=self.bf16)
        self.ex.ready(n + ".norm_out.bias", n + ".norm_out.weight")
        return dx

    def _quant_bw(self, dy, hz, z, quant, idx):
        """Through post_quant_conv, the straight-through estimator and the commitment term (and, for Quantize, the codebook), quant_conv."""
        model, w, G, s = self.model, self.model._w, self.ex.g, self._seed_scale / self.ex.micro_batches
        dq = self._lin_bw("post_quant_conv", w["post_quant_conv"], quant, dy.reshape(-1, dy.shape[-1]))
        cz = s * 2.0 * float(self.cfg.codebook_weight) / z.numel()
        dz = L.lincomb3(1.0, dq, cz, z, -cz, quant)
        if model.quantizer == "commit":
            # d/dE of beta mean((q - sg(z))^2): column k gets 2 beta / numel * (count_k e_k - sum of the z rows mapped to k);
            # the straight-through output carries no gradient to E (utils_th.py:117)
            emb = self.ex.p["quantize.embeddings"]
            counts, zsum = L.vq_ema_stats(z, idx, emb.shape[1])
            L.vq_commit_grad(emb, counts, zsum, s * 2.0 * model.beta * float(self.cfg.codebook_weight) / z.numel(), G["quantize.embeddings"],
                             accumulate=True)
            self.ex.ready("quantize.embeddings")
        return self._lin_bw("quant_conv", w["quant_conv"], hz.reshape(-1, hz.shape[-1]), dz).reshape(hz.shape)

    def optimizer_step(self):
        """Clip and Adam on the window's gradient.  Called on a partial window (Lightning's step at the end of an epoch), it steps on the
        micro-batches accumulated so far."""
        self.ex.flush()
        self.ex.wait()
        self.pending = 0
        self.step_count += 1
        gs = 1.0 / self.ex.world()
        clip = float(self.cfg.gradient_clip_val or 0.0)
        if clip > 0:
            # the reference trains under pytorch-lightning (train_codebook_th.py:69), which clips the global L2 norm of all gradients (after
            # the data-parallel mean) before the optimizer: g *= min(1, clip / (norm + 1e-6)).  flat_g's alignment padding is zero, so one
            # sum of squares over the whole buffer is that norm; the factor rides on Adam's gradient scale.
            norm = math.sqrt(float(L.sumsq(self.flat_g))) * gs
            gs *= min(1.0, clip / (norm + 1e-6))
        L.adam(self.flat_p, self.flat_g, self.flat_m, self.flat_v, lr=self.lr, beta1=self.betas[0], beta2=self.betas[1], eps=self.eps,
               step=self.step_count, grad_scale=gs)
        self._weights_changed()

    def _weights_changed(self):
        """flat_p has new values: everything derived from it is rebuilt."""
        for c in self.convs.values():                   # split-fp16 operand copies of the conv weights are stale now
            c.split.clear()
        if self.bf16:
            self._refresh_bf16_weights()
        if self.model.quantizer == "commit":
            self.model._refresh_codebook()
        else:
            self.model._refresh_decode_table()

    def training_step(self, batch, batch_idx=0):
        """vqgan_th.py:413-423 + the optimizer step Lightning runs after every ``accumulate_grad_batches``-th call.  Returns the loss of
        this micro-batch (0-d f32 tensor, not divided by the window's length)."""
        loss = self.forward_backward(batch)
        if self.pending == self.ex.micro_batches:
            self.optimizer_step()
        return loss

    # ------------------------------------------------------------------ export (reference layouts)
    def _export(self, get):
        out = {}
        for p in self.params:
            t = get(p)
            if p.kind == "conv":
                cout = t.shape[1]
                k = int(round(math.sqrt(t.shape[0] // p.cin)))
                out[p.name] = t.reshape(k, k, -1, cout).permute(3, 2, 0, 1).contiguous().cpu()
            elif p.kind == "dense":
                t4 = t.reshape(t.shape[0], t.shape[1], 1, 1).cpu()
                if p.part:
                    half = t.shape[0] // 2
                    out[p.part[0] + ".weight"], out[p.part[1] + ".weight"] = t4[:half].clone(), t4[half:].clone()
                else:
                    out[p.name] = t4.clone()
            else:
                tc = t.cpu().clone()
                if p.part:
                    half = tc.shape[0] // 2
                    out[p.part[0] + ".bias"], out[p.part[1] + ".bias"] = tc[:half].clone(), tc[half:].clone()
                else:
                    out[p.name] = tc
        return out

    def _import(self, tensors, what, strict):
        """Inverse of ``_export``: reference-keyed, reference-layout tensors -> {parameter name: kernel-layout fp32 host tensor}.  Raises on
        a wrong shape and (strict) on a missing key; nothing on the device is touched."""
        shapes = self.model.param_shapes()

        def take(key):
            if key not in tensors:
                if strict:
                    raise RuntimeError(f"{what}: missing key {key}")
                return None
            t = torch.as_tensor(tensors[key]).detach().to("cpu", torch.float32)
            if tuple(t.shape) != tuple(shapes[key]):
                raise RuntimeError(f"{what}: {key} has shape {tuple(t.shape)}, expected {tuple(shapes[key])}")
            return t

        out = {}
        for p in self.params:
            suffix = ".weight" if p.kind == "dense" else ".bias"
            parts = [take(n + suffix) for n in p.part] if p.part else [take(p.name)]
            if any(t is None for t in parts):
                continue
            t = torch.cat(parts, 0)
            if p.kind == "conv":
                t = t.permute(2, 3, 1, 0).reshape(-1, t.shape[0])
            elif p.kind == "dense":
                t = t.reshape(t.shape[0], t.shape[1])
            out[p.name] = t.contiguous()
        return out

    # ------------------------------------------------------------------ resume: everything a step reads besides the batch
    def optimizer_state(self):
        """Host copies of what ``export_state_dict()`` leaves out: Adam's moments under the reference's keys and layouts (the names of
        ``torch.optim.Adam``'s state) and the scalars.  Every rank of a data-parallel run holds the same state."""
        return dict(exp_avg=self._export(lambda p: self.ex.m[p.name]), exp_avg_sq=self._export(lambda p: self.ex.v[p.name]),
                    step_count=self.step_count, lr=self.lr, betas=tuple(self.betas), eps=self.eps, precision=self.precision)

    def load_optimizer_state(self, state, strict=True):
        """Inverse of ``optimizer_state()``; state saved by a trainer of the other precision loads too (the master copy is fp32)."""
        m, v = self._import(state["exp_avg"], "exp_avg", strict), self._import(state["exp_avg_sq"], "exp_avg_sq", strict)
        absent = [k for k in ("step_count", "lr", "betas", "eps") if k not in state]
        if strict and absent:
            raise RuntimeError(f"VQGANTrainer.load_optimizer_state: missing {absent}")
        for views, src in ((self.ex.m, m), (self.ex.v, v)):
            for k, t in src.items():
                views[k].copy_(t)
        self.step_count = int(state.get("step_count", self.step_count))
        self.lr, self.eps = float(state.get("lr", self.lr)), float(state.get("eps", self.eps))
        self.betas = tuple(state.get("betas", self.betas))
        return self

    def load_state_dict(self, state_dict, strict=True):
        """Reference-keyed weights (the keys of ``export_state_dict()``, EMA buffers included) into the fp32 master copy and the model's
        quantizer, then what an applied step does to the derived copies."""
        from .vqgan import _IGNORE
        model, shapes = self.model, self.model.param_shapes()
        sd = {k: v for k, v in state_dict.items() if not _IGNORE.match(k)}
        unknown = [k for k in sd if k not in shapes]
        if strict and unknown:
            raise RuntimeError(f"VQGANTrainer.load_state_dict: unexpected keys {unknown[:8]}")
        new = self._import(sd, "VQGANTrainer.load_state_dict", strict)
        buffers = {}
        if model.quantizer == "ema":
            for key, slot in (("quantize.embeddings", "emb"), ("quantize.ema_cluster_size_hidden", "cs"), ("quantize.ema_dw_hidden", "dw")):
                if key in sd:
                    t = torch.as_tensor(sd[key]).detach().to("cpu", torch.float32)
                    if tuple(t.shape) != tuple(shapes[key]):
                        raise RuntimeError(f"VQGANTrainer.load_state_dict: {key} has shape {tuple(t.shape)}, expected {tuple(shapes[key])}")
                    buffers[slot] = t
                elif strict:
                    raise RuntimeError(f"VQGANTrainer.load_state_dict: missing key {key}")
            if strict and "quantize.counter" not in sd:
                raise RuntimeError("VQGANTrainer.load_state_dict: missing key quantize.counter")
        for k, t in new.items():
            self.ex.p[k].copy_(t)
        q = model._w["q"]
        for slot, t in buffers.items():
            q[slot].copy_(t)
        if model.quantizer == "ema":
            q["counter"] = int(sd.get("quantize.counter", q["counter"]))
            model._refresh_codebook()                   # the EMA codebook is no parameter: re-derive its copies as load time does
        self._weights_changed()
        model._sd.update({k: torch.as_tensor(v).detach().to("cpu").clone() for k, v in sd.items() if k in shapes})
        return self

    def save_checkpoint(self, path, epoch=0):
        """A torch pickle in the pytorch-lightning layout the reference's loaders read (utils/torch.py:9-17 takes ``state_dict``; Lightning's
        ``resume_from_checkpoint`` also ``optimizer_states``, ``global_step`` and ``epoch``), with ``config.json`` next to it as the
        reference's checkpoint callback writes it (train/logging_utils_th.py:316-341).  What Lightning has no slot for sits under
        ``viewformer_b200``.  Under data parallelism call it on rank 0.  Not in the middle of an accumulation window: the checkpoint has
        no slot for a pending gradient."""
        if 0 < self.pending < self.ex.micro_batches:
            raise RuntimeError(f"save_checkpoint: {self.pending} of {self.ex.micro_batches} micro-batches of the accumulation window are "
                               "pending; save after the optimizer step that closes the window (or call optimizer_step() first)")
        st = self.optimizer_state()
        ckpt = dict(state_dict=dict(self.export_state_dict()), global_step=self.step_count, epoch=int(epoch),
                    optimizer_states=[adam_state_dict(trainable_names(self.model), st["exp_avg"], st["exp_avg_sq"], self.step_count, self.lr,
                                                      self.betas, self.eps)],
                    lr_schedulers=[], viewformer_b200=dict(precision=self.precision, quantizer=self.model.quantizer))
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(os.path.join(os.path.dirname(os.path.abspath(path)), "config.json"), "w") as f:
            json.dump(self.cfg.asdict(), f)
        torch.save(ckpt, path)

    def load_checkpoint(self, path):
        """Inverse of ``save_checkpoint``.  A file with ``state_dict`` only (what ``registry.load_model`` needs) restores the weights and
        leaves the optimizer as it is, with a warning.  Returns the checkpoint's ``epoch``."""
        ckpt = torch.load(path, map_location="cpu")
        state = None
        if ckpt.get("optimizer_states"):
            state = read_adam_state_dict(ckpt["optimizer_states"][0], trainable_names(self.model))
            # both halves are checked against this model before either is written
            self._import(state["exp_avg"], "exp_avg", True), self._import(state["exp_avg_sq"], "exp_avg_sq", True)
        self.load_state_dict(ckpt["state_dict"])
        if state is None:
            warnings.warn(f"{path} holds no optimizer state: weights restored, Adam starts from zero moments")
        else:
            if not state["exp_avg"]:                    # saved before the first step: Adam had created no moments yet
                self.flat_m.zero_(), self.flat_v.zero_()
            self.load_optimizer_state(state, strict=bool(state["exp_avg"]))
        return int(ckpt.get("epoch", 0))

    def export_gradients(self):
        """Gradient of the last forward_backward (already summed over ranks if the handles were waited for), reference layouts."""
        return self._export(lambda p: self.ex.g[p.name])

    def export_state_dict(self):
        """Reference-keyed state_dict after training; also refreshes the model's host copy."""
        sd = self.model.state_dict()
        sd.update(self._export(lambda p: p.tensor))
        self.model._sd = {k: v.clone() for k, v in sd.items()}
        return sd
