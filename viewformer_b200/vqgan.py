"""VQGAN codebook model — H100-native drop-in for the reference's torch ``VQGAN``.

Surface (same names / argument meaning / return tuples as viewformer/models/vqgan_th.py:321-398):
    VQGAN(config).load_state_dict(sd)         reference key names, [Cout,Cin,kh,kw] conv weights, [D,K] codebook
    .encode(x)        x f32 NCHW in [-1,1]  ->  (quant NCHW f32, diff scalar, codes int64 [N,h,w])   (:379-383)
    .decode(quant)    NCHW f32              ->  NCHW f32                                               (:385-388)
    .decode_code(codes)                     ->  NCHW f32                                               (:390-393)
    .__call__(x)                            ->  (dec, diff, quant, codes)                              (:395-398)
plus NHWC ("TF twin" convention, viewformer/models/vqgan.py:291-301) entry points ``encode_nhwc`` /
``decode_code_nhwc`` and the uint8 end-to-end helpers used by ``generate``.

Everything between the input and output tensors runs in libvf_b200 kernels on NHWC activations:
fp32 residual stream, GroupNorm statistics in fp64, operands of the tensor-core convolutions in the
precision's operand dtype.  No torch compute op is on the forward path (torch only allocates buffers).
"""
import re
from collections import OrderedDict
from typing import NamedTuple

import os

import torch

from . import _lib as L
from . import float_images
from .config import VQGANConfig, load_config
from .ops import Precision, Linear, gemm_nt, linear

_IGNORE = re.compile(r"(perceptual_loss\..*)|(loss\..*)")   # vqgan_th.py:322


class Stage(NamedTuple):
    """One step of the encoder or decoder walk."""
    kind: str            # conv_in | res | attn | down | up | out (norm_out + swish + conv_out)
    name: str            # reference key prefix; for "out" the half's own ("encoder" / "decoder")
    cin: int
    cout: int
    exact: bool = False  # encoder.conv_in / decoder.conv_out: always on the exact fp32 kernels

    @property
    def stride(self):    # Downsample: pad (0,1,0,1), then a VALID stride-2 conv (vqgan_th.py:45-49)
        return 2 if self.kind == "down" else 1

    @property
    def upsample(self):  # Upsample: nearest x2, then a stride-1 conv (vqgan_th.py:29-32)
        return self.kind == "up"


def layout(cfg):
    """Encoder and decoder (vqgan_th.py:147-201, 228-289) as two ordered lists of ``Stage``: conv_in, the resolution levels (res blocks,
    each followed by an AttnBlock at the attention resolutions, then a Downsample / Upsample), mid block / attention / mid block, out.
    A pure function of the config and the only place that builds an encoder / decoder key name: the parameter order, the weights, the
    forward passes and the training step all walk it."""
    ch, nres = cfg.ch, len(cfg.ch_mult)

    def level(prefix, lv, cin, nblocks):
        stages, cout = [], ch * cfg.ch_mult[lv]
        for b in range(nblocks):
            stages.append(Stage("res", f"{prefix}.block.{b}", cin, cout))
            cin = cout
            if cfg.image_size // 2 ** lv in cfg.attn_resolutions:
                stages.append(Stage("attn", f"{prefix}.attn.{b}", cout, cout))
        return stages

    def mid(half, c):
        return [Stage("res", half + ".mid.block_1", c, c), Stage("attn", half + ".mid.attn_1", c, c), Stage("res", half + ".mid.block_2", c, c)]

    enc, c = [Stage("conv_in", "encoder.conv_in", cfg.in_channels, ch, exact=True)], ch
    for lv in range(nres):
        enc += level(f"encoder.down.{lv}", lv, c, cfg.num_res_blocks)
        c = ch * cfg.ch_mult[lv]
        if lv != nres - 1:
            enc.append(Stage("down", f"encoder.down.{lv}.downsample.conv", c, c))
    enc += mid("encoder", c) + [Stage("out", "encoder", c, cfg.z_channels)]
    c = ch * cfg.ch_mult[-1]
    dec = [Stage("conv_in", "decoder.conv_in", cfg.z_channels, c)] + mid("decoder", c)
    for lv in reversed(range(nres)):
        dec += level(f"decoder.up.{lv}", lv, c, cfg.num_res_blocks + 1)
        c = ch * cfg.ch_mult[lv]
        if lv != 0:
            dec.append(Stage("up", f"decoder.up.{lv}.upsample.conv", c, c))
    dec.append(Stage("out", "decoder", c, cfg.out_ch, exact=True))
    return enc, dec


def tc_conv_shape_ok(k, cin, cout, k_align=64):
    """The conv shapes a tensor-core model runs on the tensor cores: 3x3, Cin a multiple of the K block (``Precision.k_align``
    channels), Cout a multiple of 16 and at least 64.  The bf16 codebook training step puts the same convs on bf16 wgmma."""
    return k == 3 and cin % k_align == 0 and cout % 16 == 0 and cout >= 64


def image_tensor(images, what, dtypes=(torch.uint8, torch.float32)):
    """``images`` as a tensor of one of ``dtypes`` (uint8, or float32 in [0, 1]); anything else raises TypeError instead of being cast."""
    t = torch.as_tensor(images)
    if t.dtype not in dtypes:
        raise TypeError(f"{what}: images must be {' or '.join(str(d).replace('torch.', '') for d in dtypes)}"
                        f"{' (float32 in [0, 1])' if torch.float32 in dtypes else ''}, got {t.dtype}; they are not cast")
    return t


class _Conv3:
    """3x3 (or 1x1) convolution weights in both kernel layouts."""

    def __init__(self, w, b, prec, device, *, exact=False):
        cout, cin, kh, kw = w.shape
        self.cout, self.cin, self.k = cout, cin, kh
        w = w.to(device=device, dtype=torch.float32)
        self.bias = b.to(device=device, dtype=torch.float32).contiguous()
        self.tc = (not exact) and prec.use_tc and tc_conv_shape_ok(kh, cin, cout, prec.k_align)
        self.small_cin = kh == 3 and cin in (3, 4) and cout % 16 == 0 and cout <= 128     # conv_in: dedicated exact kernel (RGB, RGBA)
        self.small_cout = kh == 3 and cin == 128 and cout in (3, 4)                       # conv_out: dedicated exact kernel
        if self.tc and prec.split:
            # exact mode: per tap [hi(Cin) | lo(Cin)] fp16 halves of the fp32 weights
            self.w_nk = L.split_f16x2(w.permute(0, 2, 3, 1).reshape(cout * kh * kw, cin).contiguous()).reshape(cout, kh * kw * 2 * cin)
        elif self.tc:
            self.w_nk = w.permute(0, 2, 3, 1).reshape(cout, kh * kw * cin).to(prec.opd).contiguous()   # [Cout, tap*Cin+c]
        else:
            self.w_kn = w.permute(2, 3, 1, 0).reshape(kh * kw * cin, cout).contiguous()                # [tap*Cin+c, Cout]


class VQGAN:
    _ignore_checkpoint_attributes = [r"perceptual_loss\..*", r"loss\..*"]

    def __init__(self, config=None, precision="bf16", device="cuda", quantizer="ema", beta=0.25, train_precision="fp32", **config_overrides):
        """``quantizer``: "ema" = QuantizeEMA (utils_th.py:8-72, what vqgan_th.py:331 instantiates) or "commit" = Quantize
        (utils_th.py:75-124: the codebook is a gradient-trained parameter, loss = |sg(q) - z|^2 + beta |q - sg(z)|^2).
        ``train_precision``: arithmetic of configure_optimizers() / training_step() on a model built with precision="fp32" — "fp32" (the
        reference's) or "bf16" (bf16 tensor-core convs over the fp32 master weights, see viewformer_b200.train)."""
        if config is None:
            config = VQGANConfig(**config_overrides)
        if quantizer not in ("ema", "commit"):
            raise ValueError("quantizer must be 'ema' (QuantizeEMA) or 'commit' (Quantize, beta-weighted commitment loss)")
        self.quantizer, self.beta = quantizer, float(beta)
        if train_precision not in ("fp32", "bf16"):
            raise ValueError("train_precision must be 'fp32' or 'bf16'")
        self.train_precision = train_precision
        self.config = load_config(config)
        # ``mixed``: the encoder (whose output feeds the bit-exact codebook argmin) runs in the fp32-faithful ``exact`` arithmetic,
        # the decoder (pixels within a tolerance) on the bf16 tensor-core path.  One precision name otherwise serves both halves.
        enc_name, dec_name = ("x3", "bf16") if precision == "mixed" else (precision, precision)
        self.precision = precision
        self.enc_prec, self.dec_prec = Precision(enc_name), Precision(dec_name)
        self.prec = self.dec_prec                  # quantizer / glue policy
        # norm2 + swish fused into conv2's operand path (vf_tc_gemm_t.norm_*, the halo tile is transformed in shared memory):
        # bit-identical to the two-kernel path and tested; the MMA warpgroups do the transform between their MMAs, so it stays
        # opt-in (VF_NORM_ON_LOAD=1) until it is measured faster than conv + vf_groupnorm_apply
        self.norm_on_load = os.environ.get("VF_NORM_ON_LOAD", "0") == "1"      # bf16 halves only
        self.exact = Precision("fp32")
        self.device = torch.device(device)
        self.training = False
        self.learning_rate = self.config.learning_rate
        self._sd = None
        self._w = None
        self.decay, self.eps = 0.99, 1e-5          # utils_th.py:9
        self.dist_world_size = 1

    # ------------------------------------------------------------------ torch-module-like plumbing
    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise L.LibraryError("viewformer_b200.VQGAN runs on CUDA (sm_90a) only; there is no CPU path")
        if self._sd is not None and device != self.device:
            sd = self.state_dict()                 # includes the live quantizer buffers (EMA updates made in train() mode)
            self.device = device
            self.load_state_dict(sd)
        self.device = device
        return self

    def cuda(self):
        return self.to("cuda")

    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        self.training = bool(mode)
        return self

    def parameters(self):
        return [v for k, v in self.state_dict().items() if not k.startswith("quantize.")]

    def param_shapes(self):
        """Ordered {name: shape} of the reference state_dict (vqgan_th.py:147-201, 228-289, 321-336)."""
        cfg = self.config
        out = OrderedDict()

        def conv(n, cout, cin, k):
            out[n + ".weight"] = (cout, cin, k, k)
            out[n + ".bias"] = (cout,)

        def norm(n, c):
            out[n + ".weight"] = (c,)
            out[n + ".bias"] = (c,)

        enc, dec = layout(cfg)
        for st in enc + dec:
            n, cin, cout = st.name, st.cin, st.cout
            if st.kind == "res":
                norm(n + ".norm1", cin); conv(n + ".conv1", cout, cin, 3); norm(n + ".norm2", cout); conv(n + ".conv2", cout, cout, 3)
                if cin != cout:
                    conv(n + ".nin_shortcut", cout, cin, 1)
            elif st.kind == "attn":
                norm(n + ".norm", cin)
                for p in ("q", "k", "v", "proj_out"):
                    conv(n + "." + p, cin, cin, 1)
            elif st.kind == "out":
                norm(n + ".norm_out", cin); conv(n + ".conv_out", cout, cin, 3)
            else:
                conv(n, cout, cin, 3)
        out["quantize.embeddings"] = (cfg.embed_dim, cfg.n_embed)
        if self.quantizer == "ema":
            out["quantize.ema_cluster_size_hidden"] = (cfg.n_embed,)
            out["quantize.ema_dw_hidden"] = (cfg.embed_dim, cfg.n_embed)
            out["quantize.counter"] = ()
        conv("quant_conv", cfg.embed_dim, cfg.z_channels, 1); conv("post_quant_conv", cfg.z_channels, cfg.embed_dim, 1)
        return out

    def expected_keys(self):
        return list(self.param_shapes().keys())

    def init_weights(self, seed=0):
        """Random initialisation with the reference's initialisers: torch Conv2d default U(+-1/sqrt(fan_in)) for
        weights and biases, GroupNorm 1/0, codebook U(+-sqrt 3) (utils_th.py:17), EMA buffers 0."""
        return self.load_state_dict(self._initial_state(seed))

    def _initial_state(self, seed=0):
        g = torch.Generator().manual_seed(int(seed))
        sd = OrderedDict()
        shapes = self.param_shapes()
        for k, shp in shapes.items():
            if k == "quantize.embeddings":
                # QuantizeEMA: U(+-sqrt 3) (utils_th.py:17); Quantize: U(+-1/K) (utils_th.py:90-91)
                sd[k] = (torch.rand(shp, generator=g) * 2 - 1) * (3 ** 0.5 if self.quantizer == "ema" else 1.0 / shp[1])
            elif k == "quantize.counter":
                sd[k] = torch.tensor(0, dtype=torch.int64)
            elif k.startswith("quantize."):
                sd[k] = torch.zeros(shp)
            elif len(shp) == 4:
                sd[k] = (torch.rand(shp, generator=g) * 2 - 1) / (shp[1] * shp[2] * shp[3]) ** 0.5
            elif ".norm" in k or "norm_out" in k:
                sd[k] = torch.ones(shp) if k.endswith("weight") else torch.zeros(shp)
            else:
                w = shapes[k[:-4] + "weight"]
                sd[k] = (torch.rand(shp, generator=g) * 2 - 1) / (w[1] * w[2] * w[3]) ** 0.5
        return sd

    @L.on_model_device
    def load_state_dict(self, state_dict, strict=True):
        """Strict key check with the reference's ignore patterns (vqgan_th.py:346-359)."""
        sd = OrderedDict((k, v) for k, v in state_dict.items() if not _IGNORE.match(k))
        if strict:
            want, got = set(self.expected_keys()), set(sd.keys())
            if want - got:
                raise RuntimeError(f"Missing keys: {want - got}")
            if got - want:
                raise RuntimeError(f"Unexpected keys: {got - want}")
        else:                                      # non-strict: unknown keys dropped, missing keys keep their current (or initial) value
            shapes = self.param_shapes()
            sd = OrderedDict((k, v) for k, v in sd.items() if k in shapes)
            missing = [k for k in shapes if k not in sd]
            if missing:
                cur = self.state_dict() if self._sd is not None else VQGAN(self.config, precision=self.precision, device=self.device,
                                                                          quantizer=self.quantizer, beta=self.beta)._initial_state(0)
                for k in missing:
                    sd[k] = cur[k]
        self._sd = OrderedDict((k, torch.as_tensor(v).detach().to("cpu").clone()) for k, v in sd.items())
        self._build()
        return self

    @L.on_model_device
    def state_dict(self):
        sd = OrderedDict((k, v.clone()) for k, v in self._sd.items())
        if self._w is not None:     # training mutates the quantizer buffers on the device
            q = self._w["q"]
            sd["quantize.embeddings"] = q["emb"].detach().cpu().clone()
            if self.quantizer == "ema":
                sd["quantize.ema_cluster_size_hidden"] = q["cs"].detach().cpu().clone()
                sd["quantize.ema_dw_hidden"] = q["dw"].detach().cpu().clone()
                sd["quantize.counter"] = torch.tensor(q["counter"], dtype=torch.int64)
        return sd

    # ------------------------------------------------------------------ weight preparation (load time only)
    def _build(self):
        L.load(require_device=True)
        sd, dev = self._sd, self.device

        def gn(n):
            return (sd[n + ".weight"].to(dev, torch.float32).contiguous(), sd[n + ".bias"].to(dev, torch.float32).contiguous())

        def conv(n, prec, exact=False):
            return _Conv3(sd[n + ".weight"], sd[n + ".bias"], prec, dev, exact=exact)

        def lin(n, prec):
            wt = sd[n + ".weight"]
            return Linear(wt.reshape(wt.shape[0], wt.shape[1]), sd[n + ".bias"], prec, dev)

        def stage(st, prec):
            """The stage's weights: a _Conv3 (conv_in / down / up), or a dict of _Conv3, Linear and GroupNorm (weight, bias) tuples."""
            n, c = st.name, st.cin
            if st.kind == "res":
                d = dict(n1=gn(n + ".norm1"), c1=conv(n + ".conv1", prec), n2=gn(n + ".norm2"), c2=conv(n + ".conv2", prec), prec=prec)
                if st.cin != st.cout:
                    d["sc"] = lin(n + ".nin_shortcut", prec)
                return d
            if st.kind == "attn":
                wq, wk, wv = (sd[f"{n}.{p}.weight"] for p in ("q", "k", "v"))
                qk = Linear(torch.cat([wq.reshape(c, c), wk.reshape(c, c)], 0), torch.cat([sd[n + ".q.bias"], sd[n + ".k.bias"]]), prec, dev)
                return dict(norm=gn(n + ".norm"), qk=qk, v=Linear(wv.reshape(c, c), sd[n + ".v.bias"], prec, dev),
                            proj=lin(n + ".proj_out", prec), prec=prec)
            if st.kind == "out":
                return dict(norm=gn(n + ".norm_out"), conv=conv(n + ".conv_out", prec, st.exact))
            return conv(n, prec, st.exact)

        enc, dec = layout(self.config)
        w = dict(enc=[(st, stage(st, self.enc_prec)) for st in enc], dec=[(st, stage(st, self.dec_prec)) for st in dec])
        # 1x1 quant convs always run in exact fp32: their output feeds the bit-exact argmin
        w["quant_conv"] = lin("quant_conv", self.exact)
        w["post_quant_conv"] = lin("post_quant_conv", self.exact)
        emb = sd["quantize.embeddings"].to(dev, torch.float32).contiguous()             # [D,K] (utils_th.py:17-18)
        w["q"] = dict(emb=emb)
        if self.quantizer == "ema":
            w["q"].update(cs=sd["quantize.ema_cluster_size_hidden"].to(dev, torch.float32).contiguous(),
                          dw=sd["quantize.ema_dw_hidden"].to(dev, torch.float32).contiguous(),
                          counter=int(sd["quantize.counter"]))
        self._w = w
        self._refresh_codebook()

    def _refresh_codebook(self):
        """Everything derived from the [D,K] codebook: transposed copy, |e|^2, tensor-core operand copies, the decode table.
        Called at load time and after a gradient step on the codebook (``quantizer="commit"``)."""
        q = self._w["q"]
        q["et"], q["esq"] = L.vq_prepare_codebook(q["emb"])
        q["eh"] = L.vq_prepare_codebook_f16(q["et"]) if (self.prec.use_tc and L.vq_fused_ok(*q["emb"].shape)) else None
        self._refresh_decode_table()

    def _refresh_decode_table(self):
        """decode_code only ever sees K distinct inputs to post_quant_conv: table[k] = post_quant_conv(E[:,k])."""
        q = self._w["q"]
        self._w["pq_table"] = linear(self.exact, q["et"], self._w["post_quant_conv"], torch.float32)

    # ------------------------------------------------------------------ building blocks (NHWC f32 in / out)
    def _conv(self, cw, x_opd_or_f32, *, residual=None, stride=1, upsample=False, stats=True, out_dtype=torch.float32):
        """``stats``: the output feeds a GroupNorm(32) — let the tensor-core epilogue accumulate its statistics.
        ``out_dtype`` bf16 is only honoured on the tensor-core path (callers check ``cw.tc``)."""
        gn = 32 if stats else 0
        if cw.tc and stride == 2:    # operand is the space-to-depth tensor [N,H/2,W/2,4C]: stride-1 tap-table conv
            return L.tc_conv(x_opd_or_f32, cw.w_nk, cw.bias, taps=L.TAPS_S2D, coffs=L.s2d_coffs(cw.cin), cin=cw.cin, gn_groups=gn)
        if cw.tc:
            return L.tc_conv(x_opd_or_f32, cw.w_nk, cw.bias, residual=residual, gn_groups=gn, out_dtype=out_dtype)
        assert out_dtype == torch.float32
        if stride == 1 and not upsample and residual is None and x_opd_or_f32.dtype == torch.float32:
            if cw.small_cin:
                return L.conv3x3_small_cin(x_opd_or_f32, cw.w_kn, cw.bias, gn_groups=gn)
            if cw.small_cout:
                return L.conv3x3_small_cout(x_opd_or_f32, cw.w_kn, cw.bias)
        pad = (1, 1) if stride == 1 else (0, 0)     # Downsample: pad (0,1,0,1) then VALID stride-2 (vqgan_th.py:45-49)
        return L.simt_conv(x_opd_or_f32, cw.w_kn, cw.bias, kh=cw.k, stride=stride, pad=pad if cw.k == 3 else (0, 0),
                           upsample=upsample, residual=residual)

    def _act_dtype(self, cw, prec):
        return prec.opd if cw.tc else torch.float32

    def _resblock(self, rbw, x):
        prec = rbw["prec"]
        bf16 = prec.name == "bf16"
        a = L.groupnorm(x, *rbw["n1"], swish=True, out_dtype=self._act_dtype(rbw["c1"], prec))
        # conv1's output is consumed by norm2 alone (the block's residual is x): in bf16 mode it travels as bf16 with the
        # GroupNorm statistics taken from the fp32 accumulators in the conv epilogue — 4 B/element less HBM traffic
        n_, h_, w_, _ = x.shape
        c1 = rbw["c1"]
        edge = torch.bfloat16 if (bf16 and c1.tc and rbw["c2"].tc
                                  and L.gn_fusable(c1.cout, 32, n_ * h_ * w_, h_ * w_, c1.cout)) else torch.float32
        h = self._conv(c1, a, out_dtype=edge)
        if h.dtype == torch.bfloat16 and self.norm_on_load and L.conv_norm_fusable(h, rbw["c2"].cout):
            # norm2 + swish applied to conv2's operand inside the kernel (while the halo tile sits in shared memory):
            # the raw bf16 edge is read once by the conv instead of being read, normalised, written and read again
            a, norm2 = h, (L.gn_mean_rstd(h), rbw["n2"][0], rbw["n2"][1], 32, True)
        else:
            a, norm2 = L.groupnorm(h, *rbw["n2"], swish=True, out_dtype=self._act_dtype(rbw["c2"], prec)), None
        if "sc" in rbw:
            n, hh, ww, c = x.shape
            xs = x if prec.opd == torch.float32 else L.groupnorm(x, None, None, swish=False, out_dtype=prec.opd, normalize=False)
            res = linear(prec, xs.reshape(n * hh * ww, -1), rbw["sc"], torch.float32).reshape(n, hh, ww, -1)
        else:
            res = x
        if norm2 is not None:
            return L.tc_conv(a, rbw["c2"].w_nk, rbw["c2"].bias, residual=res, gn_groups=32, norm=norm2)
        return self._conv(rbw["c2"], a, residual=res)

    def _attn(self, aw, x):
        """AttnBlock (vqgan_th.py:120-144): single head over HW tokens, logits scaled by C^-0.5."""
        prec = aw["prec"]
        if prec.split:
            return self._attn_exact(aw, x)
        n, hh, ww, c = x.shape
        hw = hh * ww
        a = L.groupnorm(x, *aw["norm"], swish=False, out_dtype=prec.opd).reshape(n * hw, c)
        qk = linear(prec, a, aw["qk"], prec.opd)                                      # [n*hw, 2c] = q | k
        vt = torch.empty((n, c, hw), dtype=prec.opd, device=x.device)                 # V^T per image (K-major for P.V)
        gemm_nt(prec, aw["v"].w, a, vt, M=c, N=hw, K=c, lda=c, ldb=c, ldc=hw, batch=(n, 1), a_bs=(0, 0),
                b_bs=(hw * c, 0), c_bs=(c * hw, 0), bias=aw["v"].b, bias_mode=L.BIAS_M)
        scores = torch.empty((n, hw, hw), dtype=torch.float32, device=x.device)
        gemm_nt(prec, qk, qk, scores, M=hw, N=hw, K=c, lda=2 * c, ldb=2 * c, ldc=hw, batch=(n, 1),
                a_bs=(hw * 2 * c, 0), b_bs=(hw * 2 * c, 0), c_bs=(hw * hw, 0), b_off=c, alpha=float(int(c) ** (-0.5)))
        p = torch.empty((n, hw, hw), dtype=prec.opd, device=x.device)
        L.softmax_rows(scores, p, rows_total=n * hw, rows_per_batch=hw, cols=hw, ld_in=hw, ld_out=hw)
        o = torch.empty((n * hw, c), dtype=prec.opd, device=x.device)
        gemm_nt(prec, p, vt, o, M=hw, N=c, K=hw, lda=hw, ldb=hw, ldc=c, batch=(n, 1), a_bs=(hw * hw, 0),
                b_bs=(c * hw, 0), c_bs=(hw * c, 0))
        out = linear(prec, o, aw["proj"], torch.float32, residual=x.reshape(n * hw, c), gn_rows_per_img=hw)
        out4 = out.reshape(n, hh, ww, c)
        if hasattr(out, "_gn_sums"):
            out4._gn_sums = out._gn_sums           # fused GroupNorm statistics travel with the tensor
        return out4

    def _attn_exact(self, aw, x):
        """AttnBlock on the exact tensor-core path: every GEMM takes split-fp16 operands ([hi | lo] rows, vf_tc_gemm VF_F16X2) and
        returns fp32; activations that feed another GEMM are re-split by one small elementwise pass."""
        prec = aw["prec"]
        n, hh, ww, c = x.shape
        hw = hh * ww
        f32 = torch.float32
        a = L.groupnorm(x, *aw["norm"], swish=False, out_dtype=torch.float16).reshape(n * hw, 2 * c)
        qk = linear(prec, a, aw["qk"], f32)                                            # [n*hw, 2c] = q | k
        qks = L.split_f16x2(qk)                                                        # [n*hw, 4c] = hi(q|k) | lo(q|k)
        vt = torch.empty((n, c, hw), dtype=f32, device=x.device)                       # V^T per image
        gemm_nt(prec, aw["v"].w, a, vt, M=c, N=hw, K=c, lda=2 * c, ldb=2 * c, ldc=hw, batch=(n, 1), a_bs=(0, 0),
                b_bs=(hw * 2 * c, 0), c_bs=(c * hw, 0), bias=aw["v"].b, bias_mode=L.BIAS_M)
        scores = torch.empty((n, hw, hw), dtype=f32, device=x.device)
        gemm_nt(prec, qks, qks, scores, M=hw, N=hw, K=c, lda=4 * c, ldb=4 * c, ldc=hw, batch=(n, 1), a_bs=(hw * 4 * c, 0),
                b_bs=(hw * 4 * c, 0), c_bs=(hw * hw, 0), b_off=c, alpha=float(int(c) ** (-0.5)), lo_a=2 * c, lo_b=2 * c)
        p = torch.empty((n, hw, hw), dtype=f32, device=x.device)
        L.softmax_rows(scores, p, rows_total=n * hw, rows_per_batch=hw, cols=hw, ld_in=hw, ld_out=hw)
        ps = L.split_f16x2(p.reshape(n * hw, hw))                                      # [n*hw, 2hw]
        vts = L.split_f16x2(vt.reshape(n * c, hw))                                     # [n*c, 2hw]
        o = torch.empty((n * hw, c), dtype=f32, device=x.device)
        gemm_nt(prec, ps, vts, o, M=hw, N=c, K=hw, lda=2 * hw, ldb=2 * hw, ldc=c, batch=(n, 1), a_bs=(hw * 2 * hw, 0),
                b_bs=(c * 2 * hw, 0), c_bs=(hw * c, 0))
        out = linear(prec, L.split_f16x2(o), aw["proj"], f32, residual=x.reshape(n * hw, c), gn_rows_per_img=hw)
        out4 = out.reshape(n, hh, ww, c)
        if hasattr(out, "_gn_sums"):
            out4._gn_sums = out._gn_sums
        return out4

    # ------------------------------------------------------------------ encoder / decoder (NHWC)
    def _walk(self, stages, h, prec):
        """The built stages of one half, in order, on NHWC f32 activations; ``prec``: that half's precision."""
        for st, sw in stages:
            if st.kind == "res":
                h = self._resblock(sw, h)
            elif st.kind == "attn":
                h = self._attn(sw, h)
            elif st.kind == "conv_in":    # the decoder's z goes to a tensor-core conv_in in the operand dtype
                zin = h if self._act_dtype(sw, prec) == torch.float32 else L.groupnorm(h, None, None, swish=False, out_dtype=prec.opd, normalize=False)
                h = self._conv(sw, zin)
            elif st.kind == "down":
                if sw.tc and h.shape[1] % 2 == 0 and h.shape[2] % 2 == 0:      # space-to-depth operand for the tensor-core conv
                    hs = L.groupnorm(h, None, None, swish=False, out_dtype=prec.opd, normalize=False, s2d=True)
                    h = self._conv(sw, hs, stride=2)
                elif sw.tc:
                    raise NotImplementedError("odd feature-map size in Downsample on the tensor-core path")
                else:
                    h = self._conv(sw, h, stride=2)
            elif st.kind == "up":
                if sw.tc:      # nearest x2 materialised once in the operand dtype, then the tensor-core conv
                    hu = L.groupnorm(h, None, None, swish=False, out_dtype=prec.opd, normalize=False, upsample=True)
                    h = self._conv(sw, hu)
                else:          # exact path: upsampling folded into the conv's address arithmetic
                    h = self._conv(sw, h, upsample=True)
            else:              # out: GroupNorm + swish, conv_out (whose output feeds no GroupNorm)
                a = L.groupnorm(h, *sw["norm"], swish=True, out_dtype=self._act_dtype(sw["conv"], prec))
                h = self._conv(sw["conv"], a, stats=False)
        return h

    def _encoder(self, x):
        """Encoder.forward (vqgan_th.py:203-225); x f32 [N,H,W,in_channels] -> f32 [N,h,w,z_channels]."""
        return self._walk(self._w["enc"], x, self.enc_prec)

    def _decoder(self, z):
        """Decoder.forward (vqgan_th.py:291-318); z f32 [N,h,w,z_channels] (post_quant_conv applied) -> f32 [N,H,W,out_ch]."""
        return self._walk(self._w["dec"], z, self.dec_prec)

    # ------------------------------------------------------------------ quantizer
    def _quantize(self, z_rows, want_quant=True):
        """QuantizeEMA.forward (utils_th.py:32-68) on rows [M,D]; returns (quant rows | None, diff, idx)."""
        q = self._w["q"]
        if q["eh"] is not None:
            # fused wgmma lookup: z read once, scores never leave registers, near-ties settled in fp64: same indices as the fp32 kernel
            idx, quant, dsum = L.vq_lookup_fused(z_rows, q["et"], q["esq"], q["eh"], emb_dk=q["emb"], want_quant=want_quant, want_diff=True)
        else:
            idx, quant, dsum = L.vq_lookup(z_rows, q["et"], q["esq"], want_quant=want_quant, want_diff=True)
        if self.training and self.quantizer == "ema":
            self._ema_update(z_rows, idx)
        diff = (dsum / float(z_rows.numel())).to(torch.float32).reshape(())
        if self.quantizer == "commit":
            # utils_th.py:113-114: mean((sg(q) - z)^2) + beta mean((q - sg(z))^2) — one number twice, the gradients differ (train.py)
            diff = diff + self.beta * diff
        return quant, diff, idx

    def _ema_update(self, z_rows, idx):
        """Training branch, utils_th.py:46-64: counts / embed_sum (+ one packed all-reduce), EMA, renormalise."""
        q = self._w["q"]
        d, k = q["emb"].shape
        counts, esum = L.vq_ema_stats(z_rows, idx, k)
        from .dist import allreduce_ema_stats
        counts, esum = allreduce_ema_stats(counts, esum)            # one packed NCCL call instead of the reference's two
        q["counter"] += 1
        corr = float(1.0 - torch.pow(torch.tensor(self.decay), torch.tensor(q["counter"], dtype=torch.int64)))
        alpha = 1 - self.decay
        L.vq_ema_update(counts, esum, alpha, corr, self.eps, q["cs"], q["dw"], q["emb"], q["et"], q["esq"])
        if q["eh"] is not None:
            q["eh"] = L.vq_prepare_codebook_f16(q["et"])
        self._refresh_decode_table()

    # ------------------------------------------------------------------ NHWC entry points (TF-twin convention)
    def _in(self, x, dtype=torch.float32):
        t = torch.as_tensor(x)
        if t.device != self.device or t.dtype != dtype or not t.is_contiguous():
            t = t.to(device=self.device, dtype=dtype).contiguous()
        return t

    @L.on_model_device
    def encode_rows(self, x_nhwc):
        """f32 NHWC images -> (z rows [N*h*w, D], h, w)"""
        z = self._encoder(x_nhwc)
        n, hh, ww, c = z.shape
        zr = linear(self.exact, z.reshape(n * hh * ww, c), self._w["quant_conv"], torch.float32)
        return zr, hh, ww

    def _check_layout(self, t, channel_axis, what):
        if t.dim() != 4 or t.shape[channel_axis] != self.config.in_channels:
            raise ValueError(f"{what}: expected {'NCHW' if channel_axis == 1 else 'NHWC'} images with {self.config.in_channels} channels, "
                             f"got shape {tuple(t.shape)} (the torch flavour is NCHW, the TF flavour NHWC)")

    @L.on_model_device
    def encode_nhwc(self, x_nhwc):
        """TF-twin convention (viewformer/models/vqgan.py:291-295): NHWC in, (quant NHWC, diff, codes [N,h,w])."""
        self._need_weights()
        self._check_layout(torch.as_tensor(x_nhwc), 3, "encode_nhwc")
        x = self._in(x_nhwc)
        zr, hh, ww = self.encode_rows(x)
        n = x.shape[0]
        quant, diff, idx = self._quantize(zr)
        return quant.reshape(n, hh, ww, -1), diff, idx.reshape(n, hh, ww)

    @L.on_model_device
    def encode_u8(self, images_u8_nhwc, first_views=None):
        """uint8 NHWC images -> codes int64 [N,h,w] (evaluate_transformer.py:105-110 in one device pass).
        With ``first_views=n`` the input is [B,T,H,W,C] and views 0..n-1 of every scene are encoded ([B*n,h,w]).
        Any other dtype raises TypeError: a float image in [0, 1] cast to uint8 would become 0 / 1 bytes."""
        return self.encode_images(image_tensor(images_u8_nhwc, "encode_u8", (torch.uint8,)), first_views)

    @L.on_model_device
    def encode_images(self, images_nhwc, first_views=None):
        """``encode_u8`` for uint8 images or float32 images in [0, 1], the two inputs of the reference's
        ``tf.image.convert_image_dtype(images, tf.float32) * 2 - 1`` (the identity for float32): codes int64 [N,h,w]."""
        images = image_tensor(images_nhwc, "encode_images")
        if images.shape[-1] != self.config.in_channels:
            raise ValueError(f"encode_images: the codebook takes {self.config.in_channels}-channel images, got shape {tuple(images.shape)}")
        self._need_weights()
        x = self._in(images, images.dtype)
        x = L.u8_to_unit(x, first_views) if x.dtype == torch.uint8 else float_images.f01_to_unit(x, first_views)
        zr, hh, ww = self.encode_rows(x)
        _, _, idx = self._quantize(zr, want_quant=False)
        return idx.reshape(x.shape[0], hh, ww)

    @L.on_model_device
    def decode_code_nhwc(self, codes):
        self._need_weights()
        codes = self._in(codes, torch.int64)
        n, hh, ww = codes.shape
        z = L.gather_rows(self._w["pq_table"], codes.reshape(-1)).reshape(n, hh, ww, -1)
        return self._decoder(z)

    @L.on_model_device
    def decode_code_u8(self, codes):
        """codes -> uint8 NHWC images (clip, /2+.5, ->uint8; evaluate_transformer.py:127-129)."""
        return L.unit_to_u8(self.decode_code_nhwc(codes))

    # ------------------------------------------------------------------ torch-flavour (NCHW) surface
    def _need_weights(self):
        if self._w is None:
            raise RuntimeError("VQGAN has no weights: call load_state_dict() first")

    @L.on_model_device
    def encode(self, x):
        self._need_weights()
        self._check_layout(torch.as_tensor(x), 1, "encode")
        x = L.nchw_to_nhwc(self._in(x))
        zr, hh, ww = self.encode_rows(x)
        n = x.shape[0]
        quant, diff, idx = self._quantize(zr)
        return L.nhwc_to_nchw(quant.reshape(n, hh, ww, -1)), diff, idx.reshape(n, hh, ww)

    @L.on_model_device
    def decode(self, quant):
        self._need_weights()
        q = L.nchw_to_nhwc(self._in(quant))
        n, hh, ww, c = q.shape
        z = linear(self.exact, q.reshape(-1, c), self._w["post_quant_conv"], torch.float32).reshape(n, hh, ww, -1)
        return L.nhwc_to_nchw(self._decoder(z))

    @L.on_model_device
    def decode_code(self, code_b):
        return L.nhwc_to_nchw(self.decode_code_nhwc(code_b))

    @L.on_model_device
    def forward(self, input):
        quant, diff, idx = self.encode(input)
        return self.decode(quant), diff, quant, idx

    __call__ = forward

    @L.on_model_device
    def embed_code(self, embed_id):
        """utils_th.py:70-72: ids [N,h,w] -> [N,D,h,w]."""
        ids = self._in(embed_id, torch.int64)
        n, hh, ww = ids.shape
        return L.nhwc_to_nchw(L.gather_rows(self._w["q"]["et"], ids.reshape(-1)).reshape(n, hh, ww, -1))

    # ------------------------------------------------------------------ training (Lightning surface, vqgan_th.py:413-445)
    def configure_optimizers(self, resume_from_checkpoint=None, accumulate_grad_batches=None):
        """The trainer object that owns Adam(betas=(0.5, 0.9), lr=config.learning_rate) and the flat parameter / gradient buffers.
        ``resume_from_checkpoint``: a file written by ``VQGANTrainer.save_checkpoint`` (the reference's --resume-from-checkpoint,
        train/train_codebook_th.py:29,63): weights, EMA buffers, Adam's moments and step count continue from it.
        ``accumulate_grad_batches``: micro-batches per optimizer step (the reference's option of that name, train_codebook_th.py:30,67;
        see ``VQGANTrainer``); None keeps the trainer's (1 for a new one)."""
        from .train import VQGANTrainer
        if getattr(self, "_trainer", None) is None:
            if self._w is None and resume_from_checkpoint is not None:
                self.init_weights()                     # the trainer needs device buffers to restore into
            self._trainer = VQGANTrainer(self, precision=self.train_precision, accumulate_grad_batches=1 if accumulate_grad_batches is None else accumulate_grad_batches)
        elif accumulate_grad_batches is not None:
            if int(accumulate_grad_batches) < 1:
                raise ValueError(f"accumulate_grad_batches must be >= 1, got {accumulate_grad_batches}")
            self._trainer.accumulate_grad_batches = int(accumulate_grad_batches)
        if resume_from_checkpoint is not None:
            self._trainer.load_checkpoint(resume_from_checkpoint)
        return self._trainer

    @L.on_model_device
    def training_step(self, batch, batch_idx=0):
        """Loss of one optimisation step on ``batch`` (f32 NCHW in [-1,1]); gradients are exchanged and Adam applied inside."""
        return self.configure_optimizers().training_step(batch, batch_idx)

    @L.on_model_device
    def validation_step(self, batch, batch_idx=0):
        """vqgan_th.py:425-441: reconstruction and total loss without touching weights or the codebook."""
        was = self.training
        self.training = False
        xrec, diff, _, _ = self(batch)
        self.training = was
        x = self._in(batch)
        _, l1 = L.l1_grad(L.nchw_to_nhwc(x), L.nchw_to_nhwc(xrec), 0.0)
        rec = (l1 / x.numel()).to(torch.float32).reshape(())
        return {"val/rec_loss": rec, "val/aeloss": rec + float(self.config.codebook_weight) * diff, "reconstructed_image": xrec}
