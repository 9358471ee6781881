"""Every GEMM, convolution, attention, weight-gradient and codebook-lookup launch of the real workloads, and every GroupNorm / LayerNorm
(forward, statistics, backward), column-sum, softmax-backward, cross-entropy-gradient, embedding-gradient, GELU, lincomb3, Adam, Keras AdamW,
sumsq, split / bf16 conversion and dropout launch, and the evaluation's resize, pair sums and SSIM, checked against fp64 on its own operands (tests/launch_checks.py: references and bars).  The kernel tests pin each entry point at a few hand-picked shapes; the workloads
call the same entry points at dozens of others (tile shapes, tails, split-K and tile walks all depend on the shape), which were otherwise
only held by loose end-to-end bars.

Each wrapped call snapshots what it overwrites, runs the real wrapper, and is checked at once on the same stream, before later launches
reuse its buffers.  Sampling keeps full size cheap: GEMMs up to 3 batch indices x (first 128, last 128, 64 random rows) x all columns;
convs 3 images (first, last, one random) x all pixels; attention 3 (batch, head) pairs x all rows and streams, plus, when the persistent
kernel's CTAs walk more than one item, the pair of the last item and of a CTA's later item after a change of n_kt (launch_checks.
attn_walk_pairs, from this GPU's SM count); weight gradients in full.
Calls made while a CUDA graph is being captured are counted and skipped (all workloads here are eager).

Measured on an H100 80GB HBM3 (700 W power limit), worst ratio to the bar per workload (the file runs in about 30 s of pytest time):
  mixed generate, 3 scenes x 10 views (VF_NORM_ON_LOAD 0 and 1 alike): tc_gemm bf16 0.989 (bf16-output GEMMs: the output rounding bound
      itself), tc_conv bf16 0.84, attn_block_causal 0.64, simt_gemm 0.11, conv3x3_small_cin 0.089, tc_gemm split 0.047, tc_conv split 0.010,
      vq_lookup_fused 1e-4.
  tf32 encode + decode_code: conv3x3_small_cin 0.10, tc_gemm tf32 0.062, tc_conv tf32 0.011.
  C5 KV cache (19 context views, empty slot): tc_gemm bf16 0.89, attn_block_causal 0.66.
  bf16 codebook step, medium / full size: conv3x3_small_cin 0.075 / 0.12, simt_conv 0.066 / 0.068, conv_wgrad_bf16 0.0037 / 0.035,
      conv_wgrad_tc 0.0013 / 0.020, tc_gemm bf16 0.018 / 0.019, tc_conv bf16 0.0031 / 0.0035.
  bf16 transformer step, small (dropout 0.1) / full size: tc_gemm bf16 0.97 / 0.89, attn_multiend_train 0.54 / 0.61, attn_multiend_bwd
      0.32 / 0.70, conv_wgrad 0.17 / 0.26, dense_wgrad_bf16 0.093 / 0.20.
  At the benchmarked sizes, where attention CTAs walk several items (together about 14 s):
  mixed generate, the bench's 32 scenes (attention: 1920 items on 264 CTAs): tc_gemm bf16 0.989, groupnorm 0.996 (bf16), tc_conv bf16
      0.84, attn_block_causal 0.60, tc_gemm split 0.054, tc_conv split 0.011.
  bf16 transformer step at scripts/bench_migt_train.py's size (B = 5, T = 20, dropout 0.1; 600 items per stream on 132 CTAs): tc_gemm
      bf16 0.90, attn_multiend_train 0.73, attn_multiend_bwd 0.72, migt_embed_bwd 0.33, gelu_bwd 0.32, dense_wgrad_bf16 0.026.
  fp32 trainers, small: simt_gemm 0.076 / 0.23, dense_wgrad_tc 0.22, conv_wgrad 0.026 / 0.18, tc_gemm split 0.051, tc_conv split 0.0029.
  fp32 codebook step, medium / full size: sumpool2x2 0.94 / 0.98, simt_conv 0.068 / 0.068, conv_wgrad_tc 0.0026 / 0.020, tc_gemm split
      0.026 / 0.018, conv_wgrad 0.0050 / 0.054, tc_conv split 8.2e-4 / 8.2e-4, conv3x3_small_cout 2.4e-4 / 2.6e-4.
  fp32 transformer step, full size: layernorm_bwd 0.56, dense_wgrad_tc 0.52, softmax_rows 0.33, tc_gemm split 0.31, conv_wgrad 0.28,
      simt_gemm 0.27.
  Inference paths beyond the benchmark's mixed generate (same card; together about 41 s).  Each states the (wrapper, dtype, calling
  function) triples that prove its path ran (CALLERS) and the wrappers of other paths it must not reach (ABSENT):
  loc-generate-mixed, 3 scenes x 10 views (the localising forward, _pose_head, cameras_from_relative): tc_gemm bf16 0.994, tc_conv bf16
      0.84, attn_block_causal 0.58, pose_postprocess 0.14, simt_gemm 0.14 (_pose_head 768 -> 1536 -> 7), cameras_from_relative 0.018.
  multictx-mixed, 2 scenes (3 streams, argmax of all B T 64 rows, 20 images decoded): tc_gemm bf16 0.99, tc_conv bf16 0.85,
      attn_block_multiend 0.59, pose_postprocess 0.14, simt_gemm 0.11.
  allimg-loc / allimg-noloc, 5 scenes in batches of 2, 2, 1 (3 / 2 streams): tc_gemm bf16 0.90 / 0.90, attn_block_multiend 0.65 / 0.65,
      simt_gemm 0.12 / 0.12, pose_postprocess 0.095 / -.
  kv-cache-shared (one scene, 19 context views, 8 queries on _query_block; fused decode at 18 context views, no empty slot): tc_gemm bf16
      0.994, softmax_rows 0.994 (bf16 output: its rounding bound), attn_block_causal 0.58.
  bf16-generate / tf32-generate / fp32-generate (bench.model_pair, 3 / 3 / 2 scenes): tc_conv bf16 0.84, tc_gemm bf16 0.993,
      attn_block_causal 0.60, vq_lookup_fused 3e-5 / tc_gemm tf32 0.11 (causal QK^T with skipped tiles, P.V with the k limit),
      softmax_rows 0.34, tc_conv tf32 0.011 / simt_gemm 0.13, softmax_rows 0.35, simt_conv 0.0034, vq_lookup 2e-4.
  test-step-bf16-full, 2 scenes (3 streams, losses of every row): tc_gemm bf16 0.90, attn_block_multiend 0.69, pose_loss_rows 0.35,
      row_mean 0.069, cross_entropy_rows 0.0087.
  Not audited: the tf32 and fp32 3-stream forwards at full size (multi-context generate, localising generate and test_step at those
  precisions; their kernels are audited in the single-stream generates above and in the small fp32 test_step), the x3 codebook's decoder,
  and launches replayed from a CUDA graph (GraphedPredictions equals the eager call bit for bit, tests/test_persistent_walks_gpu.py).
  tests/test_eval_paths_gpu.py checks every batch entry of the multi-stream and shared-scene query paths for batch invariance.
Normalisation, reduction, optimizer and elementwise wrappers (same card; the 14 workloads and tests/test_norm_stats_gpu.py: about 45 s):
  generate / codec / KV cache: groupnorm 0.996 (bf16 outputs: the output rounding itself), layernorm 0.995 (bf16), gn_mean_rstd 0.15 (fused
      sums of a bf16 output) / 0.0096 (statistics pass), split_f16x2 bit-exact.  Largest GroupNorm mean^2 / var: 1.14.
  codebook steps (fp32 small, bf16 medium / full; full training_step with clipping): gn_mean_rstd 0.14 (statistics pass), groupnorm 0.996,
      lincomb3 0.47, adam 0.48, softmax_bwd_rows 0.15, groupnorm_bwd 0.056, col_sums 0.053, sumsq 0.0042.  Largest mean^2 / var: 4.59.
  transformer steps (fp32 small, bf16 small / full; train_step with clipping): layernorm 0.996 (bf16), migt_embed_bwd 0.32, gelu_bwd 0.32,
      layernorm_bwd 0.25, lincomb3 0.25, gelu 0.24, cross_entropy_grad 0.22, col_sums 0.12, softmax_bwd_rows 0.09, sumsq 0.06,
      adamw_keras 0.024; to_bf16 and dropout bit-exact / exact in form.
  softmax_rows 0.995 (bf16 output, generate) / 0.18 (fp32, mask modes 0, 1, 2), sumpool2x2 0.975, pose_loss_rows 0.51, vq_commit_grad
      0.34, pose_loss_grad 0.29, vq_ema_update 0.25, vq_ema_stats 0.20, pose_postprocess 0.12, cameras_prepare 0.089, vq_prepare_codebook
      0.078, row_mean 0.052, cameras_from_relative 0.037, cross_entropy_rows 0.011, l1_grad 0.011; bit-exact: u8_to_unit, unit_to_u8, the
      layout conversions, gather_rows, vq_prepare_codebook_f16, migt_embed, argmax_rows, image_pair_sums, resize_u8 (evaluation).
  ssim_u8 0.014 (evaluation, K1 = 1; exact integer window moments, S in fp64: a bar of about 1e-14 of S).
  The whole file ran in about 105 s of pytest time with 31 workloads (H100 80GB HBM3, 700 W); the nine inference workloads above take
  about 41 s of it.  The largest GroupNorm mean^2 / var above comes from synthetic random-weight models.
"""
import os
import random
import statistics
import sys
from collections import defaultdict

import pytest
import torch

import launch_checks as lc
from oracle import synth, migt_oracle as mo
from oracle.make_golden import vq_images, SMALL_VQ, MIGT_TRAIN
from viewformer_b200.config import VQGANConfig, MIGTConfig

pytestmark = pytest.mark.gpu

_SKIP_FILES = ("_lib.py", "ops.py", "launch_checks.py", os.path.basename(__file__))


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


class Audit:
    """Wraps every checked ``_lib`` wrapper; records (calls, worst ratio) per (wrapper, operand dtype, caller file:line, caller function)."""

    def __init__(self, L, monkeypatch, seed=0):
        self.rec = defaultdict(list)
        self.skipped = 0
        self.rng = random.Random(seed)
        orig = {name: getattr(L, name) for name in lc.CHECKERS}
        groupnorm, dropout = L.groupnorm, L.dropout
        monkeypatch.setitem(lc.HOOKS, "gn_apply_bf16", lambda x, mr, gamma, beta, swish: groupnorm(
            x.contiguous(), gamma, beta, swish=swish, out_dtype=torch.bfloat16, stats=mr.contiguous(), groups=mr.shape[1]))
        monkeypatch.setitem(lc.HOOKS, "dropout_mask", lambda shape, rate, seed, device: dropout(
            torch.ones(shape, dtype=torch.float32, device=device), rate, seed))
        monkeypatch.setitem(lc.HOOKS, "ref_lookup", lambda z, et, esq: orig["vq_lookup"](z, et, esq, want_quant=False, want_diff=False)[0])
        monkeypatch.setitem(lc.HOOKS, "gn_mean_rstd", orig["gn_mean_rstd"])
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        monkeypatch.setitem(lc.HOOKS, "attn_resident", lambda train: (1 if train else 2) * sms)
        monkeypatch.setitem(lc.HOOKS, "tc_ctas", lambda: sms)
        lc.GN_COND.clear()
        for name, fn in orig.items():
            monkeypatch.setattr(L, name, self._wrap(name, fn))

    @staticmethod
    def _site():
        """(file:line, function) of the first frame outside the wrappers and the checkers: the model method that made the call."""
        f = sys._getframe(2)
        while f is not None and os.path.basename(f.f_code.co_filename) in _SKIP_FILES:
            f = f.f_back
        return ("?", "?") if f is None else (f"{os.path.basename(f.f_code.co_filename)}:{f.f_lineno}", f.f_code.co_name)

    def _wrap(self, name, fn):
        def call(*a, **k):
            if torch.cuda.is_current_stream_capturing():
                self.skipped += 1
                return fn(*a, **k)
            first = next((v for v in list(a) + list(k.values()) if isinstance(v, torch.Tensor)), None)
            dtype = "-" if first is None else str(first.dtype).replace("torch.", "")
            with torch.no_grad():
                result, r = lc.run_check(name, fn, a, k, self.rng)
            self.rec[(name, dtype) + self._site()].append(r)
            return result
        return call

    def report(self, tag):
        print(f"\n[audit {tag}] {'wrapper':<20} {'dtype':<9} {'site':<22} {'function':<36} {'calls':>5} {'worst':>8} {'median':>8}")
        bad = []
        for (name, dtype, site, func), rs in sorted(self.rec.items()):
            worst = max(rs)
            print(f"[audit {tag}] {name:<20} {dtype:<9} {site:<22} {func:<36} {len(rs):>5} {worst:>8.3g} {statistics.median(rs):>8.3g}"
                  + ("  <-- over its bar" if worst > 1.0 else ""))
            if worst > 1.0:
                bad.append(f"{name} {dtype} {site} {func}: worst ratio {worst:.3g} over {len(rs)} calls")
        per = defaultdict(float)
        for (name, dtype, _, _), rs in self.rec.items():
            per[(name, dtype)] = max(per[(name, dtype)], max(rs))
        print(f"[audit {tag}] worst per wrapper: " + ", ".join(f"{n}/{d} {v:.3g}" for (n, d), v in sorted(per.items()))
              + f"; skipped while capturing: {self.skipped}")
        if lc.GN_COND:
            print(f"[audit {tag}] largest GroupNorm mean^2/var: {max(lc.GN_COND):.3g} over {len(lc.GN_COND)} statistics calls")
        return bad

    def reached(self):
        return {(name, dtype) for name, dtype, _, _ in self.rec}

    def callers(self):
        """(wrapper, operand dtype, calling function) of every recorded call."""
        return {(name, dtype, func) for name, dtype, _, func in self.rec}


def _mixed_generate(monkeypatch, L, norm_on_load, scenes=3):
    import bench
    from viewformer_b200 import VQGAN, MIGT, generate_batch_predictions
    monkeypatch.setenv("VF_NORM_ON_LOAD", norm_on_load)
    vcfg, tcfg = VQGANConfig(), MIGTConfig(localization_weight="0")
    cb = VQGAN(vcfg, precision="mixed").load_state_dict(synth.make_vqgan_state_dict(vcfg, 0))
    tr = MIGT(tcfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(tcfg, 0))
    images, cams = bench.synth_inputs(scenes, 1234)
    generate_batch_predictions(tr, cb, images, cams)


def _tf32_codec(monkeypatch, L):
    from viewformer_b200 import VQGAN
    cfg = VQGANConfig()
    model = VQGAN(cfg, precision="tf32").load_state_dict(synth.make_vqgan_state_dict(cfg, 1))
    codes = model.encode(vq_images(2, cfg.image_size, 21))[2]
    model.decode_code(codes)


def _kv_cache(monkeypatch, L):
    from viewformer_b200 import MIGT
    cfg = MIGTConfig(localization_weight="0")
    model = MIGT(cfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(cfg, 5))
    B, T = 2, 20
    codes = synth.make_codes(B, T, seed=31)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=32))[0])
    cache = model.prefill_context(codes[:, :-1], cams[:, :-1].contiguous())
    model.query(cache, cams[:, -1].contiguous(), return_logits=True)


def _vq_step(cfg_kw, n, precision, seed, full=False):
    """forward_backward, or with ``full`` the whole training_step (the quantizer's EMA update, the clipped Adam step)."""
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    cfg = VQGANConfig(**cfg_kw)
    model = VQGAN(cfg, precision="fp32").load_state_dict(synth.make_vqgan_state_dict(cfg, 5))
    tr = VQGANTrainer(model, precision=precision)
    x = vq_images(n, cfg.image_size, seed)
    tr.training_step(x) if full else tr.forward_backward(x)


def _migt_step(cfg_kw, B, T, precision, seed, full=False):
    """forward_backward, or with ``full`` the whole train_step (per-tensor clipping, Keras AdamW, the accuracy's argmax)."""
    from viewformer_b200 import MIGT
    from viewformer_b200.train_migt import MIGTTrainer
    cfg = MIGTConfig(**cfg_kw)
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=seed)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=seed + 1))[0])
    tr = MIGTTrainer(model, seed=seed, precision=precision)
    tr.train_step((cams, codes)) if full else tr.forward_backward(cams, codes)


_EMA_KEYS = {"quantize.counter", "quantize.ema_cluster_size_hidden", "quantize.ema_dw_hidden"}


def _vq_commit_step(monkeypatch, L):
    """A full codebook training step with the commitment quantizer (Quantize): reaches vq_ema_stats + vq_commit_grad."""
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    cfg = VQGANConfig(**dict(SMALL_VQ, perceptual_weight=0.0, gradient_clip_val=0.5))
    sd = {k: v for k, v in synth.make_vqgan_state_dict(cfg, 5).items() if k not in _EMA_KEYS}        # Quantize has no EMA buffers
    model = VQGAN(cfg, precision="fp32", quantizer="commit").load_state_dict(sd)
    VQGANTrainer(model, precision="fp32").training_step(vq_images(3, cfg.image_size, 5100))


def _fp32_inference(monkeypatch, L):
    """fp32 models: the codec (AttnBlock softmax), the transformer's teacher-forced 3-stream forward with its losses (test_step: mask modes
    1 and 2, cross_entropy_rows, pose_loss_rows, row_mean, argmax_rows), and the KV-cache query of an fp32 model (mask mode 0)."""
    from viewformer_b200 import VQGAN, MIGT
    vcfg = VQGANConfig(**dict(SMALL_VQ, perceptual_weight=0.0))
    codec = VQGAN(vcfg, precision="fp32").load_state_dict(synth.make_vqgan_state_dict(vcfg, 2))
    codec.decode_code(codec.encode(vq_images(2, vcfg.image_size, 5200))[2])
    cfg = MIGTConfig(**dict(MIGT_TRAIN, localization_weight="0.5"))
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    B, T = 2, 4
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=5300)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=5301))[0])
    model.test_step((cams, codes))
    cache = model.prefill_context(codes[:, :-1], cams[:, :-1].contiguous())
    model.query(cache, cams[:, -1].contiguous(), return_logits=True)


def _evaluation(monkeypatch, L):
    """metrics.Evaluator at 128 x 128 (the reference's resize rules and SSIM K1 = 1): a 160 x 160 ground truth shrunk bilinearly, a 96 x 96
    generated view grown bilinearly, then the exact pair sums and SSIM."""
    from viewformer_b200.metrics import Evaluator
    g = torch.Generator().manual_seed(5400)
    base = torch.rand(4, 3, 20, 20, generator=g)
    gt = (torch.nn.functional.interpolate(base, size=(160, 160), mode="bilinear") * 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    gen = (torch.nn.functional.interpolate(base + 0.05 * torch.rand(4, 3, 20, 20, generator=g), size=(96, 96), mode="bilinear").clamp(0, 1)
           * 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    Evaluator(image_size=128).update_with_image(gt.cuda(), gen.cuda())


def _mixed_pair(localization_weight, seed):
    """The benchmark's mixed pair (exact encoder, bf16 decoder, bf16 transformer) at full size with synthetic weights."""
    from viewformer_b200 import VQGAN, MIGT
    vcfg, tcfg = VQGANConfig(), MIGTConfig(localization_weight=localization_weight)
    cb = VQGAN(vcfg, precision="mixed").load_state_dict(synth.make_vqgan_state_dict(vcfg, seed))
    tr = MIGT(tcfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(tcfg, seed))
    return cb, tr


def _loc_generate(monkeypatch, L, localization_weight="1"):
    """generate_batch_predictions with the default config (localisation on): the second, localising forward over all T views (T - 1 pose
    rows and the localisation token's row for the last view), then _pose_head, reduce_cameras and cameras_from_relative."""
    import bench
    from viewformer_b200 import generate_batch_predictions
    cb, tr = _mixed_pair(localization_weight, 10)
    images, cams = bench.synth_inputs(3, 6100)
    generate_batch_predictions(tr, cb, images, cams)


def _multictx(monkeypatch, L):
    """generate_batch_predictions_multictx: the 3-stream forward on attn_block_multiend, logits and argmax of all B T 64 rows, poses of
    every view, and the decoder over B T images."""
    import bench
    from viewformer_b200 import generate_batch_predictions_multictx
    cb, tr = _mixed_pair("1", 11)
    images, cams = bench.synth_inputs(2, 6200)
    generate_batch_predictions_multictx(tr, cb, images, cams)


def _allimg(monkeypatch, L, localization_weight):
    """run_with_batchsize(transformer_predict, 2, ...) over 5 scenes x 10 views: batches of 2, 2 and 1 scenes, 3 streams with
    localisation and 2 without."""
    from viewformer_b200 import MIGT
    from viewformer_b200.evaluate import run_with_batchsize, transformer_predict
    cfg = MIGTConfig(localization_weight=localization_weight)
    tr = MIGT(cfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(cfg, 12))
    cams, codes = synth.make_cameras(5, 10, seed=6300), synth.make_codes(5, 10, seed=6301)
    run_with_batchsize(transformer_predict, 2, cams, codes, transformer_model=tr)


def _kv_shared(monkeypatch, L, queries_per_scene=False):
    """The KV cache of a bf16 full-size model: one scene (19 context views) shared by 8 query poses, which runs _query_block (stride-0 cache
    batch, the softmax over S_ctx + 64 columns, the own-view P.V with the fp32 residual); then the fused decode at 2 scenes with 18 context
    views, where the query tile holds no empty view slot.  ``queries_per_scene`` gives the shared cache one query only."""
    from viewformer_b200 import MIGT
    cfg = MIGTConfig(localization_weight="0")
    model = MIGT(cfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(cfg, 13))
    codes = synth.make_codes(2, 19, seed=6400)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(2, 27, seed=6401))[0])
    shared = model.prefill_context(codes[:1], cams[:1, :19].contiguous())
    model.query(shared, cams[0, 19:20 if queries_per_scene else 27].contiguous(), return_logits=True)
    cache = model.prefill_context(codes[:, :18], cams[:, :18].contiguous())
    model.query(cache, cams[:, 18].contiguous(), return_logits=True)


def _generate(monkeypatch, L, precision, scenes):
    """The benchmark's generate at one of its other precisions: the models of bench.model_pair, localisation off."""
    import bench
    from viewformer_b200 import generate_batch_predictions
    cb, tr = bench.model_pair(precision, VQGANConfig(), MIGTConfig(localization_weight="0"), torch.device("cuda"))
    images, cams = bench.synth_inputs(scenes, 6500)
    generate_batch_predictions(tr, cb, images, cams)


def _test_step_bf16(monkeypatch, L):
    """The reference's validation step on a bf16 full-size model (localisation on): the teacher-forced 3-stream forward, cross-entropy and
    pose losses of every row, their row means, and the accuracy's argmax."""
    from viewformer_b200 import MIGT
    cfg = MIGTConfig()
    model = MIGT(cfg, precision="bf16").load_state_dict(synth.make_migt_state_dict(cfg, 14))
    codes = synth.make_codes(2, 10, seed=6600)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(2, 10, seed=6601))[0])
    model.test_step((cams, codes))


MEDIUM_VQ = dict(ch=128, ch_mult=[1, 2], attn_resolutions=[16], image_size=32, n_embed=256, perceptual_weight=0.0)
SMALL_MIGT_BF16 = dict(n_layer=2, d_model=256, n_head=4, token_image_size=8, n_loss_skip=1, weight_decay=0.01, total_steps=100, learning_rate=1e-3,
                       label_smoothing=0.05, localization_weight="0.5", image_generation_weight=0.8, pose_multiplier=1.0, dropout=0.1)
FULL_MIGT_TRAIN = dict(dropout=0.0, label_smoothing=0.1, localization_weight="0.7", total_steps=100, learning_rate=1e-4)

MIXED_NORMS = {("gn_mean_rstd", "bfloat16"), ("gn_mean_rstd", "float32"), ("groupnorm", "bfloat16"), ("groupnorm", "float32"), ("layernorm", "float32"),
               ("split_f16x2", "float32")}
VQ_BWD = {("gn_mean_rstd", "float32"), ("groupnorm", "float32"), ("groupnorm_bwd", "float32"), ("col_sums", "float32"), ("lincomb3", "float32"),
          ("softmax_bwd_rows", "float32")}
MIGT_BWD = {("layernorm", "float32"), ("layernorm_bwd", "float32"), ("gelu", "float32"), ("gelu_bwd", "float32"), ("cross_entropy_grad", "float32"),
            ("migt_embed_bwd", "float32"), ("col_sums", "float32"), ("lincomb3", "float32")}
VQ_BF16_STEP = {("tc_conv", "bfloat16"), ("tc_conv", "float16"), ("tc_gemm", "bfloat16"), ("conv_wgrad_bf16", "float32"),
                ("conv_wgrad_tc", "float32"), ("simt_conv_dgrad_s2", "float32"), ("vq_lookup", "float32")} | VQ_BWD | {("split_f16x2", "float32")}
VQ_FP32_STEP = {("tc_conv", "float16"), ("conv_wgrad_tc", "float32"), ("conv3x3_small_cout", "float32"), ("conv3x3_small_cin", "float32"),
                ("simt_conv", "float32"), ("simt_conv_dgrad_s2", "float32"), ("conv_wgrad", "float32"), ("simt_gemm", "float32"),
                ("sumpool2x2", "float32"), ("vq_lookup", "float32"), ("split_f16x2", "float32")} | VQ_BWD

# workload -> (run, the (wrapper, operand dtype) pairs it is known to reach)
WORKLOADS = {
    "mixed-generate-norm0": (lambda mp, L: _mixed_generate(mp, L, "0"),
                             {("tc_conv", "bfloat16"), ("tc_conv", "float16"), ("tc_gemm", "bfloat16"), ("attn_block_causal", "bfloat16"),
                              ("vq_lookup_fused", "float32")} | MIXED_NORMS),
    "mixed-generate-norm1": (lambda mp, L: _mixed_generate(mp, L, "1"),
                             {("tc_conv", "bfloat16"), ("tc_conv", "float16"), ("tc_gemm", "bfloat16"), ("attn_block_causal", "bfloat16"),
                              ("vq_lookup_fused", "float32")} | MIXED_NORMS),
    "mixed-generate-bench": (lambda mp, L: _mixed_generate(mp, L, "0", scenes=32),
                             {("tc_conv", "bfloat16"), ("tc_conv", "float16"), ("tc_gemm", "bfloat16"), ("attn_block_causal", "bfloat16"),
                              ("vq_lookup_fused", "float32")} | MIXED_NORMS),
    "tf32-codec": (_tf32_codec, {("tc_conv", "float32"), ("tc_gemm", "float32"), ("vq_lookup_fused", "float32"), ("gn_mean_rstd", "float32"),
                                 ("groupnorm", "float32")}),
    "kv-cache-c5": (_kv_cache, {("attn_block_causal", "bfloat16"), ("tc_gemm", "bfloat16"), ("layernorm", "float32")}),
    "vq-step-bf16-medium": (lambda mp, L: _vq_step(MEDIUM_VQ, 4, "bf16", 4100), VQ_BF16_STEP),
    "vq-step-bf16-full": (lambda mp, L: _vq_step(dict(perceptual_weight=0.0), 2, "bf16", 4200), VQ_BF16_STEP),
    "migt-step-bf16-small": (lambda mp, L: _migt_step(SMALL_MIGT_BF16, 2, 5, "bf16", 4300),
                             {("attn_multiend_train", "bfloat16"), ("attn_multiend_bwd", "bfloat16"), ("tc_gemm", "bfloat16")} | MIGT_BWD | {("to_bf16", "float32")}),
    "migt-step-bf16-full": (lambda mp, L: _migt_step(FULL_MIGT_TRAIN, 1, 5, "bf16", 4400),
                            {("attn_multiend_train", "bfloat16"), ("attn_multiend_bwd", "bfloat16"), ("tc_gemm", "bfloat16")} | MIGT_BWD | {("to_bf16", "float32")}),
    "migt-step-bf16-bench": (lambda mp, L: _migt_step(dict(FULL_MIGT_TRAIN, dropout=0.1), 5, 20, "bf16", 5500),
                             {("attn_multiend_train", "bfloat16"), ("attn_multiend_bwd", "bfloat16"), ("tc_gemm", "bfloat16")} | MIGT_BWD
                             | {("to_bf16", "float32")}),
    "vq-step-fp32-small": (lambda mp, L: _vq_step(dict(SMALL_VQ, perceptual_weight=0.0), 3, "fp32", 4500),
                           {("simt_gemm", "float32"), ("simt_conv", "float32"), ("simt_conv_dgrad_s2", "float32"), ("conv_wgrad", "float32"),
                            ("tc_conv", "float16"), ("vq_lookup", "float32")} | VQ_BWD),
    "migt-step-fp32-small": (lambda mp, L: _migt_step(MIGT_TRAIN, 2, 4, "fp32", 4600),
                             {("tc_gemm", "float16"), ("simt_gemm", "float32"), ("dense_wgrad_tc", "float32"), ("conv_wgrad", "float32")} | MIGT_BWD
                             | {("softmax_bwd_rows", "float32")}),
    "vq-step-fp32-medium": (lambda mp, L: _vq_step(MEDIUM_VQ, 4, "fp32", 5600), VQ_FP32_STEP),
    "vq-step-fp32-full": (lambda mp, L: _vq_step(dict(perceptual_weight=0.0), 2, "fp32", 5700), VQ_FP32_STEP),
    "migt-step-fp32-full": (lambda mp, L: _migt_step(FULL_MIGT_TRAIN, 1, 5, "fp32", 5800),
                            {("tc_gemm", "float16"), ("simt_gemm", "float32"), ("dense_wgrad_tc", "float32"), ("conv_wgrad", "float32")} | MIGT_BWD
                            | {("softmax_bwd_rows", "float32")}),
    "vq-train-fp32-small": (lambda mp, L: _vq_step(dict(SMALL_VQ, perceptual_weight=0.0, gradient_clip_val=0.5), 3, "fp32", 4700, full=True),
                           {("adam", "float32"), ("sumsq", "float32"), ("vq_ema_update", "float32"), ("vq_ema_stats", "float32"),
                            ("softmax_rows", "float32")} | VQ_BWD),
    "vq-train-bf16-medium": (lambda mp, L: _vq_step(dict(MEDIUM_VQ, gradient_clip_val=0.5), 4, "bf16", 4800, full=True),
                             {("adam", "float32"), ("sumsq", "float32"), ("vq_ema_update", "float32"), ("vq_ema_stats", "float32"),
                              ("vq_prepare_codebook", "float32")} | VQ_BF16_STEP),
    "vq-train-commit-fp32-small": (_vq_commit_step, {("vq_commit_grad", "float32"), ("vq_ema_stats", "float32"), ("adam", "float32"),
                                                     ("sumsq", "float32"), ("vq_prepare_codebook", "float32")} | VQ_BWD),
    "fp32-inference": (_fp32_inference, {("softmax_rows", "float32"), ("cross_entropy_rows", "float32"), ("pose_loss_rows", "float32"),
                                         ("row_mean", "float32"), ("argmax_rows", "float32"), ("migt_embed", "int32"),
                                         ("pose_postprocess", "float32"), ("layernorm", "float32"), ("gn_mean_rstd", "float32"),
                                         ("groupnorm", "float32")}),
    "evaluation": (_evaluation, {("resize_u8", "uint8"), ("image_pair_sums", "uint8"), ("ssim_u8", "uint8")}),
    "migt-train-fp32-small": (lambda mp, L: _migt_step(dict(MIGT_TRAIN, gradient_clip_val=1.0), 2, 4, "fp32", 4900, full=True),
                              {("adamw_keras", "float32"), ("sumsq", "float32")}),
    "migt-train-bf16-small": (lambda mp, L: _migt_step(dict(SMALL_MIGT_BF16, gradient_clip_val=1.0), 2, 5, "bf16", 5000, full=True),
                              {("adamw_keras", "float32"), ("sumsq", "float32")}),
    # inference paths beyond the benchmark's mixed generate
    "loc-generate-mixed": (_loc_generate, {("attn_block_causal", "bfloat16"), ("cameras_from_relative", "float32")} | MIXED_NORMS),
    "multictx-mixed": (_multictx, {("attn_block_multiend", "bfloat16"), ("argmax_rows", "float32"), ("pose_postprocess", "float32"),
                                   ("tc_conv", "bfloat16")}),
    "allimg-loc": (lambda mp, L: _allimg(mp, L, "1"), {("attn_block_multiend", "bfloat16"), ("argmax_rows", "float32")}),
    "allimg-noloc": (lambda mp, L: _allimg(mp, L, "0"), {("attn_block_multiend", "bfloat16"), ("argmax_rows", "float32")}),
    "kv-cache-shared": (_kv_shared, {("tc_gemm", "bfloat16"), ("softmax_rows", "float32"), ("attn_block_causal", "bfloat16")}),
    "bf16-generate": (lambda mp, L: _generate(mp, L, "bf16", 3), {("tc_conv", "bfloat16"), ("vq_lookup_fused", "float32"),
                                                                  ("attn_block_causal", "bfloat16")}),
    "tf32-generate": (lambda mp, L: _generate(mp, L, "tf32", 3), {("tc_gemm", "float32"), ("softmax_rows", "float32"), ("tc_conv", "float32")}),
    "fp32-generate": (lambda mp, L: _generate(mp, L, "fp32", 2), {("simt_gemm", "float32"), ("softmax_rows", "float32"), ("simt_conv", "float32"),
                                                                  ("vq_lookup", "float32")}),
    "test-step-bf16-full": (_test_step_bf16, {("attn_block_multiend", "bfloat16"), ("cross_entropy_rows", "float32"),
                                              ("pose_loss_rows", "float32"), ("row_mean", "float32")}),
}

# workload -> (wrapper, operand dtype, calling function) triples that prove its path ran: tc_gemm / bf16, say, is reached from everywhere,
# tc_gemm / bf16 from MIGT._query_block only when the shared-scene query runs
POSE_HEAD = {("layernorm", "float32", "_pose_head"), ("simt_gemm", "float32", "_pose_head"), ("pose_postprocess", "float32", "_pose_head")}
CALLERS = {
    "loc-generate-mixed": {("attn_block_causal", "bfloat16", "_attention"), ("cameras_from_relative", "float32", "generate_batch_predictions")}
                          | POSE_HEAD,
    "multictx-mixed": {("attn_block_multiend", "bfloat16", "_attention"), ("argmax_rows", "float32", "generate_batch_predictions_multictx"),
                       ("tc_conv", "bfloat16", "_conv")} | POSE_HEAD,
    "allimg-loc": {("attn_block_multiend", "bfloat16", "_attention"), ("argmax_rows", "float32", "transformer_predict"),
                   ("cameras_from_relative", "float32", "transformer_predict")} | POSE_HEAD,
    "allimg-noloc": {("attn_block_multiend", "bfloat16", "_attention"), ("argmax_rows", "float32", "transformer_predict")},
    "kv-cache-shared": {("tc_gemm", "bfloat16", "_query_block"), ("softmax_rows", "float32", "_query_block"),
                        ("attn_block_causal", "bfloat16", "_query_block_fused")},
    "bf16-generate": {("tc_conv", "bfloat16", "_conv"), ("vq_lookup_fused", "float32", "_quantize"), ("attn_block_causal", "bfloat16", "_attention")},
    "tf32-generate": {("tc_gemm", "float32", "_attention"), ("softmax_rows", "float32", "_attention")},
    "fp32-generate": {("simt_gemm", "float32", "_attention"), ("softmax_rows", "float32", "_attention"), ("simt_conv", "float32", "_conv")},
    "test-step-bf16-full": {("attn_block_multiend", "bfloat16", "_attention"), ("cross_entropy_rows", "float32", "__call__"),
                            ("pose_loss_rows", "float32", "__call__"), ("row_mean", "float32", "__call__")},
}

# workload -> (wrapper, operand dtype, calling function) patterns it must never reach (None matches anything): reaching one means the
# workload ran another path than the one it is named for
TENSOR_CORE = {(w, None, None) for w in ("tc_gemm", "tc_conv", "attn_block_causal", "attn_block_multiend", "attn_multiend_train",
                                         "attn_multiend_bwd", "vq_lookup_fused", "conv_wgrad_tc", "conv_wgrad_bf16", "dense_wgrad_tc",
                                         "dense_wgrad_bf16")}
ABSENT = {
    "allimg-noloc": {("pose_postprocess", None, None), ("simt_gemm", None, "_pose_head"), ("cameras_from_relative", None, None)},
    "bf16-generate": {("tc_conv", "float16", None), ("split_f16x2", None, None)},                   # the exact encoder
    "tf32-generate": {("attn_block_causal", None, None), ("tc_conv", "float16", None), ("tc_gemm", "bfloat16", None)},
    "fp32-generate": TENSOR_CORE,
}


@pytest.mark.parametrize("workload", list(WORKLOADS))
def test_launch_audit(L, monkeypatch, workload):
    """One eager run of the workload with every checked launch held to its fp64 bar (ratio <= 1), the expected wrappers reached (from the
    stated callers), and none of the wrappers of another path."""
    run, expected = WORKLOADS[workload]
    audit = Audit(L, monkeypatch)
    run(monkeypatch, L)
    torch.cuda.synchronize()
    bad = audit.report(workload)
    missing = expected - audit.reached()
    missing_calls = CALLERS.get(workload, set()) - audit.callers()
    present = sorted(c for c in audit.callers() for pat in ABSENT.get(workload, ())
                     if all(p is None or p == v for p, v in zip(pat, c)))
    torch.cuda.empty_cache()
    assert not missing, f"{workload}: the audit never saw {sorted(missing)}"
    assert not missing_calls, f"{workload}: the audit never saw these (wrapper, dtype, caller) calls: {sorted(missing_calls)}"
    assert not present, f"{workload}: reached wrappers of another path: {present}"
    assert not bad, "launches outside their bar:\n  " + "\n  ".join(bad)

