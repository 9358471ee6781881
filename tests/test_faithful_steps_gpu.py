"""Both fp32 training steps against fp64 autograd, tensor by tensor, at the sizes where their split-fp16 tensor-core routes run.

Each case runs one ``forward_backward`` twice from the same weights and inputs: as shipped (tensor cores) and under VF_TRAIN_TC=0 (every
kernel on the CUDA cores).  Every exported gradient g is compared with g64, fp64 autograd through the oracle (codebook: the quantizer's
codes fixed to the trainer's; transformer: ``migt_oracle.forward(..., compute_losses=True)`` in float64, dropout 0):
    e = ||g - g64|| / max(||g64||, 1e-4),   and the tensor-core step passes when  e_tc <= 2 e_cuda + STEP_FLOOR  for every tensor.
A ratio test passes trivially if the tensor-core run falls back to the CUDA cores, so each run counts the calls of its routes
(``Routes``): the tensor-core run must reach ``VQ_ROUTES`` / ``MIGT_ROUTES`` (split-fp16 ``tc_conv`` in the forward pass and in the data
gradient, ``conv_wgrad_tc`` on plain and on x2-upsampled operands, ``conv3x3_small_cout``, ``sumpool2x2``; ``dense_wgrad_tc`` and split
``tc_gemm``), and the VF_TRAIN_TC=0 run none of the tensor-core entry points (``TC_ROUTES``).

Cases: the codebook at a medium size (ch 128, ch_mult [1, 2], attention at 16 x 16, 32 x 32 images, 4 of them; both quantizers) and at
full size (VQGANConfig defaults, 2 images of 128 x 128, EMA quantizer); the transformer small (MIGT_TRAIN, B = 2, T = 4) and full size
(12 layers, d = 768, B = 1, T = 5).  The medium codebook reaches conv_wgrad_tc at 128 and 256 channels and on the upsample conv's x2
operand, conv3x3_small_cout, the split convs at 128 and 256 channels, the 16 x 16 attention block, the stride-2 data gradient and a
nin_shortcut; the small config of tests/test_exact_split_gpu.py (ch 32) reaches none of the first three.

A dropped border row in conv_wgrad_tc (its input's last pixel row zeroed, at the wrapper: no kernel changes) is flagged on exactly the
weight gradients that kernel computes (``test_faithful_bar_flags_dropped_wgrad_row``).

Measured on an H100 80GB HBM3 (700 W power limit), e per tensor, median / worst, tensor cores vs CUDA cores, and the largest ratio:
  vq-medium-ema (206 tensors)       7.3e-7 / 1.4e-6  vs  1.6e-6 / 3.7e-6,  1.25
  vq-medium-commit (207, codebook)  7.4e-7 / 1.4e-6  vs  1.6e-6 / 3.7e-6,  1.25
  vq-full-ema (342)                 1.6e-6 / 5.1e-6  vs  6.1e-6 / 1.2e-5,  1.47
  migt-small (36)                   8.4e-7 / 1.2e-6  vs  6.4e-7 / 7.9e-7,  1.58
  migt-full (156)                   6.7e-7 / 1.2e-6  vs  4.1e-7 / 1.3e-6,  2.26 (ln_f.beta, 5.0e-7 vs 2.2e-7: both near 8u, where
                                                                                 STEP_FLOOR decides)
  Closest to the bar (e_tc / (2 e_cuda + STEP_FLOOR)): 0.54, 0.54, 0.58, 0.75 and 0.93 (migt-full, h.7.attn.c_attn.weight) in the order
  above.  On the transformer the tensor-core median e is about 1.6x the CUDA cores', both at rounding level (e ~ 10u).
  Dropped conv_wgrad_tc row: e 4.5e-2 .. 1.1e-1 on all 31 weight gradients that kernel computes, nothing else flagged; the fixture
  tests' norm-and-projection metric puts 30 of the 31 at or above its 5e-3 bar (2.2e-3 .. 2.3e-1).
  The file runs in about 45 s, the fp64 references on the host's 8 CPU cores included (the full-size cases about 12 s each).
"""
import sys
from collections import Counter, defaultdict

import numpy as np
import pytest
import torch

from oracle import migt_oracle as mo
from oracle import synth
from oracle import vqgan_oracle as vo
from oracle.make_golden import MIGT_TRAIN, vq_images
from test_launch_audit_gpu import FULL_MIGT_TRAIN, MEDIUM_VQ
from viewformer_b200.config import MIGTConfig, VQGANConfig

pytestmark = pytest.mark.gpu

STEP_FLOOR = 1e-7                 # about 2u: tensors whose error is at rounding level on both paths
NORM_FLOOR = 1e-4                 # e's denominator floor: conv biases in front of a one-channel-per-group GroupNorm have a zero gradient


# ----------------------------------------------------------------------------- fp64 references
def vq_grads64(sd, cfg, x, codes, beta=None):
    """Gradient of the codebook loss in fp64 autograd through the oracle, with the quantizer's codes fixed to ``codes``.  ``beta`` None:
    QuantizeEMA (the codebook takes no gradient); a number: Quantize, mean((sg(q) - z)^2) + beta mean((q - sg(z))^2) with the
    straight-through estimator (utils_th.py:113-114), which also gives the codebook its gradient."""
    leaves = {k: v.double().clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    h = vo._conv(leaves, "quant_conv", vo.encoder(leaves, cfg, x.double()))
    emb = leaves["quantize.embeddings"]
    if beta is None:
        q = vo.embed_code(emb.detach(), codes)
        diff = (q - h).pow(2).mean()
    else:
        q = vo.embed_code(emb, codes)
        diff = (q.detach() - h).pow(2).mean() + beta * (q - h.detach()).pow(2).mean()
    dec = vo.decode(leaves, cfg, h + (q - h).detach())
    vo.compute_loss(cfg, diff, x.double(), dec).backward()
    return {k: v.grad for k, v in leaves.items() if v.grad is not None}


def migt_grads64(sd, cfg, cams, codes, loc_weight):
    """Gradient of the transformer's training loss (the batch mean of ``forward(..., compute_losses=True)["loss"]``) in fp64 autograd."""
    leaves = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    o = mo.forward(leaves, cfg, dict(input_ids=codes, poses=cams.double()), compute_losses=True, localization_weight=loc_weight)
    assert o["loss"].dtype == torch.float64
    o["loss"].mean().backward()
    return {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaves.items()}


def step_errors(grads, ref):
    return {k: float((grads[k].double() - ref[k]).norm()) / max(float(ref[k].norm()), NORM_FLOOR) for k in grads}


def faithful_report(tag, errs):
    """Prints median / worst e of both trainers and the largest ratios; returns the tensors over the bar e_tc <= 2 e_cuda + STEP_FLOOR."""
    tc, cc = errs["1"], errs["0"]
    print(f"[{tag}] {len(tc)} tensors, e median / worst: tensor cores {np.median(list(tc.values())):.2e} / {max(tc.values()):.2e}, "
          f"CUDA cores {np.median(list(cc.values())):.2e} / {max(cc.values()):.2e}")
    ratio = sorted((tc[k] / max(cc[k], 1e-12), k) for k in tc)
    print(f"[{tag}] largest e ratios tensor/CUDA cores: " + ", ".join(f"{k} {r:.2f} ({tc[k]:.1e} vs {cc[k]:.1e})" for r, k in ratio[-5:]))
    m, k = max((tc[k] / (2 * cc[k] + STEP_FLOOR), k) for k in tc)
    print(f"[{tag}] closest to the bar: {k} at {m:.2f} of 2 e_cuda + STEP_FLOOR")
    return sorted(k for k in tc if tc[k] > 2 * cc[k] + STEP_FLOOR)


# ----------------------------------------------------------------------------- route counting
TC_ROUTES = ("tc_conv", "conv_wgrad_tc", "tc_gemm", "dense_wgrad_tc", "split_f16x2")


class Routes:
    """Counts the calls of the ``_lib`` entry points a step is expected to reach, per (entry point, dtype of the first operand, where):
    where is "forward" / "data gradient" for tc_conv (the trainer method that called it) and "upsampled" / "plain" for conv_wgrad_tc
    (whether its input is the x2 map the trainer's GroupNorm pass just materialised).  Records the operand channel counts as well."""

    NAMES = TC_ROUTES + ("conv3x3_small_cout", "sumpool2x2", "simt_conv_dgrad_s2", "groupnorm")

    def __init__(self, L, monkeypatch):
        self.count, self.chans, self._up = Counter(), defaultdict(set), None
        for name in self.NAMES:
            monkeypatch.setattr(L, name, self._wrap(name, getattr(L, name)))

    def _wrap(self, name, fn):
        def call(*a, **k):
            if name == "groupnorm":
                out = fn(*a, **k)
                if k.get("upsample") and k.get("out_dtype") == torch.float32:
                    self._up = out
                return out
            dtype, where = str(a[0].dtype).replace("torch.", ""), ""
            if name == "tc_conv":
                caller = sys._getframe(1).f_code.co_name
                where = {"_conv_fw": "forward", "_conv_bw": "data gradient"}.get(caller, caller)
                self.chans[name, where].add(a[0].shape[-1] // (2 if a[0].dtype == torch.float16 else 1))
            elif name == "conv_wgrad_tc":
                where = "upsampled" if a[0] is self._up else "plain"
                self.chans[name, where].add(a[0].shape[-1])
            self.count[name, dtype, where] += 1
            return fn(*a, **k)
        return call

    def table(self):
        return ", ".join(f"{n}/{d}{'/' + w if w else ''} x{c}" + (f" ch {sorted(self.chans[n, w])}" if (n, w) in self.chans else "")
                         for (n, d, w), c in sorted(self.count.items()) if n != "groupnorm")

    def tc_calls(self):
        return sum(c for (n, _, _), c in self.count.items() if n in TC_ROUTES)


# ----------------------------------------------------------------------------- cases
VQ_ROUTES = [("tc_conv", "float16", "forward"), ("tc_conv", "float16", "data gradient"), ("conv_wgrad_tc", "float32", "plain"),
             ("conv_wgrad_tc", "float32", "upsampled"), ("conv3x3_small_cout", "float32", ""), ("sumpool2x2", "float32", ""),
             ("simt_conv_dgrad_s2", "float32", "")]
MIGT_ROUTES = [("dense_wgrad_tc", "float32", ""), ("tc_gemm", "float16", "")]

# case -> (kind, config overrides, batch, quantizer or (T, state-dict seed), input seed, channel counts the split convs must reach)
CASES = {
    "vq-medium-ema": ("vq", MEDIUM_VQ, 4, "ema", 2100, {128, 256}),
    "vq-medium-commit": ("vq", MEDIUM_VQ, 4, "commit", 2100, {128, 256}),
    "vq-full-ema": ("vq", dict(perceptual_weight=0.0), 2, "ema", 3000, {128, 256, 512}),
    "migt-small": ("migt", MIGT_TRAIN, 2, (4, 9), 50, None),
    "migt-full": ("migt", FULL_MIGT_TRAIN, 1, (5, 13), 70, None),
}
_REFS = {}                        # (case, codes) -> fp64 gradients: one reference serves both trainers


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def _vq_inputs(case):
    _, kw, n, quantizer, seed, _ = CASES[case]
    cfg = VQGANConfig(**kw)
    sd = synth.make_vqgan_state_dict(cfg, 5)
    if quantizer == "commit":                   # Quantize has no EMA buffers
        sd = {k: v for k, v in sd.items() if not k.startswith("quantize.") or k == "quantize.embeddings"}
    return cfg, sd, vq_images(n, cfg.image_size, seed)


def run_step(L, monkeypatch, case, tc):
    """One forward_backward of the case's fp32 trainer with VF_TRAIN_TC = ``tc`` -> (per-tensor e against fp64, Routes, gradients, fp64
    gradients)."""
    from viewformer_b200 import MIGT, VQGAN
    from viewformer_b200.train import VQGANTrainer
    from viewformer_b200.train_migt import MIGTTrainer
    kind, kw, n, extra, seed, _ = CASES[case]
    monkeypatch.setenv("VF_TRAIN_TC", tc)
    with monkeypatch.context() as mp:
        routes = Routes(L, mp)
        if kind == "vq":
            cfg, sd, x = _vq_inputs(case)
            tr = VQGANTrainer(VQGAN(cfg, precision="fp32", quantizer=extra).load_state_dict({k: v.clone() for k, v in sd.items()}))
            tr.forward_backward(x)
            torch.cuda.synchronize()
            grads, codes = tr.export_gradients(), tr.last["codes"].cpu().long()
            beta = tr.model.beta if extra == "commit" else None
            make_ref = lambda: vq_grads64(sd, cfg, x, codes, beta)
        else:
            T, sd_seed = extra
            cfg = MIGTConfig(**kw)
            sd = synth.make_migt_state_dict(cfg, sd_seed)
            codes = synth.make_codes(n, T, n_embed=cfg.n_embeddings, seed=seed)
            cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(n, T, seed=seed + 1))[0])
            tr = MIGTTrainer(MIGT(cfg, precision="fp32").load_state_dict({k: v.clone() for k, v in sd.items()}))
            tr.forward_backward(cams, codes)
            torch.cuda.synchronize()
            grads, lw = tr.gradients(), tr.loc_weight
            make_ref = lambda: migt_grads64(sd, cfg, cams, codes, lw)
    assert tr.use_tc == (tc == "1")
    key = (case, codes.numpy().tobytes())
    if key not in _REFS:
        _REFS[key] = make_ref()
    del tr
    torch.cuda.empty_cache()
    return step_errors(grads, _REFS[key]), routes, grads, _REFS[key]


@pytest.mark.parametrize("case", list(CASES))
def test_faithful_step_vs_fp64(L, monkeypatch, case):
    """Every gradient of one fp32 step within twice the CUDA-core trainer's fp64 error (plus STEP_FLOOR), with the tensor-core routes
    reached by the shipped trainer and by the VF_TRAIN_TC=0 one not at all."""
    kind, chans = CASES[case][0], CASES[case][5]
    errs, routes = {}, {}
    for tc in ("1", "0"):
        errs[tc], routes[tc], _, _ = run_step(L, monkeypatch, case, tc)
        print(f"[{case}] routes, VF_TRAIN_TC={tc}: {routes[tc].table()}")
    bad = faithful_report(case, errs)
    want = VQ_ROUTES if kind == "vq" else MIGT_ROUTES
    missing = [r for r in want if routes["1"].count[r] == 0]
    assert not missing, f"{case}: the tensor-core step never reached {missing}"
    if chans:
        for key in (("tc_conv", "forward"), ("tc_conv", "data gradient"), ("conv_wgrad_tc", "plain")):
            assert chans <= routes["1"].chans[key], f"{case}: {key} ran at channels {sorted(routes['1'].chans[key])}, not all of {sorted(chans)}"
    assert routes["0"].tc_calls() == 0, f"{case}: VF_TRAIN_TC=0 reached a tensor-core route: {routes['0'].table()}"
    assert not bad, f"{case}: tensor-core gradients less accurate than 2x the CUDA-core trainer's: " + ", ".join(
        f"{k} {errs['1'][k]:.2e} vs {errs['0'][k]:.2e}" for k in bad[:8])


def test_faithful_bar_flags_dropped_wgrad_row(L, monkeypatch):
    """Sensitivity of the bar (medium codebook): conv_wgrad_tc run on its input with the last pixel row zeroed, a dropped border row.  The
    comparison must flag exactly the weight gradients that conv_wgrad_tc computes (3x3 stride-1 convs with both channel counts multiples
    of 128) and nothing else, and nothing at all without the fault.  Prints what the norm-and-projection metric of the fp32 fixture tests
    (5e-3 relative) makes of the same fault."""
    case = "vq-medium-ema"
    cuda_errs, _, _, _ = run_step(L, monkeypatch, case, "0")
    clean_errs, _, _, _ = run_step(L, monkeypatch, case, "1")
    orig = L.conv_wgrad_tc

    def dropped_row(x, dy, dw, **k):
        x = x.clone()
        x[:, -1] = 0.0
        return orig(x, dy, dw, **k)

    with monkeypatch.context() as mp:
        mp.setattr(L, "conv_wgrad_tc", dropped_row)
        tc_errs, routes, grads, ref = run_step(L, monkeypatch, case, "1")
    assert routes.count["conv_wgrad_tc", "float32", "upsampled"] > 0
    assert not faithful_report(f"{case} unperturbed", {"1": clean_errs, "0": cuda_errs})
    bad = faithful_report(f"{case} dropped wgrad row", {"1": tc_errs, "0": cuda_errs})
    shapes = {k: tuple(g.shape) for k, g in grads.items()}
    hit = sorted(k for k, s in shapes.items() if len(s) == 4 and s[2:] == (3, 3) and s[0] % 128 == 0 and s[1] % 128 == 0
                 and ".downsample." not in k)                                  # stride-2 weight gradients stay on the CUDA cores
    # the norm-and-projection metric of the fp32 fixture tests on the same gradients: max(| |g| - |g64| |, |<g, p> - <g64, p>|) /
    # max(|g64|, 1e-4), p a seeded random probe
    gen = torch.Generator().manual_seed(99)
    old = {}
    for k in sorted(grads):
        p = torch.randn(shapes[k], generator=gen, dtype=torch.float64)
        g, g64 = grads[k].double(), ref[k]
        old[k] = max(abs(float(g.norm() - g64.norm())), abs(float((g * p).sum() - (g64 * p).sum()))) / max(float(g64.norm()), NORM_FLOOR)
    caught = [k for k in hit if old[k] >= 5e-3]
    print(f"[{case} dropped wgrad row] flagged {len(bad)} tensors; conv_wgrad_tc computes {len(hit)}: e {min(tc_errs[k] for k in hit):.2e} .. "
          f"{max(tc_errs[k] for k in hit):.2e}; norm/projection metric {min(old[k] for k in hit):.2e} .. {max(old[k] for k in hit):.2e}, "
          f"{len(caught)} of {len(hit)} at or above 5e-3")
    assert hit and bad == hit, f"flagged {bad}, expected {hit}"
