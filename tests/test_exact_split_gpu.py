"""The split-fp16 ("exact", VF_F16X2) tensor-core path against fp64, across operand magnitudes, dispatch options and tile edges.

An fp32 value v travels as hi = fp16(v), lo = fp16((v - hi) * 2^11); three fp16 MMA passes and chunked round-to-nearest accumulation give
fp32-faithful products, but only inside a range of magnitudes: below 2^-14 hi is an fp16 subnormal (lo's absolute floor is 2^-36), and at
|v| >= 65520 hi is inf and the product NaN.

* Producers (vf_split_f16x2, vf_groupnorm_apply with F16X2 output, vf_pad_transpose_split): bit for bit against a CPU restatement, on
  subnormal-range values and their boundaries, +-0, 65504 / 65519 / 65520 and ragged shapes.
* Accuracy bar, the same in every accuracy test: e = |got - ref64| / (sum |a||b| + |bias| + |residual|) per element; e_fp32 is the same for
  the project's CUDA-core kernel on the same fp32 inputs (vf_simt_gemm, vf_conv_wgrad).  Faithful: max e <= max(2 max e_fp32, 4u) and
  rms e <= 1.5 rms e_fp32; every result also passes the worst-case gate e <= 2 K u.
* Magnitude sweep of the exact GEMM, conv, conv_wgrad_tc and dense_wgrad_tc at operand amax 2^e: faithful for e in -10 .. 15, the ratio
  printed (not asserted) below that.
* Exact GEMM and conv dispatch options and tile edges against fp64; the weight-gradient GEMMs on gradient-like operands.
* The operand window of real training steps and of the mixed-precision encoder: every split operand's amax lies in [2^-10, 2^15].
* One codebook step's gradients against fp64 autograd, tensor cores against the CUDA-core trainer, and the gradient-seed scale that keeps
  the trainers inside the window: on the CUDA cores it changes the gradients no more than a rerun does.
"""
import math
import os
import sys
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

from oracle import migt_oracle as mo
from oracle import synth
from oracle.make_golden import MIGT_TRAIN, SMALL_VQ, vq_images
from test_faithful_steps_gpu import faithful_report, step_errors, vq_grads64
from viewformer_b200.config import MIGTConfig, VQGANConfig

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
WINDOW = (2.0 ** -10, 2.0 ** 15)


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def gen(seed):
    return torch.Generator().manual_seed(seed)


def split_ref(v):
    """CPU restatement of the VF_F16X2 pair of an fp32 tensor: hi = fp16(v), lo = fp16((v - hi) * 2^11)."""
    hi = v.half()
    lo = ((v - hi.float()) * 2048.0).half()
    return hi, lo


def bits(t):
    return t.contiguous().view(torch.int16).cpu()


def special_values(n, seed):
    """fp32 values at the edges of the split: fp16 subnormals and their boundaries, values whose lo is subnormal, +-0, the top of the fp16
    range (65504 finite, 65519 still rounds to 65504, 65520 rounds to inf), then log-uniform magnitudes 2^-40 .. 2^17 of both signs."""
    edges = [0.0, 2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -24, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -24, 2.0 ** -14 * (1 - 2.0 ** -11),
             2.0 ** -14 * (1 + 2.0 ** -10), 2.0 ** -15 + 2.0 ** -30, 3 * 2.0 ** -26, 2.0 ** -36, 2.0 ** -40, 1e-6, 1.0 + 2.0 ** -23,
             2048.0 + 1.0, 65504.0, 65519.0, 65519.996, 65520.0, 7e4, 1.0e5]
    v = torch.tensor(edges + [-e for e in edges], dtype=torch.float32)
    assert torch.signbit(v[len(edges)])                                     # -0.0
    gg = gen(seed)
    rnd = torch.sign(torch.randn(n, generator=gg)) * torch.exp2(torch.rand(n, generator=gg) * 57 - 40)
    out = torch.cat([v, rnd.float()])[:n] if n >= v.numel() else v[:n]
    return out[torch.randperm(out.numel(), generator=gg)] if n > v.numel() else out


# ----------------------------------------------------------------------------- producers, bit for bit
@pytest.mark.parametrize("rows,c", [(1003, 4), (77, 12), (5, 128)])
def test_split_f16x2_bits(L, rows, c):
    x = special_values(rows * c, rows + c).reshape(rows, c)
    hi, lo = split_ref(x)
    got = L.split_f16x2(x.cuda())
    torch.cuda.synchronize()
    assert got.shape == (rows, 2 * c)
    assert torch.equal(bits(got[:, :c]), bits(hi)) and torch.equal(bits(got[:, c:]), bits(lo))
    assert torch.isinf(hi[x.abs() >= 65520]).all() and torch.isfinite(hi[x.abs() < 65520]).all()


@pytest.mark.parametrize("layout", ["plain", "upsample", "s2d"])
@pytest.mark.parametrize("n,h,w,c", [(3, 5, 7, 4), (2, 6, 10, 4), (1, 4, 6, 64)])
def test_groupnorm_apply_split_bits(L, layout, n, h, w, c):
    if layout == "s2d" and (h % 2 or w % 2):
        pytest.skip("space-to-depth needs even maps")
    x = special_values(n * h * w * c, 7 * h + w).reshape(n, h, w, c)
    kw = dict(upsample=layout == "upsample", s2d=layout == "s2d")
    got = L.groupnorm(x.cuda(), None, None, swish=False, out_dtype=torch.float16, normalize=False, **kw).cpu()
    hi, lo = split_ref(x)

    def lay(t):
        if layout == "upsample":
            return t.repeat_interleave(2, 1).repeat_interleave(2, 2)
        if layout == "s2d":
            return t.reshape(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, h // 2, w // 2, 4 * c)
        return t

    lc = got.shape[-1] // 2
    assert torch.equal(bits(got[..., :lc]), bits(lay(hi))) and torch.equal(bits(got[..., lc:]), bits(lay(lo)))
    if c % 32 == 0:                                                          # the normalising variant: the fp32 kernel's values, split
        xs = torch.randn(n, h, w, c, generator=gen(c)) * 3e-4
        ga, be = (1 + 0.1 * torch.randn(c, generator=gen(1))).cuda(), (0.1 * torch.randn(c, generator=gen(2))).cuda()
        f = L.groupnorm(xs.cuda(), ga, be, swish=True, out_dtype=torch.float32, **kw).cpu()
        s = L.groupnorm(xs.cuda(), ga, be, swish=True, out_dtype=torch.float16, **kw).cpu()
        fh, fl = split_ref(f)
        assert torch.equal(bits(s[..., :lc]), bits(fh)) and torch.equal(bits(s[..., lc:]), bits(fl))


def pad_transpose_ref(x, pitch, copies, margin, lrow, fill):
    n, h, w, c = x.shape
    hi, lo = split_ref(x)
    out = torch.full((copies * c, 2, lrow), fill, dtype=torch.float16)
    if pitch:
        q = ((torch.arange(n)[:, None, None] * (h + 2) + torch.arange(h)[None, :, None] + 1) * pitch + torch.arange(w)[None, None, :] + 1).reshape(-1)
    else:
        q = torch.arange(n * h * w)
    for k in range(copies):
        col = margin + q - (k - copies // 2)
        out[k * c:(k + 1) * c, 0, col] = hi.reshape(-1, c).t()
        out[k * c:(k + 1) * c, 1, col] = lo.reshape(-1, c).t()
    return out


@pytest.mark.parametrize("n,h,w,c,mode", [(2, 3, 5, 4, "pad"), (1, 1, 9, 40, "pad"), (3, 4, 13, 36, "pad"), (1, 1, 77, 36, "plain"),
                                          (1, 1, 130, 4, "plain")])
def test_pad_transpose_split_bits(L, n, h, w, c, mode):
    """Interior positions bit for bit; the borders, pitch padding, margins and the row tail are never written (they keep a sentinel)."""
    x = special_values(n * h * w * c, n + h + w + c).reshape(n, h, w, c)
    if mode == "pad":
        pitch, copies = (w + 2 + 7) // 8 * 8, 3
        margin = pitch + 8
        lrow = (n * (h + 2) * pitch + 2 * margin + 8 + 7) // 8 * 8
    else:
        pitch, copies, margin = 0, 1, 0
        lrow = (n * h * w + 63) // 64 * 64 + 64
    fill = 1234.0
    out = torch.full((copies * c, 2, lrow), fill, dtype=torch.float16, device="cuda")
    lib = L.load(True)
    L._check(lib.vf_pad_transpose_split(x.cuda(), n, h, w, c, pitch, copies, margin, lrow, out, L._stream()))
    torch.cuda.synchronize()
    want = pad_transpose_ref(x, pitch, copies, margin, lrow, fill)
    assert torch.equal(bits(out), bits(want))


# ----------------------------------------------------------------------------- the accuracy bar
def bar_errors(got, ref, denom):
    return ((got.double().cpu() - ref).abs() / denom.clamp_min(1e-300)).reshape(-1)


def check_faithful(name, got, got32, ref, denom, K, strict=True):
    """The bar of the module docstring.  Returns (max e / max e_fp32, rms e / rms e_fp32)."""
    assert torch.isfinite(got).all(), f"{name}: non-finite output (or an element never written)"
    e, e32 = bar_errors(got, ref, denom), bar_errors(got32, ref, denom)
    mx, mx32 = float(e.max()), float(e32.max())
    rms, rms32 = float(e.pow(2).mean().sqrt()), float(e32.pow(2).mean().sqrt())
    rmax, rrms = mx / max(mx32, 1e-300), rms / max(rms32, 1e-300)
    print(f"[{name}] split-fp16: max e {mx:.2e} rms {rms:.2e} | fp32 CUDA cores: max {mx32:.2e} rms {rms32:.2e} | ratio max {rmax:.2f} rms {rrms:.2f}"
          f" | gate 2Ku = {2 * K * U:.1e}")
    if strict:
        assert mx <= max(2 * mx32, 4 * U), f"{name}: max e {mx:.3e} > max(2 x {mx32:.3e}, 4u)"
        assert rms <= 1.5 * rms32, f"{name}: rms e {rms:.3e} > 1.5 x {rms32:.3e}"
        assert mx <= 2 * K * U, f"{name}: max e {mx:.3e} above the worst-case gate 2 K u = {2 * K * U:.3e}"
    return rmax, rrms


def gelu64(v):
    return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))


# ----------------------------------------------------------------------------- exact GEMM
def run_gemm(L, A, B, *, M, N, K, batch=1, a_shared=False, b_shared=False, alpha=1.0, bias=None, bias_mode=None, act=None, residual=None,
             gn_rows_per_img=0):
    """C[b] = act(alpha A[b] B[b]^T + bias) + residual on the exact tensor-core GEMM and on vf_simt_gemm; A [.., M, K], B [.., N, K] fp32."""
    bm = bias_mode if bias is not None else L.BIAS_NONE
    act = L.ACT_NONE if act is None else act
    As, Bs = L.split_f16x2(A.reshape(-1, K).cuda()), L.split_f16x2(B.reshape(-1, K).cuda())
    out = torch.full((batch, M, N), float("nan"), device="cuda")
    kw = dict(M=M, N=N, K=K, ldc=N, batch=(batch, 1), c_bs=(M * N, 0), alpha=alpha, bias=None if bias is None else bias.cuda(), bias_mode=bm,
              act=act, residual=None if residual is None else residual.cuda())
    L.tc_gemm(As, Bs, out, lda=2 * K, ldb=2 * K, a_bs=(0 if a_shared else M * 2 * K, 0), b_bs=(0 if b_shared else N * 2 * K, 0), lo_a=K, lo_b=K,
              gn_rows_per_img=gn_rows_per_img, **kw)
    out32 = torch.full((batch, M, N), float("nan"), device="cuda")
    L.simt_gemm(A.cuda(), B.cuda(), out32, a_strides=(K, 1), b_strides=(1, K), a_bs=(0 if a_shared else M * K, 0), b_bs=(0 if b_shared else N * K, 0), **kw)
    torch.cuda.synchronize()
    Ad, Bd = A.double().reshape(-1, M, K), B.double().reshape(-1, N, K)
    prod = alpha * torch.matmul(Ad, Bd.transpose(1, 2))
    den = alpha * torch.matmul(Ad.abs(), Bd.abs().transpose(1, 2))
    if bias is not None:
        bb = bias.double()[None, None, :] if bm == L.BIAS_N else bias.double()[None, :, None]
        prod, den = prod + bb, den + bb.abs()
    if act == L.ACT_GELU:
        prod = gelu64(prod)
    if residual is not None:
        prod, den = prod + residual.double().reshape(prod.shape), den + residual.double().abs().reshape(prod.shape)
    return out, out32, prod.expand(batch, M, N), den.expand(batch, M, N)


# K / 64 in {1, 2, 3, 5, 6, 8} takes every accumulation chunk length (4, 3, 2, 1); 48 is a long K where unchunked accumulation shows
GEMM_CASES = {
    "kb1": dict(M=200, N=128, kb=1), "kb2": dict(M=200, N=128, kb=2), "kb3": dict(M=200, N=128, kb=3), "kb5": dict(M=200, N=128, kb=5),
    "kb6": dict(M=200, N=128, kb=6), "kb8": dict(M=200, N=128, kb=8), "kb48": dict(M=130, N=128, kb=48),
    "n64": dict(M=200, N=64, kb=2), "n72_biasM": dict(M=200, N=72, kb=3, bias="M"), "n192_biasN_gelu_res": dict(M=200, N=192, kb=5, bias="N", gelu=True, res=True),
    "alpha_res": dict(M=256, N=256, kb=2, alpha=128 ** -0.5, res=True),
    "shared_A_batch_biasM": dict(M=128, N=192, kb=2, batch=3, a_shared=True, bias="M"),
    "shared_B_batch": dict(M=200, N=128, kb=3, batch=2, b_shared=True),
}


@pytest.mark.parametrize("case", list(GEMM_CASES))
def test_exact_gemm_vs_fp64(L, case):
    c = GEMM_CASES[case]
    M, N, K, nb = c["M"], c["N"], 64 * c["kb"], c.get("batch", 1)
    gg = gen(M + N + K + nb)
    A = torch.randn(1 if c.get("a_shared") else nb, M, K, generator=gg)
    B = torch.randn(1 if c.get("b_shared") else nb, N, K, generator=gg) / math.sqrt(K)
    bias = residual = None
    bm = None
    if "bias" in c:
        bm = L.BIAS_N if c["bias"] == "N" else L.BIAS_M
        bias = torch.randn(N if c["bias"] == "N" else M, generator=gg)
    if c.get("res"):
        residual = torch.randn(nb, M, N, generator=gg)
    got, got32, ref, den = run_gemm(L, A, B, M=M, N=N, K=K, batch=nb, a_shared=c.get("a_shared", False), b_shared=c.get("b_shared", False),
                                    alpha=c.get("alpha", 1.0), bias=bias, bias_mode=bm, act=L.ACT_GELU if c.get("gelu") else None, residual=residual)
    check_faithful(f"exact gemm {case} M{M} N{N} K{K}", got, got32, ref, den, K)


def test_exact_gemm_groupnorm_sums(L):
    """gn_rows_per_img (the attention proj of the exact encoder): the fused per-(image, group) sums of the output and of its squares, against
    fp64 sums of the stored output, within 8 u of the sums of magnitudes."""
    M, N, K, rpi = 256, 128, 128, 64
    gg = gen(5)
    A, B = torch.randn(1, M, K, generator=gg), torch.randn(1, N, K, generator=gg) / math.sqrt(K)
    res = torch.randn(1, M, N, generator=gg) + 0.5
    got, got32, ref, den = run_gemm(L, A, B, M=M, N=N, K=K, residual=res, gn_rows_per_img=rpi)
    check_faithful("exact gemm + gn sums", got, got32, ref, den, K)
    assert hasattr(got, "_gn_sums") and got._gn_sums[1] == 32
    o = got.double().cpu().reshape(M // rpi, rpi, 32, N // 32)
    want = torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1)
    mag = torch.stack([o.abs().sum((1, 3)), (o * o).sum((1, 3))], -1)
    err = float(((got._gn_sums[0].cpu() - want).abs() / mag).max())
    print(f"[exact gemm gn sums] max |sum - fp64| / sum|.| = {err:.2e}")
    assert err < 8 * U


@pytest.mark.parametrize("n,hw,c", [(2, 64, 128), (2, 200, 128)])
def test_exact_gemm_scores_layout(L, n, hw, c):
    """The exact attention scores of the encoder (vqgan.py _attn_exact): q and k are the two halves of one split [hi(q|k) | lo(q|k)] row
    (lo_a = 2c > K), the key operand starts at b_off = c, alpha = c^-1/2, one batch per image; hw = 64 runs 64-wide N tiles, hw = 200 the
    scalar N tail."""
    qk = torch.randn(n * hw, 2 * c, generator=gen(hw)) * 2
    qks = L.split_f16x2(qk.cuda())
    alpha = float(c ** -0.5)
    S = torch.full((n, hw, hw), float("nan"), device="cuda")
    L.tc_gemm(qks, qks, S, M=hw, N=hw, K=c, lda=4 * c, ldb=4 * c, ldc=hw, batch=(n, 1), a_bs=(hw * 4 * c, 0), b_bs=(hw * 4 * c, 0),
              c_bs=(hw * hw, 0), b_off=c, alpha=alpha, lo_a=2 * c, lo_b=2 * c)
    S32 = torch.full((n, hw, hw), float("nan"), device="cuda")
    L.simt_gemm(qk.cuda(), qk.cuda(), S32, M=hw, N=hw, K=c, a_strides=(2 * c, 1), b_strides=(1, 2 * c), ldc=hw, batch=(n, 1),
                a_bs=(hw * 2 * c, 0), b_bs=(hw * 2 * c, 0), c_bs=(hw * hw, 0), b_off=c, alpha=alpha)
    torch.cuda.synchronize()
    q, k = qk.double().reshape(n, hw, 2 * c)[..., :c], qk.double().reshape(n, hw, 2 * c)[..., c:]
    ref = alpha * q @ k.transpose(1, 2)
    den = alpha * q.abs() @ k.abs().transpose(1, 2)
    check_faithful(f"exact scores n{n} hw{hw} c{c}", S, S32, ref, den, c)


# ----------------------------------------------------------------------------- exact conv
def run_conv(L, x, w, b, r):
    """x [n, cin, H, W], w [cout, cin, 3, 3] fp32 CPU -> (tensor-core exact, CUDA-core fp32, fp64, denominator), all NHWC."""
    n, cin, H, W = x.shape
    cout = w.shape[0]
    xh = x.permute(0, 2, 3, 1).contiguous().cuda()
    rh = r.permute(0, 2, 3, 1).contiguous().cuda() if r is not None else None
    xs = L.split_f16x2(xh.reshape(-1, cin)).reshape(n, H, W, 2 * cin)      # the trainer's operand (any Cin, unlike the GroupNorm pass)
    ws = L.split_f16x2(w.permute(0, 2, 3, 1).reshape(cout * 9, cin).contiguous().cuda()).reshape(cout, 18 * cin)
    out = torch.full((n, H, W, cout), float("nan"), device="cuda")
    got = L.tc_conv(xs, ws, b.cuda(), residual=rh, out=out)
    got32 = L.simt_conv(xh, w.permute(2, 3, 1, 0).reshape(9 * cin, cout).contiguous().cuda(), b.cuda(), kh=3, residual=rh)
    torch.cuda.synchronize()
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    den = F.conv2d(x.double().abs(), w.double().abs(), b.double().abs(), padding=1)
    if r is not None:
        ref, den = ref + r.double(), den + r.double().abs()
    return got, got32, ref.permute(0, 2, 3, 1), den.permute(0, 2, 3, 1)


CONV_CASES = {
    "halo_tw16_cin64": (2, 16, 16, 64, 128, False), "halo_tw8_cin128_ragged": (1, 20, 12, 128, 128, True),
    "tap_cin192": (2, 16, 16, 192, 128, True), "map12_tn2": (3, 12, 12, 128, 128, False), "ragged_19x27": (2, 19, 27, 64, 64, True),
    "cout192_tail": (1, 16, 16, 128, 192, True),
}


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_exact_conv_vs_fp64(L, case):
    n, H, W, cin, cout, res = CONV_CASES[case]
    gg = gen(H * W + cin + cout)
    x = torch.randn(n, cin, H, W, generator=gg) * 1.5
    w = torch.randn(cout, cin, 3, 3, generator=gg) / (9 * cin) ** 0.5
    b = torch.randn(cout, generator=gg)
    r = torch.randn(n, cout, H, W, generator=gg) if res else None
    got, got32, ref, den = run_conv(L, x, w, b, r)
    check_faithful(f"exact conv {case} n{n} {H}x{W} {cin}->{cout}", got, got32, ref, den, 9 * cin)


# ----------------------------------------------------------------------------- weight gradients on the exact GEMM
def grad_like(shape, gg, amax=1.0):
    """A backward-pass tensor: heavy-tailed (normal times log-normal), scaled to the given amax."""
    t = torch.randn(shape, generator=gg) * torch.exp(torch.randn(shape, generator=gg))
    return t * (amax / float(t.abs().max()))


def act_like(shape, gg, amax=None):
    t = torch.randn(shape, generator=gg) * 1.3 + 0.2
    t = t * torch.sigmoid(t)                                                 # swish of a GroupNorm output
    return t if amax is None else t * (amax / float(t.abs().max()))


def run_conv_wgrad(L, x, dy, upsample=False):
    """x [n, H, W, cin] (before the x2 upsample), dy [n, OH, OW, cout] fp32 CPU -> (tensor core, CUDA core, fp64, denominator) [9 cin, cout]."""
    cin, cout = x.shape[-1], dy.shape[-1]
    dw = torch.full((9 * cin, cout), float("nan"), device="cuda")
    if upsample:          # the trainer's form: the x2 upsample materialised, then the stride-1 weight gradient
        a = L.groupnorm(x.cuda(), None, None, swish=False, out_dtype=torch.float32, normalize=False, upsample=True)
    else:
        a = x.cuda()
    L.conv_wgrad_tc(a, dy.cuda(), dw, accumulate=False)
    dw32 = torch.zeros(9 * cin, cout, device="cuda")
    L.conv_wgrad(x.cuda(), dy.cuda(), dw32, kh=3, upsample=upsample)
    torch.cuda.synchronize()
    xd = x.double().permute(0, 3, 1, 2)
    if upsample:
        xd = F.interpolate(xd, scale_factor=2.0, mode="nearest")
    dyd = dy.double().permute(0, 3, 1, 2)

    def wg(a_, d_):
        return torch.nn.grad.conv2d_weight(a_, (cout, cin, 3, 3), d_, padding=1).permute(2, 3, 1, 0).reshape(9 * cin, cout)

    return dw, dw32, wg(xd, dyd), wg(xd.abs(), dyd.abs())


def run_dense_wgrad(L, x, dy):
    m, k = x.shape
    n = dy.shape[1]
    dw = torch.full((k, n), float("nan"), device="cuda")
    L.dense_wgrad_tc(x.cuda(), dy.cuda(), dw, accumulate=False)
    dw32 = torch.zeros(k, n, device="cuda")
    L.conv_wgrad(x.cuda().reshape(1, m, 1, k), dy.cuda().reshape(1, m, 1, n), dw32, kh=1, pad=(0, 0), so=(n, 1))
    torch.cuda.synchronize()
    return dw, dw32, x.double().t() @ dy.double(), x.double().abs().t() @ dy.double().abs()


@pytest.mark.parametrize("n,h,w,cin,cout,up", [(2, 10, 13, 128, 128, False), (3, 1, 20, 128, 256, False), (2, 7, 9, 128, 128, True),
                                               (1, 16, 16, 256, 128, True)])
def test_conv_wgrad_tc_vs_fp64(L, n, h, w, cin, cout, up):
    """W % 8 != 0 (pitch padding), H = 1, and the upsample conv's form (the x2 map materialised, train.py _conv_bw)."""
    gg = gen(n * h * w + cin)
    x = act_like((n, h, w, cin), gg)
    dy = grad_like((n, 2 * h if up else h, 2 * w if up else w, cout), gg)
    got, got32, ref, den = run_conv_wgrad(L, x, dy, upsample=up)
    check_faithful(f"conv_wgrad_tc n{n} {h}x{w}{' x2' if up else ''} {cin}->{cout}", got, got32, ref, den, n * h * w * (4 if up else 1))


@pytest.mark.parametrize("m,k,n", [(333, 128, 128), (1000, 256, 128), (63, 128, 384), (4100, 128, 256)])
def test_dense_wgrad_tc_vs_fp64(L, m, k, n):
    """Row counts that are not a multiple of 64 (the zero tail of the last split)."""
    gg = gen(m + k + n)
    got, got32, ref, den = run_dense_wgrad(L, act_like((m, k), gg), grad_like((m, n), gg))
    check_faithful(f"dense_wgrad_tc m{m} {k}x{n}", got, got32, ref, den, m)


# ----------------------------------------------------------------------------- magnitude sweep
SWEEP_E = [15, 8, 0, -4, -10, -16, -20, -24]


@pytest.mark.parametrize("op", ["gemm", "conv", "conv_wgrad", "dense_wgrad"])
def test_magnitude_sweep(L, op):
    """Operand amax = 2^e for both operands: faithful for e >= -10, the error ratio against the CUDA-core kernel printed below that."""
    rows = []
    for e in SWEEP_E:
        amax = 2.0 ** e
        gg = gen(100 + e)
        strict = e >= -10
        name = f"sweep {op} amax 2^{e}"
        if op == "gemm":
            M, N, K = 256, 128, 512
            A, B = grad_like((1, M, K), gg, amax), act_like((1, N, K), gg, amax)
            got, got32, ref, den = run_gemm(L, A, B, M=M, N=N, K=K)
        elif op == "conv":
            K = 9 * 128
            x = grad_like((2, 128, 16, 16), gg, amax)
            w = act_like((128, 128, 3, 3), gg, amax)
            got, got32, ref, den = run_conv(L, x, w, torch.zeros(128), None)
        elif op == "conv_wgrad":
            K = 2 * 16 * 16
            got, got32, ref, den = run_conv_wgrad(L, act_like((2, 16, 16, 128), gg, amax), grad_like((2, 16, 16, 128), gg, amax))
        else:
            K = 1000
            got, got32, ref, den = run_dense_wgrad(L, act_like((1000, 128), gg, amax), grad_like((1000, 256), gg, amax))
        rows.append((e, *check_faithful(name, got, got32, ref, den, K, strict=strict)))
    print(f"[sweep {op}] error ratio split-fp16 / fp32 CUDA cores, (max, rms) per amax exponent: "
          + ", ".join(f"2^{e}: ({a:.2f}, {r:.2f})" for e, a, r in rows))


# ----------------------------------------------------------------------------- the operand window of real steps
class OperandWindow:
    """Wraps the entry points that take split-fp16 operands and records each operand's amax per call site (caller file:line function)."""

    def __init__(self, L, monkeypatch):
        self.rec = defaultdict(list)
        self.L = L
        for name in ("split_f16x2", "conv_wgrad_tc", "dense_wgrad_tc", "tc_conv"):
            monkeypatch.setattr(L, name, self._wrap(name, getattr(L, name)))

    def _site(self):
        f = sys._getframe(2)
        return f"{os.path.basename(f.f_code.co_filename)}:{f.f_lineno} {f.f_code.co_name}"

    def _put(self, site, what, t):
        self.rec[(site, what)].append(t.detach().abs().amax().float())

    def _wrap(self, name, fn):
        def call(*a, **k):
            site = self._site()
            if name == "split_f16x2":
                self._put(site, "split x", a[0])
            elif name in ("conv_wgrad_tc", "dense_wgrad_tc"):
                self._put(site, f"{name} x", a[0])
                self._put(site, f"{name} dy", a[1])
            elif a[0].dtype == torch.float16:                             # tc_conv on split operands: the hi halves
                x, wt = a[0], a[1]
                cin = k.get("cin") or x.shape[-1] // 2
                self._put(site, "tc_conv x(hi)", x[..., :x.shape[-1] // 2])
                self._put(site, "tc_conv w(hi)", wt.reshape(wt.shape[0], -1, 2, cin)[:, :, 0])
            return fn(*a, **k)
        return call

    def table(self):
        out = []
        for (site, what), v in sorted(self.rec.items()):
            t = torch.stack(v).cpu().double()
            nz = t[t > 0]
            out.append((site, what, len(v), float(nz.min()) if nz.numel() else 0.0, float(t.max()), int((t == 0).sum())))
        return out


def _vqgan_run(cfg, images, seed):
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    model = VQGAN(cfg, precision="fp32").load_state_dict(synth.make_vqgan_state_dict(cfg, 5))
    tr = VQGANTrainer(model)
    tr.forward_backward(vq_images(images, cfg.image_size, seed))
    return tr


def _migt_run(cfg, B, T, seed):
    from viewformer_b200 import MIGT
    from viewformer_b200.train_migt import MIGTTrainer
    model = MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9))
    tr = MIGTTrainer(model)
    codes = synth.make_codes(B, T, n_embed=cfg.n_embeddings, seed=seed)
    cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=seed + 1))[0])
    tr.forward_backward(cams, codes)
    return tr


def _encoder_run():
    from viewformer_b200 import VQGAN
    cfg = VQGANConfig()
    model = VQGAN(cfg, precision="mixed").load_state_dict(synth.make_vqgan_state_dict(cfg, 5))
    model.encode(vq_images(4, cfg.image_size, 17))
    return model


WINDOW_RUNS = {
    "vqgan-small": lambda: _vqgan_run(VQGANConfig(**dict(SMALL_VQ, perceptual_weight=0.0)), 3, 2000),
    "vqgan-full": lambda: _vqgan_run(VQGANConfig(perceptual_weight=0.0), 2, 3000),
    "vqgan-full-32": lambda: _vqgan_run(VQGANConfig(perceptual_weight=0.0), 32, 3001),
    "migt-small": lambda: _migt_run(MIGTConfig(**MIGT_TRAIN), 2, 4, 50),
    "migt-full": lambda: _migt_run(MIGTConfig(dropout=0.0, label_smoothing=0.1, localization_weight="0.7", total_steps=100, learning_rate=1e-4), 1, 5, 70),
    "mixed-encoder": _encoder_run,
}


@pytest.mark.parametrize("run", list(WINDOW_RUNS))
def test_split_operand_window(L, monkeypatch, run):
    """Every split-fp16 operand of one fp32 training step (codebook: small config, full size with 2 and 32 images; transformer: small and
    full size) and of one full-size mixed-precision encoder forward has amax in [2^-10, 2^15] (all-zero operands are exact and pass).
    Prints the per-call-site table; for the encoder its last column is the margin below 65520 that nobody measured before."""
    win = OperandWindow(L, monkeypatch)
    obj = WINDOW_RUNS[run]()
    torch.cuda.synchronize()
    tab = win.table()
    assert tab, "no split-fp16 operand was recorded"
    print(f"\n[operand window {run}] {'site':<42} {'operand':<22} {'calls':>5} {'min amax':>10} {'max amax':>10} zero")
    bad = []
    for site, what, n, lo, hi, zero in tab:
        flag = "" if (lo == 0.0 or lo >= WINDOW[0]) and hi <= WINDOW[1] else "  <-- outside"
        print(f"[operand window {run}] {site:<42} {what:<22} {n:>5} {lo:>10.3e} {hi:>10.3e} {zero:>4}{flag}")
        if flag or not math.isfinite(hi):
            bad.append(f"{site} {what}: amax {lo:.3e} .. {hi:.3e}")
    hi_all = max(t[4] for t in tab)
    lo_all = min((t[3] for t in tab if t[3] > 0), default=0.0)
    print(f"[operand window {run}] overall amax {lo_all:.3e} .. {hi_all:.3e}: {math.log2(lo_all / WINDOW[0]):+.1f} octaves above 2^-10, "
          f"{math.log2(65520.0 / hi_all):.1f} octaves below 65520")
    del obj
    torch.cuda.empty_cache()
    assert not bad, "split-fp16 operands outside [2^-10, 2^15]:\n  " + "\n  ".join(bad)


# ----------------------------------------------------------------------------- one step against fp64, and the seed scale
def test_vqgan_step_gradients_vs_fp64(lib, monkeypatch):
    """One codebook training step (small config, 3 images): every exported gradient against fp64 autograd through the oracle with the
    trainer's codes.  Per tensor, the relative error ||g - g64|| / max(||g64||, 1e-4) of the tensor-core trainer is at most twice that of
    the same trainer under VF_TRAIN_TC=0, plus STEP_FLOOR (1e-7).  Measured on an H100 (400 W): median 1.8e-6 (tensor cores) vs 2.6e-6 (CUDA
    cores), worst 1.1e-4 vs 8.3e-5, largest per-tensor ratio 1.35.  At this size the unscaled seeds (1 / 9216) still leave the split
    operands at 2^-12 or above, and the same numbers (largest ratio 1.49) were measured without the seed scale: the window test, not this
    one, is what catches the trainers leaving the faithful range.  At the sizes where conv_wgrad_tc, its upsampled operand and the wider
    split convs run, and for the transformer: tests/test_faithful_steps_gpu.py."""
    from viewformer_b200 import VQGAN
    from viewformer_b200.train import VQGANTrainer
    cfg = VQGANConfig(**dict(SMALL_VQ, perceptual_weight=0.0))
    sd = synth.make_vqgan_state_dict(cfg, 5)
    x = vq_images(3, cfg.image_size, 2000)
    errs, refs = {}, {}
    for tc in ("1", "0"):
        monkeypatch.setenv("VF_TRAIN_TC", tc)
        tr = VQGANTrainer(VQGAN(cfg, precision="fp32").load_state_dict({k: v.clone() for k, v in sd.items()}))
        assert tr.use_tc == (tc == "1")
        tr.forward_backward(x)
        torch.cuda.synchronize()
        codes = tr.last["codes"].cpu().long()
        key = codes.numpy().tobytes()
        if key not in refs:
            refs[key] = vq_grads64(sd, cfg, x, codes)
        ref = refs[key]
        errs[tc] = step_errors(tr.export_gradients(), ref)
    bad = faithful_report("vqgan step vs fp64", errs)
    assert not bad, "tensor-core gradients less accurate than 2x the CUDA-core trainer's: " + ", ".join(
        f"{k} {errs['1'][k]:.2e} vs {errs['0'][k]:.2e}" for k in bad[:8])


def _pair(kind, count):
    from viewformer_b200 import MIGT, VQGAN
    from viewformer_b200.train import VQGANTrainer
    from viewformer_b200.train_migt import MIGTTrainer
    out = []
    for _ in range(count):
        if kind == "migt":
            cfg = MIGTConfig(**dict(MIGT_TRAIN, gradient_clip_val=0.05))
            out.append(MIGTTrainer(MIGT(cfg, precision="fp32").load_state_dict(synth.make_migt_state_dict(cfg, 9)), warmup_steps=0))
        else:
            quantizer = "commit" if kind == "vqgan-commit" else "ema"
            cfg = VQGANConfig(**dict(SMALL_VQ, perceptual_weight=0.0, gradient_clip_val=0.02 if quantizer == "commit" else 0.0))
            sd = synth.make_vqgan_state_dict(cfg, 5)
            if quantizer == "commit":
                sd = {k: v for k, v in sd.items() if not k.startswith("quantize.") or k == "quantize.embeddings"}
            out.append(VQGANTrainer(VQGAN(cfg, precision="fp32", quantizer=quantizer).load_state_dict(sd)))
    return out


@pytest.mark.parametrize("kind", ["vqgan", "vqgan-commit", "migt"])
def test_seed_scale_is_exact_on_cuda_cores(lib, monkeypatch, kind):
    """Under VF_TRAIN_TC=0 the gradient-seed scale is a power of two through a linear backward pass, divided back out exactly.  The CUDA-core
    weight gradients add with fp32 atomics, whose order differs between runs, so two runs of one trainer are not bit-identical; the check is
    that the scale changes the gradient no more than a rerun does: per tensor, ||g_on - g_off|| <= 2 ||g_off' - g_off|| + 1e-7 ||g_off||
    (g_off' = a second trainer with the scale off).  The loss is bit-identical."""
    monkeypatch.setenv("VF_TRAIN_TC", "0")
    on, off, off2 = _pair(kind, 3)
    off.grad_seed_scale = off2.grad_seed_scale = 1.0
    assert not on.use_tc and not off.use_tc
    if kind == "migt":
        B, T = 2, 4
        codes = synth.make_codes(B, T, n_embed=on.cfg.n_embeddings, seed=50)
        cams = mo.normalize_cameras(mo.to_relative_cameras(synth.make_cameras(B, T, seed=60))[0])
        losses = [t.forward_backward(cams, codes) for t in (on, off, off2)]
        grads = [t.gradients() for t in (on, off, off2)]
    else:
        x = vq_images(3, SMALL_VQ["image_size"], 2000)
        losses = [t.forward_backward(x) for t in (on, off, off2)]
        grads = [t.export_gradients() for t in (on, off, off2)]
    torch.cuda.synchronize()
    assert on._seed_scale > 1.0 and off._seed_scale == 1.0
    assert all(torch.equal(torch.as_tensor(v).cpu(), torch.as_tensor(losses[1]).cpu()) for v in losses)
    worst, exact, bad = 0.0, 0, []
    for k in grads[1]:
        g_on, g_off, g_rr = (gr[k].double() for gr in grads)
        d_on, d_rr, nrm = float((g_on - g_off).norm()), float((g_rr - g_off).norm()), float(g_off.norm())
        exact += d_on == 0.0
        worst = max(worst, d_on / max(nrm, 1e-30))
        if d_on > 2 * d_rr + 1e-7 * nrm:
            bad.append(f"{k}: {d_on:.3e} vs rerun {d_rr:.3e} (|g| {nrm:.3e})")
    print(f"[seed scale {kind}] scale {on._seed_scale:g}: {exact} of {len(grads[1])} gradients bit-identical with the scale off, worst relative "
          f"difference {worst:.2e}")
    assert not bad, "the seed scale changes gradients by more than a rerun:\n  " + "\n  ".join(bad[:8])
