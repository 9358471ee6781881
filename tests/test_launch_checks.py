"""The launch checkers of tests/launch_checks.py on the CPU: each accepts an output computed by an independent fp64 restatement rounded to the
output dtype, and rejects that output with one named fault put in (a dropped tap, a residual read one row off, a zeroed tail tile, a shifted
column window, a zeroed last image, swapped heads, a missing max rescale, a shifted dropout mask, swapped stream gradients, an index off by
one).  So a checker that stopped looking at part of its output would fail here, before any GPU run."""
import math
import random
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import launch_checks as lc
from viewformer_b200 import _lib as L


def gen(seed):
    return torch.Generator().manual_seed(seed)


def run(name, fn, write, *a, **k):
    """Bind ``fn``'s arguments, snapshot as the audit does, let ``write`` play the kernel, return the checker's ratio."""
    before, check = lc.CHECKERS[name]
    ba = lc.bind(fn, *a, **k)
    st = before(ba, random.Random(0))
    result = write(ba)
    return check(ba, result, st)


def assert_pass_and_catch(name, fn, good, bad, *a, **k):
    r_good = run(name, fn, good, *a, **k)
    r_bad = run(name, fn, bad, *a, **k)
    print(f"[{name}] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0, f"{name}: the fp64 restatement fails its own check ({r_good:.3g})"
    assert r_bad > 1.0, f"{name}: the mutation was not caught ({r_bad:.3g})"


@pytest.fixture(autouse=True)
def dropout_hook(monkeypatch):
    def mask(shape, rate, seed, device):
        keep = torch.rand(shape, generator=gen(int(seed))) >= rate
        return keep.float().to(device) / (1.0 - rate)
    monkeypatch.setitem(lc.HOOKS, "dropout_mask", mask)


# ----------------------------------------------------------------------------------------------- GEMM
def _gemm_ref(A, B, bias=None, res=None, gelu=False):
    y = torch.einsum("...mk,...nk->...mn", A.double(), B.double())
    if bias is not None:
        y = y + bias.double()
    if gelu:
        y = F.gelu(y)
    return y if res is None else y + res.double()


def test_tc_gemm_residual_row_offset_and_partial_tile():
    M, N, K = 200, 72, 136
    A = torch.randn(M, K, generator=gen(1)).bfloat16()
    B = (torch.randn(N, K, generator=gen(2)) / K ** 0.5).bfloat16()
    bias, res = torch.randn(N, generator=gen(3)), torch.randn(M, N, generator=gen(4))
    out = torch.empty(M, N)
    ref = _gemm_ref(A, B, bias, res).float()
    kw = dict(M=M, N=N, K=K, lda=K, ldb=K, ldc=N, bias=bias, bias_mode=L.BIAS_N, residual=res)

    def good(ba):
        return out.copy_(ref)

    def res_off(ba):                                       # residual read one row below
        return out.copy_(ref - res + torch.roll(res, 1, 0))

    def tail(ba):                                          # last partial 128-row tile never written
        out.copy_(ref)
        out[128:] = 0
        return out
    assert_pass_and_catch("tc_gemm", L.tc_gemm, good, res_off, A, B, out, **kw)
    assert_pass_and_catch("tc_gemm", L.tc_gemm, good, tail, A, B, out, **kw)


def test_tc_gemm_c_off_window_batched_gelu_out2():
    """Batched (2, 3) GELU GEMM into a column window of a wider buffer, bf16 second output."""
    b1, b2, M, N, K = 2, 3, 64, 40, 64
    A = torch.randn(b1, b2, M, K, generator=gen(5)).bfloat16()
    B = (torch.randn(b1, b2, N, K, generator=gen(6)) / 8).bfloat16()
    ref = _gemm_ref(A, B, gelu=True).float()
    ldc = 2 * N
    out = torch.zeros(b1, b2, M, ldc)
    out2 = torch.zeros(b1, b2, M, ldc, dtype=torch.bfloat16)
    kw = dict(M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, batch=(b1, b2), a_bs=(b2 * M * K, M * K), b_bs=(b2 * N * K, N * K),
              c_bs=(b2 * M * ldc, M * ldc), act=L.ACT_GELU, c_off=N, out2=out2)

    def write(shift):
        def w(ba):
            out.zero_()
            out[..., N + shift:2 * N + shift] = ref[..., :N - shift] if shift else ref
            out2.copy_(out.to(torch.bfloat16))
            return out
        return w
    assert_pass_and_catch("tc_gemm", L.tc_gemm, write(0), write(1), A, B, out, **kw)

    def bad_out2(ba):
        write(0)(ba)
        out2[1, 2, 5, N + 3] = -out2[1, 2, 5, N + 3] if float(out2[1, 2, 5, N + 3]) != 0 else 1.0
        return out
    assert run("tc_gemm", L.tc_gemm, bad_out2, A, B, out, **kw) == math.inf


def test_tc_gemm_shared_operand_stride_zero():
    """The shared-scene KV query's QK^T (MIGT._query_block): every query batch entry reads the one cached scene through a stride-0 batch
    (b_bs[0] = 0) at b_off = d, head h at column h dh; the output rows have S_ctx + 64 columns, of which this GEMM writes the first S_ctx.
    Mutant: query i reads the keys of scene i (the per-scene offset of an unshared cache where the batch stride is 0)."""
    Nq, H, dh, S_ctx = 3, 2, 64, 128
    d, ld = H * dh, S_ctx + 64
    q = torch.randn(Nq * 64, 2 * d, generator=gen(15)).bfloat16()
    kc = (torch.randn(Nq, S_ctx, 2 * d, generator=gen(16)) / 8).bfloat16()       # Nq scenes in storage, the call reads scene 0
    out = torch.zeros(Nq, H, 64, ld)
    kw = dict(M=64, N=S_ctx, K=dh, lda=2 * d, ldb=2 * d, ldc=ld, batch=(Nq, H), a_bs=(64 * 2 * d, dh), b_bs=(0, dh),
              c_bs=(H * 64 * ld, 64 * ld), b_off=d)

    def write(scene_of):
        def w(ba):
            out.zero_()
            for i in range(Nq):
                for h in range(H):
                    qi = q[i * 64:(i + 1) * 64, h * dh:(h + 1) * dh]
                    ks = kc[scene_of(i), :, d + h * dh:d + (h + 1) * dh]
                    out[i, h, :, :S_ctx] = _gemm_ref(qi, ks).float()
            return out
        return w
    assert_pass_and_catch("tc_gemm", L.tc_gemm, write(lambda i: 0), write(lambda i: i), q, kc, out, **kw)


def test_tc_gemm_operand_readings():
    """TF32 truncation, split-fp16 pairs at lo_a / lo_b, k_offsets and the causal k-limit are read as the kernel reads them."""
    M, N, K = 96, 64, 64
    A = torch.randn(M, K, generator=gen(7))
    B = torch.randn(N, K, generator=gen(8))
    out = torch.empty(M, N)
    want = (lc.tf32(A).double() @ lc.tf32(B).double().t()).float()
    assert_pass_and_catch("tc_gemm", L.tc_gemm, lambda ba: out.copy_(want), lambda ba: out.copy_((A.double() @ B.double().t()).float() + 1e-3 * want),
                          A, B, out, M=M, N=N, K=K, lda=K, ldb=K, ldc=N)
    # split fp16, lo at a larger stride, A shifted by k_offsets per batch1 index (the weight-gradient GEMM pattern)
    a32, b32 = torch.randn(M, K + 8, generator=gen(9)), torch.randn(N, K, generator=gen(10))
    ah, al = lc.split_pair(a32)
    bh, bl = lc.split_pair(b32)
    la = K + 16
    Aop = torch.zeros(M, 2 * la, dtype=torch.float16)
    Aop[:, :K + 8], Aop[:, la:la + K + 8] = ah, al
    Bop = torch.cat([bh, bl], 1)
    av = lc.split_value(a32)
    bv = lc.split_value(b32)
    outs = torch.empty(2, M, N)
    ref = torch.stack([av[:, o:o + K] @ bv.t() for o in (0, 8)]).float()
    kw = dict(M=M, N=N, K=K, lda=2 * la, ldb=2 * K, ldc=N, batch=(2, 1), c_bs=(M * N, 0), lo_a=la, lo_b=K, k_offsets=[0, 8])
    assert_pass_and_catch("tc_gemm", L.tc_gemm, lambda ba: outs.copy_(ref), lambda ba: outs.copy_(torch.stack([ref[0], ref[0]])),
                          Aop, Bop, outs, **kw)
    # causal QK^T: only visible columns are compared; the skipped tiles of a torch.empty buffer hold any bits, NaN and inf included
    S, blk = 256, 64
    q, k = torch.randn(S, 64, generator=gen(11)).bfloat16(), torch.randn(S, 64, generator=gen(12)).bfloat16()
    sc = torch.empty(S, S)
    full = (q.double() @ k.double().t()).float()
    vis = (torch.arange(S)[None, :] // blk) <= (torch.arange(S)[:, None] // blk)
    junk = torch.tensor([1e30, math.nan, math.inf, -math.inf]).repeat(S * S // 4).reshape(S, S)

    def hidden_garbage(ba):
        return sc.copy_(torch.where(vis, full, junk))

    def visible_garbage(ba):
        hidden_garbage(ba)
        sc[200, 130] += 1.0
        return sc
    assert_pass_and_catch("tc_gemm", L.tc_gemm, hidden_garbage, visible_garbage, q, k, sc, M=S, N=S, K=64, lda=64, ldb=64, ldc=S,
                          causal_block=blk, causal_skip_n=True)


def test_tc_gemm_fused_group_norm_sums():
    M, N, K = 128, 128, 64
    A, B = torch.randn(M, K, generator=gen(13)).bfloat16(), (torch.randn(N, K, generator=gen(14)) / 8).bfloat16()
    out = torch.empty(M, N)
    ref = _gemm_ref(A, B).float()

    def write(err):
        def w(ba):
            out.copy_(ref)
            y = ref.double().reshape(2, 64, 32, 4)
            sums = torch.stack([y.sum((1, 3)), (y * y).sum((1, 3))], -1)
            sums[1, 31, 0] += err
            out._gn_sums = (sums, 32)
            return out
        return w
    assert_pass_and_catch("tc_gemm", L.tc_gemm, write(0.0), write(1e-2), A, B, out, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, gn_rows_per_img=64)


def test_simt_gemm_strided_bf16_out():
    M, N, K = 130, 48, 40
    A = torch.randn(K, M, generator=gen(15))                # read transposed: a_strides = (1, M)
    B = torch.randn(K, N, generator=gen(16)).bfloat16()
    bias = torch.randn(M, generator=gen(17))
    out = torch.empty(M, N, dtype=torch.bfloat16)
    ref = (A.double().t() @ B.double() + bias.double()[:, None])
    kw = dict(M=M, N=N, K=K, a_strides=(1, M), b_strides=(N, 1), ldc=N, bias=bias, bias_mode=L.BIAS_M)
    assert_pass_and_catch("simt_gemm", L.simt_gemm, lambda ba: out.copy_(ref.to(torch.bfloat16)),
                          lambda ba: out.copy_((ref - bias.double()[:, None] + bias.double()[None, :N].mean()).to(torch.bfloat16)), A, B, out, **kw)


# ----------------------------------------------------------------------------------------------- convs
def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def test_tc_conv_dropped_tap_and_last_image():
    n, h, w, cin, cout = 3, 5, 7, 64, 128
    x = torch.randn(n, h, w, cin, generator=gen(20)).bfloat16()
    wt = (torch.randn(cout, cin, 3, 3, generator=gen(21)) / 24).bfloat16()
    w_nk = wt.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    bias, res = torch.randn(cout, generator=gen(22)), torch.randn(n, h, w, cout, generator=gen(23))
    ref = _nhwc(F.conv2d(_nchw(x.double()), wt.double(), bias.double(), padding=1)) + res.double()
    out = torch.empty(n, h, w, cout)
    wt_drop = wt.double().clone()
    wt_drop[:, :, 2, 0] = 0                                                      # tap (dy, dx) = (1, -1) left out
    dropped = _nhwc(F.conv2d(_nchw(x.double()), wt_drop, bias.double(), padding=1)) + res.double()

    def last_zero(ba):
        out.copy_(ref)
        out[-1] = 0
        return out
    kw = dict(residual=res)
    assert_pass_and_catch("tc_conv", L.tc_conv, lambda ba: out.copy_(ref), lambda ba: out.copy_(dropped), x, w_nk, bias, out=out, **kw)
    assert_pass_and_catch("tc_conv", L.tc_conv, lambda ba: out.copy_(ref), last_zero, x, w_nk, bias, out=out, **kw)


def test_tc_conv_split_space_to_depth():
    """Stride-2 conv of the exact encoder: a split-fp16 space-to-depth operand read through the tap / coff table."""
    n, h, w, c, cout = 2, 8, 6, 64, 128
    x = torch.randn(n, h, w, c, generator=gen(24))
    wt = torch.randn(cout, c, 3, 3, generator=gen(25)) / 24
    xs = x.reshape(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, h // 2, w // 2, 4 * c)
    hi, lo = lc.split_pair(xs)
    xop = torch.cat([hi, lo], -1)
    whi, wlo = lc.split_pair(wt.permute(0, 2, 3, 1).reshape(cout, 9, c))
    w_nk = torch.stack([whi, wlo], 2).reshape(cout, 18 * c)
    xv = lc.split_value(x)
    wv = (whi.double() + wlo.double() / 2048).reshape(cout, 3, 3, c).permute(0, 3, 1, 2)
    ref = _nhwc(F.conv2d(F.pad(_nchw(xv), (0, 1, 0, 1)), wv, stride=2))
    out = torch.empty(n, h // 2, w // 2, cout)
    kw = dict(taps=L.TAPS_S2D, coffs=L.s2d_coffs(c), cin=c, out=out)
    assert_pass_and_catch("tc_conv", L.tc_conv, lambda ba: out.copy_(ref), lambda ba: out.copy_(_nhwc(F.conv2d(_nchw(xv), wv, stride=2, padding=1))),
                          xop, w_nk, None, **kw)


def test_tc_conv_fused_norm_operand():
    n, h, w, c, cout = 2, 4, 4, 64, 128
    x = (torch.randn(n, h, w, c, generator=gen(26)) * 2 + 1).bfloat16()
    mr = torch.stack([torch.randn(n, 32, generator=gen(27)), torch.rand(n, 32, generator=gen(28)) + 0.5], -1)
    gamma, beta = torch.randn(c, generator=gen(29)), torch.randn(c, generator=gen(30))
    wt = (torch.randn(cout, c, 3, 3, generator=gen(31)) / 24).bfloat16()
    w_nk = wt.permute(0, 2, 3, 1).reshape(cout, 9 * c).contiguous()
    a = lc._gn_apply_bf16_torch(x, mr, gamma, beta, True).double()
    ref = _nhwc(F.conv2d(_nchw(a), wt.double(), padding=1))
    raw = _nhwc(F.conv2d(_nchw(x.double()), wt.double(), padding=1))
    out = torch.empty(n, h, w, cout)
    assert_pass_and_catch("tc_conv", L.tc_conv, lambda ba: out.copy_(ref), lambda ba: out.copy_(raw), x, w_nk, None, out=out,
                          norm=(mr, gamma, beta, 32, True))


@pytest.mark.parametrize("case", ["plain", "downsample", "upsample", "small_cin", "small_cout"])
def test_cuda_core_convs(case):
    n, h, w = 2, 6, 6
    cin, cout, kh = {"small_cin": (3, 128, 3), "small_cout": (128, 3, 3)}.get(case, (16, 24, 3))
    x = torch.randn(n, h, w, cin, generator=gen(40))
    wt = torch.randn(cout, cin, kh, kh, generator=gen(41)) / 8
    w_kn = wt.permute(2, 3, 1, 0).reshape(kh * kh * cin, cout).contiguous()
    bias = torch.randn(cout, generator=gen(42))
    xd, wd, bd = _nchw(x.double()), wt.double(), bias.double()
    if case == "downsample":
        ref, kw, fn, name = F.conv2d(F.pad(xd, (0, 1, 0, 1)), wd, bd, stride=2), dict(kh=kh, stride=2, pad=(0, 0)), L.simt_conv, "simt_conv"
    elif case == "upsample":
        ref = F.conv2d(F.interpolate(xd, scale_factor=2, mode="nearest"), wd, bd, padding=1)
        kw, fn, name = dict(kh=kh, upsample=True), L.simt_conv, "simt_conv"
    else:
        ref = F.conv2d(xd, wd, bd, padding=1)
        kw, fn, name = (dict(kh=kh), L.simt_conv, "simt_conv") if case == "plain" else ({}, getattr(L, "conv3x3_" + case), "conv3x3_" + case)
    ref = _nhwc(ref).float().contiguous()
    bad = ref.clone()
    bad[:, -1, -1] += ref.abs().max() * 1e-3                    # the last pixel row's corner off
    assert_pass_and_catch(name, fn, lambda ba: ref, lambda ba: bad, x, w_kn, bias, **kw)


def test_simt_conv_dgrad_s2():
    n, h, w, cin, cout = 2, 8, 8, 16, 24
    x = torch.randn(n, cin, h, w, generator=gen(43), dtype=torch.float64, requires_grad=True)
    wt = torch.randn(cout, cin, 3, 3, generator=gen(44), dtype=torch.float64)
    y = F.conv2d(F.pad(x, (0, 1, 0, 1)), wt, stride=2)
    dy = torch.randn(y.shape, generator=gen(45), dtype=torch.float64)
    y.backward(dy)
    ref = _nhwc(x.grad).float().contiguous()
    w_dgrad = wt.permute(2, 3, 0, 1).reshape(9 * cout, cin).float().contiguous()
    dyn = _nhwc(dy).float().contiguous()
    assert_pass_and_catch("simt_conv_dgrad_s2", L.simt_conv_dgrad_s2, lambda ba: ref, lambda ba: torch.roll(ref, 1, 2), dyn, w_dgrad, (h, w))


# ----------------------------------------------------------------------------------------------- weight gradients
def _wgrad_ref(xv, dyv, upsample=False):
    x = _nchw(xv).clone().requires_grad_()
    xi = F.interpolate(x, scale_factor=2, mode="nearest") if upsample else x
    w = torch.zeros(dyv.shape[-1], xv.shape[-1], 3, 3, dtype=torch.float64, requires_grad=True)
    F.conv2d(xi, w, padding=1).backward(_nchw(dyv))
    return w.grad.permute(2, 3, 1, 0).reshape(-1, dyv.shape[-1])


@pytest.mark.parametrize("name", ["conv_wgrad", "conv_wgrad_tc", "conv_wgrad_bf16", "dense_wgrad_tc", "dense_wgrad_bf16"])
def test_weight_gradients(name):
    n, h, w, cin, cout = 2, 5, 6, 32, 24
    upsample = name == "conv_wgrad_bf16"
    x = torch.randn(n, h, w, cin, generator=gen(50))
    dy = torch.randn(n, 2 * h if upsample else h, 2 * w if upsample else w, cout, generator=gen(51))
    pre = torch.randn(9 * cin, cout, generator=gen(52))
    fn = getattr(L, name)
    if name.startswith("dense"):
        x, dy, pre = x.reshape(-1, cin), dy.reshape(-1, cout), pre[:cin]
        rd = (lambda v: v.to(torch.bfloat16).double()) if name.endswith("bf16") else lc.split_value
        ref = pre.double() + rd(x).t() @ rd(dy)
    elif name == "conv_wgrad":
        ref = pre.double() + _wgrad_ref(x.double(), dy.double())
    elif name == "conv_wgrad_tc":
        ref = pre.double() + _wgrad_ref(lc.split_value(x), lc.split_value(dy))
    else:
        ref = pre.double() + _wgrad_ref(x.to(torch.bfloat16).double(), dy.to(torch.bfloat16).double(), upsample=True)
    dw = pre.clone()
    kw = dict(kh=3) if name == "conv_wgrad" else (dict(upsample=True) if upsample else {})

    def good(ba):
        return dw.copy_(ref.float())

    def overwrite(ba):                                                  # forgot to accumulate into dw
        return dw.copy_((ref - pre.double()).float())
    assert_pass_and_catch(name, fn, good, overwrite, x, dy, dw, **kw)


# ----------------------------------------------------------------------------------------------- attention
def _attn_case(B, S, H, ns=1, seed=60, growing=False):
    d = H * 64
    qk = torch.randn(B, ns * S, 2 * d, generator=gen(seed)) * 0.5
    if growing:                                       # later views: larger keys, the running row maximum moves
        qk[..., d:] *= (1.0 + 0.9 * (torch.arange(ns * S) % S // 64).float())[None, :, None]
    vt = torch.randn(B, d, ns * S, generator=gen(seed + 1))
    return qk.bfloat16(), vt.bfloat16()


def _attn_ref(qk, vt, B, S, H, stream=0, ns=1, mask=None, skip=-1, lazy_row=None):
    """fp64 restatement of one stream's attention, [B*S, d]; ``lazy_row`` = (b, h, r): that row's first half of the keys keeps its own
    maximum (the rescale to the final maximum omitted)."""
    d = H * 64
    out = torch.zeros(B, S, d, dtype=torch.float64)
    view_ = torch.arange(S) // 64
    for b in range(B):
        for h in range(H):
            q = qk[b, stream * S:(stream + 1) * S, h * 64:(h + 1) * 64].double()
            k0 = qk[b, :S, d + h * 64:d + (h + 1) * 64].double()
            v0 = vt[b, h * 64:(h + 1) * 64, :S].double().t()
            if stream == 0:
                kk, vv, vis = k0, v0, (view_[None, :] <= view_[:, None]) & (view_ != skip)[None, :]
            else:
                ks = qk[b, stream * S:(stream + 1) * S, d + h * 64:d + (h + 1) * 64].double()
                vs = vt[b, h * 64:(h + 1) * 64, stream * S:(stream + 1) * S].double().t()
                kk, vv = torch.cat([k0, ks]), torch.cat([v0, vs])
                vis = torch.cat([view_[None, :] < view_[:, None], view_[None, :] == view_[:, None]], 1)
            sc = (q @ kk.t()).masked_fill(~vis, -math.inf)
            p = torch.softmax(sc, 1)
            if lazy_row is not None and lazy_row[:2] == (b, h):
                r = lazy_row[2]
                half = int(vis[r].sum()) // 2
                m1, m = sc[r, :half].max(), sc[r].max()
                e = torch.exp(sc[r] - m)
                e[:half] = torch.exp(sc[r, :half] - m1)
                p[r] = e / torch.exp(sc[r] - m).sum()
            if mask is not None:
                p = p * mask[b, h]
            out[b, :, h * 64:(h + 1) * 64] = p @ vv
    return out.reshape(B * S, d)


def test_attn_block_causal_heads_and_lazy_rescale():
    B, S, H = 2, 256, 2
    qk, vt = _attn_case(B, S, H, growing=True)
    ref = _attn_ref(qk, vt, B, S, H).to(torch.bfloat16)
    swapped = ref.reshape(B * S, H, 64).flip(1).reshape(B * S, H * 64).contiguous()
    assert_pass_and_catch("attn_block_causal", L.attn_block_causal, lambda ba: ref, lambda ba: swapped, qk, vt, B, S, H, H * 64, 64)
    lazy = _attn_ref(qk, vt, B, S, H, lazy_row=(B - 1, H - 1, S - 1)).to(torch.bfloat16)
    assert_pass_and_catch("attn_block_causal", L.attn_block_causal, lambda ba: ref, lambda ba: lazy, qk, vt, B, S, H, H * 64, 64)


def test_attn_block_causal_decode_empty_slot():
    """KV-cache decode: rows below the computed tile untouched, the empty view slot's keys never visited."""
    B, H, S = 2, 1, 6 * 64
    qk, vt = _attn_case(B, S, H, seed=64)
    first, skip = 4 * 64, 3
    ref = _attn_ref(qk, vt, B, S, H, skip=skip).to(torch.bfloat16)
    leak = _attn_ref(qk, vt, B, S, H).to(torch.bfloat16)
    out = torch.full((B * S, H * 64), 7.0, dtype=torch.bfloat16)

    def write(src, keep_below=True):
        def w(ba):
            t0 = first // 128 * 128
            o = out.reshape(B, S, -1)
            o[:, t0:] = src.reshape(B, S, -1)[:, t0:]
            if not keep_below:
                o[:, t0 - 1] = 0
            return out
        return w
    args = (qk, vt, B, S, H, H * 64, 64)
    kw = dict(first_query=first, out=out, skip_view=skip)
    assert_pass_and_catch("attn_block_causal", L.attn_block_causal, write(ref), write(leak), *args, **kw)
    out.fill_(7.0)
    assert run("attn_block_causal", L.attn_block_causal, write(ref, keep_below=False), *args, **kw) == math.inf


def test_attn_multiend_and_train_dropout():
    B, S, H, ns = 1, 192, 2, 3
    qk, vt = _attn_case(B, S, H, ns=ns, seed=66)
    for s in range(ns):
        ref = _attn_ref(qk, vt, B, S, H, stream=s, ns=ns).to(torch.bfloat16)
        other = _attn_ref(qk, vt, B, S, H, stream=(s + 1) % ns, ns=ns).to(torch.bfloat16)
        assert_pass_and_catch("attn_block_multiend", L.attn_block_multiend, lambda ba: ref, lambda ba: other, qk, vt, B, S, ns, s, H, H * 64, 64)
    rate, seed, s = 0.1, 77, 1
    mask = lc.HOOKS["dropout_mask"]((B, H, S, 2 * S), rate, seed, "cpu").double()
    lse = torch.empty(B, H, S)
    o32 = torch.empty(B * S, H * 64)

    def write(m):
        def w(ba):
            o = _attn_ref(qk, vt, B, S, H, stream=s, ns=ns, mask=m)
            o32.copy_(o.float())
            for h in range(H):
                q = qk[0, s * S:(s + 1) * S, h * 64:(h + 1) * 64].double()
                _, sc, vis, _, _ = lc._logits(qk, vt, S, H * 64, 0, h, s, 64)
                lse[0, h] = torch.logsumexp(sc.masked_fill(~vis, -math.inf), 1).float()
            return o32.to(torch.bfloat16)
        return w
    assert_pass_and_catch("attn_multiend_train", L.attn_multiend_train, write(mask), write(torch.roll(mask, 1, 3)), qk, vt, B, S, ns, s, H, H * 64, 64,
                          rate=rate, seed=seed, lse=lse, out_f32=o32)


def _walk_by_cta(B, H, S, block, resident, first_query=0, stream=0, skip_view=-1):
    """The persistent kernel's walk, restated from the visible keys: all items in walk order as ((b, h), key tiles walked), and per CTA
    its items in order.  Query tiles run from the last (most keys) to the first computed one; within a tile b-major, then h; CTA c takes
    items c, c + grid, ..."""
    per_qt = []
    for qt in reversed(range(first_query // 128, -(-S // 128))):
        q0, q1 = qt * 128, min(qt * 128 + 128, S)
        if stream == 0:
            keys = [j for j in range(0, S, 64) if j < (q1 - 1) // block * block + block and j // 64 != skip_view]
            tiles = len(keys)
        else:                              # stream-0 keys of the views before the tile, the tile's first view twice, its own views
            views = (q1 - q0) // 64
            tiles = q0 // 64 + (3 if views == 2 else 1)
        per_qt += [((b, h), tiles) for b in range(B) for h in range(H)]
    grid = min(len(per_qt), resident)
    return per_qt, [per_qt[c::grid] for c in range(grid)]


@pytest.mark.parametrize("sms,train,B,H,T,kw", [
    (132, False, 32, 12, 10, {}),                                                  # the benchmark's attention: 1920 items on 264 CTAs
    (132, False, 32, 12, 9, dict(stream=1)),                                       # odd T: the last tile holds one view
    (132, True, 5, 12, 20, dict(stream=2)),                                        # the transformer step: 600 items on 132 CTAs
    (132, False, 32, 12, 11, dict(first_query=640, skip_view=9)),                  # KV-cache decode, empty slot: every n_kt alike
    (4, False, 2, 3, 7, {}),
    (132, False, 3, 12, 10, {}),                                                   # 180 items, one per CTA: nothing added
])
def test_attn_head_sampler_covers_later_items(monkeypatch, sms, train, B, H, T, kw):
    """With the resident CTA count known, the attention checks also cover the last item in walk order and an item that a CTA walks after
    one with a different number of key tiles."""
    S = T * 64
    monkeypatch.setitem(lc.HOOKS, "attn_resident", lambda tr: (1 if tr else 2) * sms)
    fn = L.attn_multiend_train if train else (L.attn_block_multiend if "stream" in kw else L.attn_block_causal)
    qk = torch.empty(0)
    if fn is L.attn_block_causal:
        ba = lc.bind(fn, qk, qk, B, S, H, H * 64, 64, **kw)
    else:
        ba = lc.bind(fn, qk, qk, B, S, 3, kw["stream"], H, H * 64, 64)
    before = lc.before_attn_train if train else lc.before_attn
    order, walk = _walk_by_cta(B, H, S, 64, (1 if train else 2) * sms, **kw)
    mixed = {pair for items in walk for k, (pair, n) in enumerate(items) if k > 0 and any(m != n for _, m in items[:k])}
    later = mixed or {pair for items in walk for pair, _ in items[1:]}
    walks = max(len(items) for items in walk) > 1
    for seed in range(5):
        monkeypatch.setitem(lc.HOOKS, "attn_resident", None)
        plain = set(before(ba, random.Random(seed))["heads"])
        monkeypatch.setitem(lc.HOOKS, "attn_resident", lambda tr: (1 if tr else 2) * sms)
        heads = set(before(ba, random.Random(seed))["heads"])
        rng = random.Random(seed)
        lc.pick(B * H, rng)                                        # the sampler draws its three pairs first
        added = lc.attn_walk_pairs(B, H, S, 64, (1 if train else 2) * sms, rng, **kw)
        assert len(plain) == min(3, B * H) and plain | set(added) == heads
        if not walks:
            assert added == [] and heads == plain
            continue
        assert added[0] == order[-1][0], f"the last item in walk order is {order[-1][0]}, not {added[0]}"
        assert added[1] in later, f"{added[1]} is not a later item of a CTA whose walk changes n_kt"
        print(f"[sampler {sms} SMs, B {B} H {H} T {T} {kw}] plain {sorted(plain)} + walk {added}; "
              f"{len(mixed)} pairs own a later item after a change of n_kt")


def _tc_walk_by_cta(order, ctas):
    """Per CTA, its tiles in walk order: CTA c takes tiles c, c + grid, ..., grid = min(tiles, ctas)."""
    grid = min(len(order), ctas)
    return [order[c::grid] for c in range(grid)]


_S2D = dict(taps=L.TAPS_S2D, coffs=L.s2d_coffs(128), cin=128)


@pytest.mark.parametrize("sms,n,hw,ctot,cout,dtype,kw,tiling", [
    (132, 3, (128, 128), 256, 128, torch.float16, {}, (16, 8, 1, True)),          # exact halo: 384 tiles, 3 per CTA
    (132, 288, (128, 128), 256, 128, torch.float16, {}, (16, 8, 1, True)),        # the benchmark's roofline conv: 36 864 tiles
    (132, 17, (32, 32), 256, 256, torch.float16, {}, (16, 8, 1, True)),          # two n tiles
    (132, 67, (8, 8), 512, 512, torch.float16, {}, (8, 8, 2, False)),            # exact tap-box, two images per tile, the last half empty
    (132, 34, (32, 32), 1024, 128, torch.float16, _S2D, (16, 8, 1, False)),      # exact stride-2 Downsample (space-to-depth taps)
    (132, 3, (128, 128), 64, 128, torch.bfloat16, {}, (8, 16, 1, True)),         # bf16 halo
    (132, 9, (64, 64), 128, 128, torch.float32, {}, (8, 16, 1, True)),           # TF32 halo
    (4, 2, (40, 20), 64, 256, torch.bfloat16, {}, (8, 16, 1, True)),             # ragged borders on a 4-SM device
    (132, 1, (32, 32), 256, 128, torch.float16, {}, (16, 8, 1, True)),           # 8 tiles, one per CTA: nothing added
])
def test_tc_conv_image_sampler_covers_later_tiles(monkeypatch, sms, n, hw, ctot, cout, dtype, kw, tiling):
    """With the SM count known, the conv check also covers the image of the last tile in walk order and the image of a tile that its CTA
    walks second or later; the tiling it assumes is the launcher's (stated here per case)."""
    h, w = hw
    x = torch.empty(1, dtype=dtype).expand(n, h, w, ctot)              # bind reads shapes only
    wn = torch.empty(1, dtype=dtype).expand(cout, 1)
    ba = lc.bind(L.tc_conv, x, wn, None, **kw)
    cin = kw.get("cin", ctot // (2 if dtype == torch.float16 else 1))
    assert lc.tc_conv_tiling(h, w, ctot, cin, h, w, ba["taps"], ba["coffs"], dtype == torch.float16, dtype == torch.float32) == tiling
    tw, th, tn, _ = tiling
    bn = 128 if cout > 64 else 64
    order = [it * tn for it in range(-(-n // tn)) for _ in range(-(-h // th)) for _ in range(-(-w // tw)) for _ in range(-(-cout // bn))]
    walk = _tc_walk_by_cta(order, sms)
    later = {img for tiles in walk for img in tiles[1:]}
    for seed in range(5):
        monkeypatch.setitem(lc.HOOKS, "tc_ctas", None)
        plain = set(lc.before_tc_conv(ba, random.Random(seed))["images"])
        monkeypatch.setitem(lc.HOOKS, "tc_ctas", lambda: sms)
        images = set(lc.before_tc_conv(ba, random.Random(seed))["images"])
        rng = random.Random(seed)
        lc.pick(n, rng)                                                   # the sampler draws its three images first
        added = [order[t] for t in lc.tc_walk_tiles(len(order), sms, rng)]
        assert plain == set(lc.pick(n, random.Random(seed))) and images == plain | set(added)
        if len(walk[0]) == 1:
            assert added == [] and images == plain
            continue
        assert added[0] == order[-1] and added[1] in later, f"{added} are not the last tile's image and a later tile's image"
        print(f"[tc sampler {sms} SMs, {n} x {hw} {ctot}->{cout} {dtype}] {len(order)} tiles, up to {len(walk[0])} per CTA: "
              f"plain {sorted(plain)} + walk {added}")


@pytest.mark.parametrize("sms,M,N,batch", [(132, 1024, 256, (3, 3)), (132, 1024, 1024, (3, 1)), (132, 1024, 64, (20, 1)),
                                           (4, 300, 200, (1, 2)), (132, 512, 256, (2, 1))])
def test_tc_gemm_batch_sampler_covers_later_tiles(monkeypatch, sms, M, N, batch):
    """With the SM count known, the GEMM check also covers the batch entry and the 128-row block of the last tile in walk order and of a
    tile that its CTA walks second or later."""
    A = torch.empty(1, dtype=torch.bfloat16).expand(M, 64)
    ba = lc.bind(L.tc_gemm, A, A, torch.empty(1).expand(M, N), M=M, N=N, K=64, lda=64, ldb=64, ldc=N, batch=batch)
    bn = 128 if N > 64 else 64
    order = [(b, m0) for b in range(batch[0] * batch[1]) for m0 in range(0, M, 128) for _ in range(-(-N // bn))]
    walk = _tc_walk_by_cta(order, sms)
    later = {tile for tiles in walk for tile in tiles[1:]}
    for seed in range(5):
        monkeypatch.setitem(lc.HOOKS, "tc_ctas", lambda: sms)
        st = lc.before_tc_gemm(ba, random.Random(seed))
        rng = random.Random(seed)
        plain_b, plain_rows = lc.pick(batch[0] * batch[1], rng), lc.pick_rows(M, rng)
        added = [order[t] for t in lc.tc_walk_tiles(len(order), sms, rng)]
        rows = set(plain_rows.tolist()) | {r for _, m0 in added for r in range(m0, min(m0 + 128, M))}
        assert st["batches"] == sorted(set(plain_b) | {b for b, _ in added}) and set(st["rows"].tolist()) == rows
        if len(walk[0]) == 1:
            assert added == []
            continue
        assert added[0] == order[-1] and added[1] in later
        print(f"[tc sampler {sms} SMs, gemm {M} x {N} batch {batch}] {len(order)} tiles, up to {len(walk[0])} per CTA: "
              f"batches {st['batches']}, walk tiles (batch, m0) {added}")


def test_attn_multiend_bwd_stream_swap():
    B, S, H, ns, rate, seed = 1, 128, 1, 3, 0.1, 90
    d = H * 64
    qk, vt = _attn_case(B, S, H, ns=ns, seed=70)
    dout = torch.randn(ns, B * S, d, generator=gen(72)).bfloat16()
    q = [qk[:, s * S:(s + 1) * S, :d].double().reshape(B, S, H, 64).permute(0, 2, 1, 3).clone().requires_grad_() for s in range(ns)]
    k = [qk[:, s * S:(s + 1) * S, d:].double().reshape(B, S, H, 64).permute(0, 2, 1, 3).clone().requires_grad_() for s in range(ns)]
    v = [vt[:, :, s * S:(s + 1) * S].double().reshape(B, H, 64, S).transpose(2, 3).clone().requires_grad_() for s in range(ns)]
    view_ = torch.arange(S) // 64
    o32, lse, total = torch.empty(ns, B * S, d), torch.empty(ns, B, H, S), 0.0
    for s in range(ns):
        if s == 0:
            lg, vis, vv = q[0] @ k[0].transpose(2, 3), view_[None, :] <= view_[:, None], v[0]
        else:
            lg = torch.cat([q[s] @ k[0].transpose(2, 3), q[s] @ k[s].transpose(2, 3)], 3)
            vis, vv = torch.cat([view_[None, :] < view_[:, None], view_[None, :] == view_[:, None]], 1), torch.cat([v[0], v[s]], 2)
        lg = lg.masked_fill(~vis, -math.inf)
        ls = torch.logsumexp(lg, 3)
        P = torch.exp(lg - ls[..., None]) * lc.HOOKS["dropout_mask"](lg.shape, rate, seed + s, "cpu").double()
        o = (P @ vv).permute(0, 2, 1, 3).reshape(B * S, d)
        o32[s], lse[s] = o.detach().float(), ls.detach().float()
        total = total + (o * dout[s].double()).sum()
    total.backward()
    f = lambda t: t.grad.permute(0, 2, 1, 3).reshape(B * S, d)
    ref = torch.stack([torch.cat([f(v[s]), f(q[s]), f(k[s])], 1) for s in range(ns)]).float()
    dvqk = torch.zeros(ns, B * S, 3 * d)
    args = (qk, vt, dout, o32, lse, B, S, ns, H, d, 64)
    kw = dict(rate=rate, seed=seed, dvqk=dvqk)
    assert_pass_and_catch("attn_multiend_bwd", L.attn_multiend_bwd, lambda ba: dvqk.copy_(ref), lambda ba: dvqk.copy_(ref[[0, 2, 1]]), *args, **kw)


# ----------------------------------------------------------------------------------------------- codebook lookup
@pytest.mark.parametrize("name", ["vq_lookup", "vq_lookup_fused"])
def test_lookup_index_off_by_one(name, monkeypatch):
    m, d, k = 300, 64, 256
    z = torch.randn(m, d, generator=gen(80))
    et = torch.randn(k, d, generator=gen(81))
    esq = (et * et).sum(1)
    dist = (z.double()[:, None, :] - et.double()[None]).pow(2).sum(2)
    idx = dist.argmin(1)
    if name != "vq_lookup":
        monkeypatch.setitem(lc.HOOKS, "ref_lookup", lambda z_, et_, esq_: idx)

    def write(ix):
        def w(ba):
            e = et[ix]
            return ix, z + (e - z), torch.tensor([float(((e.double() - z.double()) ** 2).sum())], dtype=torch.float64)
        return w
    bad = idx.clone()
    bad[-1] = (bad[-1] + 1) % k
    extra = {"vq_lookup": (), "vq_lookup_fused": (et.bfloat16(),)}[name]
    assert_pass_and_catch(name, getattr(L, name), write(idx), write(bad), z, et, esq, *extra)


# ----------------------------------------------------------------------------------------------- the checkers look where they claim
def test_removing_the_residual_from_the_reference_is_caught(monkeypatch):
    """A checker whose reference drops a term fails on a correct output: the CPU tests pin the references, not only the mutations."""
    M, N, K = 64, 64, 64
    A, B = torch.randn(M, K, generator=gen(90)).bfloat16(), torch.randn(N, K, generator=gen(91)).bfloat16()
    res = torch.randn(M, N, generator=gen(92))
    out = _gemm_ref(A, B, res=res).float()
    kw = dict(M=M, N=N, K=K, lda=K, ldb=K, ldc=N, residual=res)
    assert run("tc_gemm", L.tc_gemm, lambda ba: out, A, B, out, **kw) <= 1.0
    orig = lc.before_tc_gemm
    monkeypatch.setitem(lc.CHECKERS, "tc_gemm", (lambda ba, rng: dict(orig(ba, rng), res=None), lc.check_tc_gemm))
    assert run("tc_gemm", L.tc_gemm, lambda ba: out, A, B, out, **kw) > 1.0


def test_every_launching_wrapper_has_a_checker():
    """Every public _lib function whose code names a vf_* entry point or a checked wrapper has a checker, or is listed in
    launch_checks.UNCHECKED with its reason: a new wrapper cannot bypass the launch audit."""
    import inspect
    pat = re.compile(r"^vf_\w+$")
    checked = set(lc.CHECKERS)
    public = {name for name, fn in vars(L).items() if inspect.isfunction(fn) and fn.__module__ == L.__name__ and not name.startswith("_")
              and any(pat.match(n) or n in checked or n == "_wgrad_tc" for n in fn.__code__.co_names)}
    public -= {"load"}                                         # dlopen and the device check: launches nothing
    assert {"tc_gemm", "groupnorm", "softmax_rows", "vq_ema_update", "resize_u8", "ssim_u8", "pad_transpose_bf16"} <= public
    missing = sorted(public - checked - set(lc.UNCHECKED))
    stale = sorted(set(lc.UNCHECKED) & checked)
    print(f"[completeness] {len(public)} launching wrappers, {len(public & checked)} checked; unchecked with a reason: {sorted(lc.UNCHECKED)}")
    assert not missing, f"_lib wrappers that launch kernels without a checker in tests/launch_checks.py: {missing}"
    assert not stale, f"UNCHECKED lists wrappers that have a checker: {stale}"
    assert all(len(r) > 40 for r in lc.UNCHECKED.values())


# ----------------------------------------------------------------------------------------------- normalisation
def _gn_input(n, hw, c, ratio=3.0, seed=100):
    g = gen(seed)
    return (ratio * torch.randn(n, 1, 1, c, generator=g) + torch.randn(n, hw, 1, c, generator=g)).contiguous()


def _mr64(x, groups=32, eps=1e-6):
    m, v, _, _ = lc._gn_stats64(x, groups)
    return torch.stack([m, 1.0 / torch.sqrt(v + eps)], -1).float()


def test_gn_mean_rstd_stats_pass_and_fused_sums():
    """The stats pass at a 128 x 128 x 128 map (65 536 terms per group): a group shifted by one channel quad is caught; fused sums with
    one group's sum of squares off by 1e-4 are caught."""
    x = _gn_input(1, 128 * 128, 128)
    good = _mr64(x)
    xs = torch.roll(x, 4, -1)
    assert_pass_and_catch("gn_mean_rstd", L.gn_mean_rstd, lambda ba: good.clone(), lambda ba: _mr64(xs), x)
    xf = _gn_input(2, 256, 128, seed=101)
    xg = xf.double().reshape(2, 256, 32, 4)
    xf._gn_sums = (torch.stack([xg.sum((1, 3)), (xg * xg).sum((1, 3))], -1), 32)
    bad = xf.double().reshape(2, 256, 32, 4).clone()
    bad[1, :, 31] *= 1.0 + 1e-4
    badm = torch.stack([bad.mean((1, 3)), 1 / torch.sqrt(bad.var((1, 3), unbiased=False) + 1e-6)], -1).float()
    assert_pass_and_catch("gn_mean_rstd", L.gn_mean_rstd, lambda ba: _mr64(xf), lambda ba: badm, xf)


def _gn_apply64(x, mr, gamma, beta, swish):
    n, h, w, c = x.shape
    cidx = torch.arange(c) // (c // mr.shape[1])
    mu, rs = mr.double()[:, cidx, 0][:, None, None], mr.double()[:, cidx, 1][:, None, None]
    y = (x.double() - mu) * rs * gamma.double() + beta.double()
    return y * torch.sigmoid(y) if swish else y


@pytest.mark.parametrize("layout", ["plain_f32", "plain_bf16", "upsample_bf16", "s2d_split"])
def test_groupnorm_apply(layout, monkeypatch):
    """groupnorm with given and with computed statistics; faults: the last pixel chunk not written, groups shifted by one quad, a bf16
    output rounded toward zero."""
    n, h, w, c = 2, 8, 6, 128
    x = _gn_input(n, h * w, c, seed=102).reshape(n, h, w, c)
    g = gen(103)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g)
    mr = _mr64(x)
    monkeypatch.setitem(lc.HOOKS, "gn_mean_rstd", lambda x_, groups, eps: _mr64(x_, groups, eps))
    ref = _gn_apply64(x, mr, gamma, beta, True)
    kw = dict(swish=True, stats=None if layout == "plain_bf16" else mr)
    if layout == "plain_f32":
        kw["out_dtype"] = torch.float32
        bad_ref = ref.clone()
        bad_ref[:, -1, -1] = 0
        good, bad = ref.float(), bad_ref.float()
    elif layout == "plain_bf16":
        kw["out_dtype"] = torch.bfloat16
        good = ref.float().to(torch.bfloat16)
        f = ref.float()
        bad = (f.view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)       # truncated toward zero
    elif layout == "upsample_bf16":
        kw.update(out_dtype=torch.bfloat16, upsample=True)
        up = ref.repeat_interleave(2, 1).repeat_interleave(2, 2)
        good = up.float().to(torch.bfloat16)
        bad = _gn_apply64(x, torch.roll(mr, 1, 1), gamma, beta, True).repeat_interleave(2, 1).repeat_interleave(2, 2).float().to(torch.bfloat16)
    else:
        kw.update(out_dtype=torch.float16, s2d=True)

        def s2d(t):
            v = t.float().reshape(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, h // 2, w // 2, 4 * c)
            hi, lo = lc.split_pair(v)
            return torch.cat([hi, lo], -1)
        good = s2d(ref)
        flat = ref.clone()
        flat[:, :, :, :4] = ref[:, :, :, 4:8]                                           # one channel quad read from its neighbour
        bad = s2d(flat)
    assert_pass_and_catch("groupnorm", L.groupnorm, lambda ba: good, lambda ba: bad, x, gamma, beta, **kw)


def test_layernorm_row_tail():
    rows, d = 301, 768
    g = gen(104)
    x = 30.0 * torch.randn(rows, 1, generator=g) + torch.randn(rows, d, generator=g)
    gamma, beta = torch.rand(d, generator=g) + 0.5, torch.randn(d, generator=g)
    y = F.layer_norm(x.double(), (d,), gamma.double(), beta.double(), 1e-5).float()
    bad = y.clone()
    bad[-1, -4:] = 0                                                                    # the last quad of the last row
    assert_pass_and_catch("layernorm", L.layernorm, lambda ba: y, lambda ba: bad, x, gamma, beta, torch.float32)


def _gn_bwd64(x, dout, mr, gamma, beta, swish, add):
    n, h, w, c = x.shape
    cidx = torch.arange(c) // (c // 32)
    mu, rs = mr.double()[:, cidx, 0].reshape(n, 1, 1, c), mr.double()[:, cidx, 1].reshape(n, 1, 1, c)
    xd = x.double().requires_grad_(True)
    ga, be = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    # autograd of the normalisation with the given statistics treated as functions of x (the kernel's formula)
    xg = xd.reshape(n, h * w, 32, c // 32)
    m = xg.mean((1, 3))[:, cidx].reshape(n, 1, 1, c)
    v = ((xg - xg.mean((1, 3), keepdim=True)) ** 2).mean((1, 3))[:, cidx].reshape(n, 1, 1, c)
    xh = (xd - m) / torch.sqrt(v + 1e-6)
    xh = xh + (((x.double() - mu) * rs) - xh).detach()                                  # values from the given statistics
    y = xh * ga + be
    if swish:
        y = y * torch.sigmoid(y)
    y.backward(dout.double())
    return xd.grad + (0.0 if add is None else add.double()), ga.grad, be.grad


@pytest.mark.parametrize("fault", ["add_ignored", "dgamma_overwritten", "bf16_toward_zero"])
def test_groupnorm_bwd(fault):
    n, h, w, c = 2, 16, 16, 128
    g = gen(105)
    x = _gn_input(n, h * w, c, seed=106).reshape(n, h, w, c)
    dout = torch.randn(n, h, w, c, generator=g)
    add = torch.randn(n, h, w, c, generator=g)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.3
    mr = _mr64(x)
    dx, dg, db = _gn_bwd64(x, dout, mr, gamma, beta, True, add)
    dg0, db0 = torch.randn(c, generator=g), torch.randn(c, generator=g)
    dgam, dbet = dg0.clone(), db0.clone()

    def write(bad):
        def w_(ba):
            out = (dx - (add.double() if bad == "add_ignored" else 0.0)).float()
            dgam.copy_((dg + (0 if bad == "dgamma_overwritten" else dg0.double())).float())
            dbet.copy_((db + db0.double()).float())
            out._bf16 = ((out.view(torch.int32) & ~0xFFFF).view(torch.float32) if bad == "bf16_toward_zero" else out).to(torch.bfloat16)
            return out
        return w_

    def reset_and(f):
        def w_(ba):
            dgam.copy_(dg0)
            dbet.copy_(db0)
            return f(ba)
        return w_
    kw = dict(swish=True, add=add, out_bf16=True)
    r_good = run("groupnorm_bwd", L.groupnorm_bwd, reset_and(write(None)), x, dout, mr, gamma, beta, dgam, dbet, **kw)
    dgam.copy_(dg0), dbet.copy_(db0)
    r_bad = run("groupnorm_bwd", L.groupnorm_bwd, reset_and(write(fault)), x, dout, mr, gamma, beta, dgam, dbet, **kw)
    print(f"[groupnorm_bwd {fault}] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0 and r_bad > 1.0


def test_layernorm_bwd_dgamma_accumulates():
    rows, d = 3 * 2 * 64, 768
    g = gen(107)
    x = torch.randn(rows, d, generator=g) * 1.5 + 0.3
    dy = torch.randn(rows, d, generator=g)
    gamma = torch.rand(d, generator=g) + 0.5
    add = torch.randn(rows, d, generator=g)
    xd, gd = x.double().requires_grad_(True), gamma.double().requires_grad_(True)
    bd = torch.zeros(d, dtype=torch.float64, requires_grad=True)
    F.layer_norm(xd, (d,), gd, bd, 1e-5).backward(dy.double())
    dg0, db0 = torch.randn(d, generator=g), torch.randn(d, generator=g)
    dgam, dbet = dg0.clone(), db0.clone()

    def write(overwrite):
        def w_(ba):
            dgam.copy_((gd.grad + (0 if overwrite else dg0.double())).float())
            dbet.copy_((bd.grad + db0.double()).float())
            return (xd.grad + add.double()).float()
        return w_
    r_good = run("layernorm_bwd", L.layernorm_bwd, write(False), x, dy, gamma, dgam, dbet, add=add)
    dgam.copy_(dg0), dbet.copy_(db0)
    r_bad = run("layernorm_bwd", L.layernorm_bwd, write(True), x, dy, gamma, dgam, dbet, add=add)
    print(f"[layernorm_bwd] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0 and r_bad > 1.0


# ----------------------------------------------------------------------------------------------- reductions
def test_col_sums_dropped_chunk_at_500k_rows():
    """500 000 rows (489 row chunks of 1023): K = ceil(1023 / 8) + 8 + 489 + 1 = 626, not 500 000.  The bar 2 K u sum|x| sees a dropped
    chunk whose column sum exceeds it: here rows with a mean of 0.5 per column (as a bias gradient has), so the last chunk (776 rows) adds
    about 388 against a bar of about 33.  A chunk of zero-mean noise (its sum ~ sqrt(776) ~ 28) would sit at the bar and is not seen."""
    rows, c = 500_000, 3
    x = torch.randn(rows, c, generator=gen(108)) + 0.5
    o0 = torch.randn(c, generator=gen(109))
    out = o0.clone()
    assert lc.col_sums_chain(rows) == 626
    full = (o0.double() + x.double().sum(0)).float()
    rpb = (rows + 488) // 489
    last = (rows - 1) // rpb * rpb
    drop = (o0.double() + x[:last].double().sum(0)).float()

    def write(v):
        def w(ba):
            return out.copy_(v)
        return w
    r_good = run("col_sums", L.col_sums, write(full), x, out)
    out.copy_(o0)                                              # the mutated run snapshots the value held before, as the kernel sees it
    r_bad = run("col_sums", L.col_sums, write(drop), x, out)
    print(f"[col_sums] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0 and r_bad > 1.0


def test_softmax_bwd_and_cross_entropy_grad_tails():
    rows, cols = 37, 1024
    g = gen(110)
    logits = torch.randn(rows, cols, generator=g) * 3.0
    labels = torch.randint(0, cols, (rows,), generator=g, dtype=torch.int32)
    w = torch.rand(rows, generator=g)
    s = 0.1
    ld = logits.double().requires_grad_(True)
    y = F.one_hot(labels.long(), cols).double() * (1 - lc.f32(s)) + lc.f32(s) / cols
    (-(y * F.log_softmax(ld, -1)).sum(-1) * w.double()).sum().backward()
    good = ld.grad.float()
    y0 = F.one_hot(labels.long(), cols).double()
    ld0 = logits.double().requires_grad_(True)
    (-(y0 * F.log_softmax(ld0, -1)).sum(-1) * w.double()).sum().backward()              # label smoothing missing
    assert_pass_and_catch("cross_entropy_grad", L.cross_entropy_grad, lambda ba: good, lambda ba: ld0.grad.float(), logits, labels, w, s)
    P = torch.softmax(logits, -1)
    dP = torch.randn(rows, cols, generator=g)
    Pd, dPd = P.double(), dP.double()
    ref = (Pd * (dPd - (Pd * dPd).sum(-1, keepdim=True))).float()
    bad = (Pd * (dPd - (Pd[:, :-32] * dPd[:, :-32]).sum(-1, keepdim=True))).float()      # the last 32 columns left out of the row sum
    assert_pass_and_catch("softmax_bwd_rows", L.softmax_bwd_rows, lambda ba: ref, lambda ba: bad, P, dP)


def test_sumsq_dropped_block():
    n = 1_000_000
    x = torch.randn(n, generator=gen(111))
    want = torch.tensor([(x.double() ** 2).sum()])
    bad = torch.tensor([(x[:-256].double() ** 2).sum()])
    assert_pass_and_catch("sumsq", L.sumsq, lambda ba: want, lambda ba: bad, x)


def test_migt_embed_bwd_collisions_and_fixed_token():
    """1024 codes, 3 streams of 2 x 64 tokens with heavy code collisions; the fault scatters every token to fixed_token."""
    BT, Lt, d, V = 6, 64, 96, 1025
    g = gen(112)
    dh = torch.randn(BT * Lt, d, generator=g)
    ids = torch.randint(0, 40, (BT * Lt,), generator=g, dtype=torch.int32)
    fixed = 1024
    w0, p0, q0 = torch.randn(V, d, generator=g), torch.randn(Lt, d, generator=g), torch.randn(BT, d, generator=g)
    dwte, dwpe, dpose = w0.clone(), p0.clone(), q0.clone()

    def write(index):
        def w_(ba):
            dwte.copy_(w0.double().index_add(0, index, dh.double()).float())
            dwpe.copy_(p0.double().index_add(0, torch.arange(BT * Lt) % Lt, dh.double()).float())
            dpose.copy_(q0.double().index_add(0, torch.arange(BT * Lt) // Lt, dh.double()).float())
        return w_
    r_good = run("migt_embed_bwd", L.migt_embed_bwd, write(ids.long()), dh, ids, fixed, BT, Lt, dwte, dwpe, dpose)
    for t, t0 in ((dwte, w0), (dwpe, p0), (dpose, q0)):
        t.copy_(t0)
    r_bad = run("migt_embed_bwd", L.migt_embed_bwd, write(torch.full((BT * Lt,), fixed)), dh, ids, fixed, BT, Lt, dwte, dwpe, dpose)
    print(f"[migt_embed_bwd] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0 and r_bad > 1.0


# ----------------------------------------------------------------------------------------------- elementwise
def test_gelu_and_gelu_bwd():
    x = torch.randn(20000, generator=gen(113)) * 3
    dy = torch.randn(20000, generator=gen(114))
    xd = x.double()
    cdf = 0.5 * (1 + torch.erf(xd / math.sqrt(2)))
    pdf = torch.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi)
    y = (xd * cdf).float()
    tanh = F.gelu(x, approximate="tanh")
    assert_pass_and_catch("gelu", L.gelu, lambda ba: y, lambda ba: tanh, x)
    db = (dy.double() * (cdf + xd * pdf)).float()
    assert_pass_and_catch("gelu_bwd", L.gelu_bwd, lambda ba: db, lambda ba: (dy.double() * cdf).float(), x, dy)


def test_lincomb3_in_place_bucket_rescale():
    """out aliasing x (the gradient bucket rescaled in place): the snapshot, not the overwritten x, is the reference."""
    x = torch.randn(50000, generator=gen(115))
    x0 = x.clone()
    a = 1.0 / 1024

    def good(ba):
        return x.copy_((lc.f32(a) * x0.double()).float())

    def tail(ba):
        good(ba)
        x[-100:] = x0[-100:]                                   # the tail of the buffer left unscaled
        return x
    r_good = run("lincomb3", L.lincomb3, good, a, x, out=x)
    x.copy_(x0)
    r_bad = run("lincomb3", L.lincomb3, tail, a, x, out=x)
    print(f"[lincomb3] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0 and r_bad > 1.0


def _adam_ref(p, g, m, v, lr, b1, b2, eps, t, gs):
    b1, b2, eps, lr = lc.f32(b1), lc.f32(b2), lc.f32(eps), lc.f32(lr)
    gi = g.double() * lc.f32(gs)
    m1 = m.double() + (1 - b1) * (gi - m.double())
    v1 = b2 * v.double() + (1 - b2) * gi * gi
    bc1, bc2 = lc._pow32(b1, t), lc._pow32(b2, t)
    return p.double() - lr / bc1 * m1 / (v1.sqrt() / math.sqrt(bc2) + eps), m1, v1


@pytest.mark.parametrize("opt", ["adam", "adamw_keras"])
def test_optimizers_step_count_and_decay_order(opt):
    """A 1 M-element flat buffer, sampled ranges.  adam: the step count off by one (bias corrections of t + 1); adamw_keras: the weight
    decay applied after the update instead of before."""
    n = 1 << 20
    g_ = gen(116)
    p0, g, m0, v0 = torch.randn(n, generator=g_), torch.randn(n, generator=g_) * 1e-3, torch.randn(n, generator=g_) * 1e-3, torch.rand(n, generator=g_) * 1e-6
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    t = 3
    if opt == "adam":
        kw = dict(lr=1e-4, beta1=0.5, beta2=0.9, eps=1e-8, step=t, grad_scale=0.5)

        def write(tt):
            def w_(ba):
                pr, mr, vr = _adam_ref(p0, g, m0, v0, 1e-4, 0.5, 0.9, 1e-8, tt, 0.5)
                p.copy_(pr.float()), m.copy_(mr.float()), v.copy_(vr.float())
            return w_
        good, bad, fn = write(t), write(t + 1), L.adam
    else:
        kw = dict(lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.05, step=t, grad_scale=1.0, clip_scale=0.5)

        def write(after):
            def w_(ba):
                gi = g.double() * 0.5
                mr = m0.double() + (gi - m0.double()) * (1 - lc.f32(0.9))
                vr = v0.double() + (gi * gi - v0.double()) * (1 - lc.f32(0.999))
                upd = lc.keras_lr_t(1e-4, 0.9, 0.999, t) * mr / (vr.sqrt() + lc.f32(1e-8))
                wd = lc.f32(np.float32(1e-4) * np.float32(0.05))
                pr = (p0.double() - upd) * (1 - wd) if after else p0.double() * (1 - wd) - upd
                p.copy_(pr.float()), m.copy_(mr.float()), v.copy_(vr.float())
            return w_
        good, bad, fn = write(False), write(True), L.adamw_keras
    r_good = run(opt, fn, good, p, g, m, v, **kw)
    p.copy_(p0), m.copy_(m0), v.copy_(v0)
    r_bad = run(opt, fn, bad, p, g, m, v, **kw)
    print(f"[{opt}] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0 and r_bad > 1.0


# ----------------------------------------------------------------------------------------------- bit-exact conversions, dropout
def test_split_to_bf16_and_dropout():
    x = torch.randn(300, 64, generator=gen(117)) * 100
    hi, lo = lc.split_pair(x)
    good = torch.cat([hi, lo], 1)
    bad = torch.cat([hi, (((x - hi.float()) * 1024.0).half())], 1)                     # lo without the 2^11
    assert_pass_and_catch("split_f16x2", L.split_f16x2, lambda ba: good, lambda ba: bad, x)
    rate, seed = 0.1, 5
    y = x * lc.HOOKS["dropout_mask"](tuple(x.shape), rate, seed, "cpu").float()
    shifted = x * lc.HOOKS["dropout_mask"](tuple(x.shape), rate, seed + 1, "cpu").float()
    assert_pass_and_catch("to_bf16", L.to_bf16, lambda ba: (y, y.to(torch.bfloat16)), lambda ba: (y, shifted.to(torch.bfloat16)), x, rate, seed,
                          out_f32=True)
    trunc = (x.view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)
    assert_pass_and_catch("to_bf16", L.to_bf16, lambda ba: x.to(torch.bfloat16), lambda ba: trunc, x)
    sc = float(np.float32(1.0) / np.float32(1.0 - np.float32(rate)))
    keep = torch.rand(x.shape, generator=gen(118)) >= rate
    assert_pass_and_catch("dropout", L.dropout, lambda ba: torch.where(keep, x * sc, torch.zeros_like(x)),
                          lambda ba: torch.where(keep, x / (1 - rate), torch.zeros_like(x)).double().float() * (1 + 2 ** -20), x, rate, seed)
    assert_pass_and_catch("dropout", L.dropout, lambda ba: x.clone(), lambda ba: x * sc, x, 0.0, seed)


# ----------------------------------------------------------------------------------------------- pixels, layouts, glue, losses, quantizer
def _last_changed(t):
    """t with its last element changed (a dropped tail)."""
    b = t.clone()
    flat = b.reshape(-1)
    if b.dtype == torch.uint8:
        flat[-1] = (int(flat[-1]) + 1) % 256
    elif b.dtype == torch.bfloat16 or b.dtype == torch.float16:
        flat[-1] = -flat[-1] if float(flat[-1]) != 0 else 1.0
    elif b.is_floating_point():
        flat[-1] = flat[-1] * 1.01 + 1.0
    else:
        flat[-1] += 1
    return b


def _bitexact_cases():
    g = gen(120)
    u8 = torch.randint(0, 256, (2, 3, 5, 6, 3), generator=g, dtype=torch.uint8)
    x = torch.randn(2, 3, 5, 8, generator=g) * 3
    table, idx = torch.randn(40, 16, generator=g), torch.randint(-2, 45, (70,), generator=g)
    et = torch.randn(64, 32, generator=g)
    ids = torch.randint(-1, 30, (6 * 16,), generator=g, dtype=torch.int32)
    wte, wpe, pose = torch.randn(33, 32, generator=g), torch.randn(16, 32, generator=g), torch.randn(6, 32, generator=g)
    logits = torch.randn(37, 1024, generator=g)
    logits[5, 3] = logits[5, 900] = 50.0                       # a tie: the first index wins
    a8, b8 = torch.randint(0, 256, (3, 8, 8, 3), generator=g, dtype=torch.uint8), torch.randint(0, 256, (3, 8, 8, 3), generator=g, dtype=torch.uint8)
    ar = torch.arange(96)
    emb = torch.where(ids.long() < 0, 0, ids.long())
    k = torch.tensor(1.0 / 255.0, dtype=torch.float32)
    return [
        ("u8_to_unit", L.u8_to_unit, (u8,), dict(first_views=2), (u8[:, :2].reshape(4, 5, 6, 3).float() * k) * 2.0 - 1.0),
        ("unit_to_u8", L.unit_to_u8, (x.clamp(-1.2, 1.2),), {}, ((x.clamp(-1, 1) * 0.5 + 0.5) * 255.5).clamp(0, 255).to(torch.uint8)),
        ("nchw_to_nhwc", L.nchw_to_nhwc, (x,), {}, x.permute(0, 2, 3, 1).contiguous()),
        ("nhwc_to_nchw", L.nhwc_to_nchw, (x,), {}, x.permute(0, 3, 1, 2).contiguous()),
        ("gather_rows", L.gather_rows, (table, idx), {}, table[idx.clamp(0, 39)]),
        ("vq_prepare_codebook_f16", L.vq_prepare_codebook_f16, (et,), {}, (-2.0 * et).half()),
        ("migt_embed", L.migt_embed, (ids, 32, wte, wpe, pose, 6, 16), {}, (wte[torch.where(ids.long() < 0, 32, emb)] + wpe[ar % 16]) + pose[ar // 16]),
        ("argmax_rows", L.argmax_rows, (logits,), {}, torch.argmax(logits, 1)),
        ("image_pair_sums", L.image_pair_sums, (a8, b8), {},
         torch.stack([(a8.long() - b8.long()).abs().reshape(3, -1).sum(1), ((a8.long() - b8.long()) ** 2).reshape(3, -1).sum(1)], 1)),
    ]


@pytest.mark.parametrize("case", range(9))
def test_bit_exact_wrappers(case):
    """The bit-exact checkers accept the restatement and reject it with its last element changed (a dropped tail)."""
    name, fn, a, k, good = _bitexact_cases()[case]
    assert_pass_and_catch(name, fn, lambda ba: good, lambda ba: _last_changed(good), *a, **k)


def test_migt_embed_fixed_token_and_argmax_tie():
    g = gen(121)
    ids = torch.randint(0, 30, (96,), generator=g, dtype=torch.int32)
    wte, wpe, pose = torch.randn(33, 32, generator=g), torch.randn(16, 32, generator=g), torch.randn(6, 32, generator=g)
    ar = torch.arange(96)
    good = (wte[ids.long()] + wpe[ar % 16]) + pose[ar // 16]
    bad = (wte[torch.full((96,), 32)] + wpe[ar % 16]) + pose[ar // 16]
    assert_pass_and_catch("migt_embed", L.migt_embed, lambda ba: good, lambda ba: bad, ids, 32, wte, wpe, pose, 6, 16)
    x = torch.zeros(4, 300)
    x[:, 7] = x[:, 250] = 1.0
    assert_pass_and_catch("argmax_rows", L.argmax_rows, lambda ba: torch.full((4,), 7), lambda ba: torch.full((4,), 250), x)


def test_sumpool_l1_row_mean():
    g = gen(122)
    x = torch.randn(2, 6, 10, 5, generator=g)
    good = x.double().reshape(2, 3, 2, 5, 2, 5).sum((2, 4)).float()
    bad = x.double().reshape(2, 3, 2, 5, 2, 5)[:, :, :, :, :1].sum((2, 4)).float()
    assert_pass_and_catch("sumpool2x2", L.sumpool2x2, lambda ba: good, lambda ba: bad, x)
    a, b = torch.randn(5000, generator=g), torch.randn(5000, generator=g)
    d = b.double() - a.double()
    want = (torch.sign(d).float() * lc.f32(0.25) + 0.0, d.abs().sum().reshape(1))
    assert_pass_and_catch("l1_grad", L.l1_grad, lambda ba: want, lambda ba: (want[0], d[:-1].abs().sum().reshape(1)), a, b, 0.25)
    r = torch.randn(6, 3 * 64, generator=g) + 2.0
    assert_pass_and_catch("row_mean", L.row_mean, lambda ba: r[:, 64:].double().mean(1).float(), lambda ba: r.double().mean(1).float(), r, 64)


def _masked_softmax(sc, rows_per_batch, mode, block, row0=0, shift=0):
    rows, cols = sc.shape
    pos = torch.arange(rows) % rows_per_batch + row0
    vw = (pos // block)[:, None] + shift
    c = torch.arange(cols)[None, :]
    if mode == 1:
        vis = c < ((vw + 1) * block).clamp(max=cols)
    else:
        half = cols // 2
        vis = (c < (vw * block).clamp(max=half)) | ((c >= half + vw * block) & (c < half + (vw + 1) * block))
    return torch.softmax(sc.double().masked_fill(~vis, -math.inf), 1).masked_fill(~vis, 0).float()


@pytest.mark.parametrize("fault", ["mode2_view_off_by_one", "row0_ignored"])
def test_softmax_rows_masks(fault):
    S, blk = 4 * 16, 16
    sc = torch.randn(2 * S, 2 * S, generator=gen(123)) * 3
    kw = dict(rows_total=2 * S, rows_per_batch=S, cols=2 * S, ld_in=2 * S, ld_out=2 * S, block=blk)
    P = torch.empty(2 * S, 2 * S)
    if fault == "mode2_view_off_by_one":
        kw["mask_mode"] = 2
        good, bad = _masked_softmax(sc, S, 2, blk), _masked_softmax(sc, S, 2, blk, shift=1)
    else:
        kw.update(mask_mode=1, row0=blk, cols=2 * S)
        good, bad = _masked_softmax(sc, S, 1, blk, row0=blk), _masked_softmax(sc, S, 1, blk)
    assert_pass_and_catch("softmax_rows", L.softmax_rows, lambda ba: P.copy_(good), lambda ba: P.copy_(bad), sc, P, **kw)


def test_softmax_rows_all_keys_bf16():
    """The shared-scene KV query's softmax (MIGT._query_block): mask mode 0 over S_ctx + 64 columns, 64 rows per batch entry, bf16
    probabilities.  Mutant: the last column (the query view's last own key) masked out."""
    rows, cols = 2 * 2 * 64, 3 * 64 + 64
    sc = torch.randn(rows, cols, generator=gen(125)) * 3
    P = torch.empty(rows, cols, dtype=torch.bfloat16)
    good = torch.softmax(sc.double(), 1).to(torch.bfloat16)
    bad = torch.softmax(sc.double()[:, :-1], 1)
    bad = torch.cat([bad, torch.zeros(rows, 1, dtype=torch.float64)], 1).to(torch.bfloat16)
    kw = dict(rows_total=rows, rows_per_batch=64, cols=cols, ld_in=cols, ld_out=cols)
    assert_pass_and_catch("softmax_rows", L.softmax_rows, lambda ba: P.copy_(good), lambda ba: P.copy_(bad), sc, P, **kw)


def test_cross_entropy_and_pose_losses():
    g = gen(124)
    rows, cols, s = 37, 1024, 0.1
    lg = torch.randn(rows, cols, generator=g) * 3
    lab = torch.randint(0, cols, (rows,), generator=g, dtype=torch.int32)
    x = lg.double()
    lse = torch.logsumexp(x, 1)
    xl = x.gather(1, lab.long()[:, None])[:, 0]
    good = ((1 - lc.f32(s)) * (lse - xl) + lc.f32(s) * (lse - x.mean(1))).float()
    assert_pass_and_catch("cross_entropy_rows", L.cross_entropy_rows, lambda ba: good, lambda ba: (lse - xl).float(), lg, lab, s)
    tpv, views = 16, 5
    raw, poses, w = torch.randn(tpv * views, 7, generator=g), torch.randn(views, 7, generator=g), torch.rand(tpv * views, generator=g)
    y = poses.double().repeat_interleave(tpv, 0)
    m = 2.5
    pos = ((y[:, :3] * lc.f32(m) - raw.double()[:, :3]) ** 2).mean(1).float()
    ori = ((y[:, 3:] - raw.double()[:, 3:]) ** 2).mean(1).float()
    y1 = poses.double().roll(1, 0).repeat_interleave(tpv, 0)                                   # the previous view's pose
    bad = ((y1[:, :3] * lc.f32(m) - raw.double()[:, :3]) ** 2).mean(1).float()
    assert_pass_and_catch("pose_loss_rows", L.pose_loss_rows, lambda ba: (pos, ori), lambda ba: (bad, ori), raw, poses, tpv, m)
    mv = torch.tensor([lc.f32(m)] * 3 + [1.0] * 4, dtype=torch.float64)
    scl = torch.tensor([lc.f32(0.6) * 2 / 3] * 3 + [lc.f32(1.7) * 2 / 4] * 4, dtype=torch.float64)
    gr = (-w.double()[:, None] * scl * (y * mv - raw.double())).float()
    bad = (-w.double()[:, None] * scl * (y - raw.double())).float()                           # multiplier left out
    assert_pass_and_catch("pose_loss_grad", L.pose_loss_grad, lambda ba: gr, lambda ba: bad, raw, poses, w, tpv, m, 0.6, 1.7)
    pp = torch.cat([raw[:, :3].double() / lc.f32(m), lc._quat_unit(raw[:, 3:].double())], 1).float()
    assert_pass_and_catch("pose_postprocess", L.pose_postprocess, lambda ba: pp, lambda ba: torch.cat([pp[:, :3], -pp[:, 3:]], 1), raw, m)


def test_cameras():
    g = gen(125)
    cams = torch.randn(2, 5, 7, generator=g)
    c = cams.double()
    inv = lc._conj(c[:, :1, 3:])
    d = torch.cat([torch.zeros_like(c[..., :1]), c[..., :3] - c[:, :1, :3]], -1)
    p = lc._qmul(lc._qmul(inv.expand(2, 5, 4), d), lc._conj(inv).expand(2, 5, 4))[..., 1:]
    q = lc._quat_unit(lc._qmul(inv.expand(2, 5, 4), c[..., 3:]))
    out = torch.cat([p, q], -1).float()
    tr = cams[:, 0].contiguous()
    bad = torch.cat([(c[..., :3] - c[:, :1, :3]), q], -1).float()                              # translation not rotated
    assert_pass_and_catch("cameras_prepare", L.cameras_prepare, lambda ba: (out, tr), lambda ba: (bad, tr), cams, True)
    t = torch.randn(2, 7, generator=g).double()
    tq = t[:, None, 3:].expand(2, 5, 4)
    pq = torch.cat([torch.zeros_like(c[..., :1]), c[..., :3]], -1)
    back = torch.cat([lc._qmul(lc._qmul(tq, pq), lc._conj(tq))[..., 1:] + t[:, None, :3], lc._qmul(tq, c[..., 3:])], -1).float()
    bad = torch.cat([c[..., :3] + t[:, None, :3], lc._qmul(tq, c[..., 3:])], -1).float()
    assert_pass_and_catch("cameras_from_relative", L.cameras_from_relative, lambda ba: back, lambda ba: bad, cams, t.float())


def test_quantizer_ema_and_commit():
    """EMA statistics with colliding codes; the commitment gradient; the EMA update with a code getting eps twice (codes 0..15 unused,
    so their cluster size is eps-dominated and the doubled eps is an O(1) change)."""
    g = gen(126)
    D, K, m = 16, 64, 600
    z = torch.randn(m, D, generator=g)
    idx = torch.randint(16, K, (m,), generator=g)
    cnt = torch.bincount(idx, minlength=K).float()
    zs = torch.zeros(K, D, dtype=torch.float64).index_add_(0, idx, z.double()).t().float().contiguous()
    bad_zs = zs.clone()
    bad_zs[:, -1] = 0
    assert_pass_and_catch("vq_ema_stats", L.vq_ema_stats, lambda ba: (cnt, zs), lambda ba: (cnt, bad_zs), z, idx, K)
    emb = torch.randn(D, K, generator=g)
    coef = 0.5 / (m * D)
    good = (lc.f32(coef) * (cnt.double() * emb.double() - zs.double())).float()
    assert_pass_and_catch("vq_commit_grad", L.vq_commit_grad, lambda ba: good, lambda ba: (lc.f32(coef) * (emb.double() - zs.double())).float(),
                          emb, cnt, zs, coef, torch.empty(D, K))
    a, corr, eps = 0.01, 1 - 0.99 ** 3, 1e-5
    cs0, dw0 = torch.rand(K, generator=g) * 1e-6, torch.randn(D, K, generator=g)
    cs, dw, e_out, et, esq = cs0.clone(), dw0.clone(), torch.empty(D, K), torch.empty(K, D), torch.empty(K)

    def write(eps2):
        def w_(ba):
            fa, fc, fe = lc.f32(a), lc.f32(corr), lc.f32(eps)
            cs1 = cs0.double() + fa * (cnt.double() - cs0.double())
            n = (cs1 / fc).sum()
            cl = (cs1 / fc + fe * eps2) / (n + K * fe) * n
            dw1 = dw0.double() + fa * (zs.double() - dw0.double())
            e = (dw1 / fc) / cl[None, :]
            cs.copy_(cs1.float()), dw.copy_(dw1.float()), e_out.copy_(e.float()), et.copy_(e_out.t()), esq.copy_((e * e).sum(0).float())
        return w_
    args = (cnt, zs, a, corr, eps, cs, dw, e_out, et, esq)
    r_good = run("vq_ema_update", L.vq_ema_update, write(1.0), *args)
    cs.copy_(cs0), dw.copy_(dw0)
    r_bad = run("vq_ema_update", L.vq_ema_update, write(2.0), *args)
    print(f"[vq_ema_update] clean {r_good:.3g}  mutated {r_bad:.3g}")
    assert r_good <= 1.0 and r_bad > 1.0
    et2 = emb.t().contiguous()
    sq = (emb.double() ** 2).sum(0).float()
    assert_pass_and_catch("vq_prepare_codebook", L.vq_prepare_codebook, lambda ba: (et2, sq), lambda ba: (et2, (emb.double()[:-1] ** 2).sum(0).float()), emb)


def _torch_resize(x, size, method):
    v = x.permute(0, 3, 1, 2).float() / 255.0
    if method == "nearest":
        y = F.interpolate(v, size=(size, size), mode="nearest")
    else:
        y = F.interpolate(v, size=(size, size), mode="bilinear", align_corners=False)
    return (y.clamp(0, 1) * 255.0).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("method,hw", [pytest.param("nearest", None, id="nearest"), pytest.param("bilinear", None, id="bilinear")]
                         + [pytest.param(None, hw, id=f"{hw[0]}x{hw[1]}") for hw in ((96, 160), (160, 96), (128, 200), (200, 128), (480, 640))])
def test_resize_u8(method, hw):
    """The fp64 restatement accepts torch's uint8 resize of the same image (nearest: F.interpolate; bilinear: the same formula) and rejects
    the image shifted by one source row.  Non-square frames to 128 under the default rule: the method follows the height (96 x 160 grows
    with nearest, 160 x 96 shrinks bilinearly), and a width-keyed choice is rejected; 128 x 200 and 200 x 128 must come back as the input
    itself, and a resized copy is rejected."""
    g = gen(127)
    if hw is None:
        h = 48 if method == "bilinear" else 12
        x = torch.randint(0, 256, (2, h, h, 3), generator=g, dtype=torch.uint8)
        size = 32
        good = _torch_resize(x, size, method)
        assert_pass_and_catch("resize_u8", L.resize_u8, lambda ba: good, lambda ba: torch.roll(good, 1, 1), x, size, method)
        return
    h, w = hw
    x = torch.randint(0, 256, (2, h, w, 3), generator=g, dtype=torch.uint8)
    size = 128
    by_w = _torch_resize(x, size, "nearest" if size > w else "bilinear")
    if size in (h, w):
        assert_pass_and_catch("resize_u8", L.resize_u8, lambda ba: ba["x_u8"], lambda ba: by_w, x, size)
        return
    good = _torch_resize(x, size, "nearest" if size > h else "bilinear")
    bad = torch.roll(good, 1, 1) if (size > h) == (size > w) else by_w
    assert_pass_and_catch("resize_u8", L.resize_u8, lambda ba: good, lambda ba: bad, x, size)


# ----------------------------------------------------------------------------------------------- SSIM
def _ssim_ld(a, b, k1=0.01, k2=0.03):
    """ssim() (metrics.py:17-73) in numpy long double, in the reference's own order: 1/49 box means of X = x / 255, X^2, XY, then
    49/48 (E[XY] - E[X] E[Y]).  Long double carries 64 significant bits, so a flat window's cancellation costs ~1e-17 of S."""
    assert np.finfo(np.longdouble).nmant >= 63
    from numpy.lib.stride_tricks import sliding_window_view
    X, Y = a.numpy().astype(np.longdouble) / 255, b.numpy().astype(np.longdouble) / 255
    box = lambda t: sliding_window_view(t, (7, 7), axis=(1, 2)).sum((-2, -1)) / 49
    ux, uy, uxx, uyy, uxy = box(X), box(Y), box(X * X), box(Y * Y), box(X * Y)
    cn = np.longdouble(49) / 48
    vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
    C1, C2 = np.longdouble(float(k1) * float(k1)), np.longdouble(float(k2) * float(k2))        # fp64 K^2, as the kernel takes it
    S = (2 * ux * uy + C1) * (2 * vxy + C2) / ((ux * ux + uy * uy + C1) * (vx + vy + C2))
    return torch.from_numpy(S.reshape(S.shape[0], -1).mean(1).astype(np.float64))


def _ssim_f32(a, b, k1=0.01, k2=0.03):
    """The parent kernel's arithmetic in torch fp32: exact window sums, then means, E[x^2] - E[x]^2 and S one fp32 operation at a time."""
    sx, sy, sxx, syy, sxy = (lc.box7(t).float() for t in (a, b, a.long() * a.long(), b.long() * b.long(), a.long() * b.long()))
    d1, d2, cn = 49.0 * 255.0, 49.0 * 65025.0, torch.tensor(49.0 / 48.0, dtype=torch.float32)
    ux, uy, uxx, uyy, uxy = sx / d1, sy / d1, sxx / d2, syy / d2, sxy / d2
    vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
    C1, C2 = lc.f32(lc.f32(k1) * lc.f32(k1)), lc.f32(lc.f32(k2) * lc.f32(k2))
    S = ((2.0 * ux * uy + C1) * (2.0 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2))
    return S.double().reshape(S.shape[0], -1).mean(1)


def test_ssim_u8_flat_level_pairs_and_fp32_moments():
    """Flat images at level pairs 1 to 3 apart: the variances are exactly 0 and C2 dominates B2, so the fp32 E[x^2] - E[x]^2 of the
    parent kernel leaves ~1e-4 in S (199 / 196, 224 / 223 are the worst) in every window alike.  The long-double restatement passes
    (K1 = 0.01 and the Evaluator's K1 = 1), the fp32 one is caught."""
    pairs = [(199, 196), (224, 223), (100, 101), (37, 40), (255, 254), (1, 0), (128, 128)]
    a = torch.tensor([p[0] for p in pairs], dtype=torch.uint8)[:, None, None, None].expand(-1, 9, 11, 1).contiguous()
    b = torch.tensor([p[1] for p in pairs], dtype=torch.uint8)[:, None, None, None].expand(-1, 9, 11, 1).contiguous()
    for k1 in (0.01, 1.0):
        good, bad = _ssim_ld(a, b, k1), _ssim_f32(a, b, k1)
        print(f"[ssim flat K1={k1}] fp32 moments off by {float((bad - good).abs().max()):.3g}")
        assert_pass_and_catch("ssim_u8", L.ssim_u8, lambda ba: good, lambda ba: bad, a, b, k1=k1)


def test_ssim_u8_windows_channels_images_constants():
    """Noisy synthetic pairs 13 x 29 x 3: the long-double restatement passes; dropping the last row or the last column of windows,
    pairing a's channel 0 with b's channel 1, swapping the two images' results, or using K1 = 0.01 where 1 was asked are caught."""
    from oracle import synth
    g = gen(131)
    a = synth.make_images_uint8(1, 2, size=32, seed=7)[0][:, :13, :29].contiguous()
    b = (a.int() + torch.randint(-30, 31, a.shape, generator=g)).clamp(0, 255).to(torch.uint8)
    good = _ssim_ld(a, b)
    mutants = {"last window row": _ssim_ld(a[:, :-1], b[:, :-1]), "last window column": _ssim_ld(a[:, :, :-1], b[:, :, :-1]),
               "channels": _ssim_ld(a, b[..., [1, 0, 2]]), "images": good[[1, 0]]}
    for name, bad in mutants.items():
        print(f"[ssim {name}]", end=" ")
        assert_pass_and_catch("ssim_u8", L.ssim_u8, lambda ba: good, lambda ba: bad, a, b)
    assert_pass_and_catch("ssim_u8", L.ssim_u8, lambda ba: _ssim_ld(a, b, 1.0), lambda ba: good, a, b, k1=1.0)
    assert_pass_and_catch("ssim_u8", L.ssim_u8, lambda ba: _ssim_ld(a, b, 0.01, 0.1), lambda ba: good, a, b, k2=0.1)


def test_ssim_u8_rejects_mismatched_images_before_any_launch(monkeypatch):
    """a and b of different shapes (a smaller b would be read past its end by the kernel): a ValueError before the library is called."""
    calls = []

    class Lib:
        def __getattr__(self, name):
            return lambda *args: calls.append(name) or 0
    monkeypatch.setattr(L, "load", lambda require_device=False: Lib())
    a = torch.zeros(2, 16, 16, 3, dtype=torch.uint8)
    for b in (torch.zeros(2, 8, 16, 3, dtype=torch.uint8), torch.zeros(2, 16, 15, 3, dtype=torch.uint8), torch.zeros(1, 16, 16, 3, dtype=torch.uint8),
              torch.zeros(2, 16, 16, 1, dtype=torch.uint8), a[0]):
        for k1 in (None, 1.0):
            with pytest.raises(ValueError, match="one shape"):
                L.ssim_u8(a, b, k1=k1)
            with pytest.raises(ValueError, match="one shape"):
                L.ssim_u8(b, a, k1=k1)
    assert not calls
