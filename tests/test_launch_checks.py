"""The launch checkers of tests/launch_checks.py on the CPU: each accepts an output computed by an independent fp64 restatement rounded to the
output dtype, and rejects that output with one named fault put in (a dropped tap, a residual read one row off, a zeroed tail tile, a shifted
column window, a zeroed last image, swapped heads, a missing max rescale, a shifted dropout mask, swapped stream gradients, an index off by
one).  So a checker that stopped looking at part of its output would fail here, before any GPU run."""
import math
import random

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
    # causal QK^T: only visible columns are compared
    S, blk = 256, 64
    q, k = torch.randn(S, 64, generator=gen(11)).bfloat16(), torch.randn(S, 64, generator=gen(12)).bfloat16()
    sc = torch.empty(S, S)
    full = (q.double() @ k.double().t()).float()
    vis = (torch.arange(S)[None, :] // blk) <= (torch.arange(S)[:, None] // blk)

    def hidden_garbage(ba):
        return sc.copy_(torch.where(vis, full, torch.full_like(full, 1e30)))

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
@pytest.mark.parametrize("name", ["vq_lookup", "vq_lookup_fused", "vq_lookup_tc"])
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
    extra = {"vq_lookup": (), "vq_lookup_fused": (et.bfloat16(),), "vq_lookup_tc": (et.bfloat16(),)}[name]
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
    """Every _lib function that launches a GEMM, conv, attention, weight-gradient or lookup kernel, or calls a checked wrapper (the
    tensor-core weight gradients and lookup do), has a checker: a new wrapper cannot bypass the launch audit."""
    import inspect
    import re
    pat = re.compile(r"^(vf_(tc_gemm|simt_gemm|attn_\w+|conv_wgrad|conv3x3_small_\w+|vq_lookup\w*)|tc_gemm|_wgrad_tc)$")
    public = {name for name, fn in vars(L).items() if inspect.isfunction(fn) and fn.__module__ == L.__name__ and not name.startswith("_")
              and any(pat.match(n) for n in fn.__code__.co_names)}
    assert {"tc_gemm", "tc_conv", "vq_lookup_tc", "conv_wgrad_bf16", "attn_multiend_bwd", "conv3x3_small_cin"} <= public
    missing = sorted(public - set(lc.CHECKERS))
    print(f"[completeness] {len(public)} launching wrappers: {sorted(public)}")
    assert not missing, f"_lib wrappers that launch checked kernels without a checker in tests/launch_checks.py: {missing}"
