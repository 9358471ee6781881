"""Backward-pass and optimizer kernels (GPU) against fp64 computations of the same operation on the CPU.

Every reduction is held to a worst-case bound that holds for any summation or atomic order: |err| <= c K u sum|terms| element-wise, with
K the number of terms added into that output, u = 2^-24 and sum|terms| computed in fp64 from the same inputs.  The structural cases keep
K u << 1, so a missing term or a wrong index lands orders of magnitude above the bar; where an edge of the kernel's tiling lives (the last
pixel chunk, the tail rows, the border taps, the last channel of a partial tile) the inputs are made large, so that dropping it is an O(1)
relative error.  The few large cases that exist to run the chunking / grid-stride logic use c sqrt(K) u sum|terms| instead, a statistical
bar (random-order rounding errors grow as sqrt(K)); their docstrings say so.  Elementwise kernels get a few ulps plus an absolute floor.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def gen(seed):
    return torch.Generator().manual_seed(seed)


def check(name, got, want, bar):
    """Element-wise |got - want| <= bar; prints the worst ratio error / bar."""
    got, want, bar = got.double().cpu(), want.double().cpu(), bar.double().cpu().expand_as(want)
    err = (got - want).abs()
    ratio = err / bar.clamp_min(1e-300)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    i = int(ratio.argmax()) if ratio.numel() else 0
    print(f"[{name}] worst err/bar {worst:.3e} (max err {float(err.max()):.3e}; at {i}: err {float(err.reshape(-1)[i]):.3e} "
          f"bar {float(bar.reshape(-1)[i]):.3e})")
    assert worst <= 1.0, f"{name}: error {worst:.3e} x the bar at flat index {i} (got {float(got.reshape(-1)[i])!r}, want {float(want.reshape(-1)[i])!r})"


def f32(x):
    """A hyperparameter as the kernels see it (passed as a C float), in fp64."""
    return float(np.float32(x))


def keras_lr_t(lr, b1, b2, t):
    """lr sqrt(1 - b2^t) / (1 - b1^t) evaluated in fp32, as vf_adamw_keras does on the host and TF 2.4's Adam does for fp32 variables.  1 - b2^t
    cancels (b2 = 0.999), so an fp64 evaluation differs by up to u / (1 - b2^t), 3e-5 relative at t = 2: more than the optimizer bars."""
    one = np.float32(1.0)
    return float(np.float32(lr) * np.sqrt(one - np.float32(b2) ** np.float32(t)) / (one - np.float32(b1) ** np.float32(t)))


# ----------------------------------------------------------------------------- convolution weight / data gradients
def _conv_ref(x, dy, cout, kh, stride, pad, upsample):
    """fp64 dW of the convolution the trainer runs, in the kernel layout [kh*kh*Cin, Cout] (k = tap * Cin + c); x NHWC, dy NHWC."""
    xd = x.double().permute(0, 3, 1, 2)
    if upsample:
        xd = F.interpolate(xd, scale_factor=2, mode="nearest")
    if stride == 2:                                          # the reference Downsample: pad right / bottom by one, then a valid conv
        xd = F.pad(xd, (0, 1, 0, 1))
    wt = torch.zeros(cout, x.shape[-1], kh, kh, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(xd, wt, stride=stride, padding=pad[0] if stride == 1 else 0)
    assert tuple(y.shape[2:]) == tuple(dy.shape[1:3])
    y.backward(dy.double().permute(0, 3, 1, 2))
    return wt.grad.permute(2, 3, 1, 0).reshape(kh * kh * x.shape[-1], cout)


CONV_WGRAD_CASES = [
    # n, h, w, cin, cout, kh, stride, upsample
    (2, 12, 10, 3, 16, 3, 1, False),          # conv_in: Cin = 3
    (2, 12, 10, 16, 32, 3, 1, False),         # partial 64-wide tiles on both sides
    (2, 12, 10, 32, 96, 3, 1, False),
    (2, 12, 10, 96, 128, 3, 1, False),
    (2, 12, 10, 128, 3, 3, 1, False),         # conv_out: Cout = 3
    (2, 24, 24, 64, 64, 3, 1, False),         # 1152 pixels: five chunks of 256, the last one partial (multi-chunk atomics)
    (2, 8, 8, 32, 48, 3, 2, False),           # Downsample, even map (the padded bottom / right taps are cut by the bounds check)
    (2, 9, 7, 32, 48, 3, 2, False),           # Downsample, odd map (the last row / column are real taps)
    (2, 6, 5, 16, 32, 3, 1, True),            # Upsample: nearest x2, then the conv
]


@pytest.mark.parametrize("n,h,w,cin,cout,kh,stride,upsample", CONV_WGRAD_CASES)
def test_conv_wgrad_cuda_cores(L, n, h, w, cin, cout, kh, stride, upsample):
    """vf_conv_wgrad (CUDA-core atomics) == fp64 autograd dW of conv2d (stride 2: F.pad(x, (0,1,0,1)) then the stride-2 conv; upsample:
    nearest x2 then the conv), accumulated onto what dw held.  K = output pixels per weight; the border rows / columns of x and the last 16
    output pixels of dy are large, so a missed boundary tap or a dropped tail chunk is an O(1) error."""
    gg = gen(1000 + 7 * cin + cout + h + stride)
    x = torch.randn(n, h, w, cin, generator=gg)
    x[:, -1] *= 30.0
    x[:, :, -1] *= 30.0
    x[:, 0] *= 10.0
    vh, vw = (2 * h, 2 * w) if upsample else (h, w)
    oh, ow = (vh // 2, vw // 2) if stride == 2 else (vh, vw)
    dy = torch.randn(n, oh, ow, cout, generator=gg)
    dy.reshape(-1, cout)[-16:] *= 100.0
    pad = (1, 1) if stride == 1 else (0, 0)
    want = _conv_ref(x, dy, cout, kh, stride, pad, upsample)
    absum = _conv_ref(x.abs(), dy.abs(), cout, kh, stride, pad, upsample)
    d0 = torch.randn(kh * kh * cin, cout, generator=gg)
    dw = d0.cuda()
    L.conv_wgrad(x.cuda(), dy.cuda(), dw, kh=kh, stride=stride, pad=pad, upsample=upsample)
    K = n * oh * ow
    check(f"conv_wgrad n{n} {h}x{w} {cin}->{cout} k{kh} s{stride} up{int(upsample)} K={K}", dw, d0.double() + want,
          2 * K * U * absum + 2 * U * (d0.double().abs() + want.abs()))


@pytest.mark.parametrize("k,n,so", [(96, 160, "nk"), (128, 7, "kn")])
def test_conv_wgrad_linear_layouts(L, k, n, so):
    """The 1x1 / Linear weight gradients: ``so=(1, k)`` writes dW as [out, in] (VQGAN's nin_shortcut, quant_conv, attention projections),
    ``so=(n, 1)`` as [in, out] (the transformer's Conv1D layers and, with (d, 1), its tied head).  fp64 x^T dy; 300 rows (two chunks),
    the last rows large."""
    gg = gen(k + n)
    m = 300
    x = torch.randn(m, k, generator=gg)
    dy = torch.randn(m, n, generator=gg)
    dy[-5:] *= 100.0
    want = x.double().t() @ dy.double()
    absum = x.double().abs().t() @ dy.double().abs()
    if so == "nk":
        want, absum, stride = want.t(), absum.t(), (1, k)
    else:
        stride = (n, 1)
    d0 = torch.randn(want.shape, generator=gg)
    dw = d0.cuda()
    L.conv_wgrad(x.reshape(1, m, 1, k).cuda(), dy.reshape(1, m, 1, n).cuda(), dw, kh=1, pad=(0, 0), so=stride)
    check(f"conv_wgrad 1x1 so={stride} m{m} {k}->{n}", dw, d0.double() + want, 2 * m * U * absum + 2 * U * (d0.double().abs() + want.abs()))


@pytest.mark.parametrize("m,k,n", [(200, 128, 128), (1000, 256, 128), (333, 128, 256), (1500, 768, 3072)])
def test_dense_wgrad_tc(L, m, k, n):
    """dense_wgrad_tc (exact split-fp16 GEMM over the row axis, split-K, vf_sum_splits) == fp64 x^T dy; m is not a multiple of 64 nor of the
    split length, and the last rows are large (the tail of the last split).  accumulate=True adds onto dw, accumulate=False overwrites it."""
    gg = gen(m + k + n)
    x = torch.randn(m, k, generator=gg)
    dy = torch.randn(m, n, generator=gg)
    x[-3:] *= 50.0
    want = x.double().t() @ dy.double()
    bar = 2 * m * U * (x.double().abs().t() @ dy.double().abs())
    d0 = torch.randn(k, n, generator=gg)
    dw = d0.cuda()
    L.dense_wgrad_tc(x.cuda(), dy.cuda(), dw, accumulate=True)
    check(f"dense_wgrad_tc m{m} {k}x{n} accumulate", dw, d0.double() + want, bar + 2 * U * (d0.double().abs() + want.abs()))
    dw = torch.full((k, n), float("nan"), device="cuda")
    L.dense_wgrad_tc(x.cuda(), dy.cuda(), dw, accumulate=False)
    check(f"dense_wgrad_tc m{m} {k}x{n} overwrite", dw, want, bar)


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 8, 8, 32, 48), (2, 9, 7, 48, 32), (1, 5, 11, 16, 64)])
def test_simt_conv_dgrad_s2(L, n, h, w, cin, cout):
    """simt_conv_dgrad_s2 == fp64 autograd dx of the Downsample conv (F.pad(x, (0,1,0,1)), 3x3 stride 2), even and odd maps, Cin != Cout.
    K = 9 Cout terms per dx element; the last output row / column of dy are large (they reach the last input row / column)."""
    gg = gen(n + h + w + cin)
    wt = torch.randn(cout, cin, 3, 3, generator=gg, dtype=torch.float64)
    w_kn = wt.permute(2, 3, 1, 0).reshape(9 * cin, cout).float()            # the trainer's conv layout [tap * Cin + c, Cout]
    oh, ow = h // 2, w // 2
    dy = torch.randn(n, oh, ow, cout, generator=gg)
    dy[:, -1] *= 30.0
    dy[:, :, -1] *= 30.0

    def ref(wd, dyd):
        x = torch.zeros(n, cin, h, w, dtype=torch.float64, requires_grad=True)
        F.conv2d(F.pad(x, (0, 1, 0, 1)), wd, stride=2).backward(dyd.permute(0, 3, 1, 2))
        return x.grad.permute(0, 2, 3, 1)

    want = ref(w_kn.double().reshape(3, 3, cin, cout).permute(3, 2, 0, 1), dy.double())
    absum = ref(w_kn.double().abs().reshape(3, 3, cin, cout).permute(3, 2, 0, 1), dy.double().abs())
    wd = w_kn.reshape(3, 3, cin, cout).permute(0, 1, 3, 2).reshape(9 * cout, cin).contiguous()      # as VQGANTrainer._conv_bw builds it
    dx = L.simt_conv_dgrad_s2(dy.cuda(), wd.cuda(), (h, w))
    check(f"simt_conv_dgrad_s2 n{n} {h}x{w} {cout}->{cin}", dx, want, 2 * 9 * cout * U * absum)


# ----------------------------------------------------------------------------- reductions
@pytest.mark.parametrize("rows,C", [(1, 37), (7, 37), (1023, 37), (1025, 100), (1024 * 1024 + 3, 5)])
def test_col_sums(L, rows, C):
    """vf_col_sums == fp64 column sums, added onto ``out``; C is not a multiple of 32 and the last row is large.  The 1M-row case
    (1024 row chunks of 1025 rows, atomics across them) is held to the statistical bar 2 sqrt(K) u sum|x|; the others to 2 K u sum|x|."""
    gg = gen(rows + C)
    x = torch.randn(rows, C, generator=gg)
    x[-1] *= 1000.0
    o0 = torch.randn(C, generator=gg)
    out = o0.cuda()
    L.col_sums(x.cuda(), out)
    absum = x.double().abs().sum(0)
    kf = math.sqrt(rows) if rows > 1 << 20 else rows
    check(f"col_sums rows{rows} C{C}", out, o0.double() + x.double().sum(0), 2 * kf * U * absum + 2 * U * o0.double().abs())


def _gn_ref(x, dout, gamma, beta, groups, swish, eps=1e-6):
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    ga = gamma.double().requires_grad_(True)
    be = beta.double().requires_grad_(True)
    y = F.group_norm(xd, groups, ga, be, eps)
    if swish:
        y = y * torch.sigmoid(y)
    y.backward(dout.double().permute(0, 3, 1, 2))
    return xd.grad.permute(0, 2, 3, 1), ga.grad, be.grad


@pytest.mark.parametrize("n,hw,C,swish,add", [(2, 35, 32, True, False), (2, 35, 64, False, True), (3, 1, 128, True, True),
                                              (2, 63, 512, True, False), (1, 4099, 128, True, True)])
def test_groupnorm_bwd(L, n, hw, C, swish, add):
    """vf_groupnorm_bwd == fp64 autograd through F.group_norm(32) (+ swish): dx (+ add), and dgamma / dbeta added onto what they held.
    The kernel is given the fp64 statistics rounded to fp32.  C = 32 is one channel per group; HW odd and HW = 1.  The last pixel's dout is
    large, so a dropped tail pixel moves the group sums by O(1).  Bars: the group sums have K = HW C/32 terms, dgamma / dbeta K = N HW;
    sum|terms| includes the rounding of the mean (|mean| rstd) and of the swish derivative."""
    groups = 32
    gg = gen(n * 1000 + hw + C)
    x = torch.randn(n, hw, 1, C, generator=gg) * 2.0 + 0.5
    dout = torch.randn(n, hw, 1, C, generator=gg)
    dout[:, -1] *= 20.0
    gamma = torch.rand(C, generator=gg) + 0.5
    beta = torch.randn(C, generator=gg) * 0.3
    addt = torch.randn(n, hw, 1, C, generator=gg) if add else None
    xg = x.double().reshape(n, hw, groups, C // groups)
    mu = xg.mean((1, 3))
    rs = 1.0 / torch.sqrt(xg.var((1, 3), unbiased=False) + 1e-6)
    mr = torch.stack([mu, rs], -1).float()
    dx_w, dg_w, db_w = _gn_ref(x, dout, gamma, beta, groups, swish)
    if add:
        dx_w = dx_w + addt.double()
    dg0, db0 = torch.randn(C, generator=gg), torch.randn(C, generator=gg)
    dgam, dbet = dg0.cuda(), db0.cuda()
    dx = L.groupnorm_bwd(x.cuda(), dout.cuda(), mr.cuda(), gamma.cuda(), beta.cuda(), dgam, dbet, swish=swish,
                         add=addt.cuda() if add else None)
    # sum|terms| in fp64: g = dL/d(normalised) before gamma, xh the normalised input
    cidx = torch.arange(C) // (C // groups)
    mu_c, rs_c = mu[:, cidx].reshape(n, 1, 1, C), rs[:, cidx].reshape(n, 1, 1, C)
    xh = (x.double() - mu_c) * rs_c
    g = dout.double()
    if swish:
        z = xh * gamma.double() + beta.double()
        sg = torch.sigmoid(z)
        g = g * sg * (1 + z * (1 - sg))
    xh_err = xh.abs() + rs_c * mu_c.abs() + 1.0
    dgg = (g * gamma.double()).abs()
    A1 = dgg.reshape(n, hw, groups, -1).mean((1, 3))[:, cidx].reshape(n, 1, 1, C)
    A2 = (dgg * xh_err).reshape(n, hw, groups, -1).mean((1, 3))[:, cidx].reshape(n, 1, 1, C)
    Kg = hw * (C // groups)
    s_dx = rs_c * (dgg * xh_err + A1 + xh_err * A2) + (addt.double().abs() if add else 0.0)
    check(f"groupnorm_bwd dx n{n} hw{hw} C{C} swish{int(swish)} add{int(add)}", dx, dx_w, 4 * (Kg + 8) * U * s_dx)
    Kc = n * hw
    s_dg = (g.abs() * xh_err).sum((0, 1, 2))
    check(f"groupnorm_bwd dgamma n{n} hw{hw} C{C}", dgam, dg0.double() + dg_w, 4 * (Kc + 8) * U * s_dg + 2 * U * dg0.double().abs())
    check(f"groupnorm_bwd dbeta n{n} hw{hw} C{C}", dbet, db0.double() + db_w, 4 * (Kc + 8) * U * g.abs().sum((0, 1, 2)) + 2 * U * db0.double().abs())


@pytest.mark.parametrize("rows,D,add", [(37, 4, False), (37, 96, True), (21, 768, False), (13, 1024, True), (13, 3072, True)])
def test_layernorm_bwd(L, rows, D, add):
    """vf_layernorm_bwd == fp64 autograd through F.layer_norm (eps 1e-5): dx (+ add) and dgamma / dbeta added onto what they held.  The
    kernel recomputes the row statistics in fp32 (K = D terms); rows is not a multiple of 8 and the last row is large."""
    gg = gen(rows * 7 + D)
    x = torch.randn(rows, D, generator=gg) * 1.5 + 0.3
    dy = torch.randn(rows, D, generator=gg)
    dy[-1] *= 50.0
    gamma = torch.rand(D, generator=gg) + 0.5
    addt = torch.randn(rows, D, generator=gg) if add else None
    xd = x.double().requires_grad_(True)
    gd = gamma.double().requires_grad_(True)
    bd = torch.zeros(D, dtype=torch.float64, requires_grad=True)
    F.layer_norm(xd, (D,), gd, bd, 1e-5).backward(dy.double())
    dx_w = xd.grad + (addt.double() if add else 0.0)
    dg0, db0 = torch.randn(D, generator=gg), torch.randn(D, generator=gg)
    dgam, dbet = dg0.cuda(), db0.cuda()
    dx = L.layernorm_bwd(x.cuda(), dy.cuda(), gamma.cuda(), dgam, dbet, eps=1e-5, add=addt.cuda() if add else None)
    mu = x.double().mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(x.double().var(1, unbiased=False, keepdim=True) + 1e-5)
    xh = (x.double() - mu) * rs
    xh_err = xh.abs() + rs * (x.double().abs().mean(1, keepdim=True)) + 1.0        # the fp32 mean / rstd carry K = D rounding errors
    dgg = (dy.double() * gamma.double()).abs()
    s_dx = rs * (dgg * xh_err + dgg.mean(1, keepdim=True) + xh_err * (dgg * xh_err).mean(1, keepdim=True)) + (addt.double().abs() if add else 0.0)
    check(f"layernorm_bwd dx rows{rows} D{D} add{int(add)}", dx, dx_w, 4 * (D + 8) * U * s_dx)
    K = rows + D
    check(f"layernorm_bwd dgamma rows{rows} D{D}", dgam, dg0.double() + gd.grad, 4 * K * U * (dy.double().abs() * xh_err).sum(0) + 2 * U * dg0.double().abs())
    check(f"layernorm_bwd dbeta rows{rows} D{D}", dbet, db0.double() + bd.grad, 4 * K * U * dy.double().abs().sum(0) + 2 * U * db0.double().abs())


@pytest.mark.parametrize("cols", [1, 31, 33, 640])
def test_softmax_bwd_rows(L, cols):
    """vf_softmax_bwd_rows == fp64 P (dP - sum_j P_j dP_j) on the same fp32 P, dP; one warp per row, so cols 31 / 33 / 640 cover a partial
    lane, one spare lane and a long row.  The last column of dP is large.  K = cols terms in the row sum."""
    gg = gen(cols)
    rows = 37
    P = torch.softmax(torch.randn(rows, cols, generator=gg) * 2.0, -1)
    dP = torch.randn(rows, cols, generator=gg)
    dP[:, -1] *= 100.0
    Pd, dPd = P.double(), dP.double()
    s = (Pd * dPd).sum(-1, keepdim=True)
    want = Pd * (dPd - s)
    bar = 2 * (cols + 2) * U * Pd * (dPd.abs() + (Pd * dPd).abs().sum(-1, keepdim=True))
    dS = L.softmax_bwd_rows(P.cuda(), dP.cuda())
    check(f"softmax_bwd_rows cols{cols}", dS, want, bar)
    if cols == 1:
        assert torch.equal(dS.cpu(), torch.zeros_like(dS.cpu()))


def test_gelu_and_gelu_bwd(L):
    """vf_gelu_fwd / vf_gelu_bwd == fp64 erf GELU x Phi(x) and its derivative Phi(x) + x phi(x), for |x| <= 10 and +-0.  Bars: 4 ulps of the
    result plus an absolute floor of 4 u |x| (erff's 2-ulp error on 1 + erf, which cancels for negative x) and 4 u |dy| for the derivative."""
    gg = gen(5)
    x = torch.cat([torch.linspace(-10, 10, 4001), torch.tensor([0.0, -0.0, 1e-30, -1e-30, 6.0, -6.0]), torch.randn(1000, generator=gg) * 3])
    dy = torch.randn(x.shape, generator=gg)
    xd = x.double()
    cdf = 0.5 * (1 + torch.erf(xd / math.sqrt(2)))
    pdf = torch.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi)
    y = L.gelu(x.cuda())
    check("gelu", y, xd * cdf, 4 * U * (xd * cdf).abs() + 4 * U * xd.abs() + 1e-38)
    dx = L.gelu_bwd(x.cuda(), dy.cuda())
    want = dy.double() * (cdf + xd * pdf)
    check("gelu_bwd", dx, want, 4 * U * want.abs() + 4 * U * dy.double().abs() * (1 + (xd * pdf).abs()))
    yc = y.cpu()
    assert float(yc[4001]) == 0.0 and float(yc[4002]) == 0.0


@pytest.mark.parametrize("n", [1000, 132 * 16 * 256 + 1000])
def test_l1_grad(L, n):
    """vf_l1_grad: dy = scale sign(y - x) exactly (0 where y == x) and loss_sum == fp64 sum |y - x| (bar: the fp32 subtraction, u/2 per term,
    with fp64 accumulation).  n is not a multiple of 256; the large n exceeds the grid (grid-stride loop); the last element is large."""
    gg = gen(n)
    x = torch.randn(n, generator=gg)
    y = torch.randn(n, generator=gg)
    tie = torch.rand(n, generator=gg) < 0.1
    tie[-1] = False
    y[tie] = x[tie]
    y[-1] = x[-1] + 1e4
    scale = 1.0 / 3.0
    dy, ls = L.l1_grad(x.cuda(), y.cuda(), scale)
    d = y.double() - x.double()
    want = torch.sign(d) * f32(scale)
    assert torch.equal(dy.cpu().double(), want), "l1_grad: gradient is not scale * sign(y - x)"
    assert int((dy.cpu() == 0).sum()) == int(tie.sum())
    check(f"l1_grad loss_sum n{n}", ls, d.abs().sum().reshape(1), torch.tensor([(U + n * 2.0 ** -53) * float(d.abs().sum())]))


@pytest.mark.parametrize("use_y,use_z", [(True, True), (True, False), (False, True), (False, False)])
def test_lincomb3(L, use_y, use_z):
    """vf_lincomb3 == fp64 a x + b y + c z with y and / or z null (their terms dropped).  Bar 4 u sum|terms|: the product and the two fmas
    each round once (3 u sum|terms| at worst)."""
    gg = gen(int(use_y) * 2 + int(use_z))
    n = 1000
    x, y, z = (torch.randn(n, generator=gg) for _ in range(3))
    a, b, c = 0.7, -1.3, 2.5e-3
    out = L.lincomb3(a, x.cuda(), b, y.cuda() if use_y else None, c, z.cuda() if use_z else None)
    terms = [f32(a) * x.double()] + ([f32(b) * y.double()] if use_y else []) + ([f32(c) * z.double()] if use_z else [])
    check(f"lincomb3 y{int(use_y)} z{int(use_z)}", out, sum(terms), 4 * U * sum(t.abs() for t in terms) + 1e-38)


@pytest.mark.parametrize("n,H,W,C", [(2, 3, 5, 3), (1, 7, 1, 64)])
def test_sumpool2x2(L, n, H, W, C):
    """vf_sumpool2x2 (backward of the nearest x2 upsample) == fp64 sum over each 2x2 window; odd pooled sizes, C = 3."""
    gg = gen(H * W + C)
    x = torch.randn(n, 2 * H, 2 * W, C, generator=gg)
    y = L.sumpool2x2(x.cuda())
    xw = x.double().reshape(n, H, 2, W, 2, C)
    check(f"sumpool2x2 {H}x{W}x{C}", y, xw.sum((2, 4)), 2 * 4 * U * xw.abs().sum((2, 4)))


@pytest.mark.parametrize("with_ids", [True, False])
def test_migt_embed_bwd(L, with_ids):
    """vf_migt_embed_bwd == fp64 index_add_: dwte[id] += dh (ids repeat, so the atomics collide; ids=None scatters everything to
    fixed_token), dwpe[l] += dh, dpose[bt] += dh (or no dpose).  All three accumulate onto what they held."""
    gg = gen(int(with_ids))
    BT, Lt, d, V = 6, 16, 96, 40
    dh = torch.randn(BT * Lt, d, generator=gg)
    ids = torch.randint(0, 5, (BT * Lt,), generator=gg, dtype=torch.int32)       # 5 ids over 96 tokens: heavy repeats
    fixed = 37
    w0, p0, q0 = torch.randn(V, d, generator=gg), torch.randn(Lt, d, generator=gg), torch.randn(BT, d, generator=gg)
    dwte, dwpe = w0.cuda(), p0.cuda()
    dpose = q0.cuda() if with_ids else None
    L.migt_embed_bwd(dh.cuda(), ids.cuda() if with_ids else None, fixed, BT, Lt, dwte, dwpe, dpose)
    idx = ids.long() if with_ids else torch.full((BT * Lt,), fixed, dtype=torch.long)
    hd, ha = dh.double(), dh.double().abs()
    rows_l = torch.arange(BT * Lt) % Lt
    rows_bt = torch.arange(BT * Lt) // Lt

    def acc(base, index, v):
        return base.double().index_add_(0, index, v)

    K = BT * Lt
    check("migt_embed_bwd dwte", dwte, acc(w0, idx, hd), 2 * K * U * acc(w0.abs(), idx, ha))
    check("migt_embed_bwd dwpe", dwpe, acc(p0, rows_l, hd), 2 * K * U * acc(p0.abs(), rows_l, ha))
    if with_ids:
        check("migt_embed_bwd dpose", dpose, acc(q0, rows_bt, hd), 2 * K * U * acc(q0.abs(), rows_bt, ha))


@pytest.mark.parametrize("cols,smoothing", [(1024, 0.0), (1025, 0.1), (1024, 0.1), (1025, 0.0)])
def test_cross_entropy_grad(L, cols, smoothing):
    """vf_cross_entropy_grad == fp64 autograd of sum_r w_r CE_s(logits_r, label_r) with the smoothed target (1 - s) onehot + s / cols, on the
    same fp32 logits.  Some rows have weight 0; several labels sit in the last column, which also holds the row's largest logit (the
    tail of the lane loop).  Bar: the softmax's K = cols term sum and a few ulps of each term."""
    gg = gen(cols + int(smoothing * 10))
    rows = 37
    logits = torch.randn(rows, cols, generator=gg) * 3.0
    logits[::3, -1] += 12.0
    labels = torch.randint(0, cols, (rows,), generator=gg, dtype=torch.int32)
    labels[::4] = cols - 1
    w = torch.rand(rows, generator=gg)
    w[::5] = 0.0
    ld = logits.double().requires_grad_(True)
    y = F.one_hot(labels.long(), cols).double() * (1 - f32(smoothing)) + f32(smoothing) / cols
    (-(y * F.log_softmax(ld, -1)).sum(-1) * w.double()).sum().backward()
    got = L.cross_entropy_grad(logits.cuda(), labels.cuda(), w.cuda(), smoothing)
    p = torch.softmax(logits.double(), -1)
    bar = 2 * U * w.double()[:, None] * ((cols + 8) * p + 4 * y) + 1e-38
    check(f"cross_entropy_grad cols{cols} s{smoothing}", got, ld.grad, bar)
    assert torch.equal(got.cpu()[::5], torch.zeros_like(got.cpu()[::5]))


def test_pose_loss_grad(L):
    """vf_pose_loss_grad == fp64 autograd of sum_r w_r (ps mean_3 (y m - raw)^2 + os mean_4 (y - raw)^2), y the pose of the row's view
    (tokens_per_view rows share it), with pose_multiplier m, pos_scale ps and ori_scale os all != 1.  8 ulps of |y m| + |raw|."""
    gg = gen(9)
    tpv, views = 16, 5
    rows = tpv * views
    raw = torch.randn(rows, 7, generator=gg)
    poses = torch.randn(views, 7, generator=gg)
    w = torch.rand(rows, generator=gg)
    mult, ps, os_ = 2.5, 0.6, 1.7
    rd = raw.double().requires_grad_(True)
    y = poses.double().repeat_interleave(tpv, 0)
    m = torch.tensor([f32(mult)] * 3 + [1.0] * 4, dtype=torch.float64)
    diff2 = (y * m - rd) ** 2
    loss = (w.double() * (f32(ps) * diff2[:, :3].mean(-1) + f32(os_) * diff2[:, 3:].mean(-1))).sum()
    loss.backward()
    got = L.pose_loss_grad(raw.cuda(), poses.cuda(), w.cuda(), tpv, mult, ps, os_)
    scl = torch.tensor([f32(ps) * 2 / 3] * 3 + [f32(os_) * 2 / 4] * 4, dtype=torch.float64)
    check("pose_loss_grad", got, rd.grad, 8 * U * w.double()[:, None] * scl * ((y * m).abs() + rd.detach().abs()) + 1e-38)


# ----------------------------------------------------------------------------- optimizers
def _opt_inputs(n, seed):
    gg = gen(seed)
    p = torch.randn(n, generator=gg)
    grads = [torch.randn(n, generator=gg) * s for s in (1.0, 0.3, 2.0)]
    grads[1][:7] = 0.0                                                    # zero gradients: the update runs on the moments alone
    return p, grads


def test_adam(L):
    """vf_adam == torch.optim.Adam in fp64 (betas (0.5, 0.9), eps 1e-8, the hyperparameters rounded to fp32 as the kernel receives them) run
    three steps from the same fp32 start, with grad_scale != 1 and n not a multiple of 256.  Bar per element: 12 u |p| (the fp32 weight
    rounded at each step) + 100 u lr (a few ulps of each of the three updates, |m / denom| <= ~3)."""
    n, lr, gs = 1000, 1e-3, 0.25
    p, grads = _opt_inputs(n, 11)
    pg, mg, vg = p.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pr = p.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([pr], lr=f32(lr), betas=(f32(0.5), f32(0.9)), eps=f32(1e-8))
    for step, g in enumerate(grads, 1):
        gc = g.cuda()
        L.adam(pg, gc, mg, vg, lr=lr, beta1=0.5, beta2=0.9, eps=1e-8, step=step, grad_scale=gs)
        pr.grad = (g * gs).double()        # g * 0.25 is exact in fp32
        opt.step()
    check("adam 3 steps", pg, pr.detach(), 12 * U * pr.detach().abs() + 100 * U * lr)


@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_adamw_keras(L, wd):
    """vf_adamw_keras == the Keras AdamWeightDecay step (models/utils.py:507-515 over TF 2.4 Adam) restated in fp64: p -= lr wd p;
    m += (g - m)(1 - b1); v += (g^2 - v)(1 - b2); p -= lr sqrt(1 - b2^t) / (1 - b1^t) m / (sqrt(v) + eps), with g = grad * grad_scale *
    clip_scale, three steps from the same fp32 start, hyperparameters rounded to fp32 and lr_t evaluated in fp32 (keras_lr_t).  Bar as
    test_adam."""
    n, lr, gs, cs = 1000, 2e-3, 1.0 / 1024, 0.37
    p, grads = _opt_inputs(n, 12)
    pg, mg, vg = p.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    b1, b2, eps = f32(0.9), f32(0.999), f32(1e-8)
    pr, mr, vr = p.double(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for step, g in enumerate(grads, 1):
        L.adamw_keras(pg, g.cuda(), mg, vg, lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=wd, step=step, grad_scale=gs, clip_scale=cs)
        gd = g.double() * f32(gs) * f32(cs)
        pr = pr - f32(lr) * f32(wd) * pr
        mr = mr + (gd - mr) * (1 - b1)
        vr = vr + (gd * gd - vr) * (1 - b2)
        lr_t = keras_lr_t(lr, 0.9, 0.999, step)
        pr = pr - lr_t * mr / (vr.sqrt() + eps)
    check(f"adamw_keras wd{wd} 3 steps", pg, pr, 12 * U * pr.abs() + 100 * U * lr)


@pytest.mark.parametrize("n", [1, 600001])
def test_sumsq(L, n):
    """vf_sumsq == fp64 sum of squares (squares are exact in fp64, the sum is fp64: K 2^-53 sum x^2); n = 1, and n past the grid (grid-stride
    loop) with the last element large."""
    gg = gen(n)
    x = torch.randn(n, generator=gg)
    x[-1] = 3e3
    got = L.sumsq(x.cuda())
    want = (x.double() ** 2).sum()
    check(f"sumsq n{n}", got, want.reshape(1), torch.tensor([2 * n * 2.0 ** -53 * float(want) + 1e-300]))


# ----------------------------------------------------------------------------- dropout: properties
def test_dropout_properties(L):
    """vf_dropout: no reference exists (a hash of (seed, index)), so its properties: the output is exactly 0 or x * (1 / (1 - rate)) (both in
    fp32), the keep fraction is within 5 sigma of the binomial, the same seed gives the same bits, the masks of seeds s and s + 1 overlap as
    independent masks would (within 5 sigma), rate 0 is the identity, and element i's mask does not depend on the tensor length."""
    n = 1_000_003
    x = torch.randn(n, generator=gen(3)).cuda()
    for rate in (0.1, 0.5):
        sc = torch.tensor(1.0, dtype=torch.float32) / (torch.tensor(1.0, dtype=torch.float32) - torch.tensor(rate, dtype=torch.float32))
        y = L.dropout(x, rate, 1234)
        keep = y != 0
        assert torch.equal(y[keep], x[keep] * sc.cuda()), "kept elements are not x / (1 - rate)"
        frac_sigma = math.sqrt(n * rate * (1 - rate))
        kept = int(keep.sum())
        print(f"[dropout rate {rate}] kept {kept} of {n}: {abs(kept - n * (1 - rate)) / frac_sigma:.2f} sigma from the binomial mean")
        assert abs(kept - n * (1 - rate)) < 5 * frac_sigma
        assert torch.equal(L.dropout(x, rate, 1234), y)
        k2 = L.dropout(x, rate, 1235) != 0
        both = int((keep & k2).sum())
        q = (1 - rate) ** 2
        print(f"[dropout rate {rate}] seeds s, s+1 both keep {both}: {abs(both - n * q) / math.sqrt(n * q * (1 - q)):.2f} sigma from independence")
        assert abs(both - n * q) < 5 * math.sqrt(n * q * (1 - q))
        short = L.dropout(x[:4097].contiguous(), rate, 1234)
        assert torch.equal(short, y[:4097])
    assert torch.equal(L.dropout(x, 0.0, 99), x)


# ----------------------------------------------------------------------------- codebook
def test_vq_commit_grad(L):
    """vf_vq_commit_grad (with the counts and row sums of vf_vq_ema_stats) == fp64 2 beta / numel (count_k e_k - sum of the z rows mapped to k)
    in the codebook layout [D, K].  A third of the codes are never used: their gradient is exactly 0."""
    gg = gen(21)
    D, K, m = 16, 96, 500
    emb = torch.randn(D, K, generator=gg)
    z = torch.randn(m, D, generator=gg)
    idx = torch.randint(0, 64, (m,), generator=gg)                         # codes 64..95 unused
    counts, zsum = L.vq_ema_stats(z.cuda(), idx.cuda(), K)
    coef = 2.0 * 0.25 / (m * D)
    grad = torch.full((D, K), float("nan"), device="cuda")
    L.vq_commit_grad(emb.cuda(), counts, zsum, coef, grad)
    cnt = torch.bincount(idx, minlength=K).double()
    zs = torch.zeros(K, D, dtype=torch.float64).index_add_(0, idx, z.double()).t()
    za = torch.zeros(K, D, dtype=torch.float64).index_add_(0, idx, z.double().abs()).t()
    want = f32(coef) * (cnt * emb.double() - zs)
    check("vq_commit_grad", grad, want, 2 * (cnt + 4) * U * f32(coef) * (cnt * emb.double().abs() + za) + 1e-38)
    assert torch.equal(grad.cpu()[:, 64:], torch.zeros(D, K - 64))
