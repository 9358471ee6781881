"""Per-kernel parity (GPU): every libvf_b200 entry point against a plain PyTorch fp32/fp64 CPU computation of the
same op, called through the C-ABI (viewformer_b200._lib helpers pass raw pointers + stream)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def g(seed):
    return torch.Generator().manual_seed(seed)


def report(name, got, want, atol, rtol):
    got, want = got.double().cpu(), want.double().cpu()
    err = (got - want).abs()
    tol = atol + rtol * want.abs()
    bad = int((err > tol).sum())
    print(f"[{name}] max_abs_err={err.max():.3e} ref_scale={want.abs().mean():.3e} bad={bad}/{err.numel()}")
    if bad:
        i = int((err - tol).argmax())
        print(f"   worst at flat index {i}: got {got.reshape(-1)[i]:.6f} want {want.reshape(-1)[i]:.6f}")
    assert bad == 0, f"{name}: {bad} elements out of tolerance (max err {err.max():.3e})"


# ----------------------------------------------------------------------------- pixels / layout
def test_pixel_conversions(L):
    u8 = torch.randint(0, 256, (3, 16, 16, 3), generator=g(0), dtype=torch.uint8)
    got = L.u8_to_unit(u8.cuda())
    want = u8.float() * torch.tensor(1.0 / 255.0) * 2 - 1
    assert torch.equal(got.cpu(), want)
    x = torch.randn(5, 7, 9, 3, generator=g(1)) * 0.8
    got = L.unit_to_u8(x.cuda())
    want = ((x.clamp(-1, 1) / 2 + 0.5) * 255.5).clamp(0, 255).to(torch.uint8)
    assert torch.equal(got.cpu(), want)
    y = torch.randn(2, 5, 6, 7, generator=g(2))
    assert torch.equal(L.nchw_to_nhwc(y.cuda()).cpu(), y.permute(0, 2, 3, 1).contiguous())
    assert torch.equal(L.nhwc_to_nchw(y.permute(0, 2, 3, 1).contiguous().cuda()).cpu(), y)


# ----------------------------------------------------------------------------- norms
@pytest.mark.parametrize("C,H,W", [(128, 16, 16), (256, 8, 8), (512, 4, 4), (32, 8, 8), (64, 5, 7)])
def test_groupnorm(L, C, H, W):
    x = torch.randn(3, C, H, W, generator=g(C)) * 2 + 0.5
    ga, be = 1 + 0.1 * torch.randn(C, generator=g(1)), 0.1 * torch.randn(C, generator=g(2))
    want = F.group_norm(x.double(), 32, ga.double(), be.double(), eps=1e-6)
    want_s = want * torch.sigmoid(want)
    xh = x.permute(0, 2, 3, 1).contiguous().cuda()
    got = L.groupnorm(xh, ga.cuda(), be.cuda(), swish=False, out_dtype=torch.float32)
    report("gn", got.permute(0, 3, 1, 2), want, 2e-5, 1e-5)
    got = L.groupnorm(xh, ga.cuda(), be.cuda(), swish=True, out_dtype=torch.float32)
    report("gn+swish", got.permute(0, 3, 1, 2), want_s, 2e-5, 1e-5)
    got = L.groupnorm(xh, ga.cuda(), be.cuda(), swish=True, out_dtype=torch.bfloat16)
    report("gn+swish bf16", got.float().permute(0, 3, 1, 2), want_s, 2e-2, 1e-2)
    got = L.groupnorm(xh, None, None, swish=False, out_dtype=torch.float32, normalize=False, upsample=True)
    report("upsample", got.permute(0, 3, 1, 2), F.interpolate(x, scale_factor=2.0, mode="nearest"), 0, 0)


@pytest.mark.parametrize("n,hw,C", [(2, 64, 128), (3, 24, 256), (1, 8, 512)])
def test_groupnorm_layouts_and_chunking(L, n, hw, C):
    """several pixel chunks per image (grid.x > 1), the upsample / space-to-depth stores, and the bf16 -> bf16 edge."""
    x = (torch.randn(n, hw, hw, C, generator=g(hw + C)) * 1.5 + 0.3).cuda()
    ga, be = (1 + 0.1 * torch.randn(C, generator=g(1))).cuda(), (0.1 * torch.randn(C, generator=g(2))).cuda()
    want = F.group_norm(x.permute(0, 3, 1, 2).double().cpu(), 32, ga.double().cpu(), be.double().cpu(), eps=1e-6)
    want = (want * torch.sigmoid(want)).permute(0, 2, 3, 1)
    base = L.groupnorm(x, ga, be, swish=True, out_dtype=torch.float32)
    report("gn chunked", base, want, 2e-5, 1e-5)
    up = L.groupnorm(x, ga, be, swish=True, out_dtype=torch.float32, upsample=True)
    assert torch.equal(up, base.repeat_interleave(2, 1).repeat_interleave(2, 2))
    s2 = L.groupnorm(x, ga, be, swish=True, out_dtype=torch.float32, s2d=True)
    want_s2 = base.reshape(n, hw // 2, 2, hw // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(n, hw // 2, hw // 2, 4 * C)
    assert torch.equal(s2, want_s2)
    # bf16 input carrying fp32-accumulated statistics (what a conv epilogue hands over)
    xb = x.bfloat16()
    o = x.double().reshape(n, hw * hw, 32, C // 32)
    xb._gn_sums = (torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1).contiguous(), 32)
    got = L.groupnorm(xb, ga, be, swish=True, out_dtype=torch.bfloat16)
    report("gn bf16->bf16", got.float(), want, 4e-2, 2e-2)
    with pytest.raises(Exception):
        L.groupnorm(x.bfloat16(), ga, be, swish=True, out_dtype=torch.bfloat16)      # bf16 input without statistics


def test_layernorm(L):
    x = torch.randn(70, 768, generator=g(3)) * 3 + 1
    ga, be = 1 + 0.1 * torch.randn(768, generator=g(4)), 0.1 * torch.randn(768, generator=g(5))
    want = F.layer_norm(x.double(), (768,), ga.double(), be.double(), 1e-5)
    report("ln f32", L.layernorm(x.cuda(), ga.cuda(), be.cuda(), torch.float32), want, 2e-5, 1e-5)
    report("ln bf16", L.layernorm(x.cuda(), ga.cuda(), be.cuda(), torch.bfloat16).float(), want, 2e-2, 1e-2)
    x = torch.randn(9, 128, generator=g(6))
    want = F.layer_norm(x.double(), (128,), ga[:128].double(), be[:128].double(), 1e-5)
    report("ln d128", L.layernorm(x.cuda(), ga[:128].contiguous().cuda(), be[:128].contiguous().cuda(), torch.float32), want, 2e-5, 1e-5)


# ----------------------------------------------------------------------------- SIMT conv / gemm
def _w_kn(w):
    return w.permute(2, 3, 1, 0).reshape(-1, w.shape[0]).contiguous()


@pytest.mark.parametrize("cin,cout,hw,k,mode", [(3, 128, 20, 3, "same"), (128, 3, 12, 3, "same"), (64, 96, 9, 3, "same"),
                                                 (64, 64, 10, 3, "down"), (32, 48, 6, 3, "up"), (72, 40, 7, 1, "same")])
def test_simt_conv(L, cin, cout, hw, k, mode):
    x = torch.randn(2, cin, hw, hw, generator=g(cin + cout))
    w = torch.randn(cout, cin, k, k, generator=g(7)) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g(8))
    xd = x.double()
    if mode == "down":
        want = F.conv2d(F.pad(xd, (0, 1, 0, 1)), w.double(), b.double(), stride=2)
        kw = dict(stride=2, pad=(0, 0))
    elif mode == "up":
        want = F.conv2d(F.interpolate(xd, scale_factor=2.0, mode="nearest"), w.double(), b.double(), padding=1)
        kw = dict(upsample=True)
    else:
        want = F.conv2d(xd, w.double(), b.double(), padding=k // 2)
        kw = dict(pad=(k // 2, k // 2))
    res = torch.randn(want.shape, generator=g(9))
    got = L.simt_conv(x.permute(0, 2, 3, 1).contiguous().cuda(), _w_kn(w).cuda(), b.cuda(), kh=k,
                      residual=res.permute(0, 2, 3, 1).contiguous().cuda(), **kw)
    report(f"simt_conv {mode}", got.permute(0, 3, 1, 2), want + res.double(), 2e-5, 1e-5)


def test_simt_gemm_batched_strided(L):
    B1, B2, M, N, K = 2, 3, 70, 50, 37
    A = torch.randn(B1, B2, M, K, generator=g(10))
    Bm = torch.randn(B1, B2, N, K, generator=g(11))
    bias = torch.randn(M, generator=g(12))
    want = torch.einsum("abmk,abnk->abmn", A.double(), Bm.double()) * 0.5 + bias.double()[None, None, :, None]
    out = torch.empty(B1, B2, M, N, device="cuda")
    L.simt_gemm(A.cuda(), Bm.cuda(), out, M=M, N=N, K=K, a_strides=(K, 1), b_strides=(1, K), ldc=N, batch=(B1, B2),
                a_bs=(B2 * M * K, M * K), b_bs=(B2 * N * K, N * K), c_bs=(B2 * M * N, M * N), alpha=0.5, bias=bias.cuda(),
                bias_mode=L.BIAS_M)
    report("simt_gemm", out, want, 2e-5, 1e-5)


# ----------------------------------------------------------------------------- tensor-core (wgmma) GEMM
def _tc_case(L, dtype, M, N, K, batch=(1, 1), bias_mode=0, act=0, residual=False, alpha=1.0, out_dtype=torch.float32, seed=0):
    B1, B2 = batch
    A = torch.randn(B1, B2, M, K, generator=g(seed))
    Bm = torch.randn(B1, B2, N, K, generator=g(seed + 1)) / K ** 0.5
    Aq, Bq = A.to(dtype).cuda(), Bm.to(dtype).cuda()
    Ar, Br = Aq.double().cpu(), Bq.double().cpu()
    if dtype == torch.float32:      # TF32 truncates mantissas to 10 bits inside the tensor core
        def trunc(t):
            return (t.float().view(torch.int32) & ~0x1FFF).view(torch.float32).double()
        Ar, Br = trunc(Ar), trunc(Br)
    want = torch.einsum("abmk,abnk->abmn", Ar, Br) * alpha
    bias = None
    if bias_mode == 1:
        bias = torch.randn(N, generator=g(seed + 2)); want = want + bias.double()
    elif bias_mode == 2:
        bias = torch.randn(M, generator=g(seed + 2)); want = want + bias.double()[:, None]
    if act:
        want = F.gelu(want)
    res = None
    if residual:
        res = torch.randn(B1, B2, M, N, generator=g(seed + 3)); want = want + res.double()
    out = torch.full((B1, B2, M, N), float("nan"), dtype=out_dtype, device="cuda")
    L.tc_gemm(Aq, Bq, out, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, batch=batch, a_bs=(B2 * M * K, M * K), b_bs=(B2 * N * K, N * K),
              c_bs=(B2 * M * N, M * N), alpha=alpha, bias=None if bias is None else bias.cuda(), bias_mode=bias_mode, act=act,
              residual=None if res is None else res.cuda())
    torch.cuda.synchronize()
    tol = 2e-2 if out_dtype == torch.bfloat16 else (2e-3 if dtype == torch.bfloat16 else 2e-3)
    report(f"tc_gemm {dtype} M{M} N{N} K{K} b{batch} bias{bias_mode} act{act} res{residual}", out.float(), want, tol, tol)


def test_tc_gemm_single_tile_bf16(L):
    _tc_case(L, torch.bfloat16, 128, 128, 64)


def test_tc_gemm_k_loop_bf16(L):
    _tc_case(L, torch.bfloat16, 128, 128, 1024, seed=3)      # > kStages k-blocks: exercises ring wrap + phases


def test_tc_gemm_multi_tile_bf16(L):
    _tc_case(L, torch.bfloat16, 512, 384, 256, seed=5)


def test_tc_gemm_tails_bf16(L):
    _tc_case(L, torch.bfloat16, 200, 72, 136, seed=7)          # M, N, K tails
    _tc_case(L, torch.bfloat16, 64, 40, 64, seed=8)            # BLOCK_N = 64 variant, M < 128


def test_tc_gemm_epilogues_bf16(L):
    _tc_case(L, torch.bfloat16, 256, 256, 192, bias_mode=1, act=1, seed=9)
    _tc_case(L, torch.bfloat16, 256, 128, 192, bias_mode=2, residual=True, alpha=0.25, seed=10)
    _tc_case(L, torch.bfloat16, 256, 128, 192, bias_mode=1, out_dtype=torch.bfloat16, seed=11)


def test_tc_gemm_wide_tiles(L):
    """un-batched bf16 GEMMs with >= 256 rows and N > 64, so several 128 x 128 tiles (block_n 128) per launch: row tails, K tails, every
    epilogue combination (bias, GELU with fp32 and bf16 outputs, residual with alpha), and a batch with shared weights whose entries are
    contiguous."""
    _tc_case(L, torch.bfloat16, 256, 128, 64, seed=40)
    _tc_case(L, torch.bfloat16, 1000, 768, 776, bias_mode=1, residual=True, seed=41)               # M tail (1000 = 3*256+232), K tail
    _tc_case(L, torch.bfloat16, 300, 256, 512, bias_mode=1, act=1, out_dtype=torch.bfloat16, seed=42)   # GELU -> bf16 (fast erf)
    _tc_case(L, torch.bfloat16, 2048, 384, 3072, bias_mode=1, act=1, seed=43)                       # GELU -> f32 (exact erf), long K
    _tc_case(L, torch.bfloat16, 513, 128, 192, residual=True, alpha=0.25, seed=44)
    # contiguous batch with shared weights == one flat row range (the q|k projection pattern)
    Bn, S, d, N = 3, 192, 128, 256
    X = torch.randn(Bn, S, d, generator=g(45)).bfloat16().cuda()
    W = (torch.randn(N, d, generator=g(46)) / d ** 0.5).bfloat16().cuda()
    bias = torch.randn(N, generator=g(47))
    out = torch.empty(Bn, S, N, dtype=torch.bfloat16, device="cuda")
    L.tc_gemm(X, W, out, M=S, N=N, K=d, lda=d, ldb=d, ldc=N, batch=(Bn, 1), a_bs=(S * d, 0), b_bs=(0, 0), c_bs=(S * N, 0),
              bias=bias.cuda(), bias_mode=L.BIAS_N)
    want = torch.einsum("bmk,nk->bmn", X.double().cpu(), W.double().cpu()) + bias.double()
    report("wide gemm flattened batch", out.float(), want, 3e-2, 2e-2)


def test_tc_gemm_batched_bf16(L):
    _tc_case(L, torch.bfloat16, 192, 128, 128, batch=(2, 3), bias_mode=1, seed=12)


def test_tc_gemm_tf32(L):
    _tc_case(L, torch.float32, 128, 128, 32, seed=13)
    _tc_case(L, torch.float32, 300, 200, 416, bias_mode=1, residual=True, seed=14)


def test_tc_gemm_broadcast_and_offsets(L):
    """shared A (weights) across the batch, bias along M, column-offset output: the V^T projection pattern."""
    Bn, d, S = 3, 128, 192
    W = (torch.randn(d, d, generator=g(20)) / d ** 0.5).bfloat16().cuda()
    X = torch.randn(Bn, S, d, generator=g(21)).bfloat16().cuda()
    bias = torch.randn(d, generator=g(22))
    out = torch.zeros(Bn, d, 2 * S, dtype=torch.bfloat16, device="cuda")
    L.tc_gemm(W, X, out, M=d, N=S, K=d, lda=d, ldb=d, ldc=2 * S, batch=(Bn, 1), a_bs=(0, 0), b_bs=(S * d, 0),
              c_bs=(d * 2 * S, 0), c_off=S, bias=bias.cuda(), bias_mode=L.BIAS_M)
    want = torch.einsum("mk,bnk->bmn", W.double().cpu(), X.double().cpu()) + bias.double()[None, :, None]
    report("tc_gemm bcast", out[:, :, S:].float(), want, 3e-2, 2e-2)
    assert float(out[:, :, :S].abs().max()) == 0.0


def test_tc_gemm_causal(L):
    """block-causal k-limit (P.V) and n-tile skipping (QK^T) give the same visible values as the dense product."""
    S, dh, blk = 384, 64, 64
    q = torch.randn(S, dh, generator=g(30)).bfloat16().cuda()
    k = torch.randn(S, dh, generator=g(31)).bfloat16().cuda()
    sc = torch.full((S, S), float("nan"), device="cuda")
    L.tc_gemm(q, k, sc, M=S, N=S, K=dh, lda=dh, ldb=dh, ldc=S, causal_block=blk, causal_skip_n=True)
    want = q.double().cpu() @ k.double().cpu().t()
    view = torch.arange(S) // blk
    vis = view[:, None] >= view[None, :]
    got = sc.cpu().double()
    assert torch.isfinite(got[vis]).all()
    report("qk causal", torch.where(vis, got, torch.zeros_like(got)), torch.where(vis, want, torch.zeros_like(want)), 2e-2, 1e-2)
    p = torch.rand(S, S, generator=g(32)) * vis
    vt = torch.randn(dh, S, generator=g(33)).bfloat16().cuda()
    o = torch.empty(S, dh, device="cuda")
    L.tc_gemm(p.bfloat16().cuda(), vt, o, M=S, N=dh, K=S, lda=S, ldb=S, ldc=dh, causal_block=blk)
    report("pv causal", o, p.bfloat16().double() @ vt.double().cpu().t(), 2e-2, 1e-2)


# ----------------------------------------------------------------------------- tensor-core (wgmma) conv
@pytest.mark.parametrize("dtype,cin,cout,n,hw", [(torch.bfloat16, 64, 128, 2, 16), (torch.bfloat16, 128, 128, 1, 32),
                                                  (torch.bfloat16, 256, 64, 3, 8), (torch.bfloat16, 128, 256, 2, 4),
                                                  (torch.float32, 64, 128, 2, 16), (torch.bfloat16, 128, 128, 1, 20)])
def test_tc_conv3x3(L, dtype, cin, cout, n, hw):
    x = torch.randn(n, cin, hw, hw, generator=g(cin + hw)).to(dtype)
    w = (torch.randn(cout, cin, 3, 3, generator=g(40)) / (9 * cin) ** 0.5).to(dtype)
    b = torch.randn(cout, generator=g(41))
    res = torch.randn(n, cout, hw, hw, generator=g(42))
    xr, wr = x.double(), w.double()
    if dtype == torch.float32:
        tr = lambda t: (t.float().view(torch.int32) & ~0x1FFF).view(torch.float32).double()
        xr, wr = tr(x), tr(w)
    want = F.conv2d(xr, wr, b.double(), padding=1) + res.double()
    w_nk = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous().cuda()
    got = L.tc_conv(x.permute(0, 2, 3, 1).contiguous().cuda(), w_nk, b.cuda(), residual=res.permute(0, 2, 3, 1).contiguous().cuda())
    torch.cuda.synchronize()
    report(f"tc_conv {dtype} {cin}->{cout} n{n} hw{hw}", got.permute(0, 3, 1, 2), want, 3e-3, 3e-3)


@pytest.mark.parametrize("n,H,W,cin,cout,res,out_bf16", [(2, 64, 64, 128, 128, True, False), (1, 40, 20, 64, 256, True, False),
                                                          (3, 32, 8, 256, 128, False, True), (1, 128, 128, 128, 128, True, False),
                                                          (2, 33, 9, 64, 128, False, False)])
def test_tc_conv3x3_wide_tiles(L, n, H, W, cin, cout, res, out_bf16):
    """bf16 3x3 convs on maps >= 16 rows tall take the halo path (8 x 16-pixel tiles, one halo tile per 64-channel block, the 9 taps
    as shifted descriptors into it): ragged heights / widths, one to four channel blocks, two n tiles, residual, bf16 output and the
    fused GroupNorm statistics."""
    x = torch.randn(n, cin, H, W, generator=g(H + W)).bfloat16()
    w = (torch.randn(cout, cin, 3, 3, generator=g(43)) / (9 * cin) ** 0.5).bfloat16()
    b = torch.randn(cout, generator=g(44))
    r = torch.randn(n, cout, H, W, generator=g(45)) if res else None
    want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    if res:
        want = want + r.double()
    w_nk = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous().cuda()
    fus = L.gn_fusable(cout, 32, n * H * W, H * W, cout)
    got = L.tc_conv(x.permute(0, 2, 3, 1).contiguous().cuda(), w_nk, b.cuda(),
                    residual=r.permute(0, 2, 3, 1).contiguous().cuda() if res else None, gn_groups=32,
                    out_dtype=torch.bfloat16 if out_bf16 else torch.float32)
    torch.cuda.synchronize()
    tol = 2e-2 if out_bf16 else 3e-3
    report(f"wide conv n{n} {H}x{W} {cin}->{cout}", got.float().permute(0, 3, 1, 2), want, tol, tol)
    if fus:
        assert hasattr(got, "_gn_sums")
        o = want.permute(0, 2, 3, 1).reshape(n, H * W, 32, cout // 32)
        ws = torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1)
        report("wide conv fused gn sums", got._gn_sums[0].cpu(), ws, 0.5, 2e-3)


@pytest.mark.parametrize("n,H,W,cin,cout", [(2, 64, 64, 128, 128), (1, 40, 20, 64, 256), (2, 33, 9, 128, 128), (3, 32, 8, 256, 128)])
def test_tc_conv_normalise_on_load(L, n, H, W, cin, cout):
    """GroupNorm + swish applied to the halo tile of the conv operand inside the kernel == vf_groupnorm_apply followed by the conv, bit for
    bit (same arithmetic on the same bf16 values); padding stays zero after normalisation (ragged tiles exercise the border)."""
    xr = (torch.randn(n, H, W, cin, generator=g(H * W + cin)) * 1.3 + 0.4).cuda()
    xb = xr.bfloat16()
    o = xr.double().reshape(n, H * W, 32, cin // 32)
    sums = torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1).contiguous()          # fp32-accurate statistics of the producer
    ga, be = (1 + 0.1 * torch.randn(cin, generator=g(1))).cuda(), (0.1 * torch.randn(cin, generator=g(2))).cuda()
    w = (torch.randn(cout, 9 * cin, generator=g(3)) / (9 * cin) ** 0.5).bfloat16().cuda()
    b = torch.randn(cout, generator=g(4)).cuda()
    res = torch.randn(n, H, W, cout, generator=g(5)).cuda()
    assert L.conv_norm_fusable(xb, cout)
    xb._gn_sums = (sums, 32)
    a = L.groupnorm(xb, ga, be, swish=True, out_dtype=torch.bfloat16)
    want = L.tc_conv(a, w, b, residual=res)
    xb2 = xr.bfloat16()
    xb2._gn_sums = (sums, 32)
    got = L.tc_conv(xb2, w, b, residual=res, norm=(L.gn_mean_rstd(xb2), ga, be, 32, True))
    torch.cuda.synchronize()
    diff = (got - want).abs().max().item()
    print(f"[norm-on-load n{n} {H}x{W} {cin}->{cout}] max |fused - (gn_apply; conv)| = {diff:.3e}")
    assert torch.equal(got, want)
    # and against an fp64 reference of norm -> swish -> conv (tolerance of the bf16 operand rounding)
    xn = F.group_norm(xb.double().cpu().permute(0, 3, 1, 2), 32, ga.double().cpu(), be.double().cpu(), eps=1e-6)
    mean = (sums[..., 0] / (H * W * cin // 32)).cpu()
    ref = F.conv2d((xn * torch.sigmoid(xn)), w.double().cpu().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2), b.double().cpu(), padding=1)
    report("norm-on-load vs fp64", got.permute(0, 3, 1, 2), ref + res.double().cpu().permute(0, 3, 1, 2), 5e-2, 3e-2)
    with pytest.raises(Exception):      # shapes outside the halo-tile path are rejected, not silently un-normalised
        small = torch.randn(1, 16, 16, 64).bfloat16().cuda()
        L.tc_conv(small, (torch.randn(128, 9 * 64) / 24).bfloat16().cuda(), None,
                  norm=(torch.zeros(1, 32, 2, device="cuda"), torch.ones(64, device="cuda"), torch.zeros(64, device="cuda"), 32, True))


# ----------------------------------------------------------------------------- codebook
def test_vq_lookup_bit_exact_vs_reference_golden(L, golden_dir):
    import os
    from oracle import synth
    gd = np.load(os.path.join(golden_dir, "vq_lookup.npz"))
    E, z = synth.make_lookup_inputs(int(gd["seed"]))
    et, esq = L.vq_prepare_codebook(E.cuda())
    assert torch.equal(et.cpu(), E.t().contiguous())
    idx, quant, dsum = L.vq_lookup(z.cuda(), et, esq)
    idx = idx.cpu().numpy()
    mism = int((idx != gd["idx"]).sum())
    print(f"[vq_lookup] mismatches vs reference fp32 expression: {mism}/{idx.size}; vs fp64: {int((idx != gd['idx_f64']).sum())}")
    assert np.array_equal(idx, gd["idx"])
    e = E.t()[torch.from_numpy(idx)]
    assert torch.equal(quant.cpu(), z + (e - z))                        # straight-through value, utils_th.py:67
    want = float(((e - z).double() ** 2).sum())
    assert abs(float(dsum) - want) / want < 1e-6
    # ragged M (not a multiple of the 64-row tile) and M = 0
    idx2, _, _ = L.vq_lookup(z[:77].contiguous().cuda(), et, esq)
    assert np.array_equal(idx2.cpu().numpy(), gd["idx"][:77])
    idx0, _, _ = L.vq_lookup(z[:0].contiguous().cuda(), et, esq)
    assert idx0.numel() == 0


def test_gather_rows(L):
    t = torch.randn(50, 64, generator=g(50))
    i = torch.randint(0, 50, (33,), generator=g(51))
    assert torch.equal(L.gather_rows(t.cuda(), i.cuda()).cpu(), t[i])


def test_vq_ema_matches_reference_golden(L, golden_dir):
    import os
    gd = np.load(os.path.join(golden_dir, "quantizer.npz"))
    E, z = torch.from_numpy(gd["E"]).cuda(), torch.from_numpy(gd["z"])
    D, K = E.shape
    zr = z.permute(0, 2, 3, 1).reshape(-1, D).contiguous().cuda()
    emb = E.clone()
    et, esq = L.vq_prepare_codebook(emb)
    cs, dw = torch.zeros(K, device="cuda"), torch.zeros(D, K, device="cuda")
    for step in range(2):
        idx, _, dsum = L.vq_lookup(zr, et, esq)
        assert np.array_equal(idx.cpu().numpy().reshape(gd[f"ids{step}"].shape), gd[f"ids{step}"])
        np.testing.assert_allclose(float(dsum) / zr.numel(), float(gd[f"diff{step}"]), rtol=1e-5)
        counts, esum = L.vq_ema_stats(zr, idx, K)
        corr = float(1.0 - torch.pow(torch.tensor(0.99), torch.tensor(step + 1)))
        L.vq_ema_update(counts, esum, 1 - 0.99, corr, 1e-5, cs, dw, emb, et, esq)
        np.testing.assert_allclose(cs.cpu().numpy(), gd[f"cs{step}"], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(dw.cpu().numpy(), gd[f"dw{step}"], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(emb.cpu().numpy(), gd[f"emb{step}"], rtol=2e-5, atol=1e-5)
        assert torch.equal(et.cpu(), emb.t().contiguous().cpu())


# ----------------------------------------------------------------------------- transformer glue
def test_softmax_masks_and_argmax(L):
    S, blk = 192, 64
    sc = torch.randn(2 * S, S, generator=g(60)) * 4
    view = torch.arange(S) // blk
    m = (view[:, None] >= view[None, :]).float().repeat(2, 1)
    w = sc * m - 1e4 * (1 - m)                       # branching_attention.py:13
    want = F.softmax(w.double(), -1)
    p = torch.empty(2 * S, S, device="cuda")
    L.softmax_rows(sc.cuda(), p, rows_total=2 * S, rows_per_batch=S, cols=S, ld_in=S, ld_out=S, mask_mode=1, block=blk)
    report("softmax causal", p, want, 1e-6, 1e-5)
    # multi-end mask (branching_attention.py:96-124)
    sc2 = torch.randn(S, 2 * S, generator=g(61)) * 3
    m_old = (view[:, None] > view[None, :]).float()
    m_new = (view[:, None] == view[None, :]).float()
    w2 = torch.cat([sc2[:, :S] * m_old - 1e4 * (1 - m_old), torch.where(m_new > 0, sc2[:, S:], torch.full_like(sc2[:, S:], -1e30))], 1)
    want2 = F.softmax(w2.double(), -1)
    p2 = torch.empty(S, 2 * S, device="cuda")
    L.softmax_rows(sc2.cuda(), p2, rows_total=S, rows_per_batch=S, cols=2 * S, ld_in=2 * S, ld_out=2 * S, mask_mode=2, block=blk)
    report("softmax multiend", p2, want2, 1e-6, 1e-5)
    x = torch.randn(37, 1024, generator=g(62))
    x[3, 10] = x[3, 900] = 50.0                       # tie -> first index
    assert torch.equal(L.argmax_rows(x.cuda()).cpu(), x.argmax(-1))
    assert int(L.argmax_rows(x.cuda())[3]) == 10


def test_embed_and_pose_post(L):
    from oracle import migt_oracle as mo
    wte, wpe = torch.randn(1026, 64, generator=g(70)), torch.randn(256, 64, generator=g(71))
    ids = torch.randint(0, 1026, (3, 2, 64), generator=g(72), dtype=torch.int32)
    pose = torch.randn(6, 64, generator=g(73))
    got = L.migt_embed(ids.cuda(), 0, wte.cuda(), wpe.cuda(), pose.cuda(), 6, 64)
    want = wte[ids.long()] + wpe[:64][None, None] + pose.reshape(3, 2, 1, 64)
    assert torch.equal(got.cpu().reshape(3, 2, 64, 64), want)
    got = L.migt_embed(None, 1024, wte.cuda(), wpe.cuda(), pose.cuda(), 6, 64)
    assert torch.equal(got.cpu().reshape(3, 2, 64, 64), wte[1024] + wpe[:64][None, None] + pose.reshape(3, 2, 1, 64))
    raw = torch.randn(40, 7, generator=g(74))
    got = L.pose_postprocess(raw.cuda(), 2.0).cpu()
    want = torch.cat([raw[:, :3] / 2.0, mo.quaternion_remove_sign(mo.quaternion_normalize(raw[:, 3:]))], -1)
    report("pose_post", got, want, 1e-6, 1e-6)


def test_camera_kernels_and_strided_u8(L):
    from oracle import synth, migt_oracle as mo
    cams = synth.make_cameras(5, 4, seed=80)
    cams[:, :, 3:] *= 1.7                                   # un-normalised quaternions on purpose
    got, tr = L.cameras_prepare(cams.cuda(), True)
    rel, tr_want = mo.to_relative_cameras(cams)
    report("cams relative", got, mo.normalize_cameras(rel), 2e-6, 1e-5)
    assert torch.equal(tr.cpu(), tr_want[:, 0])
    got2, _ = L.cameras_prepare(cams.cuda(), False)
    report("cams normalise", got2, mo.normalize_cameras(cams), 1e-6, 1e-6)
    back = L.cameras_from_relative(rel.contiguous().cuda(), tr)
    report("cams from_relative", back, mo.from_relative_cameras(rel, tr_want), 2e-6, 1e-5)
    u8 = torch.randint(0, 256, (3, 4, 8, 8, 3), generator=g(81), dtype=torch.uint8)
    got = L.u8_to_unit(u8.cuda(), first_views=3).cpu()
    want = (u8[:, :3].float() * torch.tensor(1.0 / 255.0) * 2 - 1).reshape(9, 8, 8, 3)
    assert torch.equal(got, want)


def test_small_channel_convs(L):
    x = torch.randn(3, 3, 37, 70, generator=g(90))
    w = torch.randn(128, 3, 3, 3, generator=g(91)) / 27 ** 0.5
    b = torch.randn(128, generator=g(92))
    want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    got = L.conv3x3_small_cin(x.permute(0, 2, 3, 1).contiguous().cuda(), _w_kn(w).cuda(), b.cuda())
    report("conv_in small_cin", got.permute(0, 3, 1, 2), want, 2e-5, 1e-5)
    got = L.conv3x3_small_cin(x.permute(0, 2, 3, 1).contiguous().cuda(), _w_kn(w).cuda(), b.cuda(), gn_groups=32)   # + fused GN sums
    report("conv_in small_cin (+stats)", got.permute(0, 3, 1, 2), want, 2e-5, 1e-5)
    o = want.permute(0, 2, 3, 1).reshape(3, 37 * 70, 32, 4)
    report("conv_in fused gn sums", got._gn_sums[0].cpu(), torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1), 2e-2, 1e-5)
    w64, b64 = w[:64].contiguous(), b[:64].contiguous()
    got = L.conv3x3_small_cin(x.permute(0, 2, 3, 1).contiguous().cuda(), _w_kn(w64).cuda(), b64.cuda())
    report("conv_in small_cin cout64", got.permute(0, 3, 1, 2), want[:, :64], 2e-5, 1e-5)
    x = torch.randn(2, 128, 19, 45, generator=g(93))
    w = torch.randn(3, 128, 3, 3, generator=g(94)) / 1152 ** 0.5
    b = torch.randn(3, generator=g(95))
    want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    xh = x.permute(0, 2, 3, 1).contiguous().cuda()
    report("conv_out small_cout f32", L.conv3x3_small_cout(xh, _w_kn(w).cuda(), b.cuda()).permute(0, 3, 1, 2), want, 2e-5, 1e-5)
    want16 = F.conv2d(x.bfloat16().double(), w.double(), b.double(), padding=1)
    report("conv_out small_cout bf16", L.conv3x3_small_cout(xh.bfloat16(), _w_kn(w).cuda(), b.cuda()).permute(0, 3, 1, 2), want16, 2e-5, 1e-5)


@pytest.mark.parametrize("cin,cout,n,hw", [(64, 128, 2, 16), (128, 128, 1, 32), (256, 256, 3, 8)])
def test_tc_downsample_space_to_depth(L, cin, cout, n, hw):
    """pad(0,1,0,1) + stride-2 3x3 conv (vqgan_th.py:45-49) as a stride-1 tap-table conv over the space-to-depth operand."""
    x = torch.randn(n, cin, hw, hw, generator=g(cin))
    w = (torch.randn(cout, cin, 3, 3, generator=g(96)) / (9 * cin) ** 0.5).bfloat16()
    b = torch.randn(cout, generator=g(97))
    xs = L.groupnorm(x.permute(0, 2, 3, 1).contiguous().cuda(), None, None, swish=False, out_dtype=torch.bfloat16, normalize=False, s2d=True)
    assert list(xs.shape) == [n, hw // 2, hw // 2, 4 * cin]
    want = F.conv2d(F.pad(x.bfloat16().double(), (0, 1, 0, 1)), w.double(), b.double(), stride=2)
    w_nk = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous().cuda()
    got = L.tc_conv(xs, w_nk, b.cuda(), taps=L.TAPS_S2D, coffs=L.s2d_coffs(cin), cin=cin)
    torch.cuda.synchronize()
    report(f"tc downsample {cin}->{cout} hw{hw}", got.permute(0, 3, 1, 2), want, 3e-3, 3e-3)


@pytest.mark.parametrize("cin,cout,n,hw", [(128, 128, 3, 16), (128, 256, 2, 8), (256, 512, 5, 8)])
def test_tc_conv_fused_groupnorm_statistics(L, cin, cout, n, hw):
    """GroupNorm(32) statistics accumulated in the conv epilogue == statistics of the stored output."""
    x = torch.randn(n, hw, hw, cin, generator=g(cin + n)).bfloat16().cuda()
    w = (torch.randn(cout, 9 * cin, generator=g(98)) / (9 * cin) ** 0.5).bfloat16().cuda()
    b = torch.randn(cout, generator=g(99)).cuda()
    res = torch.randn(n, hw, hw, cout, generator=g(100)).cuda()
    out = L.tc_conv(x, w, b, residual=res, gn_groups=32)
    assert hasattr(out, "_gn_sums"), "fusion expected for this shape"
    sums = out._gn_sums[0].cpu()
    o = out.double().cpu().reshape(n, hw * hw, 32, cout // 32)
    want = torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1)
    report("fused gn sums", sums, want, 1e-2, 1e-5)
    ga, be = (1 + 0.1 * torch.randn(cout, generator=g(101))).cuda(), (0.1 * torch.randn(cout, generator=g(102))).cuda()
    y_fused = L.groupnorm(out, ga, be, swish=True, out_dtype=torch.float32)
    plain = out.clone()                                        # clone drops the attached statistics -> stats kernel path
    y_plain = L.groupnorm(plain, ga, be, swish=True, out_dtype=torch.float32)
    report("gn via fused stats vs stats kernel", y_fused, y_plain, 2e-5, 1e-5)
    # bf16 output edge: same statistics (taken from the fp32 accumulators), output rounded once
    out_b = L.tc_conv(x, w, b, residual=res, gn_groups=32, out_dtype=torch.bfloat16)
    assert out_b.dtype == torch.bfloat16 and torch.equal(out_b._gn_sums[0].cpu(), sums) is not None
    report("bf16-edge gn sums", out_b._gn_sums[0].cpu(), want, 1e-2, 1e-5)
    assert torch.equal(out_b, out.bfloat16())
    y_edge = L.groupnorm(out_b, ga, be, swish=True, out_dtype=torch.bfloat16)
    report("gn over bf16 edge", y_edge.float(), y_plain, 6e-2, 3e-2)


@pytest.mark.parametrize("B,T,H,blk", [(2, 4, 3, 64), (1, 10, 2, 64), (2, 3, 2, 64), (1, 5, 1, 32)])
def test_fused_block_causal_attention(L, B, T, H, blk):
    """Fused wgmma attention == softmax(q k^T * m - 1e4 (1-m)) v of branching_attention.py:5-18,41-61 (no 1/sqrt(d))."""
    d, S = H * 64, T * blk
    qk = (torch.randn(B, S, 2 * d, generator=g(S + H)) * 0.6).bfloat16()
    v = torch.randn(B, S, d, generator=g(S + H + 1)).bfloat16()
    vt = v.permute(0, 2, 1).contiguous()
    out = L.attn_block_causal(qk.cuda(), vt.cuda(), B, S, H, d, blk)
    torch.cuda.synchronize()
    q = qk[..., :d].double().reshape(B, S, H, 64).permute(0, 2, 1, 3)
    k = qk[..., d:].double().reshape(B, S, H, 64).permute(0, 2, 1, 3)
    vv = v.double().reshape(B, S, H, 64).permute(0, 2, 1, 3)
    view = torch.arange(S) // blk
    m = (view[:, None] >= view[None, :]).double()
    w = q @ k.transpose(-1, -2)
    w = w * m - 1e4 * (1 - m)
    want = (torch.softmax(w, -1) @ vv).permute(0, 2, 1, 3).reshape(B * S, d)
    report(f"fused attention B{B} T{T} H{H} blk{blk}", out.float(), want, 2e-2, 2e-2)


def _attn_reference(qk, v, B, S, H, d, blk):
    q = qk[..., :d].double().reshape(B, S, H, 64).permute(0, 2, 1, 3)
    k = qk[..., d:].double().reshape(B, S, H, 64).permute(0, 2, 1, 3)
    vv = v.double().reshape(B, S, H, 64).permute(0, 2, 1, 3)
    view = torch.arange(S) // blk
    m = (view[:, None] >= view[None, :]).double()
    w = q @ k.transpose(-1, -2)
    w = w * m - 1e4 * (1 - m)
    return (torch.softmax(w, -1) @ vv).permute(0, 2, 1, 3).reshape(B * S, d)


@pytest.mark.parametrize("B,T,H,blk,first", [(2, 6, 2, 64, 0), (1, 20, 2, 64, 0), (2, 20, 3, 64, 19 * 64), (1, 7, 1, 64, 6 * 64)])
def test_fused_attention_growing_logits_and_tail(L, B, T, H, blk, first):
    """Single-pass softmax: key norms grow from view to view, so the running reference maximum has to move (and the register accumulator be
    rescaled) several times per row; `first` > 0 is the KV-cache decode call (only the last view's query rows are computed)."""
    d, S = H * 64, T * blk
    qk = (torch.randn(B, S, 2 * d, generator=g(S + H + 7)) * 0.5)
    scale = (1.0 + 0.9 * (torch.arange(S) // blk).float())[None, :, None]
    qk[..., d:] *= scale                       # later views: larger keys -> the row maximum keeps growing along the key axis
    qk = qk.bfloat16()
    v = torch.randn(B, S, d, generator=g(S + H + 8)).bfloat16()
    vt = v.permute(0, 2, 1).contiguous()
    out = torch.full((B * S, d), 7.0, dtype=torch.bfloat16, device="cuda")
    L.attn_block_causal(qk.cuda(), vt.cuda(), B, S, H, d, blk, first_query=first, out=out)
    torch.cuda.synchronize()
    want = _attn_reference(qk, v, B, S, H, d, blk)
    t0 = (first // 128) * 128
    got = out.float().cpu().reshape(B, S, d)
    report(f"fused attention (growing logits) B{B} T{T} H{H} first{first}", got[:, t0:].reshape(-1, d), want.reshape(B, S, d)[:, t0:].reshape(-1, d), 2e-2, 2e-2)
    if t0 > 0:
        assert bool((got[:, :t0] == 7.0).all()), "rows below the first computed tile must stay untouched"


@pytest.mark.parametrize("B,Tc,H", [(2, 5, 2), (3, 19, 1), (2, 4, 2), (1, 1, 1)])
def test_fused_attention_decode_with_empty_view_slot(L, B, Tc, H):
    """KV-cache decode layout of MIGT.prefill_context: context views, an EMPTY view slot when their number is odd (garbage the kernel must
    never read), the query view at the start of a 128-row tile.  Result == block-causal attention over [context | query]."""
    blk = 64
    d = H * 64
    pad = Tc % 2
    S_c = (Tc + 1) * blk                       # compact sequence: context + query
    S_tot = (Tc + pad + 1) * blk
    gg = g(Tc * 11 + H)
    qk = (torch.randn(B, S_c, 2 * d, generator=gg) * 0.6).bfloat16()
    v = torch.randn(B, S_c, d, generator=gg).bfloat16()
    want = _attn_reference(qk, v, B, S_c, H, d, blk).reshape(B, S_c, d)[:, Tc * blk:]
    qk_p = torch.full((B, S_tot, 2 * d), 300.0).bfloat16()                 # the empty slot holds huge values: any leak shows
    v_p = torch.full((B, S_tot, d), -77.0).bfloat16()
    qk_p[:, :Tc * blk] = qk[:, :Tc * blk]; v_p[:, :Tc * blk] = v[:, :Tc * blk]
    r0 = (Tc + pad) * blk
    qk_p[:, r0:] = qk[:, Tc * blk:]; v_p[:, r0:] = v[:, Tc * blk:]
    out = torch.zeros((B * S_tot, d), dtype=torch.bfloat16, device="cuda")
    L.attn_block_causal(qk_p.cuda(), v_p.permute(0, 2, 1).contiguous().cuda(), B, S_tot, H, d, blk, first_query=r0, out=out,
                        skip_view=(Tc if pad else -1))
    torch.cuda.synchronize()
    got = out.float().cpu().reshape(B, S_tot, d)[:, r0:]
    report(f"fused attention decode Tc{Tc} pad{pad}", got.reshape(-1, d), want.reshape(-1, d), 2e-2, 2e-2)


@pytest.mark.parametrize("B,T,H", [(2, 5, 2), (1, 10, 3), (1, 3, 1), (2, 2, 1)])
def test_fused_multiend_attention(L, B, T, H):
    """Fused branching attention == branching_attention.py:82-126 (oracle restatement): stream 0 block-causal, streams 1 and 2 attend to the
    stream-0 keys of strictly earlier views plus their own view of their own stream, one joint softmax."""
    from oracle import migt_oracle as mo
    blk, ns = 64, 3
    d, S = H * 64, T * blk
    gg = g(T * 7 + H)
    qk = (torch.randn(B, ns * S, 2 * d, generator=gg) * 0.5).bfloat16()
    v = torch.randn(B, ns * S, d, generator=gg).bfloat16()
    vt = v.permute(0, 2, 1).contiguous()
    split = lambda x: [x[:, s * S:(s + 1) * S].double().reshape(B, T, blk, H, 64).permute(0, 3, 1, 2, 4) for s in range(ns)]      # [B,H,T,L,dh]
    want = mo.causal_block_multiend_attention(split(qk[..., d:]), split(v), split(qk[..., :d]))
    for s in range(ns):
        out = L.attn_block_multiend(qk.cuda(), vt.cuda(), B, S, ns, s, H, d, blk)
        torch.cuda.synchronize()
        w = want[s].permute(0, 2, 3, 1, 4).reshape(B * S, d)
        report(f"fused multi-end attention stream {s} B{B} T{T} H{H}", out.float(), w, 2e-2, 2e-2)


# ----------------------------------------------------------------------------- exact (split-fp16, chunked accumulation) convolutions
def _split_ref(v):
    """CPU restatement of the VF_F16X2 pair: hi = fp16(v), lo = fp16((v - hi) * 2^11)."""
    hi = v.half()
    lo = ((v - hi.float()) * 2048.0).half()
    return hi, lo


def test_split_f16x2_layouts(L):
    x = torch.randn(2, 6, 4, 128, generator=g(7)) * 3
    hi, lo = _split_ref(x)
    y = L.groupnorm(x.cuda(), None, None, swish=False, out_dtype=torch.float16, normalize=False).cpu()
    assert list(y.shape) == [2, 6, 4, 256]
    assert torch.equal(y[..., :128], hi) and torch.equal(y[..., 128:], lo)
    rec = y[..., :128].double() + y[..., 128:].double() / 2048.0
    assert float(((rec - x.double()).abs() / x.abs().double().clamp_min(1e-3)).max()) < 2.0 ** -21
    # space-to-depth: [N,H/2,W/2, hi(4C) | lo(4C)], block (a*2+b) <- pixel (2y+a, 2x+b)
    ys = L.groupnorm(x.cuda(), None, None, swish=False, out_dtype=torch.float16, normalize=False, s2d=True).cpu()
    assert list(ys.shape) == [2, 3, 2, 1024]
    for a in (0, 1):
        for b in (0, 1):
            blk = (a * 2 + b) * 128
            assert torch.equal(ys[..., blk:blk + 128], hi[:, a::2, b::2]) and torch.equal(ys[..., 512 + blk:512 + blk + 128], lo[:, a::2, b::2])
    # nearest x2 upsample
    yu = L.groupnorm(x.cuda(), None, None, swish=False, out_dtype=torch.float16, normalize=False, upsample=True).cpu()
    assert torch.equal(yu[:, ::2, ::2], y) and torch.equal(yu[:, 1::2, 1::2], y)
    # normalising variant == the fp32 kernel's values, split
    ga, be = (1 + 0.1 * torch.randn(128, generator=g(8))).cuda(), (0.1 * torch.randn(128, generator=g(9))).cuda()
    f = L.groupnorm(x.cuda(), ga, be, swish=True, out_dtype=torch.float32).cpu()
    s = L.groupnorm(x.cuda(), ga, be, swish=True, out_dtype=torch.float16).cpu()
    fh, fl = _split_ref(f)
    assert torch.equal(s[..., :128], fh) and torch.equal(s[..., 128:], fl)


@pytest.mark.parametrize("n,H,W,cin,cout,res", [(2, 64, 64, 128, 128, True), (1, 40, 20, 64, 256, False), (2, 33, 9, 128, 128, True),
                                                 (3, 16, 16, 256, 256, True), (5, 8, 8, 512, 256, False), (2, 4, 4, 128, 64, True)])
def test_tc_conv_exact_split_fp16(L, n, H, W, cin, cout, res):
    """fp32-faithful conv on the tensor cores (VF_F16X2 operands, 3 MMA passes, chunked RN accumulation) against fp64, next to the
    fp32 CUDA-core conv of the exact path: the tensor-core result must be at least as close to fp64 as the FFMA chain."""
    x = torch.randn(n, cin, H, W, generator=g(H + W + cin)) * 1.5
    w = torch.randn(cout, cin, 3, 3, generator=g(143)) / (9 * cin) ** 0.5
    b = torch.randn(cout, generator=g(144))
    r = torch.randn(n, cout, H, W, generator=g(145)) if res else None
    want = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    if res:
        want = want + r.double()
    xh = x.permute(0, 2, 3, 1).contiguous().cuda()
    rh = r.permute(0, 2, 3, 1).contiguous().cuda() if res else None
    xs = L.groupnorm(xh, None, None, swish=False, out_dtype=torch.float16, normalize=False)
    ws = L.split_f16x2(w.permute(0, 2, 3, 1).reshape(cout * 9, cin).contiguous().cuda()).reshape(cout, 18 * cin)
    got = L.tc_conv(xs, ws, b.cuda(), residual=rh, gn_groups=32)
    ref32 = L.simt_conv(xh, w.permute(2, 3, 1, 0).reshape(9 * cin, cout).contiguous().cuda(), b.cuda(), kh=3, residual=rh)
    torch.cuda.synchronize()
    wantp = want.permute(0, 2, 3, 1)
    scale = float(wantp.abs().mean())
    e_tc = (got.double().cpu() - wantp).abs()
    e_32 = (ref32.double().cpu() - wantp).abs()
    print(f"[exact conv n{n} {H}x{W} {cin}->{cout}] tensor-core: max {e_tc.max() / scale:.2e} rms {e_tc.pow(2).mean().sqrt() / scale:.2e} | "
          f"FFMA: max {e_32.max() / scale:.2e} rms {e_32.pow(2).mean().sqrt() / scale:.2e} (relative to mean |y|)")
    assert float(e_tc.max()) / scale < 4e-6
    assert float(e_tc.pow(2).mean().sqrt()) <= 1.5 * float(e_32.pow(2).mean().sqrt()) + 1e-9
    if L.gn_fusable(cout, 32, n * H * W, H * W, cout):
        assert hasattr(got, "_gn_sums")
        o = got.double().cpu().reshape(n, H * W, 32, cout // 32)
        report("exact conv fused gn sums", got._gn_sums[0].cpu(), torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1), 1e-2, 1e-5)


@pytest.mark.parametrize("cin,cout,n,hw", [(128, 128, 2, 32), (256, 256, 3, 8)])
def test_tc_downsample_exact_split_fp16(L, cin, cout, n, hw):
    """stride-2 Downsample conv (vqgan_th.py:45-49) on the exact path: split-fp16 space-to-depth operand + tap table."""
    x = torch.randn(n, cin, hw, hw, generator=g(cin + 1))
    w = torch.randn(cout, cin, 3, 3, generator=g(196)) / (9 * cin) ** 0.5
    b = torch.randn(cout, generator=g(197))
    want = F.conv2d(F.pad(x.double(), (0, 1, 0, 1)), w.double(), b.double(), stride=2).permute(0, 2, 3, 1)
    xs = L.groupnorm(x.permute(0, 2, 3, 1).contiguous().cuda(), None, None, swish=False, out_dtype=torch.float16, normalize=False, s2d=True)
    ws = L.split_f16x2(w.permute(0, 2, 3, 1).reshape(cout * 9, cin).contiguous().cuda()).reshape(cout, 18 * cin)
    got = L.tc_conv(xs, ws, b.cuda(), taps=L.TAPS_S2D, coffs=L.s2d_coffs(cin), cin=cin)
    torch.cuda.synchronize()
    e = (got.double().cpu() - want).abs()
    print(f"[exact downsample {cin}->{cout} hw{hw}] max {e.max() / want.abs().mean():.2e}")
    assert float(e.max() / want.abs().mean()) < 4e-6


# ----------------------------------------------------------------------------- fused wgmma codebook lookup
def test_vq_lookup_fused_bit_exact(L, golden_dir):
    """One-pass fused lookup (fp16 wgmma distance GEMM, top-2 from the accumulator registers, fp64 settlement of near-ties) == the REAL
    reference's indices on the golden rows (4096 gaussian + 512 adversarial near-ties + 64 exact codes), ragged / empty M,
    quant + commit-loss outputs, and == the exact fp32 kernel on 40 960 random rows."""
    import os
    from oracle import synth
    gd = np.load(os.path.join(golden_dir, "vq_lookup.npz"))
    E, z = synth.make_lookup_inputs(int(gd["seed"]))
    et, esq = L.vq_prepare_codebook(E.cuda())
    eh = L.vq_prepare_codebook_f16(et)
    assert torch.equal(eh.cpu(), (-2.0 * E.t()).half())
    idx, quant, dsum, cnt = L.vq_lookup_fused(z.cuda(), et, esq, eh, return_counts=True)
    torch.cuda.synchronize()
    idx = idx.cpu().numpy()
    print(f"[vq_lookup_fused] mismatches vs reference: {int((idx != gd['idx']).sum())}/{idx.size}; settled exactly: pair {int(cnt[0])}, all-codes {int(cnt[1])}")
    assert np.array_equal(idx, gd["idx"])
    e = E.t()[torch.from_numpy(idx)]
    assert torch.equal(quant.cpu(), z + (e - z))
    want = float(((e - z).double() ** 2).sum())
    assert abs(float(dsum) - want) / want < 1e-6
    for m in (77, 128, 129, 255, 257, 1000):
        i2, _, _ = L.vq_lookup_fused(z[:m].contiguous().cuda(), et, esq, eh, want_quant=False, want_diff=False)
        assert np.array_equal(i2.cpu().numpy(), gd["idx"][:m]), m
    i0, _, _ = L.vq_lookup_fused(z[:0].contiguous().cuda(), et, esq, eh)
    assert i0.numel() == 0
    zz = torch.randn(40960, 256, generator=g(123)).cuda()
    a, _, _, cnt = L.vq_lookup_fused(zz, et, esq, eh, want_quant=False, want_diff=False, return_counts=True)
    b, _, _ = L.vq_lookup(zz, et, esq, want_quant=False, want_diff=False)
    print(f"[vq_lookup_fused] 40960 random rows: mismatches {int((a != b).sum())}; settled exactly: pair {int(cnt[0])}, all-codes {int(cnt[1])}")
    assert torch.equal(a, b)
    # a quarter of the worst-case tolerance (the default, tol_factor = 1): same indices on random rows, fewer rows take the exact pass
    a1, _, _, cnt1 = L.vq_lookup_fused(zz, et, esq, eh, want_quant=False, want_diff=False, tol_factor=0.25, return_counts=True)
    assert torch.equal(a1, b) and int(cnt1.sum()) <= int(cnt.sum())
    # rows beyond fp16 range / non-finite rows go to the exact pass instead of producing garbage
    zbig = zz[:300].clone()
    zbig[5] *= 1e5
    zbig[17, 3] = 7e4
    ab, _, _ = L.vq_lookup_fused(zbig, et, esq, eh, want_quant=False, want_diff=False)
    bb, _, _ = L.vq_lookup(zbig, et, esq, want_quant=False, want_diff=False)
    assert torch.equal(ab, bb)


@pytest.mark.parametrize("D,K", [(64, 256), (128, 512)])
def test_vq_lookup_fused_small_codebooks(L, D, K):
    E = (torch.rand(D, K, generator=g(D)) * 2 - 1) * 3 ** 0.5
    z = torch.randn(3000, D, generator=g(K))
    z[:200] = E.t()[torch.randint(0, K, (200,), generator=g(1))] + 1e-3 * torch.randn(200, D, generator=g(2))      # near codes
    et, esq = L.vq_prepare_codebook(E.cuda())
    eh = L.vq_prepare_codebook_f16(et)
    a, qa, da = L.vq_lookup_fused(z.cuda(), et, esq, eh)
    b, qb, db = L.vq_lookup(z.cuda(), et, esq)
    assert torch.equal(a, b) and torch.equal(qa, qb) and abs(float(da) - float(db)) <= 1e-9 * abs(float(db))


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 16, 16, 128, 128), (3, 8, 8, 256, 128), (1, 32, 24, 128, 256), (5, 8, 8, 128, 128)])
def test_conv_weight_gradient_on_tensor_cores(L, n, h, w, cin, cout):
    """conv_wgrad_tc (nine exact split-fp16 GEMMs over the zero-padded, transposed pixel axis, K offsets per tap, split-K) == the fp64
    weight gradient of a 3x3 stride-1 pad-1 convolution, and agrees with the fp32 CUDA-core atomics kernel."""
    gg = g(n * 100 + h + cin)
    x = torch.randn(n, h, w, cin, generator=gg)
    dy = torch.randn(n, h, w, cout, generator=gg)
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(False)
    wt = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, requires_grad=True)
    y = torch.nn.functional.conv2d(xd, wt, padding=1)
    y.backward(dy.double().permute(0, 3, 1, 2))
    want = wt.grad.permute(2, 3, 1, 0).reshape(9 * cin, cout)             # [tap*Cin + c, Cout]
    dw = torch.zeros(9 * cin, cout, device="cuda")
    L.conv_wgrad_tc(x.cuda(), dy.cuda(), dw)
    torch.cuda.synchronize()
    scale = float(want.abs().max())
    err = float((dw.double().cpu() - want).abs().max()) / scale
    dw32 = torch.zeros(9 * cin, cout, device="cuda")
    L.conv_wgrad(x.cuda(), dy.cuda(), dw32, kh=3)
    err32 = float((dw32.double().cpu() - want).abs().max()) / scale
    print(f"[conv_wgrad_tc n{n} {h}x{w} {cin}->{cout}] max err / max|dW|: tensor-core exact {err:.2e}, fp32 atomics {err32:.2e}")
    assert err < 5e-6 and err32 < 5e-5
    # accumulate semantics
    L.conv_wgrad_tc(x.cuda(), dy.cuda(), dw)
    assert float((dw.double().cpu() - 2 * want).abs().max()) / scale < 1e-5
