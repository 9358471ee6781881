"""The exact (split-fp16) tensor-core conv / GEMM kernel's staging handover, at launches where the busiest CTA walks 8 or more tiles.

In exact mode tc_gemm_kernel (viewformer_b200/csrc/vf_tc_gemm.cu) splits each tile's epilogue between two sides: the eight MMA warps
write the tile's chunk sums to the shared staging tile and arrive on an mbarrier (stg_full), then start the next tile's MMAs; warps
9..11 of the producer warpgroup wait on it, add bias and residual, store, fold the GroupNorm sums and arrive on a second mbarrier
(stg_empty), which the MMA warps wait on before they overwrite the staging tile with the next tile.  The phases flip once per tile, so
a parity slip shows up as a tile stored from another tile's staging (or one stored twice and another never) only after several tiles
of one CTA; hence 8 tiles or more per CTA here, on 132 SMs.

Every case goes through the helpers of test_persistent_tc_walks_gpu.py: the launcher's plan against the restated tiling, every image
or batch entry against fp64 (tests/launch_checks.py), and every image (TN = 1), image pair (TN = 2) or batch entry against a launch of
that part alone, bit for bit, with the fused GroupNorm sums at rtol 1e-12 (fp64 atomics in schedule order).  Covered: the halo conv
at 128^2 and 64^2 with a residual, without one and with the residual aliased to the output; the tap-box conv 256 -> 256 at 32^2 and
its TN = 2 case at 8^2; the Downsample; a split-fp16 GEMM with an N tail, whose last n tile takes the epilogue's generic (scalar)
path; and a launch with fewer tiles than SMs.
"""
import random

import pytest
import torch

import launch_checks as lc
from test_persistent_tc_walks_gpu import _bias_res, _conv_case, _conv_operands, _conv_plan, _gemm_case, _mat, _same_bits, _split

pytestmark = pytest.mark.gpu

WALK = 8          # tiles the busiest CTA walks in every many-tile case


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


@pytest.mark.parametrize("n,side,residual,gn", [
    (9, 128, True, 32),           # 1152 tiles
    (9, 128, False, 32),
    (34, 64, True, 32),           # 1088 tiles
    (34, 64, False, 0),
], ids=["128sq-res-gn", "128sq-gn", "64sq-res-gn", "64sq"])
def test_exact_halo_conv_handover(L, n, side, residual, gn):
    seed = 1100 + n + side
    x, w_nk = _conv_operands("exact", n, side, side, 128, 128, seed)
    b, r = _bias_res(n, side, side, 128, seed, residual)
    _conv_case(L, f"exact halo {n} x {side}^2{' res' if residual else ''}{' gn' if gn else ''}", x, w_nk, b, WALK, residual=r,
               gn_groups=gn)


@pytest.mark.parametrize("n,side", [(9, 128), (34, 64)], ids=["128sq", "64sq"])
def test_exact_halo_conv_handover_residual_aliased_to_output(L, n, side):
    """out = conv(x) + out: the epilogue warps read each residual row just before they overwrite it."""
    c = 128
    x, w_nk = _conv_operands("exact", n, side, side, c, c, 1200 + side)
    b, r = _bias_res(n, side, side, c, 1200 + side, True)
    tag = f"exact halo aliased residual {n} x {side}^2"
    _conv_plan(L, tag, x, w_nk, WALK)
    before, check = lc.CHECKERS["tc_conv"]
    out = r.clone()
    ba = lc.bind(L.tc_conv, x, w_nk, b, residual=out, out=out, gn_groups=32)
    st = before(ba, random.Random(0))
    L.tc_conv(x, w_nk, b, residual=out, out=out, gn_groups=32)
    torch.cuda.synchronize()
    worst = 0.0
    for i0 in range(0, n, 16):
        st["images"] = list(range(i0, min(n, i0 + 16)))
        worst = max(worst, check(ba, out, st))
    print(f"[fp64 {tag}] every image of {n}: worst ratio {worst:.3g}")
    assert worst <= 1.0
    gn = out._gn_sums[0]
    for i in range(n):
        one = r[i:i + 1].clone()
        L.tc_conv(x[i:i + 1], w_nk, b, residual=one, out=one, gn_groups=32)
        _same_bits(f"{tag} image {i}", out[i:i + 1], one)
        torch.testing.assert_close(gn[i:i + 1], one._gn_sums[0], rtol=1e-12, atol=0)


@pytest.mark.parametrize("n,side,cin,cout", [
    (67, 32, 256, 256),           # 1072 tiles
    (535, 8, 256, 512),           # TN = 2: 268 image pairs x 4 n tiles = 1072 tiles, the last pair half empty
], ids=["32sq-256", "8sq-tn2"])
def test_exact_tap_box_conv_handover(L, n, side, cin, cout):
    x, w_nk = _conv_operands("exact", n, side, side, cin, cout, 1300 + n)
    b, r = _bias_res(n, side, side, cout, 1300 + n, True)
    _conv_case(L, f"exact tap-box {n} x {side}^2 {cin}->{cout} res", x, w_nk, b, WALK, residual=r, gn_groups=32)


def test_exact_downsample_conv_handover(L):
    """The stride-2 Downsample (space-to-depth operand, TAPS_S2D): 134 x 64^2 -> 32^2, 1072 tiles."""
    n, c = 134, 128
    x, w_nk = _conv_operands("exact", n, 64, 64, c, c, 1400, s2d=True)
    b, _ = _bias_res(n, 32, 32, c, 1400, False)
    _conv_case(L, "exact downsample 134 x 64^2", x, w_nk, b, WALK, taps=L.TAPS_S2D, coffs=L.s2d_coffs(c), cin=c, gn_groups=32)


def test_exact_gemm_handover_n_tail(L):
    """Split-fp16 GEMM, N = 200: n tile 0 takes the vector epilogue, n tile 1 (72 columns) the generic one; 9 x 64 x 2 = 1152 tiles
    with BIAS_N and a residual."""
    M, N, K, b1 = 8192, 200, 128, 9
    A = _split(_mat((b1, M, K), 1500) * 1.5)
    B = _split(_mat((N, K), 1501) / K ** 0.5)
    R = _mat((b1, M, N), 1502)
    out = torch.empty((b1, M, N), device="cuda")
    _gemm_case(L, "exact gemm N tail", A, B, out, WALK, M=M, N=N, K=K, lda=2 * K, ldb=2 * K, ldc=N, batch=(b1, 1), a_bs=(M * 2 * K, 0),
               c_bs=(M * N, 0), bias=_mat(N, 1503), bias_mode=L.BIAS_N, residual=R)


def test_exact_halo_conv_fewer_tiles_than_sms(L):
    """2 x 64^2: 64 tiles, one per CTA, so every CTA's epilogue warps store one tile and exit."""
    n, side = 2, 64
    x, w_nk = _conv_operands("exact", n, side, side, 128, 128, 1600)
    b, r = _bias_res(n, side, side, 128, 1600, True)
    _conv_case(L, "exact halo 2 x 64^2 (64 tiles)", x, w_nk, b, 1, residual=r, gn_groups=32)
