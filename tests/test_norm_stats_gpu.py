"""GroupNorm and LayerNorm statistics under a large mean, against fp64 statistics of the stored fp32 input.

var = E[x^2] - mean^2 loses 1 + mean^2 / var of relative precision to the cancellation: an fp32 sum of squares over a chain of K terms
carries K u sum x^2 of error, so rstd would be off by K u (1 + mean^2 / var) relatively.  An fp32-faithful implementation keeps rstd within a
few u K relatively, independent of the mean.  Inputs: x = mean + std z per group / row with |mean| / std in {1, 30, 300, 3000}, signs mixed.

Bars (u = 2^-24, K the longest fp32 addition chain of one statistic):
  GroupNorm mean   |mean - mean64| <= (K + 2) u mean|x|       (the fp32 chain and the rounding of the result)
  GroupNorm rstd   |rstd - rstd64| <= 2 (K + 4) u rstd64       (no conditioning factor)
                   vf_groupnorm_stats sums x and x^2 per thread in fp32, so it meets this bar only up to |mean| / std ~ 10 (measured on an
                   H100: err/bar 0.56 at 30 with K = 10 pixels per thread, 1.6 at 30 with K = 34, 5e3 at 3000).  The real workloads reach
                   mean^2 / var <= 4.6 (|mean| / std 2.1, with synthetic random weights; tests/test_launch_audit_gpu.py prints it), so the
                   kernel keeps its fp32 sums:
                   above |mean| / std = 10 the test holds it to the conditioned bar 2 (K + 4) u (1 + mean^2 / var) rstd64 instead, the
                   limit DESIGN.md section 7 states.
  LayerNorm y      |y - y64| <= 2 (K + 4) u (|xhat| + rstd mean|x|) |gamma| + 2 u |beta|: the fp32 mean carries K u mean|x|, which every
                   element's x - mean inherits; an rstd off by K u (1 + mean^2 / var) would add that factor times |xhat|.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RATIOS = [1.0, 30.0, 300.0, 3000.0]
STATS_PASS_FAITHFUL = 10.0          # |mean| / std up to which vf_groupnorm_stats meets the unconditioned bar


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def _group_input(n, hw, c, groups, ratio, seed):
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(n, groups, generator=g) < 0.5, -1.0, 1.0)
    std = torch.rand(n, groups, generator=g) * 2 + 0.5
    mean = sign * ratio * std
    z = torch.randn(n, hw, groups, c // groups, generator=g)
    x = (mean[:, None, :, None] + std[:, None, :, None] * z).reshape(n, hw, 1, c)
    return x.float().contiguous()


def _stats64(x, groups):
    n, hw, _, c = x.shape
    xg = x.double().reshape(n, hw, groups, c // groups)
    return xg.mean((1, 3)), xg.var((1, 3), unbiased=False), xg.abs().mean((1, 3))


def _check_stats(tag, mr, x, groups, K, eps=1e-6, conditioned=False):
    m64, v64, amean = _stats64(x, groups)
    r64 = 1.0 / torch.sqrt(v64 + eps)
    mr = mr.double().cpu()
    e_mean = float(((mr[..., 0] - m64).abs() / ((K + 2) * U * amean)).max())
    factor = 1 + m64 * m64 / v64 if conditioned else 1.0
    e_rstd = float(((mr[..., 1] - r64).abs() / (2 * (K + 4) * U * r64 * factor)).max())
    cond = float((m64 * m64 / v64).max())
    print(f"[{tag}] max mean^2/var {cond:.3g}: mean err/bar {e_mean:.3g}, rstd err/bar {e_rstd:.3g}")
    assert e_mean <= 1.0, f"{tag}: mean off by {e_mean:.3g} x its bar"
    assert e_rstd <= 1.0, f"{tag}: rstd off by {e_rstd:.3g} x its bar (mean^2/var up to {cond:.3g})"


@pytest.mark.parametrize("ratio", [1.0, STATS_PASS_FAITHFUL] + RATIOS[1:])
@pytest.mark.parametrize("n,hw,c", [(2, 64 * 64, 128), (1, 128 * 128, 128), (4, 32 * 32, 512)])
def test_groupnorm_stats_pass_large_mean(L, n, hw, c, ratio):
    """vf_groupnorm_stats (the statistics pass of gn_mean_rstd on an fp32 input).  K (launch_checks.gn_stats_chain): one thread sums
    ceil(pixels per block / pixel lanes) pixels of its channel quad, then folds the quad (+2); the block and grid partial sums meet in fp64.
    Faithful up to STATS_PASS_FAITHFUL, conditioned above it (module docstring)."""
    import launch_checks as lc
    x = _group_input(n, hw, c, 32, ratio, int(ratio) + hw + c)
    mr = L.gn_mean_rstd(x.cuda())
    K = lc.gn_stats_chain(n, hw, c)
    _check_stats(f"gn stats pass n{n} hw{hw} C{c} K{K} |mean|/std {ratio:g}", mr, x, 32, K=K, conditioned=ratio > STATS_PASS_FAITHFUL)


@pytest.mark.parametrize("ratio", RATIOS)
def test_groupnorm_finalize_large_mean(L, ratio):
    """vf_groupnorm_finalize (gn_mean_rstd of a tensor carrying fused sums) from exact fp64 sums of the stored x: the fp64 division step
    alone must be faithful (its cancellation costs 2^-53 (1 + mean^2 / var), below u even at 3000^2).  This does not measure the sums a
    conv epilogue fuses: those fold fp32 partial sums across a warp before their fp64 atomic, a shorter chain with the same cancellation."""
    n, hw, c = 2, 1024, 256
    x = _group_input(n, hw, c, 32, ratio, 7 + int(ratio))
    xg = x.double().reshape(n, hw, 32, c // 32)
    xd = x.cuda()
    xd._gn_sums = (torch.stack([xg.sum((1, 3)), (xg * xg).sum((1, 3))], -1).cuda(), 32)
    mr = L.gn_mean_rstd(xd)
    _check_stats(f"gn finalize |mean|/std {ratio:g}", mr, x, 32, K=0)


@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("d", [256, 768])
def test_layernorm_large_mean(L, d, ratio):
    """vf_layernorm (two passes in fp32: the mean, then the sum of squared deviations): K = d / 128 per-lane terms + 2 (quad fold) + 5 (the
    shuffle tree).  The output of rows with |mean| / std = ratio is held to the faithful bar of the module docstring."""
    rows = 333
    g = torch.Generator().manual_seed(d + int(ratio))
    sign = torch.where(torch.rand(rows, 1, generator=g) < 0.5, -1.0, 1.0)
    std = torch.rand(rows, 1, generator=g) + 0.5
    x = (sign * ratio * std + std * torch.randn(rows, d, generator=g)).float()
    gamma, beta = torch.rand(d, generator=g) + 0.5, torch.randn(d, generator=g)
    y = L.layernorm(x.cuda(), gamma.cuda(), beta.cuda(), torch.float32, eps=1e-5).double().cpu()
    xd = x.double()
    mu = xd.mean(1, keepdim=True)
    var = xd.var(1, unbiased=False, keepdim=True)
    rs = 1.0 / torch.sqrt(var + 1e-5)
    xh = (xd - mu) * rs
    want = xh * gamma.double() + beta.double()
    K = d // 128 + 7
    bar = 2 * (K + 4) * U * (xh.abs() + rs * xd.abs().mean(1, keepdim=True)) * gamma.double() + 2 * U * beta.double().abs()
    worst = float(((y - want).abs() / bar).max())
    print(f"[layernorm d{d} |mean|/std {ratio:g}] max mean^2/var {float((mu * mu / var).max()):.3g}: y err/bar {worst:.3g}")
    assert worst <= 1.0, f"layernorm d{d} ratio {ratio}: output off by {worst:.3g} x the faithful bar"
