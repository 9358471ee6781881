"""The codebook lookups at their numerical edges, on the host: row and codebook generators for tests/test_vq_lookup_edges_gpu.py, and an
fp16 model of the fused lookup's decision (vf_vq_fused.cu): fp16 operands z and -2e, products summed in fp64, and the kernel's tolerance
(the rounding bound scaled by tol_factor, plus the accumulation, fixed-point and subnormal slack) with the fixed-point step G and the row cap
computed as the kernel computes them.  The model shows what the GPU tests then check: rows whose fp16 roundings all align are misranked
beyond the 0.25 x bound tolerance, the full bound (tol_factor 1) catches them, and at operand scales below 2^-14 the relative bound alone
lets misranked rows through while the subnormal term does not."""
import math

import numpy as np
import pytest

U = 2.0 ** -24


# ----------------------------------------------------------------------------------------------- generators
def uniform_codebook(D, K, seed, scale=1.0):
    """Et [K, D] float32, uniform in +-sqrt(3) (unit variance, as scripts/bench_vq.py), times scale."""
    rng = np.random.default_rng(seed)
    return (rng.uniform(-1.0, 1.0, (K, D)) * math.sqrt(3.0) * scale).astype(np.float32)


def gaussian_rows(M, D, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((M, D)) * scale).astype(np.float32)


def esq32(et):
    """|e|^2 per code as vf_vq_prepare_codebook sums it: fp32, square then add, in dimension order."""
    s = np.zeros(et.shape[0], np.float32)
    for d in range(et.shape[1]):
        s = (s + et[:, d] * et[:, d]).astype(np.float32)
    return s


def kernel_constants(esq):
    """(G, zcap) of vq_lookup_fused_kernel for a codebook with these |e|^2 (vf_vq_fused.cu, the fixed-point set-up), in fp32 as there."""
    f = np.float32
    esqmax = max(f(np.nan_to_num(esq, nan=np.inf).max()), f(1e-30))
    kexp = int((np.array([f(17.2) * esqmax], np.float32).view(np.int32)[0] >> 23) & 255) - 127 + 2
    g_step = f(2.0 ** (kexp - 23))
    half_range = f(2.0 ** (kexp - 1))
    zcap = f((half_range - esqmax) / (f(2.02) * np.sqrt(esqmax, dtype=np.float32)))
    return float(g_step), float(zcap)


def lookup_bar(z, et):
    """Per row, the fp32 tie bar of tests/launch_checks.check_lookup: a row is decisive when its fp64 gap to the runner-up exceeds it."""
    z64, e64 = z.astype(np.float64), et.astype(np.float64)
    return 4 * (z.shape[1] + 2) * U * ((z64 * z64).sum(1) + (e64 * e64).sum(1).max())


def fp64_distances(z, et):
    """fp64 |z - e|^2 [M, K], direct sums of squared differences (NaN where an operand is NaN)."""
    z64, e64 = z.astype(np.float64), et.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.stack([((e64 - r[None, :]) ** 2).sum(1) for r in z64])


def nearest64(dist):
    """(index, gap to the runner-up) per row: NaN reads as +inf, ties go to the smaller index (the rule both lookups follow)."""
    d = np.where(np.isnan(dist), np.inf, dist)
    idx = d.argmin(1)                                           # first index among equal minima
    best = d[np.arange(len(d)), idx]
    rest = d.copy()
    rest[np.arange(len(d)), idx] = np.inf
    with np.errstate(invalid="ignore"):
        gap = rest.min(1) - best
    return idx, np.where(np.isnan(gap), 0.0, gap)


def aligned_pair_rows(D, K, n_rows, seed, a=1.0, m_extra=None, margin_bars=1.25, pair=(3, 200)):
    """Rows whose fp16 roundings all push one way, against a codebook holding one pair of fp16-exact codes e_a = a s, e_b = -a s
    (s: D/2 +1 and D/2 -1) at ``pair`` and far fillers of smaller norm.  Row elements are fp16 grid points in [1, 1 + 2^-10] moved by
    eps_i < 0.49 ulp against s (z_i = z16_i + s_i eps_i), so fp16(z) = z16 exactly and every rounding error lowers the fp16 score of b
    against a by the same sign: the fp16 gap  4a 2^-10 (D/2 - m)  favours b, while the eps_i are set so that the fp64 distances favour
    a by ``margin_bars`` x the fp32 tie bar of check_lookup.  Returns (z [n, D] float32, Et [K, D] float32, (i_a, i_b))."""
    rng = np.random.default_rng(seed)
    ia, ib = pair
    s = np.concatenate([np.ones(D // 2), -np.ones(D // 2)])
    rng.shuffle(s)
    et = (-0.75 + rng.uniform(-0.25, 0.25, (K, D))).astype(np.float32)       # |z - f|^2 ~ 3 D: far; |f|^2 < D = |e_a|^2
    et[ia], et[ib] = a * s, -a * s
    bar = 4 * (D + 2) * U * (D * 1.0 + (et.astype(np.float64) ** 2).sum(1).max())    # |z|^2 ~ D
    eps_max = 0.49 * 2.0 ** -10
    if m_extra is None:                         # the smallest m with room for the margin: sum eps = 2^-10 (D/2 - m) + margin / (4a)
        m_extra = int(math.ceil(D / 2 - (D * eps_max - margin_bars * bar / (4 * a)) / 2.0 ** -10))
    rows = []
    for _ in range(n_rows):
        k = np.where(s < 0, 1.0, 0.0)
        plus = np.flatnonzero(s > 0)
        k[rng.choice(plus, m_extra, replace=False)] = 1.0
        z16 = 1.0 + k * 2.0 ** -10                                             # fp16 grid points in [1, 2)
        want = 2.0 ** -10 * (D / 2 - m_extra) + margin_bars * bar / (4 * a)    # sum eps
        eps = np.full(D, want / D) * (1 + 0.02 * rng.uniform(-1, 1, D))
        eps *= want / eps.sum()
        assert eps.max() < 0.5 * 2.0 ** -10, "no room for the margin: lower margin_bars or raise m_extra"
        rows.append(z16 + s * eps)
    return np.array(rows, dtype=np.float32), et, (ia, ib)


# ----------------------------------------------------------------------------------------------- the fused kernel's decision
def fused_model(z, et, tol_factor, subnormal=True):
    """fp16 model of vq_lookup_fused_kernel per row: (best code of the fp16 scores, queued for the exact pass, fp16 gap of the first code
    outside the tolerance over its tolerance).  Scores s_c = fp16(z) . fp16(-2 e_c) (fp64 sums) + |e_c|^2, the tolerance of the merge step
    with the rounding bound tol_factor 2^-9 |z| (|e_b| + |e_c|), the slack 2^-16 (|s_b| + |s_c|) + 4 G, and (subnormal=True, as the
    kernel does) the subnormal term 2^-23 sqrt(D) (|z| + |e_b| + |e_c|) + D 2^-48."""
    D = z.shape[1]
    esq = esq32(et)
    g_step, _ = kernel_constants(esq)
    z16 = z.astype(np.float16).astype(np.float64)
    e16 = (np.float32(-2.0) * et).astype(np.float16).astype(np.float64)
    s = z16 @ e16.T + esq.astype(np.float64)[None, :]
    b = s.argmin(1)
    sb = s[np.arange(len(s)), b]
    zn = np.sqrt((z.astype(np.float64) ** 2).sum(1))[:, None]
    en = np.sqrt(esq.astype(np.float64))
    tol = tol_factor * 2.0 ** -9 * zn * (en[b][:, None] + en[None, :]) + 2.0 ** -16 * (np.abs(s) + np.abs(sb)[:, None]) + 4 * g_step
    if subnormal:
        tol = tol + 2.0 ** -23 * math.sqrt(D) * (zn + en[b][:, None] + en[None, :]) + D * 2.0 ** -48
    gap = s - sb[:, None]
    gap[np.arange(len(s)), b] = np.inf
    queued = (gap <= tol).any(1)
    return b, queued, (gap / tol).min(1)


def misranked_unqueued(z, et, tol_factor, subnormal=True):
    """Rows the model says the fused kernel gets wrong: the fp16 scores pick another code than the fp64 nearest, the row is not queued,
    and the fp64 gap exceeds the fp32 tie bar."""
    b, queued, _ = fused_model(z, et, tol_factor, subnormal)
    idx, gap = nearest64(fp64_distances(z, et))
    return (b != idx) & ~queued & (gap > lookup_bar(z, et))


# ----------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("D,K", [(64, 256), (128, 512), (256, 1024)])
def test_aligned_rounding_rows_beat_the_quarter_tolerance(D, K):
    """The aligned-rounding rows are adversarial under the model: decisive in fp64 for code a, ranked b first by the fp16 scores, by more
    than 0.25 x bound + slack (not queued), and inside the full bound (tol_factor 1, queued)."""
    z, et, (ia, ib) = aligned_pair_rows(D, K, 6, seed=D)
    idx, gap = nearest64(fp64_distances(z, et))
    assert (idx == ia).all() and (gap > lookup_bar(z, et)).all()
    b, queued, ratio = fused_model(z, et, 0.25)
    assert (b == ib).all() and not queued.any()
    print(f"[aligned D={D} K={K}] fp16 gap / (0.25 x bound + slack) = {ratio.min():.3f} .. {ratio.max():.3f}")
    assert ratio.min() > 1.2
    assert misranked_unqueued(z, et, 0.25).all()
    b1, queued1, ratio1 = fused_model(z, et, 1.0)
    assert queued1.all() and not misranked_unqueued(z, et, 1.0).any()
    print(f"[aligned D={D} K={K}] fp16 gap / (1.0 x bound + slack) = {ratio1.max():.3f}")


def test_aligned_rounding_rows_are_fp16_exact_where_claimed():
    """The construction's premises: the pair codes and their -2e are fp16-exact, and fp16(z) is the fp16 grid point every element was
    built from (so every rounding error has the chosen sign)."""
    z, et, (ia, ib) = aligned_pair_rows(256, 1024, 4, seed=5)
    for c in (ia, ib):
        assert np.array_equal((np.float32(-2.0) * et[c]).astype(np.float16).astype(np.float32), np.float32(-2.0) * et[c])
    z16 = z.astype(np.float16).astype(np.float64)
    err = z16 - z.astype(np.float64)
    s = np.sign(et[ia])
    assert (np.abs(err) < 0.5 * 2.0 ** -10).all() and (np.sign(err) == -s[None, :]).all()


def test_subnormal_scales_need_the_absolute_term():
    """4096 gaussian rows against a uniform 1024 x 256 codebook, both scaled by 2^p: under a relative-only tolerance (no subnormal term)
    misranked, unqueued, decisive rows appear once operands fall below fp16's normal range (none at 2^0 and 2^-14, some at 2^-18, more at
    2^-20); with the subnormal term there are none at any scale."""
    D, K = 256, 1024
    counts = {}
    for p in (0, -14, -18, -20):
        z = gaussian_rows(4096, D, 1, 2.0 ** p)
        et = uniform_codebook(D, K, 2, 2.0 ** p)
        counts[p] = (int(misranked_unqueued(z, et, 0.25, subnormal=False).sum()), int(misranked_unqueued(z, et, 0.25).sum()))
    print(f"[subnormal] misranked, unqueued, decisive rows per scale 2^p (relative bound only, with the subnormal term): {counts}")
    assert counts[0][0] == 0 and counts[-14][0] == 0
    assert 0 < counts[-18][0] < counts[-20][0]
    assert all(c[1] == 0 for c in counts.values())


def test_kernel_constants_cap_rows():
    """zcap as the kernel computes it keeps 2 |z| |e| (1 + 2^-10) + |e|^2 below the fixed-point half range 2^(k-1), with G = 2^(k-23)."""
    for D, K in ((64, 256), (256, 1024)):
        esq = esq32(uniform_codebook(D, K, 3))
        g_step, zcap = kernel_constants(esq)
        half = g_step * 2.0 ** 22
        emax = math.sqrt(float(esq.max()))
        assert 2 * zcap * emax * (1 + 2.0 ** -10) + emax ** 2 < half
        assert half >= 17.2 * float(esq.max())


def test_nearest64_rules():
    """NaN reads as +inf and equal distances go to the smaller index: all-NaN / all-inf rows -> 0, NaN codes are never chosen."""
    et = np.array([[0, 0], [1, 1], [np.nan, 0], [1, 1]], np.float32)
    z = np.array([[1, 1], [np.nan, 0], [np.inf, 0], [-np.inf, 5], [0.9, 0.9]], np.float32)
    idx, _ = nearest64(fp64_distances(z, et))
    assert idx.tolist() == [1, 0, 0, 0, 1]
