"""Both codebook lookups (vf_vq_lookup, the fp32 kernel; vf_vq_lookup_fused, fp16 wgmma scores + the fp64 settlement of near-ties) against
fp64 nearest codes at their edges: operand scales down to fp16 subnormals, rows at the fused kernel's row cap, aligned-rounding near-ties
(tests/test_vq_lookup_edges_host.py), near-tie and duplicate pairs on 64-code set and 256-code sub-tile boundaries, several codes inside
the tolerance in one set or one column group, the >64-candidate fallback, non-finite rows and codes, and the persistent walk over many
tiles.  Rules checked on every row: a decisive row (fp64 gap to the runner-up above check_lookup's fp32 tie bar) gets the fp64 nearest
code, every chosen code lies within the bar, exact ties go to the smaller index, a row with a NaN or +-inf element gets code 0, quant is
z + (e - z) bit for bit and diff_sum is within 1e-6 of its fp64 value."""
import math

import numpy as np
import pytest
import torch

from test_vq_lookup_edges_host import aligned_pair_rows, esq32, fused_model, gaussian_rows, kernel_constants, uniform_codebook

pytestmark = pytest.mark.gpu

SHAPES = [(64, 256), (128, 512), (256, 1024)]
U = 2.0 ** -24


@pytest.fixture(scope="module")
def L(lib):
    from viewformer_b200 import _lib
    _lib.load(require_device=True)
    return _lib


def nearest64(z, et):
    """fp64 direct distances on the GPU -> (index, gap to the runner-up, chosen-code distance table); NaN reads as +inf, ties to the
    smaller index."""
    z64, e64 = z.double(), et.double()
    d = torch.cat([((e64[None] - z64[r:r + 128, None, :]) ** 2).sum(2) for r in range(0, z.shape[0], 128)])
    d = torch.nan_to_num(d, nan=math.inf)
    idx = d.argmin(1)                                           # first minimal index
    best = d.gather(1, idx[:, None])[:, 0]
    rest = d.scatter(1, idx[:, None], math.inf)
    gap = torch.nan_to_num(rest.min(1).values - best, nan=0.0)
    return idx, gap, d


def bar(z, et):
    """check_lookup's fp32 tie bar per row (a NaN code does not count towards the largest |e|^2)."""
    z64, e64 = z.double(), et.double()
    return 4 * (z.shape[1] + 2) * U * ((z64 * z64).sum(1) + torch.nan_to_num((e64 * e64).sum(1), nan=0.0).max())


def lookups(L, z, et, tol_factor=None):
    """Both kernels on z [M, D] against Et [K, D] (all on the GPU): index-only calls first, their indices checked to lie in [0, K) before
    the calls that gather codes for quant and diff_sum.  Returns {name: (idx, quant, diff_sum)} and the fused kernel's counters."""
    K = et.shape[0]
    emb = et.t().contiguous()
    et_, esq = L.vq_prepare_codebook(emb)
    eh = L.vq_prepare_codebook_f16(et_)
    kw = {} if tol_factor is None else dict(tol_factor=tol_factor)
    calls = {"vq_lookup": lambda **a: L.vq_lookup(z, et_, esq, **a),
             "vq_lookup_fused": lambda **a: L.vq_lookup_fused(z, et_, esq, eh, emb_dk=emb, **kw, **a)}
    out = {}
    for name, fn in calls.items():
        idx = fn(want_quant=False, want_diff=False)[0]
        torch.cuda.synchronize()
        lo, hi = int(idx.min()), int(idx.max())
        assert 0 <= lo and hi < K, f"{name}: index out of range [{lo}, {hi}] for K = {K}"
        out[name] = fn()
    cnt = L.vq_lookup_fused(z, et_, esq, eh, emb_dk=emb, want_quant=False, want_diff=False, return_counts=True, **kw)[3]
    torch.cuda.synchronize()
    return out, cnt.cpu()


def check(tag, L, z, et, expect=None, tol_factor=None):
    """Runs both lookups and checks every rule; expect = {row: index} pins rows (exact ties, non-finite rows).  Returns the fused kernel's
    (PAIR, SETS) counts."""
    z, et = z.contiguous().cuda(), et.contiguous().cuda()
    M = z.shape[0]
    out, cnt = lookups(L, z, et, tol_factor)
    want, gap, d = nearest64(z, et)
    b = bar(z, et)
    decisive = gap > b
    finite = torch.isfinite(z).all(1)
    expect = dict(expect or {})
    for r in torch.nonzero(~finite)[:, 0].tolist():
        expect.setdefault(r, 0)
    for name, (idx, quant, dsum) in out.items():
        bad = torch.nonzero(decisive & (idx != want))[:, 0]
        assert bad.numel() == 0, f"[{tag}] {name}: {bad.numel()} decisive rows off the fp64 nearest code, first row {int(bad[0])}: " \
                                 f"got {int(idx[bad[0]])} want {int(want[bad[0]])}, gap {float(gap[bad[0]]):.3e} > bar {float(b[bad[0]]):.3e}"
        over = (d.gather(1, idx[:, None])[:, 0] - d.gather(1, want[:, None])[:, 0])[finite]
        assert not bool((over > b[finite]).any()), f"[{tag}] {name}: a chosen code lies beyond the tie bar ({float(over.max()):.3e})"
        for r, i in expect.items():
            assert int(idx[r]) == i, f"[{tag}] {name}: row {r} got {int(idx[r])}, want {i}"
        e = et[idx]
        q_want = z + (e - z)
        same = (quant == q_want) | (torch.isnan(quant) & torch.isnan(q_want))
        assert bool(same.all()), f"[{tag}] {name}: quant differs from z + (e - z)"
        d64 = float(((e.double() - z.double()) ** 2).sum())
        got = float(dsum.reshape(-1)[0])
        if math.isfinite(d64):
            assert abs(got - d64) <= 1e-6 * d64 + 1e-300, f"[{tag}] {name}: diff_sum {got!r} vs fp64 {d64!r}"
        else:
            assert not math.isfinite(got), f"[{tag}] {name}: diff_sum {got!r} vs fp64 {d64!r}"
    assert int(cnt[0]) + int(cnt[1]) <= M
    print(f"[{tag}] M={M} decisive {int(decisive.sum())}, settled exactly: PAIR {int(cnt[0])}, SETS {int(cnt[1])}")
    return int(cnt[0]), int(cnt[1])


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


# ----------------------------------------------------------------------------------------------- scales and the row cap
@pytest.mark.parametrize("D,K", SHAPES)
@pytest.mark.parametrize("p", [0, -8, -14, -16, -18, -20, -24])
def test_scale_sweep(L, D, K, p):
    """Gaussian rows and a uniform codebook scaled together by 2^p (exact): below 2^-14 the fp16 operands are subnormal, and the fused
    kernel's tolerance has to bound their absolute rounding."""
    z = t(gaussian_rows(2048, D, 10 + D, 2.0 ** p))
    et = t(uniform_codebook(D, K, 20 + K, 2.0 ** p))
    check(f"scale 2^{p} D={D} K={K}", L, z, et)


@pytest.mark.parametrize("D,K", SHAPES)
def test_rows_at_the_row_cap(L, D, K):
    """Rows with |z| at 0.98x and 1.02x the fused kernel's zcap (computed as the kernel does): just inside the fixed-point range, and just
    outside it (decided by the exact pass)."""
    et = uniform_codebook(D, K, 30 + K)
    _, zcap = kernel_constants(esq32(et))
    z = gaussian_rows(512, D, 31 + D).astype(np.float64)
    z /= np.linalg.norm(z, axis=1, keepdims=True)
    z[:256] *= 0.98 * zcap
    z[256:] *= 1.02 * zcap
    check(f"row cap D={D} K={K} zcap={zcap:.1f}", L, t(z.astype(np.float32)), t(et))


# ----------------------------------------------------------------------------------------------- aligned fp16 roundings
@pytest.mark.parametrize("D,K", SHAPES)
def test_aligned_rounding_near_ties(L, D, K):
    """Rows whose fp16 roundings all favour the wrong code of a pair by 1.7x the 0.25 x bound tolerance (host model), decisive in fp64:
    the default (worst-case) tolerance settles them exactly; what 0.25 does is printed."""
    for pair in ((3, K - 50), (64, 65), (0, K - 1)):
        z, et, (ia, ib) = aligned_pair_rows(D, K, 64, seed=D + pair[0], pair=pair)
        _, _, ratio = fused_model(z, et, 0.25)
        z_, et_ = t(z), t(et)
        check(f"aligned D={D} K={K} pair={pair} model ratio {ratio.min():.3f}", L, z_, et_, expect={r: ia for r in range(64)})
        zc, ec = z_.cuda(), et_.cuda()
        et2, esq = L.vq_prepare_codebook(ec.t().contiguous())
        q, _, _ = L.vq_lookup_fused(zc, et2, esq, L.vq_prepare_codebook_f16(et2), want_quant=False, want_diff=False, tol_factor=0.25)
        print(f"[aligned D={D} K={K} pair={pair}] tol_factor 0.25: {int((q.cpu() != ia).sum())}/64 rows misranked")


# ----------------------------------------------------------------------------------------------- set and sub-tile boundaries
def boundary_pairs(K):
    return [pq for pq in ((63, 64), (255, 256), (511, 512), (0, K - 1), (5, 40)) if pq[1] < K]


@pytest.mark.parametrize("D,K", SHAPES)
def test_pairs_on_set_and_subtile_boundaries(L, D, K):
    """Near-tie pairs (code j = code i + small offset, rows between them with an fp64 gap of +-2 and +-0.5 tie bars) and exact-duplicate
    pairs (ties -> the smaller index) at codes (63, 64), (255, 256), (511, 512), (0, K-1) and within one set."""
    rng = np.random.default_rng(D + K)
    base = uniform_codebook(D, K, 40 + K).astype(np.float64)
    for i, j in boundary_pairs(K):
        et = base.copy()
        et[j] = et[i] + 0.05 * rng.standard_normal(D)
        et32 = et.astype(np.float32)
        e_i, e_j = et32[i].astype(np.float64), et32[j].astype(np.float64)
        w = e_j - e_i
        mid = 0.5 * (e_i + e_j)
        rows = []
        b0 = 4 * (D + 2) * U * ((mid * mid).sum() + (et32.astype(np.float64) ** 2).sum(1).max())
        for f in (2.0, -2.0, 0.5, -0.5) * 8:
            n = rng.standard_normal(D)
            n -= n.dot(w) / w.dot(w) * w
            zr = mid + 0.02 * n / np.linalg.norm(n) * math.sqrt(D)
            zr += f * b0 / (2 * w.dot(w)) * w                                # |z-e_i|^2 - |z-e_j|^2 = 2 lambda |w|^2 = f * bar
            rows.append(zr)
        check(f"near-tie pair ({i},{j}) D={D} K={K}", L, t(np.array(rows, np.float32)), t(et32))
        dup = base.astype(np.float32).copy()
        dup[j] = dup[i]
        zd = dup[i][None, :] + 0.1 * rng.standard_normal((32, D)).astype(np.float32)
        check(f"duplicate pair ({i},{j}) D={D} K={K}", L, t(zd), t(dup), expect={r: i for r in range(32)})


# ----------------------------------------------------------------------------------------------- codes hidden behind the reported keys
@pytest.mark.parametrize("D,K", SHAPES)
def test_many_codes_inside_the_tolerance(L, D, K):
    """Four codes of one 64-code set within the tolerance of each other (only two per set reach the merge), and one code per sub-tile of
    one column group plus more in its first set (only three per column group reach the merge): the exact pass must find the hidden ones."""
    rng = np.random.default_rng(K + 7)
    base = uniform_codebook(D, K, 50 + K).astype(np.float64)
    groups = {"one set": [17, 18, 19, 20, 41],
              "one column group": [7 + 256 * n for n in range(K // 256)] + [8, 9, 30]}
    for tag, codes in groups.items():
        et = base.copy()
        c = et[codes[0]].copy()
        for k in codes:
            et[k] = c + 2e-3 * rng.standard_normal(D)
        et32 = et.astype(np.float32)
        z = (c[None, :] + 0.3 * rng.standard_normal((256, D))).astype(np.float32)
        check(f"{tag} {codes} D={D} K={K}", L, t(z), t(et32))


@pytest.mark.parametrize("D,K", SHAPES)
def test_all_codes_equidistant(L, D, K):
    """z = 0 against sign-flipped copies of one vector: every fp64 distance is the same, every code is a candidate (the >64-candidate
    fallback of the exact pass), and the index is 0."""
    rng = np.random.default_rng(K)
    v = rng.uniform(0.5, 1.5, D)
    et = (v[None, :] * rng.choice([-1.0, 1.0], (K, D))).astype(np.float32)
    check(f"equidistant D={D} K={K}", L, torch.zeros(40, D), t(et), expect={r: 0 for r in range(40)})


# ----------------------------------------------------------------------------------------------- non-finite values
@pytest.mark.parametrize("D,K", SHAPES)
def test_non_finite_rows_and_codes(L, D, K):
    """Rows with one NaN, +inf or -inf element and all-NaN rows get code 0 in both kernels (their fp64 distances are all NaN or +inf: NaN
    reads as +inf, ties go to the smaller index); a NaN code is never chosen for a finite row; a code beyond the fused kernel's fp16
    codebook range sends every row to the exact pass."""
    et = uniform_codebook(D, K, 60 + K)
    z = gaussian_rows(300, D, 61 + D)
    z[3, 5] = np.nan
    z[4, D - 1] = np.inf
    z[5, 0] = -np.inf
    z[6] = np.nan
    z[7, 1], z[7, 2] = np.inf, -np.inf
    z[130, 9] = np.nan
    z[299, 0] = np.inf
    check(f"non-finite rows D={D} K={K}", L, t(z), t(et))
    zf = gaussian_rows(300, D, 62 + D)
    zf[:20] = et[5]                                                    # rows at the NaN code's finite original
    zf[:20, 3] = 0.0
    want, gap, _ = nearest64(t(zf).cuda(), t(et).cuda())
    decisive = (gap > bar(t(zf).cuda(), t(et).cuda())).cpu()
    expect = {r: int(want[r]) for r in torch.nonzero(decisive)[:, 0].tolist()}     # decisive against the codebook without the odd code
    nan_code = et.copy()
    nan_code[5, 3] = np.nan
    check(f"NaN code D={D} K={K}", L, t(zf), t(nan_code), expect={r: i for r, i in expect.items() if i != 5})
    huge = et.copy()
    huge[K - 2] = 4.0e4                                                # |e|^2 = 1.6e9 D: outside codebook_ok's range
    check(f"huge code D={D} K={K}", L, t(zf), t(huge), expect={r: i for r, i in expect.items() if i != K - 2})


# ----------------------------------------------------------------------------------------------- persistent walk
def test_persistent_walk_with_special_rows(L):
    """M = 2 * 132 * 128 + 77 rows (every CTA walks several tiles, ragged tail): exact-code rows, exact-duplicate ties, near-tie rows,
    non-finite rows and zero rows at tile starts, tile ends and in the tail."""
    D, K = 256, 1024
    M = 2 * 132 * 128 + 77
    rng = np.random.default_rng(5)
    et = uniform_codebook(D, K, 70)
    et[901] = et[900]                                                  # duplicate pair: ties -> 900
    z = gaussian_rows(M, D, 71)
    spots = sorted({r for tile in (0, 1, 131, 132, 263) for r in (128 * tile, 128 * tile + 127)} | set(range(M - 77, M, 7)) | {M - 1})
    expect = {}
    for n, r in enumerate(spots):
        kind = n % 5
        if kind == 0:
            z[r] = et[n % K]
            expect[r] = n % K if n % K != 901 else 900
        elif kind == 1:
            z[r] = et[900] + 0.01 * rng.standard_normal(D)
            expect[r] = 900
        elif kind == 2:
            a, b = et[10].astype(np.float64), et[700].astype(np.float64)
            z[r] = 0.5 * (a + b) + 1e-3 * rng.standard_normal(D)
        elif kind == 3:
            z[r, n % D] = (np.nan, np.inf, -np.inf)[n % 3]
        else:
            z[r] = 0.0
    pair, sets = check(f"persistent walk M={M}", L, t(z), t(et), expect=expect)
    assert pair + sets <= M
