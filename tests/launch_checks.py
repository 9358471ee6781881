"""Pure checkers of the libvf_b200 wrappers in ``viewformer_b200._lib``: each one restates a wrapper's result in fp64 from the operand
values the kernel consumed (bf16 as stored, fp32 read as TF32 by the tensor cores, split-fp16 pairs as hi + lo 2^-11, the bf16 operands a
weight-gradient transposer rounds), so that only accumulation order and output rounding separate kernel and reference.  A check returns
the worst ratio of error to its bar (<= 1 passes); bit-for-bit conditions return inf when they fail.

Bars, elementwise (u = 2^-24):
  GEMM / conv / weight gradient:  |got - ref| <= 2 K u (|alpha| S + |bias| + |residual|),  S = sum_k |a_k b_k|, K the reduction length
      (the exact-mode bar of DESIGN.md section 7: a length-K fp32 sum of exactly represented products).  After GELU the bar is multiplied
      by 1.13 (the largest slope of GELU) and gains 4 u |ref| (evaluation of erf).  A bf16 output is rounded once more: bf16 carries 8
      significant bits, so its unit roundoff is 2^-8 and the bar becomes (1 + 2^-8) bar + 2^-8 |ref| (the rounding acts on a value already
      within bar of ref); bf16-output GEMMs of the workloads reach 0.99 of it.  ``out2`` must be ``out`` converted, bit for bit.  Fused
      GroupNorm sums ``_gn_sums`` of an image and group: within 1e-5 of the fp64 sum / sum of squares of the stored fp32 output (relative to
      sum |y| and sum y^2), 2^-8 when the stored output is bf16 (the sums come from the fp32 accumulators, the stored values are rounded once).
  attention forward:  |O - O64| <= (2^-8 + n u) sum_j p_j |v_j| + 2^-8 |O64|, p the exact probabilities after dropout and its 1 / (1 - rate),
      n the visible keys: the unnormalised P is rounded once to bf16 (unit roundoff 2^-8 per term), the fp32 P.V and row sums over n keys
      add n u, and the output is rounded once to bf16 (2^-8 |O|); out_f32 drops the output term.
      LSE: |lse - lse64| <= 2^-20 |row max| + n 2^-23 + 2 dh u max_j sum_c |q_c k_jc| (ex2 / log and the fp32 row sum over n keys, and the
      fp32 scores).
  attention backward (P recomputed from the given lse, D = rowsum(dO * out_f32) from the given out_f32, as the kernel does):
      dV_j <= (2^-8 + n u) sum_q p'_qj |dO_q|   (dropped P rounded once to bf16, unit roundoff 2^-8; fp32 sums over the n query rows),
      dQ_q <= 2^-7 sum_j p_qj (|dP'_qj| + |D_q| + 2^-14 (|dO_q|.|V_j| m_qj + |dO_q|.|O_q|)) |K_j|, dK likewise with |Q_q|: dS = P (dP' - D) is
      rounded once to bf16 (2^-8), which leaves a factor 2 for the fp32 sums; the 2^-14 term covers the fp32 dot products behind dP and D
      (64 terms, 2^-18 each, times 4) when they cancel.  p' = dropped probabilities, dP' = m (dO . V), m the dropout multiplier.
  codebook lookup: the chosen code's fp64 distance is within a near-tie tolerance of the minimum (and equals ``ref_lookup``'s index when the
      hook is set), quant == z + (e - z) bit for bit, the distance sum within 1e-6 relative.

The checkers are device-agnostic torch code.  Device-specific pieces are the HOOKS: the bf16 GroupNorm+swish operand of the fused-norm conv
and of the bf16 weight-gradient transposer, the dropout mask of the attention kernels, the reference lookup, and the number of resident
CTAs of the persistent attention and tensor-core GEMM / conv kernels (which (batch, head) pairs, batch entries and images a CTA computes
as its second or later work item).
"""
import math
import random

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
GELU_SLOPE = 1.13
BF16_OUT = 2.0 ** -8
ACT_GELU, BIAS_N, BIAS_M = 1, 1, 2


def _gn_apply_bf16_torch(x, mr, gamma, beta, swish):
    """GroupNorm with given (mean, rstd) [N, groups, 2] [+ swish], fp32 arithmetic, one rounding to bf16 (vf_groupnorm_apply's bf16 output)."""
    n, h, w, c = x.shape
    g = mr.shape[1]
    xf = x.float().reshape(n, h * w, g, c // g)
    y = ((xf - mr[:, None, :, None, 0]) * mr[:, None, :, None, 1]).reshape(n, h, w, c) * gamma.float() + beta.float()
    if swish:
        y = y / (1.0 + torch.exp(-y))
    return y.to(torch.bfloat16)


def _dropout_mask_missing(shape, rate, seed, device):
    raise RuntimeError("launch_checks.HOOKS['dropout_mask'] is not set: the attention checkers need the kernels' dropout mask")


HOOKS = {
    "gn_apply_bf16": _gn_apply_bf16_torch,       # (x [n,h,w,c], mean_rstd [n,g,2], gamma, beta, swish) -> bf16 operand
    "dropout_mask": _dropout_mask_missing,       # (shape, rate, seed, device) -> fp32 multipliers (0 or 1 / (1 - rate))
    "ref_lookup": None,                          # (z_rows, et, esq) -> int64 indices, or None: fp64 argmin with a near-tie tolerance
    "gn_mean_rstd": None,                        # (x, groups, eps) -> the (mean, rstd) groupnorm computes when not given stats
    "attn_resident": None,                       # (train) -> CTAs of the persistent attention kernel resident at once, or None
    "tc_ctas": None,                             # () -> CTAs of the persistent tensor-core GEMM / conv kernel (the SM count), or None
}


# ----------------------------------------------------------------------------------------------- helpers
def pick(n, rng, edge=1, extra=1):
    """First ``edge``, last ``edge`` and ``extra`` seeded random indices of range(n), sorted, without repeats."""
    s = set(range(min(edge, n))) | set(range(max(0, n - edge), n))
    rest = [i for i in range(n) if i not in s] if n <= 4096 else None
    for _ in range(extra):
        if rest:
            s.add(rest.pop(rng.randrange(len(rest))))
        elif rest is None:
            s.add(rng.randrange(n))
    return sorted(s)


def pick_rows(m, rng):
    """GEMM rows: the first 128, the last 128 and 64 random ones."""
    if m <= 320:
        return torch.arange(m)
    mid = rng.sample(range(128, m - 128), min(64, m - 256))
    return torch.tensor(sorted(set(range(128)) | set(range(m - 128, m)) | set(mid)))


def view(t, off, size, stride):
    return t.as_strided(size, stride, t.storage_offset() + int(off))


def tf32(t):
    return (t.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def operand64(t):
    """fp64 value of a stored tensor-core operand: bf16 as stored, fp32 read as TF32."""
    return tf32(t).double() if t.dtype == torch.float32 else t.double()


def split_pair(v):
    """The split-fp16 pair of fp32 values: hi = fp16(v), lo = fp16((v - hi) 2^11)."""
    v = v.float()
    hi = v.half()
    return hi, ((v - hi.float()) * 2048.0).half()


def split_value(v):
    hi, lo = split_pair(v)
    return hi.double() + lo.double() / 2048.0


def ratio(err, bar):
    """max err / bar over all elements; an error where the bar is 0 is inf, NaN anywhere is inf."""
    if err.numel() == 0:
        return 0.0
    if not bool(torch.isfinite(err).all()):
        return math.inf
    r = torch.where(bar > 0, err / bar.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max())


_INT = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def bits_equal(a, b):
    """0 when a and b hold the same bits (NaN payloads included), else inf."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return math.inf
    if a.is_floating_point():
        a, b = a.view(_INT[a.element_size()]), b.view(_INT[b.element_size()])
    return 0.0 if torch.equal(a, b) else math.inf


def _epilogue(acc, s, K, ba, bias, res, out_bf16):
    """ref and bar of C = act(alpha acc + bias) + residual."""
    alpha = float(ba.get("alpha", 1.0))
    pre = alpha * acc + (0.0 if bias is None else bias)
    den = abs(alpha) * s + (0.0 if bias is None else bias.abs())
    gelu = ba.get("act", 0) == ACT_GELU
    ref = F.gelu(pre) if gelu else pre
    bar = 2.0 * K * U * den * (GELU_SLOPE if gelu else 1.0)
    if res is not None:
        ref = ref + res
        bar = bar + 2.0 * K * U * res.abs()
    if gelu:
        bar = bar + 4 * U * ref.abs()
    if out_bf16:
        bar = (1 + BF16_OUT) * bar + BF16_OUT * ref.abs()
    return ref, bar


def _outputs(out, out2):
    """(fp32 output | None, bf16 output | None) of the tensor-core epilogue."""
    f32 = b16 = None
    for o in (out, out2):
        if o is None:
            continue
        if o.dtype == torch.float32:
            f32 = o
        else:
            b16 = o
    return f32, b16


def _gn_ratio(y, sums, groups, rows_per_img, images, bf16):
    """fused (sum, sum of squares) per image and group against fp64 sums of the stored output y [rows, C] (sampled images)."""
    c = y.shape[1]
    worst = 0.0
    tol = BF16_OUT if bf16 else 1e-5
    for i in images:
        yi = y[i * rows_per_img:(i + 1) * rows_per_img].double().reshape(rows_per_img, groups, c // groups)
        s1, s2 = yi.sum((0, 2)), (yi * yi).sum((0, 2))
        a1, a2 = yi.abs().sum((0, 2)), s2
        got = sums[i].double()
        worst = max(worst, ratio((got[:, 0] - s1).abs(), tol * a1), ratio((got[:, 1] - s2).abs(), tol * a2))
    return worst


def _snapshot_if_aliased(res, out):
    if res is None or out is None:
        return res
    if res.untyped_storage().data_ptr() == out.untyped_storage().data_ptr():
        return res.clone()
    return res


# ----------------------------------------------------------------------------------------------- tensor-core walk
TC_BM = 128            # output rows (GEMM) or pixels (conv) per tile of tc_gemm_kernel


def tc_block_n(ncols):
    """Output columns per tile: 128 when Ncols > 64, else 64."""
    return 128 if ncols > 64 else 64


def tc_conv_tiling(h, w, ctot, cin, oh, ow, taps, coffs, exact, tf32):
    """(TW, TH, TN, halo) the vf_tc_gemm launcher picks for a conv: a tile of TN images x TH rows x TW columns = 128 pixels; halo for
    the plain 3x3 stride-1 pad-1 conv (exact: <= 2 channel blocks of [hi | lo] channels, one image per tile; bf16 / TF32: maps >= 16 rows,
    which then take 8 x 16-pixel tiles)."""
    tw = 16 if ow >= 16 else 8 if ow >= 8 else 4 if ow >= 4 else 2 if ow >= 2 else 1
    th = 128 // tw
    if th > oh:
        th = 1
        while th * 2 <= oh:
            th *= 2
    tn = 128 // (tw * th)
    bk = 32 if tf32 else 64
    halo = len(taps) == 9 and (oh, ow) == (h, w) and (
        (ctot == 2 * cin and cin <= 2 * bk and tn == 1 and tw >= 8) if exact else (ctot == cin and oh >= 16 and ow >= 8))
    halo = halo and all(tuple(taps[t]) == (t // 3 - 1, t % 3 - 1) and (coffs is None or coffs[t] == 0) for t in range(9))
    if halo and not exact:
        tw, th, tn = 8, 16, 1
    return tw, th, tn, halo


def tc_conv_geometry(ba):
    """(tiles_x, tiles_y, image tiles, n tiles, TN) of a tc_conv call; its tile t is (image tile, y tile, x tile, n tile), n fastest."""
    n, h, w, ctot = ba["x"].shape
    split = ba["x"].dtype == torch.float16
    cin = ctot // (2 if split else 1) if ba["cin"] is None else ba["cin"]
    oh, ow = (h, w) if ba["out_hw"] is None else ba["out_hw"]
    tw, th, tn, _ = tc_conv_tiling(h, w, ctot, cin, oh, ow, ba["taps"], ba["coffs"], split, ba["x"].dtype == torch.float32)
    return -(-ow // tw), -(-oh // th), -(-n // tn), -(-ba["w_nk"].shape[0] // tc_block_n(ba["w_nk"].shape[0])), tn


def tc_walk_tiles(total, ctas, rng):
    """Tiles of a persistent tc_gemm_kernel launch (CTA c walks tiles c, c + grid, ..., grid = min(total, ctas)) that a CTA computes as
    its second or later tile: the last tile in walk order and one seeded tile from the second round on.  Empty when no CTA walks a second
    tile or ``ctas`` is None."""
    if ctas is None or total <= ctas:
        return []
    return [total - 1, rng.randrange(ctas, total)]


# ----------------------------------------------------------------------------------------------- tensor-core GEMM
def before_tc_gemm(ba, rng):
    """Up to 3 batch entries and pick_rows, plus the batch entry and 128-row block of each tc_walk_tiles tile."""
    b1, b2 = ba["batch"]
    batches, rows = set(pick(b1 * b2, rng)), pick_rows(ba["M"], rng)
    tiles_m, tiles_n = -(-ba["M"] // TC_BM), -(-ba["N"] // tc_block_n(ba["N"]))
    walk = tc_walk_tiles(tiles_m * tiles_n * b1 * b2, HOOKS["tc_ctas"] and HOOKS["tc_ctas"](), rng)
    extra = []
    for t in walk:
        batches.add(t // (tiles_n * tiles_m))
        m0 = (t // tiles_n) % tiles_m * TC_BM
        extra += range(m0, min(m0 + TC_BM, ba["M"]))
    if extra:
        rows = torch.tensor(sorted(set(rows.tolist()) | set(extra)))
    return dict(batches=sorted(batches), rows=rows, res=_snapshot_if_aliased(ba["residual"], ba["out"]),
                gn_prev=getattr(ba["out"], "_gn_sums", None))


def _gemm_operand(t, off, rows, ld, K, lo, koff):
    """fp64 [len(rows), K] of a K-major tensor-core operand (rows ``rows`` of a matrix at element ``off``, row stride ``ld``)."""
    nrows = int(rows.max()) + 1
    if t.dtype == torch.float16:
        hi = view(t, off + koff, (nrows, K), (ld, 1))[rows]
        lo = view(t, off + koff + lo, (nrows, K), (ld, 1))[rows]
        return hi.double() + lo.double() / 2048.0
    return operand64(view(t, off + koff, (nrows, K), (ld, 1))[rows])


def check_tc_gemm(ba, result, st):
    A, B, out, out2 = ba["A"], ba["B"], ba["out"], ba["out2"]
    M, N, K, lda, ldb, ldc = ba["M"], ba["N"], ba["K"], ba["lda"], ba["ldb"], ba["ldc"]
    b1n, b2n = ba["batch"]
    a_bs, b_bs, c_bs = ba["a_bs"], ba["b_bs"], ba["c_bs"]
    koffs = ba["k_offsets"]
    lo_a = K if ba["lo_a"] is None else ba["lo_a"]
    lo_b = K if ba["lo_b"] is None else ba["lo_b"]
    rows = st["rows"].to(A.device)
    bias = ba["bias"] if ba["bias_mode"] else None
    blk = ba["causal_block"]
    bk = 128 // (2 if A.dtype != torch.float32 else 4)
    f32, b16 = _outputs(out, out2)
    got_t = f32 if f32 is not None else b16
    worst = 0.0
    for bi in st["batches"]:
        i1, i2 = divmod(bi, b2n)
        koff = 0 if koffs is None else int(koffs[i1])
        a = _gemm_operand(A, ba["a_off"] + i1 * a_bs[0] + i2 * a_bs[1], rows, lda, K, lo_a, koff)
        b = _gemm_operand(B, ba["b_off"] + i1 * b_bs[0] + i2 * b_bs[1], torch.arange(N, device=A.device), ldb, K, lo_b, 0)
        cols = torch.arange(N, device=A.device)
        keep = torch.ones((len(rows), N), dtype=torch.bool, device=A.device)
        if blk:
            m0 = rows // 128 * 128
            lim = ((((m0 + 127) // blk + 1) * blk + bk - 1) // bk * bk).clamp(max=K)
            kmask = torch.arange(K, device=A.device)[None, :] < lim[:, None]
            a = a * kmask
            if ba["causal_skip_n"]:
                keep = cols[None, :] < ((rows // blk + 1) * blk)[:, None]
        acc, s = a @ b.t(), a.abs() @ b.abs().t()
        bv = None
        if bias is not None:
            bv = bias.double()[None, :N] if ba["bias_mode"] == BIAS_N else bias.double()[rows][:, None]
        c_off = ba["c_off"] + i1 * c_bs[0] + i2 * c_bs[1]
        res = None
        if st["res"] is not None:
            res = view(st["res"], c_off, (M, N), (ldc, 1))[rows].double()
        ref, bar = _epilogue(acc, s, K, ba, bv, res, got_t.dtype == torch.bfloat16)
        got = view(got_t, c_off, (M, N), (ldc, 1))[rows].double()
        worst = max(worst, ratio(torch.where(keep, (got - ref).abs(), 0.0), bar))      # skipped tiles hold any bits, NaN included
        if f32 is not None and b16 is not None:
            worst = max(worst, bits_equal(view(b16, c_off, (M, N), (ldc, 1))[rows], view(f32, c_off, (M, N), (ldc, 1))[rows].to(torch.bfloat16)))
    gn = getattr(result, "_gn_sums", None)
    if gn is not None and gn is not st["gn_prev"]:
        rpi = ba["gn_rows_per_img"]
        y = view(got_t, ba["c_off"], (M, N), (ldc, 1))
        worst = max(worst, _gn_ratio(y, gn[0], gn[1], rpi, pick(M // rpi, random.Random(M)), got_t.dtype == torch.bfloat16))
    return worst


# ----------------------------------------------------------------------------------------------- tensor-core conv
def before_tc_conv(ba, rng):
    """First, last and one random image, plus the first image of each tc_walk_tiles tile."""
    n = ba["x"].shape[0]
    images = set(pick(n, rng))
    tiles_x, tiles_y, tiles_img, tiles_n, tn = tc_conv_geometry(ba)
    for t in tc_walk_tiles(tiles_x * tiles_y * tiles_img * tiles_n, HOOKS["tc_ctas"] and HOOKS["tc_ctas"](), rng):
        images.add(t // tiles_n // (tiles_x * tiles_y) * tn)
    return dict(images=sorted(images), res=_snapshot_if_aliased(ba["residual"], ba["out"]), gn_prev=getattr(ba["out"], "_gn_sums", None))


def _tap_conv(xv, w, taps, coffs, cin, oh, ow):
    """fp64 tap-table conv and its absolute-value twin: out[y,x] = sum_t x[y+dy_t, x+dx_t, coff_t : coff_t+cin] . w[:, t]; zero outside."""
    n, h, wd, _ = xv.shape
    p = 2
    xp = F.pad(xv, (0, 0, p, p + max(0, oh - h), p, p + max(0, ow - wd)))
    acc = s = 0.0
    for t, (dy, dx) in enumerate(taps):
        c0 = 0 if coffs is None else coffs[t]
        sl = xp[:, p + dy:p + dy + oh, p + dx:p + dx + ow, c0:c0 + cin]
        acc = acc + torch.einsum("nyxc,oc->nyxo", sl, w[:, t])
        s = s + torch.einsum("nyxc,oc->nyxo", sl.abs(), w[:, t].abs())
    return acc, s


def check_tc_conv(ba, result, st):
    x, w_nk, out, out2 = ba["x"], ba["w_nk"], result, ba["out2"]
    taps, coffs = ba["taps"], ba["coffs"]
    n, h, wd, ctot = x.shape
    split = x.dtype == torch.float16
    cin = ctot // (2 if split else 1) if ba["cin"] is None else ba["cin"]
    cout = w_nk.shape[0]
    oh, ow = (h, wd) if ba["out_hw"] is None else ba["out_hw"]
    imgs = torch.tensor(st["images"], device=x.device)
    xs = x[imgs]
    if ba["norm"] is not None:
        mr, gamma, beta, groups, swish = ba["norm"]
        assert mr.shape[1] == groups
        xv = HOOKS["gn_apply_bf16"](xs, mr[imgs], gamma, beta, bool(swish)).double()
    elif split:
        cl = ctot // 2
        xv = xs[..., :cl].double() + xs[..., cl:].double() / 2048.0
    else:
        xv = operand64(xs)
    T = len(taps)
    if split:
        wv = w_nk.reshape(cout, T, 2, cin)
        wv = wv[:, :, 0].double() + wv[:, :, 1].double() / 2048.0
    else:
        wv = operand64(w_nk).reshape(cout, T, cin)
    acc, s = _tap_conv(xv, wv, taps, coffs, cin, oh, ow)
    bias = None if ba["bias"] is None else ba["bias"].double()
    res = None if st["res"] is None else st["res"][imgs].double()
    f32, b16 = _outputs(out, out2)
    got_t = f32 if f32 is not None else b16
    ref, bar = _epilogue(acc, s, T * cin, {}, bias, res, got_t.dtype == torch.bfloat16)
    worst = ratio((got_t[imgs].double() - ref).abs(), bar)
    if f32 is not None and b16 is not None:
        worst = max(worst, bits_equal(b16[imgs], f32[imgs].to(torch.bfloat16)))
    gn = getattr(result, "_gn_sums", None)
    if gn is not None and gn is not st["gn_prev"]:
        y = got_t.reshape(n * oh * ow, cout)
        worst = max(worst, _gn_ratio(y, gn[0], gn[1], oh * ow, st["images"], got_t.dtype == torch.bfloat16))
    return worst


# ----------------------------------------------------------------------------------------------- CUDA-core GEMM and convs
def before_simt_gemm(ba, rng):
    b1, b2 = ba["batch"]
    return dict(batches=pick(b1 * b2, rng), rows=pick_rows(ba["M"], rng), res=_snapshot_if_aliased(ba["residual"], ba["out"]))


def check_simt_gemm(ba, result, st):
    A, B, out = ba["A"], ba["B"], ba["out"]
    M, N, K, ldc = ba["M"], ba["N"], ba["K"], ba["ldc"]
    (sm, sk), (bsk, bsn) = ba["a_strides"], ba["b_strides"]
    b2n = ba["batch"][1]
    a_bs, b_bs, c_bs = ba["a_bs"], ba["b_bs"], ba["c_bs"]
    rows = st["rows"].to(A.device)
    bias = ba["bias"] if ba["bias_mode"] else None
    worst = 0.0
    for bi in st["batches"]:
        i1, i2 = divmod(bi, b2n)
        a = view(A, ba["a_off"] + i1 * a_bs[0] + i2 * a_bs[1], (int(rows.max()) + 1, K), (sm, sk))[rows].double()
        b = view(B, ba["b_off"] + i1 * b_bs[0] + i2 * b_bs[1], (K, N), (bsk, bsn)).double()
        acc, s = a @ b, a.abs() @ b.abs()
        bv = None
        if bias is not None:
            bv = bias.double()[None, :N] if ba["bias_mode"] == BIAS_N else bias.double()[rows][:, None]
        c_off = ba["c_off"] + i1 * c_bs[0] + i2 * c_bs[1]
        res = None if st["res"] is None else view(st["res"], c_off, (M, N), (ldc, 1))[rows].double()
        ref, bar = _epilogue(acc, s, K, ba, bv, res, out.dtype == torch.bfloat16)
        got = view(out, c_off, (M, N), (ldc, 1))[rows].double()
        worst = max(worst, ratio((got - ref).abs(), bar))
    return worst


def _window_conv(xv, w, kh, stride, pad, oh, ow):
    """fp64 conv over the (already upsampled) image: out[y,x] = sum x[y s - pad_t + ky, x s - pad_l + kx] . w[ky,kx]; zero outside."""
    n, h, wd, c = xv.shape
    xp = F.pad(xv, (0, 0, pad[1], kh + stride * ow, pad[0], kh + stride * oh))
    acc = s = 0.0
    for ky in range(kh):
        for kx in range(kh):
            sl = xp[:, ky:ky + stride * (oh - 1) + 1:stride, kx:kx + stride * (ow - 1) + 1:stride]
            acc = acc + torch.einsum("nyxc,co->nyxo", sl, w[ky, kx])
            s = s + torch.einsum("nyxc,co->nyxo", sl.abs(), w[ky, kx].abs())
    return acc, s


def before_conv(ba, rng):
    x = ba.get("x", ba.get("dy"))
    out = ba.get("out")
    return dict(images=pick(x.shape[0], rng), res=_snapshot_if_aliased(ba.get("residual"), out),
                gn_prev=None if out is None else getattr(out, "_gn_sums", None))


def _check_window_conv(ba, result, st, kh, stride, pad, upsample, res_t):
    x, w_kn = ba["x"], ba["w_kn"]
    cin, cout = x.shape[-1], w_kn.shape[1]
    imgs = torch.tensor(st["images"], device=x.device)
    xv = x[imgs].double()
    if upsample:
        xv = xv.repeat_interleave(2, 1).repeat_interleave(2, 2)
    oh, ow = result.shape[1:3]
    acc, s = _window_conv(xv, w_kn.double().reshape(kh, kh, cin, cout), kh, stride, pad, oh, ow)
    bias = None if ba["bias"] is None else ba["bias"].double()
    res = None if res_t is None else res_t[imgs].double()
    ref, bar = _epilogue(acc, s, kh * kh * cin, {}, bias, res, result.dtype == torch.bfloat16)
    worst = ratio((result[imgs].double() - ref).abs(), bar)
    gn = getattr(result, "_gn_sums", None)
    if gn is not None and gn is not st["gn_prev"]:
        worst = max(worst, _gn_ratio(result.reshape(-1, cout), gn[0], gn[1], oh * ow, st["images"], False))
    return worst


def check_simt_conv(ba, result, st):
    return _check_window_conv(ba, result, st, ba["kh"], ba["stride"], ba["pad"], ba["upsample"], st["res"])


def check_conv3x3_small_cin(ba, result, st):
    return _check_window_conv(ba, result, st, 3, 1, (1, 1), False, None)


check_conv3x3_small_cout = check_conv3x3_small_cin


def check_simt_conv_dgrad_s2(ba, result, st):
    """dx of the Downsample conv (pad (0,1,0,1), VALID stride 2): dx[2 oy + ky, 2 ox + kx] += dy[oy, ox] . w[ky, kx]^T."""
    dy, w = ba["dy"], ba["w_dgrad_kn"]
    n, oh, ow, cout = dy.shape
    h, wd = ba["in_hw"]
    cin = w.shape[1]
    imgs = torch.tensor(st["images"], device=dy.device)
    d = dy[imgs].double()
    wv = w.double().reshape(3, 3, cout, cin)
    big = torch.zeros((len(imgs), 2 * oh + 2, 2 * ow + 2, cin), dtype=torch.float64, device=dy.device)
    sbig = torch.zeros_like(big)
    for ky in range(3):
        for kx in range(3):
            big[:, ky:ky + 2 * oh:2, kx:kx + 2 * ow:2] += torch.einsum("nyxo,oc->nyxc", d, wv[ky, kx])
            sbig[:, ky:ky + 2 * oh:2, kx:kx + 2 * ow:2] += torch.einsum("nyxo,oc->nyxc", d.abs(), wv[ky, kx].abs())
    ref, s = big[:, :h, :wd], sbig[:, :h, :wd]
    return ratio((result[imgs].double() - ref).abs(), 2.0 * 9 * cout * U * s)


# ----------------------------------------------------------------------------------------------- weight gradients
def before_wgrad(ba, rng):
    return dict(dw=ba["dw"].clone() if "dw" in ba else ba["dw_kn"].clone())


def _wgrad_window(xv, dy, kh, stride, pad):
    """fp64 dW [kh, kh, Cin, Cout] = sum over output pixels of x(gathered as the forward conv) dy, and its absolute-value twin."""
    n, oh, ow, cout = dy.shape
    xp = F.pad(xv, (0, 0, pad[1], kh + stride * ow, pad[0], kh + stride * oh))
    acc = torch.zeros((kh, kh, xv.shape[-1], cout), dtype=torch.float64, device=xv.device)
    s = torch.zeros_like(acc)
    for ky in range(kh):
        for kx in range(kh):
            sl = xp[:, ky:ky + stride * (oh - 1) + 1:stride, kx:kx + stride * (ow - 1) + 1:stride]
            acc[ky, kx] = torch.einsum("nyxc,nyxo->co", sl, dy)
            s[ky, kx] = torch.einsum("nyxc,nyxo->co", sl.abs(), dy.abs())
    return acc.reshape(-1, cout), s.reshape(-1, cout)


def _wgrad_ratio(got, pre, acc, s, K):
    ref = acc + pre
    return ratio((got - ref).abs(), 2.0 * K * U * (s + pre.abs()))


def check_conv_wgrad(ba, result, st):
    x, dy, dw = ba["x"], ba["dy"], ba["dw"]
    kh = ba["kh"]
    xv = x.double()
    if ba["upsample"]:
        xv = xv.repeat_interleave(2, 1).repeat_interleave(2, 2)
    acc, s = _wgrad_window(xv, dy.double(), kh, ba["stride"], ba["pad"])
    cout = dy.shape[-1]
    so = (cout, 1) if ba["so"] is None else ba["so"]
    k = acc.shape[0]
    got = view(dw, 0, (k, cout), so).double()
    pre = view(st["dw"], 0, (k, cout), so).double()
    return _wgrad_ratio(got, pre, acc, s, dy.shape[0] * dy.shape[1] * dy.shape[2])


def _wgrad_tc_check(x, dy, dw, st, *, bf16, conv, norm=None, upsample=False, accumulate=True):
    if bf16:
        if norm is not None:
            mr, gamma, beta, swish = norm
            xv = HOOKS["gn_apply_bf16"](x, mr, gamma, beta, bool(swish)).double()
        else:
            xv = x.to(torch.bfloat16).double()
        dv = dy.to(torch.bfloat16).double()
    else:
        xv, dv = split_value(x), split_value(dy)
    pre = st["dw"].double() if accumulate else torch.zeros_like(st["dw"], dtype=torch.float64)
    if conv:
        if upsample:
            xv = xv.repeat_interleave(2, 1).repeat_interleave(2, 2)
        acc, s = _wgrad_window(xv, dv, 3, 1, (1, 1))
        K = dy.shape[0] * dy.shape[1] * dy.shape[2]
    else:
        xr, dr = xv.reshape(-1, x.shape[-1]), dv.reshape(-1, dy.shape[-1])
        acc, s = xr.t() @ dr, xr.abs().t() @ dr.abs()
        K = xr.shape[0]
    return _wgrad_ratio(dw.double(), pre, acc, s, K)


def check_conv_wgrad_tc(ba, result, st):
    return _wgrad_tc_check(ba["x"], ba["dy"], ba["dw"], st, bf16=False, conv=True, accumulate=ba["accumulate"])


def check_conv_wgrad_bf16(ba, result, st):
    return _wgrad_tc_check(ba["x"], ba["dy"], ba["dw"], st, bf16=True, conv=True, norm=ba["norm"], upsample=ba["upsample"],
                           accumulate=ba["accumulate"])


def check_dense_wgrad_tc(ba, result, st):
    return _wgrad_tc_check(ba["x_rows"], ba["dy_rows"], ba["dw_kn"], st, bf16=False, conv=False, accumulate=ba["accumulate"])


def check_dense_wgrad_bf16(ba, result, st):
    return _wgrad_tc_check(ba["x_rows"], ba["dy_rows"], ba["dw_kn"], st, bf16=True, conv=False, accumulate=ba["accumulate"])


# ----------------------------------------------------------------------------------------------- attention
ATTN_QT, ATTN_KT = 128, 64         # query rows per work item and keys per tile of attn_block_causal_kernel


def attn_items(B, H, S, first_query=0):
    """Work items of one persistent attention launch (attn_launch): B H n_qtiles, n_qtiles = ceil(S / 128) - first_query / 128."""
    return B * H * (-(-S // ATTN_QT) - first_query // ATTN_QT)


def attn_item(item, B, H, S, block, first_query=0, stream=0, skip_view=-1):
    """(b, h, n_kt) of work item ``item`` (item_coords of vf_attn_fused.cu): heaviest query tile first, then batch * head; n_kt = the key
    tiles the item walks (stream >= 1: q0/64 + 3, or + 1 when the tile holds one view; an empty view slot of the KV cache is not walked)."""
    qt0 = first_query // ATTN_QT
    n_qt = -(-S // ATTN_QT) - qt0
    BH = B * H
    q0 = (qt0 + n_qt - 1 - item // BH) * ATTN_QT
    last_q = min(q0 + ATTN_QT, S) - 1
    n_kt = -(-min(S, (last_q // block + 1) * block) // ATTN_KT)
    if stream > 0:
        n_kt = q0 // ATTN_KT + (3 if q0 + ATTN_KT < S else 1)
    elif 0 <= skip_view < n_kt:
        n_kt -= 1
    bh = item % BH
    return bh // H, bh % H, n_kt


def attn_walk_pairs(B, H, S, block, resident, rng, first_query=0, stream=0, skip_view=-1):
    """(b, h) pairs a persistent launch computes as some CTA's second or later work item (CTA c walks items c, c + grid, ...): the last
    item in walk order (always (B - 1, H - 1), which the plain sample holds as well), and one seeded item whose CTA walked an item with
    a different n_kt before it, so the K / V ring counters and parities it starts from were carried across items of different lengths
    (any later item when every item has the same n_kt).  Empty when no CTA walks a second item or ``resident`` is None."""
    items = attn_items(B, H, S, first_query)
    if resident is None or items <= resident:
        return []
    coords = [attn_item(i, B, H, S, block, first_query, stream, skip_view) for i in range(items)]
    later = [i for i in range(resident, items) if any(coords[j][2] != coords[i][2] for j in range(i % resident, i, resident))]
    later = later or list(range(resident, items))
    return [coords[-1][:2], coords[later[rng.randrange(len(later))]][:2]]


def _heads(ba, rng, train):
    """The (batch, head) pairs an attention check covers: first, last and one random pair, and the attn_walk_pairs of the launch (of the
    training instance's stream-0 launch for the backward, which is not persistent but reads that forward's lse and out_f32)."""
    B, H = ba["B"], ba["H"]
    pairs = [(b, h) for b in range(B) for h in range(H)]
    sampled = {pairs[i] for i in pick(len(pairs), rng)}
    resident = None if HOOKS["attn_resident"] is None else HOOKS["attn_resident"](train)
    walk = attn_walk_pairs(B, H, ba["S"], ba["block"], resident, rng, first_query=int(ba.get("first_query", 0)),
                           stream=int(ba.get("stream", 0)), skip_view=int(ba.get("skip_view", -1)))
    return sorted(sampled | set(walk))


def _stream_qkv(qk, vt, s, S, d, b, h):
    """fp64 q, k [S, 64] and v [S, 64] of stream s, batch b, head h (qk [B, ns*S, 2d], vt [B, d, ns*S])."""
    q = qk[b, s * S:(s + 1) * S, h * 64:(h + 1) * 64].double()
    k = qk[b, s * S:(s + 1) * S, d + h * 64:d + (h + 1) * 64].double()
    v = vt[b, h * 64:(h + 1) * 64, s * S:(s + 1) * S].double().t()
    return q, k, v


def _logits(qk, vt, S, d, b, h, stream, block, skip_view=-1):
    """Scores [S, cols], visibility, keys and values of one stream (cols = S for stream 0, 2S for streams >= 1: stream-0 keys | own keys).
    Keys no row may see (the empty view slot of the KV cache) are zeroed: the kernel never reads them and they may hold any bits."""
    view_ = torch.arange(S, device=qk.device) // block
    q, k, v = _stream_qkv(qk, vt, stream, S, d, b, h)
    if stream == 0:
        vis = view_[None, :] <= view_[:, None]
        if skip_view >= 0:
            vis = vis & (view_ != skip_view)[None, :]
        kk, vv = k, v
    else:
        _, k0, v0 = _stream_qkv(qk, vt, 0, S, d, b, h)
        vis = torch.cat([view_[None, :] < view_[:, None], view_[None, :] == view_[:, None]], 1)
        kk, vv = torch.cat([k0, k]), torch.cat([v0, v])
    dead = ~vis.any(0)
    kk, vv = kk.masked_fill(dead[:, None], 0.0), vv.masked_fill(dead[:, None], 0.0)
    return q, (q @ kk.t()).masked_fill(~vis, 0.0), vis, kk, vv


def _softmax(sc, vis):
    sc = sc.masked_fill(~vis, -math.inf)
    lse = torch.logsumexp(sc, 1)
    p = torch.exp(sc - lse[:, None])
    return p, lse, sc.amax(1)


def _drop(shape, rate, seed, device):
    return HOOKS["dropout_mask"](shape, rate, seed, device).double() if rate > 0 else None


def _attn_forward(ba, st, S, stream, block, out_rows, skip_view=-1, rate=0.0, seed=0, lse=None, out_f32=None, t0=0):
    qk, vt, B, H, d = ba["qk"], ba["vt"], ba["B"], ba["H"], ba["d"]
    out = out_rows.reshape(B, S, d)
    mask = None
    if rate > 0:
        cols = S if stream == 0 else 2 * S
        mask = _drop((B, H, S, cols), rate, seed, qk.device)
    worst = 0.0
    for b, h in st["heads"]:
        q, sc, vis, kk, vv = _logits(qk, vt, S, d, b, h, stream, block, skip_view)
        p, lse64, rmax = _softmax(sc, vis)
        if mask is not None:
            p = p * mask[b, h]
        o = p @ vv
        pv = p @ vv.abs()
        got = out[b, t0:, h * 64:(h + 1) * 64].double()
        pbar = (BF16_OUT + vis.sum(1, keepdim=True).double() * U) * pv
        worst = max(worst, ratio((got - o[t0:]).abs(), pbar[t0:] + BF16_OUT * o[t0:].abs()))
        if out_f32 is not None:
            g32 = out_f32.reshape(B, S, d)[b, :, h * 64:(h + 1) * 64].double()
            worst = max(worst, ratio((g32 - o).abs(), pbar))
            worst = max(worst, bits_equal(out[b, :, h * 64:(h + 1) * 64], g32.float().to(torch.bfloat16)))
        if lse is not None:
            n = vis.sum(1).double()
            qs = (q.abs() @ kk.abs().t()).masked_fill(~vis, 0).amax(1)
            bar = 2.0 ** -20 * rmax.abs() + n * 2.0 ** -23 + 2 * 64 * U * qs
            worst = max(worst, ratio((lse[b, h].double() - lse64).abs(), bar))
    return worst


def before_attn(ba, rng, train=False):
    st = dict(heads=_heads(ba, rng, train))
    if ba.get("out") is not None:
        st["out"] = ba["out"].clone()
    return st


def before_attn_train(ba, rng):
    return before_attn(ba, rng, train=True)


def check_attn_block_causal(ba, result, st):
    S, d, B = ba["S"], ba["d"], ba["B"]
    fq = int(ba["first_query"])
    t0 = (fq // 128) * 128 if fq > 0 else 0
    worst = _attn_forward(ba, st, S, 0, ba["block"], result, skip_view=int(ba["skip_view"]), t0=t0)
    if t0 > 0 and "out" in st:
        worst = max(worst, bits_equal(result.reshape(B, S, d)[:, :t0], st["out"].reshape(B, S, d)[:, :t0]))
    return worst


def check_attn_block_multiend(ba, result, st):
    return _attn_forward(ba, st, ba["S"], ba["stream"], ba["block"], result)


def check_attn_multiend_train(ba, result, st):
    return _attn_forward(ba, st, ba["S"], ba["stream"], ba["block"], result, rate=float(ba["rate"]), seed=int(ba["seed"]), lse=ba["lse"],
                         out_f32=ba["out_f32"])


def before_attn_bwd(ba, rng):
    st = dict(heads=_heads(ba, rng, True))
    st["dvqk"] = None if ba["dvqk"] is None else ba["dvqk"].clone()
    return st


def check_attn_multiend_bwd(ba, result, st):
    """dV, dQ, dK of every stream against fp64 on the kernel's operands: bf16 Q, K, V, dO, the given lse and out_f32 (D)."""
    qk, vt, dout, o32, lse = ba["qk"], ba["vt"], ba["dout"], ba["out_f32"], ba["lse"]
    B, S, ns, H, d, block = ba["B"], ba["S"], ba["n_streams"], ba["H"], ba["d"], ba["block"]
    rate, seed = float(ba["rate"]), int(ba["seed"])
    pre = st["dvqk"]
    got = result.reshape(ns, B, S, 3 * d)
    worst = 0.0
    for b, h in st["heads"]:
        sl = slice(h * 64, (h + 1) * 64)
        dv = torch.zeros((ns, S, 64), dtype=torch.float64, device=qk.device)
        dq, dk = torch.zeros_like(dv), torch.zeros_like(dv)
        bv, bq, bk = torch.zeros_like(dv), torch.zeros_like(dv), torch.zeros_like(dv)
        for s in range(ns):
            q, sc, vis, kk, vv = _logits(qk, vt, S, d, b, h, s, block)
            p = torch.exp(sc - lse[s, b, h].double()[:, None]).masked_fill(~vis, 0.0)
            m = _drop((B, H, S, sc.shape[1]), rate, seed + s, qk.device)
            m = torch.ones_like(p) if m is None else m[b, h]
            do = dout[s].reshape(B, S, d)[b, :, sl].double()
            oo = o32[s].reshape(B, S, d)[b, :, sl].double()
            D = (do * oo).sum(1)
            dpp = (do @ vv.t()) * m
            ds = p * (dpp - D[:, None])
            slack = 2.0 ** -14 * ((do.abs() @ vv.abs().t()) * m + (do.abs() * oo.abs()).sum(1)[:, None])
            w = p * (dpp.abs() + D.abs()[:, None] + slack)
            pd = p * m
            keys = [(0, slice(0, S))] if s == 0 else [(0, slice(0, S)), (s, slice(S, 2 * S))]
            dq[s] += ds @ kk
            bq[s] += w @ kk.abs()
            for ks, cs in keys:
                dv[ks] += pd[:, cs].t() @ do
                bv[ks] += pd[:, cs].t() @ do.abs()
                dk[ks] += ds[:, cs].t() @ q
                bk[ks] += w[:, cs].t() @ q.abs()
        for s in range(ns):
            for j, (ref, bar, scale) in enumerate(((dv[s], bv[s], BF16_OUT + ns * S * U), (dq[s], bq[s], 2.0 ** -7), (dk[s], bk[s], 2.0 ** -7))):
                cs = slice(j * d + h * 64, j * d + (h + 1) * 64)
                p0 = 0.0 if pre is None else pre.reshape(ns, B, S, 3 * d)[s, b, :, cs].double()
                g = got[s, b, :, cs].double()
                worst = max(worst, ratio((g - p0 - ref).abs(), scale * bar + 2 * U * (ref + p0).abs()))
    return worst


# ----------------------------------------------------------------------------------------------- codebook lookup
def before_lookup(ba, rng):
    return dict(rows=pick_rows(ba["z_rows"].shape[0], rng))


def check_lookup(ba, result, st, use_hook=True):
    z, et, esq = ba["z_rows"], ba["et"], ba["esq"]
    idx, quant, dsum = result[:3]
    m, dd = z.shape
    worst = 0.0
    ref_lookup = HOOKS["ref_lookup"] if use_hook else None
    if ref_lookup is not None:
        worst = max(worst, bits_equal(idx, ref_lookup(z, et, esq)))
    rows = st["rows"].to(z.device)
    zr, e64 = z[rows].double(), et.double()
    dist = (zr * zr).sum(1)[:, None] - 2 * zr @ e64.t() + (e64 * e64).sum(1)[None, :]
    chosen = dist.gather(1, idx[rows][:, None])[:, 0]
    tie = 4 * (dd + 2) * U * ((zr * zr).sum(1) + (e64 * e64).sum(1).max())
    worst = max(worst, ratio(chosen - dist.min(1).values, tie))
    e = et[idx]
    if quant is not None:
        worst = max(worst, bits_equal(quant, z + (e - z)))
    if dsum is not None:
        want = float(((e.double() - z.double()) ** 2).sum())
        worst = max(worst, abs(float(dsum.reshape(-1)[0]) - want) / max(1e-6 * want, 1e-300) if want > 0 else (0.0 if float(dsum) == 0 else math.inf))
    return worst


def check_vq_lookup(ba, result, st):
    return check_lookup(ba, result, st, use_hook=False)


# ----------------------------------------------------------------------------------------------- normalisation
GN_COND = []          # mean^2 / var of every GroupNorm group whose statistics were checked (the audit prints the largest)
GN_USED = {}          # (x.data_ptr(), groups) -> the (mean, rstd) the last checked gn_mean_rstd call returned (what groupnorm then consumes)


def f32(x):
    """A hyperparameter as the kernel receives it (a C float), in fp64."""
    return float(np.float32(x))


def _gn_stats64(x, groups):
    """fp64 (mean, var, mean |x|, mean x^2) [N, groups] of the stored x [N,H,W,C]."""
    n = x.shape[0]
    xg = x.double().reshape(n, -1, groups, x.shape[-1] // groups)
    m = xg.mean((1, 3))
    return m, (xg * xg).mean((1, 3)) - m * m, xg.abs().mean((1, 3)), (xg * xg).mean((1, 3))


def gn_stats_chain(n, hw, c):
    """Longest fp32 chain of vf_groupnorm_stats: a thread sums ceil(ppb / lanes) pixels of its channel quad, then folds the quad (+2); the
    block's threads and the chunks then meet in fp64 atomics."""
    lanes = 256 // (c // 4)
    chunks = max(1, min((hw + 63) // 64, (132 * 8 + n - 1) // n))
    ppb = (hw + chunks - 1) // chunks
    return (ppb + lanes - 1) // lanes + 2


def before_gn_mean_rstd(ba, rng):
    x = ba["x"]
    fused = getattr(x, "_gn_sums", None)
    return dict(fused=fused is not None and fused[1] == ba["groups"])


def check_gn_mean_rstd(ba, result, st):
    """mean / rstd against the fp64 statistics of the stored x.  Sums with relative error t (of sum |x| and sum x^2) give
    |mean err| <= t mean|x| + u |mean| and |var err| <= (2t + t^2) E x^2 + 2 t |mean| mean|x| + t^2 (mean|x|)^2, so rstd is within var_err / (2 (var + eps)) + 2u
    relatively: the conditioning factor E x^2 / var = 1 + mean^2 / var appears explicitly.  t = 1e-5 for fused sums of an fp32 output,
    2^-8 for a bf16 one (as _gn_ratio), and (K + 1) u for the statistics pass (K = gn_stats_chain; the squares round once).  Every
    checked call appends its largest mean^2 / var to GN_COND."""
    x, groups, eps = ba["x"], ba["groups"], f32(ba["eps"])
    m, v, am, m2 = _gn_stats64(x, groups)
    n, h, w, c = x.shape
    if st["fused"]:
        t = BF16_OUT if x.dtype == torch.bfloat16 else 1e-5
    else:
        t = (gn_stats_chain(n, h * w, c) + 1) * U
    got = result.double()
    verr = (2 * t + t * t) * m2 + 2 * t * m.abs() * am + t * t * am * am
    r64 = 1.0 / torch.sqrt(v.clamp_min(0) + eps)
    GN_COND.append(float((m * m / v.clamp_min(1e-300)).max()))
    if len(GN_USED) > 64:
        GN_USED.clear()
    GN_USED[(x.data_ptr(), groups)] = result
    return max(ratio((got[..., 0] - m).abs(), t * am + U * m.abs()),
               ratio((got[..., 1] - r64).abs(), r64 * (verr / (2 * (v.clamp_min(0) + eps)) + 2 * U)))


def _unlayout(y, n, h, w, c, upsample, s2d):
    """fp64 [N,H,W,C] view(s) of a groupnorm output: the 4 copies of the x2 upsample, the space-to-depth blocks, split pairs decoded."""
    if y.dtype == torch.float16:
        cl = y.shape[-1] // 2
        y = y[..., :cl].double() + y[..., cl:].double() / 2048.0
    else:
        y = y.double()
    if upsample:
        y6 = y.reshape(n, h, 2, w, 2, c)
        return [y6[:, :, a, :, b] for a in (0, 1) for b in (0, 1)]
    if s2d:
        return [y.reshape(n, h // 2, w // 2, 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, h, w, c)]
    return [y]


def before_groupnorm(ba, rng):
    return dict(images=pick(ba["x"].shape[0], rng))


def _groupnorm_stats(ba):
    """The (mean, rstd) groupnorm consumed: the given ``stats``, else what its own gn_mean_rstd call returned (recorded by
    check_gn_mean_rstd when that call is audited), else HOOKS['gn_mean_rstd']."""
    if ba["stats"] is not None:
        return ba["stats"]
    used = GN_USED.pop((ba["x"].data_ptr(), ba["groups"]), None)
    return used if used is not None else HOOKS["gn_mean_rstd"](ba["x"], ba["groups"], ba["eps"])


def check_groupnorm(ba, result, st):
    """y = ((x - mean) rstd) gamma + beta [swish] from the given (mean, rstd): 4 u (|xhat gamma| + |mean rstd gamma| + |beta|) (the
    rounded operations, and the bf16 path's folded shift beta - mean rstd gamma), times 1.1 (the largest slope of swish) + 8 u |y| (its exp
    and division); a bf16 output adds 2^-8 |y|, a split pair 2^-21 |y| + 2^-36 (hi + lo 2^-11 carries 22 bits)."""
    x = ba["x"]
    n, h, w, c = x.shape
    imgs = torch.tensor(st["images"], device=x.device)
    xv = x[imgs].double()
    if ba["normalize"]:
        g = ba["groups"]
        mr = _groupnorm_stats(ba)[imgs].double()
        cidx = torch.arange(c, device=x.device) // (c // g)
        mu, rs = mr[:, cidx, 0][:, None, None], mr[:, cidx, 1][:, None, None]
        ga, be = ba["gamma"].double(), ba["beta"].double()
        ref = (xv - mu) * rs * ga + be
        bar = 4 * U * (((xv - mu) * rs * ga).abs() + (mu * rs * ga).abs() + be.abs())
    else:
        ref, bar = xv, torch.zeros_like(xv)
    if ba["swish"]:
        ref = ref * torch.sigmoid(ref)
        bar = 1.1 * bar + 8 * U * ref.abs()
    if result.dtype == torch.bfloat16:
        bar = (1 + BF16_OUT) * bar + BF16_OUT * ref.abs()
    elif result.dtype == torch.float16:
        bar = bar + 2.0 ** -21 * ref.abs() + 2.0 ** -36
    worst = 0.0
    for got in _unlayout(result[imgs], len(imgs), h, w, c, ba["upsample"], ba["s2d"]):
        worst = max(worst, ratio((got - ref).abs(), bar))
    return worst


def before_layernorm(ba, rng):
    x = ba["x"]
    return dict(rows=pick_rows(x.numel() // x.shape[-1], rng))


def check_layernorm(ba, result, st):
    """Two fp32 passes per row (one warp): K = ceil(d / 128) quads per lane (+2 for the quad fold) + 5 shuffle levels.  The fp32 mean carries
    K u mean|x|, which every x - mean inherits: |y - y64| <= 2 (K + 4) u (|xhat| + rstd mean|x|) |gamma| + 2 u |beta| (+ 2^-8 |y| for bf16);
    an rstd off by the conditioning factor 1 + mean^2 / var would not fit (tests/test_norm_stats_gpu.py)."""
    x, d = ba["x"], ba["x"].shape[-1]
    rows = st["rows"].to(x.device)
    xv = x.reshape(-1, d)[rows].double()
    mu = xv.mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(xv.var(1, unbiased=False, keepdim=True) + f32(ba["eps"]))
    xh = (xv - mu) * rs
    ga, be = ba["gamma"].double(), ba["beta"].double()
    ref = xh * ga + be
    K = (d + 127) // 128 + 7
    bar = 2 * (K + 4) * U * (xh.abs() + rs * xv.abs().mean(1, keepdim=True)) * ga.abs() + 2 * U * be.abs()
    if result.dtype == torch.bfloat16:
        bar = (1 + BF16_OUT) * bar + BF16_OUT * ref.abs()
    return ratio((result.reshape(-1, d)[rows].double() - ref).abs(), bar)


def _gn_bwd_chains(n, hw, c):
    """(K of the group sums, K of dgamma / dbeta) of vf_groupnorm_bwd: a thread sums ppb / lanes pixels of its quad in fp32 (the group sums
    then meet in fp64); dgamma / dbeta then add the block's lanes in shared fp32 atomics and the N x chunks blocks in global ones, onto
    the value held before."""
    lanes = 256 // (c // 4)
    ppb = lanes * 128
    while ppb > lanes * 4 and ((hw + ppb - 1) // ppb) * n < 132 * 4:
        ppb >>= 1
    per = ppb // lanes
    return per + 2, per + lanes + n * ((hw + ppb - 1) // ppb) + 1


def before_groupnorm_bwd(ba, rng):
    return dict(dgamma=ba["dgamma"].clone(), dbeta=ba["dbeta"].clone())


def check_groupnorm_bwd(ba, result, st):
    """dx = rstd (g gamma - mean(g gamma) - xhat mean(g gamma xhat)) [+ add], g = dout [x swish'], from the given (mean, rstd); dgamma /
    dbeta added onto their snapshots.  The sum|terms| expressions of tests/test_backward_kernels_gpu.py::test_groupnorm_bwd with this
    kernel's chains (_gn_bwd_chains) for K; the bf16 copy must be dx rounded to nearest even, bit for bit."""
    x, dout, mr, gamma, beta, groups = ba["x"], ba["dout"], ba["mean_rstd"], ba["gamma"], ba["beta"], ba["groups"]
    n, h, w, c = x.shape
    cidx = torch.arange(c, device=x.device) // (c // groups)
    mu_c, rs_c = mr.double()[:, cidx, 0].reshape(n, 1, 1, c), mr.double()[:, cidx, 1].reshape(n, 1, 1, c)
    xh = (x.double() - mu_c) * rs_c
    g = dout.double()
    if ba["swish"]:
        z = xh * gamma.double() + beta.double()
        sg = torch.sigmoid(z)
        g = g * sg * (1 + z * (1 - sg))
    gg_ = g * gamma.double()
    m1 = gg_.reshape(n, -1, groups, c // groups).mean((1, 3))[:, cidx].reshape(n, 1, 1, c)
    m2 = (gg_ * xh).reshape(n, -1, groups, c // groups).mean((1, 3))[:, cidx].reshape(n, 1, 1, c)
    add = ba["add"]
    ref = rs_c * (gg_ - m1 - xh * m2) + (0.0 if add is None else add.double())
    xh_err = xh.abs() + rs_c * mu_c.abs() + 1.0
    dgg = gg_.abs()
    A1 = dgg.reshape(n, -1, groups, c // groups).mean((1, 3))[:, cidx].reshape(n, 1, 1, c)
    A2 = (dgg * xh_err).reshape(n, -1, groups, c // groups).mean((1, 3))[:, cidx].reshape(n, 1, 1, c)
    Kg, Kc = _gn_bwd_chains(n, h * w, c)
    s_dx = rs_c * (dgg * xh_err + A1 + xh_err * A2) + (0.0 if add is None else add.double().abs())
    worst = ratio((result.double() - ref).abs(), 4 * (Kg + 8) * U * s_dx)
    dg0, db0 = st["dgamma"].double(), st["dbeta"].double()
    worst = max(worst, ratio((ba["dgamma"].double() - dg0 - (g * xh).sum((0, 1, 2))).abs(),
                             4 * (Kc + 8) * U * (g.abs() * xh_err).sum((0, 1, 2)) + 2 * U * dg0.abs()))
    worst = max(worst, ratio((ba["dbeta"].double() - db0 - g.sum((0, 1, 2))).abs(), 4 * (Kc + 8) * U * g.abs().sum((0, 1, 2)) + 2 * U * db0.abs()))
    if ba["out_bf16"]:
        worst = max(worst, bits_equal(result._bf16, result.to(torch.bfloat16)))
    return worst


def before_layernorm_bwd(ba, rng):
    return dict(dgamma=ba["dgamma"].clone(), dbeta=ba["dbeta"].clone())


def check_layernorm_bwd(ba, result, st):
    """tests/test_backward_kernels_gpu.py::test_layernorm_bwd's bars with this kernel's chains: a row's statistics and mean(dy gamma),
    mean(dy gamma xhat) are one warp's (K = ceil(d / 32) + 5); dgamma / dbeta meet the block's 8 rows in shared fp32 atomics, then
    ceil(rows / 8) blocks in global ones, onto the snapshot (Kc = 8 + ceil(rows / 8) + 1)."""
    x, dy, gamma = ba["x"], ba["dy"], ba["gamma"]
    d = x.shape[-1]
    xv, dv = x.reshape(-1, d).double(), dy.reshape(-1, d).double()
    rows = xv.shape[0]
    mu = xv.mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(xv.var(1, unbiased=False, keepdim=True) + f32(ba["eps"]))
    xh = (xv - mu) * rs
    dg = dv * gamma.double()
    ref = rs * (dg - dg.mean(1, keepdim=True) - xh * (dg * xh).mean(1, keepdim=True))
    add = ba["add"]
    if add is not None:
        ref = ref + add.reshape(-1, d).double()
    K = (d + 31) // 32 + 5
    xh_err = xh.abs() + rs * xv.abs().mean(1, keepdim=True) + 1.0
    dgg = dg.abs()
    s_dx = rs * (dgg * xh_err + dgg.mean(1, keepdim=True) + xh_err * (dgg * xh_err).mean(1, keepdim=True))
    if add is not None:
        s_dx = s_dx + add.reshape(-1, d).double().abs()
    worst = ratio((result.reshape(-1, d).double() - ref).abs(), 4 * (K + 8) * U * s_dx)
    Kc = 8 + (rows + 7) // 8 + 1 + K
    dg0, db0 = st["dgamma"].double(), st["dbeta"].double()
    worst = max(worst, ratio((ba["dgamma"].double() - dg0 - (dv * xh).sum(0)).abs(), 4 * Kc * U * (dv.abs() * xh_err).sum(0) + 2 * U * dg0.abs()))
    worst = max(worst, ratio((ba["dbeta"].double() - db0 - dv.sum(0)).abs(), 4 * Kc * U * dv.abs().sum(0) + 2 * U * db0.abs()))
    return worst


# ----------------------------------------------------------------------------------------------- reductions
def col_sums_chain(rows):
    """K of vf_col_sums: ceil(rpb / 8) rows per thread, 8 warps folded, the row chunks' atomics, the value held before."""
    chunks = min((rows + 1023) // 1024, 1024)
    rpb = (rows + chunks - 1) // chunks
    chunks = (rows + rpb - 1) // rpb
    return (rpb + 7) // 8 + 8 + chunks + 1


def before_col_sums(ba, rng):
    return dict(out=ba["out"].clone())


def check_col_sums(ba, result, st):
    """out += column sums of x [rows, C], against the snapshot: 2 K u (sum |x| + |out0|), K = col_sums_chain(rows)."""
    x = ba["x_rows"]
    c = x.shape[-1]
    xv = x.reshape(-1, c).double()
    K = col_sums_chain(xv.shape[0])
    o0 = st["out"].double()
    return ratio((result.double() - o0 - xv.sum(0)).abs(), 2 * K * U * (xv.abs().sum(0) + o0.abs()))


def check_softmax_bwd_rows(ba, result, st):
    """dS = P (dP - sum_j P_j dP_j), one warp per row: 2 (K + 2) u P (|dP| + sum|P dP|), K = ceil(cols / 32) + 5."""
    P, dP = ba["P"], ba["dP"]
    cols = P.shape[-1]
    rows = st["rows"].to(P.device)
    p, d = P.reshape(-1, cols)[rows].double(), dP.reshape(-1, cols)[rows].double()
    K = (cols + 31) // 32 + 5
    ref = p * (d - (p * d).sum(-1, keepdim=True))
    return ratio((result.reshape(-1, cols)[rows].double() - ref).abs(), 2 * (K + 2) * U * p * (d.abs() + (p * d).abs().sum(-1, keepdim=True)))


def before_rows(key):
    def before(ba, rng):
        t = ba[key]
        return dict(rows=pick_rows(t.numel() // t.shape[-1], rng))
    return before


def check_cross_entropy_grad(ba, result, st):
    """w (softmax - (1 - s) onehot - s / cols), one warp per row: 2 u w ((K + 8) p + 4 y) with K = ceil(cols / 32) + 5 (the row sum of
    exponentials) and y the smoothed target (tests/test_backward_kernels_gpu.py::test_cross_entropy_grad with this kernel's K)."""
    lg, lab, w = ba["logits_rows"], ba["labels_i32"], ba["row_weight"]
    cols = lg.shape[-1]
    rows = st["rows"].to(lg.device)
    s = f32(ba["smoothing"])
    x = lg[rows].double()
    p = torch.softmax(x, -1)
    y = F.one_hot(lab[rows].long(), cols).double() * (1 - s) + s / cols
    wr = w[rows].double()[:, None]
    K = (cols + 31) // 32 + 5
    return ratio((result[rows].double() - wr * (p - y)).abs(), 2 * U * wr.abs() * ((K + 8) * p + 4 * y) + 1e-38)


def check_sumsq(ba, result, st):
    """sum x^2 in fp64 (squares exact): per-thread chains over a grid-stride loop, 5 shuffle levels, 8 warps, one fp64 atomic per block:
    2 K 2^-53 sum x^2."""
    x = ba["x"]
    n = x.numel()
    blocks = min((n + 255) // 256, 132 * 16)
    K = (n + blocks * 256 - 1) // (blocks * 256) + 5 + 8 + blocks
    want = (x.double() ** 2).sum()
    return ratio((result.double().reshape(-1)[:1] - want).abs(), torch.full((1,), 2 * K * 2.0 ** -53 * float(want) + 1e-300,
                                                                           dtype=torch.float64, device=x.device))


def before_migt_embed_bwd(ba, rng):
    return {k: (None if ba[k] is None else ba[k].clone()) for k in ("dwte", "dwpe", "dpose")}


def check_migt_embed_bwd(ba, result, st):
    """dwte[id] += dh (id = ids, or fixed_token where ids is null or < 0), dwpe[l] += dh, dpose[bt] += dh, onto the snapshots.  Every
    token adds with one fp32 atomic, so an element's chain is the number of tokens that hit it, plus the value held before:
    2 (hits + 1) u (|snapshot| + sum |dh|)."""
    dh, ids, BT, Lt = ba["dh"], ba["ids_i32"], ba["BT"], ba["L"]
    d = dh.shape[-1]
    tok = BT * Lt
    hd = dh.reshape(tok, d).double()
    dev = dh.device
    idx = torch.full((tok,), int(ba["fixed_token"]), dtype=torch.long, device=dev) if ids is None else ids.long().reshape(-1)
    if ids is not None:
        idx = torch.where(idx < 0, torch.full_like(idx, int(ba["fixed_token"])), idx)
    worst = 0.0
    for key, index in (("dwte", idx), ("dwpe", torch.arange(tok, device=dev) % Lt), ("dpose", torch.arange(tok, device=dev) // Lt)):
        if st[key] is None:
            continue
        b0 = st[key].double()
        want = b0.index_add(0, index, hd)
        hits = torch.zeros(b0.shape[0], dtype=torch.float64, device=dev).index_add_(0, index, torch.ones(tok, dtype=torch.float64, device=dev))
        absum = b0.abs().index_add(0, index, hd.abs())
        worst = max(worst, ratio((ba[key].double() - want).abs(), 2 * (hits[:, None] + 1) * U * absum))
    return worst


# ----------------------------------------------------------------------------------------------- elementwise
def _ranges(n, rng, block=4096):
    """Sampled flat ranges of a buffer of n elements: the first block, the last block, and 3 random blocks."""
    nb = (n + block - 1) // block
    return [slice(b * block, min(n, (b + 1) * block)) for b in pick(nb, rng, extra=3)]


def _snap(ba, keys, rng, n):
    rs = _ranges(n, rng)
    return dict(ranges=rs, snap={k: [None if ba[k] is None else ba[k].reshape(-1)[r].clone() for r in rs] for k in keys})


def before_elementwise(*keys, size="x"):
    def before(ba, rng):
        return _snap(ba, keys, rng, ba[size].numel())
    return before


def check_gelu(ba, result, st):
    """x Phi(x): 4 u |y| + 4 u |x| (erff's error on 1 + erf, which cancels for negative x) (tests/test_backward_kernels_gpu.py)."""
    worst = 0.0
    for r, x in zip(st["ranges"], st["snap"]["x"]):
        xd = x.double()
        want = xd * 0.5 * (1 + torch.erf(xd / math.sqrt(2)))
        worst = max(worst, ratio((result.reshape(-1)[r].double() - want).abs(), 4 * U * want.abs() + 4 * U * xd.abs() + 1e-38))
    return worst


def check_gelu_bwd(ba, result, st):
    """dy (Phi(x) + x phi(x)): 4 u |ref| + 4 u |dy| (1 + |x phi(x)|) (tests/test_backward_kernels_gpu.py)."""
    worst = 0.0
    for r, x, dy in zip(st["ranges"], st["snap"]["pre"], st["snap"]["dy"]):
        xd = x.double()
        cdf = 0.5 * (1 + torch.erf(xd / math.sqrt(2)))
        pdf = torch.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi)
        want = dy.double() * (cdf + xd * pdf)
        worst = max(worst, ratio((result.reshape(-1)[r].double() - want).abs(), 4 * U * want.abs() + 4 * U * dy.double().abs() * (1 + (xd * pdf).abs())))
    return worst


def check_lincomb3(ba, result, st):
    """a x + b y + c z (null operands dropped), from the snapshots (``out`` may alias ``x``): one product and two fmas, 4 u sum|terms|."""
    worst = 0.0
    for i, r in enumerate(st["ranges"]):
        terms = [f32(ba["a"]) * st["snap"]["x"][i].double()]
        for k, cf in (("y", "b"), ("z", "c")):
            if st["snap"][k][i] is not None:
                terms.append(f32(ba[cf]) * st["snap"][k][i].double())
        worst = max(worst, ratio((result.reshape(-1)[r].double() - sum(terms)).abs(), 4 * U * sum(t.abs() for t in terms) + 1e-38))
    return worst


def _update_bar(scale, m, v, gi, m1, v1, den, sq_bc2):
    """Bar of scale m1 / den: m1 and v1 are within em = 4 u (|m| + |g|) and ev = 4 u (|v| + g^2) (3 roundings each, and the rounded
    gradient), den moves by ev / (2 sqrt(v1) sq_bc2); 8 u |update| for the quotient, the scale and the square root."""
    em, ev = 4 * U * (m.abs() + gi.abs()), 4 * U * (v.abs() + gi * gi)
    dden = torch.where(v1 > 0, ev / (2 * v1.sqrt().clamp_min(1e-300) * sq_bc2), ev.sqrt() / sq_bc2)
    return abs(scale) * (em / den + m1.abs() * dden / (den * den)) + 8 * U * (scale * m1 / den).abs()


def _pow32(b, t):
    return float(np.float32(1.0) - np.float32(b) ** np.float32(t))


def keras_lr_t(lr, b1, b2, t):
    """lr sqrt(1 - b2^t) / (1 - b1^t) in fp32, as vf_adamw_keras's host code and TF 2.4's Adam evaluate it (1 - b2^t cancels)."""
    one = np.float32(1.0)
    return float(np.float32(lr) * np.sqrt(one - np.float32(b2) ** np.float32(t)) / (one - np.float32(b1) ** np.float32(t)))


def check_adam(ba, result, st):
    """torch.optim.Adam's step in fp64 from the snapshots of p, m, v (sampled ranges), hyperparameters as fp32, the bias corrections
    1 - beta^t in fp32 (as the host code): m, v within 4 u of their terms, p within 2 u |p| + 16 u |update|."""
    b1, b2, eps, lr, gs, t = f32(ba["beta1"]), f32(ba["beta2"]), f32(ba["eps"]), f32(ba["lr"]), f32(ba["grad_scale"]), int(ba["step"])
    bc1, bc2 = _pow32(b1, t), _pow32(b2, t)
    worst = 0.0
    for i, r in enumerate(st["ranges"]):
        p, g, m, v = (st["snap"][k][i].double() for k in ("p", "g", "m", "v"))
        gi = g * gs
        m1 = m + (1 - b1) * (gi - m)
        v1 = b2 * v + (1 - b2) * gi * gi
        den = v1.sqrt() / math.sqrt(bc2) + eps
        upd = lr / bc1 * m1 / den
        ubar = _update_bar(lr / bc1, m, v, gi, m1, v1, den, math.sqrt(bc2))
        worst = max(worst, ratio((ba["m"].reshape(-1)[r].double() - m1).abs(), 4 * U * (m.abs() + gi.abs()) + 1e-38),
                    ratio((ba["v"].reshape(-1)[r].double() - v1).abs(), 4 * U * (v.abs() + gi * gi) + 1e-38),
                    ratio((ba["p"].reshape(-1)[r].double() - (p - upd)).abs(), 2 * U * p.abs() + ubar + 1e-38))
    return worst


def check_adamw_keras(ba, result, st):
    """The Keras AdamWeightDecay step in fp64 from the snapshots: p -= lr wd p; m += (g - m)(1 - b1); v += (g^2 - v)(1 - b2);
    p -= lr_t m / (sqrt(v) + eps) with g = grad grad_scale clip_scale and lr_t = keras_lr_t (fp32).  Bars as check_adam, plus 2 u |lr wd p|."""
    b1, b2, eps, lr, wd = f32(ba["beta1"]), f32(ba["beta2"]), f32(ba["eps"]), f32(ba["lr"]), f32(ba["weight_decay"])
    lr_t = keras_lr_t(ba["lr"], ba["beta1"], ba["beta2"], int(ba["step"]))
    worst = 0.0
    for i, r in enumerate(st["ranges"]):
        p, g, m, v = (st["snap"][k][i].double() for k in ("p", "g", "m", "v"))
        gi = g * f32(ba["grad_scale"]) * f32(ba["clip_scale"])
        p1 = p - f32(np.float32(lr) * np.float32(wd)) * p
        m1 = m + (gi - m) * (1 - b1)
        v1 = v + (gi * gi - v) * (1 - b2)
        den = v1.sqrt() + eps
        upd = lr_t * m1 / den
        ubar = _update_bar(lr_t, m, v, gi, m1, v1, den, 1.0)
        worst = max(worst, ratio((ba["m"].reshape(-1)[r].double() - m1).abs(), 4 * U * (m.abs() + gi.abs()) + 1e-38),
                    ratio((ba["v"].reshape(-1)[r].double() - v1).abs(), 4 * U * (v.abs() + gi * gi) + 1e-38),
                    ratio((ba["p"].reshape(-1)[r].double() - (p1 - upd)).abs(), 2 * U * p.abs() + 2 * U * (lr * wd * p).abs() + ubar + 1e-38))
    return worst


# ----------------------------------------------------------------------------------------------- bit-exact conversions, dropout
def before_none(ba, rng):
    return {}


def check_split_f16x2(ba, result, st):
    """[hi | lo] with hi = fp16(v), lo = fp16((v - hi) 2^11), bit for bit."""
    hi, lo = split_pair(ba["x_rows"])
    return bits_equal(result, torch.cat([hi, lo], 1))


def _dropped(x, rate, seed):
    """fp32 dropout(x) with the kernels' mask: x times the multiplier (0 or fp32(1 / (1 - rate))), one fp32 product."""
    if rate <= 0:
        return x.float()
    return x.float() * HOOKS["dropout_mask"](tuple(x.shape), rate, seed, x.device).float()


def check_to_bf16(ba, result, st):
    """bf16(dropout(x)) rounded to nearest even, and the fp32 dropout(x) when requested, bit for bit."""
    y = _dropped(ba["x"], float(ba["rate"]), int(ba["seed"]))
    if ba["out_f32"]:
        return max(bits_equal(result[0], y), bits_equal(result[1], y.to(torch.bfloat16)))
    return bits_equal(result, y.to(torch.bfloat16))


def check_dropout(ba, result, st):
    """The mask is a hash of (seed, index) with no independent reference, so only its form is checked: every element is exactly 0 or
    x fp32(1 / (1 - rate)), and rate 0 is the identity.  A wrong keep fraction or a mask shifted between sites is invisible here (the
    kernel test checks the fraction; the attention checkers read the same mask)."""
    x, rate = ba["x"], float(ba["rate"])
    if rate <= 0:
        return bits_equal(result, x)
    sc = np.float32(1.0) / (np.float32(1.0) - np.float32(rate))
    ok = (result == 0) | (result == x * float(sc))
    return 0.0 if bool(ok.all()) else math.inf


# ----------------------------------------------------------------------------------------------- pixels, layouts, glue (bit-exact)
def check_u8_to_unit(ba, result, st):
    """(x fp32(1/255)) 2 - 1, op by op in fp32, bit for bit; ``first_views=n`` reads views 0..n-1 of every scene."""
    x, fv = ba["x_u8"], ba["first_views"]
    if fv is not None:
        x = x[:, :fv].reshape((-1,) + tuple(x.shape[2:]))
    k = torch.tensor(1.0 / 255.0, dtype=torch.float32, device=x.device)
    return bits_equal(result, (x.float() * k) * 2.0 - 1.0)


def check_unit_to_u8(ba, result, st):
    """clamp(x, -1, 1) 0.5 + 0.5, times 255.5, clamped to [0, 255], truncated, op by op in fp32, bit for bit."""
    v = ba["x"].float().clamp(-1.0, 1.0) * 0.5 + 0.5
    return bits_equal(result, (v * 255.5).clamp(0.0, 255.0).to(torch.uint8))


def check_nchw_to_nhwc(ba, result, st):
    return bits_equal(result, ba["x"].permute(0, 2, 3, 1).contiguous())


def check_nhwc_to_nchw(ba, result, st):
    return bits_equal(result, ba["x"].permute(0, 3, 1, 2).contiguous())


def check_gather_rows(ba, result, st):
    """table[idx], the index clamped into the table, bit for bit."""
    t = ba["table"]
    return bits_equal(result, t[ba["idx"].clamp(0, t.shape[0] - 1)])


def check_vq_prepare_codebook_f16(ba, result, st):
    """fp16(-2 e) of the codebook rows Et [K, D] (-2 e is exact in fp32), bit for bit."""
    return bits_equal(result, (-2.0 * ba["et"].float()).half())


def check_vq_prepare_codebook(ba, result, st):
    """Et = emb^T bit for bit; |e|^2 a sequential fp32 sum of D rounded squares: 2 (D + 1) u sum e^2."""
    emb = ba["emb_dk"]
    et, esq = result
    e = emb.double()
    want = (e * e).sum(0)
    return max(bits_equal(et, emb.t().contiguous()), ratio((esq.double() - want).abs(), 2 * (emb.shape[0] + 1) * U * want + 1e-300))


def check_migt_embed(ba, result, st):
    """(wte[id] + wpe[l]) + pose[bt] in fp32, in the reference's order, bit for bit (id = ids, or fixed_token where null or < 0)."""
    ids, wte, wpe, pose, BT, Lt = ba["ids_i32"], ba["wte"], ba["wpe"], ba["pose_rows"], ba["BT"], ba["L"]
    tok = BT * Lt
    dev = wte.device
    fixed = torch.full((tok,), int(ba["fixed_token"]), dtype=torch.long, device=dev)
    idx = fixed if ids is None else torch.where(ids.long().reshape(-1) < 0, fixed, ids.long().reshape(-1))
    ar = torch.arange(tok, device=dev)
    return bits_equal(result, (wte[idx] + wpe[ar % Lt]) + pose[ar // Lt])


def check_argmax_rows(ba, result, st):
    """Index of the row maximum, ties to the first index, exactly."""
    return bits_equal(result, torch.argmax(ba["x_rows"], 1))


def check_image_pair_sums(ba, result, st):
    """(sum |a - b|, sum (a - b)^2) per image in int64, exactly."""
    a, b = ba["a_u8"], ba["b_u8"]
    d = (a.long() - b.long()).reshape(a.shape[0], -1)
    return bits_equal(result, torch.stack([d.abs().sum(1), (d * d).sum(1)], 1))


def check_sumpool2x2(ba, result, st):
    """(x00 + x01) + (x10 + x11) per 2 x 2 window: 2 u sum|terms| (bit-exact where the sums are exact)."""
    x = ba["x"]
    n, h2, w2, c = x.shape
    xw = x.double().reshape(n, h2 // 2, 2, w2 // 2, 2, c)
    return ratio((result.double() - xw.sum((2, 4))).abs(), 2 * U * xw.abs().sum((2, 4)))


def check_l1_grad(ba, result, st):
    """dy = scale sign(y - x) bit for bit (the fp32 difference keeps the sign and is 0 only where y == x); the fp64 loss sum within
    (u + K 2^-53) sum |y - x| (the fp32 subtraction, then an fp64 chain: per-thread + 5 shuffles + 8 warps + the blocks)."""
    x, y = ba["x"], ba["y"]
    dy, ls = result
    d = y.double() - x.double()
    sc = torch.tensor(f32(ba["scale"]), dtype=torch.float32, device=x.device)
    want_dy = torch.sign(d).float() * sc
    n = y.numel()
    blocks = min((n + 255) // 256, 132 * 16)
    K = (n + blocks * 256 - 1) // (blocks * 256) + 13 + blocks
    s = d.abs().sum()
    return max(bits_equal(dy, want_dy + 0.0), ratio((ls.double().reshape(-1)[:1] - s).abs(), ((U + K * 2.0 ** -53) * s + 1e-300).reshape(1)))


def check_row_mean(ba, result, st):
    """mean of x[b, start:]: one block per row, ceil((n - start) / 256) terms per thread, 5 shuffles, 8 warps, then the division:
    2 (K + 1) u mean|x|."""
    x, start = ba["x_rows"], int(ba["start"])
    xs = x[:, start:].double()
    K = (xs.shape[1] + 255) // 256 + 13
    return ratio((result.double() - xs.mean(1)).abs(), 2 * (K + 1) * U * xs.abs().mean(1) + 1e-300)


# ----------------------------------------------------------------------------------------------- softmax, losses, poses
def before_softmax_rows(ba, rng):
    return dict(rows=pick_rows(int(ba["rows_total"]), rng))


def check_softmax_rows(ba, result, st):
    """Masked row softmax (one warp per row; row r of its batch at position r + row0, view = position // block): mode 0 all columns,
    mode 1 columns < (view + 1) block, mode 2 columns < view block of the first half and the view's own block of the second half.  Masked
    columns exactly 0.  Visible: 2 (K + 8) u p (+ 2^-8 p for bf16), K = ceil(visible / 32) + 5 (the sum of exponentials; expf and the
    reciprocal a few ulps)."""
    rows = st["rows"].to(ba["scores"].device)
    cols, mode, blk = int(ba["cols"]), int(ba["mask_mode"]), int(ba["block"])
    rt = int(ba["rows_total"])
    sc = view(ba["scores"], 0, (rt, cols), (int(ba["ld_in"]), 1))[rows].double()
    got = view(result, 0, (rt, cols), (int(ba["ld_out"]), 1))[rows].double()
    pos = rows % int(ba["rows_per_batch"]) + int(ba["row0"])
    c = torch.arange(cols, device=sc.device)[None, :]
    vw = (pos // blk if blk > 0 else torch.zeros_like(pos))[:, None]
    if mode == 1:
        vis = c < ((vw + 1) * blk).clamp(max=cols)
    elif mode == 2:
        half = cols // 2
        vis = (c < (vw * blk).clamp(max=half)) | ((c >= half + vw * blk) & (c < half + (vw + 1) * blk))
    else:
        vis = c >= 0
    p = torch.softmax(sc.masked_fill(~vis, -math.inf), 1).masked_fill(~vis, 0.0)
    K = (vis.sum(1, keepdim=True).double() + 31) // 32 + 5
    bar = 2 * (K + 8) * U * p
    if result.dtype == torch.bfloat16:
        bar = bar + BF16_OUT * p
    return ratio((got - p).abs(), bar)


def check_cross_entropy_rows(ba, result, st):
    """(1 - s) (lse - x_label) + s (lse - mean x), one warp per row: lse carries K u (the sum of exponentials, K = ceil(cols / 32) + 5)
    plus a few ulps of |lse|, the row sum K u sum|x|: 4 (K + 4) u (1 + |lse| + |x_label| + mean|x|)."""
    lg, lab = ba["logits_rows"], ba["labels_i32"]
    cols = lg.shape[-1]
    rows = st["rows"].to(lg.device)
    x = lg[rows].double()
    s = f32(ba["smoothing"])
    lse = torch.logsumexp(x, 1)
    xl = x.gather(1, lab[rows].long()[:, None])[:, 0]
    want = (1 - s) * (lse - xl) + s * (lse - x.mean(1))
    K = (cols + 31) // 32 + 5
    return ratio((result[rows].double() - want).abs(), 4 * (K + 4) * U * (1 + lse.abs() + xl.abs() + x.abs().mean(1)))


def _pose_target(ba, rows):
    return ba["poses_bt7"].reshape(-1, 7)[rows // int(ba["tokens_per_view"])].double()


def check_pose_loss_rows(ba, result, st):
    """pos = mean_3 (y m - r)^2, ori = mean_4 (y - r)^2 per row (y the pose of the row's view): 8 u mean (|y m| + |r|)^2."""
    raw = ba["raw_rows"]
    rows = torch.arange(raw.shape[0], device=raw.device)
    y, r = _pose_target(ba, rows), raw.double()
    m = f32(ba["mult"])
    pos, ori = result
    ym = y[:, :3] * m
    return max(ratio((pos.double() - ((ym - r[:, :3]) ** 2).mean(1)).abs(), 8 * U * ((ym.abs() + r[:, :3].abs()) ** 2).mean(1) + 1e-38),
               ratio((ori.double() - ((y[:, 3:] - r[:, 3:]) ** 2).mean(1)).abs(), 8 * U * ((y[:, 3:].abs() + r[:, 3:].abs()) ** 2).mean(1) + 1e-38))


def check_pose_loss_grad(ba, result, st):
    """d/draw of sum w (ps mean_3 (y m - r)^2 + os mean_4 (y - r)^2): 8 u w scale (|y m| + |r|) (tests/test_backward_kernels_gpu.py)."""
    raw, w = ba["raw_rows"], ba["row_weight"].double()[:, None]
    rows = torch.arange(raw.shape[0], device=raw.device)
    y, r = _pose_target(ba, rows), raw.double()
    mv = torch.tensor([f32(ba["mult"])] * 3 + [1.0] * 4, dtype=torch.float64, device=raw.device)
    scl = torch.tensor([f32(ba["pos_scale"]) * 2 / 3] * 3 + [f32(ba["ori_scale"]) * 2 / 4] * 4, dtype=torch.float64, device=raw.device)
    want = -w * scl * (y * mv - r)
    return ratio((result.double() - want).abs(), 8 * U * w.abs() * scl * ((y * mv).abs() + r.abs()) + 1e-38)


def _quat_unit(q):
    q = q / q.norm(dim=-1, keepdim=True).clamp_min(1e-6)
    return q * torch.where(q[..., :1] >= 0, 1.0, -1.0)


def check_pose_postprocess(ba, result, st):
    """xyz / mult (one rounding: u |xyz / mult|), the quaternion normalised with w >= 0: its squared norm is a 4-term chain (4 u relative),
    rsqrtf is within 2 ulp (4 u), the product rounds once (u), and the result may be one rounding of the stored unit value away (u):
    16 u absolute on each unit-quaternion component."""
    raw = ba["raw_rows"].double()
    want = torch.cat([raw[:, :3] / f32(ba["mult"]), _quat_unit(raw[:, 3:])], 1)
    bar = torch.cat([U * want[:, :3].abs(), torch.full_like(want[:, 3:], 16 * U)], 1)
    return ratio((result.double() - want).abs(), bar + 1e-38)


def _qmul(a, b):
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def _conj(q):
    return q * torch.tensor([1.0, -1.0, -1.0, -1.0], dtype=q.dtype, device=q.device)


def check_cameras_prepare(ba, result, st):
    """relative: xyz - xyz0 rotated by conj(q0), q = conj(q0) q; then q normalised with w >= 0; the transform is view 0's camera bit for
    bit.  Bars: 16 u (|xyz| + |xyz0|) on positions (two quaternion products), 16 u on the unit quaternion."""
    cams = ba["cams"].double()
    out, tr = result
    p, q = cams[..., :3], cams[..., 3:]
    worst = 0.0
    if ba["relative"]:
        inv = _conj(q[:, :1])
        d = torch.cat([torch.zeros_like(p[..., :1]), p - p[:, :1]], -1)
        p = _qmul(_qmul(inv.expand_as(q), d), _conj(inv).expand_as(q))[..., 1:]
        q = _qmul(inv.expand_as(q), q)
        worst = bits_equal(tr, ba["cams"][:, 0].contiguous())
    want = torch.cat([p, _quat_unit(q)], -1)
    sc = (cams[..., :3].abs().sum(-1, keepdim=True) + cams[:, :1, :3].abs().sum(-1, keepdim=True)) * (cams[..., 3:].abs().sum(-1, keepdim=True) ** 2)
    bar = torch.cat([16 * U * sc.expand_as(p), torch.full_like(q, 16 * U)], -1)
    return max(worst, ratio((out.double() - want).abs(), bar + 1e-38))


def check_cameras_from_relative(ba, result, st):
    """q = qt q, xyz = qt xyz conj(qt) + t (the inverse of the relative transform): 16 u (|xyz| |qt|^2 + |t|), 8 u |qt| |q| on q."""
    c, t = ba["cams"].double(), ba["transform"].double()[:, None]
    tq = t[..., 3:].expand(c.shape[:-1] + (4,))
    q = _qmul(tq, c[..., 3:])
    pp = torch.cat([torch.zeros_like(c[..., :1]), c[..., :3]], -1)
    xyz = _qmul(_qmul(tq, pp), _conj(tq))[..., 1:] + t[..., :3]
    want = torch.cat([xyz, q], -1)
    n2 = tq.abs().sum(-1, keepdim=True)
    bar = torch.cat([16 * U * (c[..., :3].abs().sum(-1, keepdim=True) * n2 * n2 + t[..., :3].abs()).expand_as(xyz),
                     8 * U * (n2 * c[..., 3:].abs().sum(-1, keepdim=True)).expand_as(q)], -1)
    return ratio((result.double() - want).abs(), bar + 1e-38)


# ----------------------------------------------------------------------------------------------- quantizer
def check_vq_ema_stats(ba, result, st):
    """counts exact (integers below 2^24); esum [D, K] = sum of the z rows mapped to each code, one fp32 atomic per row: an element's
    chain is its code's count, 2 (count + 1) u sum |z|."""
    z, idx, k = ba["z_rows"], ba["idx"], int(ba["k"])
    counts, esum = result
    cnt = torch.bincount(idx, minlength=k).float()
    zs = torch.zeros(k, z.shape[1], dtype=torch.float64, device=z.device).index_add_(0, idx, z.double()).t()
    za = torch.zeros(k, z.shape[1], dtype=torch.float64, device=z.device).index_add_(0, idx, z.double().abs()).t()
    return max(bits_equal(counts, cnt), ratio((esum.double() - zs).abs(), 2 * (cnt.double() + 1) * U * za + 1e-38))


def check_vq_commit_grad(ba, result, st):
    """coef (count_k e - esum) from the given counts and row sums, three roundings: 4 u |coef| (count |e| + |esum|)."""
    emb, counts, esum = ba["emb_dk"].double(), ba["counts"].double(), ba["esum"].double()
    c = f32(ba["coef"])
    want = c * (counts * emb - esum)
    return ratio((result.double() - want).abs(), 4 * U * abs(c) * (counts * emb.abs() + esum.abs()) + 1e-38)


def before_vq_ema_update(ba, rng):
    return dict(cs=ba["cs_hidden"].clone(), dw=ba["dw_hidden"].clone())


def check_vq_ema_update(ba, result, st):
    """QuantizeEMA's update in fp64 from the snapshots of the hidden EMAs: cs' = cs + a (counts - cs), n = sum cs' / corr (fp32 chain
    Kn = ceil(K / 1024) + 10), cluster = (cs' / corr + eps) / (n + K eps) n, dw' = dw + a (esum - dw), e = (dw' / corr) / cluster written
    to emb [D, K] and (bit for bit the same values) Et [K, D], |e|^2 a chain of D fmas.  Bars: cs', dw' 4 u of their terms;
    e 2 (Kn + 12) u |e| + the dw' error / (corr cluster); |e|^2 2 (D + 2) u sum e^2 + 2 |e| that bar."""
    a, corr, eps = f32(ba["alpha"]), f32(ba["corr"]), f32(ba["eps"])
    counts, esum = ba["counts"].double(), ba["esum"].double()
    cs0, dw0 = st["cs"].double(), st["dw"].double()
    k = cs0.shape[0]
    cs1 = cs0 + a * (counts - cs0)
    n = (cs1 / corr).sum()
    cluster = (cs1 / corr + eps) / (n + k * eps) * n
    dw1 = dw0 + a * (esum - dw0)
    e = (dw1 / corr) / cluster[None, :]
    Kn = (k + 1023) // 1024 + 10
    ebar = 2 * (Kn + 12) * U * e.abs() + 4 * U * (dw0.abs() + a * esum.abs()) / (corr * cluster.abs()[None, :])
    emb, et, esq = ba["emb_dk"], ba["et"], ba["esq"]
    worst = max(ratio((ba["cs_hidden"].double() - cs1).abs(), 4 * U * (cs0.abs() + a * counts.abs()) + 1e-38),
                ratio((ba["dw_hidden"].double() - dw1).abs(), 4 * U * (dw0.abs() + a * esum.abs()) + 1e-38),
                ratio((emb.double() - e).abs(), ebar + 1e-38), bits_equal(et, emb.t().contiguous()))
    sq = (e * e).sum(0)
    return max(worst, ratio((esq.double() - sq).abs(), 2 * (emb.shape[0] + 2) * U * sq + 2 * (e.abs() * ebar).sum(0) + 1e-38))


# ----------------------------------------------------------------------------------------------- evaluation
def check_resize_u8(ba, result, st):
    """fp64 restatement of the nearest / bilinear (align_corners=False) resize of x / 255, times 255, truncated; the source indices and
    interpolation weights are formed in fp32 as the kernel forms them.  Bit-exact, except where
    the fp64 value lies within 64 u (of 255) of an integer: there the kernel's fp32 rounding may land on either side, so k or k - 1 is
    accepted for a value within that distance of k."""
    x, size = ba["x_u8"], int(ba["size"])
    n, h, w, c = x.shape
    # resize() hands NHWC to resize_th() unless shape[-2] = W is the size; resize_th() returns NCHW unchanged when shape[-2] = H is the
    # size, and otherwise grows the height with nearest and shrinks it bilinearly, whatever the width does
    if size in (w, h):
        return 0.0 if result is x else math.inf
    method = ba["method"] or ("nearest" if size > h else "bilinear")
    xv = x.double() / 255.0
    sh, sw = f32(np.float32(h) / np.float32(size)), f32(np.float32(w) / np.float32(size))
    o = torch.arange(size, device=x.device, dtype=torch.float32)          # source indices and weights in fp32, as the kernel forms them
    if method == "nearest":
        sy = torch.floor(o * sh).long().clamp(max=h - 1)
        sx = torch.floor(o * sw).long().clamp(max=w - 1)
        v = xv[:, sy][:, :, sx]
    else:
        fy, fx = ((o + 0.5) * sh - 0.5).clamp_min(0), ((o + 0.5) * sw - 0.5).clamp_min(0)
        y0, x0 = fy.long(), fx.long()
        y1, x1 = (y0 + 1).clamp(max=h - 1), (x0 + 1).clamp(max=w - 1)
        ly, lx = (fy - y0).double()[None, :, None, None], (fx - x0).double()[None, None, :, None]
        g = lambda yy, xx: xv[:, yy][:, :, xx]
        v = (1 - ly) * ((1 - lx) * g(y0, x0) + lx * g(y0, x1)) + ly * ((1 - lx) * g(y1, x0) + lx * g(y1, x1))
    t = v.clamp(0, 1) * 255.0
    k = torch.floor(t)
    near_up = (torch.ceil(t) - t) <= 64 * U * 255
    near_dn = (t - k) <= 64 * U * 255
    got = result.double()
    ok = (got == k) | (near_up & (got == k + 1)) | (near_dn & (got == k - 1))
    return 0.0 if bool(ok.all()) else math.inf


U64 = 2.0 ** -53
SSIM_M, SSIM_D = 49 * 49 * 65025, 48 * 49 * 65025      # 49^2 255^2 and 48 49 255^2: the scales of the window sums' moments


def box7(t):
    """Exact 7 x 7 VALID window sums of an integer tensor [N, H, W, C] -> int64 [N, H-6, W-6, C], from a 2-D cumulative sum."""
    n, h, w, c = t.shape
    s = torch.zeros(n, h + 1, w + 1, c, dtype=torch.int64, device=t.device)
    s[:, 1:, 1:] = t.long().cumsum(1).cumsum(2)
    return s[:, 7:, 7:] - s[:, :-7, 7:] - s[:, 7:, :-7] + s[:, :-7, :-7]


def pairwise_sum(x):
    """Sum over the last dimension by halving: ceil(log2 n) additions per element's chain."""
    while x.shape[-1] > 1:
        if x.shape[-1] % 2:
            x = F.pad(x, (0, 1))
        x = x[..., 0::2] + x[..., 1::2]
    return x[..., 0]


def ssim64(a, b, k1=0.01, k2=0.03):
    """SSIM of ``ssim()`` (7 x 7 uniform window, VALID, sample covariance, data range 1) of uint8 images [N, H, W, C] in fp64, from exact
    integer window moments: with x = 255 X, M = 49^2 255^2 and D = 48 49 255^2, 2 ux uy + C1 = (2 sx sy + C1 M) / M and
    2 vxy + C2 = (2 (49 sxy - sx sy) + C2 D) / D, and likewise B1, B2; the integers are exact in int64 and the scales cancel in S.
    C1 = K1^2 and C2 = K2^2 are rounded once in fp64.  Returns (per-window S, the mean per image, T = |A1| |2 vxy| / (B1 B2) per window)."""
    C1, C2 = float(k1) * float(k1), float(k2) * float(k2)
    xa, xb = a.long(), b.long()
    sx, sy, sxx, syy, sxy = box7(xa), box7(xb), box7(xa * xa), box7(xb * xb), box7(xa * xb)
    n2xy = 2 * (49 * sxy - sx * sy)
    a1 = (2 * sx * sy).double() + C1 * SSIM_M
    a2 = n2xy.double() + C2 * SSIM_D
    b1 = (sx * sx + sy * sy).double() + C1 * SSIM_M
    b2 = ((49 * sxx - sx * sx) + (49 * syy - sy * sy)).double() + C2 * SSIM_D
    den = b1 * b2
    S = (a1 * a2) / den
    flat = S.reshape(S.shape[0], -1)
    return S, pairwise_sum(flat) / flat.shape[1], a1.abs() * n2xy.double().abs() / den


def ssim_bar(S, T, h, w, c):
    """The bar of ``check_ssim_u8`` per image (see there) from ssim64's per-window S and T."""
    total = (h - 6) * (w - 6) * c
    chunks = min((total + 255) // 256, 64)
    kc = -(-total // (chunks * 256)) + 5 + 8 + chunks + 1            # kernel: windows per thread, shuffles, warps, chunk atomics, / total
    kr = math.ceil(math.log2(total)) + 1 if total > 1 else 1           # reference: pairwise sum, / total
    Sa, Ta = S.abs().reshape(S.shape[0], -1), T.reshape(T.shape[0], -1)
    return (24 * U64 * (Sa + Ta).sum(1) + (kc + kr) * U64 * Sa.sum(1)) / total


def check_ssim_u8(ba, result, st):
    """Mean SSIM per image against ``ssim64`` (exact int64 window sums, S in fp64).  The kernel also sums each window exactly in integers
    and forms the numerators 49 sxx - sx^2, 49 sxy - sx sy exactly (|.| < 2^29); S follows in fp64 with the same C1 = K1^2, C2 = K2^2.
    Per window (u = 2^-53), the kernel: A1 = 2 sx sy / M + C1, B1, B2 one division and one addition of non-negative terms each (2 u
    relative); A2 = q + C2 with q = 2 nxy / D, which cancels when the covariance is negative: u |q| + u |A2|; the two products and the
    quotient 3 u: in all 10 u |S| + u T with T = |A1| |q| / (B1 B2).  The reference rounds C1 M, C2 D and its sums (2 u each of A1, B1,
    B2; u (|q| + 2 |A2|) on A2) and 3 u in S: 11 u |S| + u T.  So each window's S is within 21 u |S| + 2 u T of the exact one; the bar
    takes 24 u (|S| + T), which covers the second-order terms.  The mean: a per-thread fp64 chain over ceil(total / (chunks 256))
    windows, 5 shuffles, 8 warp partials, up to 64 chunk atomics (chunks = min(ceil(total / 256), 64)), then / total: a chain of
    Kc = that sum + 1 roundings of partial sums bounded by sum |S|; the reference's pairwise sum adds ceil(log2 total) + 1.  Bar per
    image: (24 u sum (|S| + T) + (Kc + Kr) u sum |S|) / total, about 1e-14 at 128 x 128 x 3.  An fp32 E[x^2] - E[x]^2, a dropped row of
    windows, swapped channels or images, or K1 = 0.01 for 1 is off by 1e-5 or more."""
    a, b = ba["a_u8"], ba["b_u8"]
    k1 = 0.01 if ba["k1"] is None else ba["k1"]
    k2 = 0.03 if ba["k2"] is None else ba["k2"]
    S, mean, T = ssim64(a, b, k1, k2)
    _, h, w, c = a.shape
    return ratio((result.double() - mean).abs(), ssim_bar(S, T, h, w, c))


# ----------------------------------------------------------------------------------------------- registry
CHECKERS = {
    "tc_gemm": (before_tc_gemm, check_tc_gemm),
    "tc_conv": (before_tc_conv, check_tc_conv),
    "simt_gemm": (before_simt_gemm, check_simt_gemm),
    "simt_conv": (before_conv, check_simt_conv),
    "simt_conv_dgrad_s2": (before_conv, check_simt_conv_dgrad_s2),
    "conv3x3_small_cin": (before_conv, check_conv3x3_small_cin),
    "conv3x3_small_cout": (before_conv, check_conv3x3_small_cout),
    "conv_wgrad": (before_wgrad, check_conv_wgrad),
    "conv_wgrad_tc": (before_wgrad, check_conv_wgrad_tc),
    "conv_wgrad_bf16": (before_wgrad, check_conv_wgrad_bf16),
    "dense_wgrad_tc": (before_wgrad, check_dense_wgrad_tc),
    "dense_wgrad_bf16": (before_wgrad, check_dense_wgrad_bf16),
    "attn_block_causal": (before_attn, check_attn_block_causal),
    "attn_block_multiend": (before_attn, check_attn_block_multiend),
    "attn_multiend_train": (before_attn_train, check_attn_multiend_train),
    "attn_multiend_bwd": (before_attn_bwd, check_attn_multiend_bwd),
    "vq_lookup": (before_lookup, check_vq_lookup),
    "vq_lookup_fused": (before_lookup, check_lookup),
    "gn_mean_rstd": (before_gn_mean_rstd, check_gn_mean_rstd),
    "groupnorm": (before_groupnorm, check_groupnorm),
    "layernorm": (before_layernorm, check_layernorm),
    "groupnorm_bwd": (before_groupnorm_bwd, check_groupnorm_bwd),
    "layernorm_bwd": (before_layernorm_bwd, check_layernorm_bwd),
    "col_sums": (before_col_sums, check_col_sums),
    "softmax_bwd_rows": (before_rows("P"), check_softmax_bwd_rows),
    "cross_entropy_grad": (before_rows("logits_rows"), check_cross_entropy_grad),
    "sumsq": (before_none, check_sumsq),
    "migt_embed_bwd": (before_migt_embed_bwd, check_migt_embed_bwd),
    "gelu": (before_elementwise("x"), check_gelu),
    "gelu_bwd": (before_elementwise("pre", "dy", size="pre"), check_gelu_bwd),
    "lincomb3": (before_elementwise("x", "y", "z"), check_lincomb3),
    "adam": (before_elementwise("p", "g", "m", "v", size="p"), check_adam),
    "adamw_keras": (before_elementwise("p", "g", "m", "v", size="p"), check_adamw_keras),
    "split_f16x2": (before_none, check_split_f16x2),
    "to_bf16": (before_none, check_to_bf16),
    "dropout": (before_none, check_dropout),
    "u8_to_unit": (before_none, check_u8_to_unit),
    "unit_to_u8": (before_none, check_unit_to_u8),
    "nchw_to_nhwc": (before_none, check_nchw_to_nhwc),
    "nhwc_to_nchw": (before_none, check_nhwc_to_nchw),
    "gather_rows": (before_none, check_gather_rows),
    "vq_prepare_codebook_f16": (before_none, check_vq_prepare_codebook_f16),
    "vq_prepare_codebook": (before_none, check_vq_prepare_codebook),
    "migt_embed": (before_none, check_migt_embed),
    "argmax_rows": (before_none, check_argmax_rows),
    "image_pair_sums": (before_none, check_image_pair_sums),
    "sumpool2x2": (before_none, check_sumpool2x2),
    "l1_grad": (before_none, check_l1_grad),
    "row_mean": (before_none, check_row_mean),
    "softmax_rows": (before_softmax_rows, check_softmax_rows),
    "cross_entropy_rows": (before_rows("logits_rows"), check_cross_entropy_rows),
    "pose_loss_rows": (before_none, check_pose_loss_rows),
    "pose_loss_grad": (before_none, check_pose_loss_grad),
    "pose_postprocess": (before_none, check_pose_postprocess),
    "cameras_prepare": (before_none, check_cameras_prepare),
    "cameras_from_relative": (before_none, check_cameras_from_relative),
    "vq_ema_stats": (before_none, check_vq_ema_stats),
    "vq_commit_grad": (before_none, check_vq_commit_grad),
    "vq_ema_update": (before_vq_ema_update, check_vq_ema_update),
    "resize_u8": (before_none, check_resize_u8),
    "ssim_u8": (before_none, check_ssim_u8),
}

# Launching wrappers without a checker of their own, each with the reason.  test_every_launching_wrapper_has_a_checker allows exactly these.
UNCHECKED = {
    "pad_transpose_split": "internal operand builder of the split-fp16 weight gradient (_wgrad_tc): a misplaced or non-zero border value "
                           "changes dW, which check_conv_wgrad_tc / check_dense_wgrad_tc restate from x and dy directly",
    "pad_transpose_bf16": "internal operand builder of the bf16 weight gradient (_wgrad_tc), held the same way by check_conv_wgrad_bf16 / "
                          "check_dense_wgrad_bf16 (GroupNorm operand through HOOKS['gn_apply_bf16'])",
    "dense_weights_bf16": "its table holds raw device pointers, which a device-agnostic checker cannot dereference; the bf16 copies it "
                          "writes are the operands every bf16 dense tc_gemm check reads, and tests/test_train_migt_bf16_gpu.py pins them "
                          "bit for bit against torch",
    "conv_weights_bf16": "raw device pointers in its table, as dense_weights_bf16; its copies are the operands of the bf16 tc_conv checks "
                         "and are pinned bit for bit in tests/test_train_bf16_gpu.py",
}


def bind(fn, *a, **k):
    """The wrapper's arguments by name, defaults filled in."""
    import inspect
    b = inspect.signature(fn).bind(*a, **k)
    b.apply_defaults()
    return dict(b.arguments)


def run_check(name, fn, a, k, rng):
    """Call wrapper ``fn`` with its snapshot taken first; return (result, worst ratio)."""
    before, check = CHECKERS[name]
    ba = bind(fn, *a, **k)
    st = before(ba, rng)
    result = fn(*a, **k)
    return result, check(ba, result, st)
