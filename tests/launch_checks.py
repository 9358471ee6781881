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
and of the bf16 weight-gradient transposer, the dropout mask of the attention kernels, and the reference lookup.
"""
import math
import random

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


# ----------------------------------------------------------------------------------------------- tensor-core GEMM
def before_tc_gemm(ba, rng):
    b1, b2 = ba["batch"]
    return dict(batches=pick(b1 * b2, rng), rows=pick_rows(ba["M"], rng), res=_snapshot_if_aliased(ba["residual"], ba["out"]),
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
        worst = max(worst, ratio(((got - ref).abs() * keep), bar))
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
    n = ba["x"].shape[0]
    return dict(images=pick(n, rng), res=_snapshot_if_aliased(ba["residual"], ba["out"]), gn_prev=getattr(ba["out"], "_gn_sums", None))


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
def _heads(B, H, rng):
    pairs = [(b, h) for b in range(B) for h in range(H)]
    return [pairs[i] for i in pick(len(pairs), rng)]


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


def before_attn(ba, rng):
    st = dict(heads=_heads(ba["B"], ba["H"], rng))
    if ba.get("out") is not None:
        st["out"] = ba["out"].clone()
    return st


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
    st = dict(heads=_heads(ba["B"], ba["H"], rng))
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
    "attn_multiend_train": (before_attn, check_attn_multiend_train),
    "attn_multiend_bwd": (before_attn_bwd, check_attn_multiend_bwd),
    "vq_lookup": (before_lookup, check_vq_lookup),
    "vq_lookup_fused": (before_lookup, check_lookup),
    "vq_lookup_tc": (before_lookup, check_lookup),
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
