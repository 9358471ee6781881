"""Precision policy + operator dispatch shared by the VQGAN and MIGT host classes.

Three precisions, all of them CUDA (there is no CPU path):
  * ``bf16``  tensor-core path: bf16 operands, fp32 accumulation in registers (wgmma), fp32 residual stream,
              fp32 norms / softmax / argmin.  This is the benchmarked configuration.
  * ``tf32``  same kernels with fp32 operands fed to ``wgmma.mma_async ... .tf32`` (the arithmetic the reference
              itself ran on A100 with torch 1.7 / TF 2.4 defaults).
  * ``fp32``  exact CUDA-core path (FFMA), used for strict parity against the oracle.
  * ``x3``    (VQGAN only) fp32-faithful 3x3 convolutions on the tensor cores (split-fp16 operands, 3 MMAs per product,
              chunked accumulation); 1x1 convs / attention blocks on the fp32 CUDA-core path.  Same codebook indices as ``fp32``.
"""
import torch

from . import _lib as L


class Precision:
    def __init__(self, name):
        if name not in ("bf16", "tf32", "fp32", "x3"):
            raise ValueError(f"precision must be bf16|tf32|fp32|x3, got {name}")
        self.name = name
        self.use_tc = name != "fp32"
        # x3: fp32-faithful tensor-core convolutions — operands travel as split fp16 pairs (torch.float16, [hi | lo] channels),
        # three MMAs per product block, chunked accumulation (vf_tc_gemm.cu EXACT_LO_SCALE); everything else as in fp32
        self.split = name == "x3"
        self.opd = {"bf16": torch.bfloat16, "x3": torch.float16}.get(name, torch.float32)   # dtype of conv operands
        self.k_align = 32 if name == "tf32" else 64                      # channels per 128-byte K block

    def __repr__(self):
        return f"Precision({self.name})"


class Linear:
    """y = x @ W^T + b with W stored K-major [out, in] in the operand dtype (Conv1D / 1x1 conv sites)."""

    def __init__(self, w_out_in, bias, prec, device):
        self.n, self.k = w_out_in.shape
        if getattr(prec, "split", False):      # exact mode: rows [hi(k) | lo(k)] fp16 (vf_tc_gemm VF_F16X2)
            self.w = L.split_f16x2(w_out_in.to(device=device, dtype=torch.float32).contiguous())
        else:
            self.w = w_out_in.to(device=device, dtype=prec.opd).contiguous()
        self.ld = self.w.shape[1]              # row stride of w (2k for split operands)
        self.b = None if bias is None else bias.reshape(-1).to(device=device, dtype=torch.float32).contiguous()


def gemm_nt(prec, A, B, out, *, M, N, K, lda, ldb, ldc, batch=(1, 1), a_bs=(0, 0), b_bs=(0, 0), c_bs=(0, 0),
            alpha=1.0, bias=None, bias_mode=L.BIAS_NONE, act=L.ACT_NONE, residual=None, a_off=0, b_off=0, c_off=0,
            causal_block=0, causal_skip_n=False, gn_rows_per_img=0, lo_a=None, lo_b=None):
    """C[m,n] = act(alpha * sum_k A[m,k]*B[n,k] + bias) + residual  (both operands K-major)."""
    es = A.element_size()
    tc_ok = (prec.use_tc and A.dtype == B.dtype and A.dtype == prec.opd
             and (lda * es) % 16 == 0 and (ldb * es) % 16 == 0 and (K * es) % 16 == 0
             and (a_off * es) % 16 == 0 and (b_off * es) % 16 == 0
             and all((s * es) % 16 == 0 for s in (*a_bs, *b_bs)))
    if tc_ok:
        return L.tc_gemm(A, B, out, M=M, N=N, K=K, lda=lda, ldb=ldb, ldc=ldc, batch=batch, a_bs=a_bs, b_bs=b_bs,
                         c_bs=c_bs, alpha=alpha, bias=bias, bias_mode=bias_mode, act=act, residual=residual,
                         a_off=a_off, b_off=b_off, c_off=c_off, causal_block=causal_block,
                         causal_skip_n=causal_skip_n, gn_rows_per_img=gn_rows_per_img, lo_a=lo_a, lo_b=lo_b)
    if A.dtype == torch.float16:
        raise L.LibraryError("split-fp16 (exact) operands have no CUDA-core GEMM: shape not supported by vf_tc_gemm")
    L.simt_gemm(A, B, out, M=M, N=N, K=K, a_strides=(lda, 1), b_strides=(1, ldb), ldc=ldc, batch=batch, a_bs=a_bs,
                b_bs=b_bs, c_bs=c_bs, alpha=alpha, bias=bias, bias_mode=bias_mode, act=act, residual=residual,
                a_off=a_off, b_off=b_off, c_off=c_off)
    return out


def linear(prec, x_rows, lin, out_dtype, *, act=L.ACT_NONE, residual=None, out=None, gn_rows_per_img=0):
    """x_rows [M, K] (operand dtype) -> [M, N]."""
    M = x_rows.shape[0]
    if out is None:
        out = torch.empty((M, lin.n), dtype=out_dtype, device=x_rows.device)
    gemm_nt(prec, x_rows, lin.w, out, M=M, N=lin.n, K=lin.k, lda=x_rows.shape[1], ldb=lin.ld, ldc=lin.n,
            bias=lin.b, bias_mode=L.BIAS_N if lin.b is not None else L.BIAS_NONE, act=act, residual=residual,
            gn_rows_per_img=gn_rows_per_img)
    return out
