/* vf_b200.h — C-ABI of libvf_b200.so, the sm_90a kernel library underneath
 * viewformer_b200.{VQGAN,MIGT}.
 *
 * The reference (jkulhanek/viewformer) has no FFI layer: its hot path is Python calling
 * torch / TensorFlow library ops.  Each entry point below therefore names the reference
 * *library-call site* it replaces (file:line in the reference tree).  All functions are
 * extern "C", take raw device pointers, plain sizes and a cudaStream_t (as void*), never
 * allocate persistent memory, never synchronise the stream, and return 0 on success or a
 * negative code (message via vf_last_error()).  No torch types cross this boundary.
 *
 * Layout conventions: activations are NHWC ("pixel rows x channels"), i.e. every image
 * tensor is a row-major matrix [N*H*W, C]; transformer activations are [B*T*64, d].
 */
#ifndef VF_B200_H
#define VF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* vf_stream_t; /* cudaStream_t */

enum { VF_F32 = 0, VF_BF16 = 1, VF_F16X2 = 2 /* fp32 value as two fp16: [.., hi(C) | lo(C)], lo = fp16((v - hi) * 2^11); fp32-faithful for
                                                   tensors with amax in [2^-10, 2^15], NaN products at |v| >= 65520; see vf_tc_gemm */ };
enum { VF_ACT_NONE = 0, VF_ACT_GELU_ERF = 1 };
enum { VF_BIAS_NONE = 0, VF_BIAS_N = 1, VF_BIAS_M = 2 };
enum { VF_OK = 0, VF_ERR_ARG = -1, VF_ERR_CUDA = -2, VF_ERR_UNSUPPORTED = -3 };

const char* vf_last_error(void);
int vf_version(void);
/* struct sizes, so a foreign-language binding can verify its mirror of the parameter structs */
int vf_sizeof_simt_gemm(void);
int vf_sizeof_tc_gemm(void);
/* 0 when the current device is compute capability 9.0 (H100); negative otherwise. */
int vf_device_check(void);

/* ------------------------------------------------------------------------------------------
 * Pixel / layout conversion
 * replaces: evaluate/evaluate_transformer.py:106-108 (uint8 -> f32, *2-1), :128-129 (clip, ->uint8),
 *           the NCHW<->NHWC permutes of models/utils_th.py:34,72 and utils/convert.py:61-67.
 * ---------------------------------------------------------------------------------------- */
/* out[r, :] = in[r*in_row_stride : +row_len] * (1/255) * 2 - 1 for r < rows (rows=1: flat array; rows=B with
 * in_row_stride = T*H*W*3 selects the first views of every scene without a gather copy) */
int vf_u8_to_unit_f32(const uint8_t* in, float* out, int64_t rows, int64_t row_len, int64_t in_row_stride, vf_stream_t s);
/* the same strided read of f32 images in [0, 1]: out = in * 2 - 1 (convert_image_dtype is the identity for float32 input) */
int vf_f01_to_unit_f32(const float* in, float* out, int64_t rows, int64_t row_len, int64_t in_row_stride, vf_stream_t s);
int vf_unit_f32_to_u8(const float* in, uint8_t* out, int64_t n, vf_stream_t s);      /* clip[-1,1]/2+.5 -> trunc(x*255.5) */
int vf_nchw_to_nhwc_f32(const float* in, float* out, int N, int C, int H, int W, vf_stream_t s);
int vf_nhwc_to_nchw_f32(const float* in, float* out, int N, int C, int H, int W, vf_stream_t s);

/* ------------------------------------------------------------------------------------------
 * GroupNorm(32 groups) [+ swish] [+ nearest x2 upsample] [+ cast]
 * replaces: models/vqgan_th.py:11-17 (Normalize, nonlinearity), :29-30 (F.interpolate nearest)
 * x f32 [N, HW, C].  vf_groupnorm_stats: sums = double [N, groups, 2] scratch (zeroed + accumulated here),
 * mean_rstd = float [N, groups, 2] result (mean, 1/sqrt(var+eps)) consumed by vf_groupnorm_apply.
 * vf_groupnorm_apply: y = ((x-mean)*rstd*gamma+beta) [swish]; normalize=0 -> plain cast/upsample.
 *   layout: 0 = same shape; 1 = nearest x2 upsample, y is [N, 2H, 2W, C]; 2 = space-to-depth, y is [N, H/2, W/2, 4C]
 *   with channel block (a*2+b)*C holding pixel (2y+a, 2x+b) — the operand layout that turns the reference's
 *   pad(0,1,0,1)+stride-2 3x3 conv (vqgan_th.py:45-49) into a stride-1 tap-table conv.
 *   (x_dtype, y_dtype): (F32,F32) exact order of operations; (F32,BF16) and (BF16,BF16) tensor-core operand producers
 *   (affine folded to one FMA, ex2/rcp swish); (F32,F16X2) = the (F32,F32) arithmetic, each result stored as the
 *   split-fp16 pair [.., hi(Cl) | lo(Cl)] (Cl = C, or 4C for layout 2) that vf_tc_gemm's exact convolution consumes.
 *   grid = (pixel chunks, N): N <= 65535.
 * ---------------------------------------------------------------------------------------- */
/* fp32 [rows, C] -> split fp16 [rows, hi(C) | lo(C)] (hi = fp16(v), lo = fp16((v - hi) * 2^11)): the VF_F16X2 operand of vf_tc_gemm for
 * tensors that do not come out of a GroupNorm pass (any C % 4 == 0). */
int vf_split_f16x2(const float* x, int64_t rows, int C, void* out_f16, vf_stream_t s);
int vf_groupnorm_stats(const float* x, int N, int HW, int C, int groups, float eps, double* sums, float* mean_rstd,
                       vf_stream_t s);
/* (sum, sumsq) -> (mean, rstd) for `count` elements per (image, group); n_stats = images*groups */
int vf_groupnorm_finalize(const double* sums, int n_stats, double count, float eps, float* mean_rstd, vf_stream_t s);
int vf_groupnorm_apply(const void* x, int x_dtype, const float* mean_rstd, const float* gamma, const float* beta,
                       int N, int H, int W, int C, int groups, float eps, int normalize, int swish,
                       int layout, void* y, int y_dtype, vf_stream_t s);

/* Exact fp32 3x3 stride-1 pad-1 convolutions for the two tiny-channel layers (vqgan_th.py:159-163 conv_in C->128,
 * :285-289 conv_out 128->C), C = 3 (RGB) or 4 (RGB + mask); other counts are rejected.  NHWC; weights [9*Cin, Cout] fp32
 * (k = tap*Cin + c). */
int vf_conv3x3_small_cin(const float* x, const float* w_kn, const float* bias, int N, int H, int W, int Cin, int Cout,
                         float* y, double* gn_sums /* optional [N][32][2]: GroupNorm(32) sums of y, Cout = 128 only */,
                         vf_stream_t s);
int vf_conv3x3_small_cout(const void* x, int x_dtype, const float* w_kn, const float* bias, int N, int H, int W, int Cin,
                          int Cout, float* y, vf_stream_t s);

/* LayerNorm over the last dim — replaces tf.keras LayerNormalization at models/migt.py:225-227,292. */
int vf_layernorm(const float* x, const float* gamma, const float* beta, int64_t rows, int D, float eps,
                 void* y, int y_dtype, vf_stream_t s);

/* ------------------------------------------------------------------------------------------
 * Generic fp32 CUDA-core implicit GEMM ("exact" path + the small-channel convs)
 * replaces: torch.nn.Conv2d at models/vqgan_th.py:23-49,60-76,98-117,159-163,197-201,249-253,285-289,
 *           332-333; torch.bmm at :128-140; tf.matmul at models/migt.py:93 and branching_attention.py:7,18.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    /* A operand: conv gather (conv=1) or dense strided matrix (conv=0) */
    const void* A; int a_dtype; int conv;   /* conv: 0 dense, 1 forward conv gather, 2 data-gradient gather of a stride-2 conv */
    int N, H, W, Cin;            /* conv: input NHWC dims */
    int OH, OW, KH, KW, stride, pad_t, pad_l, upsample2x;
    int64_t a_sm, a_sk;          /* dense: element strides of A(m,k) */
    /* B operand (weights / second matrix): element (k,n) at k*b_sk + n*b_sn, fp32 or bf16 */
    const void* B; int b_dtype; int64_t b_sk, b_sn;
    /* problem */
    int M, Ncols, K;             /* per batch */
    int batch1, batch2;          /* grid.z = batch1*batch2 */
    int64_t a_sb1, a_sb2, b_sb1, b_sb2, c_sb1, c_sb2;   /* batch strides (elements) */
    /* epilogue: C = act(alpha*acc + bias) + residual */
    float alpha; const float* bias; int bias_mode; int act;
    const float* residual;       /* f32, same indexing as C */
    float* C_f32; void* C_bf16;  /* either or both */
    int64_t ldc;
} vf_simt_gemm_t;
int vf_simt_gemm(const vf_simt_gemm_t* p, vf_stream_t s);

/* ------------------------------------------------------------------------------------------
 * tensor-core GEMM / implicit-GEMM conv (TMA -> 128B-swizzled smem -> wgmma -> register accumulators)
 * replaces the same call sites as vf_simt_gemm on the fast path.
 *   GEMM:  C[b1,b2][m,n] = act(alpha * sum_k A[b1,b2][m,k] * B[b1,b2][n,k] + bias) + residual
 *          A and B are K-major (k contiguous), 16-byte aligned rows, dtype bf16 (or f32 -> TF32).
 *   CONV:  A is an NHWC activation tensor [N,H,W,Cin] (Cin % (128/elsize) == 0); taps describe the
 *          filter footprint: tap t reads pixel (oy+dy[t], ox+dx[t]) and channels coff[t]..coff[t]+Cin-1
 *          of a [N,H,W,Ctot] tensor; weights B are [Cout, ntaps*Cin] K-major.  Out-of-image taps are
 *          zero (TMA out-of-bounds fill), which implements both the symmetric pad-1 and the
 *          reference's asymmetric (0,1,0,1) pad.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    int conv;                    /* 0 gemm, 1 conv */
    int ab_dtype;                /* VF_BF16 | VF_F32 (TF32 math) */
    const void* A; const void* B;
    /* gemm geometry */
    int M, Ncols, K; int batch1, batch2;
    int64_t lda, ldb;            /* row strides (elements) */
    int64_t a_sb1, a_sb2, b_sb1, b_sb2;
    /* conv geometry */
    int N, H, W, Ctot, Cin, OH, OW, ntaps;
    int tap_dy[9], tap_dx[9], tap_coff[9];
    /* k-range limit for block-causal attention: if causal_block > 0, output row tile [m0, m0+128) only
       accumulates k < round_up(((m0+127)/causal_block + 1) * causal_block, BK); for the QK^T GEMM
       (causal_skip_n=1) column tiles that start at or beyond that bound are skipped entirely. */
    int causal_block, causal_skip_n;
    /* epilogue */
    float alpha; const float* bias; int bias_mode; int act; const float* residual;
    float* C_f32; void* C_bf16; int64_t ldc, c_sb1, c_sb2;
    /* optional: GroupNorm statistics of the OUTPUT fused into the epilogue (vqgan_th.py:16-17 of the NEXT layer):
       gn_sums double [images, gn_groups, 2] is zeroed and receives (sum, sum of squares) per image and group;
       an image = OH*OW consecutive rows (conv) or gn_rows_per_img rows (gemm).  Feed it to vf_groupnorm_finalize. */
    double* gn_sums; int gn_groups; int gn_rows_per_img;
    /* optional: GroupNorm(+swish) of the INPUT applied while the operand sits in shared memory (3x3 stride-1 bf16 convs on
       maps >= 32 rows tall, Cin % 64 == 0, Cout % 128 == 0 — the halo-tile path of the kernel; other shapes are rejected):
       A then is the RAW activation (e.g. the bf16 output of the previous conv), norm_mean_rstd float [N, norm_groups, 2]
       from vf_groupnorm_finalize, norm_gamma / norm_beta float [Cin].  Padding stays zero AFTER normalisation, as in
       vqgan_th.py:69-78 (norm -> swish -> conv with padding=1).  Removes the separate vf_groupnorm_apply pass.
       norm_swish: 0 = no activation, 1 = x / (1 + e^-x) in fp32 (ex2/rcp; bit-identical to vf_groupnorm_apply's bf16 output),
       2 = packed bf16 h (1 + tanh h), h = x / 2 (one MUFU op per two elements). */
    const float* norm_mean_rstd; const float* norm_gamma; const float* norm_beta; int norm_groups; int norm_swish;
    /* ab_dtype = VF_F16X2 ("exact" mode: fp32-faithful products on the tensor cores — three fp16 MMA passes hi.hi + 2^-11 (hi.lo +
       lo.hi), accumulation drained from the accumulators in short chunks and summed with round-to-nearest FFMAs; fp32 output only):
         conv: A = [N,H,W, hi(Cl) | lo(Cl)] with Ctot = 2*Cl, B = [Cout][tap][hi(Cin) | lo(Cin)];
         gemm: a row of A holds hi(K) at column 0 and lo(K) at column exact_lo_a (elements), B rows likewise at exact_lo_b;
               K %% 64 == 0; lda / ldb are the full row strides.
       Faithful range: the products are as accurate as an fp32 FFMA chain for operands whose amax lies in [2^-10, 2^15].  Below
       2^-14 hi is an fp16 subnormal and lo's absolute floor is 2^-36, so relative precision falls below fp32's once a tensor's amax
       drops under about 2^-12; at |v| >= 65520 hi = inf and the result is NaN (no guard).  Callers keep their operands inside the range
       (the fp32 trainers scale their gradient seeds, DESIGN.md §6). */
    int64_t exact_lo_a, exact_lo_b;
} vf_tc_gemm_t;
int vf_tc_gemm(const vf_tc_gemm_t* p, vf_stream_t s);
/* The tiling vf_tc_gemm chooses for p, without launching or reading any operand: plan[8] = {block_n, TW, TH, TN, halo, exact,
   tiles, CTAs} (TW / TH / TN / halo are 0 for a GEMM).  The persistent grid is CTAs = min(tiles, SMs); CTA c walks tiles c, c + CTAs, ..
   with the n tile fastest, then the m tile (conv: x tile, y tile, image tile), then the batch. */
int vf_tc_gemm_plan(const vf_tc_gemm_t* p, int* plan);

/* ------------------------------------------------------------------------------------------
 * Fused block-causal attention on wgmma (single-stream forward):  out = softmax(mask(Q K^T)) V, no 1/sqrt(dh) scale
 * replaces: models/branching_attention.py:41-61 via models/migt.py:211-217.
 *   qk  bf16 [B, S, 2d]  rows = tokens, columns [0,d) = q, [d,2d) = k (head h at columns h*64..h*64+63)
 *   vt  bf16 [B, d, S]   V transposed (row = channel, contiguous over tokens)
 *   out bf16 [B*S, d]    a token of view v attends to all tokens of views <= v; view = token / block
 *   head dim must be 64; S % block == 0.
 *   first_query: only the query rows >= first_query (rounded down to a 128-row tile) are computed (0: all rows); rows of `out` below the
 *     first computed tile are left untouched.  With first_query > 0 this is the KV-cache decode step — the context's q|k rows and V^T
 *     columns stay in `qk` / `vt` from the prefill and the query view's are appended behind them.
 *   skip_view: the 64 keys of this view are never visited (-1: none; needs block == 64).  Lets the host keep the query view at the start of
 *     a 128-row tile whatever the number of cached context views.
 * ---------------------------------------------------------------------------------------- */
int vf_attn_block_causal_decode(const void* qk_bf16, const void* vt_bf16, int B, int S, int H, int d, int block, int first_query,
                                int skip_view, void* out_bf16, vf_stream_t s);
/* Branching (multi-end) attention of the 3-stream forward — viewformer/models/branching_attention.py:82-126.  qk [B, n_streams*S, 2d] and
 * vt [B, d, n_streams*S] hold the streams side by side.  stream 0: block-causal over its own keys; stream s >= 1: a query of view t attends
 * to the stream-0 keys of views < t and to its own stream's keys of view t (one joint softmax).  out bf16 [B*S, d] = that stream's output.
 * Streams >= 1 need block == 64.  Same fused kernel: the key-tile schedule changes, nothing is materialised in HBM. */
int vf_attn_block_multiend(const void* qk_bf16, const void* vt_bf16, int B, int S, int n_streams, int stream, int H, int d, int block,
                           void* out_bf16, vf_stream_t s);
/* Training forward of one stream (bf16 transformer training step): vf_attn_block_multiend plus the natural-log log-sum-exp of every query
 * row (lse [B, H, S], nullable), an fp32 copy of the output (out_f32 [B*S, d], nullable) and inverted dropout of the probabilities before
 * the P.V product, with vf_dropout's hash mask over this stream's [B, H, S, cols] probability tensor (cols = S for stream 0, 2S with the
 * own-stream keys at columns S + j for streams >= 1).  rate 0 and no outputs: the bits of vf_attn_block_multiend. */
int vf_attn_multiend_train(const void* qk_bf16, const void* vt_bf16, int B, int S, int n_streams, int stream, int H, int d, int block,
                           float rate, uint64_t seed, float* lse, float* out_f32, void* out_bf16, vf_stream_t s);
/* Fused backward of the multi-end attention of all n_streams streams: P is recomputed from Q, K and lse ([n_streams, B, H, S]) with the
 * forward pass's dropout mask (stream s uses seed + s); dout bf16 [n_streams, B*S, d], out fp32 [n_streams, B*S, d] (D = rowsum(dout*out)).
 * dvqk fp32 [n_streams, B*S, 3d], columns v | q | k (zeroed by the caller): stream-0 keys / values get gradient from every stream's
 * queries, stream-s keys / values only from stream s.  Head dim 64, block = 64; no S x S tensor in global memory. */
int vf_attn_multiend_bwd(const void* qk_bf16, const void* vt_bf16, const void* dout_bf16, const float* out, const float* lse, int B, int S,
                         int n_streams, int H, int d, int block, float rate, uint64_t seed, float* dvqk, vf_stream_t s);

/* ------------------------------------------------------------------------------------------
 * Backward pass of the codebook training step (models/vqgan_th.py:395-423, 443-445), fp32.  Data gradients of convolutions and dense
 * layers are calls to vf_simt_gemm / vf_tc_gemm with flipped / transposed weights; what has no forward twin lives here.
 *   vf_conv_wgrad: dW[(tap*Cin + ci) * so_k + co * so_n] += sum over output pixels of X(gathered exactly as the forward conv does:
 *     stride, pad_t / pad_l, optional nearest x2 upsampling) * dY[pixel][co]   (fp32 atomics; dW must be zeroed by the caller).
 *     KH = KW = 1 with so_k = 1, so_n = Cin gives the [Cout, Cin] gradient of a dense layer.
 *   vf_col_sums: out[c] += sum_rows x[row][c]  (bias gradients).
 *   vf_groupnorm_bwd: GroupNorm(groups) [+ swish] backward of y = act(xhat*gamma + beta): dx = rstd (dg gamma - mean - xhat mean2) + add,
 *     dgamma += sum dg xhat, dbeta += sum dg;  mean_rstd from the forward pass; gsums = double [N, groups, 2] scratch;
 *     dx_bf16 (nullable) receives a second copy of dx rounded to bf16 (nearest even), the operand of the next tensor-core data gradient.
 *   vf_softmax_bwd_rows: dS = P (dP - rowsum(dP P)).   vf_l1_grad: dy = scale * sign(y - x), loss_sum += sum |y - x|.
 *   vf_lincomb3: out = a x + b y + c z (y, z nullable).   vf_sumpool2x2: [N,2H,2W,C] -> [N,H,W,C] (nearest-upsample backward).
 *   vf_adam: torch.optim.Adam step number `step` (>= 1) on flat buffers; the gradient is multiplied by grad_scale first (1 / world size).
 * ---------------------------------------------------------------------------------------- */
int vf_conv_wgrad(const float* x, const float* dy, int N, int H, int W, int Cin, int OH, int OW, int Cout, int KH, int KW, int stride,
                  int pad_t, int pad_l, int upsample2x, int64_t so_k, int64_t so_n, float* dw, vf_stream_t s);
int vf_col_sums(const float* x, int64_t rows, int C, float* out, vf_stream_t s);
int vf_groupnorm_bwd(const float* x, const float* dout, const float* mean_rstd, const float* gamma, const float* beta, int N, int HW,
                     int C, int groups, int swish, const float* add, double* gsums, float* dgamma, float* dbeta, float* dx, void* dx_bf16,
                     vf_stream_t s);
int vf_softmax_bwd_rows(const float* P, const float* dP, int64_t rows, int cols, float* dS, vf_stream_t s);
int vf_l1_grad(const float* x, const float* y, int64_t n, float scale, float* dy, double* loss_sum, vf_stream_t s);
int vf_lincomb3(float a, const float* x, float b, const float* y, float c, const float* z, int64_t n, float* out, vf_stream_t s);
/* Tensor-core weight gradient of a 3x3 stride-1 convolution = exact split-fp16 GEMMs with K = pixels (vf_tc_gemm, gemm mode with
 * ntaps = batch1 = 3: tap_coff[ky] shifts the K coordinate of the activation operand by whole rows of the padded grid; the three horizontal
 * shifts are three row blocks of the operand, so M = 3 Cin).  vf_pad_transpose_split lays an NHWC fp32 tensor out as that K-major split
 * operand, fp16 [copies*C][2][L], over the zero-padded pixel grid of row pitch `pitch` (a multiple of 8: TMA box starts stay 16-byte
 * aligned): column margin + ((n (H+2) + y + 1) pitch + x + 1) - (k - copies/2) of copy k; pitch = 0 (copies = 1): plain transpose, column
 * margin + pixel index (weight gradient of a dense layer: K = rows); the caller clears the buffer.
 * vf_sum_splits folds the split-K partial products: out[g*n + i] (+)= sum_s partial[(g*splits + s)*n + i]. */
int vf_pad_transpose_split(const float* x_nhwc, int N, int H, int W, int C, int pitch, int copies, int64_t margin, int64_t L, void* out_f16,
                           vf_stream_t s);
int vf_sum_splits(const float* partial, int groups, int splits, int64_t n, int accumulate, float* out, vf_stream_t s);
/* bf16 training step.  vf_pad_transpose_bf16: the single-pass bf16 operand of the same weight-gradient GEMM (vf_tc_gemm, VF_BF16):
 * bf16 [copies*C][L], the column map of vf_pad_transpose_split with no lo half, over the logical image x (upsample2x = 0) or its nearest x2
 * upsample (upsample2x = 1: [N,2H,2W,C], pitch >= 2W + 2).  mean_rstd (nullable, [N, groups, 2] from the forward pass) applies
 * GroupNorm(groups) [+ swish] on the way, with vf_groupnorm_apply's bf16-output arithmetic; the caller clears the buffer.
 * vf_conv_weights_bf16: one launch over `n` convs (table in device memory) writes the bf16 operands of each from its fp32 master
 * weights w_kn [9*Cin, Cout]: fw [Cout][9*Cin] (forward conv, also the space-to-depth stride-2 conv) and, when bw_bf16 is not null,
 * bw [Cin][9*Cout] = the flipped-tap, channel-swapped weights of the data gradient. */
typedef struct { const float* w_kn; void* fw_bf16; void* bw_bf16; int64_t cin, cout; } vf_conv_weights_bf16_t;
int vf_pad_transpose_bf16(const float* x_nhwc, int N, int H, int W, int C, int upsample2x, int pitch, int copies, int64_t margin, int64_t L,
                          const float* mean_rstd, const float* gamma, const float* beta, int groups, int swish, void* out_bf16, vf_stream_t s);
int vf_conv_weights_bf16(const vf_conv_weights_bf16_t* table, int n, vf_stream_t s);
int vf_sumpool2x2(const float* x, int N, int H, int W, int C, float* y, vf_stream_t s);
int vf_adam(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps, int step,
            float grad_scale, vf_stream_t s);
/* Transformer training step (models/migt.py:464-505, models/utils.py:371-564):
 *   vf_layernorm_bwd: LayerNorm backward over rows of D (statistics recomputed): dx (+ add), dgamma / dbeta accumulated.
 *   vf_gelu_bwd: out = dy * d/dx gelu_erf(pre).   vf_migt_embed_bwd: backward of vf_migt_embed (scatter-add into wte / wpe / pose rows).
 *   vf_cross_entropy_grad: dlogits = w[row] (softmax - smoothed one-hot).   vf_pose_loss_grad: gradient of vf_pose_loss_rows' pos_scale * pos + ori_scale * ori
 *     (both 1 for the plain sum; exp(-w) of DynamicLossWeightingCriterion, migt.py:107-120).
 *   vf_adamw_keras: Keras Adam update (epsilon outside the bias correction) preceded by AdamWeightDecay's p -= lr * wd * p;
 *     the gradient is multiplied by grad_scale * clip_scale first (1 / world size, tf.clip_by_norm factor).
 *   vf_sumsq: out += sum x^2 (per-tensor gradient norms for clip_by_norm).   vf_dropout: stateless inverted dropout, hash(seed, i). */
int vf_layernorm_bwd(const float* x, const float* dy, const float* gamma, const float* add, int64_t rows, int D, float eps,
                     float* dgamma, float* dbeta, float* dx, vf_stream_t s);
int vf_gelu_fwd(const float* x, int64_t n, float* y, vf_stream_t s);      /* exact erf GELU (migt.py:13), kept separate so the pre-activation survives for the backward pass */
int vf_gelu_bwd(const float* pre, const float* dy, int64_t n, float* out, vf_stream_t s);
int vf_migt_embed_bwd(const float* dh, const int32_t* ids, int fixed_token, int64_t BT, int L, int d, float* dwte, float* dwpe,
                      float* dpose, vf_stream_t s);
int vf_cross_entropy_grad(const float* logits, const int32_t* labels, const float* row_weight, int64_t rows, int cols, float smoothing,
                          float* dlogits, vf_stream_t s);
int vf_pose_loss_grad(const float* raw, const float* poses, const float* row_weight, int64_t rows, int tokens_per_view,
                      float pose_multiplier, float pos_scale, float ori_scale, float* draw, vf_stream_t s);
int vf_adamw_keras(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                   float weight_decay, int step, float grad_scale, float clip_scale, vf_stream_t s);
int vf_sumsq(const float* x, int64_t n, double* out, vf_stream_t s);
int vf_dropout(const float* x, int64_t n, float rate, uint64_t seed, float* y, vf_stream_t s);
/* bf16 transformer training step.
 *   vf_to_bf16: y_bf16 = bf16(dropout(x)) with vf_dropout's mask (rate 0: plain round-to-nearest-even); y (nullable) = the fp32 dropout(x).
 *   vf_dense_weights_bf16: one launch over `n` dense layers (table in device memory) writes the bf16 operands of each from its fp32 master
 *     weights w_kn [k, n]: fw [n][k] (the forward GEMM's K-major weights) and bw [k][n] (the data gradient's), either nullable. */
typedef struct { const float* w_kn; void* fw_bf16; void* bw_bf16; int64_t k, n; } vf_dense_weights_bf16_t;
int vf_to_bf16(const float* x, int64_t n, float rate, uint64_t seed, float* y, void* y_bf16, vf_stream_t s);
int vf_dense_weights_bf16(const vf_dense_weights_bf16_t* table, int n, vf_stream_t s);

/* ------------------------------------------------------------------------------------------
 * Evaluation-side kernels (SURVEY.md §8 f2 / f3)
 *   vf_resize_u8: data/_common.py:19-44 (resize_th) on uint8 NHWC images: bilinear (align_corners = False) when `bilinear`, else
 *     torch 'nearest'; result = uint8(clamp(interp(x / 255), 0, 1) * 255).
 *   vf_resize_f32: the same on f32 NHWC images in [0, 1]: result = clamp(interp(x), 0, 1), not quantised.
 *   vf_image_pair_sums: out[2n] = sum |a - b|, out[2n+1] = sum (a - b)^2 over image n (exact integers) -> MSE / MAE / RMSE / PSNR.
 *   vf_ssim_u8: utils/metrics.py:17-73 (7x7 uniform window, VALID, sample covariance, data range 1); out[n] = mean SSIM of image n.
 *   vf_ssim_u8_k: the same with explicit K1 / K2 — utils/metrics.py:176-184 (SSIMMetric, the one the evaluators use) calls
 *     ssim(gt, images, 1), i.e. K1 = 1, so C1 = 1 instead of 1e-4.
 * ---------------------------------------------------------------------------------------- */
int vf_resize_u8(const void* x_u8, int N, int H, int W, int C, int OH, int OW, int bilinear, void* y_u8, vf_stream_t s);
int vf_resize_f32(const float* x, int N, int H, int W, int C, int OH, int OW, int bilinear, float* y, vf_stream_t s);
int vf_image_pair_sums(const void* a_u8, const void* b_u8, int N, int64_t per_image, uint64_t* out, vf_stream_t s);
int vf_ssim_u8(const void* a_u8, const void* b_u8, int N, int H, int W, int C, double* out, vf_stream_t s);
int vf_ssim_u8_k(const void* a_u8, const void* b_u8, int N, int H, int W, int C, double K1, double K2, double* out, vf_stream_t s);

/* ------------------------------------------------------------------------------------------
 * Codebook
 * replaces: models/utils_th.py:34-44 (distance, argmax(-dist), gather), :66 (diff), :70-72 (embed_code)
 *   z [M,D] f32 rows; codebook given TRANSPOSED as Et [K,D] (built once at weight load) with esq[K]=|e|^2.
 *   idx int64 [M]; quant (nullable) f32 [M,D]; diff_sum (nullable) double[1], += sum((e-z)^2).
 *   Index rule of both lookups: the nearest code, equal distances to the smaller index; a NaN distance counts as +inf.  So a row
 *   with a NaN or +-inf element (all its distances NaN or +inf) gets code 0, as argmax(-dist) gives for NaN in the reference, and a
 *   NaN code is never chosen over a finite one; quant and diff_sum follow from that index (NaN / inf for such rows).
 * ---------------------------------------------------------------------------------------- */
int vf_vq_lookup(const float* z, const float* Et, const float* esq, int64_t M, int D, int K,
                 int64_t* idx, float* quant, double* diff_sum, vf_stream_t s);
/* Fused lookup (same result as vf_vq_lookup; viewformer_b200/csrc/vf_vq_fused.cu): one wgmma kernel reads every z row ONCE
 * (fp32 -> fp16 in shared memory), scores it against Eh = fp16(-2 e) [K,D] (vf_vq_prepare_codebook_f16) with wgmma and keeps the
 * two best codes per row straight from the accumulator registers — no score matrix in HBM, 4*D + 8 bytes of traffic per row.  Rows whose two best scores
 * lie within the fp16 rounding bound are settled exactly in fp64 by a second kernel.  tol_factor scales the bound's relative part:
 * 1.0 is the proven worst case (fp16 subnormals and accumulation included), under which every row whose fp64 gap exceeds the bound
 * gets the fp64 nearest code; below 1.0, rows whose fp16 roundings align can be misranked.  Rows outside the fp16 / fixed-point
 * range and codebooks with a code beyond it (or a NaN code) are decided by the exact pass.
 *   D % 64 == 0, D <= 256, K % 256 == 0, K <= 1024, M < 2^31.  worklist: int4[M] scratch; counter: int[2] scratch, on return
 *   counter[0] = rows settled between two candidates, counter[1] = rows settled over all codes.  quant / diff_sum nullable. */
int vf_vq_prepare_codebook_f16(const float* Et, int K, int D, void* Eh_f16, vf_stream_t s);
int vf_vq_lookup_fused(const float* z, const void* Eh_f16, const float* Et /* [K,D] */, const float* E_dk /* the same codebook as [D,K] */,
                       const float* esq, int64_t M, int D, int K,
                       float tol_factor, int64_t* idx, void* worklist, int* counter, float* quant, double* diff_sum, vf_stream_t s);
int vf_gather_rows(const float* table, const int64_t* idx, int64_t M, int D, int64_t n_rows, float* out, vf_stream_t s);
/* training statistics of QuantizeEMA (utils_th.py:47-48): counts[K] += onehot, embed_sum[D,K] += z^T onehot */
int vf_vq_ema_stats(const float* z, const int64_t* idx, int64_t M, int D, int K,
                    float* counts, float* embed_sum_dk, vf_stream_t s);
/* Quantize (utils_th.py:75-124, the gradient-trained codebook variant): gradient of beta * mean((q - sg(z))^2) with respect to the [D,K]
 * codebook from the per-code counts / row sums of vf_vq_ema_stats: grad[d,k] = coef * (counts[k] * E[d,k] - embed_sum[d,k]), or with
 * accumulate != 0 grad[d,k] += that (gradient accumulation over several backward passes). */
int vf_vq_commit_grad(const float* embeddings_dk, const float* counts, const float* embed_sum_dk, int D, int K, float coef,
                      int accumulate, float* grad_dk, vf_stream_t s);
/* EMA update + Laplace-smoothed renormalisation (utils_th.py:55-64).  alpha = float32(1 - decay);
 * corr = 1 - decay^counter (post-increment counter), both computed by the host exactly as torch does.
 * Updates cs_hidden[K], dw_hidden[D,K], embeddings[D,K] and the derived Et[K,D], esq[K]. */
int vf_vq_ema_update(const float* counts, const float* embed_sum_dk, int D, int K, float alpha, float corr, float eps,
                     float* cs_hidden, float* dw_hidden, float* embeddings_dk, float* Et, float* esq, vf_stream_t s);
/* Et[K,D], esq[K] from embeddings[D,K] (weight-load time) */
int vf_vq_prepare_codebook(const float* embeddings_dk, int D, int K, float* Et, float* esq, vf_stream_t s);

/* ------------------------------------------------------------------------------------------
 * Transformer glue
 * ---------------------------------------------------------------------------------------- */
/* h[b,t,l,:] = wte[ids[b,t,l]] + wpe[l] + pose[b,t,:]   (models/migt.py:358-392).
 * ids int32 (negative id -> use fixed_token, e.g. MASK for stream 1); pose f32 [B*T, d]. */
int vf_migt_embed(const int32_t* ids, int fixed_token, const float* wte, const float* wpe, const float* pose,
                  int64_t BT, int L, int d, float* out, vf_stream_t s);
/* Row softmax of fp32 scores -> probabilities (bf16 or f32), written over the first `cols` columns.
 *   mask_mode 0: none.  1: block-causal (branching_attention.py:41-61): row r (view (row0+r)/block)
 *   keeps columns < (view+1)*block; masked entries get probability 0 (reference: logit -1e4 -> exp underflows
 *   to exactly 0 in fp32).  2: multi-end (:82-126): columns [0,half) are stream-0 keys kept when
 *   key view < query view, columns [half, 2*half) are own-stream keys kept when key view == query view. */
int vf_softmax_rows(const float* scores, int64_t rows_total, int rows_per_batch, int cols, int64_t ld_in,
                    int mask_mode, int block, int row0, void* P, int p_dtype, int64_t ld_out, vf_stream_t s);
/* argmax over the last dim (first index wins) — tf.argmax at evaluate/evaluate_transformer.py:123 */
int vf_argmax_rows(const float* x, int64_t rows, int cols, int64_t ld, int64_t* out, vf_stream_t s);
/* pose head post-processing (models/migt.py:159-164): in [rows,7] raw MLP output ->
 * xyz/pose_multiplier | normalised, sign-fixed quaternion */
int vf_pose_postprocess(const float* raw, int64_t rows, float pose_multiplier, float* out, vf_stream_t s);
/* camera pre-processing of generate() in one launch (evaluate/evaluate_transformer.py:70-78, 90-94):
 * cams f32 [B,T,7] (xyz | wxyz).  relative != 0: express every pose relative to view 0 (rotate by the conjugate of
 * view 0's quaternion), then L2-normalise the quaternion (eps 1e-12) and flip it to w >= 0.
 * out [B,T,7]; transform (nullable) [B,7] receives view 0's original pose. */
int vf_cameras_prepare(const float* cams, int B, int T, int relative, float* out, float* transform, vf_stream_t s);
/* inverse map (evaluate_transformer.py:81-87): out[b,i] = transform[b] o cams[b,i];  cams [B,n,7], transform [B,7] */
int vf_cameras_from_relative(const float* cams, const float* transform, int B, int n, float* out, vf_stream_t s);
/* nearest cameras of 7-Scenes localisation: for each of Q query cameras [Q,7] (xyz | wxyz), the k database cameras of least distance,
 * ascending, ties to the lower database index (a stable sort: tf.argsort at evaluate/evaluate_sevenscenes.py:189, tf.argmin at
 * evaluate_sevenscenes_baseline.py:93).  Distances in fp32 with x1 = the database camera, x2 = the query:
 *   mode 0: 0.3 |xyz1 - xyz2| + 2 asin |vec(n(q1) n(q2)*)|   (evaluate_sevenscenes.py:36-45, n = l2 normalisation, eps 1e-12)
 *   mode 1: |xyz1 - xyz2|;  mode 2: 2 asin |vec(n(q1) n(q2)*)|  (evaluate_sevenscenes_baseline.py:43-51)
 * The argument of asin is clamped to 1: for a pose 180 degrees from the query it can round above 1, where the reference's distance is
 * NaN and its argsort order undefined; here it is pi.
 * db [N,7] shared by all queries when db_stride == 0, else query q reads db + q * db_stride (floats, >= 7 N).
 * 1 <= k <= 64, k <= N.  idx_out int32 [Q,k], dist_out f32 [Q,k]. */
int vf_camera_knn(const float* db, int64_t N, int64_t db_stride, const float* queries, int Q, int mode, int k, int32_t* idx_out,
                  float* dist_out, vf_stream_t s);
/* evaluation losses of MIGT.call(compute_losses=True) — models/migt.py:417-448, 165-177 */
int vf_cross_entropy_rows(const float* logits, const int32_t* labels, int64_t rows, int cols, float smoothing, float* out,
                          vf_stream_t s);                       /* sparse softmax CE per row (fp32) */
int vf_pose_loss_rows(const float* raw, const float* poses, int64_t rows, int tokens_per_view, float pose_multiplier,
                      float* pos_out, float* ori_out, vf_stream_t s);   /* per-token MSE of position / raw quaternion */
int vf_row_mean(const float* x, int64_t rows, int n, int start, float* out, vf_stream_t s);   /* out[r] = mean(x[r, start:n]) */

#ifdef __cplusplus
}
#endif
#endif /* VF_B200_H */
