// Generic fp32 CUDA-core implicit GEMM: exact-precision path and the small-channel convolutions
// (3->128 conv_in, 128->3 conv_out, K=7 pose MLP).  64x64x16 tiles, 4x4 register micro-tiles.
// C = act(alpha * A*B + bias) + residual, A gathered either as an NHWC convolution patch matrix
// (models/vqgan_th.py conv sites) or as a dense strided matrix (bmm / Conv1D sites).
#include "vf_common.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, PAD = 4;

__device__ __forceinline__ float ld_elem(const void* p, int dtype, int64_t off) {
    if (dtype == VF_F32) return __ldg(reinterpret_cast<const float*>(p) + off);
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[off]);
}

__global__ void __launch_bounds__(256) simt_gemm_kernel(const vf_simt_gemm_t p) {
    __shared__ float As[BK][BM + PAD];
    __shared__ float Bs[BK][BN + PAD];

    const int tid = threadIdx.x;
    const int bz = blockIdx.z;
    const int b1 = bz / p.batch2, b2 = bz % p.batch2;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;

    const int64_t a_boff = (int64_t)b1 * p.a_sb1 + (int64_t)b2 * p.a_sb2;
    const int64_t b_boff = (int64_t)b1 * p.b_sb1 + (int64_t)b2 * p.b_sb2;
    const int64_t c_boff = (int64_t)b1 * p.c_sb1 + (int64_t)b2 * p.c_sb2;

    // A-load assignment: row am, 4 consecutive k starting at ak0
    const int am = tid >> 2, ak0 = (tid & 3) * 4;
    // B-load assignment: row bk, 4 consecutive n starting at bn0
    const int bk = tid >> 4, bn0 = (tid & 15) * 4;

    // conv: decode the output pixel of row (m0+am) once
    int pn = 0, poy = 0, pox = 0;
    const int gm = m0 + am;
    const bool m_ok = gm < p.M;
    if (p.conv && m_ok) {
        pox = gm % p.OW;
        int t = gm / p.OW;
        poy = t % p.OH;
        pn = t / p.OH;
    }
    const int VH = p.upsample2x ? p.H * 2 : p.H;   // virtual (upsampled) input size
    const int VW = p.upsample2x ? p.W * 2 : p.W;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int ty = tid >> 4, tx = tid & 15;

    for (int k0 = 0; k0 < p.K; k0 += BK) {
        // ---- load A tile
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int gk = k0 + ak0 + i;
            float v = 0.f;
            if (m_ok && gk < p.K) {
                if (p.conv == 2) {
                    // data gradient of a stride-2 convolution (Downsample, vqgan_th.py:45-49: pad (0,1,0,1), VALID): row m is an INPUT
                    // pixel (poy, pox) of the forward conv, A holds dY [N, H, W, Cin=Cout_fwd]; tap (kh, kw) contributes dY[(poy - kh) / 2,
                    // (pox - kw) / 2] when both differences are even and inside dY
                    const int ci = gk % p.Cin;
                    const int tap = gk / p.Cin;
                    const int kw = tap % p.KW, kh = tap / p.KW;
                    const int ty2 = poy + p.pad_t - kh, tx2 = pox + p.pad_l - kw;
                    if (ty2 >= 0 && tx2 >= 0 && !(ty2 & 1) && !(tx2 & 1) && (ty2 >> 1) < p.H && (tx2 >> 1) < p.W)
                        v = ld_elem(p.A, p.a_dtype, a_boff + (((int64_t)pn * p.H + (ty2 >> 1)) * p.W + (tx2 >> 1)) * p.Cin + ci);
                } else if (p.conv) {
                    const int ci = gk % p.Cin;
                    const int tap = gk / p.Cin;
                    const int kw = tap % p.KW, kh = tap / p.KW;
                    const int iy = poy * p.stride + kh - p.pad_t;
                    const int ix = pox * p.stride + kw - p.pad_l;
                    if (iy >= 0 && iy < VH && ix >= 0 && ix < VW) {
                        const int sy = p.upsample2x ? (iy >> 1) : iy;
                        const int sx = p.upsample2x ? (ix >> 1) : ix;
                        v = ld_elem(p.A, p.a_dtype, a_boff + (((int64_t)pn * p.H + sy) * p.W + sx) * p.Cin + ci);
                    }
                } else {
                    v = ld_elem(p.A, p.a_dtype, a_boff + (int64_t)gm * p.a_sm + (int64_t)gk * p.a_sk);
                }
            }
            As[ak0 + i][am] = v;
        }
        // ---- load B tile
        {
            const int gk = k0 + bk;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int gn = n0 + bn0 + j;
                float v = 0.f;
                if (gk < p.K && gn < p.Ncols) v = ld_elem(p.B, p.b_dtype, b_boff + (int64_t)gk * p.b_sk + (int64_t)gn * p.b_sn);
                Bs[bk][bn0 + j] = v;
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w};
            const float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }

    // ---- epilogue
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= p.Ncols) continue;
            float v = acc[i][j] * p.alpha;
            if (p.bias_mode == VF_BIAS_N) v += __ldg(p.bias + n);
            else if (p.bias_mode == VF_BIAS_M) v += __ldg(p.bias + m);
            if (p.act == VF_ACT_GELU_ERF) v = vf_gelu_erf(v);
            const int64_t off = c_boff + (int64_t)m * p.ldc + n;
            if (p.residual) v += __ldg(p.residual + off);
            if (p.C_f32) p.C_f32[off] = v;
            if (p.C_bf16) reinterpret_cast<__nv_bfloat16*>(p.C_bf16)[off] = __float2bfloat16(v);
        }
    }
}

}  // namespace

extern "C" int vf_simt_gemm(const vf_simt_gemm_t* p, vf_stream_t s) {
    VF_CHECK_ARG(p && p->A && p->B, "vf_simt_gemm: null operand");
    VF_CHECK_ARG(p->C_f32 || p->C_bf16, "vf_simt_gemm: no output");
    VF_CHECK_ARG(p->M > 0 && p->Ncols > 0 && p->K > 0, "vf_simt_gemm: bad shape M=%d N=%d K=%d", p->M, p->Ncols, p->K);
    VF_CHECK_ARG(p->batch1 > 0 && p->batch2 > 0, "vf_simt_gemm: bad batch");
    VF_CHECK_ARG(p->act == VF_ACT_NONE || p->act == VF_ACT_GELU_ERF, "vf_simt_gemm: activation %d unsupported (none or GELU)", p->act);
    if (p->conv) {
        VF_CHECK_ARG(p->K == p->KH * p->KW * p->Cin, "vf_simt_gemm: conv K mismatch");
        VF_CHECK_ARG(p->M == p->N * p->OH * p->OW, "vf_simt_gemm: conv M mismatch");
        VF_CHECK_ARG(p->stride == 1 || p->stride == 2, "vf_simt_gemm: stride");
    }
    VF_CHECK_ARG(p->bias_mode == VF_BIAS_NONE || p->bias, "vf_simt_gemm: bias pointer missing");
    dim3 grid((p->M + BM - 1) / BM, (p->Ncols + BN - 1) / BN, p->batch1 * p->batch2);
    VF_CHECK_ARG(grid.y <= 65535 && grid.z <= 65535, "vf_simt_gemm: grid too large");
    simt_gemm_kernel<<<grid, 256, 0, vf_s(s)>>>(*p);
    VF_CHECK_LAUNCH("vf_simt_gemm");
    return VF_OK;
}
