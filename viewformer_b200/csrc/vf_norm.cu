// GroupNorm (two-phase: statistics, then normalise [+swish] [+nearest x2] [+cast]) and LayerNorm.
// HBM-bound kernels: 128-bit loads, one pass each.  NHWC layout: x is [N, HW, C] fp32.
#include "vf_common.cuh"
#include <cuda_fp16.h>

namespace {

// VF_F16X2 output: an fp32 value as (hi, lo) fp16 pair, hi = fp16(v), lo = fp16((v - hi) * 2^11), stored [.., hi(C) | lo(C)]
// — the operand format of the exact tensor-core convolution (vf_tc_gemm.cu, EXACT_LO_SCALE).  v - hi is exact in fp32.
struct f16x2_t { __half h; };
template <typename T> struct out_traits { static constexpr bool fast = false, split = false; };
template <> struct out_traits<__nv_bfloat16> { static constexpr bool fast = true, split = false; };
template <> struct out_traits<f16x2_t> { static constexpr bool fast = false, split = true; };

// ---------------------------------------------------------------------------------------------
// Statistics: per (n, group) sum and sum of squares in double.
// grid = (chunks, N), block = 256.  Each thread owns one channel quad (4 consecutive channels; a quad
// never straddles a group because C/groups is a multiple of 4) and strides over the chunk's pixels.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, int HW, int C, int groups,
                                                       int pix_per_block, double* __restrict__ stats) {
    extern __shared__ double sh[];   // [groups][2]
    const int n = blockIdx.y;
    const int quads = C >> 2;
    const int lanes = 256 / quads;              // pixel lanes per block (quads in {8..128})
    const int cq = threadIdx.x % quads;
    const int pl = threadIdx.x / quads;
    for (int i = threadIdx.x; i < groups * 2; i += 256) sh[i] = 0.0;
    __syncthreads();
    const int p0 = blockIdx.x * pix_per_block;
    const int p1 = min(HW, p0 + pix_per_block);
    float s[4] = {0.f, 0.f, 0.f, 0.f}, ss[4] = {0.f, 0.f, 0.f, 0.f};
    if (pl < lanes) {
        const float4* base = reinterpret_cast<const float4*>(x + (int64_t)n * HW * C) + cq;
        int p = p0 + pl;
        for (; p + 3 * lanes < p1; p += 4 * lanes) {          // 4 independent 128-bit loads in flight
            float4 v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = __ldg(base + (int64_t)(p + k * lanes) * quads);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s[0] += v[k].x; s[1] += v[k].y; s[2] += v[k].z; s[3] += v[k].w;
                ss[0] += v[k].x * v[k].x; ss[1] += v[k].y * v[k].y; ss[2] += v[k].z * v[k].z; ss[3] += v[k].w * v[k].w;
            }
        }
        for (; p < p1; p += lanes) {
            const float4 v = __ldg(base + (int64_t)p * quads);
            s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
            ss[0] += v.x * v.x; ss[1] += v.y * v.y; ss[2] += v.z * v.z; ss[3] += v.w * v.w;
        }
        const int cpg = C / groups;
        if ((cpg & 3) == 0) {        // the quad lies inside one group
            const int g = (cq * 4) / cpg;
            atomicAdd(&sh[g * 2 + 0], (double)((s[0] + s[1]) + (s[2] + s[3])));
            atomicAdd(&sh[g * 2 + 1], (double)((ss[0] + ss[1]) + (ss[2] + ss[3])));
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int g = (cq * 4 + j) / cpg;
                atomicAdd(&sh[g * 2 + 0], (double)s[j]);
                atomicAdd(&sh[g * 2 + 1], (double)ss[j]);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < groups * 2; i += 256) atomicAdd(&stats[(int64_t)n * groups * 2 + i], sh[i]);
}

// sums (double) -> (mean, rstd) floats, one thread per (n, group): keeps fp64 math out of the streaming kernel
__global__ void gn_finalize_kernel(const double* __restrict__ sums, int total, double cnt, float eps, float* __restrict__ mr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const double mean = sums[2 * i] / cnt;
    double var = sums[2 * i + 1] / cnt - mean * mean;
    if (var < 0) var = 0;
    mr[2 * i] = (float)mean;
    mr[2 * i + 1] = (float)(1.0 / sqrt(var + (double)eps));
}

// ---------------------------------------------------------------------------------------------
// Apply: one thread per channel quad of one pixel.
// ---------------------------------------------------------------------------------------------
template <typename OutT>
__device__ __forceinline__ void store4(OutT* p, float a, float b, float c, float d);
template <>
__device__ __forceinline__ void store4<float>(float* p, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
template <>
__device__ __forceinline__ void store4<__nv_bfloat16>(__nv_bfloat16* p, float a, float b, float c, float d) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&lo);
    u.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(p) = u;
}

// 128-bit (fp32) / 64-bit (bf16) channel-quad loads
template <typename InT>
__device__ __forceinline__ float4 load4(const InT* p);
template <>
__device__ __forceinline__ float4 load4<float>(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}
template <>
__device__ __forceinline__ float4 load4<__nv_bfloat16>(const __nv_bfloat16* p) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xffff0000u));
}

// hi halves at p, lo halves at p + lo_off
__device__ __forceinline__ void store4_split(f16x2_t* p, int64_t lo_off, float a, float b, float c, float d) {
    const float v[4] = {a, b, c, d};
    __half hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        hi[j] = __float2half_rn(v[j]);
        lo[j] = __float2half_rn((v[j] - __half2float(hi[j])) * 2048.0f);
    }
    uint2 uh, ul;
    uh.x = (uint32_t)__half_as_ushort(hi[0]) | ((uint32_t)__half_as_ushort(hi[1]) << 16);
    uh.y = (uint32_t)__half_as_ushort(hi[2]) | ((uint32_t)__half_as_ushort(hi[3]) << 16);
    ul.x = (uint32_t)__half_as_ushort(lo[0]) | ((uint32_t)__half_as_ushort(lo[1]) << 16);
    ul.y = (uint32_t)__half_as_ushort(lo[2]) | ((uint32_t)__half_as_ushort(lo[3]) << 16);
    *reinterpret_cast<uint2*>(p) = uh;
    *reinterpret_cast<uint2*>(p + lo_off) = ul;
}

template <typename OutT>
__device__ __forceinline__ float gn_swish(float v) {
    // bf16 operand output: ex2.approx / rcp.approx (rel. error ~1e-6, far below bf16 rounding) keep this kernel
    // memory-bound; the fp32 and split-fp16 (exact-path) instantiations use expf and a true division
    if constexpr (out_traits<OutT>::fast) return __fdividef(v, 1.0f + __expf(-v));
    else return vf_swish(v);
}

// Apply: grid (pixel chunks, N).  A thread owns ONE channel quad of ONE image for its whole life, so the affine
// (x - mean) * rstd * gamma + beta is folded once into (scale, shift) registers — the bf16 instantiation evaluates it as
// one FMA per element; the exact fp32 instantiation keeps the reference's operation order — and the streaming loop is
// load -> fma -> swish -> store with four independent 128-bit loads in flight and no integer division.
// layout: 0 same, 1 nearest-neighbour x2 upsample, 2 space-to-depth ([N,H,W,C] -> [N,H/2,W/2,4C], block a*2+b <- (2y+a, 2x+b))
template <typename InT, typename OutT, int kLayout>
__global__ void __launch_bounds__(256) gn_apply_kernel(const InT* __restrict__ x, const float* __restrict__ mr,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta, int H, int W,
                                                       int C, int groups, int normalize, int swish, int pix_per_block,
                                                       OutT* __restrict__ y) {
    const int quads = C >> 2;                               // 256 % quads == 0 (checked by the launcher)
    const int lanes = 256 / quads;
    const int cq = threadIdx.x % quads, pl = threadIdx.x / quads;
    const int n = blockIdx.y, HW = H * W;
    float mu[4] = {0.f, 0.f, 0.f, 0.f}, rs[4] = {1.f, 1.f, 1.f, 1.f}, ga[4] = {1.f, 1.f, 1.f, 1.f}, be[4] = {0.f, 0.f, 0.f, 0.f};
    if (normalize) {
        const int cpg = C / groups;
        const float4 g4 = __ldg(reinterpret_cast<const float4*>(gamma) + cq);
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(beta) + cq);
        ga[0] = g4.x; ga[1] = g4.y; ga[2] = g4.z; ga[3] = g4.w;
        be[0] = b4.x; be[1] = b4.y; be[2] = b4.z; be[3] = b4.w;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 m = __ldg(reinterpret_cast<const float2*>(mr) + (int64_t)n * groups + (cq * 4 + j) / cpg);
            mu[j] = m.x;
            rs[j] = m.y;
        }
    }
    float sc[4], sh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { sc[j] = rs[j] * ga[j]; sh[j] = be[j] - mu[j] * sc[j]; }

    auto body = [&](float4 v, int p) {
        float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (normalize) {
                if constexpr (out_traits<OutT>::fast) e[j] = fmaf(e[j], sc[j], sh[j]);
                else e[j] = (e[j] - mu[j]) * rs[j] * ga[j] + be[j];
            }
            if (swish) e[j] = gn_swish<OutT>(e[j]);
        }
        if constexpr (out_traits<OutT>::split) {
            // pixel stride doubles ([hi | lo]); the lo half starts after the LOGICAL channel count of the output layout
            if constexpr (kLayout == 0) {
                store4_split(y + ((int64_t)n * HW + p) * (2 * C) + cq * 4, C, e[0], e[1], e[2], e[3]);
            } else if constexpr (kLayout == 2) {
                const int yy = p / W, xx = p - yy * W;
                const int64_t o = (((int64_t)n * (H >> 1) + (yy >> 1)) * (W >> 1) + (xx >> 1)) * (8 * (int64_t)C) + ((yy & 1) * 2 + (xx & 1)) * C + cq * 4;
                store4_split(y + o, 4 * (int64_t)C, e[0], e[1], e[2], e[3]);
            } else {
                const int yy = p / W, xx = p - yy * W;
                const int64_t W2 = 2 * (int64_t)W, C2 = 2 * (int64_t)C;
                const int64_t o = (((int64_t)n * 2 * H + 2 * yy) * W2 + 2 * xx) * C2 + cq * 4;
                store4_split(y + o, C, e[0], e[1], e[2], e[3]);
                store4_split(y + o + C2, C, e[0], e[1], e[2], e[3]);
                store4_split(y + o + W2 * C2, C, e[0], e[1], e[2], e[3]);
                store4_split(y + o + W2 * C2 + C2, C, e[0], e[1], e[2], e[3]);
            }
        } else if constexpr (kLayout == 0) {
            store4<OutT>(y + ((int64_t)n * HW + p) * C + cq * 4, e[0], e[1], e[2], e[3]);
        } else if constexpr (kLayout == 2) {
            const int yy = p / W, xx = p - yy * W;
            const int64_t o = ((((int64_t)n * (H >> 1) + (yy >> 1)) * (W >> 1) + (xx >> 1)) * 4 + ((yy & 1) * 2 + (xx & 1))) * C + cq * 4;
            store4<OutT>(y + o, e[0], e[1], e[2], e[3]);
        } else {
            const int yy = p / W, xx = p - yy * W;
            const int64_t W2 = 2 * (int64_t)W;
            const int64_t o = (((int64_t)n * 2 * H + 2 * yy) * W2 + 2 * xx) * C + cq * 4;
            store4<OutT>(y + o, e[0], e[1], e[2], e[3]);
            store4<OutT>(y + o + C, e[0], e[1], e[2], e[3]);
            store4<OutT>(y + o + W2 * C, e[0], e[1], e[2], e[3]);
            store4<OutT>(y + o + W2 * C + C, e[0], e[1], e[2], e[3]);
        }
    };

    const int p0 = blockIdx.x * pix_per_block;
    const int p1 = min(HW, p0 + pix_per_block);
    const InT* base = x + (int64_t)n * HW * C + cq * 4;
    int p = p0 + pl;
    for (; p + 3 * lanes < p1; p += 4 * lanes) {
        float4 v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = load4<InT>(base + (int64_t)(p + k * lanes) * C);
#pragma unroll
        for (int k = 0; k < 4; ++k) body(v[k], p + k * lanes);
    }
    for (; p < p1; p += lanes) body(load4<InT>(base + (int64_t)p * C), p);
}

// ---------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row cached in registers (D <= 1024, D % 4 == 0).
// ---------------------------------------------------------------------------------------------
template <typename OutT>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, int64_t rows, int D, float eps,
                                                        OutT* __restrict__ y) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const int quads = D >> 2;
    const float4* xr = reinterpret_cast<const float4*>(x + row * D);
    float4 v[8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int q = lane + i * 32;
        if (q < quads) {
            v[i] = __ldg(xr + q);
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
    }
    s = warp_sum(s);
    const float mean = s / (float)D;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int q = lane + i * 32;
        if (q < quads) {
            const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            ss += (a * a + b * b) + (c * c + d * d);
        }
    }
    ss = warp_sum(ss);
    const float rstd = rsqrtf(ss / (float)D + eps);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int q = lane + i * 32;
        if (q < quads) {
            const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma) + q);
            const float4 be = __ldg(reinterpret_cast<const float4*>(beta) + q);
            store4<OutT>(y + row * D + q * 4, (v[i].x - mean) * rstd * ga.x + be.x, (v[i].y - mean) * rstd * ga.y + be.y,
                         (v[i].z - mean) * rstd * ga.z + be.z, (v[i].w - mean) * rstd * ga.w + be.w);
        }
    }
}

// fp32 [rows, C] -> split fp16 [rows, hi(C) | lo(C)] for any C % 4 == 0: the operand form of the exact tensor-core GEMM
__global__ void split_rows_kernel(const float* __restrict__ x, long long quads_total, int quads_per_row, __half* __restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < quads_total; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        const long long r = i / quads_per_row;
        const int q = (int)(i - r * quads_per_row);
        const float e[4] = {v.x, v.y, v.z, v.w};
        __half hi[4], lo[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            hi[j] = __float2half_rn(e[j]);
            lo[j] = __float2half_rn((e[j] - __half2float(hi[j])) * 2048.0f);
        }
        __half* o = out + r * (8LL * quads_per_row) + 4 * q;
        *reinterpret_cast<uint2*>(o) = *reinterpret_cast<const uint2*>(hi);
        *reinterpret_cast<uint2*>(o + 4 * quads_per_row) = *reinterpret_cast<const uint2*>(lo);
    }
}

}  // namespace

extern "C" int vf_split_f16x2(const float* x, int64_t rows, int C, void* out_f16, vf_stream_t s) {
    VF_CHECK_ARG(x && out_f16 && C > 0 && C % 4 == 0, "vf_split_f16x2: C must be a positive multiple of 4 (C=%d)", C);
    if (rows == 0) return VF_OK;
    const long long quads = rows * (C / 4);
    long long blocks = (quads + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    split_rows_kernel<<<(unsigned)blocks, 256, 0, vf_s(s)>>>(x, quads, C / 4, reinterpret_cast<__half*>(out_f16));
    VF_CHECK_LAUNCH("vf_split_f16x2");
    return VF_OK;
}

extern "C" int vf_groupnorm_stats(const float* x, int N, int HW, int C, int groups, float eps, double* stats, float* mean_rstd,
                                  vf_stream_t s) {
    VF_CHECK_ARG(x && stats && mean_rstd, "vf_groupnorm_stats: null pointer");
    VF_CHECK_ARG(C % groups == 0 && C % 4 == 0 && C / 4 <= 256 && 256 % (C / 4) == 0,
                 "vf_groupnorm_stats: unsupported C=%d groups=%d", C, groups);
    cudaError_t e = cudaMemsetAsync(stats, 0, sizeof(double) * 2 * groups * N, vf_s(s));
    if (e != cudaSuccess) { vf_set_error("vf_groupnorm_stats: memset: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
    // enough blocks to fill the machine, at least 64 pixels per block
    int chunks = (HW + 63) / 64;
    const int target = (132 * 8 + N - 1) / N;
    if (chunks > target) chunks = target;
    if (chunks < 1) chunks = 1;
    const int ppb = (HW + chunks - 1) / chunks;
    chunks = (HW + ppb - 1) / ppb;
    dim3 grid(chunks, N);
    gn_stats_kernel<<<grid, 256, sizeof(double) * 2 * groups, vf_s(s)>>>(x, HW, C, groups, ppb, stats);
    VF_CHECK_LAUNCH("vf_groupnorm_stats");
    gn_finalize_kernel<<<(N * groups + 127) / 128, 128, 0, vf_s(s)>>>(stats, N * groups, (double)HW * (C / groups), eps, mean_rstd);
    VF_CHECK_LAUNCH("vf_groupnorm_stats(finalize)");
    return VF_OK;
}

extern "C" int vf_groupnorm_finalize(const double* sums, int n_stats, double count, float eps, float* mean_rstd, vf_stream_t s) {
    VF_CHECK_ARG(sums && mean_rstd && n_stats >= 0 && count > 0, "vf_groupnorm_finalize: bad args");
    if (n_stats == 0) return VF_OK;
    gn_finalize_kernel<<<(n_stats + 127) / 128, 128, 0, vf_s(s)>>>(sums, n_stats, count, eps, mean_rstd);
    VF_CHECK_LAUNCH("vf_groupnorm_finalize");
    return VF_OK;
}

template <typename InT, typename OutT>
static void gn_apply_launch(const void* x, const float* stats, const float* gamma, const float* beta, int N, int H, int W, int C,
                            int groups, int normalize, int swish, int layout, void* y, cudaStream_t st) {
    const int HW = H * W;
    const int lanes = 256 / (C / 4);
    // 16 pixel rounds per thread (4 x 4 loads in flight) unless that leaves the machine short of blocks
    int ppb = lanes * 16;
    while (ppb > lanes * 4 && (int64_t)((HW + ppb - 1) / ppb) * N < 132 * 8) ppb >>= 1;
    dim3 grid((HW + ppb - 1) / ppb, N);
    const InT* xi = reinterpret_cast<const InT*>(x);
    OutT* yo = reinterpret_cast<OutT*>(y);
    if (layout == 0)
        gn_apply_kernel<InT, OutT, 0><<<grid, 256, 0, st>>>(xi, stats, gamma, beta, H, W, C, groups, normalize, swish, ppb, yo);
    else if (layout == 1)
        gn_apply_kernel<InT, OutT, 1><<<grid, 256, 0, st>>>(xi, stats, gamma, beta, H, W, C, groups, normalize, swish, ppb, yo);
    else
        gn_apply_kernel<InT, OutT, 2><<<grid, 256, 0, st>>>(xi, stats, gamma, beta, H, W, C, groups, normalize, swish, ppb, yo);
}

extern "C" int vf_groupnorm_apply(const void* x, int x_dtype, const float* stats, const float* gamma, const float* beta, int N,
                                  int H, int W, int C, int groups, float eps, int normalize, int swish, int layout,
                                  void* y, int y_dtype, vf_stream_t s) {
    (void)eps;
    VF_CHECK_ARG(x && y, "vf_groupnorm_apply: null pointer");
    VF_CHECK_ARG(C % 4 == 0 && C / 4 <= 256 && 256 % (C / 4) == 0, "vf_groupnorm_apply: unsupported C=%d", C);
    VF_CHECK_ARG((int64_t)H * W < (1ll << 30) && N <= 65535, "vf_groupnorm_apply: image too large");
    VF_CHECK_ARG(layout >= 0 && layout <= 2, "vf_groupnorm_apply: bad layout %d", layout);
    VF_CHECK_ARG(layout != 2 || (H % 2 == 0 && W % 2 == 0), "vf_groupnorm_apply: space-to-depth needs even H, W");
    if (normalize) {
        VF_CHECK_ARG(stats && gamma && beta, "vf_groupnorm_apply: normalize needs stats/gamma/beta");
        VF_CHECK_ARG(C % groups == 0, "vf_groupnorm_apply: unsupported C=%d groups=%d", C, groups);
    }
    if (N == 0 || H * W == 0) return VF_OK;
    if (x_dtype == VF_F32 && y_dtype == VF_F32)
        gn_apply_launch<float, float>(x, stats, gamma, beta, N, H, W, C, groups, normalize, swish, layout, y, vf_s(s));
    else if (x_dtype == VF_F32 && y_dtype == VF_BF16)
        gn_apply_launch<float, __nv_bfloat16>(x, stats, gamma, beta, N, H, W, C, groups, normalize, swish, layout, y, vf_s(s));
    else if (x_dtype == VF_BF16 && y_dtype == VF_BF16)
        gn_apply_launch<__nv_bfloat16, __nv_bfloat16>(x, stats, gamma, beta, N, H, W, C, groups, normalize, swish, layout, y, vf_s(s));
    else if (x_dtype == VF_F32 && y_dtype == VF_F16X2)
        gn_apply_launch<float, f16x2_t>(x, stats, gamma, beta, N, H, W, C, groups, normalize, swish, layout, y, vf_s(s));
    else
        VF_CHECK_ARG(false, "vf_groupnorm_apply: unsupported dtype pair (x %d, y %d)", x_dtype, y_dtype);
    VF_CHECK_LAUNCH("vf_groupnorm_apply");
    return VF_OK;
}

extern "C" int vf_layernorm(const float* x, const float* gamma, const float* beta, int64_t rows, int D, float eps, void* y,
                            int y_dtype, vf_stream_t s) {
    VF_CHECK_ARG(x && gamma && beta && y, "vf_layernorm: null pointer");
    VF_CHECK_ARG(D % 4 == 0 && D <= 1024, "vf_layernorm: unsupported D=%d", D);
    if (rows == 0) return VF_OK;
    const unsigned blocks = (unsigned)((rows + 7) / 8);
    if (y_dtype == VF_F32)
        layernorm_kernel<float><<<blocks, 256, 0, vf_s(s)>>>(x, gamma, beta, rows, D, eps, reinterpret_cast<float*>(y));
    else if (y_dtype == VF_BF16)
        layernorm_kernel<__nv_bfloat16><<<blocks, 256, 0, vf_s(s)>>>(x, gamma, beta, rows, D, eps,
                                                                     reinterpret_cast<__nv_bfloat16*>(y));
    else
        VF_CHECK_ARG(false, "vf_layernorm: bad dtype");
    VF_CHECK_LAUNCH("vf_layernorm");
    return VF_OK;
}
