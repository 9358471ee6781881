// LPIPS-VGG16 (include/vf_b200_lpips.h): the max-pool that feeds the next exact convolution its split-fp16 operand, and the fused
// per-tap head (channel normalisation, squared difference, 1x1 "lin" layer, spatial mean).  The convolutions themselves are
// vf_lpips_conv_in (vf_conv_small.cu) and vf_tc_gemm.
#include "vf_common.cuh"
#include "../../include/vf_b200_lpips.h"
#include <cuda_fp16.h>

namespace {

// max that keeps a NaN from either side, as torch's max_pool2d does (fmaxf would drop it)
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }

// one thread per (output pixel, 4 channels): four float4 loads of the 2x2 window, one hi and one lo 8-byte store
__global__ void maxpool2x2_split_kernel(const float* __restrict__ x, int H, int W, int C, int OH, int OW, long long total,
                                        __half* __restrict__ out) {
    const int quads = C / 4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long pix = i / quads;
        const int q = (int)(i - pix * quads);
        const int ox = (int)(pix % OW);
        const long long t = pix / OW;
        const int oy = (int)(t % OH);
        const long long n = t / OH;
        const float* p = x + ((n * H + 2 * oy) * W + 2 * ox) * C + 4 * q;
        const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + C));
        const float4 c = __ldg(reinterpret_cast<const float4*>(p + (long long)W * C)), d = __ldg(reinterpret_cast<const float4*>(p + (long long)W * C + C));
        const float e[4] = {nan_max(nan_max(a.x, b.x), nan_max(c.x, d.x)), nan_max(nan_max(a.y, b.y), nan_max(c.y, d.y)),
                            nan_max(nan_max(a.z, b.z), nan_max(c.z, d.z)), nan_max(nan_max(a.w, b.w), nan_max(c.w, d.w))};
        __half hi[4], lo[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {                    // vf_split_f16x2's split: hi = fp16(v), lo = fp16((v - hi) * 2^11)
            hi[j] = __float2half_rn(e[j]);
            lo[j] = __float2half_rn((e[j] - __half2float(hi[j])) * 2048.0f);
        }
        __half* o = out + pix * (2LL * C) + 4 * q;
        *reinterpret_cast<uint2*>(o) = *reinterpret_cast<const uint2*>(hi);
        *reinterpret_cast<uint2*>(o + C) = *reinterpret_cast<const uint2*>(lo);
    }
}

constexpr int TAP_PIX = 64;          // pixels per block of the head; a warp takes 8 of them in order

// the same value in every lane: the butterfly sum of lane 0
__device__ __forceinline__ float warp_sum_bcast(float v) { return __shfl_sync(0xffffffffu, warp_sum(v), 0); }

// V = C / 32 channels per lane.  Block (pixel chunk, pair): every pixel's term in fp32, the chunk's sum in fp64 in pixel order.
template <int V>
__global__ void __launch_bounds__(256) lpips_tap_kernel(const float* __restrict__ f, int HW, int Npairs, const float* __restrict__ lin,
                                                        double* __restrict__ partial) {
    constexpr int C = 32 * V;
    __shared__ double warp_part[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = blockIdx.y;
    float w[V];
#pragma unroll
    for (int j = 0; j < V; ++j) w[j] = __ldg(lin + lane * V + j);
    double acc = 0.0;
    for (int k = 0; k < TAP_PIX / 8; ++k) {
        const int p = blockIdx.x * TAP_PIX + warp * (TAP_PIX / 8) + k;
        if (p >= HW) break;
        const float* p0 = f + ((long long)n * HW + p) * C + lane * V;
        const float* p1 = f + ((long long)(n + Npairs) * HW + p) * C + lane * V;
        float a[V], b[V];
#pragma unroll
        for (int j = 0; j < V; j += 2) {
            const float2 u = __ldg(reinterpret_cast<const float2*>(p0 + j)), v = __ldg(reinterpret_cast<const float2*>(p1 + j));
            a[j] = u.x; a[j + 1] = u.y; b[j] = v.x; b[j + 1] = v.y;
        }
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) { s0 = __fmaf_rn(a[j], a[j], s0); s1 = __fmaf_rn(b[j], b[j], s1); }
        const float n0 = __fadd_rn(sqrtf(warp_sum_bcast(s0)), 1e-10f), n1 = __fadd_rn(sqrtf(warp_sum_bcast(s1)), 1e-10f);
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const float r = __fsub_rn(__fdiv_rn(a[j], n0), __fdiv_rn(b[j], n1));
            t = __fmaf_rn(w[j], __fmul_rn(r, r), t);
        }
        t = warp_sum(t);
        acc += (double)t;                               // lane 0's sum is the one kept
    }
    if (lane == 0) warp_part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += warp_part[i];
        partial[(long long)n * gridDim.x + blockIdx.x] = s;
    }
}

// one warp per pair: the chunk sums in a fixed order, then out[n] += sum / HW
__global__ void lpips_tap_finish_kernel(const double* __restrict__ partial, int nblk, int HW, double* __restrict__ out) {
    const int n = blockIdx.x, lane = threadIdx.x;
    double s = 0.0;
    for (int i = lane; i < nblk; i += 32) s += partial[(long long)n * nblk + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[n] += s / (double)HW;
}

}  // namespace

extern "C" int vf_maxpool2x2_split(const float* x, int N, int H, int W, int C, void* out_f16, vf_stream_t s) {
    VF_CHECK_ARG(x && out_f16, "vf_maxpool2x2_split: null pointer");
    VF_CHECK_ARG(N >= 0 && H >= 0 && W >= 0 && C > 0 && C % 4 == 0, "vf_maxpool2x2_split: C must be a positive multiple of 4 (C=%d)", C);
    const int OH = H / 2, OW = W / 2;
    const long long total = (long long)N * OH * OW * (C / 4);
    if (total == 0) return VF_OK;
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 64) blocks = 132 * 64;
    maxpool2x2_split_kernel<<<(unsigned)blocks, 256, 0, vf_s(s)>>>(x, H, W, C, OH, OW, total, reinterpret_cast<__half*>(out_f16));
    VF_CHECK_LAUNCH("vf_maxpool2x2_split");
    return VF_OK;
}

extern "C" int vf_lpips_tap(const float* f, int N, int H, int W, int C, const float* lin, double* partial, double* out, vf_stream_t s) {
    VF_CHECK_ARG(f && lin && partial && out, "vf_lpips_tap: null pointer");
    VF_CHECK_ARG(C == 64 || C == 128 || C == 256 || C == 512, "vf_lpips_tap: C must be 64, 128, 256 or 512 (got %d)", C);
    VF_CHECK_ARG(N >= 0 && N <= 65535 && H > 0 && W > 0 && (long long)H * W < (1ll << 31), "vf_lpips_tap: shape out of range");
    if (N == 0) return VF_OK;
    const int HW = H * W, nblk = (HW + TAP_PIX - 1) / TAP_PIX;
    const dim3 grid(nblk, N);
    if (C == 64) lpips_tap_kernel<2><<<grid, 256, 0, vf_s(s)>>>(f, HW, N, lin, partial);
    else if (C == 128) lpips_tap_kernel<4><<<grid, 256, 0, vf_s(s)>>>(f, HW, N, lin, partial);
    else if (C == 256) lpips_tap_kernel<8><<<grid, 256, 0, vf_s(s)>>>(f, HW, N, lin, partial);
    else lpips_tap_kernel<16><<<grid, 256, 0, vf_s(s)>>>(f, HW, N, lin, partial);
    VF_CHECK_LAUNCH("vf_lpips_tap");
    lpips_tap_finish_kernel<<<N, 32, 0, vf_s(s)>>>(partial, nblk, HW, out);
    VF_CHECK_LAUNCH("vf_lpips_tap");
    return VF_OK;
}
