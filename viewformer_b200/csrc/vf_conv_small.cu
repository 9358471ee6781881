// Exact fp32 3x3 convolutions for the two layers whose channel counts are too small for a tensor-core tile:
//   conv_in   C -> 128 @128x128  (viewformer/models/vqgan_th.py:159-163): output-write bound
//   conv_out  128 -> C @128x128  (vqgan_th.py:285-289): input-read bound
// C = 3 (RGB) or 4 (RGB + mask: the CO3Dv2 codebooks, data/loaders/co3dv2.py:149-153).  Both are stride-1, pad-1, NHWC.
// The small-Cin kernel also runs LPIPS's first VGG16 layer (vf_lpips_conv_in, 3 -> 64 + ReLU) straight from the uint8 images.
#include "vf_common.cuh"
#include "../../include/vf_b200_lpips.h"

namespace {

// Input readers of the small-Cin conv: element i (channel c) of an NHWC tensor as the conv sees it.
struct InputF32 {                   // fp32, as stored
    const float* x;
    __device__ __forceinline__ float operator()(int64_t i, int) const { return __ldg(x + i); }
};
struct InputU8Scaled {              // uint8 through tf.image.convert_image_dtype (x * fp32(1/255)) and lpips' ScalingLayer ((v - shift) / scale)
    const uint8_t* x; const float* shift; const float* scale;
    __device__ __forceinline__ float operator()(int64_t i, int c) const {
        const float v = __fmul_rn((float)__ldg(x + i), (float)(1.0 / 255.0));
        return __fdiv_rn(__fsub_rn(v, __ldg(shift + c)), __ldg(scale + c));
    }
};

// ------------------------------------------------------------------------------------------------
// Small Cin (<= 4): block = 32 lanes (pixels along x) x (Cout/16) warps; each thread computes 2 pixels
// (x, x+32) x 16 output channels.  Weights [9*Cin][Cout] live in shared memory and are read as broadcast float4.
// Padding is zero in the input the conv sees (after In's conversion); RELU: max(y, 0) on the output.
// ------------------------------------------------------------------------------------------------
template <int CIN, typename In, bool RELU>
__global__ void __launch_bounds__(256) conv3x3_small_cin_kernel(const In x, const float* __restrict__ w_kn,
                                                                  const float* __restrict__ bias, int N, int H, int W, int Cout,
                                                                  float* __restrict__ y) {
    extern __shared__ float ws[];                       // [9*CIN][Cout]
    constexpr int K = 9 * CIN;
    for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) ws[i] = w_kn[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;      // g: group of 16 output channels
    const int xb = blockIdx.x * 64;
    const int yy = blockIdx.y, n = blockIdx.z;
    float in[2][K];
#pragma unroll
    for (int px = 0; px < 2; ++px) {
        const int xx = xb + lane + px * 32;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const int iy = yy + t / 3 - 1, ix = xx + t % 3 - 1;
            const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
            for (int c = 0; c < CIN; ++c) in[px][t * CIN + c] = ok ? x((((int64_t)n * H + iy) * W + ix) * CIN + c, c) : 0.f;
        }
    }
    float acc[2][16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float b = bias ? __ldg(bias + g * 16 + j) : 0.f;
        acc[0][j] = b;
        acc[1][j] = b;
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
            const float4 w4 = *reinterpret_cast<const float4*>(&ws[k * Cout + g * 16 + j4 * 4]);
#pragma unroll
            for (int px = 0; px < 2; ++px) {
                acc[px][j4 * 4 + 0] = fmaf(in[px][k], w4.x, acc[px][j4 * 4 + 0]);
                acc[px][j4 * 4 + 1] = fmaf(in[px][k], w4.y, acc[px][j4 * 4 + 1]);
                acc[px][j4 * 4 + 2] = fmaf(in[px][k], w4.z, acc[px][j4 * 4 + 2]);
                acc[px][j4 * 4 + 3] = fmaf(in[px][k], w4.w, acc[px][j4 * 4 + 3]);
            }
        }
    }
#pragma unroll
    for (int px = 0; px < 2; ++px) {
        const int xx = xb + lane + px * 32;
        if (xx >= W) continue;
        float* o = y + (((int64_t)n * H + yy) * W + xx) * Cout + g * 16;
        if (RELU) {
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[px][j] = vf_relu(acc[px][j]);
        }
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4)
            *reinterpret_cast<float4*>(o + j4 * 4) = make_float4(acc[px][j4 * 4], acc[px][j4 * 4 + 1], acc[px][j4 * 4 + 2], acc[px][j4 * 4 + 3]);
    }
}

// ------------------------------------------------------------------------------------------------
// Cin = CIN (3 or 4), Cout = 128 (conv_in of the released models).  Block = 8 warps over a ROWS x 64-pixel tile:
//   * the (ROWS+2) x 66 x CIN input patch is staged once in shared memory (zero padded to 4 floats per pixel), so every input read in
//     the main loop is a warp-uniform LDS.128 broadcast;
//   * lane l owns output channels 4l..4l+3 (exactly one GroupNorm(32) group) and keeps its 9 CIN x 4 weights in registers;
//   * every store is one coalesced 512-byte pixel row;
//   * the GroupNorm statistics of the OUTPUT (sum, sum of squares per (image, group)) are accumulated on the fly —
//     one fp64 RED per (block, group, statistic) — which removes the separate 2.4 GB statistics pass of the encoder.
// FFMA-bound: 9 CIN * 128 FMA per pixel.  The FMA order is (dy, dx, channel) for every CIN.
// ------------------------------------------------------------------------------------------------
constexpr int CI_ROWS = 4, CI_W = 64;
template <int CIN>
__global__ void __launch_bounds__(256) conv3x3_cin_cout128_kernel(const float* __restrict__ x, const float* __restrict__ w_kn,
                                                                  const float* __restrict__ bias, int N, int H, int W,
                                                                  float* __restrict__ y, double* __restrict__ gn_sums) {
    static_assert(CIN == 3 || CIN == 4, "conv_in: 3 or 4 input channels");
    constexpr int KR = 3 * CIN;                          // inputs per filter row: 3 columns x CIN channels
    // patch[r][c][k]: r = 0..ROWS+1 input rows, c = 0..CI_W+1 input columns, k = 0..CIN-1 channels, padded to 4 floats per pixel
    __shared__ __align__(16) float patch[(CI_ROWS + 2) * (CI_W + 2) * 4];
    __shared__ float red[8][32][2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int x0 = blockIdx.x * CI_W, y0 = blockIdx.y * CI_ROWS, n = blockIdx.z;
    for (int i = threadIdx.x; i < (CI_ROWS + 2) * (CI_W + 2); i += 256) {
        const int r = i / (CI_W + 2), c = i - r * (CI_W + 2);
        const int iy = y0 + r - 1, ix = x0 + c - 1;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
            const float* px = x + (((int64_t)n * H + iy) * W + ix) * CIN;
            v.x = __ldg(px); v.y = __ldg(px + 1); v.z = __ldg(px + 2);
            if (CIN == 4) v.w = __ldg(px + 3);
        }
        *reinterpret_cast<float4*>(&patch[i * 4]) = v;
    }
    float4 wr[3 * KR];
#pragma unroll
    for (int k = 0; k < 3 * KR; ++k) wr[k] = __ldg(reinterpret_cast<const float4*>(w_kn + k * 128) + lane);
    const float4 b4 = bias ? __ldg(reinterpret_cast<const float4*>(bias) + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    float gs = 0.f, gq = 0.f;
    // warp w: row (w / 2) of the tile, pixels [(w & 1) * 32, +32), two pixels per iteration
    const int r = warp >> 1;
    const int yy = y0 + r;
    const int cbase = (warp & 1) * 32;
    if (yy < H) {
#pragma unroll 2
        for (int j = 0; j < 32; j += 2) {
            const int c = cbase + j;                      // tile column of the first pixel
            float4 a0 = b4, a1 = b4;
#pragma unroll
            for (int dy = 0; dy < 3; ++dy) {
                const float4* row = reinterpret_cast<const float4*>(&patch[((r + dy) * (CI_W + 2) + c) * 4]);
                const float4 p[4] = {row[0], row[1], row[2], row[3]};      // input columns c-1 .. c+2 (tile-relative + 1)
                float in0[KR], in1[KR];
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const float q0[4] = {p[dx].x, p[dx].y, p[dx].z, p[dx].w};
                    const float q1[4] = {p[dx + 1].x, p[dx + 1].y, p[dx + 1].z, p[dx + 1].w};
#pragma unroll
                    for (int ch = 0; ch < CIN; ++ch) {
                        in0[dx * CIN + ch] = q0[ch];
                        in1[dx * CIN + ch] = q1[ch];
                    }
                }
#pragma unroll
                for (int k = 0; k < KR; ++k) {
                    const float4 w4 = wr[dy * KR + k];
                    a0.x = fmaf(in0[k], w4.x, a0.x); a0.y = fmaf(in0[k], w4.y, a0.y); a0.z = fmaf(in0[k], w4.z, a0.z); a0.w = fmaf(in0[k], w4.w, a0.w);
                    a1.x = fmaf(in1[k], w4.x, a1.x); a1.y = fmaf(in1[k], w4.y, a1.y); a1.z = fmaf(in1[k], w4.z, a1.z); a1.w = fmaf(in1[k], w4.w, a1.w);
                }
            }
            const int xx = x0 + c;
            float* o = y + (((int64_t)n * H + yy) * W + xx) * 128 + lane * 4;
            // sums of squares contracted explicitly, so that every CIN instance rounds them alike
            if (xx < W) {
                *reinterpret_cast<float4*>(o) = a0;
                gs += (a0.x + a0.y) + (a0.z + a0.w);
                gq += fmaf(a0.x, a0.x, a0.y * a0.y) + fmaf(a0.z, a0.z, a0.w * a0.w);
            }
            if (xx + 1 < W) {
                *reinterpret_cast<float4*>(o + 128) = a1;
                gs += (a1.x + a1.y) + (a1.z + a1.w);
                gq += fmaf(a1.x, a1.x, a1.y * a1.y) + fmaf(a1.z, a1.z, a1.w * a1.w);
            }
        }
    }
    if (gn_sums) {      // lane = group: fold the 8 warps, then one RED per (group, statistic)
        red[warp][lane][0] = gs;
        red[warp][lane][1] = gq;
        __syncthreads();
        if (threadIdx.x < 64) {
            const int g = threadIdx.x >> 1, st = threadIdx.x & 1;
            float t = 0.f;
#pragma unroll
            for (int w8 = 0; w8 < 8; ++w8) t += red[w8][g][st];
            atomicAdd(gn_sums + ((int64_t)n * 32 + g) * 2 + st, (double)t);
        }
    }
}


// ------------------------------------------------------------------------------------------------
// Small Cout (<= 4), Cin == 128: one warp walks a run of pixels along x; lane l owns input channels 4l..4l+3 and keeps
// its 9 x 4 x COUT weights in registers; per pixel 9 coalesced 512-byte loads, COUT warp reductions.
// ------------------------------------------------------------------------------------------------
template <typename InT> __device__ __forceinline__ float4 ld4(const InT* p);
template <> __device__ __forceinline__ float4 ld4<float>(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
template <> __device__ __forceinline__ float4 ld4<__nv_bfloat16>(const __nv_bfloat16* p) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&u.x), b = *reinterpret_cast<const __nv_bfloat162*>(&u.y);
    const float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
    return make_float4(fa.x, fa.y, fb.x, fb.y);
}

// COUT = 3 or 4, Cin = 128 (conv_out of the released models): a warp walks a 32-pixel run of one row four pixels at a time.
// Lane l owns input channels 4l..4l+3; the 3 x 6 input float4 of the 4-pixel window are all requested before the first FMA;
// weights sit in shared memory as [tap][out][128] (conflict-free LDS.128); the 4 COUT partial sums (4 pixels x COUT outputs, in
// 16 slots) are folded across the warp with one butterfly that halves the value count every step (16 shuffles instead of 60) and
// land as 4 COUT consecutive floats of the output row.
template <int COUT, typename InT>
__global__ void __launch_bounds__(256) conv3x3_cout_kernel(const InT* __restrict__ x, const float* __restrict__ w_kn,
                                                           const float* __restrict__ bias, int N, int H, int W,
                                                           float* __restrict__ y) {
    static_assert(COUT == 3 || COUT == 4, "conv_out: 3 or 4 output channels");
    constexpr int CIN = 128;
    __shared__ __align__(16) float ws[9 * COUT * CIN];    // [(tap * COUT + o)][c]
    for (int i = threadIdx.x; i < 9 * COUT * CIN; i += 256) {
        const int to = i / CIN, c = i - to * CIN;
        const int t = to / COUT, o = to - t * COUT;
        ws[i] = __ldg(w_kn + (int64_t)(t * CIN + c) * COUT + o);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int runs_per_row = (W + 31) / 32;
    const int run = warp_global % runs_per_row;
    const int row = warp_global / runs_per_row;           // n*H + y
    if (row >= N * H) return;
    const int yy = row % H, n = row / H;
    const float b_lane = bias ? __ldg(bias + ((lane >> 1) % COUT)) : 0.f;   // lanes 2i, 2i+1 end up with value i = px*COUT + o
    const int x0 = run * 32, x1 = min(W, x0 + 32);
    for (int xx = x0; xx < x1; xx += 4) {
        float4 in[3][6];                                  // rows yy-1..yy+1, columns xx-1..xx+4
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const int iy = yy + dy - 1;
            const bool oky = iy >= 0 && iy < H;
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                const int ix = xx + c - 1;
                const bool ok = oky && ix >= 0 && ix < W;                   // warp-uniform
                // clamped address keeps all 18 loads unconditional and in flight together
                const int cy = oky ? iy : yy, cx = (ix >= 0 && ix < W) ? ix : xx;
                const float4 v = ld4<InT>(x + (((int64_t)n * H + cy) * W + cx) * CIN + lane * 4);
                in[dy][c] = ok ? v : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = 0.f;
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx)
#pragma unroll
                for (int o = 0; o < COUT; ++o) {
                    const float4 w4 = *reinterpret_cast<const float4*>(&ws[((dy * 3 + dx) * COUT + o) * CIN + lane * 4]);
#pragma unroll
                    for (int px = 0; px < 4; ++px) {
                        const float4 a = in[dy][px + dx];
                        float t = v[px * COUT + o];
                        t = fmaf(a.x, w4.x, t); t = fmaf(a.y, w4.y, t); t = fmaf(a.z, w4.z, t); t = fmaf(a.w, w4.w, t);
                        v[px * COUT + o] = t;
                    }
                }
        // butterfly: after the step with offset `off` a lane keeps the half of the values selected by its bit `off`
#pragma unroll
        for (int half = 8, off = 16; half >= 1; half >>= 1, off >>= 1) {
            const bool upper = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < half; ++i) {
                const float send = upper ? v[i] : v[i + half];
                const float keep = upper ? v[i + half] : v[i];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
        }
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
        const int idx = lane >> 1;                        // = px * COUT + o
        if ((lane & 1) == 0 && idx < 4 * COUT && xx + idx / COUT < x1)
            y[(((int64_t)n * H + yy) * W + xx) * COUT + idx] = v[0] + b_lane;
    }
}

}  // namespace

extern "C" int vf_conv3x3_small_cin(const float* x, const float* w_kn, const float* bias, int N, int H, int W, int Cin, int Cout,
                                    float* y, double* gn_sums, vf_stream_t s) {
    VF_CHECK_ARG(x && w_kn && y, "vf_conv3x3_small_cin: null pointer");
    VF_CHECK_ARG((Cin == 3 || Cin == 4) && Cout % 16 == 0 && Cout <= 128,
                 "vf_conv3x3_small_cin: supports Cin = 3 or 4, Cout%%16==0, Cout<=128 (got %d->%d)", Cin, Cout);
    VF_CHECK_ARG(!gn_sums || Cout == 128, "vf_conv3x3_small_cin: fused GroupNorm(32) statistics need Cout = 128");
    if (N == 0) return VF_OK;
    VF_CHECK_ARG(H <= 65535 * CI_ROWS && N <= 65535, "vf_conv3x3_small_cin: grid too large");
    if (Cout == 128) {
        if (gn_sums) {
            cudaError_t e = cudaMemsetAsync(gn_sums, 0, sizeof(double) * 2 * 32 * N, vf_s(s));
            if (e != cudaSuccess) { vf_set_error("vf_conv3x3_small_cin: memset: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
        }
        dim3 grid((W + CI_W - 1) / CI_W, (H + CI_ROWS - 1) / CI_ROWS, N);
        if (Cin == 3)
            conv3x3_cin_cout128_kernel<3><<<grid, 256, 0, vf_s(s)>>>(x, w_kn, bias, N, H, W, y, gn_sums);
        else
            conv3x3_cin_cout128_kernel<4><<<grid, 256, 0, vf_s(s)>>>(x, w_kn, bias, N, H, W, y, gn_sums);
        VF_CHECK_LAUNCH("vf_conv3x3_small_cin");
        return VF_OK;
    }
    dim3 grid((W + 63) / 64, H, N);
    VF_CHECK_ARG(H <= 65535, "vf_conv3x3_small_cin: grid too large");
    if (Cin == 3)
        conv3x3_small_cin_kernel<3, InputF32, false><<<grid, 32 * (Cout / 16), sizeof(float) * 27 * Cout, vf_s(s)>>>(InputF32{x}, w_kn, bias, N, H, W, Cout, y);
    else
        conv3x3_small_cin_kernel<4, InputF32, false><<<grid, 32 * (Cout / 16), sizeof(float) * 36 * Cout, vf_s(s)>>>(InputF32{x}, w_kn, bias, N, H, W, Cout, y);
    VF_CHECK_LAUNCH("vf_conv3x3_small_cin");
    return VF_OK;
}

extern "C" int vf_lpips_conv_in(const uint8_t* x, const float* shift, const float* scale, const float* w_kn, const float* bias, int N, int H,
                                int W, int Cout, float* y, vf_stream_t s) {
    VF_CHECK_ARG(x && shift && scale && w_kn && bias && y, "vf_lpips_conv_in: null pointer");
    VF_CHECK_ARG(Cout % 16 == 0 && Cout > 0 && Cout <= 128, "vf_lpips_conv_in: Cout %% 16 == 0, Cout <= 128 (got %d)", Cout);
    VF_CHECK_ARG(N >= 0 && N <= 65535 && H >= 0 && H <= 65535 && W >= 0, "vf_lpips_conv_in: shape out of range");
    if (N == 0 || H == 0 || W == 0) return VF_OK;
    dim3 grid((W + 63) / 64, H, N);
    conv3x3_small_cin_kernel<3, InputU8Scaled, true><<<grid, 32 * (Cout / 16), sizeof(float) * 27 * Cout, vf_s(s)>>>(
        InputU8Scaled{x, shift, scale}, w_kn, bias, N, H, W, Cout, y);
    VF_CHECK_LAUNCH("vf_lpips_conv_in");
    return VF_OK;
}

extern "C" int vf_conv3x3_small_cout(const void* x, int x_dtype, const float* w_kn, const float* bias, int N, int H, int W, int Cin,
                                     int Cout, float* y, vf_stream_t s) {
    VF_CHECK_ARG(x && w_kn && y, "vf_conv3x3_small_cout: null pointer");
    VF_CHECK_ARG(Cin == 128 && (Cout == 3 || Cout == 4), "vf_conv3x3_small_cout: supports 128->3 and 128->4 (got %d->%d)", Cin, Cout);
    VF_CHECK_ARG(x_dtype == VF_F32 || x_dtype == VF_BF16, "vf_conv3x3_small_cout: x must be fp32 or bf16");
    if (N == 0) return VF_OK;
    const long long warps = (long long)N * H * ((W + 31) / 32);
    VF_CHECK_ARG(warps < (1ll << 31), "vf_conv3x3_small_cout: too many pixels");
    const unsigned blocks = (unsigned)((warps + 7) / 8);
    if (Cout == 3 && x_dtype == VF_F32)
        conv3x3_cout_kernel<3, float><<<blocks, 256, 0, vf_s(s)>>>((const float*)x, w_kn, bias, N, H, W, y);
    else if (Cout == 3)
        conv3x3_cout_kernel<3, __nv_bfloat16><<<blocks, 256, 0, vf_s(s)>>>((const __nv_bfloat16*)x, w_kn, bias, N, H, W, y);
    else if (x_dtype == VF_F32)
        conv3x3_cout_kernel<4, float><<<blocks, 256, 0, vf_s(s)>>>((const float*)x, w_kn, bias, N, H, W, y);
    else
        conv3x3_cout_kernel<4, __nv_bfloat16><<<blocks, 256, 0, vf_s(s)>>>((const __nv_bfloat16*)x, w_kn, bias, N, H, W, y);
    VF_CHECK_LAUNCH("vf_conv3x3_small_cout");
    return VF_OK;
}
