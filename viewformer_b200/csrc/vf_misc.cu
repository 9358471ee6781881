// Small HBM-bound kernels: pixel conversion, layout permutes, transformer glue
// (embedding sum, row softmax with block-causal masks, argmax, pose post-processing), casts, loss sums.
#include "vf_common.cuh"
#include "../../include/vf_b200_pose.h"
#include <stdarg.h>

// ------------------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
void vf_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char* vf_last_error(void) { return g_err; }
extern "C" int vf_version(void) { return 100; }
extern "C" int vf_sizeof_simt_gemm(void) { return (int)sizeof(vf_simt_gemm_t); }
extern "C" int vf_sizeof_tc_gemm(void) { return (int)sizeof(vf_tc_gemm_t); }
extern "C" int vf_device_check(void) {
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
        vf_set_error("vf_device_check: no CUDA device");
        return VF_ERR_CUDA;
    }
    if (prop.major != 9 || prop.minor != 0) {
        vf_set_error("vf_device_check: device %s is sm_%d%d, this library is built for sm_90a only", prop.name, prop.major,
                     prop.minor);
        return VF_ERR_UNSUPPORTED;
    }
    return VF_OK;
}

namespace {

// ------------------------------------------------------------------------------------------ pixels
__global__ void u8_to_unit_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int64_t n, int64_t in_row_stride) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    in += (int64_t)blockIdx.y * in_row_stride;
    out += (int64_t)blockIdx.y * n;
    const float k = 1.0f / 255.0f;   // tf.image.convert_image_dtype: multiply by float32(1/255)
    if (i + 3 < n && ((reinterpret_cast<uintptr_t>(in + i) & 3) == 0)) {
        const uchar4 v = *reinterpret_cast<const uchar4*>(in + i);
        // explicit mul then mul/sub, no contraction, to match (x * k) * 2 - 1 evaluated op by op
        float4 o;
        o.x = __fsub_rn(__fmul_rn(__fmul_rn((float)v.x, k), 2.0f), 1.0f);
        o.y = __fsub_rn(__fmul_rn(__fmul_rn((float)v.y, k), 2.0f), 1.0f);
        o.z = __fsub_rn(__fmul_rn(__fmul_rn((float)v.z, k), 2.0f), 1.0f);
        o.w = __fsub_rn(__fmul_rn(__fmul_rn((float)v.w, k), 2.0f), 1.0f);
        *reinterpret_cast<float4*>(out + i) = o;
    } else {
        for (int64_t j = i; j < n && j < i + 4; ++j)
            out[j] = __fsub_rn(__fmul_rn(__fmul_rn((float)in[j], k), 2.0f), 1.0f);
    }
}

// f32 images in [0, 1] -> x * 2 - 1 (convert_image_dtype is the identity for float32 input), op by op
__global__ void f01_to_unit_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t n, int64_t in_row_stride) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[(int64_t)blockIdx.y * n + i] = __fsub_rn(__fmul_rn(__ldg(in + (int64_t)blockIdx.y * in_row_stride + i), 2.0f), 1.0f);
}

__global__ void unit_to_u8_kernel(const float* __restrict__ in, uint8_t* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = fminf(fmaxf(in[i], -1.0f), 1.0f);
    v = __fadd_rn(__fmul_rn(v, 0.5f), 0.5f);          // x / 2 + 0.5
    v = __fmul_rn(v, 255.5f);                         // convert_image_dtype(float -> uint8): scale = max + 0.5
    v = fminf(fmaxf(v, 0.0f), 255.0f);                // saturate_cast
    out[i] = (uint8_t)v;                              // truncation
}

// NCHW -> NHWC: thread per (n, pixel); reads C planes (coalesced per plane), writes C contiguous values.
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int64_t HW, int64_t total) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // n*HW + p
    if (i >= total) return;
    const int64_t n = i / HW, p = i % HW;
    const float* src = in + n * C * HW + p;
    float* dst = out + i * C;
    for (int c = 0; c < C; ++c) dst[c] = __ldg(src + (int64_t)c * HW);
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int64_t HW, int64_t total) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // n*HW + p
    if (i >= total) return;
    const int64_t n = i / HW, p = i % HW;
    const float* src = in + i * C;
    float* dst = out + n * C * HW + p;
    for (int c = 0; c < C; ++c) dst[(int64_t)c * HW] = __ldg(src + c);
}

// ------------------------------------------------------------------------------------------ transformer glue
// one thread per float4 of the output
__global__ void migt_embed_kernel(const int32_t* __restrict__ ids, int fixed_token, const float* __restrict__ wte,
                                  const float* __restrict__ wpe, const float* __restrict__ pose, int64_t BT, int L, int d,
                                  float* __restrict__ out) {
    const int quads = d >> 2;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= BT * L * quads) return;
    const int q = (int)(i % quads);
    const int64_t tok = i / quads;           // bt*L + l
    const int l = (int)(tok % L);
    const int64_t bt = tok / L;
    int id = ids ? ids[tok] : -1;
    if (id < 0) id = fixed_token;
    const float4 a = __ldg(reinterpret_cast<const float4*>(wte + (int64_t)id * d) + q);
    const float4 b = __ldg(reinterpret_cast<const float4*>(wpe + (int64_t)l * d) + q);
    const float4 c = __ldg(reinterpret_cast<const float4*>(pose + bt * d) + q);
    // reference: sum((inputs_embeds, position_embeds, pose_embeddings)) == (0 + a) + b) + c
    float4 o;
    o.x = (a.x + b.x) + c.x; o.y = (a.y + b.y) + c.y; o.z = (a.z + b.z) + c.z; o.w = (a.w + b.w) + c.w;
    reinterpret_cast<float4*>(out)[i] = o;
}

template <typename OutT> __device__ __forceinline__ void st1(OutT* p, float v);
template <> __device__ __forceinline__ void st1<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st1<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }

// one warp per row
template <typename OutT>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ scores, int64_t rows_total,
                                                           int rows_per_batch, int cols, int64_t ld_in, int mask_mode,
                                                           int block, int row0, OutT* __restrict__ P, int64_t ld_out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + warp;
    if (row >= rows_total) return;
    const int r = (int)(row % rows_per_batch) + row0;        // position of the query token in its sequence
    const float* src = scores + row * ld_in;
    OutT* dst = P + row * ld_out;
    const int view = block > 0 ? r / block : 0;
    // keep(c): is column c visible?
    int lim0 = cols, lo1 = 0, hi1 = 0;    // visible: [0,lim0) U [lo1,hi1)
    if (mask_mode == 1) {
        lim0 = min(cols, (view + 1) * block);
    } else if (mask_mode == 2) {
        const int half = cols / 2;
        lim0 = min(half, view * block);
        lo1 = half + view * block;
        hi1 = min(cols, lo1 + block);
    }
    float mx = -INFINITY;
    for (int c = lane; c < lim0; c += 32) mx = fmaxf(mx, src[c]);
    for (int c = lo1 + lane; c < hi1; c += 32) mx = fmaxf(mx, src[c]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int c = lane; c < lim0; c += 32) sum += expf(src[c] - mx);
    for (int c = lo1 + lane; c < hi1; c += 32) sum += expf(src[c] - mx);
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
    for (int c = lane; c < cols; c += 32) {
        const bool keep = (c < lim0) || (c >= lo1 && c < hi1);
        st1<OutT>(dst + c, keep ? expf(src[c] - mx) * inv : 0.0f);
    }
}

__global__ void __launch_bounds__(256) argmax_rows_kernel(const float* __restrict__ x, int64_t rows, int cols, int64_t ld,
                                                          int64_t* __restrict__ out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const float* src = x + row * ld;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < cols; c += 32) {
        const float v = src[c];
        if (v > best || (v == best && c < bi)) { best = v; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) out[row] = (bi == 0x7fffffff) ? 0 : bi;
}

__global__ void pose_post_kernel(const float* __restrict__ raw, int64_t rows, float mult, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const float* r = raw + i * 7;
    float* o = out + i * 7;
    o[0] = r[0] / mult; o[1] = r[1] / mult; o[2] = r[2] / mult;
    const float w = r[3], x = r[4], y = r[5], z = r[6];
    const float n2 = fmaxf(((w * w + x * x) + y * y) + z * z, 1e-12f);
    const float inv = rsqrtf(n2);
    float qw = w * inv, qx = x * inv, qy = y * inv, qz = z * inv;
    const float sg = (qw >= 0.f) ? 1.f : -1.f;
    o[3] = qw * sg; o[4] = qx * sg; o[5] = qy * sg; o[6] = qz * sg;
}

// quaternion helpers, (w,x,y,z) order — viewformer/utils/geometry_tf.py:6-13, 53-91
struct Quat { float w, x, y, z; };
__device__ __forceinline__ Quat qmul(Quat a, Quat b) {
    Quat r;
    r.x = a.x * b.w + a.y * b.z - a.z * b.y + a.w * b.x;
    r.y = -a.x * b.z + a.y * b.w + a.z * b.x + a.w * b.y;
    r.z = a.x * b.y - a.y * b.x + a.z * b.w + a.w * b.z;
    r.w = -a.x * b.x - a.y * b.y - a.z * b.z + a.w * b.w;
    return r;
}
__global__ void cameras_prepare_kernel(const float* __restrict__ cams, int B, int T, int relative, float* __restrict__ out,
                                       float* __restrict__ transform) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * T) return;
    const int b = i / T, t = i % T;
    const float* c = cams + (int64_t)i * 7;
    const float* c0 = cams + (int64_t)b * T * 7;
    float px = c[0], py = c[1], pz = c[2];
    Quat q = {c[3], c[4], c[5], c[6]};
    if (relative) {
        const Quat inv = {c0[3], -c0[4], -c0[5], -c0[6]};          // conjugate of view 0's rotation
        const Quat p = {0.f, px - c0[0], py - c0[1], pz - c0[2]};
        const Quat conj_inv = {inv.w, -inv.x, -inv.y, -inv.z};
        const Quat r = qmul(qmul(inv, p), conj_inv);               // quaternion_rotate(xyz - t, inv)
        px = r.x; py = r.y; pz = r.z;
        q = qmul(inv, q);
        if (t == 0 && transform) {
            float* tr = transform + (int64_t)b * 7;
            for (int j = 0; j < 7; ++j) tr[j] = c0[j];
        }
    }
    const float n2 = fmaxf(((q.w * q.w + q.x * q.x) + q.y * q.y) + q.z * q.z, 1e-12f);
    const float inv_n = rsqrtf(n2);
    q.w *= inv_n; q.x *= inv_n; q.y *= inv_n; q.z *= inv_n;
    const float sg = (q.w >= 0.f) ? 1.f : -1.f;
    float* o = out + (int64_t)i * 7;
    o[0] = px; o[1] = py; o[2] = pz; o[3] = q.w * sg; o[4] = q.x * sg; o[5] = q.y * sg; o[6] = q.z * sg;
}

__global__ void cameras_from_relative_kernel(const float* __restrict__ cams, const float* __restrict__ transform, int B, int n,
                                             float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * n) return;
    const float* c = cams + (int64_t)i * 7;
    const float* t = transform + (int64_t)(i / n) * 7;
    const Quat tq = {t[3], t[4], t[5], t[6]};
    const Quat q = qmul(tq, Quat{c[3], c[4], c[5], c[6]});
    const Quat p = {0.f, c[0], c[1], c[2]};
    const Quat r = qmul(qmul(tq, p), Quat{tq.w, -tq.x, -tq.y, -tq.z});
    float* o = out + (int64_t)i * 7;
    o[0] = r.x + t[0]; o[1] = r.y + t[1]; o[2] = r.z + t[2];
    o[3] = q.w; o[4] = q.x; o[5] = q.y; o[6] = q.z;
}

// nearest cameras (evaluate_sevenscenes.py:36-45, 187-189; evaluate_sevenscenes_baseline.py:43-51, 93): one CTA per query.  Each
// database camera becomes a 64-bit key (order-preserving bits of its fp32 distance | its index), so keys are unique and ascending key
// order is ascending distance with ties to the lower index; k rounds of a block-wide min over the keys above the last one picked.
// The first KNN_CACHE keys are kept in shared memory; a larger database recomputes the rest each round.
constexpr int KNN_THREADS = 256;
constexpr int KNN_CACHE = 8192;                    // 64 KB of keys: a 7-Scenes training split (1 000 - 7 000 frames) fits whole

__device__ __forceinline__ Quat qnormalize(Quat q) {   // l2_normalize(axis=-1, epsilon=1e-12), geometry_tf.py:44-45
    const float r = rsqrtf(fmaxf(((q.w * q.w + q.x * q.x) + q.y * q.y) + q.z * q.z, 1e-12f));
    return Quat{q.w * r, q.x * r, q.y * r, q.z * r};
}

__device__ __forceinline__ unsigned long long knn_key(const float* __restrict__ c, float px, float py, float pz, Quat qconj, int mode,
                                                      uint32_t i) {
    float d = 0.f;
    if (mode != 2) {
        const float dx = c[0] - px, dy = c[1] - py, dz = c[2] - pz;
        d = sqrtf((dx * dx + dy * dy) + dz * dz);
        if (mode == 0) d = __fmul_rn(d, 0.3f);     // pos * 0.3, rounded before the sum as the reference rounds it
    }
    if (mode != 1) {
        const Quat r = qmul(qnormalize(Quat{c[3], c[4], c[5], c[6]}), qconj);
        d = __fadd_rn(d, 2.f * asinf(fminf(sqrtf((r.x * r.x + r.y * r.y) + r.z * r.z), 1.f)));
    }
    uint32_t u = __float_as_uint(d);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((unsigned long long)u << 32) | i;
}

__global__ void __launch_bounds__(KNN_THREADS) camera_knn_kernel(const float* __restrict__ db, int64_t N, int64_t db_stride,
                                                                 const float* __restrict__ queries, int mode, int k, int ncache,
                                                                 int32_t* __restrict__ idx_out, float* __restrict__ dist_out) {
    extern __shared__ unsigned long long keys[];
    __shared__ unsigned long long warp_min[KNN_THREADS / 32];
    __shared__ unsigned long long picked;
    const int64_t qi = blockIdx.x;
    const float* q = queries + qi * 7;
    const float* base = db + qi * db_stride;
    const float px = q[0], py = q[1], pz = q[2];
    const Quat qn = qnormalize(Quat{q[3], q[4], q[5], q[6]});
    const Quat qconj = {qn.w, -qn.x, -qn.y, -qn.z};
    for (int i = threadIdx.x; i < ncache; i += KNN_THREADS) keys[i] = knn_key(base + (int64_t)i * 7, px, py, pz, qconj, mode, (uint32_t)i);
    __syncthreads();
    unsigned long long lo = 0;                     // keys are unique: round r takes the least key >= (round r-1's key) + 1
    for (int r = 0; r < k; ++r) {
        unsigned long long best = ~0ull;
        for (int64_t i = threadIdx.x; i < N; i += KNN_THREADS) {
            const unsigned long long key = i < ncache ? keys[i] : knn_key(base + i * 7, px, py, pz, qconj, mode, (uint32_t)i);
            if (key >= lo && key < best) best = key;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
            best = other < best ? other : best;
        }
        if ((threadIdx.x & 31) == 0) warp_min[threadIdx.x >> 5] = best;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long b = warp_min[0];
            for (int w = 1; w < KNN_THREADS / 32; ++w) b = warp_min[w] < b ? warp_min[w] : b;
            uint32_t u = (uint32_t)(b >> 32);
            u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
            idx_out[qi * k + r] = (int32_t)(uint32_t)b;
            dist_out[qi * k + r] = __uint_as_float(u);
            picked = b;
        }
        __syncthreads();
        lo = picked + 1;
    }
}

// sparse softmax cross-entropy per row (tf.nn.sparse_softmax_cross_entropy_with_logits, models/migt.py:99-104,419-423);
// label smoothing s: loss = (1-s) * nll + s * (lse - mean(logits)).  One warp per row.
__global__ void __launch_bounds__(256) ce_rows_kernel(const float* __restrict__ logits, const int32_t* __restrict__ labels,
                                                      int64_t rows, int cols, float smoothing, float* __restrict__ out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const float* x = logits + row * cols;
    float mx = -INFINITY;
    for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, x[c]);
    mx = warp_max(mx);
    float se = 0.f, sx = 0.f;
    for (int c = lane; c < cols; c += 32) { se += expf(x[c] - mx); sx += x[c]; }
    se = warp_sum(se);
    sx = warp_sum(sx);
    if (lane == 0) {
        const float lse = mx + logf(se);
        const float nll = lse - x[labels[row]];
        out[row] = (1.0f - smoothing) * nll + smoothing * (lse - sx / (float)cols);
    }
}

// pose regression losses per token (models/migt.py:158-171): raw [rows,7] MLP output, target pose of the token's view
// (poses [BT,7], tokens_per_view consecutive rows share a view) scaled by [m,m,m,1,1,1,1]; pos = mean_3 (y-xyz/c)^2, ori = mean_4 (y-q)^2
// with c = scene_mult[view / views_per_scene] (the training-time pose scale of the view's scene), or 1 when scene_mult is null
__global__ void pose_loss_kernel(const float* __restrict__ raw, const float* __restrict__ poses, int64_t rows, int tokens_per_view,
                                 float mult, int views_per_scene, const float* __restrict__ scene_mult, float* __restrict__ pos_out,
                                 float* __restrict__ ori_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const float* r = raw + i * 7;
    const int64_t view = i / tokens_per_view;
    const float* y = poses + view * 7;
    const float c = scene_mult ? scene_mult[view / views_per_scene] : 1.0f;      // x / 1 == x: the unscaled path keeps its bits
    float p = 0.f, o = 0.f;
#pragma unroll
    for (int j = 0; j < 3; ++j) { const float d = y[j] * mult - r[j] / c; p += d * d; }
#pragma unroll
    for (int j = 3; j < 7; ++j) { const float d = y[j] - r[j]; o += d * d; }
    pos_out[i] = p / 3.0f;
    ori_out[i] = o / 4.0f;
}

// get_model_input (models/migt.py:139-145): out [rows,7] = [(xyz * mult) * c | quaternion] of poses [rows,7], rounded after each product
// as the reference does, c = scene_mult[row / views_per_scene] (omitted when scene_mult is null)
__global__ void pose_model_input_kernel(const float* __restrict__ poses, int64_t rows, int views_per_scene, float mult,
                                        const float* __restrict__ scene_mult, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * 7) return;
    const int64_t row = i / 7;
    float v = poses[i];
    if (i - row * 7 < 3) {
        v = v * mult;
        if (scene_mult) v = v * scene_mult[row / views_per_scene];
    }
    out[i] = v;
}

// out[b] = mean(x[b, start:n])  — one block per b
__global__ void __launch_bounds__(256) row_mean_kernel(const float* __restrict__ x, int n, int start, float* __restrict__ out) {
    __shared__ float sh[8];
    const float* xr = x + (int64_t)blockIdx.x * n;
    float s = 0.f;
    for (int i = start + threadIdx.x; i < n; i += 256) s += xr[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += sh[w];
        out[blockIdx.x] = t / (float)(n - start);
    }
}


}  // namespace

static inline unsigned nblk(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

extern "C" int vf_u8_to_unit_f32(const uint8_t* in, float* out, int64_t rows, int64_t row_len, int64_t in_row_stride,
                                 vf_stream_t s) {
    VF_CHECK_ARG(in && out && rows >= 0 && row_len >= 0 && rows <= 65535, "vf_u8_to_unit_f32: bad args");
    if (rows == 0 || row_len == 0) return VF_OK;
    dim3 grid(nblk(row_len, 1024), (unsigned)rows);
    u8_to_unit_kernel<<<grid, 256, 0, vf_s(s)>>>(in, out, row_len, in_row_stride);
    VF_CHECK_LAUNCH("vf_u8_to_unit_f32");
    return VF_OK;
}
extern "C" int vf_f01_to_unit_f32(const float* in, float* out, int64_t rows, int64_t row_len, int64_t in_row_stride, vf_stream_t s) {
    VF_CHECK_ARG(in && out && rows >= 0 && row_len >= 0 && rows <= 65535, "vf_f01_to_unit_f32: bad args");
    if (rows == 0 || row_len == 0) return VF_OK;
    dim3 grid(nblk(row_len, 256), (unsigned)rows);
    f01_to_unit_kernel<<<grid, 256, 0, vf_s(s)>>>(in, out, row_len, in_row_stride);
    VF_CHECK_LAUNCH("vf_f01_to_unit_f32");
    return VF_OK;
}
extern "C" int vf_unit_f32_to_u8(const float* in, uint8_t* out, int64_t n, vf_stream_t s) {
    VF_CHECK_ARG(in && out && n >= 0, "vf_unit_f32_to_u8: bad args");
    if (n == 0) return VF_OK;
    unit_to_u8_kernel<<<nblk(n, 256), 256, 0, vf_s(s)>>>(in, out, n);
    VF_CHECK_LAUNCH("vf_unit_f32_to_u8");
    return VF_OK;
}
extern "C" int vf_nchw_to_nhwc_f32(const float* in, float* out, int N, int C, int H, int W, vf_stream_t s) {
    VF_CHECK_ARG(in && out, "vf_nchw_to_nhwc_f32: null");
    const int64_t total = (int64_t)N * H * W;
    if (total == 0) return VF_OK;
    nchw_to_nhwc_kernel<<<nblk(total, 256), 256, 0, vf_s(s)>>>(in, out, C, (int64_t)H * W, total);
    VF_CHECK_LAUNCH("vf_nchw_to_nhwc_f32");
    return VF_OK;
}
extern "C" int vf_nhwc_to_nchw_f32(const float* in, float* out, int N, int C, int H, int W, vf_stream_t s) {
    VF_CHECK_ARG(in && out, "vf_nhwc_to_nchw_f32: null");
    const int64_t total = (int64_t)N * H * W;
    if (total == 0) return VF_OK;
    nhwc_to_nchw_kernel<<<nblk(total, 256), 256, 0, vf_s(s)>>>(in, out, C, (int64_t)H * W, total);
    VF_CHECK_LAUNCH("vf_nhwc_to_nchw_f32");
    return VF_OK;
}
extern "C" int vf_migt_embed(const int32_t* ids, int fixed_token, const float* wte, const float* wpe, const float* pose,
                             int64_t BT, int L, int d, float* out, vf_stream_t s) {
    VF_CHECK_ARG(wte && wpe && pose && out, "vf_migt_embed: null");
    VF_CHECK_ARG(d % 4 == 0, "vf_migt_embed: d %% 4");
    const int64_t total = BT * L * (d / 4);
    if (total == 0) return VF_OK;
    migt_embed_kernel<<<nblk(total, 256), 256, 0, vf_s(s)>>>(ids, fixed_token, wte, wpe, pose, BT, L, d, out);
    VF_CHECK_LAUNCH("vf_migt_embed");
    return VF_OK;
}
extern "C" int vf_softmax_rows(const float* scores, int64_t rows_total, int rows_per_batch, int cols, int64_t ld_in,
                               int mask_mode, int block, int row0, void* P, int p_dtype, int64_t ld_out, vf_stream_t s) {
    VF_CHECK_ARG(scores && P && rows_per_batch > 0 && cols > 0, "vf_softmax_rows: bad args");
    VF_CHECK_ARG(mask_mode == 0 || block > 0, "vf_softmax_rows: mask needs block");
    if (rows_total == 0) return VF_OK;
    if (p_dtype == VF_F32)
        softmax_rows_kernel<float><<<nblk(rows_total, 8), 256, 0, vf_s(s)>>>(scores, rows_total, rows_per_batch, cols, ld_in,
                                                                            mask_mode, block, row0, (float*)P, ld_out);
    else
        softmax_rows_kernel<__nv_bfloat16><<<nblk(rows_total, 8), 256, 0, vf_s(s)>>>(
            scores, rows_total, rows_per_batch, cols, ld_in, mask_mode, block, row0, (__nv_bfloat16*)P, ld_out);
    VF_CHECK_LAUNCH("vf_softmax_rows");
    return VF_OK;
}
extern "C" int vf_argmax_rows(const float* x, int64_t rows, int cols, int64_t ld, int64_t* out, vf_stream_t s) {
    VF_CHECK_ARG(x && out && cols > 0, "vf_argmax_rows: bad args");
    if (rows == 0) return VF_OK;
    argmax_rows_kernel<<<nblk(rows, 8), 256, 0, vf_s(s)>>>(x, rows, cols, ld, out);
    VF_CHECK_LAUNCH("vf_argmax_rows");
    return VF_OK;
}
extern "C" int vf_pose_postprocess(const float* raw, int64_t rows, float pose_multiplier, float* out, vf_stream_t s) {
    VF_CHECK_ARG(raw && out, "vf_pose_postprocess: null");
    if (rows == 0) return VF_OK;
    pose_post_kernel<<<nblk(rows, 256), 256, 0, vf_s(s)>>>(raw, rows, pose_multiplier, out);
    VF_CHECK_LAUNCH("vf_pose_postprocess");
    return VF_OK;
}
extern "C" int vf_cameras_prepare(const float* cams, int B, int T, int relative, float* out, float* transform, vf_stream_t s) {
    VF_CHECK_ARG(cams && out && B >= 0 && T > 0, "vf_cameras_prepare: bad args");
    if (B == 0) return VF_OK;
    cameras_prepare_kernel<<<(B * T + 127) / 128, 128, 0, vf_s(s)>>>(cams, B, T, relative, out, transform);
    VF_CHECK_LAUNCH("vf_cameras_prepare");
    return VF_OK;
}
extern "C" int vf_cameras_from_relative(const float* cams, const float* transform, int B, int n, float* out, vf_stream_t s) {
    VF_CHECK_ARG(cams && transform && out && B >= 0 && n > 0, "vf_cameras_from_relative: bad args");
    if (B == 0) return VF_OK;
    cameras_from_relative_kernel<<<(B * n + 127) / 128, 128, 0, vf_s(s)>>>(cams, transform, B, n, out);
    VF_CHECK_LAUNCH("vf_cameras_from_relative");
    return VF_OK;
}
extern "C" int vf_camera_knn(const float* db, int64_t N, int64_t db_stride, const float* queries, int Q, int mode, int k, int32_t* idx_out,
                             float* dist_out, vf_stream_t s) {
    VF_CHECK_ARG(db && queries && idx_out && dist_out, "vf_camera_knn: null");
    VF_CHECK_ARG(Q >= 0 && N >= 1 && N < (1ll << 31) && db_stride >= 0, "vf_camera_knn: bad sizes (N %lld, Q %d)", (long long)N, Q);
    VF_CHECK_ARG(mode >= 0 && mode <= 2, "vf_camera_knn: mode %d (0 combined, 1 position, 2 orientation)", mode);
    VF_CHECK_ARG(k >= 1 && k <= 64 && k <= N, "vf_camera_knn: k %d outside [1, min(64, N = %lld)]", k, (long long)N);
    VF_CHECK_ARG(db_stride == 0 || db_stride >= N * 7, "vf_camera_knn: db_stride %lld overlaps the %lld cameras of a query",
                 (long long)db_stride, (long long)N);
    if (Q == 0) return VF_OK;
    static vf_per_device_flag flag;
    bool& configured = flag.current();
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(camera_knn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, KNN_CACHE * 8);
        if (e != cudaSuccess) { vf_set_error("vf_camera_knn: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
        configured = true;
    }
    const int ncache = (int)(N < KNN_CACHE ? N : KNN_CACHE);
    camera_knn_kernel<<<(unsigned)Q, KNN_THREADS, (size_t)ncache * 8, vf_s(s)>>>(db, N, db_stride, queries, mode, k, ncache, idx_out, dist_out);
    VF_CHECK_LAUNCH("vf_camera_knn");
    return VF_OK;
}
extern "C" int vf_cross_entropy_rows(const float* logits, const int32_t* labels, int64_t rows, int cols, float smoothing, float* out,
                                     vf_stream_t s) {
    VF_CHECK_ARG(logits && labels && out && cols > 0, "vf_cross_entropy_rows: bad args");
    if (rows == 0) return VF_OK;
    ce_rows_kernel<<<nblk(rows, 8), 256, 0, vf_s(s)>>>(logits, labels, rows, cols, smoothing, out);
    VF_CHECK_LAUNCH("vf_cross_entropy_rows");
    return VF_OK;
}
extern "C" int vf_pose_loss_rows(const float* raw, const float* poses, int64_t rows, int tokens_per_view, float pose_multiplier,
                                 float* pos_out, float* ori_out, vf_stream_t s) {
    VF_CHECK_ARG(raw && poses && pos_out && ori_out && tokens_per_view > 0, "vf_pose_loss_rows: bad args");
    if (rows == 0) return VF_OK;
    pose_loss_kernel<<<nblk(rows, 256), 256, 0, vf_s(s)>>>(raw, poses, rows, tokens_per_view, pose_multiplier, 1, nullptr, pos_out, ori_out);
    VF_CHECK_LAUNCH("vf_pose_loss_rows");
    return VF_OK;
}
extern "C" int vf_pose_loss_rows_scaled(const float* raw, const float* poses, int64_t rows, int tokens_per_view, float pose_multiplier,
                                        int views_per_scene, const float* scene_mult, float* pos_out, float* ori_out, vf_stream_t s) {
    VF_CHECK_ARG(raw && poses && pos_out && ori_out && tokens_per_view > 0 && views_per_scene > 0, "vf_pose_loss_rows_scaled: bad args");
    if (rows == 0) return VF_OK;
    pose_loss_kernel<<<nblk(rows, 256), 256, 0, vf_s(s)>>>(raw, poses, rows, tokens_per_view, pose_multiplier, views_per_scene, scene_mult,
                                                          pos_out, ori_out);
    VF_CHECK_LAUNCH("vf_pose_loss_rows_scaled");
    return VF_OK;
}
extern "C" int vf_pose_model_input(const float* poses, int64_t rows, int views_per_scene, float pose_multiplier, const float* scene_mult,
                                   float* out, vf_stream_t s) {
    VF_CHECK_ARG(poses && out && rows >= 0 && views_per_scene > 0, "vf_pose_model_input: bad args");
    if (rows == 0) return VF_OK;
    pose_model_input_kernel<<<nblk(rows * 7, 256), 256, 0, vf_s(s)>>>(poses, rows, views_per_scene, pose_multiplier, scene_mult, out);
    VF_CHECK_LAUNCH("vf_pose_model_input");
    return VF_OK;
}
extern "C" int vf_row_mean(const float* x, int64_t rows, int n, int start, float* out, vf_stream_t s) {
    VF_CHECK_ARG(x && out && n > start && start >= 0, "vf_row_mean: bad args");
    if (rows == 0) return VF_OK;
    row_mean_kernel<<<(unsigned)rows, 256, 0, vf_s(s)>>>(x, n, start, out);
    VF_CHECK_LAUNCH("vf_row_mean");
    return VF_OK;
}
