// Codebook kernels: exact fp32 L2 nearest-neighbour lookup (+gather, +commit-loss sum), embed_code gather,
// QuantizeEMA training statistics and EMA update.   Reference: viewformer/models/utils_th.py:32-72.
#include "vf_common.cuh"

namespace {

constexpr int LM = 64, LN = 64, LK = 16, LPAD = 4;

// One CTA = 64 z rows against the whole codebook.  64x64x16 register-tiled fp32 dot products, running
// (min dist, first index) per row; distance evaluated in the reference's order (|z|^2 - 2 z.e) + |e|^2.
// Non-finite distances: NaN counts as +inf and equal distances go to the smaller index, so a row with a NaN or +-inf element
// (every distance NaN or +inf) returns code 0, as the reference's argmax(-dist) does for NaN, and a NaN code is never chosen
// over a finite one.
__global__ void __launch_bounds__(256) vq_lookup_kernel(const float* __restrict__ z, const float* __restrict__ Et,
                                                        const float* __restrict__ esq, int64_t M, int D, int K,
                                                        int64_t* __restrict__ idx, float* __restrict__ quant,
                                                        double* __restrict__ diff_sum) {
    __shared__ float As[LK][LM + LPAD];
    __shared__ float Bs[LK][LN + LPAD];
    __shared__ float zz[LM];
    __shared__ int best_i[LM];
    __shared__ int second_i[LM];
    __shared__ double dsum_sh[8];

    const int tid = threadIdx.x;
    const int64_t m0 = (int64_t)blockIdx.x * LM;
    const int lr = tid >> 2, lk0 = (tid & 3) * 4;       // loader: row lr, 4 consecutive k
    const int ty = tid >> 4, tx = tid & 15;

    // |z|^2 per row: 4 threads per row
    {
        const int64_t gm = m0 + lr;
        float s = 0.f;
        if (gm < M) {
            const float* zr = z + gm * D;
            for (int d = (tid & 3); d < D; d += 4) s = fmaf(zr[d], zr[d], s);
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if ((tid & 3) == 0) zz[lr] = s;
    }
    __syncthreads();

    // running best and runner-up (distance, index) per owned row; order = (smaller distance, then smaller index)
    float bd[4], sd[4];
    int bi[4], si[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { bd[i] = sd[i] = INFINITY; bi[i] = si[i] = 0x7fffffff; }

    for (int c0 = 0; c0 < K; c0 += LN) {
        float acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
        for (int k0 = 0; k0 < D; k0 += LK) {
            {
                const int64_t gm = m0 + lr;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (gm < M) v = __ldg(reinterpret_cast<const float4*>(z + gm * D + k0 + lk0));
                As[lk0 + 0][lr] = v.x; As[lk0 + 1][lr] = v.y; As[lk0 + 2][lr] = v.z; As[lk0 + 3][lr] = v.w;
                const int gc = c0 + lr;
                float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
                if (gc < K) w = __ldg(reinterpret_cast<const float4*>(Et + (int64_t)gc * D + k0 + lk0));
                Bs[lk0 + 0][lr] = w.x; Bs[lk0 + 1][lr] = w.y; Bs[lk0 + 2][lr] = w.z; Bs[lk0 + 3][lr] = w.w;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < LK; ++kk) {
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
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float zi = zz[ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = c0 + tx * 4 + j;
                if (c < K) {
                    // NaN reads as +inf, and +inf distances tie: a row with a NaN or +-inf element gets code 0
                    const float dist = fminf(__fadd_rn(__fsub_rn(zi, 2.0f * acc[i][j]), __ldg(esq + c)), INFINITY);
                    if (dist < bd[i] || (dist == bd[i] && c < bi[i])) { sd[i] = bd[i]; si[i] = bi[i]; bd[i] = dist; bi[i] = c; }
                    else if (dist < sd[i] || (dist == sd[i] && c < si[i])) { sd[i] = dist; si[i] = c; }
                }
            }
        }
    }
    // merge the (best, runner-up) pairs of the 16 threads (tx) that share rows: 16 consecutive lanes of one warp
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            const float obd = __shfl_xor_sync(0xffffffffu, bd[i], o), osd = __shfl_xor_sync(0xffffffffu, sd[i], o);
            const int obi = __shfl_xor_sync(0xffffffffu, bi[i], o), osi = __shfl_xor_sync(0xffffffffu, si[i], o);
            if (obd < bd[i] || (obd == bd[i] && obi < bi[i])) {
                // other's best wins; runner-up = min(my best, other's runner-up)
                if (bd[i] < osd || (bd[i] == osd && bi[i] < osi)) { sd[i] = bd[i]; si[i] = bi[i]; } else { sd[i] = osd; si[i] = osi; }
                bd[i] = obd; bi[i] = obi;
            } else {
                // my best stays; runner-up = min(my runner-up, other's best)
                if (obd < sd[i] || (obd == sd[i] && obi < si[i])) { sd[i] = obd; si[i] = obi; }
            }
        }
        if (tx == 0) {
            best_i[ty * 4 + i] = bi[i];
            // near-tie: the fp32 gap is within the rounding error of a 256-term fp32 dot product -> settle it in fp64
            const float scale = zz[ty * 4 + i] + fabsf(bd[i]) + fabsf(sd[i]);
            second_i[ty * 4 + i] = (si[i] != 0x7fffffff && (sd[i] - bd[i]) <= 2e-5f * scale) ? si[i] : -1;
        }
    }
    __syncthreads();
    // fp64 re-score of flagged rows (direct sum of squared differences, 4 threads per row): the index returned is the
    // exact-arithmetic nearest neighbour, ties to the smaller index (== argmax(-dist) first-index rule, utils_th.py:41)
    {
        const int64_t gm = m0 + lr;
        const int cand = second_i[lr];
        if (gm < M && cand >= 0) {           // uniform across the 4 threads of the row
            const int b0 = best_i[lr];
            const float* zr = z + gm * D;
            const float* e0 = Et + (int64_t)b0 * D;
            const float* e1 = Et + (int64_t)cand * D;
            double d0 = 0.0, d1 = 0.0;
            for (int d = (tid & 3); d < D; d += 4) {
                const double zv = (double)zr[d];
                const double a = (double)e0[d] - zv, b = (double)e1[d] - zv;
                d0 += a * a;
                d1 += b * b;
            }
            const unsigned qmask = 0xFu << (tid & 28);      // only the 4 lanes of this row take this branch together
            d0 += __shfl_xor_sync(qmask, d0, 1); d0 += __shfl_xor_sync(qmask, d0, 2);
            d1 += __shfl_xor_sync(qmask, d1, 1); d1 += __shfl_xor_sync(qmask, d1, 2);
            if ((tid & 3) == 0 && (d1 < d0 || (d1 == d0 && cand < b0))) best_i[lr] = cand;
        }
    }
    __syncthreads();
    if (tid < LM && m0 + tid < M) idx[m0 + tid] = (int64_t)best_i[tid];

    // gather + commit-loss partial sum: 4 threads per row
    double ds = 0.0;
    {
        const int64_t gm = m0 + lr;
        if (gm < M && (quant || diff_sum)) {
            const float* e = Et + (int64_t)best_i[lr] * D;
            const float* zr = z + gm * D;
            for (int d = (tid & 3) * 4; d < D; d += 16) {
                const float4 ev = __ldg(reinterpret_cast<const float4*>(e + d));
                const float4 zv = __ldg(reinterpret_cast<const float4*>(zr + d));
                if (quant)   // reference returns the straight-through value input + (quantize - input) (utils_th.py:67)
                    *reinterpret_cast<float4*>(quant + gm * D + d) =
                        make_float4(__fadd_rn(zv.x, __fsub_rn(ev.x, zv.x)), __fadd_rn(zv.y, __fsub_rn(ev.y, zv.y)),
                                    __fadd_rn(zv.z, __fsub_rn(ev.z, zv.z)), __fadd_rn(zv.w, __fsub_rn(ev.w, zv.w)));
                const float a = ev.x - zv.x, b = ev.y - zv.y, c = ev.z - zv.z, dd = ev.w - zv.w;
                ds += (double)(a * a) + (double)(b * b) + (double)(c * c) + (double)(dd * dd);
            }
        }
    }
    if (diff_sum) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ds += __shfl_xor_sync(0xffffffffu, ds, o);
        if ((tid & 31) == 0) dsum_sh[tid >> 5] = ds;
        __syncthreads();
        if (tid == 0) {
            double t = 0;
            for (int w = 0; w < 8; ++w) t += dsum_sh[w];
            atomicAdd(diff_sum, t);
        }
    }
}

__global__ void gather_rows_kernel(const float* __restrict__ table, const int64_t* __restrict__ idx, int64_t M, int D,
                                   int64_t n_rows, float* __restrict__ out) {
    const int quads = D >> 2;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * quads) return;
    const int64_t m = i / quads;
    const int q = (int)(i % quads);
    int64_t r = idx[m];
    if (r < 0) r = 0;
    if (r >= n_rows) r = n_rows - 1;
    reinterpret_cast<float4*>(out)[i] = __ldg(reinterpret_cast<const float4*>(table + r * D) + q);
}

__global__ void ema_stats_kernel(const float* __restrict__ z, const int64_t* __restrict__ idx, int64_t M, int D, int K,
                                 float* __restrict__ counts, float* __restrict__ embed_sum_dk) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * D) return;
    const int64_t m = i / D;
    const int d = (int)(i % D);
    const int64_t k = idx[m];
    atomicAdd(embed_sum_dk + (int64_t)d * K + k, z[i]);
    if (d == 0) atomicAdd(counts + k, 1.0f);
}

__global__ void commit_grad_kernel(const float* __restrict__ emb, const float* __restrict__ counts, const float* __restrict__ esum, long long n,
                                   int K, float coef, int accumulate, float* __restrict__ grad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const float g = coef * (counts[i % K] * emb[i] - esum[i]);
        grad[i] = accumulate ? __fadd_rn(grad[i], g) : g;
    }
}

// single block of 1024 threads; thread k owns code k (K <= 1024 handled by striding)
__global__ void __launch_bounds__(1024) ema_update_kernel(const float* __restrict__ counts, const float* __restrict__ esum, int D,
                                                          int K, float alpha, float corr, float eps, float* __restrict__ cs,
                                                          float* __restrict__ dw, float* __restrict__ emb, float* __restrict__ Et,
                                                          float* __restrict__ esq) {
    __shared__ float red[32];
    __shared__ float n_sh;
    float local = 0.f;
    for (int k = threadIdx.x; k < K; k += 1024) {
        const float h = cs[k];
        const float nh = h + alpha * (counts[k] - h);     // add_(x - h, alpha)
        cs[k] = nh;
        local += nh / corr;
    }
    local = warp_sum(local);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = red[threadIdx.x];
        v = warp_sum(v);
        if (threadIdx.x == 0) n_sh = v;
    }
    __syncthreads();
    const float n = n_sh;
    for (int k = threadIdx.x; k < K; k += 1024) {
        const float ecs = cs[k] / corr;
        const float cluster = (ecs + eps) / (n + (float)K * eps) * n;
        float sq = 0.f;
        for (int d = 0; d < D; ++d) {
            const int64_t o = (int64_t)d * K + k;
            const float h = dw[o];
            const float nh = h + alpha * (esum[o] - h);
            dw[o] = nh;
            const float e = (nh / corr) / cluster;
            emb[o] = e;
            Et[(int64_t)k * D + d] = e;
            sq = fmaf(e, e, sq);
        }
        esq[k] = sq;
    }
}

__global__ void prepare_codebook_kernel(const float* __restrict__ emb, int D, int K, float* __restrict__ Et,
                                        float* __restrict__ esq) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    float sq = 0.f;
    for (int d = 0; d < D; ++d) {
        const float e = emb[(int64_t)d * K + k];
        Et[(int64_t)k * D + d] = e;
        sq = __fadd_rn(sq, __fmul_rn(e, e));     // embeddings.pow(2).sum(0): square then add, no contraction
    }
    esq[k] = sq;
}

}  // namespace

extern "C" int vf_vq_lookup(const float* z, const float* Et, const float* esq, int64_t M, int D, int K, int64_t* idx,
                            float* quant, double* diff_sum, vf_stream_t s) {
    if (M == 0) return VF_OK;
    VF_CHECK_ARG(z && Et && esq && idx, "vf_vq_lookup: null pointer");
    VF_CHECK_ARG(D % 16 == 0 && K > 0 && M >= 0, "vf_vq_lookup: unsupported D=%d K=%d", D, K);
    const unsigned blocks = (unsigned)((M + LM - 1) / LM);
    vq_lookup_kernel<<<blocks, 256, 0, vf_s(s)>>>(z, Et, esq, M, D, K, idx, quant, diff_sum);
    VF_CHECK_LAUNCH("vf_vq_lookup");
    return VF_OK;
}

extern "C" int vf_gather_rows(const float* table, const int64_t* idx, int64_t M, int D, int64_t n_rows, float* out,
                              vf_stream_t s) {
    VF_CHECK_ARG(table && idx && out && D % 4 == 0 && n_rows > 0, "vf_gather_rows: bad args");
    if (M == 0) return VF_OK;
    const int64_t total = M * (D / 4);
    gather_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, vf_s(s)>>>(table, idx, M, D, n_rows, out);
    VF_CHECK_LAUNCH("vf_gather_rows");
    return VF_OK;
}

extern "C" int vf_vq_ema_stats(const float* z, const int64_t* idx, int64_t M, int D, int K, float* counts,
                               float* embed_sum_dk, vf_stream_t s) {
    VF_CHECK_ARG(z && idx && counts && embed_sum_dk, "vf_vq_ema_stats: null pointer");
    if (M == 0) return VF_OK;
    const int64_t total = M * D;
    ema_stats_kernel<<<(unsigned)((total + 255) / 256), 256, 0, vf_s(s)>>>(z, idx, M, D, K, counts, embed_sum_dk);
    VF_CHECK_LAUNCH("vf_vq_ema_stats");
    return VF_OK;
}

// Gradient of the commitment term of Quantize (utils_th.py:113-114, beta mean((q - sg(z))^2)) with respect to the [D,K] codebook:
// column k collects coef * (count_k e_k - sum of the z rows mapped to k); counts / sums come from vf_vq_ema_stats.  accumulate: added to
// grad (one more backward pass into the same gradient buffer), else written over it.
extern "C" int vf_vq_commit_grad(const float* embeddings_dk, const float* counts, const float* embed_sum_dk, int D, int K, float coef,
                                 int accumulate, float* grad_dk, vf_stream_t s) {
    VF_CHECK_ARG(embeddings_dk && counts && embed_sum_dk && grad_dk && D > 0 && K > 0, "vf_vq_commit_grad: bad args");
    const long long n = (long long)D * K;
    commit_grad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, vf_s(s)>>>(embeddings_dk, counts, embed_sum_dk, n, K, coef, accumulate, grad_dk);
    VF_CHECK_LAUNCH("vf_vq_commit_grad");
    return VF_OK;
}

extern "C" int vf_vq_ema_update(const float* counts, const float* embed_sum_dk, int D, int K, float alpha, float corr,
                                float eps, float* cs_hidden, float* dw_hidden, float* embeddings_dk, float* Et, float* esq,
                                vf_stream_t s) {
    VF_CHECK_ARG(counts && embed_sum_dk && cs_hidden && dw_hidden && embeddings_dk && Et && esq, "vf_vq_ema_update: null");
    ema_update_kernel<<<1, 1024, 0, vf_s(s)>>>(counts, embed_sum_dk, D, K, alpha, corr, eps, cs_hidden, dw_hidden,
                                               embeddings_dk, Et, esq);
    VF_CHECK_LAUNCH("vf_vq_ema_update");
    return VF_OK;
}

extern "C" int vf_vq_prepare_codebook(const float* embeddings_dk, int D, int K, float* Et, float* esq, vf_stream_t s) {
    VF_CHECK_ARG(embeddings_dk && Et && esq, "vf_vq_prepare_codebook: null");
    prepare_codebook_kernel<<<(K + 127) / 128, 128, 0, vf_s(s)>>>(embeddings_dk, D, K, Et, esq);
    VF_CHECK_LAUNCH("vf_vq_prepare_codebook");
    return VF_OK;
}
