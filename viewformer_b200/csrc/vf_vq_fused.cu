// Fused codebook lookup on Hopper tensor cores (sm_90a, wgmma):  idx[m] = argmin_k |z_m - e_k|^2   — viewformer/models/utils_th.py:34-41.
//
// HBM traffic is the algorithmic minimum: every z row (fp32, 4*D bytes) is read ONCE, one int64 index is written; the distance
// matrix never exists outside registers.  Per CTA and 128-row tile (persistent CTAs walk the tiles):
//   convert (8 warps) z fp32 [128 rows x D] --LDG.128--> fp16 --> 128B-swizzled K-major A tile in shared memory;
//                     also |z|^2 per row and a range check (|z_i| beyond fp16 -> the row goes to the exact path)
//   TMA producer      B stages (256 codes x 64 k) of Eh = fp16(-2 e)   [K, D] K-major, running ahead across sub-tiles and tiles
//   MMA (2 warpgroups) S[64 rows, 256 codes] = A . B^T per warpgroup and sub-tile, fp32 in registers; s = S + |e|^2 (fp32, shared
//                     memory table), the code index is packed into the 6 low mantissa bits and a running (min, second min) pair
//                     per (row, 64-code set) is kept with integer min / max, merged over the 4 lanes that share a row
//   merge (4 warps)   per row: best code over the 16 sets; if the runner-up lies within the fp16 rounding bound of the best the row
//                     is queued for the exact pass (PAIR: both candidates known; FULL: a third may hide inside one set)
// vq_rescue_kernel then settles queued rows in fp64 (direct sum of squared differences, ties to the smaller index — the same rule as
// vf_vq_lookup), so with tol_factor = 1 the index returned is the fp64 nearest code on every row whose fp64 gap to the runner-up
// exceeds the fp16 rounding bound below, and the fp32 kernel's index wherever the fp32 kernel itself is decisive.  Non-finite rows
// (a NaN or +-inf element) are settled over all codes with NaN read as +inf, so they return code 0, as vf_vq_lookup does.
//
// Rounding model (why the tolerance is safe): an fp16 operand x carries an error of at most max(2^-11 |x|, 2^-25) (relative in
// the normal range, absolute among the subnormals below 2^-14).  The relative part gives |d(z.e)| <= 2^-10 sum|z_i e_i| <=
// 2^-10 |z||e|, so the score -2 z.e + |e|^2 of two codes moves by at most 2^-9 |z| (|e_a| + |e_b|) against each other; this is
// reached when all roundings align (tests/test_vq_lookup_edges_host.py builds such rows), while random roundings move it ~40x
// less.  `tol_factor` scales that bound: 1.0 (the default of viewformer_b200._lib) is the proven worst case, smaller factors are
// a statistical bet that aligned rows do not occur.  Always included unscaled: the subnormal part, 2^-23 sqrt(D) (|z| + |e_a| +
// |e_b|) + D 2^-48; index packing (6 mantissa bits) and the truncating tensor-core accumulation, 2^-16 |s| + 4 G.
#include "vf_wgmma.cuh"
#include <cuda_fp16.h>

namespace {
using namespace vftc;

constexpr int TM = 128;                 // z rows per CTA tile
constexpr int TN = 256;                 // codes per sub-tile (MMA N)
constexpr int KB_BYTES = TM * 128;      // one A k-block: 128 rows x 128 B
constexpr int A_BYTES = 4 * KB_BYTES;   // up to D = 256
constexpr int B_STAGE = TN * 128;       // one (256 codes x 64 k) stage
constexpr int B_STAGES = 4;
constexpr int NCONV = 8;                // converter warps (= the MMA warps)
constexpr int MMA_THREADS = 32 * NCONV;
constexpr int THREADS = MMA_THREADS + 128;     // + the producer warpgroup (one elected thread issues TMA; see setmaxnreg_dec)
constexpr int MAXK = 1024;
constexpr int RES_BYTES = 4 * TM * 16;  // 4 column groups x 128 rows x (3 best keys + pad)
constexpr int SMEM = A_BYTES + B_STAGES * B_STAGE + MAXK * 4 + TM * 4 * 2 + RES_BYTES + 8 * 2 * B_STAGES + 1024;

struct VqParams {
    CUtensorMap tmB;            // Eh [K, D] fp16: box {64, 128}
    const float* z;             // [M, D]
    const float* esq;           // [K]
    long long M;
    int D, K, kblocks, nsub;
    long long n_tiles;          // ceil(M / 128)
    float tol_factor;
    int key_mul;                // 256, passed as data so the key is ONE IMAD (fma pipe) instead of a shift + add on the alu pipe
    long long* idx;             // [M]
    int4* worklist;             // {row, c1, c2 (-1: all codes), 0}
    int* counter;               // [0] queued rows, [1] of which FULL
};

// explicit shared-state-space accesses: pointers derived from the aligned dynamic-smem base are "generic" to the compiler, and a
// generic LD to shared memory is tracked on the long scoreboard like a global load
__device__ __forceinline__ uint4 lds_u4(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_u4(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float lds_f(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}

__global__ void __launch_bounds__(THREADS, 1) vq_lookup_fused_kernel(const __grid_constant__ VqParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;                                          // [A_BYTES]
    uint8_t* sB = sA + A_BYTES;                                  // [B_STAGES][B_STAGE]
    float* esq_s = reinterpret_cast<float*>(sB + B_STAGES * B_STAGE);            // [MAXK]
    float* zz_s = esq_s + MAXK;                                  // [TM]
    int* bad_s = reinterpret_cast<int*>(zz_s + TM);              // [TM]
    uint8_t* res_s = reinterpret_cast<uint8_t*>(bad_s + TM);     // [4 groups][TM] x uint4 (3 best keys of the (row, group))
    uint64_t* b_full = reinterpret_cast<uint64_t*>(res_s + RES_BYTES);          // [B_STAGES]
    uint64_t* b_empty = b_full + B_STAGES;                       // [B_STAGES]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        prefetch_tmap(&p.tmB);
        for (int s = 0; s < B_STAGES; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], MMA_THREADS); }
        mbar_fence_init();
    }
    // Fixed-point scores: with C = 1.5 * 2^k and |score| < 2^(k-1), the fp32 sum  t = acc + (|e|^2 + C)  stays inside the binade [2^k, 2^(k+1)),
    // so its BIT PATTERN is an order-preserving integer with step G = 2^(k-23).  key = t_bits * 256 + code index is then one IMAD, and
    // the top-2 tracking runs on integer min / max.  k is chosen from the codebook (2^(k-1) >= 17.2 max|e|^2): rows with |z| up to
    // 8 max|e| fit; rows beyond that go to the exact pass like rows outside the fp16 range.
    __shared__ int esqmax_bits;
    if (threadIdx.x == 0) esqmax_bits = 0;
    __syncthreads();
    {
        float mx = 0.f;
        for (int i = threadIdx.x; i < p.K; i += THREADS) {
            const float v = __ldg(p.esq + i);
            mx = fmaxf(mx, v == v ? v : INFINITY);              // fmaxf drops NaN: a NaN code must fail codebook_ok below
        }
        mx = warp_max(mx);
        if ((threadIdx.x & 31) == 0) atomicMax(&esqmax_bits, __float_as_int(mx));      // non-negative floats order like their bit patterns
    }
    __syncthreads();
    const float esqmax = fmaxf(__int_as_float(esqmax_bits), 1e-30f);
    const bool codebook_ok = esqmax < 1.0e9f;                    // every -2 e_i representable in fp16 (|e_i| <= |e| < 31623); NaN / inf fail
    const int kexp = ((__float_as_int(17.2f * esqmax) >> 23) & 255) - 127 + 2;          // 2^(kexp - 1) > 17.2 max|e|^2
    const int c_bits = ((kexp + 127) << 23) | 0x400000;          // C = 1.5 * 2^kexp
    const float c_off = __int_as_float(c_bits);
    const int key0 = (int)((uint32_t)c_bits << 8);               // key of score 0 and index 0: +-2^30 (exponent parity), keys never wrap
    const float g_step = __int_as_float((kexp - 23 + 127) << 23);              // G = 2^(kexp - 23)
    const float half_range = __int_as_float((kexp - 1 + 127) << 23);           // 2^(kexp - 1)
    const float zcap = (half_range - esqmax) / (2.02f * sqrtf(esqmax));        // 2 |z| |e| (1 + 2^-10 ...) + |e|^2 < 2^(kexp - 1)
    const float zz_cap = codebook_ok ? fminf(zcap * zcap, 3.6e9f) : -1.0f;     // |z_i| <= |z| < 60000: inside the fp16 range
    for (int i = threadIdx.x; i < p.K; i += THREADS) esq_s[i] = __ldg(p.esq + i) + c_off;
    __syncthreads();

    if (warp >= MMA_THREADS / 32) {
        // ===================== TMA producer: every B stage (256 codes x 64 k) =====================
        setmaxnreg_dec<40>();
        if (warp == MMA_THREADS / 32 && elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (long long t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
                for (int n = 0; n < p.nsub; ++n)
                    for (int kb = 0; kb < p.kblocks; ++kb) {
                        mbar_wait(&b_empty[stage], phase ^ 1, "vq_fused(b_empty)");
                        mbar_expect_tx(&b_full[stage], B_STAGE);
                        tma_load_4d(sB + stage * B_STAGE, &p.tmB, &b_full[stage], kb * 64, n * TN, 0, 0);
                        if (++stage == B_STAGES) { stage = 0; phase ^= 1; }
                    }
            }
        }
        return;
    }

    // ===================== warps 0..7: convert, MMA (warpgroup wg = rows [64 wg, +64)), top-2 per (row, 64-code set), merge ==========
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);     // accumulator rows r0, r0 + 8 (layout: vf_wgmma.cuh)
    const int c_ln = 2 * (lane & 3);
    const int my_g = lane & 3;                                   // the 64-code column group whose keys this lane folds
    const uint32_t esq_a = smem_u32(esq_s), res_a = smem_u32(res_s);
    const int EMPTY = 0x7fffffff;
    const int key_mul = p.key_mul;
    int stage = 0;
    uint32_t phase = 0;
    float acc[TN / 2];
    for (long long t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
        named_sync(1, MMA_THREADS);                              // the previous tile's merge is done with sA, zz_s, bad_s, res_s
        // ---- converters: z fp32 -> fp16 swizzled A tile, |z|^2, range check
        {
            const int kb = lane >> 3, ch = lane & 7;              // this lane's 8 elements of a row: k = kb*64 + ch*8 ..
            const bool lane_ok = lane * 8 < p.D;
            const long long row0 = t * TM;
#pragma unroll 1
            for (int rb = 0; rb < TM / NCONV; rb += 4) {           // 4 rows of this warp in flight: 8 x LDG.128 per lane
                float4 v[4][2];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int r = warp + (rb + u) * NCONV;
                    const long long gr = row0 + r;
                    if (gr < p.M && lane_ok) {
                        const float4* src = reinterpret_cast<const float4*>(p.z + gr * p.D + lane * 8);
                        v[u][0] = __ldg(src);
                        v[u][1] = __ldg(src + 1);
                    } else {
                        v[u][0] = v[u][1] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int r = warp + (rb + u) * NCONV;
                    const float e[8] = {v[u][0].x, v[u][0].y, v[u][0].z, v[u][0].w, v[u][1].x, v[u][1].y, v[u][1].z, v[u][1].w};
                    float ss = 0.f;
                    uint32_t w[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        ss = fmaf(e[2 * q], e[2 * q], ss);
                        ss = fmaf(e[2 * q + 1], e[2 * q + 1], ss);
                        const __half2 h = __floats2half2_rn(e[2 * q], e[2 * q + 1]);
                        w[q] = *reinterpret_cast<const uint32_t*>(&h);
                    }
                    if (lane_ok)
                        *reinterpret_cast<uint4*>(sA + kb * KB_BYTES + r * 128 + ((ch ^ (r & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
                    ss = warp_sum(ss);
                    if (lane == 0) {
                        zz_s[r] = ss;
                        // |z|^2 below the cap keeps every element inside the fp16 range and every score inside the fixed-point range;
                        // NaN / inf fail the comparison too.  Rows that fail are decided by the exact pass.
                        bad_s[r] = !(ss < zz_cap);
                    }
                }
            }
        }
        fence_async_smem();                                      // generic-proxy A tile -> visible to wgmma
        named_sync(1, MMA_THREADS);

        // ---- S = A . B^T per 256-code sub-tile, then this thread's keys
        int tk[2][3] = {{EMPTY, EMPTY, EMPTY}, {EMPTY, EMPTY, EMPTY}};     // three best keys of (row r0 + 8 hh, group my_g) over the sets
        const uint32_t a_addr = smem_u32(sA) + (uint32_t)(wg * 64 * 128);
        for (int n = 0; n < p.nsub; ++n) {
            for (int kb = 0; kb < p.kblocks; ++kb) {
                mbar_wait(&b_full[stage], phase, "vq_fused(b_full)");
                const uint64_t adesc = sw128_desc(a_addr + kb * KB_BYTES), bdesc = sw128_desc(smem_u32(sB + stage * B_STAGE));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_ss<TN, F16>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(acc);
                mbar_arrive(&b_empty[stage]);
                if (++stage == B_STAGES) { stage = 0; phase ^= 1; }
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    int m1 = EMPTY, m2 = EMPTY;
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int col = 64 * g + 8 * jj + c_ln;                                   // column of acc[4 j + 2 hh], j = 8 g + jj
                        const float2 e = *reinterpret_cast<const float2*>(esq_s + n * TN + col);
                        const int tb0 = __float_as_int(acc[4 * (8 * g + jj) + 2 * hh] + e.x);     // score + C, one binade
                        const int tb1 = __float_as_int(acc[4 * (8 * g + jj) + 2 * hh + 1] + e.y);
                        const int k0 = tb0 * key_mul + (col & 63), k1 = tb1 * key_mul + (col & 63) + 1;    // low byte = index in the set
                        m2 = min(m2, max(m1, k0));
                        m1 = min(m1, k0);
                        m2 = min(m2, max(m1, k1));
                        m1 = min(m1, k1);
                    }
                    // the set's 64 codes are spread over the 4 lanes of the row: merge their (best, second best) pairs
#pragma unroll
                    for (int o = 1; o < 4; o <<= 1) {
                        const int b1 = __shfl_xor_sync(0xffffffffu, m1, o), b2 = __shfl_xor_sync(0xffffffffu, m2, o);
                        m2 = min(max(m1, b1), min(m2, b2));
                        m1 = min(m1, b1);
                    }
                    if (g == my_g) {
                        // fold the set's two best into the three best of (row, group) (set number into bits 6..7 of the index)
#pragma unroll
                        for (int q = 0; q < 2; ++q) {
                            const int mk = q ? m2 : m1;
                            const int k = mk == EMPTY ? EMPTY : (mk | (n << 6));                  // bits 6..7 of the index byte are zero so far
                            const int a = max(tk[hh][0], k);
                            tk[hh][0] = min(tk[hh][0], k);
                            const int b2 = max(tk[hh][1], a);
                            tk[hh][1] = min(tk[hh][1], a);
                            tk[hh][2] = min(tk[hh][2], b2);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
            sts_u4(res_a + (uint32_t)((my_g * TM + r0 + 8 * hh) * 16), make_uint4((uint32_t)tk[hh][0], (uint32_t)tk[hh][1], (uint32_t)tk[hh][2], 0u));
        named_sync(1, MMA_THREADS);                              // the tile's keys are in res_s
        // ---- merge (threads 0..127, thread = row): best code over the sets; rows whose runner-up is within the bound are queued
        if (threadIdx.x < TM) {
            const int row = threadIdx.x;
            const long long gr = t * TM + row;
            if (gr < p.M) {
                uint32_t ks[12];
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const uint4 v = lds_u4(res_a + (uint32_t)((g * TM + row) * 16));
                    ks[3 * g] = v.x; ks[3 * g + 1] = v.y; ks[3 * g + 2] = v.z;
                }
                    // key -> (value, code, set): value = ((key - key0) >> 8) * G, code = n*256 + g*64 + idx6, set = n*4 + g
                    const float vscale = g_step * 0.00390625f;            // G / 256
                    const float sub_k = 1.1920929e-7f * sqrtf((float)p.D), sub_0 = (float)p.D * 3.5527137e-15f;    // 2^-23 sqrt(D), D 2^-48
                    float bv = __int_as_float(0x7f800000);
                    int bc = 0x7fffffff, bset = -1;
#pragma unroll
                    for (int i = 0; i < 12; ++i) {
                        const uint32_t k = ks[i];
                        const float v = (float)((int)(k & 0xFFFFFF00u) - key0) * vscale;
                        const int n = (int)((k >> 6) & 3u), g = i / 3;
                        const int c = n * TN + g * 64 + (int)(k & 63u);
                        if (k != 0x7fffffffu && (v < bv || (v == bv && c < bc))) { bv = v; bc = c; bset = n * 4 + g; }
                    }
                    const uint32_t zslot = (uint32_t)(row * 4);
                    bool bad = bad_s[row] != 0;
                    if (bset < 0) { bc = 0; bad = true; }
                    const float znorm = sqrtf(lds_f(smem_u32(zz_s) + zslot));
                    const float eb = sqrtf(__ldg(p.esq + bc));
                    int within = 0, oc = -1, oset = -1;
                    uint32_t inside = 0;                                   // bit i: key i lies inside the tolerance (the best code itself included)
#pragma unroll
                    for (int i = 0; i < 12; ++i) {
                        const uint32_t k = ks[i];
                        if (k == 0x7fffffffu) continue;                                      // empty slot
                        const float v = (float)((int)(k & 0xFFFFFF00u) - key0) * vscale;
                        const int n = (int)((k >> 6) & 3u), g = i / 3;
                        const int c = n * TN + g * 64 + (int)(k & 63u);
                        if (c == bc) { inside |= 1u << i; continue; }
                        // truncating tensor-core accumulation (2^-16 relative, generous) + the fixed-point step of both scores
                        // + fp16 subnormal operands (absolute rounding 2^-25, see the rounding model above)
                        const float ec = sqrtf(__ldg(p.esq + c));
                        const float slack = 1.52587891e-5f * (fabsf(v) + fabsf(bv)) + 4.0f * g_step + sub_k * (znorm + eb + ec) + sub_0;
                        const float tol = p.tol_factor * 0.001953125f * znorm * (eb + ec) + slack;
                        if (v - bv <= tol) { ++within; inside |= 1u << i; oc = c; oset = n * 4 + g; }
                    }
                    p.idx[gr] = (long long)bc;
                    if (within > 0 || bad) {
                        // A code inside the tolerance that is NOT among the 12 keys sits either in a set whose two reported best are both
                        // inside the tolerance (the sets of all inside keys are masked) or behind a thread whose three reported keys are all
                        // inside (then any of that thread's sets may hide it) — proof sketch in DESIGN.md.  One other candidate in a different
                        // set than the best: PAIR (two known codes).  Everything else: SETS (all codes of the masked 64-code sets).
                        uint32_t mask = 0;                                 // 64-code sets (sub-tile * 4 + column group) the exact pass looks at
#pragma unroll
                        for (int i = 0; i < 12; ++i)
                            if ((inside >> i) & 1u) mask |= 1u << ((((ks[i] >> 6) & 3u) << 2) | (uint32_t)(i / 3));
#pragma unroll
                        for (int g = 0; g < 4; ++g)
                            if (((inside >> (3 * g)) & 7u) == 7u) mask |= 0x1111u << g;
                        const bool pair = !bad && within == 1 && oset != bset;
                        if (bad) mask = 0xFFFFu;
                        // PAIR entries fill the worklist from the front, SETS entries from the back
                        if (!pair) p.worklist[p.M - 1 - atomicAdd(p.counter + 1, 1)] = make_int4((int)gr, bc, -1, (int)mask);
                        else p.worklist[atomicAdd(p.counter, 1)] = make_int4((int)gr, bc, oc, 0);
                    }
            }
        }
    }
}

__device__ __forceinline__ float warp_min_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Exact pass over the queued rows: fp64 direct sum of squared differences, ties to the smaller index.
// PAIR entries (front of the worklist): one warp per entry, the two known candidates.  SETS entries (back of the worklist): one CTA per
// entry, the codes of the 64-code sets named by the entry's mask (all sets for rows outside the fp16 range), block-wide argmin.
__global__ void __launch_bounds__(256) vq_rescue_kernel(const float* __restrict__ z, const float* __restrict__ Et, const float* __restrict__ Edk,
                                                        const float* __restrict__ esq, int D, int K, long long M,
                                                        const int4* __restrict__ worklist, const int* __restrict__ counter,
                                                        long long* __restrict__ idx) {
    constexpr int MAXCAND = 64;
    __shared__ double sd[8];
    __shared__ int si[8];
    __shared__ __align__(16) float zs[256];
    __shared__ int cands[MAXCAND];
    __shared__ float scores[1024];
    __shared__ float part[4][64];
    __shared__ int ncand;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    const int n_pair = counter[0], n_full = counter[1];
    for (int i = gw; i < n_pair; i += nw) {
        const int4 e = worklist[i];
        const float* zr = z + (long long)e.x * D;
        double d0 = 0.0, d1 = 0.0;
        const float* e0 = Et + (long long)e.y * D;
        const float* e1 = Et + (long long)e.z * D;
        for (int d = lane; d < D; d += 32) {
            const double zv = (double)zr[d];
            const double a = (double)e0[d] - zv, b = (double)e1[d] - zv;
            d0 += a * a;
            d1 += b * b;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { d0 += __shfl_xor_sync(0xffffffffu, d0, o); d1 += __shfl_xor_sync(0xffffffffu, d1, o); }
        if (lane == 0) idx[e.x] = (long long)((d1 < d0 || (d1 == d0 && e.z < e.y)) ? e.z : e.y);
    }
    // SETS entries: fp32 screening of the codes of the masked 64-code sets by the whole CTA (the reference's expanded form), then fp64
    // only for the codes whose fp32 score lies within the fp32 rounding bound of the minimum (almost always one or two)
    const int nsets = K >> 6;
    for (int i = blockIdx.x; i < n_full; i += gridDim.x) {
        const int4 e = worklist[M - 1 - i];
        const uint32_t all_sets = nsets >= 32 ? 0xffffffffu : ((1u << nsets) - 1u);
        const uint32_t mask = (e.w ? (uint32_t)e.w : all_sets) & all_sets;
        const float* zr = z + (long long)e.x * D;
        for (int d = threadIdx.x; d < D; d += 256) zs[d] = zr[d];
        if (threadIdx.x == 0) ncand = 0;
        __syncthreads();
        float zz = 0.f;
        for (int d = 0; d < D; ++d) zz = fmaf(zs[d], zs[d], zz);
        // screening: thread = (code of the set, quarter of the dimensions); the codebook is read in its [D, K] layout so that a warp's 32
        // codes are one coalesced 128-byte row per dimension; z broadcast from shared memory; 8 independent loads in flight per thread
        float smin = INFINITY;
        {
            const int cs = threadIdx.x & 63, slice = threadIdx.x >> 6, dq = D >> 2;
            for (uint32_t rest = mask; rest; rest &= rest - 1) {
                const int set = __ffs(rest) - 1;
                const int c = (set >> 2) * 256 + (set & 3) * 64 + cs;          // set = sub-tile * 4 + column group (main kernel's numbering)
                const float* ep = Edk + (long long)(slice * dq) * K + c;
                const float* zp = zs + slice * dq;
                float a0 = 0.f, a1 = 0.f;
                for (int d = 0; d < dq; d += 8) {
                    float ev[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) ev[q] = __ldg(ep + (long long)(d + q) * K);
#pragma unroll
                    for (int q = 0; q < 8; q += 2) { a0 = fmaf(zp[d + q], ev[q], a0); a1 = fmaf(zp[d + q + 1], ev[q + 1], a1); }
                }
                part[slice][cs] = a0 + a1;
                __syncthreads();
                if (slice == 0) {
                    const float sco = __ldg(esq + c) - 2.0f * ((part[0][cs] + part[1][cs]) + (part[2][cs] + part[3][cs]));
                    scores[c] = sco;
                    smin = fminf(smin, sco);
                }
                __syncthreads();
            }
        }
        smin = warp_min_f(smin);
        if (lane == 0) sd[warp] = (double)smin;
        __syncthreads();
        if (threadIdx.x == 0) {
            double m = sd[0];
            for (int w = 1; w < 8; ++w) m = sd[w] < m ? sd[w] : m;
            sd[0] = m;
        }
        __syncthreads();
        const float gmin = (float)sd[0];
        __syncthreads();
        const bool finite = gmin == gmin && fabsf(gmin) < INFINITY && zz == zz && zz < INFINITY;
        for (int c = threadIdx.x; c < K; c += 256) {
            if (!((mask >> (((c >> 8) << 2) | ((c >> 6) & 3))) & 1u)) continue;
            // fp32 error of a D-term dot product: <= D * 2^-24 * |z||e| per score; 6e-5 * (|z|^2 + |s|) covers it with margin
            const float sco = scores[c];
            if (!finite || sco - gmin <= 6e-5f * (zz + fabsf(gmin) + fabsf(sco))) {
                const int slot = atomicAdd(&ncand, 1);
                if (slot < MAXCAND) cands[slot] = c;
            }
        }
        __syncthreads();
        const int nc = ncand;
        double bd = INFINITY;
        int bi = 0x7fffffff;
        auto score64 = [&](int c) {
            const float* ec = Et + (long long)c * D;
            double dd = 0.0;
            for (int d = lane; d < D; d += 32) {
                const double tt = (double)ec[d] - (double)zs[d];
                dd += tt * tt;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) dd += __shfl_xor_sync(0xffffffffu, dd, o);
            dd = fmin(dd, (double)INFINITY);                  // NaN reads as +inf; +inf ties go to the smaller index (vf_vq_lookup's rule)
            if (dd < bd || (dd == bd && c < bi)) { bd = dd; bi = c; }
        };
        if (nc <= MAXCAND) {
            for (int k = warp; k < nc; k += 8) score64(cands[k]);
        } else {                                              // degenerate row (all codes nearly equidistant, or non-finite): every masked code in fp64
            for (int c = warp; c < K; c += 8)
                if ((mask >> (((c >> 8) << 2) | ((c >> 6) & 3))) & 1u) score64(c);
        }
        if (lane == 0) { sd[warp] = bd; si[warp] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 0; w < 8; ++w)
                if (sd[w] < bd || (sd[w] == bd && si[w] < bi)) { bd = sd[w]; bi = si[w]; }
            idx[e.x] = (long long)bi;
        }
        __syncthreads();
    }
}

// quant = z + (e - z) (straight-through value, utils_th.py:67) and the commit-loss sum  sum (e - z)^2  for given indices
__global__ void __launch_bounds__(256) vq_gather_diff_kernel(const float* __restrict__ z, const float* __restrict__ Et,
                                                             const long long* __restrict__ idx, long long M, int D,
                                                             float* __restrict__ quant, double* __restrict__ diff_sum) {
    __shared__ double dsum_sh[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * 8 + warp;
    double ds = 0.0;
    if (row < M) {
        const float* e = Et + idx[row] * D;
        const float* zr = z + row * D;
        for (int d = lane * 4; d < D; d += 128) {
            const float4 ev = __ldg(reinterpret_cast<const float4*>(e + d));
            const float4 zv = __ldg(reinterpret_cast<const float4*>(zr + d));
            if (quant)
                *reinterpret_cast<float4*>(quant + row * D + d) =
                    make_float4(__fadd_rn(zv.x, __fsub_rn(ev.x, zv.x)), __fadd_rn(zv.y, __fsub_rn(ev.y, zv.y)),
                                __fadd_rn(zv.z, __fsub_rn(ev.z, zv.z)), __fadd_rn(zv.w, __fsub_rn(ev.w, zv.w)));
            const float a = ev.x - zv.x, b = ev.y - zv.y, c = ev.z - zv.z, dd = ev.w - zv.w;
            ds += (double)(a * a) + (double)(b * b) + (double)(c * c) + (double)(dd * dd);
        }
    }
    if (diff_sum) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ds += __shfl_xor_sync(0xffffffffu, ds, o);
        if (lane == 0) dsum_sh[warp] = ds;
        __syncthreads();
        if (threadIdx.x == 0) {
            double tsum = 0;
            for (int w = 0; w < 8; ++w) tsum += dsum_sh[w];
            atomicAdd(diff_sum, tsum);
        }
    }
}

__global__ void codebook_f16_kernel(const float* __restrict__ Et, long long n, __half* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __float2half_rn(-2.0f * Et[i]);
}

}  // namespace

extern "C" int vf_vq_prepare_codebook_f16(const float* Et, int K, int D, void* Eh_f16, vf_stream_t s) {
    VF_CHECK_ARG(Et && Eh_f16 && K > 0 && D > 0, "vf_vq_prepare_codebook_f16: bad args");
    const long long n = (long long)K * D;
    codebook_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, vf_s(s)>>>(Et, n, reinterpret_cast<__half*>(Eh_f16));
    VF_CHECK_LAUNCH("vf_vq_prepare_codebook_f16");
    return VF_OK;
}

extern "C" int vf_vq_lookup_fused(const float* z, const void* Eh_f16, const float* Et, const float* E_dk, const float* esq, int64_t M, int D, int K,
                                  float tol_factor, int64_t* idx, void* worklist, int* counter, float* quant, double* diff_sum,
                                  vf_stream_t s) {
    if (M == 0) return VF_OK;
    VF_CHECK_ARG(z && Eh_f16 && Et && E_dk && esq && idx && worklist && counter, "vf_vq_lookup_fused: null pointer");
    VF_CHECK_ARG(D % 64 == 0 && D <= 256 && K % 256 == 0 && K <= MAXK && M < (1ll << 31),
                 "vf_vq_lookup_fused: unsupported D=%d K=%d (D %% 64 == 0, D <= 256, K %% 256 == 0, K <= 1024)", D, K);
    VF_CHECK_ARG((reinterpret_cast<uintptr_t>(z) & 15) == 0, "vf_vq_lookup_fused: z must be 16-byte aligned");
    cudaStream_t st = vf_s(s);
    VqParams prm;
    memset(&prm, 0, sizeof(prm));
    const uint64_t dims[4] = {(uint64_t)D, (uint64_t)K, 1, 1};
    const uint64_t str[3] = {(uint64_t)D * 2, (uint64_t)D * 2 * K, (uint64_t)D * 2 * K};
    const uint32_t box[4] = {64, (uint32_t)TN, 1, 1};
    int rc;
    if ((rc = make_tmap_16bit(&prm.tmB, Eh_f16, dims, str, box)) != VF_OK) return rc;
    prm.z = z; prm.esq = esq; prm.M = M; prm.D = D; prm.K = K;
    prm.kblocks = D / 64; prm.nsub = K / TN;
    prm.n_tiles = (M + TM - 1) / TM;
    prm.tol_factor = tol_factor;
    prm.key_mul = 256;
    prm.idx = reinterpret_cast<long long*>(idx);
    prm.worklist = reinterpret_cast<int4*>(worklist);
    prm.counter = counter;
    cudaError_t e = cudaMemsetAsync(counter, 0, 2 * sizeof(int), st);
    if (e != cudaSuccess) { vf_set_error("vf_vq_lookup_fused: memset: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
    static vf_per_device_flag configured_pd;          // function attributes are per device
    bool& configured = configured_pd.current();
    if (!configured) {
        e = cudaFuncSetAttribute(vq_lookup_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
        if (e != cudaSuccess) { vf_set_error("vf_vq_lookup_fused: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
        configured = true;
    }
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || num_sms <= 0) num_sms = 132;
    }
    const unsigned grid = (unsigned)(prm.n_tiles < num_sms ? prm.n_tiles : num_sms);       // persistent CTAs
    vq_lookup_fused_kernel<<<grid, THREADS, SMEM, st>>>(prm);
    VF_CHECK_LAUNCH("vf_vq_lookup_fused");
    vq_rescue_kernel<<<num_sms * 8, 256, 0, st>>>(z, Et, E_dk, esq, D, K, M, prm.worklist, counter, prm.idx);
    VF_CHECK_LAUNCH("vf_vq_lookup_fused(rescue)");
    if (quant || diff_sum) {
        vq_gather_diff_kernel<<<(unsigned)((M + 7) / 8), 256, 0, st>>>(z, Et, prm.idx, M, D, quant, diff_sum);
        VF_CHECK_LAUNCH("vf_vq_lookup_fused(gather)");
    }
    return VF_OK;
}
