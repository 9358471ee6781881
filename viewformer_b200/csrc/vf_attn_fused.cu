// Fused block-causal attention on Hopper tensor cores (sm_90a, wgmma):  O = softmax(mask(Q K^T)) V  per (batch, head).
//
// Replaces viewformer/models/branching_attention.py:41-61 (compute_causal_block_attention: a view attends to all tokens
// of its own and of every earlier view; logits are NOT scaled by 1/sqrt(dh); masked logits are -1e4 in the reference,
// whose exp underflows to exactly 0 in fp32, so masked keys are simply skipped here) for the single-stream forward.
//
// One CTA = 128 queries (two 64-token views) of one (batch, head); two CTAs share an SM (~90 KB of shared memory each), so one
// CTA's prologue / epilogue hides behind the other's main loop.  Keys are walked ONCE in 64-key tiles; each of the two MMA
// warpgroups owns 64 query rows:
//   S_j = Q K_j^T   64x64 fp32 in registers (wgmma, Q and K from shared memory)
//   row max of the tile (4 lanes per row), P_j = exp2(S_j log2e - m_ref) packed to bf16 straight into the A-operand registers
//   O  += P_j V_j   (wgmma with A from registers, V^T from shared memory), O 64x64 fp32 in registers.
// Online softmax with a lazy reference maximum: m_ref only moves when a tile's maximum exceeds it by more than 2^8, and only
// then is the O accumulator row rescaled.  The final O / l does not depend on which reference was used, so this is the same
// softmax, not an approximation.  Fully masked key tiles are never loaded; a warpgroup whose rows cannot see a tile skips it.
//
// Warp roles (288 threads): warps 0..7 two MMA / softmax warpgroups, warp 8 TMA producer.
#include "vf_wgmma.cuh"

namespace {
using namespace vftc;

constexpr int QT = 128;            // queries per CTA
constexpr int KT = 64;             // keys per tile (= one 128-byte swizzle row of V^T)
constexpr int DH = 64;             // head dim (one 128-byte swizzle row)
constexpr int KSTAGES = 4;         // K tile ring
constexpr int VSTAGES = 3;         // V^T tile ring
constexpr int Q_BYTES = QT * 128;              // 16 KB (double-buffered: the next work item's Q streams in behind the current one)
constexpr int K_BYTES = KT * 128;              // 8 KB
constexpr int V_BYTES = DH * 128;              // [64 dh rows x 64 keys] = 8 KB
constexpr int MMA_THREADS = 256;
constexpr int ATTN_THREADS = MMA_THREADS + 32;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LAZY_LOG2 = 8.0f;              // the reference maximum moves only when a tile exceeds it by more than 2^8

struct AttnParams {
    CUtensorMap tmQ, tmK, tmV;
    int S, H, d, block, n_qtiles, qt0, BH;  // query tiles qt0 .. qt0 + n_qtiles - 1 are computed (qt0 > 0: KV-cache query mode)
    int stream, stream_rows;                // multi-end mode (stream > 0): rows of stream s start at s * stream_rows in qk / V^T
    int skip_tile;                          // >= 0: this 64-key tile of stream 0 is never visited (an unused view slot of the KV cache)
    __nv_bfloat16* out;
    // training instance only (attn_block_causal_kernel<true>):
    float* lse;                             // nullable [B, H, S]: natural-log log-sum-exp of every query row's masked logits
    float* out_f32;                         // nullable [B*S, d]: O in fp32 as well
    unsigned long long drop_seed;           // vf_dropout's seed of this stream's [B, H, S, cols] probability tensor
    uint32_t drop_thr;                      // vf_drop_threshold(rate); 0 = no dropout
    float drop_scale;                       // 1 / (1 - rate)
};

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

__device__ __forceinline__ uint32_t use_parity(int t) { return (uint32_t)(t >> 1) & 1u; }

// TRAIN: also the per-row log-sum-exp for the backward pass, an fp32 copy of O, and the hash dropout mask of the fp32 trainer applied to P
// before the P V product (the row sum l stays undropped, as in softmax -> dropout -> matmul).  The training instance is
// built for one CTA per SM: under the two-CTA register cap its dropout and log-sum-exp bookkeeping would spill.  The inference instance (TRAIN = false) is the
// same code without those three; the training instance with neither output and no dropout computes the same bits.
template <bool TRAIN>
__global__ void __launch_bounds__(ATTN_THREADS, TRAIN ? 1 : 2) attn_block_causal_kernel(const __grid_constant__ AttnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sQ = smem;                                    // [2][Q_BYTES]
    uint8_t* sK = sQ + 2 * Q_BYTES;
    uint8_t* sV = sK + KSTAGES * K_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + VSTAGES * V_BYTES);
    uint64_t* q_full = bars;                 // 2
    uint64_t* q_empty = q_full + 2;          // 2: the item's last Q K^T retired (every MMA thread arrives)
    uint64_t* k_full = q_empty + 2;          // KSTAGES
    uint64_t* k_empty = k_full + KSTAGES;    // KSTAGES
    uint64_t* v_full = k_empty + KSTAGES;    // VSTAGES
    uint64_t* v_empty = v_full + VSTAGES;    // VSTAGES

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_items = p.BH * p.n_qtiles;

    if (threadIdx.x == 0) {
        prefetch_tmap(&p.tmQ); prefetch_tmap(&p.tmK); prefetch_tmap(&p.tmV);
        for (int i = 0; i < 2; ++i) { mbar_init(&q_full[i], 1); mbar_init(&q_empty[i], MMA_THREADS); }
        for (int i = 0; i < KSTAGES; ++i) { mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], MMA_THREADS); }
        for (int i = 0; i < VSTAGES; ++i) { mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], MMA_THREADS); }
        mbar_fence_init();
    }
    __syncthreads();

    // Work items = (query tile, batch*head), heaviest query tiles (most visible keys) first; a CTA walks items blockIdx.x, + gridDim.x, ...
    // Every role derives the same sequence, so nothing has to be broadcast; tile counters run on across items (ring parities stay valid).
    auto item_coords = [&](int item, int& b, int& h, int& q0, int& n_kt) {
        const int qt = p.qt0 + p.n_qtiles - 1 - item / p.BH;
        const int bh = item % p.BH;
        h = bh % p.H; b = bh / p.H;
        q0 = qt * QT;
        const int last_q = min(q0 + QT, p.S) - 1;                                   // keys visible to the tile's last valid query
        const int kv_lim = min(p.S, (last_q / p.block + 1) * p.block);
        n_kt = (kv_lim + KT - 1) / KT;
        if (p.stream > 0) n_kt = q0 / KT + ((q0 + KT < p.S) ? 3 : 1);               // multi-end schedule, see tile_at
        else if (p.skip_tile >= 0 && p.skip_tile < n_kt) --n_kt;
    };
    // Key tile j of the item whose first query is q0: row of the tile in qk / V^T and which half of the 128 query rows sees it
    // (bit 0: rows 0..63, bit 1: rows 64..127).  Stream 0 (block-causal, branching_attention.py:41-61): tile j of stream 0, the masks
    // come from the per-row visibility arithmetic.  Stream s >= 1 (branching_attention.py:82-126; one view per 64-key tile): a query of
    // view t sees stream-0 keys of views < t and its own stream's keys of view t — for the tile's two views (t0, t0 + 1):
    //   stream 0, views 0 .. t0-1 (both halves) | stream 0, view t0 (upper half) | stream s, view t0 (lower half) | stream s, view t0+1 (upper)
    auto tile_at = [&](int q0, int j, int& krow, uint32_t& halves) {
        if (p.stream == 0) { krow = ((p.skip_tile >= 0 && j >= p.skip_tile) ? j + 1 : j) * KT; halves = 3u; return; }
        const int t0 = q0 / KT;
        const bool two = q0 + KT < p.S;
        if (j < t0) { krow = j * KT; halves = 3u; }
        else if (two && j == t0) { krow = t0 * KT; halves = 2u; }
        else if (j == t0 + (two ? 1 : 0)) { krow = p.stream * p.stream_rows + t0 * KT; halves = 1u; }
        else { krow = p.stream * p.stream_rows + (t0 + 1) * KT; halves = 2u; }
    };

    if (warp == MMA_THREADS / 32) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            int ks = 0, vs = 0, it = 0;
            uint32_t kph = 0, vph = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++it) {
                int b, h, q0, n_kt;
                item_coords(item, b, h, q0, n_kt);
                if (it >= 2) mbar_wait(&q_empty[it & 1], use_parity(it - 2), "vf_attn producer(Q)");
                mbar_expect_tx(&q_full[it & 1], Q_BYTES);
                tma_load_4d(sQ + (it & 1) * Q_BYTES, &p.tmQ, &q_full[it & 1], 0, p.stream * p.stream_rows + q0, h, b);
                for (int j = 0; j < n_kt; ++j) {
                    int krow;
                    uint32_t halves;
                    tile_at(q0, j, krow, halves);
                    mbar_wait(&k_empty[ks], kph ^ 1, "vf_attn producer(K)");
                    mbar_expect_tx(&k_full[ks], K_BYTES);
                    tma_load_4d(sK + ks * K_BYTES, &p.tmK, &k_full[ks], 0, krow, h, b);
                    if (++ks == KSTAGES) { ks = 0; kph ^= 1; }
                    mbar_wait(&v_empty[vs], vph ^ 1, "vf_attn producer(V)");
                    mbar_expect_tx(&v_full[vs], V_BYTES);
                    tma_load_4d(sV + vs * V_BYTES, &p.tmV, &v_full[vs], krow, h * DH, b, 0);
                    if (++vs == VSTAGES) { vs = 0; vph ^= 1; }
                }
            }
        }
        return;
    }

    // ===================== MMA + softmax + epilogue: warpgroup wg = query rows [64 wg, 64 wg + 64) of the tile =====================
    // accumulator layout (vf_wgmma.cuh): this thread holds rows r_h = 16 (warp % 4) + lane / 4 + 8 h (h = 0, 1) and, for every
    // 8-column block j, columns 8 j + 2 (lane % 4) + {0, 1}: acc[4 j + 2 h + {0, 1}]
    const int wg = warp >> 2;
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int c_ln = 2 * (lane & 3);
    int ks = 0, vs = 0, it = 0;
    uint32_t kph = 0, vph = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++it) {
        int b, h, q0, n_kt;
        item_coords(item, b, h, q0, n_kt);
        const int wq0 = q0 + 64 * wg;                       // first query of this warpgroup
        const bool wg_live = wq0 < p.S;                     // rows beyond the sequence are never stored: skip their arithmetic
        const int vis_lo = min(p.S, (min(wq0, p.S - 1) / p.block + 1) * p.block);
        const int vis_hi = min(p.S, (min(wq0 + 63, p.S - 1) / p.block + 1) * p.block);
        int vis[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) vis[hh] = min(p.S, (min(q0 + r0 + 8 * hh, p.S - 1) / p.block + 1) * p.block);
        mbar_wait(&q_full[it & 1], use_parity(it), "vf_attn mma(Q)");
        const uint64_t qdesc = sw128_desc(smem_u32(sQ + (it & 1) * Q_BYTES + wg * 64 * 128));
        float o[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = 0.f;
        float m2[2] = {-INFINITY, -INFINITY};               // reference maximum per row, in log2 units (S * log2 e)
        float l[2] = {0.f, 0.f};
        for (int j = 0; j < n_kt; ++j) {
            int kbase;
            uint32_t halves;
            tile_at(q0, j, kbase, halves);
            bool sees = wg_live && kbase < vis_hi, partial = kbase + KT > vis_lo;
            if (p.stream > 0) {                 // multi-end: whole 64-row halves see or do not see a tile, nothing is partially masked
                sees = wg_live && ((halves >> wg) & 1u) != 0;
                partial = false;
            }
            float s[32];
            mbar_wait(&k_full[ks], kph, "vf_attn mma(K)");
            if (sees) {
                const uint64_t kdesc = sw128_desc(smem_u32(sK + ks * K_BYTES));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_ss<64, BF16>(s, qdesc + 2 * k, kdesc + 2 * k, k > 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(s);
            }
            mbar_arrive(&k_empty[ks]);
            if (++ks == KSTAGES) { ks = 0; kph ^= 1; }
            mbar_wait(&v_full[vs], vph, "vf_attn mma(V)");
            if (sees) {
                if (partial) {
#pragma unroll
                    for (int i = 0; i < 32; ++i)
                        if (kbase + 8 * (i >> 2) + c_ln + (i & 1) >= vis[(i >> 1) & 1]) s[i] = -INFINITY;
                }
                uint32_t pa[4][4];
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float mx = -INFINITY;
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    const float mt = mx * LOG2E;      // log2 e > 0: the maximum commutes with the scaling
                    if (m2[hh] == -INFINITY) {
                        m2[hh] = mt;                  // first tile this row sees: nothing accumulated yet, nothing to rescale
                    } else if (mt > m2[hh] + LAZY_LOG2) {
                        const float sc = ex2(m2[hh] - mt);
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) { o[4 * jj + 2 * hh] *= sc; o[4 * jj + 2 * hh + 1] *= sc; }
                        l[hh] *= sc;
                        m2[hh] = mt;
                    }
                    const float nm = m2[hh] == -INFINITY ? 0.f : -m2[hh];
                    float ls = 0.f;
                    // dropout: element (b, h, query, column) of the fp32 trainer's [B, H, S, cols] probability tensor; cols = S (stream 0) or
                    // 2S with the stream's own keys at columns S + j
                    unsigned long long drow = 0;
                    if constexpr (TRAIN) {
                        const int cols = p.stream == 0 ? p.S : 2 * p.S;
                        const int kcol = kbase >= p.S ? kbase - (p.stream - 1) * p.stream_rows : kbase;
                        drow = ((unsigned long long)(b * p.H + h) * p.S + (q0 + r0 + 8 * hh)) * cols + kcol + c_ln;
                    }
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        float e0 = ex2(fmaf(s[4 * jj + 2 * hh], LOG2E, nm));          // exp2(-inf) = 0 for masked keys
                        float e1 = ex2(fmaf(s[4 * jj + 2 * hh + 1], LOG2E, nm));
                        ls += e0 + e1;
                        if constexpr (TRAIN) {
                            if (p.drop_thr) {
                                if (!vf_drop_keep(p.drop_seed, drow + 8 * jj, p.drop_thr)) e0 = 0.f;
                                if (!vf_drop_keep(p.drop_seed, drow + 8 * jj + 1, p.drop_thr)) e1 = 0.f;
                            }
                        }
                        // A fragment of k-step jj / 2: regs {0, 1} = rows (r0, r0 + 8) of its first 8 keys, {2, 3} of its last 8
                        pa[jj >> 1][2 * (jj & 1) + hh] = pack_bf16(e0, e1);
                    }
                    l[hh] += ls;
                }
                const uint64_t vdesc = sw128_desc(smem_u32(sV + vs * V_BYTES));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) wgmma_rs_bf16_n64(o, pa[k], vdesc + 2 * k, 1u);     // 64 keys = 4 steps of 16
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(o);
            }
            mbar_arrive(&v_empty[vs]);
            if (++vs == VSTAGES) { vs = 0; vph ^= 1; }
        }
        mbar_arrive(&q_empty[it & 1]);                      // every Q K^T of this item has retired
        // ---- epilogue: O / l -> bf16 (row sums: the 4 lanes of a row hold disjoint key columns)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            float lt = l[hh];
            lt += __shfl_xor_sync(0xffffffffu, lt, 1);
            lt += __shfl_xor_sync(0xffffffffu, lt, 2);
            const int qpos = q0 + r0 + 8 * hh;
            if (!wg_live || qpos >= p.S) continue;
            float inv;
            if constexpr (TRAIN) inv = p.drop_scale / lt;
            else inv = 1.0f / lt;
            __nv_bfloat16* orow = p.out + ((long long)b * p.S + qpos) * p.d + h * DH;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
                *reinterpret_cast<uint32_t*>(orow + 8 * jj + c_ln) = pack_bf16(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
            if constexpr (TRAIN) {
                if (p.lse) p.lse[((long long)b * p.H + h) * p.S + qpos] = (m2[hh] + log2f(lt)) * 0.69314718055994531f;
                if (p.out_f32) {
                    float* frow = p.out_f32 + ((long long)b * p.S + qpos) * p.d + h * DH;
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj)
                        *reinterpret_cast<float2*>(frow + 8 * jj + c_ln) = make_float2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
                }
            }
        }
    }
}

}  // namespace

struct AttnTrain {           // training-instance options of attn_launch (null: the inference instance)
    float* lse;
    float* out_f32;
    float rate;
    unsigned long long seed;
};
static int attn_launch(const void* qk, const void* vt, int B, int S, int n_streams, int stream, int H, int d, int block, int first_query,
                       int skip_view, void* out, vf_stream_t s, const AttnTrain* train = nullptr);

// Single-stream block-causal attention.  Only the query rows >= first_query (rounded down to a 128-row tile) are computed (0: all of
// them): with the context's q|k rows and V^T columns kept from a prefill and the query view appended behind them, this is the KV-cache
// decode step (BASELINE config 5) — the same fused kernel, no score matrix in HBM.  Rows of `out` below the first computed tile are left
// untouched.  The keys of view `skip_view` (64 tokens per view; -1: none) are never visited.  With an odd number of cached context views
// the query view would share its 128-row tile with the last context view (half of the tile's softmax work recomputes context rows nobody
// reads); leaving one slot empty puts the query view at the start of a tile.
extern "C" int vf_attn_block_causal_decode(const void* qk, const void* vt, int B, int S, int H, int d, int block, int first_query, int skip_view,
                                           void* out, vf_stream_t s) {
    VF_CHECK_ARG(skip_view < 0 || block == KT, "vf_attn_block_causal_decode: skipping a view needs 64 tokens per view (block=%d)", block);
    return attn_launch(qk, vt, B, S, 1, 0, H, d, block, first_query, skip_view, out, s);
}

// Branching (multi-end) attention, branching_attention.py:82-126: qk [B, n_streams * S, 2d] and V^T [B, d, n_streams * S] hold the streams
// side by side.  stream = 0: block-causal attention of stream 0 over its own keys (the first S rows of each batch element);
// stream = s >= 1: a query of view t of stream s attends to the stream-0 keys of views < t and to the stream-s keys of view t, one joint
// softmax.  out [B * S, d] receives that stream's attention output.  Streams >= 1 need block == 64 (one view per key tile).
extern "C" int vf_attn_block_multiend(const void* qk, const void* vt, int B, int S, int n_streams, int stream, int H, int d, int block,
                                      void* out, vf_stream_t s) {
    VF_CHECK_ARG(n_streams >= 1 && stream >= 0 && stream < n_streams, "vf_attn_block_multiend: stream %d of %d", stream, n_streams);
    VF_CHECK_ARG(stream == 0 || (block == KT && S % KT == 0), "vf_attn_block_multiend: streams >= 1 need 64 tokens per view (block=%d S=%d)", block, S);
    return attn_launch(qk, vt, B, S, n_streams, stream, H, d, block, 0, -1, out, s);
}

// Training forward of one stream of the multi-end attention: vf_attn_block_multiend plus the per-row log-sum-exp (nullable lse [B, H, S]),
// an fp32 copy of O (nullable out_f32 [B*S, d]) and inverted dropout of the probabilities with vf_dropout's mask of this stream's
// [B, H, S, cols] tensor (seed as for vf_dropout; rate 0: none).
extern "C" int vf_attn_multiend_train(const void* qk, const void* vt, int B, int S, int n_streams, int stream, int H, int d, int block, float rate,
                                      uint64_t seed, float* lse, float* out_f32, void* out, vf_stream_t s) {
    VF_CHECK_ARG(n_streams >= 1 && stream >= 0 && stream < n_streams, "vf_attn_multiend_train: stream %d of %d", stream, n_streams);
    VF_CHECK_ARG(stream == 0 || (block == KT && S % KT == 0), "vf_attn_multiend_train: streams >= 1 need 64 tokens per view (block=%d S=%d)", block, S);
    VF_CHECK_ARG(rate >= 0.f && rate < 1.f, "vf_attn_multiend_train: dropout rate %g", (double)rate);
    const AttnTrain tr{lse, out_f32, rate, (unsigned long long)seed};
    return attn_launch(qk, vt, B, S, n_streams, stream, H, d, block, 0, -1, out, s, &tr);
}

static int attn_launch(const void* qk, const void* vt, int B, int S, int n_streams, int stream, int H, int d, int block, int first_query,
                       int skip_view, void* out, vf_stream_t s, const AttnTrain* train) {
    VF_CHECK_ARG(qk && vt && out, "vf_attn_block_causal: null pointer");
    VF_CHECK_ARG(first_query >= 0 && first_query < S, "vf_attn_block_causal: first_query out of range");
    VF_CHECK_ARG(H > 0 && d == H * DH, "vf_attn_block_causal: head dim must be 64 (d=%d H=%d)", d, H);
    VF_CHECK_ARG(block > 0 && S % block == 0 && S % 8 == 0, "vf_attn_block_causal: S=%d must be a multiple of block=%d and of 8", S, block);
    if (B == 0 || S == 0) return VF_OK;
    AttnParams prm;
    memset(&prm, 0, sizeof(prm));
    prm.S = S; prm.H = H; prm.d = d; prm.block = block; prm.BH = B * H;
    prm.stream = stream; prm.stream_rows = S; prm.skip_tile = skip_view;
    const uint64_t rows_all = (uint64_t)n_streams * S;          // rows of qk / columns of V^T per batch element (all streams)
    prm.qt0 = first_query / QT;
    prm.n_qtiles = (S + QT - 1) / QT - prm.qt0;
    prm.out = reinterpret_cast<__nv_bfloat16*>(out);
    prm.drop_scale = 1.0f;
    if (train) {
        prm.lse = train->lse;
        prm.out_f32 = train->out_f32;
        prm.drop_seed = train->seed;
        prm.drop_thr = vf_drop_threshold(train->rate);
        prm.drop_scale = 1.0f / (1.0f - train->rate);
    }
    int rc;
    const uint64_t row = (uint64_t)2 * d * 2;                  // bytes per qk row
    {   // Q / K: [B, S, 2d] viewed as (dh, S, H, B); K is the second half of every row
        const uint64_t dims[4] = {(uint64_t)DH, rows_all, (uint64_t)H, (uint64_t)B};
        const uint64_t str[3] = {row, (uint64_t)DH * 2, row * rows_all};
        const uint32_t boxq[4] = {(uint32_t)DH, (uint32_t)QT, 1, 1};
        const uint32_t boxk[4] = {(uint32_t)DH, (uint32_t)KT, 1, 1};
        if ((rc = make_tmap_16bit(&prm.tmQ, qk, dims, str, boxq)) != VF_OK) return rc;
        if ((rc = make_tmap_16bit(&prm.tmK, reinterpret_cast<const __nv_bfloat16*>(qk) + d, dims, str, boxk)) != VF_OK) return rc;
    }
    {   // V^T: [B, d, S] viewed as (S, d, B, 1); one box = 64 keys x 64 dh rows
        const uint64_t dims[4] = {rows_all, (uint64_t)d, (uint64_t)B, 1};
        const uint64_t str[3] = {rows_all * 2, rows_all * 2 * d, rows_all * 2 * d * B};
        const uint32_t box[4] = {(uint32_t)KT, (uint32_t)DH, 1, 1};
        if ((rc = make_tmap_16bit(&prm.tmV, vt, dims, str, box)) != VF_OK) return rc;
    }
    constexpr int smem = 2 * Q_BYTES + KSTAGES * K_BYTES + VSTAGES * V_BYTES + 1024 + 256;     // ~90 KB: two CTAs per SM
    static vf_per_device_flag configured_pd[2];       // function attributes are per device and per instance
    bool& configured = configured_pd[train ? 1 : 0].current();
    auto kernel = train ? attn_block_causal_kernel<true> : attn_block_causal_kernel<false>;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        if (e != cudaSuccess) { vf_set_error("vf_attn: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
        configured = true;
    }
    const long long items = (long long)B * H * prm.n_qtiles;
    VF_CHECK_ARG(items < (1ll << 31), "vf_attn_block_causal: too many work items");
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || num_sms <= 0) num_sms = 132;
    }
    // persistent: two CTAs per SM (one for the training instance), every CTA walks items blockIdx.x, blockIdx.x + gridDim.x, ...
    const long long resident = (train ? 1ll : 2ll) * num_sms;
    const unsigned grid = (unsigned)(items < resident ? items : resident);
    kernel<<<grid, ATTN_THREADS, smem, vf_s(s)>>>(prm);
    VF_CHECK_LAUNCH("vf_attn_block_causal");
    return VF_OK;
}

// ===================================================================================================================================
// Fused multi-end attention backward (bf16 training step).  One CTA = the 64 keys of one view of one key stream, one (batch, head):
// dK and dV of those keys stay in registers while the CTA walks every query view of every stream that sees them
//   key stream 0, view v:  stream-0 queries of views v .. T-1 (block-causal) and stream-s queries (s >= 1) of views v+1 .. T-1
//   key stream s >= 1, view v:  stream-s queries of view v only
// and per (query stream, query view) step, with the 64 x 64 tiles in shared memory and four warps of 16 query rows:
//   S = Q K^T,  P = exp(S - lse) (recomputed from the forward pass's log-sum-exp),  dP = dO V^T,
//   Pd = P * mask / (1 - rate),  dS = P * (dP * mask / (1 - rate) - D),  D = rowsum(dO * O)
//   dQ += dS K        (fp32 atomics into the caller-zeroed q columns: query rows get gradient from several key CTAs)
//   dV += Pd^T dO,  dK += dS^T Q   (each warp 16 keys; stored once at the end, the CTA owns those rows)
// The mask is the forward pass's: element (b, h, query, column) of the fp32 trainer's [B, H, S, cols] probability tensor of the query stream.
// Every MMA is a bf16 mma.sync m16n8k16 with fp32 accumulation, operands read with ldmatrix (.trans for the transposed products).
// Nothing of size S x S reaches global memory.
namespace {

constexpr int BW_THREADS = 128;
constexpr int BW_LD = 72;                      // shared tile row pitch in bf16 (144 bytes: conflict-free ldmatrix rows)
constexpr int BW_TILE = 64 * BW_LD;

struct AttnBwdParams {
    const __nv_bfloat16* qk;                   // [B, ns*S, 2d] (q | k), as in the forward pass
    const __nv_bfloat16* vt;                   // [B, d, ns*S]
    const __nv_bfloat16* dout;                 // [ns, B*S, d]
    const float* out;                          // [ns, B*S, d] forward outputs O
    const float* lse;                          // [ns, B, H, S]
    float* dvqk;                               // [ns, B*S, 3d] columns v | q | k
    int B, S, H, d, ns, T;
    unsigned long long seed0;                  // query stream qs uses seed0 + qs
    uint32_t drop_thr;
    float drop_scale;
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const __nv_bfloat16* ptr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(ptr)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const __nv_bfloat16* ptr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(ptr)));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// acc[8][4] (16 rows x 64 columns, m16n8 fragments) += A[16 x 64] B[64 x 64] over 4 k-steps of 16.
//   A_T = false: A row-major [m][k] at a (rows m0..m0+15);  true: A stored transposed [k][m] at a (columns m0..m0+15)
//   B_T = false: B stored [n][k] (rows = output columns);   true: B stored [k][n]
template <bool A_T, bool B_T>
__device__ __forceinline__ void mma_16x64x64(float (&acc)[8][4], const __nv_bfloat16* a, int m0, const __nv_bfloat16* b, int lane) {
    const int rr = lane & 7, i = lane >> 3;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        uint32_t af[4];
        if (A_T) ldsm_x4_t(af, a + (16 * kk + rr + 8 * (i >> 1)) * BW_LD + m0 + 8 * (i & 1));
        else ldsm_x4(af, a + (m0 + rr + 8 * (i & 1)) * BW_LD + 16 * kk + 8 * (i >> 1));
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
            uint32_t bf[4];
            if (B_T) ldsm_x4_t(bf, b + (16 * kk + rr + 8 * (i & 1)) * BW_LD + 16 * nb + 8 * (i >> 1));
            else ldsm_x4(bf, b + (16 * nb + rr + 8 * (i >> 1)) * BW_LD + 16 * kk + 8 * (i & 1));
            mma_bf16(acc[2 * nb], af, bf[0], bf[1]);
            mma_bf16(acc[2 * nb + 1], af, bf[2], bf[3]);
        }
    }
}

// 64 rows x 64 bf16 from global (row stride ld elements) into a shared tile: 16-byte vectors, 4 per thread
__device__ __forceinline__ void load_tile(__nv_bfloat16* dst, const __nv_bfloat16* src, long long ld) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int v = threadIdx.x + BW_THREADS * it, r = v >> 3, c = (v & 7) * 8;
        *reinterpret_cast<uint4*>(dst + r * BW_LD + c) = __ldg(reinterpret_cast<const uint4*>(src + r * ld + c));
    }
}

__global__ void __launch_bounds__(BW_THREADS) attn_multiend_bwd_kernel(const __grid_constant__ AttnBwdParams p) {
    extern __shared__ __align__(16) uint8_t bw_smem[];
    __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(bw_smem);   // [key][dh]
    __nv_bfloat16* sVt = sK + BW_TILE;                                 // [dh][key]
    __nv_bfloat16* sQ = sVt + BW_TILE;                                 // [query][dh]
    __nv_bfloat16* sdO = sQ + BW_TILE;                                 // [query][dh]
    __nv_bfloat16* sP = sdO + BW_TILE;                                 // [query][key]  dropped P
    __nv_bfloat16* sdS = sP + BW_TILE;                                 // [query][key]
    float* sLse = reinterpret_cast<float*>(sdS + BW_TILE);             // [64] log2 units
    float* sD = sLse + 64;                                             // [64]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = p.S, T = p.T, d = p.d, H = p.H;
    // work unit: heaviest (stream-0 keys of early views) first
    const int BH = p.B * H;
    const int unit = blockIdx.x / BH, bh = blockIdx.x % BH;
    const int b = bh / H, h = bh % H;
    const int ks = unit < T ? 0 : 1 + (unit - T) / T;
    const int kv = unit < T ? unit : (unit - T) % T;
    const long long rows_all = (long long)p.ns * S;
    const int krow = ks * S + kv * 64;                                 // key rows in qk / columns in V^T
    load_tile(sK, p.qk + ((long long)b * rows_all + krow) * 2 * d + d + h * DH, 2 * d);
    load_tile(sVt, p.vt + ((long long)b * d + h * DH) * rows_all + krow, rows_all);
    const int n0 = ks == 0 ? T - kv : 1;                               // query views of stream 0 (or the one step of a stream-s key tile)
    const int n1 = ks == 0 ? T - 1 - kv : 0;                           // query views of every stream s >= 1
    const int steps = n0 + (p.ns - 1) * n1;

    float dv[8][4], dk[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) { dv[j][e] = 0.f; dk[j][e] = 0.f; }

    const int rq = 16 * warp + (lane >> 2);                            // this thread's first query row / key row in the tile
    const int c2 = 2 * (lane & 3);
    for (int st = 0; st < steps; ++st) {
        int qs, qv;
        if (ks > 0) { qs = ks; qv = kv; }
        else if (st < n0) { qs = 0; qv = kv + st; }
        else { qs = 1 + (st - n0) / n1; qv = kv + 1 + (st - n0) % n1; }
        const long long qrow = (long long)b * S + qv * 64;            // row of the query view in [B*S, .] stream tensors
        __syncthreads();                                               // the previous step is done with sQ / sdO / sP / sdS
        load_tile(sQ, p.qk + ((long long)b * rows_all + qs * S + qv * 64) * 2 * d + h * DH, 2 * d);
        load_tile(sdO, p.dout + ((long long)qs * p.B * S + qrow) * d + h * DH, d);
        {   // lse (log2 units) and D = rowsum(dO * O): two threads per row, 32 columns each
            const int r = threadIdx.x >> 1, c0 = (threadIdx.x & 1) * 32;
            const long long g = ((long long)qs * p.B * S + qrow + r) * d + h * DH + c0;
            const __nv_bfloat16* dor = p.dout + g;
            const float* orow = p.out + g;
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 32; c += 2) {
                const float2 o2 = __ldg(reinterpret_cast<const float2*>(orow + c));
                const float2 d2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(dor + c));
                acc = fmaf(d2.x, o2.x, fmaf(d2.y, o2.y, acc));
            }
            acc += __shfl_xor_sync(0xffffffffu, acc, 1);
            if ((threadIdx.x & 1) == 0) {
                sD[r] = acc;
                sLse[r] = __ldg(p.lse + (((long long)qs * p.B + b) * H + h) * S + qv * 64 + r) * LOG2E;
            }
        }
        __syncthreads();
        // ---- per warp: 16 query rows x 64 keys
        float sc[8][4], dp[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) { sc[j][e] = 0.f; dp[j][e] = 0.f; }
        mma_16x64x64<false, false>(sc, sQ, 16 * warp, sK, lane);      // S = Q K^T   (K stored [key][dh] = [n][k])
        mma_16x64x64<false, true>(dp, sdO, 16 * warp, sVt, lane);     // dP = dO V^T (V^T stored [dh][key] = [k][n])
        const int cols = qs == 0 ? S : 2 * S;
        const int kcol = (ks == 0 ? 0 : S) + kv * 64;                  // column of key 0 of the tile in the query stream's P
        const unsigned long long seed = p.seed0 + (unsigned long long)qs;
        uint32_t dsa[4][4];                                            // dS as A fragments (16 rows x 64 keys) for dQ = dS K
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = rq + 8 * hh;
            const float lse2 = sLse[r], Dr = sD[r];
            const unsigned long long drow = ((unsigned long long)(b * H + h) * S + qv * 64 + r) * cols + kcol + c2;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float pe[2], ds[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pr = ex2(fmaf(sc[j][2 * hh + e], LOG2E, -lse2));
                    float g = dp[j][2 * hh + e], pd = pr;
                    if (p.drop_thr) {
                        const bool keep = vf_drop_keep(seed, drow + 8 * j + e, p.drop_thr);
                        pd = keep ? pr * p.drop_scale : 0.f;
                        g = keep ? g * p.drop_scale : 0.f;
                    }
                    pe[e] = pd;
                    ds[e] = pr * (g - Dr);
                }
                const uint32_t pp = pack_bf16(pe[0], pe[1]), dd = pack_bf16(ds[0], ds[1]);
                *reinterpret_cast<uint32_t*>(sP + r * BW_LD + 8 * j + c2) = pp;
                *reinterpret_cast<uint32_t*>(sdS + r * BW_LD + 8 * j + c2) = dd;
                dsa[j >> 1][2 * (j & 1) + hh] = dd;
            }
        }
        {   // dQ (16 rows x 64 dh) = dS K: A from registers, B = K stored [key][dh] = [k][n]
            float dq[8][4];
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) dq[j][e] = 0.f;
            const int rr = lane & 7, i = lane >> 3;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
                for (int nb = 0; nb < 4; ++nb) {
                    uint32_t bf[4];
                    ldsm_x4_t(bf, sK + (16 * kk + rr + 8 * (i & 1)) * BW_LD + 16 * nb + 8 * (i >> 1));
                    mma_bf16(dq[2 * nb], dsa[kk], bf[0], bf[1]);
                    mma_bf16(dq[2 * nb + 1], dsa[kk], bf[2], bf[3]);
                }
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float* g = p.dvqk + ((long long)qs * p.B * S + qrow + rq + 8 * hh) * 3 * d + d + h * DH + c2;
#pragma unroll
                for (int j = 0; j < 8; ++j) atomicAdd(reinterpret_cast<float2*>(g + 8 * j), make_float2(dq[j][2 * hh], dq[j][2 * hh + 1]));
            }
        }
        __syncthreads();                                               // sP / sdS complete
        // ---- per warp: keys 16 warp .. 16 warp + 15
        mma_16x64x64<true, true>(dv, sP, 16 * warp, sdO, lane);       // dV += Pd^T dO (Pd stored [q][key] = [k][m], dO [q][dh] = [k][n])
        mma_16x64x64<true, true>(dk, sdS, 16 * warp, sQ, lane);       // dK += dS^T Q
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        float* g = p.dvqk + ((long long)ks * p.B * S + (long long)b * S + kv * 64 + rq + 8 * hh) * 3 * d + h * DH + c2;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            *reinterpret_cast<float2*>(g + 8 * j) = make_float2(dv[j][2 * hh], dv[j][2 * hh + 1]);
            *reinterpret_cast<float2*>(g + 2 * d + 8 * j) = make_float2(dk[j][2 * hh], dk[j][2 * hh + 1]);
        }
    }
}

}  // namespace

// Backward of the multi-end attention of all streams (see attn_multiend_bwd_kernel): qk / vt as in the forward pass, dout bf16 [ns, B*S, d],
// out fp32 [ns, B*S, d] and lse [ns, B, H, S] from vf_attn_multiend_train, dropout (rate, seed of stream 0; stream s uses seed + s) as there.
// dvqk fp32 [ns, B*S, 3d] (columns v | q | k per stream, the layout of the c_attn output): the caller zeroes it; the v and k columns are
// written, the q columns accumulated.  Needs head dim 64 and 64 tokens per view.
extern "C" int vf_attn_multiend_bwd(const void* qk, const void* vt, const void* dout, const float* out, const float* lse, int B, int S, int n_streams,
                                    int H, int d, int block, float rate, uint64_t seed, float* dvqk, vf_stream_t s) {
    VF_CHECK_ARG(qk && vt && dout && out && lse && dvqk, "vf_attn_multiend_bwd: null pointer");
    VF_CHECK_ARG(H > 0 && d == H * DH, "vf_attn_multiend_bwd: head dim must be 64 (d=%d H=%d)", d, H);
    VF_CHECK_ARG(block == KT && S > 0 && S % KT == 0 && n_streams >= 1 && n_streams <= 3, "vf_attn_multiend_bwd: needs 64 tokens per view (block=%d S=%d ns=%d)",
                 block, S, n_streams);
    VF_CHECK_ARG(rate >= 0.f && rate < 1.f, "vf_attn_multiend_bwd: dropout rate %g", (double)rate);
    if (B == 0) return VF_OK;
    AttnBwdParams prm;
    prm.qk = reinterpret_cast<const __nv_bfloat16*>(qk);
    prm.vt = reinterpret_cast<const __nv_bfloat16*>(vt);
    prm.dout = reinterpret_cast<const __nv_bfloat16*>(dout);
    prm.out = out; prm.lse = lse; prm.dvqk = dvqk;
    prm.B = B; prm.S = S; prm.H = H; prm.d = d; prm.ns = n_streams; prm.T = S / KT;
    prm.seed0 = (unsigned long long)seed;
    prm.drop_thr = vf_drop_threshold(rate);
    prm.drop_scale = 1.0f / (1.0f - rate);
    const long long ctas = (long long)n_streams * prm.T * B * H;
    VF_CHECK_ARG(ctas < (1ll << 31), "vf_attn_multiend_bwd: too many work items");
    constexpr int smem = 6 * BW_TILE * 2 + 128 * 4;
    static vf_per_device_flag configured_pd;
    bool& configured = configured_pd.current();
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(attn_multiend_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) { vf_set_error("vf_attn_multiend_bwd: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
        configured = true;
    }
    attn_multiend_bwd_kernel<<<(unsigned)ctas, BW_THREADS, smem, vf_s(s)>>>(prm);
    VF_CHECK_LAUNCH("vf_attn_multiend_bwd");
    return VF_OK;
}
