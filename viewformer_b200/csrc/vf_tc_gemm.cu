// Tensor-core GEMMs and implicit-GEMM convolutions for sm_90a (Hopper): one persistent kernel, tc_gemm_kernel, 128 x (64|128)
// output tiles: plain / batched / causal GEMMs, tap-table and halo-tile convolutions, bf16, fp16 (split-fp16 "exact" mode) and TF32.
// Structure:
//   TMA (cp.async.bulk.tensor, 128B swizzle)  ->  smem ring (mbarrier full / empty pairs)  ->  two MMA warpgroups, each issuing
//   wgmma.mma_async for 64 rows of the tile with fp32 accumulators in registers  ->  the same 8 warps as epilogue: accumulators ->
//   shared-memory staging tile -> alpha, bias, GELU, residual, GroupNorm statistics, f32/bf16 stores.
//
// Warp roles (384 threads): warps 0..7 = MMA + epilogue (warpgroup g owns tile rows [64g, 64g+64)), warps 8..11 = TMA producer
// warpgroup (one elected thread issues the loads; the warpgroup hands its registers to the MMA warpgroups).  Exact mode moves the
// epilogue's stores onto warps 9..11 of the producer warpgroup: the MMA warps write the staging tile, hand it over through an
// mbarrier pair and go straight on to the next tile's MMAs while those warps add bias and residual, store and fold the GroupNorm sums.
// Both roles run the same epilogue function, store_slice.  vf_tc_gemm_plan and vf_tc_gemm share one validation and tiling, tc_setup.
// A CTA walks 128 x BLOCK_N output tiles; the producer runs ahead across tiles, so the next tile's operands stream in while the
// epilogue of this one runs.  GEMM operands are K-major; the convolution reads its A operand straight from the NHWC activation
// tensor with a 4-D tensor map: for every filter tap the box [TN images x TH rows x TW cols x 64 channels] shifted by (dy,dx)
// lands in shared memory as a 128-row K-major tile, out-of-image pixels zero-filled by TMA — no im2col buffer exists anywhere.
//
// Replaces: torch.nn.Conv2d sites of viewformer/models/vqgan_th.py (3x3 stride-1 convs, 1x1 convs),
//           tf.matmul sites of viewformer/models/migt.py:93 (Conv1D), :54 (tied LM head) and
//           viewformer/models/branching_attention.py:7,18 (QK^T, PV) on the fast path.
#include "vf_wgmma.cuh"
#include <stdlib.h>

namespace {
using namespace vftc;

constexpr int BLOCK_M = 128;
constexpr int ROW_BYTES = 128;                 // one swizzle-128B row = one K block
constexpr int A_STAGE_BYTES = BLOCK_M * ROW_BYTES;
constexpr int NUM_EPI_WARPS = 8;               // the two MMA warpgroups; in the epilogue 2 warps per 32-row quarter of the tile
constexpr int NUM_MMA_THREADS = 32 * NUM_EPI_WARPS;
constexpr int NUM_THREADS = NUM_MMA_THREADS + 128;  // + the producer warpgroup (one elected thread issues TMA; see setmaxnreg_dec)

struct TcParams {
    CUtensorMap tmA, tmB;
    int conv;
    int M, Ncols;
    int num_k_blocks;          // total K blocks (gemm: ceil(K/BKe); conv: ntaps * cin_blocks)
    int batch2;
    int tiles_m, tiles_n, total_tiles;
    int a_bm1, a_bm2, b_bm1, b_bm2;   // 0 => operand is shared by all batches along that batch dim
    // conv tiling
    int TW, TH, TN, tiles_x, tiles_y, OH, OW, Nimg, cin_blocks, bk_elems;
    int tap_dy[9], tap_dx[9], tap_coff[9];
    int gemm_koff;             // gemm mode: tap_coff[b1] is added to the K coordinate of A for batch1 index b1 (shifted views of one operand)
    int causal_block, causal_skip_n;
    float alpha;
    const float* bias;
    int bias_mode, act;
    const float* residual;
    float* C_f32;
    __nv_bfloat16* C_bf16;
    long long ldc, c_sb1, c_sb2;
    int vec_ok;                // output/residual/bias addressing is 16-byte friendly -> vector epilogue
    int halo;                  // conv only: 1 = load one (TH+2)x(TW+2) halo tile per 64-channel block (exact: per block and half)
                               // and address the 9 taps as row-shifted wgmma descriptors into it (9x fewer A bytes from L2);
                               // 0 = one shifted TMA box per tap
    double* gn_sums;           // optional fused GroupNorm statistics of the OUTPUT: [images][groups][2] (sum, sum of squares)
    int gn_groups, gn_cpg, gn_rows_per_img;
    int exact_kc;              // k-blocks per accumulation chunk (divides ntaps * cin_blocks)
    int exact_clog;            // logical channels of the split activation tensor (= Ctot / 2): the lo half starts there
    int exact_kpp;             // k-blocks per product pass = ntaps * cin_blocks (conv) or K / 64 (gemm)
    int exact_lo_b;            // gemm only: element offset of the lo half inside a B row (exact_clog is the A side's)
    const float2* norm_mr;     // halo mode only, optional GroupNorm(+swish) of the INPUT applied to each halo tile in shared memory:
    const float* norm_gamma;   //   (mean, rstd) [N][groups], gamma / beta [Cin]
    const float* norm_beta;
    int norm_groups, norm_cpg, norm_swish;
};

// ---- exact mode (VF_F16X2 operands): fp32-faithful GEMMs and convolutions on the tensor cores ----------------------------------
// An fp32 value v travels as TWO fp16 numbers  hi = fp16(v),  lo = fp16((v - hi) * 2^11)  (22-23 significand bits; the scaling keeps
// lo out of the fp16 subnormal range), activations as [.., hi(C) | lo(C)], weights as [Cout][tap][hi(Cin) | lo(Cin)].
//   x * w  =  hi_x hi_w  +  2^-11 (hi_x lo_w + lo_x hi_w)  +  O(2^-22 |x w|)            -> three fp16 MMAs per product block
// The tensor cores add into their fp32 accumulators without round-to-nearest, so a long K loop is not fp32-faithful.  The
// accumulator is therefore drained every `exact_kc` k-blocks (a "chunk" of MMA steps from a ZERO accumulator) and the chunks are
// summed in a second register array with round-to-nearest FFMA, scaled by 2^-11 for the cross terms, small terms first.
constexpr float EXACT_LO_SCALE = 1.0f / 2048.0f;

struct TileInfo {
    int m0, n0, b1, b2, img0, oy0, ox0, nkb;
    bool skip;
};

__device__ __forceinline__ TileInfo decode_tile(const TcParams& p, int t, int block_n) {
    TileInfo ti;
    const int n_tile = t % p.tiles_n;
    const int r = t / p.tiles_n;
    const int m_tile = r % p.tiles_m;
    const int bz = r / p.tiles_m;
    ti.b1 = bz / p.batch2;
    ti.b2 = bz % p.batch2;
    ti.m0 = m_tile * BLOCK_M;
    ti.n0 = n_tile * block_n;
    ti.nkb = p.num_k_blocks;
    ti.skip = false;
    if (p.causal_block > 0) {
        const int lim = ((ti.m0 + BLOCK_M - 1) / p.causal_block + 1) * p.causal_block;   // keys visible to the tile's last row
        if (p.causal_skip_n) {
            ti.skip = ti.n0 >= lim;                                                      // whole tile masked: never read
        } else {
            const int kb = (lim + p.bk_elems - 1) / p.bk_elems;
            if (kb < ti.nkb) ti.nkb = kb;
        }
    }
    ti.img0 = ti.oy0 = ti.ox0 = 0;
    if (p.conv) {
        const int tx = m_tile % p.tiles_x;
        const int q = m_tile / p.tiles_x;
        ti.img0 = (q / p.tiles_y) * p.TN;
        ti.oy0 = (q % p.tiles_y) * p.TH;
        ti.ox0 = tx * p.TW;
    }
    return ti;
}

constexpr int HALO_BYTES = 23552;  // one (16+2) x (8+2) halo tile of 128-byte rows, rounded up to 1024
// Halo mode carves the operand region into halo buffers followed by a ring of weight-tile slots.  bf16 / TF32: 2 halo buffers
// (double-buffered over the channel blocks), 6 slots.  Exact: 4 buffers, the lo and hi halves of up to 2 channel blocks, all
// resident for the whole tile, 4 slots.
__host__ __device__ constexpr int halo_buffers(bool exact) { return exact ? 4 : 2; }
__host__ __device__ constexpr int halo_slots(bool exact) { return exact ? 4 : 6; }
__host__ __device__ constexpr int operand_bytes(int stages, int stage_bytes, int b_stage_bytes, bool exact) {
    return stages * stage_bytes > halo_buffers(exact) * HALO_BYTES + halo_slots(exact) * b_stage_bytes
               ? stages * stage_bytes
               : halo_buffers(exact) * HALO_BYTES + halo_slots(exact) * b_stage_bytes;
}
constexpr int MAX_STAGES = 8;
template <int kBlockN, int kStages, bool kExact>
__host__ __device__ constexpr int tc_smem_bytes() {
    return operand_bytes(kStages, A_STAGE_BYTES + kBlockN * ROW_BYTES, kBlockN * ROW_BYTES, kExact) +
           NUM_EPI_WARPS * 32 * (kBlockN / 2 + 4) * 4 /*epilogue staging*/ + 1024 /*align slack*/ +
           8 * (2 * MAX_STAGES + 2 * halo_buffers(kExact) + 2) /*barriers: ring, halo tiles, staging handover (exact)*/;
}

// Exact mode's staging handover: MMA warps arrive on stg_full once the tile's chunk sums are in the staging tile, the epilogue warps
// (9..11 of the producer warpgroup) on stg_empty once they have stored it.  Every thread of either side arrives.
constexpr int NUM_STORE_WARPS = 3;
static_assert(NUM_EPI_WARPS + 1 + NUM_STORE_WARPS == NUM_THREADS / 32, "warp roles");
constexpr int STORE_RES_VECS = 4;              // residual float4 loads in flight per lane of an epilogue warp (fits 80 registers)

// L2 prefetch of the residual rows a conv tile's epilogue will read: one bulk prefetch per (image, output row) of the tile, spanning
// its valid pixels from channel n0 on (the columns between the tile's channel slices ride along).
__device__ __forceinline__ void prefetch_residual_l2(const TcParams& p, const TileInfo& ti, int block_n) {
    const int tw = min(p.TW, p.OW - ti.ox0);
    const uint32_t bytes = (uint32_t)(((long long)(tw - 1) * p.ldc + block_n) * 4);
    for (int r = 0; r < p.TN * p.TH; ++r) {
        const int img = ti.img0 + r / p.TH, oy = ti.oy0 + r % p.TH;
        if (img >= p.Nimg || oy >= p.OH) continue;
        const float* src = p.residual + ((long long)(img * p.OH + oy) * p.OW + ti.ox0) * p.ldc + ti.n0;
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
    }
}

// Normalise-on-load: GroupNorm (+ swish) of the raw halo tile of channel block cb, in place, by the 256 MMA threads.  The tile holds
// (TH+2) x (TW+2) rows (pixels) of 64 bf16 channels, 128B-swizzled: physical 16-byte chunk pc of row r holds logical chunk
// pc ^ (r & 7) (the buffers are 1024-byte aligned).  Rows outside the image were zero-filled by TMA and stay zero (the reference
// pads AFTER norm + swish, vqgan_th.py:69-78).  Same arithmetic as vf_groupnorm_apply, so the operand is bit-identical.
__device__ __forceinline__ void normalise_halo(const TcParams& p, uint8_t* tile, int cb, int img, int oy0, int ox0, int tid) {
    const int rows = (p.TW + 2) * (p.TH + 2);
    for (int idx = tid; idx < rows * 8; idx += NUM_MMA_THREADS) {
        const int r = idx >> 3, pc = idx & 7;
        const int py = r / (p.TW + 2), px = r - py * (p.TW + 2);
        const int iy = oy0 - 1 + py, ix = ox0 - 1 + px;
        if (iy < 0 || iy >= p.OH || ix < 0 || ix >= p.OW) continue;
        const int c0 = cb * 64 + ((pc ^ (r & 7)) << 3);                  // first of the chunk's 8 channels
        uint4* ptr = reinterpret_cast<uint4*>(tile + r * ROW_BYTES + pc * 16);
        const uint4 v = *ptr;
        uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = c0 + 2 * k;
            const float2 ma = __ldg(p.norm_mr + (img * p.norm_groups + c / p.norm_cpg));
            const float2 mb = __ldg(p.norm_mr + (img * p.norm_groups + (c + 1) / p.norm_cpg));
            const float sa = ma.y * __ldg(p.norm_gamma + c), sb = mb.y * __ldg(p.norm_gamma + c + 1);
            float a = __uint_as_float(w[k] << 16), b = __uint_as_float(w[k] & 0xffff0000u);
            a = fmaf(a, sa, __ldg(p.norm_beta + c) - ma.x * sa);
            b = fmaf(b, sb, __ldg(p.norm_beta + c + 1) - mb.x * sb);
            if (p.norm_swish == 1) {          // same arithmetic as vf_groupnorm_apply (bit-identical operand)
                a = __fdividef(a, 1.0f + __expf(-a));
                b = __fdividef(b, 1.0f + __expf(-b));
            }
            __nv_bfloat162 o = __floats2bfloat162_rn(a, b);
            w[k] = *reinterpret_cast<uint32_t*>(&o);
            if (p.norm_swish == 2) {
                // packed bf16: swish(y) = h * (1 + tanh(h)), h = y / 2 — ONE MUFU op per two elements instead of four
                uint32_t h, th;
                asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(h) : "r"(w[k]), "r"(0x3f003f00u));
                asm("tanh.approx.bf16x2 %0, %1;" : "=r"(th) : "r"(h));
                asm("fma.rn.bf16x2 %0, %1, %2, %1;" : "=r"(w[k]) : "r"(h), "r"(th));
            }
        }
        *ptr = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

// ---- epilogue: one 32-row x HALF_N slice of the staging tile -> bias, GELU, residual, f32 / bf16 stores, GroupNorm statistics ----
// Slice s = quarter + 4 col_half holds tile rows [32 quarter, +32) and columns [HALF_N col_half, +HALF_N).  In the bf16 / TF32
// instances MMA warp s stores slice s; in exact mode epilogue warp e (9..11) stores slices e, e + 3, e + 6.  Both run store_slice, so
// exact mode keeps the lanes' rows and columns, the arithmetic order and the GroupNorm shuffle tree of the other instances.
// Vector path geometry: VPR float4 vectors span a slice row, a warp covers RPI rows per iteration, ITERS iterations.
template <int kBlockN>
struct EpiGeom {
    static constexpr int HALF_N = kBlockN / 2, STG_LD = HALF_N + 4, VPR = HALF_N / 4, RPI = 32 / VPR, ITERS = 32 / RPI;
};

// Row bookkeeping: lane l owns tile row 32 quarter + l; the other lanes of the warp read it with shuffles.
struct EpiLane {
    long long off;      // the row's element offset in C and in the residual
    int ok, gm;         // the row lies inside the output; its global row (GEMM) or pixel (conv)
    float bias_m;       // VF_BIAS_M: the row's bias
};

__device__ __forceinline__ EpiLane epi_lane(const TcParams& p, const TileInfo& ti, int quarter, int lane) {
    const int row = quarter * 32 + lane;
    long long off;
    int ok, gm;
    if (p.conv) {
        const int lx = row % p.TW;
        const int q = row / p.TW;
        const int ly = q % p.TH;
        const int ln = q / p.TH;
        const int img = ti.img0 + ln, oy = ti.oy0 + ly, ox = ti.ox0 + lx;
        ok = (img < p.Nimg) && (oy < p.OH) && (ox < p.OW);
        gm = (img * p.OH + oy) * p.OW + ox;
        off = (long long)gm * p.ldc;
    } else {
        gm = ti.m0 + row;
        ok = gm < p.M;
        off = (long long)ti.b1 * p.c_sb1 + (long long)ti.b2 * p.c_sb2 + (long long)gm * p.ldc;
    }
    const float bias_m = (p.bias_mode == VF_BIAS_M && ok) ? __ldg(p.bias + gm) : 0.f;
    return {off, ok, gm, bias_m};
}

// The vector path's residual float4 of slice row rr at column n_ln.  Unconditional (out-of-range rows read row 0 and are never
// stored): a predicated load would make the compiler funnel a batch of loads through one temporary and serialise their latencies.
__device__ __forceinline__ float4 residual_vec(const TcParams& p, const EpiLane& el, int rr, int n_ln) {
    const int ok = __shfl_sync(0xffffffffu, el.ok, rr);
    const long long off_row = __shfl_sync(0xffffffffu, el.off, rr);
    return __ldg(reinterpret_cast<const float4*>(p.residual + (ok ? off_row + n_ln : (long long)n_ln)));
}

// stg: the slice, [32][STG_LD].  fast: the vector path (full-width tile, 16-byte aligned rows), whose VF_BIAS_N bias (bias4) and
// residual (resv) each role loads on its own schedule.  The bf16 / TF32 MMA warps pass all three in, the residual as all ITERS vectors
// loaded into registers before their K loop, so the DRAM latency hides under the tile's MMAs.  Exact mode's epilogue warps have 80
// registers: they pass nothing, and store_slice computes them here, the residual from L2 (the producer prefetched it) STORE_RES_VECS
// vectors at a time.
template <int kBlockN, bool kExact>
__device__ __forceinline__ void store_slice(const TcParams& p, const TileInfo& ti, const EpiLane& el, const float* stg, int col_half,
                                            int lane, bool fast, float4 bias4, const float4* resv) {
    using G = EpiGeom<kBlockN>;
    constexpr int RB = kExact ? STORE_RES_VECS : G::ITERS;     // residual vectors per batch
    static_assert(G::ITERS % RB == 0, "residual batches");
    const int r_sub = lane / G::VPR;
    const int c_ln = (lane % G::VPR) * 4;         // column inside the slice
    const int n_ln = ti.n0 + col_half * G::HALF_N + c_ln;
    if constexpr (kExact) fast = p.vec_ok && (ti.n0 + kBlockN <= p.Ncols);
    if (fast) {
        if constexpr (kExact) {
            bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.bias_mode == VF_BIAS_N) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + n_ln));
        }
        float gs = 0.f, gq = 0.f;                 // fused GroupNorm statistics of this lane's 4 channels
#pragma unroll 1
        for (int i0 = 0; i0 < G::ITERS; i0 += RB) {
            float4 resb[RB];
            if (kExact && p.residual) {
#pragma unroll
                for (int k = 0; k < RB; ++k) resb[k] = residual_vec(p, el, (i0 + k) * G::RPI + r_sub, n_ln);
            }
#pragma unroll
            for (int k = 0; k < RB; ++k) {
                const int rr = (i0 + k) * G::RPI + r_sub;
                const int ok = __shfl_sync(0xffffffffu, el.ok, rr);
                const long long off_row = __shfl_sync(0xffffffffu, el.off, rr);
                const float bm = __shfl_sync(0xffffffffu, el.bias_m, rr);
                float4 v = *reinterpret_cast<const float4*>(stg + rr * G::STG_LD + c_ln);
                if (p.bias_mode == VF_BIAS_N) { v.x += bias4.x; v.y += bias4.y; v.z += bias4.z; v.w += bias4.w; }
                else { v.x += bm; v.y += bm; v.z += bm; v.w += bm; }
                if (p.act == VF_ACT_GELU_ERF) { v.x = vf_gelu_erf(v.x); v.y = vf_gelu_erf(v.y); v.z = vf_gelu_erf(v.z); v.w = vf_gelu_erf(v.w); }
                if (p.residual) {
                    const float4 r = kExact ? resb[k] : resv[i0 + k];
                    v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
                }
                if (ok) {
                    gs += (v.x + v.y) + (v.z + v.w);
                    // the GroupNorm partials (recorded for exact mode in tests/golden/exact_conv_bits.json) are this rounding; written
                    // out, so that which product the compiler would fuse into the add cannot change it
                    gq += __fmaf_rn(v.y, v.y, __fmul_rn(v.x, v.x)) + __fmaf_rn(v.w, v.w, __fmul_rn(v.z, v.z));
                    const long long off = off_row + n_ln;
                    if (p.C_f32) *reinterpret_cast<float4*>(p.C_f32 + off) = v;
                    if (p.C_bf16) {
                        __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
                        uint2 u;
                        u.x = *reinterpret_cast<uint32_t*>(&lo);
                        u.y = *reinterpret_cast<uint32_t*>(&hi);
                        *reinterpret_cast<uint2*>(p.C_bf16 + off) = u;
                    }
                }
            }
        }
        if (p.gn_sums) {
            // the 32 rows of a slice lie in one image; lanes with equal column vector (different r_sub) and the cpg/4 neighbouring
            // lanes of a group are folded with shuffles, then one fp64 RED per (image, group)
            const unsigned okmask = __ballot_sync(0xffffffffu, el.ok);
#pragma unroll
            for (int o = G::VPR; o < 32; o <<= 1) {
                gs += __shfl_xor_sync(0xffffffffu, gs, o);
                gq += __shfl_xor_sync(0xffffffffu, gq, o);
            }
            const int lpg = p.gn_cpg >> 2;
            for (int o = 1; o < lpg; o <<= 1) {
                gs += __shfl_xor_sync(0xffffffffu, gs, o);
                gq += __shfl_xor_sync(0xffffffffu, gq, o);
            }
            const int gm_first = __shfl_sync(0xffffffffu, el.gm, okmask ? (__ffs(okmask) - 1) : 0);
            if (okmask && r_sub == 0 && (lane % lpg) == 0) {
                const long long slot = ((long long)(gm_first / p.gn_rows_per_img) * p.gn_groups + n_ln / p.gn_cpg) * 2;
                atomicAdd(p.gn_sums + slot, (double)gs);
                atomicAdd(p.gn_sums + slot + 1, (double)gq);
            }
        }
    } else {
        // generic path (N tails, unaligned leading dimensions): scalar, same arithmetic order
#pragma unroll 1
        for (int rr = 0; rr < 32; ++rr) {
            const int ok = __shfl_sync(0xffffffffu, el.ok, rr);
            const long long off_row = __shfl_sync(0xffffffffu, el.off, rr);
            const float bm = __shfl_sync(0xffffffffu, el.bias_m, rr);
            if (!ok) continue;
            for (int c = lane; c < G::HALF_N; c += 32) {
                const int n = ti.n0 + col_half * G::HALF_N + c;
                if (n >= p.Ncols) continue;
                float x = stg[rr * G::STG_LD + c];
                x += (p.bias_mode == VF_BIAS_N) ? __ldg(p.bias + n) : bm;
                if (p.act == VF_ACT_GELU_ERF) x = vf_gelu_erf(x);
                const long long off = off_row + n;
                if (p.residual) x += __ldg(p.residual + off);
                if (p.C_f32) p.C_f32[off] = x;
                if (p.C_bf16) p.C_bf16[off] = __float2bfloat16(x);
            }
        }
    }
}

// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles t = blockIdx.x, +gridDim.x, ...
template <int kBlockN, int kStages, WgKind kKind>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_gemm_kernel(const __grid_constant__ TcParams p) {
    constexpr int B_STAGE_BYTES = kBlockN * ROW_BYTES;
    constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
    constexpr int K_STEPS = 4;                 // MMA steps per 128-byte K block: 16 bf16/fp16 or 8 tf32 elements (32 bytes) each
    constexpr int HALF_N = kBlockN / 2;        // columns per epilogue warp
    constexpr int STG_LD = HALF_N + 4;         // staging row stride (floats): +4 keeps 128-bit row reads conflict-free
    constexpr int STG_BYTES = NUM_EPI_WARPS * 32 * STG_LD * 4;
    constexpr int NACC = kBlockN / 2;          // accumulator registers per thread (64 rows x kBlockN per warpgroup)
    constexpr bool kExact = kKind == F16;      // fp16 operands are always split-fp16 pairs (VF_F16X2)

    extern __shared__ uint8_t smem_raw[];
    // 1024B alignment required by the 128B swizzle atoms
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int OPER_BYTES = operand_bytes(kStages, STAGE_BYTES, B_STAGE_BYTES, kExact);
    float* staging = reinterpret_cast<float*>(smem + OPER_BYTES);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OPER_BYTES + STG_BYTES);   // [MAX_STAGES]
    uint64_t* empty_bar = full_bar + MAX_STAGES;        // [MAX_STAGES]
    constexpr int NHB = halo_buffers(kExact);
    uint64_t* a_full_bar = empty_bar + MAX_STAGES;      // [NHB]  halo mode: A halo tiles
    uint64_t* a_empty_bar = a_full_bar + NHB;           // [NHB]
    uint64_t* stg_full = a_empty_bar + NHB;             // exact mode: staging tile written (MMA warps -> epilogue warps)
    uint64_t* stg_empty = stg_full + 1;                 //             staging tile stored  (epilogue warps -> MMA warps)
    constexpr int NG = kStages;                         // ring depth (normal mode)
    // halo mode carves the same operand region differently: NHB halo buffers, then a ring of B-only slots
    constexpr int NGH = halo_slots(kExact);
    uint8_t* halo_b_base = smem + NHB * HALO_BYTES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        prefetch_tmap(&p.tmA);
        prefetch_tmap(&p.tmB);
        for (int s = 0; s < MAX_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], NUM_MMA_THREADS);     // every MMA thread arrives once its wgmma reading the slot retired
        }
        for (int a = 0; a < NHB; ++a) {
            mbar_init(&a_full_bar[a], 1);
            mbar_init(&a_empty_bar[a], NUM_MMA_THREADS);
        }
        if constexpr (kExact) {
            mbar_init(stg_full, NUM_MMA_THREADS);
            mbar_init(stg_empty, 32 * NUM_STORE_WARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp >= NUM_EPI_WARPS) {
        // ===================== TMA producer (warp 8), exact mode's epilogue (warps 9..11) =====================
        setmaxnreg_dec<kExact ? 80 : 40>();           // 208 x 256 + 80 x 128 <= 64K (exact), 232 x 256 + 40 x 128 (bf16 / TF32)
        if constexpr (kExact) {
            if (warp > NUM_EPI_WARPS) {
                // every role walks the same tiles; epilogue warp e stores staging slices e, e + 3, e + 6
                const int e = warp - NUM_EPI_WARPS - 1;
                uint32_t spar = 0;
                for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
                    const TileInfo ti = decode_tile(p, t, kBlockN);
                    if (ti.skip) continue;
                    mbar_wait(stg_full, spar, "vf_tc_gemm epilogue");      // spans one K loop: well under a millisecond
#pragma unroll 1
                    for (int s = e; s < NUM_EPI_WARPS; s += NUM_STORE_WARPS)
                        store_slice<kBlockN, true>(p, ti, epi_lane(p, ti, s & 3, lane), staging + s * (32 * STG_LD), s >> 2, lane,
                                                   false, float4(), nullptr);
                    mbar_arrive(stg_empty);
                    spar ^= 1;
                }
                return;
            }
        }
        if (warp == NUM_EPI_WARPS && elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            int ab = 0;
            uint32_t aphase = 0, tpar = 0;
            for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, tpar ^= 1) {
                const TileInfo ti = decode_tile(p, t, kBlockN);
                if (ti.skip) continue;
                const uint32_t halo_bytes = (uint32_t)((p.TW + 2) * (p.TH + 2)) * ROW_BYTES;
                if (kExact && p.halo) {
                    // Halo buffer 2 h + cb holds half h (0 = lo, 1 = hi) of channel block cb and is loaded once per tile.  The lo
                    // halves are read by product pass 0 only, so they load first; the hi halves, still read by the previous
                    // tile's last pass when this tile starts, load NGH k-blocks into pass 0.
                    auto load_halves = [&](int h) {
                        for (int cb = 0; cb < p.cin_blocks; ++cb) {
                            const int hb = 2 * h + cb;
                            mbar_wait(&a_empty_bar[hb], tpar ^ 1, "vf_tc_gemm producer(halo)");
                            mbar_expect_tx(&a_full_bar[hb], halo_bytes);
                            tma_load_4d(smem + hb * HALO_BYTES, &p.tmA, &a_full_bar[hb], (h ? 0 : p.exact_clog) + cb * p.bk_elems,
                                        ti.ox0 - 1, ti.oy0 - 1, ti.img0);
                        }
                    };
                    load_halves(0);
                    if (p.residual && p.vec_ok && ti.n0 + kBlockN <= p.Ncols) prefetch_residual_l2(p, ti, kBlockN);
                    int j = 0, tap = 0, cb = 0;     // the tap-box walk: product pass, tap, channel block
                    for (int kb = 0; kb < ti.nkb; ++kb) {
                        if (kb == NGH) load_halves(1);
                        mbar_wait(&empty_bar[stage], phase ^ 1, "vf_tc_gemm producer");
                        mbar_expect_tx(&full_bar[stage], (uint32_t)B_STAGE_BYTES);
                        tma_load_4d(halo_b_base + stage * B_STAGE_BYTES, &p.tmB, &full_bar[stage],
                                    ((tap * 2 + (j == 1 ? 1 : 0)) * p.cin_blocks + cb) * p.bk_elems, ti.n0, 0, 0);
                        if (++cb == p.cin_blocks) { cb = 0; if (++tap == 9) { tap = 0; ++j; } }
                        if (++stage == NGH) { stage = 0; phase ^= 1; }
                    }
                    continue;
                }
                if (p.halo) {
                    const int nkb = 9 * p.cin_blocks;
                    int tap = 0, cb = 0;
                    for (int kb = 0; kb < nkb; ++kb) {
                        mbar_wait(&empty_bar[stage], phase ^ 1, "vf_tc_gemm producer");
                        mbar_expect_tx(&full_bar[stage], (uint32_t)B_STAGE_BYTES);
                        if (tap == 0) {      // first tap of a channel block: its halo tile
                            mbar_wait(&a_empty_bar[ab], aphase ^ 1, "vf_tc_gemm producer(halo)");
                            mbar_expect_tx(&a_full_bar[ab], halo_bytes);
                            tma_load_4d(smem + ab * HALO_BYTES, &p.tmA, &a_full_bar[ab], cb * p.bk_elems, ti.ox0 - 1, ti.oy0 - 1, ti.img0);
                            if (++ab == 2) { ab = 0; aphase ^= 1; }
                        }
                        tma_load_4d(halo_b_base + stage * B_STAGE_BYTES, &p.tmB, &full_bar[stage], (tap * p.cin_blocks + cb) * p.bk_elems,
                                    ti.n0, 0, 0);
                        if (++tap == 9) { tap = 0; ++cb; }
                        if (++stage == NGH) { stage = 0; phase ^= 1; }
                    }
                    continue;
                }
                if constexpr (kExact) {
                    // tap-box convs and GEMMs: product pass j (0 = (lo_x, hi_w), 1 = (hi_x, lo_w), 2 = (hi_x, hi_w)), k-block kbr of
                    // the pass, for a conv its tap and channel block cb.  Walked by counters: the ring is 4 k-blocks deep, so the one
                    // producer thread's latency per k-block (divisions, dependent constant loads) would show in the MMA rate.
                    if (p.conv && p.residual && p.vec_ok && ti.n0 + kBlockN <= p.Ncols) prefetch_residual_l2(p, ti, kBlockN);
                    int j = 0, kbr = 0, tap = 0, cb = 0;
                    for (int kb = 0; kb < ti.nkb; ++kb) {
                        mbar_wait(&empty_bar[stage], phase ^ 1, "vf_tc_gemm producer");
                        mbar_expect_tx(&full_bar[stage], (uint32_t)STAGE_BYTES);
                        uint8_t* sa = smem + stage * STAGE_BYTES;
                        uint8_t* sb = sa + A_STAGE_BYTES;
                        if (p.conv) {
                            tma_load_4d(sa, &p.tmA, &full_bar[stage], (j == 0 ? p.exact_clog : 0) + p.tap_coff[tap] + cb * p.bk_elems,
                                        ti.ox0 + p.tap_dx[tap], ti.oy0 + p.tap_dy[tap], ti.img0);
                            tma_load_4d(sb, &p.tmB, &full_bar[stage], ((tap * 2 + (j == 1 ? 1 : 0)) * p.cin_blocks + cb) * p.bk_elems,
                                        ti.n0, 0, 0);
                        } else {
                            const int kcoord_a = (j == 0 ? p.exact_clog : 0) + kbr * p.bk_elems + (p.gemm_koff ? p.tap_coff[ti.b1] : 0);
                            tma_load_4d(sa, &p.tmA, &full_bar[stage], kcoord_a, ti.m0, ti.b2 * p.a_bm2, ti.b1 * p.a_bm1);
                            tma_load_4d(sb, &p.tmB, &full_bar[stage], (j == 1 ? p.exact_lo_b : 0) + kbr * p.bk_elems, ti.n0,
                                        ti.b2 * p.b_bm2, ti.b1 * p.b_bm1);
                        }
                        if (++kbr == p.exact_kpp) { kbr = tap = cb = 0; ++j; }
                        else if (++cb == p.cin_blocks) { cb = 0; ++tap; }
                        if (++stage == NG) { stage = 0; phase ^= 1; }
                    }
                } else {
                    for (int kb = 0; kb < ti.nkb; ++kb) {
                        mbar_wait(&empty_bar[stage], phase ^ 1, "vf_tc_gemm producer");
                        mbar_expect_tx(&full_bar[stage], (uint32_t)STAGE_BYTES);
                        uint8_t* sa = smem + stage * STAGE_BYTES;
                        uint8_t* sb = sa + A_STAGE_BYTES;
                        if (p.conv) {
                            const int tap = kb / p.cin_blocks;
                            const int cb = kb - tap * p.cin_blocks;
                            tma_load_4d(sa, &p.tmA, &full_bar[stage], p.tap_coff[tap] + cb * p.bk_elems, ti.ox0 + p.tap_dx[tap],
                                        ti.oy0 + p.tap_dy[tap], ti.img0);
                        } else {
                            int kcoord_a = kb * p.bk_elems;
                            if (p.gemm_koff) kcoord_a += p.tap_coff[ti.b1];
                            tma_load_4d(sa, &p.tmA, &full_bar[stage], kcoord_a, ti.m0, ti.b2 * p.a_bm2, ti.b1 * p.a_bm1);
                        }
                        tma_load_4d(sb, &p.tmB, &full_bar[stage], kb * p.bk_elems, ti.n0, ti.b2 * p.b_bm2, ti.b1 * p.b_bm1);
                        if (++stage == NG) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        return;
    }

    // ===================== MMA + epilogue (warps 0..7; exact mode: MMA and staging only) =====================
    setmaxnreg_inc<kExact ? 208 : 232>();       // exact: the chunk sums, no epilogue state
    const int wg = warp >> 2;                          // MMA: warpgroup wg computes tile rows [64 wg, 64 wg + 64)
    const int quarter = warp & 3;                      // epilogue: this warp stores tile rows [32 quarter, +32) ...
    const int col_half = warp >> 2;                    // ... of column half col_half
    float* stg = staging + warp * (32 * STG_LD);       // the epilogue's staging tile of this warp [32][STG_LD]
    int stage = 0, ab = 0;
    uint32_t phase = 0, aphase = 0, tpar = 0, spar = 0;

    // fragment -> staging: element (r, c) of the 128 x kBlockN tile goes to the staging slice of the warp that stores it (slice
    // quarter + 4 col_half: MMA+epilogue warp of that number, or in exact mode the epilogue warp that takes it).
    // Exact halo mode with 16 x 8-pixel tiles: MMA row group g of warpgroup wg is image row g, columns [8 wg, 8 wg + 8), stored as
    // tile row 16 g + 8 wg + i, so that every epilogue warp sums the same pixels as on the tap-box path (same GroupNorm partials).
    const bool col_split = kExact && p.halo && p.TW == 16;
    auto to_staging = [&](const float (&v)[NACC], float sc) {
        const int r_lo = 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
        for (int j = 0; j < NACC / 4; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = col_split ? 16 * (2 * (warp & 3) + h) + 8 * wg + (lane >> 2) : r_lo + 8 * h;
                const int c = 8 * j + 2 * (lane & 3);
                float* dst = staging + ((c / HALF_N) * 4 + (r >> 5)) * (32 * STG_LD) + (r & 31) * STG_LD + (c % HALF_N);
                *reinterpret_cast<float2*>(dst) = make_float2(v[4 * j + 2 * h] * sc, v[4 * j + 2 * h + 1] * sc);
            }
        }
    };

    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, tpar ^= 1) {
        const TileInfo ti = decode_tile(p, t, kBlockN);
        if (ti.skip) continue;

        // Declared per tile, so that neither array is live in the epilogue (every tile's first wgmma starts from a zero accumulator).
        // csum (exact mode): the running sum of the chunks in the accumulator's fragment layout, first chunk acc * sc, then
        // fma(acc, sc, csum).
        float acc[NACC];
        float csum[kExact ? NACC : 1];
        auto k_loop = [&]() {
            // ---- phase 1: K loop.  One wgmma group (4 MMA steps of one k-block) stays in flight: once the group of k-block kb is
            // issued, wait for kb-1's and hand its ring slot back to the producer.
            const int nkb = (p.halo && !kExact) ? 9 * p.cin_blocks : ti.nkb;
            const int nsmall = kExact ? 2 * p.exact_kpp / p.exact_kc : 0;      // exact mode: cross-term chunks come first
            int prev_stage = -1, prev_halo = -1, in_chunk = 0, ck = 0, tap = 0, j = 0, cb = 0;
            bool fresh = true;
            uint32_t a_base = 0;
            const uint32_t pitch = (uint32_t)(p.TW + 2);
            // halo rows between the two warpgroups' first pixels: TW = 8 -> 8 image rows apart, TW = 16 -> 8 columns apart
            const uint32_t wg_rows = p.TW == 16 ? 8u : 8u * pitch;
            auto retire_prev = [&]() {
                if (prev_stage >= 0) mbar_arrive(&empty_bar[prev_stage]);
                if (prev_halo >= 0) mbar_arrive(&a_empty_bar[prev_halo]);
                prev_stage = prev_halo = -1;
            };
#pragma unroll 1
            for (int kb = 0; kb < nkb; ++kb) {
                uint64_t adesc, bdesc;
                int this_halo = (p.halo && tap == 8) ? ab : -1;
                if (kExact && p.halo) {
                    // the tap-box walk (pass j, tap, channel block cb) over the resident halo tiles: pass 0 reads the lo halves
                    // (buffers 0, 1), passes 1 and 2 the hi halves (buffers 2, 3); a buffer is released after its last read
                    const int hb = (j == 0 ? 0 : 2) + cb;
                    if (tap == 0 && j < 2) mbar_wait(&a_full_bar[hb], tpar, "vf_tc_gemm mma(halo)");
                    this_halo = (tap == 8 && j != 1) ? hb : -1;
                    mbar_wait(&full_bar[stage], phase, "vf_tc_gemm mma");
                    const uint32_t a_addr = smem_u32(smem + hb * HALO_BYTES) +
                                            ((uint32_t)(tap / 3) * pitch + (uint32_t)(tap % 3) + (uint32_t)wg * wg_rows) * ROW_BYTES;
                    adesc = sw128_desc(a_addr, pitch * ROW_BYTES);
                    bdesc = sw128_desc(smem_u32(halo_b_base + stage * B_STAGE_BYTES));
                } else if (p.halo) {
                    // tile = TH rows of TW=8 pixels: MMA row group g (8 rows) = image row g of the tile; inside the halo tile
                    // (pitch TW+2 rows) tap (dy,dx) starts (dy*(TW+2)+dx) rows in, consecutive groups are (TW+2) rows apart
                    if (tap == 0) {
                        mbar_wait(&a_full_bar[ab], aphase, "vf_tc_gemm mma(halo)");
                        a_base = smem_u32(smem + ab * HALO_BYTES);
                        if (!kExact && p.norm_mr) {  // every thread's MMAs read the whole tile: transform, then publish it to the async proxy
                            normalise_halo(p, smem + ab * HALO_BYTES, kb / 9, ti.img0, ti.oy0, ti.ox0, threadIdx.x);
                            fence_async_smem();
                            named_sync(1, NUM_MMA_THREADS);
                        }
                    }
                    mbar_wait(&full_bar[stage], phase, "vf_tc_gemm mma");
                    const uint32_t a_addr = a_base + ((uint32_t)(tap / 3) * pitch + (uint32_t)(tap % 3) + (uint32_t)(8 * wg) * pitch) * ROW_BYTES;
                    adesc = sw128_desc(a_addr, pitch * ROW_BYTES);
                    bdesc = sw128_desc(smem_u32(halo_b_base + stage * B_STAGE_BYTES));
                } else {
                    mbar_wait(&full_bar[stage], phase, "vf_tc_gemm mma");
                    const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
                    adesc = sw128_desc(sa + (uint32_t)(wg * 64 * ROW_BYTES));
                    bdesc = sw128_desc(sa + A_STAGE_BYTES);
                }
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < K_STEPS; ++k)      // +32 bytes along K inside the swizzle atom => +2 in the (addr >> 4) field
                    wgmma_ss<kBlockN, kKind>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (fresh && k == 0) ? 0u : 1u);
                wgmma_commit();
                fresh = false;
                wgmma_wait<1>();
                retire_prev();
                prev_stage = stage;
                prev_halo = this_halo;
                if (kExact && p.halo) {
                    if (++stage == NGH) { stage = 0; phase ^= 1; }
                    if (++cb == p.cin_blocks) { cb = 0; if (++tap == 9) { tap = 0; ++j; } }
                } else if (p.halo) {
                    if (++stage == NGH) { stage = 0; phase ^= 1; }
                    if (++tap == 9) { tap = 0; if (++ab == 2) { ab = 0; aphase ^= 1; } }
                } else {
                    if (++stage == NG) { stage = 0; phase ^= 1; }
                }
                if (kExact && ++in_chunk == p.exact_kc) {
                    // chunk complete: fold it into the running sum with round-to-nearest FFMA, restart from a zero accumulator
                    in_chunk = 0;
                    wgmma_wait<0>();
                    reg_fence(acc);
                    const float sc = (ck < nsmall ? EXACT_LO_SCALE : 1.0f) * p.alpha;
                    if (ck == 0) {
#pragma unroll
                        for (int i = 0; i < NACC; ++i) csum[i] = acc[i] * sc;
                    } else {
#pragma unroll
                        for (int i = 0; i < NACC; ++i) csum[i] = fmaf(acc[i], sc, csum[i]);
                    }
                    ++ck;
                    fresh = true;
                }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            retire_prev();
        };
        if constexpr (kExact) {
            // hand the chunk sums over to the epilogue warps and go straight on to the next tile
            k_loop();
            mbar_wait(stg_empty, spar ^ 1, "vf_tc_gemm mma(staging)");    // the epilogue warps have stored the previous tile
            to_staging(csum, 1.0f);
            mbar_arrive(stg_full);
            spar ^= 1;
            continue;
        }

        // vector path: the bias and the whole residual of this warp's slice go into registers BEFORE the K loop, so their DRAM latency
        // hides behind this tile's MMAs
        using G = EpiGeom<kBlockN>;
        const EpiLane el = epi_lane(p, ti, quarter, lane);
        const int n_ln = ti.n0 + col_half * HALF_N + (lane % G::VPR) * 4;
        const bool fast = p.vec_ok && (ti.n0 + kBlockN <= p.Ncols);
        float4 resv[G::ITERS];
        if (fast && p.residual) {
#pragma unroll
            for (int i = 0; i < G::ITERS; ++i) resv[i] = residual_vec(p, el, i * G::RPI + lane / G::VPR, n_ln);
        }
        float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (fast && p.bias_mode == VF_BIAS_N) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + n_ln));

        k_loop();
        named_sync(1, NUM_MMA_THREADS);                           // the previous tile's epilogue is done with the staging tile
        to_staging(acc, p.alpha);
        named_sync(1, NUM_MMA_THREADS);                           // staging tile complete
        store_slice<kBlockN, false>(p, ti, el, stg, col_half, lane, fast, bias4, resv);
    }
}

// 4-D tensor map, dims innermost first, 128B swizzle, zero OOB fill.  strides[i] = byte stride of dim i+1.
int make_tmap(CUtensorMap* tm, int dtype, const void* base, const uint64_t dims[4], const uint64_t strides_bytes[3],
              const uint32_t box[4]) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) { vf_set_error("vf_tc_gemm: cuTensorMapEncodeTiled unavailable"); return VF_ERR_CUDA; }
    cuuint64_t gdim[4] = {dims[0], dims[1], dims[2], dims[3]};
    cuuint64_t gstr[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
    cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = fn(tm, dtype == VF_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
                    const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        vf_set_error("vf_tc_gemm: cuTensorMapEncodeTiled failed (%d): dims=[%llu,%llu,%llu,%llu] strides=[%llu,%llu,%llu] box=[%u,%u,%u,%u]",
                     (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
                     (unsigned long long)dims[3], (unsigned long long)strides_bytes[0], (unsigned long long)strides_bytes[1],
                     (unsigned long long)strides_bytes[2], box[0], box[1], box[2], box[3]);
        return VF_ERR_CUDA;
    }
    return VF_OK;
}

template <int kBlockN, int kStages, WgKind kKind>
int launch(const TcParams& prm, dim3 grid, cudaStream_t st) {
    constexpr int smem = tc_smem_bytes<kBlockN, kStages, kKind == F16>();
    static_assert(kStages <= MAX_STAGES, "ring depth");
    static_assert(smem <= 232448, "shared memory budget");
    static vf_per_device_flag configured_pd;          // function attributes are per device
    bool& configured = configured_pd.current();
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(tc_gemm_kernel<kBlockN, kStages, kKind>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) { vf_set_error("vf_tc_gemm: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
        configured = true;
    }
    tc_gemm_kernel<kBlockN, kStages, kKind><<<grid, NUM_THREADS, smem, st>>>(prm);
    VF_CHECK_LAUNCH("vf_tc_gemm");
    return VF_OK;
}

template <int kBlockN, int kStages>
int launch_kind(const TcParams& prm, WgKind kind, dim3 grid, cudaStream_t st) {
    if (kind == TF32) return launch<kBlockN, kStages, TF32>(prm, grid, st);
    if (kind == F16) return launch<kBlockN, kStages, F16>(prm, grid, st);
    return launch<kBlockN, kStages, BF16>(prm, grid, st);
}

// Output tile of a convolution, TN images x TH rows x TW cols = 128 pixels, and whether it takes the halo path (returned).
bool conv_tiling(const vf_tc_gemm_t* q, bool exact, int bk, int* TWo, int* THo, int* TNo) {
    int TW = q->OW >= 16 ? 16 : (q->OW >= 8 ? 8 : (q->OW >= 4 ? 4 : (q->OW >= 2 ? 2 : 1)));
    int TH = 128 / TW;
    if (TH > q->OH) { TH = 1; while (TH * 2 <= q->OH) TH *= 2; }
    int TN = 128 / (TW * TH);
    // halo mode: plain stride-1 pad-1 3x3 conv on maps at least 16 rows tall -> 8x16-pixel tiles, one halo load per channel block.
    // Exact mode: one halo per channel block and half, all resident for the tile (so at most 2 channel blocks), on the tap-box
    // path's own 16x8 or 8x16 tiles, which keeps the fused GroupNorm partial sums of each epilogue warp.
    bool halo = q->ntaps == 9 && q->OH == q->H && q->OW == q->W &&
                (exact ? q->Ctot == 2 * q->Cin && q->Cin <= 2 * bk && TN == 1 && TW >= 8
                       : q->Ctot == q->Cin && q->OH >= 16 && q->OW >= 8);
    for (int t = 0; halo && t < 9; ++t) halo = q->tap_dy[t] == t / 3 - 1 && q->tap_dx[t] == t % 3 - 1 && q->tap_coff[t] == 0;
    if (halo && !exact) { TW = 8; TH = 16; TN = 1; }
    *TWo = TW; *THo = TH; *TNo = TN;
    return halo;
}

// Persistent CTAs of a launch: one per SM (the device's count, read once).
int persistent_ctas() {
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || num_sms <= 0) num_sms = 132;
    }
    return num_sms;
}

// Validates a parameter block and fills the kernel parameters that decide the tile walk: shapes, tiling, tile counts, the epilogue
// and normalise-on-load options, block_n and the persistent CTA count.  vf_tc_gemm_plan reports from it and vf_tc_gemm launches it,
// so the plan is the launch's tiling; vf_tc_gemm adds the tensor maps, vec_ok and the GroupNorm sums.
int tc_setup(const vf_tc_gemm_t* q, TcParams& prm, int& block_n, int& ctas) {
    VF_CHECK_ARG(q->A && q->B, "vf_tc_gemm: null operand");
    VF_CHECK_ARG(q->C_f32 || q->C_bf16, "vf_tc_gemm: no output");
    VF_CHECK_ARG(q->ab_dtype == VF_BF16 || q->ab_dtype == VF_F32 || q->ab_dtype == VF_F16X2, "vf_tc_gemm: bad dtype");
    const bool exact = q->ab_dtype == VF_F16X2;
    if (exact) {
        VF_CHECK_ARG(q->C_f32 && !q->C_bf16 && !q->norm_mean_rstd && q->causal_block == 0,
                     "vf_tc_gemm: VF_F16X2 (exact split-fp16) operands need an fp32 output and no causal / fused-norm options");
        if (q->conv) VF_CHECK_ARG(q->Ctot % 2 == 0 && q->alpha == 1.0f, "vf_tc_gemm: exact conv needs [hi | lo] channels and alpha = 1");
        else VF_CHECK_ARG(q->K % 64 == 0 && q->exact_lo_a >= q->K && q->exact_lo_b >= q->K && q->exact_lo_a % 8 == 0 && q->exact_lo_b % 8 == 0,
                          "vf_tc_gemm: exact GEMM needs K %% 64 == 0 and lo-half offsets >= K (K=%d lo_a=%lld lo_b=%lld)", q->K,
                          (long long)q->exact_lo_a, (long long)q->exact_lo_b);
    }
    VF_CHECK_ARG(q->bias_mode == VF_BIAS_NONE || q->bias, "vf_tc_gemm: bias pointer missing");
    VF_CHECK_ARG(!q->norm_mean_rstd || q->conv, "vf_tc_gemm: fused input GroupNorm is a convolution option");
    const int es = q->ab_dtype == VF_F32 ? 4 : 2;
    const int bk = ROW_BYTES / es;                       // K elements per block: 64 bf16 / 32 tf32

    memset(&prm, 0, sizeof(prm));
    prm.conv = q->conv;
    prm.Ncols = q->Ncols;
    prm.bk_elems = bk;
    prm.alpha = q->alpha;
    prm.bias = q->bias;
    prm.bias_mode = q->bias_mode;
    prm.act = q->act;
    prm.residual = q->residual;
    prm.C_f32 = q->C_f32;
    prm.C_bf16 = reinterpret_cast<__nv_bfloat16*>(q->C_bf16);
    prm.ldc = q->ldc;
    prm.causal_block = q->causal_block;
    prm.causal_skip_n = q->causal_skip_n;

    // N tile: 128 when the problem is wide enough, else 64 (fewer wasted MMA columns and accumulator registers)
    block_n = (q->Ncols > 64) ? 128 : 64;
    dim3 grid;
    if (q->conv) {
        VF_CHECK_ARG(q->ntaps >= 1 && q->ntaps <= 9 && q->OW > 0 && q->OH > 0 && q->N > 0, "vf_tc_gemm: conv shape");
        VF_CHECK_ARG(q->Cin % bk == 0 && q->Ctot % (16 / es) == 0, "vf_tc_gemm: conv Cin=%d must be a multiple of %d", q->Cin, bk);
        VF_CHECK_ARG(q->causal_block == 0, "vf_tc_gemm: causal with conv");
        int TW, TH, TN;
        const bool halo = conv_tiling(q, exact, bk, &TW, &TH, &TN);
        prm.halo = halo ? 1 : 0;
        if (q->norm_mean_rstd) {
            VF_CHECK_ARG(halo && q->ab_dtype == VF_BF16 && q->H >= 32 && q->Ncols % 128 == 0 && q->Cin % 64 == 0,
                         "vf_tc_gemm: fused input GroupNorm needs a 3x3 stride-1 bf16 conv on a map >= 32 rows (Cin %% 64 == 0, Cout %% 128 == 0)");
            VF_CHECK_ARG(q->norm_gamma && q->norm_beta && q->norm_groups > 0 && q->Cin % q->norm_groups == 0,
                         "vf_tc_gemm: fused input GroupNorm needs gamma, beta and a group count dividing Cin");
            prm.norm_mr = reinterpret_cast<const float2*>(q->norm_mean_rstd);
            prm.norm_gamma = q->norm_gamma;
            prm.norm_beta = q->norm_beta;
            prm.norm_groups = q->norm_groups;
            prm.norm_cpg = q->Cin / q->norm_groups;
            prm.norm_swish = q->norm_swish;
        }
        VF_CHECK_ARG(TW * TH * TN == 128 && TN <= 256, "vf_tc_gemm: cannot tile %dx%d output", q->OH, q->OW);
        prm.TW = TW; prm.TH = TH; prm.TN = TN;
        prm.tiles_x = (q->OW + TW - 1) / TW;
        prm.tiles_y = (q->OH + TH - 1) / TH;
        prm.OH = q->OH; prm.OW = q->OW; prm.Nimg = q->N;
        prm.cin_blocks = q->Cin / bk;
        prm.num_k_blocks = q->ntaps * prm.cin_blocks;
        if (exact) {
            prm.exact_kpp = prm.num_k_blocks;
            prm.exact_clog = q->Ctot / 2;
            prm.exact_kc = (prm.num_k_blocks % 3 == 0) ? 3 : 1;      // k-blocks (= 4 MMA steps each) per accumulation chunk
            prm.num_k_blocks *= 3;
        }
        prm.M = q->N * q->OH * q->OW;
        prm.batch2 = 1;
        for (int t = 0; t < q->ntaps; ++t) { prm.tap_dy[t] = q->tap_dy[t]; prm.tap_dx[t] = q->tap_dx[t]; prm.tap_coff[t] = q->tap_coff[t]; }
        const int ntiles_img = (q->N + TN - 1) / TN;
        grid = dim3(prm.tiles_x * prm.tiles_y * ntiles_img, (q->Ncols + block_n - 1) / block_n, 1);
    } else {
        VF_CHECK_ARG(q->M > 0 && q->Ncols > 0 && q->K > 0 && q->batch1 > 0 && q->batch2 > 0, "vf_tc_gemm: bad shape");
        VF_CHECK_ARG((q->lda * es) % 16 == 0 && (q->ldb * es) % 16 == 0, "vf_tc_gemm: row strides must be 16-byte multiples");
        VF_CHECK_ARG((q->a_sb1 * es) % 16 == 0 && (q->a_sb2 * es) % 16 == 0 && (q->b_sb1 * es) % 16 == 0 && (q->b_sb2 * es) % 16 == 0,
                     "vf_tc_gemm: batch strides must be 16-byte multiples");
        VF_CHECK_ARG(q->causal_block == 0 || (q->causal_block % bk == 0 || bk % q->causal_block == 0), "vf_tc_gemm: causal block");
        prm.M = q->M;
        prm.batch2 = q->batch2;
        prm.num_k_blocks = (q->K + bk - 1) / bk;
        if (exact) {
            prm.exact_kpp = prm.num_k_blocks;
            prm.exact_clog = (int)q->exact_lo_a;
            prm.exact_lo_b = (int)q->exact_lo_b;
            prm.exact_kc = prm.exact_kpp % 4 == 0 ? 4 : (prm.exact_kpp % 3 == 0 ? 3 : (prm.exact_kpp % 2 == 0 ? 2 : 1));
            prm.num_k_blocks *= 3;
        }
        prm.c_sb1 = q->c_sb1; prm.c_sb2 = q->c_sb2;
        // ntaps > 0 in gemm mode: batch1 index b reads A shifted by tap_coff[b] >= 0 elements along K (one operand, several shifted
        // views — the weight gradient of a 3x3 convolution over a transposed, zero-padded activation: vf_conv_wgrad_tc)
        if (q->ntaps > 0) {
            VF_CHECK_ARG(q->ntaps == q->batch1 && q->ntaps <= 9, "vf_tc_gemm: gemm K offsets need ntaps == batch1 <= 9");
            prm.gemm_koff = 1;
            for (int t = 0; t < q->ntaps; ++t) {
                VF_CHECK_ARG(q->tap_coff[t] >= 0 && q->tap_coff[t] % 8 == 0, "vf_tc_gemm: K offsets must be non-negative multiples of 8 (16-byte TMA box starts)");
                prm.tap_coff[t] = q->tap_coff[t];
            }
        }
        // an operand with batch stride 0 is shared by every batch: its tensor map gets a size-1 batch dim and the
        // kernel multiplies the batch coordinate by 0
        prm.a_bm1 = (q->batch1 > 1 && q->a_sb1 != 0) ? 1 : 0;
        prm.a_bm2 = (q->batch2 > 1 && q->a_sb2 != 0) ? 1 : 0;
        prm.b_bm1 = (q->batch1 > 1 && q->b_sb1 != 0) ? 1 : 0;
        prm.b_bm2 = (q->batch2 > 1 && q->b_sb2 != 0) ? 1 : 0;
        grid = dim3((q->M + BLOCK_M - 1) / BLOCK_M, (q->Ncols + block_n - 1) / block_n, q->batch1 * q->batch2);
    }
    // persistent launch: `grid` is the tile space (m tiles, n tiles, batches); one CTA per SM walks it, n fastest
    prm.tiles_m = (int)grid.x;
    prm.tiles_n = (int)grid.y;
    const long long total = (long long)prm.tiles_m * grid.y * grid.z;
    VF_CHECK_ARG(total > 0 && total < (1ll << 31), "vf_tc_gemm: tile count out of range");
    prm.total_tiles = (int)total;
    const int num_sms = persistent_ctas();
    ctas = (int)(total < num_sms ? total : num_sms);
    return VF_OK;
}

}  // namespace

extern "C" int vf_tc_gemm_plan(const vf_tc_gemm_t* q, int* plan) {
    VF_CHECK_ARG(q && plan, "vf_tc_gemm_plan: null argument");
    TcParams prm;
    int block_n, ctas, rc;
    if ((rc = tc_setup(q, prm, block_n, ctas)) != VF_OK) return rc;
    const int vals[8] = {block_n, prm.TW, prm.TH, prm.TN, prm.halo, q->ab_dtype == VF_F16X2 ? 1 : 0, prm.total_tiles, ctas};
    for (int i = 0; i < 8; ++i) plan[i] = vals[i];
    return VF_OK;
}

extern "C" int vf_tc_gemm(const vf_tc_gemm_t* q, vf_stream_t s) {
    VF_CHECK_ARG(q, "vf_tc_gemm: null argument");
    TcParams prm;
    int block_n, ctas, rc;
    if ((rc = tc_setup(q, prm, block_n, ctas)) != VF_OK) return rc;
    const bool exact = q->ab_dtype == VF_F16X2;
    const bool tf32 = q->ab_dtype == VF_F32;
    const int tm_dtype = tf32 ? VF_F32 : VF_BF16;        // tensor-map element type (fp16 and bf16 move identically)
    const int es = tf32 ? 4 : 2;
    const int bk = prm.bk_elems;
    if (q->conv) {
        const bool halo = prm.halo;
        const uint64_t dimsA[4] = {(uint64_t)q->Ctot, (uint64_t)q->W, (uint64_t)q->H, (uint64_t)q->N};
        const uint64_t strA[3] = {(uint64_t)q->Ctot * es, (uint64_t)q->W * q->Ctot * es, (uint64_t)q->H * q->W * q->Ctot * es};
        const uint32_t boxA[4] = {(uint32_t)bk, (uint32_t)(halo ? prm.TW + 2 : prm.TW), (uint32_t)(halo ? prm.TH + 2 : prm.TH), (uint32_t)prm.TN};
        if ((rc = make_tmap(&prm.tmA, tm_dtype, q->A, dimsA, strA, boxA)) != VF_OK) return rc;
        const uint64_t Ktot = (uint64_t)q->ntaps * q->Cin * (exact ? 2 : 1);
        const uint64_t dimsB[4] = {Ktot, (uint64_t)q->Ncols, 1, 1};
        const uint64_t strB[3] = {Ktot * es, Ktot * es * q->Ncols, Ktot * es * q->Ncols};
        const uint32_t boxB[4] = {(uint32_t)bk, (uint32_t)block_n, 1, 1};
        if ((rc = make_tmap(&prm.tmB, tm_dtype, q->B, dimsB, strB, boxB)) != VF_OK) return rc;
    } else {
        long long max_koff = 0;
        for (int t = 0; t < q->ntaps; ++t) max_koff = q->tap_coff[t] > max_koff ? q->tap_coff[t] : max_koff;
        const uint64_t fbA = (uint64_t)q->lda * es * (uint64_t)q->M, fbB = (uint64_t)q->ldb * es * (uint64_t)q->Ncols;
        const uint64_t dimsA[4] = {(uint64_t)((exact ? q->exact_lo_a + q->K : q->K) + max_koff), (uint64_t)q->M, prm.a_bm2 ? (uint64_t)q->batch2 : 1, prm.a_bm1 ? (uint64_t)q->batch1 : 1};
        const uint64_t strA[3] = {(uint64_t)q->lda * es, prm.a_bm2 ? (uint64_t)q->a_sb2 * es : fbA, prm.a_bm1 ? (uint64_t)q->a_sb1 * es : fbA};
        const uint32_t boxA[4] = {(uint32_t)bk, (uint32_t)BLOCK_M, 1, 1};
        if ((rc = make_tmap(&prm.tmA, tm_dtype, q->A, dimsA, strA, boxA)) != VF_OK) return rc;
        const uint64_t dimsB[4] = {(uint64_t)(exact ? q->exact_lo_b + q->K : q->K), (uint64_t)q->Ncols, prm.b_bm2 ? (uint64_t)q->batch2 : 1, prm.b_bm1 ? (uint64_t)q->batch1 : 1};
        const uint64_t strB[3] = {(uint64_t)q->ldb * es, prm.b_bm2 ? (uint64_t)q->b_sb2 * es : fbB, prm.b_bm1 ? (uint64_t)q->b_sb1 * es : fbB};
        const uint32_t boxB[4] = {(uint32_t)bk, (uint32_t)block_n, 1, 1};
        if ((rc = make_tmap(&prm.tmB, tm_dtype, q->B, dimsB, strB, boxB)) != VF_OK) return rc;
    }
    {
        auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
        auto a8 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; };
        prm.vec_ok = (q->ldc % 4 == 0) && (q->c_sb1 % 4 == 0) && (q->c_sb2 % 4 == 0) && a16(q->C_f32) && a8(q->C_bf16) && a16(q->residual) &&
                     a16(q->bias);
    }
    if (q->gn_sums) {
        const int C = q->Ncols;
        VF_CHECK_ARG(q->gn_groups > 0 && C % q->gn_groups == 0, "vf_tc_gemm: gn_groups");
        const int cpg = C / q->gn_groups;
        const long long rpi = q->conv ? (long long)q->OH * q->OW : q->gn_rows_per_img;
        const long long rows = q->conv ? (long long)q->N * q->OH * q->OW : (long long)q->M;
        VF_CHECK_ARG(cpg % 4 == 0 && cpg <= 32 && 32 % cpg == 0 && C % block_n == 0 && prm.vec_ok && rpi >= 32 && rpi % 32 == 0 &&
                         rows % rpi == 0 && (q->conv ? (prm.TW * prm.TH) % 32 == 0 : q->batch1 * q->batch2 == 1),
                     "vf_tc_gemm: fused GroupNorm statistics unsupported for this shape (C=%d groups=%d rows/img=%lld)", C, q->gn_groups, rpi);
        prm.gn_sums = q->gn_sums;
        prm.gn_groups = q->gn_groups;
        prm.gn_cpg = cpg;
        prm.gn_rows_per_img = (int)rpi;
        cudaError_t e = cudaMemsetAsync(q->gn_sums, 0, sizeof(double) * 2 * q->gn_groups * (rows / rpi), vf_s(s));
        if (e != cudaSuccess) { vf_set_error("vf_tc_gemm: memset gn_sums: %s", cudaGetErrorString(e)); return VF_ERR_CUDA; }
    }
    cudaStream_t st = vf_s(s);
    const WgKind kind = tf32 ? TF32 : (exact ? F16 : BF16);
    const dim3 pgrid((unsigned)ctas, 1, 1);
    if (block_n == 128) return launch_kind<128, 4>(prm, kind, pgrid, st);
    return launch_kind<64, 6>(prm, kind, pgrid, st);
}
