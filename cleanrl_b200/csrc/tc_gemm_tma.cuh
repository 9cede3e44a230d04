// TMA-fed wgmma GEMM (fc forward / data-gradient) and fc weight-gradient kernels + launcher.
#pragma once
#include "tc_base.cuh"

namespace b200rl {
using namespace tc;

// Plain GEMM out[M, N] = A[M, 64*nchunks] . Bw[N, 64*nchunks]^T with a fused epilogue (tc_gemm_tma: fc layer)
struct KGemmParams {
    const void* A;         // row-major bf16 [M, 64*nchunks]
    int64_t M;
    int nchunks;           // K = 64*nchunks
    const bf16* Bw;        // packed weights [N, 64*nchunks]
    int N;
    // ---- epilogue
    bf16* out;
    int ldo;
    const float* bias;
    float scale;
    int relu;
    // ReLU masks as bits, word (row * N/32 + col/32) of a dense [M, N] tensor (see WinParams)
    const uint32_t* mask_bits;   // multiply the output by the mask (data-gradient)
    uint32_t* mask_out;          // record (output > 0) (forward with relu)
    // fc data-gradient only: write dact3 on the 9x9 linear grid (out) and zero-padded 11x11 grid (out2)
    int dual_dact3;
    bf16* out2;
    // fp32 output instead of bf16 (wide heads): columns [0, ncols_f32) of out_f32 [M, ldo]; null = bf16 `out`
    float* out_f32;
    int ncols_f32;
};

// ------------------------------------------------------------------ kernel 1d: TMA-fed GEMM (fc forward / data-gradient)
// Plain row-major operands => the tiles are rectangular boxes: one thread per ring issues cp.async.bulk.tensor (TMA,
// SWIZZLE_128B) loads for the A chunk [BN x 64] and the weight chunk [BN x 64]; the hardware does the address generation,
// zero-fills out-of-range rows and signals the stage's mbarrier with complete_tx.  A tile is BN rows x BN columns (BN / 64
// m64 halves).  Warpgroups 1 and 2 take alternate tiles of the CTA (tile blockIdx.x + i * gridDim.x goes to warpgroup
// i % 2), each with its own accumulators and its own ring of STAGES stages fed by its own producer lane (lane 0 of warp 0
// / warp 1), so one warpgroup's epilogue runs under the other warpgroup's MMAs.  Every output is the same bf16 products
// summed over the same K sequence (chunks and k16 steps in order, the first MMA with scale-d = 0) as with any other
// tiling: which warpgroup or m64 half owns a row does not change its sums.
// The epilogue is per warp: a warp stages 8 of its accumulator rows at a time in shared memory (no warpgroup barrier),
// one lane per row and 32-column group applies the fp32 epilogue and packs bf16 back into the row, then the packed rows
// are stored as whole 128-byte lines, 8 lanes per line, instead of 16 bytes in each of 32 rows per warp store.
constexpr int kGemmThreads = 384;
constexpr int kGemmRegsProducer = 40, kGemmRegsMma = 232;   // setmaxnreg: the accumulators + the epilogue need > 168
static_assert(128 * kGemmRegsProducer + 256 * kGemmRegsMma <= 65536, "register budgets exceed the SM");
template <int BN>
__host__ __device__ constexpr size_t gemm_acc_bytes() { return (size_t)8 * 8 * (BN + 4) * sizeof(float); }   // 8 rows per warp

// One warpgroup's main loop over the nch K chunks of a tile: chunk j's batch of MH x 4 MMAs is one commit group, and
// chunk j-1's stage is released once chunk j has been issued (wgmma_wait<1>), so the tensor pipe does not drain between
// chunks.  The last chunk is peeled: its MMAs, the final wait and the accumulator reads then share one basic block, which
// keeps ptxas from serialising the MMAs (C7520).  nch >= 1 (launch_gemm_tma checks it).
template <int BN, int STAGES>
__device__ __forceinline__ void gemm_tile_mma(float (&d)[BN / 64][BN / 2], uint32_t ring, uint64_t* full_bar,
                                              uint64_t* empty_bar, uint32_t q0, int nch, int tid) {
    constexpr int MH = BN / 64;
    constexpr int A_BYTES = BN * 128;
    constexpr int STAGE_BYTES = A_BYTES + BN * 128;
    auto chunk = [&](int j) {
        const uint32_t q = q0 + (uint32_t)j, s = q % STAGES;
        mbar_wait(&full_bar[s], (q / STAGES) & 1);
        wgmma_fence();
        const uint32_t stage_addr = ring + s * STAGE_BYTES;
        const uint64_t b = desc_kmajor(stage_addr + A_BYTES);
#pragma unroll
        for (int h = 0; h < MH; ++h) {
            const uint64_t a = desc_kmajor(stage_addr + h * 64 * 128);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) WgmmaBf16<BN, 0, 0>::mma(d[h], a + 2 * kk, b + 2 * kk, (j | kk) != 0 ? 1u : 0u);
        }
        wgmma_commit();
    };
    for (int j = 0; j + 1 < nch; ++j) {
        chunk(j);
        wgmma_wait<1>();
        if (j > 0 && (tid & 31) == 0) mbar_arrive(&empty_bar[(q0 + (uint32_t)j - 1u) % STAGES]);
    }
    chunk(nch - 1);
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < MH; ++h) wgmma_fence_operands(d[h]);
    if ((tid & 31) == 0) {
        if (nch > 1) mbar_arrive(&empty_bar[(q0 + (uint32_t)nch - 2u) % STAGES]);
        mbar_arrive(&empty_bar[(q0 + (uint32_t)nch - 1u) % STAGES]);
    }
}

// STAGES: ring depth per consumer warpgroup
template <int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1) tc_gemm_tma(const __grid_constant__ CUtensorMap tmA,
                                                               const __grid_constant__ CUtensorMap tmB,
                                                               const KGemmParams p, int total_tiles, int ntiles_n) {
    static_assert(BN == 64 || BN == 128, "one epilogue lane per row and 32-column group of 8 rows");
    constexpr int MH = BN / 64;
    constexpr int A_BYTES = BN * 128;
    constexpr int STAGE_BYTES = A_BYTES + BN * 128;
    constexpr int LDA = BN + 4;
    constexpr int NW = BN / 32;                               // 32-column groups (mask words) per row
    constexpr int PR = BN / 8;                                // 16-byte pieces of a packed row
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[2][STAGES], empty_bar[2][STAGES];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* sAcc = reinterpret_cast<float*>(smem + (size_t)2 * STAGES * STAGE_BYTES);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nch = p.nchunks;
    if (tid == 0) {
        for (int w = 0; w < 2; ++w)
            for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[w][s], 1); mbar_init(&empty_bar[w][s], 4); }   // the ring's 4 consumer warps
        fence_barrier_init();
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
    }
    __syncthreads();

    if (warp < 4) {
        // ======================= TMA producer of ring w (warp w, lane 0): the chunks of consumer warpgroup w's tiles, in order
        setmaxnreg_dec<kGemmRegsProducer>();
        if (warp < 2 && lane == 0) {
            const int w = warp;
            uint8_t* ring = smem + (size_t)w * STAGES * STAGE_BYTES;
            uint32_t q = 0;
            for (int tile = blockIdx.x + w * gridDim.x; tile < total_tiles; tile += 2 * gridDim.x) {
                const int mt = tile / ntiles_n, n0 = (tile - mt * ntiles_n) * BN;
                for (int j = 0; j < nch; ++j, ++q) {
                    const uint32_t s = q % STAGES;
                    if (q >= (uint32_t)STAGES) mbar_wait(&empty_bar[w][s], ((q / STAGES) - 1) & 1);
                    const uint32_t dst = smem_u32(ring + (size_t)s * STAGE_BYTES);
                    mbar_arrive_expect_tx(&full_bar[w][s], STAGE_BYTES);
                    tma_load_2d(dst, &tmA, j * 64, mt * BN, &full_bar[w][s]);
                    tma_load_2d(dst + A_BYTES, &tmB, j * 64, n0, &full_bar[w][s]);
                }
            }
        }
    } else {
        setmaxnreg_inc<kGemmRegsMma>();
        const int wg = (warp - 4) >> 2, ww = (warp - 4) & 3;
        float* st = sAcc + (warp - 4) * 8 * LDA;             // this warp's 8 staged rows
        const uint32_t ring = smem_u32(smem + (size_t)wg * STAGES * STAGE_BYTES);
        const int nwords = p.N >> 5;                         // mask words per row (N is a multiple of 32)
        const int er = lane & 7, eg = lane >> 3;             // epilogue lane: row er of the 8, 32-column group eg
        uint32_t q = 0;
        for (int tile = blockIdx.x + wg * gridDim.x; tile < total_tiles; tile += 2 * gridDim.x, q += (uint32_t)nch) {
            const int mt = tile / ntiles_n, n0 = (tile - mt * ntiles_n) * BN;
            // accumulators local to the tile: carried across tiles, their copies make ptxas serialise the MMAs (C7520)
            float d[MH][BN / 2];
#pragma unroll
            for (int h = 0; h < MH; ++h)
#pragma unroll
                for (int e = 0; e < BN / 2; ++e) d[h][e] = 0.f;
            gemm_tile_mma<BN, STAGES>(d, ring, full_bar[wg], empty_bar[wg], q, nch, tid);
#pragma unroll
            for (int pass = 0; pass < 2 * MH; ++pass) {
                // rows 64 h + 16 ww + 8 hi + (0..7) of the tile: fragment elements d[h][4 j + 2 hi + 0/1]
                const int h = pass >> 1, hi = pass & 1;
                const int row0 = mt * BN + 64 * h + 16 * ww + 8 * hi;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
                    *reinterpret_cast<float2*>(st + (lane >> 2) * LDA + 8 * j + 2 * (lane & 3)) =
                        make_float2(d[h][4 * j + 2 * hi], d[h][4 * j + 2 * hi + 1]);
                __syncwarp();
                const int r = row0 + er, col = n0 + eg * 32;
                const bool live = eg < NW && r < (int)p.M && col < p.N;   // rows past M, the ragged last column tile
                int4 w[4];
                if (live) {
                    const int64_t wb = (int64_t)r * nwords + (col >> 5);
                    uint32_t v[32];
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const float4 f = *reinterpret_cast<const float4*>(st + er * LDA + eg * 32 + 4 * e);
                        v[4 * e] = __float_as_uint(f.x); v[4 * e + 1] = __float_as_uint(f.y);
                        v[4 * e + 2] = __float_as_uint(f.z); v[4 * e + 3] = __float_as_uint(f.w);
                    }
                    const uint32_t mbw = p.mask_bits != nullptr ? __ldg(p.mask_bits + wb) : 0xFFFFFFFFu;
                    if (p.bias) {
                        const float4* bp = reinterpret_cast<const float4*>(p.bias + col);
#pragma unroll
                        for (int e = 0; e < 8; ++e) {
                            const float4 bv = __ldg(bp + e);
                            v[4 * e] = __float_as_uint(fmaf(__uint_as_float(v[4 * e]), p.scale, bv.x));
                            v[4 * e + 1] = __float_as_uint(fmaf(__uint_as_float(v[4 * e + 1]), p.scale, bv.y));
                            v[4 * e + 2] = __float_as_uint(fmaf(__uint_as_float(v[4 * e + 2]), p.scale, bv.z));
                            v[4 * e + 3] = __float_as_uint(fmaf(__uint_as_float(v[4 * e + 3]), p.scale, bv.w));
                        }
                    } else {
#pragma unroll
                        for (int e = 0; e < 32; ++e) v[e] = __float_as_uint(__uint_as_float(v[e]) * p.scale);
                    }
                    if (p.relu) {
                        uint32_t bits = 0u;
#pragma unroll
                        for (int e = 0; e < 32; ++e) {
                            const bool pos = __uint_as_float(v[e]) > 0.f;
                            bits |= (pos ? 1u : 0u) << e;
                            v[e] = pos ? v[e] : 0u;
                        }
                        if (p.mask_out) p.mask_out[wb] = bits;
                    }
                    if (p.mask_bits) {
#pragma unroll
                        for (int e = 0; e < 32; ++e) if (!((mbw >> e) & 1u)) v[e] = 0u;
                    }
                    if (p.out_f32) {
                        float* dst = p.out_f32 + (int64_t)r * p.ldo + col;
#pragma unroll
                        for (int e = 0; e < 32; ++e) if (col + e < p.ncols_f32) dst[e] = __uint_as_float(v[e]);
                    }
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        w[e].x = (int)pack_bf16x2(__uint_as_float(v[8 * e]), __uint_as_float(v[8 * e + 1]));
                        w[e].y = (int)pack_bf16x2(__uint_as_float(v[8 * e + 2]), __uint_as_float(v[8 * e + 3]));
                        w[e].z = (int)pack_bf16x2(__uint_as_float(v[8 * e + 4]), __uint_as_float(v[8 * e + 5]));
                        w[e].w = (int)pack_bf16x2(__uint_as_float(v[8 * e + 6]), __uint_as_float(v[8 * e + 7]));
                    }
                }
                __syncwarp();                                // every lane has read its fp32 values
                if (live) {
                    int4* brow = reinterpret_cast<int4*>(st + er * LDA) + 4 * eg;   // packed bf16: bytes [64 eg, 64 eg + 64)
#pragma unroll
                    for (int e = 0; e < 4; ++e) brow[e] = w[e];
                }
                __syncwarp();
                if (p.out_f32 == nullptr) {
#pragma unroll
                    for (int k = lane; k < 8 * PR; k += 32) {
                        const int rr = k / PR, pc = k % PR;
                        const int rs = row0 + rr, cs = n0 + pc * 8;
                        if (rs >= (int)p.M || cs >= p.N) continue;
                        const int4 val = reinterpret_cast<const int4*>(st + rr * LDA)[pc];
                        if (p.dual_dact3) {
                            // a 64-column group is one 7x7 position of act3 (64 channels): one 128-byte line per grid
                            const int px = cs >> 6;
                            const int oy = px / 7, ox = px - oy * 7;
                            *reinterpret_cast<int4*>(p.out + ((int64_t)rs * 81 + oy * 9 + ox) * 64 + (cs & 63)) = val;
                            *reinterpret_cast<int4*>(p.out2 + ((int64_t)rs * 121 + (oy + 2) * 11 + ox + 2) * 64 + (cs & 63)) = val;
                        } else {
                            *reinterpret_cast<int4*>(p.out + (int64_t)rs * p.ldo + cs) = val;
                        }
                    }
                }
                __syncwarp();                                // the packed rows have been read before the next staging
            }
        }
    }
}

// A: row-major [M, 64*nchunks] bf16 (p.A), weights p.Bw [N, 64*nchunks]; epilogue fields as KGemmParams.  Tiles of BN rows
// x BN columns; STAGES stages per consumer warpgroup.
template <int BN, int STAGES>
static int launch_gemm_tma(const KGemmParams& p, cudaStream_t s, const char* what) {
    const size_t smem = (size_t)2 * STAGES * (BN * 128 + BN * 128) + gemm_acc_bytes<BN>() + 1024;
    static SmemAttrCache attr;
    int rc;
    if (p.N % 64 != 0 || BN % 64 != 0) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: N must be a multiple of 64", what);
    if (p.nchunks < 1) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: K must be at least 64", what);
    if (p.out_f32 == nullptr && !p.dual_dact3 && p.ldo % 8 != 0)
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: output pitch must be a multiple of 8 (16-byte stores)", what);
    if ((rc = attr.ensure(tc_gemm_tma<BN, STAGES>, smem, what))) return rc;
    CUtensorMap tmA, tmB;
    const int64_t K = (int64_t)p.nchunks * 64;
    if ((rc = make_tmap_2d(&tmA, p.A, p.M, K, BN, what))) return rc;
    if ((rc = make_tmap_2d(&tmB, p.Bw, p.N, K, BN, what))) return rc;
    const int ntn = (int)ceil_div(p.N, BN);
    const int total = (int)ceil_div(p.M, BN) * ntn;
    int grid = num_sms();
    if (grid > total) grid = total;
    tc_gemm_tma<BN, STAGES><<<grid, kGemmThreads, smem, s>>>(tmA, tmB, p, total, ntn);
    return check_launch(what);
}

// ------------------------------------------------------------------ kernel 2d: TMA-fed weight gradient (fc)
// D[o, k] = sum_m dhid[m, o] * act3[m, k]: both operands are row-major, so each 64-row x 64-column chunk image is
// one TMA box; they are consumed as MN-major operands.  grid = (row splits, X groups of 2 chunks, Y groups of 4).
// Consumer warpgroup w accumulates X chunk w against all kFcWgradYChunks Y chunks (N = 256, 64-element MN atoms chunk_img
// apart); the geometry is fixed: 2 X chunks (one per consumer warpgroup) x 4 Y chunks per CTA.
constexpr int kWgradTmaThreads = 384;
constexpr int kFcWgradXChunks = 2, kFcWgradYChunks = 4;
static __global__ void __launch_bounds__(kWgradTmaThreads, 1) tc_wgrad_tma(const __grid_constant__ CUtensorMap tmX,
                                                                    const __grid_constant__ CUtensorMap tmY,
                                                                    int64_t M, int64_t rows_per_cta, float* ws) {
    constexpr int R = 64, STAGES = 4, nxc = kFcWgradXChunks, nyc = kFcWgradYChunks, NY = 64 * nyc;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, warp = tid >> 5;
    const int xc0 = blockIdx.y * nxc, yc0 = blockIdx.z * nyc;
    constexpr int chunk_img = R * 128;
    constexpr int stage_bytes = (nxc + nyc) * chunk_img;
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
        fence_barrier_init();
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmY);
    }
    __syncthreads();
    const int64_t m_begin = (int64_t)blockIdx.x * rows_per_cta;
    int64_t m_end = m_begin + rows_per_cta;
    if (m_end > M) m_end = M;
    const int nsteps = m_end > m_begin ? (int)((m_end - m_begin + R - 1) / R) : 0;

    if (warp == 0 && (tid & 31) == 0) {
        for (int it = 0; it < nsteps; ++it) {
            const int s = it % STAGES;
            if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
            const uint32_t dst = smem_u32(smem + (size_t)s * stage_bytes);
            const int m0 = (int)(m_begin + (int64_t)it * R);
            mbar_arrive_expect_tx(&full_bar[s], (uint32_t)stage_bytes);
            for (int c = 0; c < nxc; ++c) tma_load_2d(dst + c * chunk_img, &tmX, (xc0 + c) * 64, m0, &full_bar[s]);
            for (int c = 0; c < nyc; ++c) tma_load_2d(dst + (nxc + c) * chunk_img, &tmY, (yc0 + c) * 64, m0, &full_bar[s]);
        }
    } else if (warp >= 4) {
        const int wg = (warp - 4) >> 2, wt = tid & 127;
        float d[NY / 2];
#pragma unroll
        for (int e = 0; e < NY / 2; ++e) d[e] = 0.f;
        auto step = [&](int it) {                            // one batch of 4 MMAs on the stage of step it, one commit group
            const int s = it % STAGES;
            mbar_wait(&full_bar[s], (it / STAGES) & 1);
            wgmma_fence();
            const uint32_t xa = smem_u32(smem + (size_t)s * stage_bytes), ya = xa + nxc * chunk_img;
#pragma unroll
            for (int kk = 0; kk < R / 16; ++kk) {
                const uint64_t adesc = desc_mnmajor(xa + wg * chunk_img + kk * 2048, chunk_img);
                const uint64_t bdesc = desc_mnmajor(ya + kk * 2048, chunk_img);
                WgmmaBf16<NY, 1, 1>::mma(d, adesc, bdesc, (it | kk) != 0 ? 1u : 0u);
            }
            wgmma_commit();
        };
        // Step it-1's stage is released once step it's batch has been issued (wgmma_wait<1>), so the tensor pipe does not
        // drain between steps; the last step is peeled so that its MMAs, the final wait and the stores share one basic
        // block (as in tc_wgrad_win).  Every split has at least one step (wgrad_plan).
        for (int it = 0; it + 1 < nsteps; ++it) {
            step(it);
            wgmma_wait<1>();
            if (it > 0 && (tid & 31) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
        }
        step(nsteps - 1);
        wgmma_wait<0>();
        wgmma_fence_operands(d);
        const int64_t NYtot = (int64_t)gridDim.z * nyc * 64;
        const int64_t KXtot = (int64_t)gridDim.y * nxc * 64;
        float* wsb = ws + (int64_t)blockIdx.x * KXtot * NYtot;
        const int row = ((wt >> 5) << 4) + ((wt & 31) >> 2), col = (wt & 3) * 2;
        float* d0 = wsb + ((int64_t)xc0 * 64 + wg * 64 + row) * NYtot + (int64_t)yc0 * 64 + col;
        float* d8 = d0 + 8 * NYtot;
#pragma unroll
        for (int j = 0; j < NY / 8; ++j) {
            *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
            *reinterpret_cast<float2*>(d8 + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
        }
    }
}

// ---- row splits of the weight gradients: every CTA owns rows_per_cta rows (a multiple of `quantum`)
static int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }
struct WPlan { int64_t rows_per_cta; int splits; };
static WPlan wgrad_plan(int64_t M, int target_ctas, int quantum = 32) {
    WPlan w;
    w.rows_per_cta = round_up(ceil_div(M, target_ctas), quantum);
    if (w.rows_per_cta < quantum) w.rows_per_cta = quantum;
    w.splits = (int)ceil_div(M, w.rows_per_cta);
    if (w.splits < 1) w.splits = 1;
    return w;
}
constexpr int kFcSplits = 8;                 // row splits of tc_wgrad_tma

// partials ws[splits][xcols][ycols rounded up to 256] (fp32) written by launch_wgrad_tma
static size_t wgrad_tma_bytes(int64_t M, int xcols, int ycols) {
    return (size_t)wgrad_plan(M, kFcSplits, 64).splits * xcols * round_up(ycols, 64 * kFcWgradYChunks) * sizeof(float);
}
// ws[split] = X[rows of the split]^T . Y[rows of the split] for row-major bf16 X [M, xcols] and Y [M, ycols] (Y columns
// past ycols are zero-filled by TMA); returns the number of row splits (fold them with tc_fold_fc), or an error (< 0)
static int launch_wgrad_tma(const void* X, int xcols, const void* Y, int ycols, int64_t M, float* ws, cudaStream_t s,
                            const char* what) {
    if (xcols % (64 * kFcWgradXChunks) != 0) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: X columns must be a multiple of 128", what);
    const WPlan pl = wgrad_plan(M, kFcSplits, 64);
    if (M < 1) {                                         // no rows: one split of zero partials (the kernel runs >= 1 step)
        const cudaError_t e = cudaMemsetAsync(ws, 0, wgrad_tma_bytes(M, xcols, ycols), s);
        if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "%s: cudaMemsetAsync: %s", what, cudaGetErrorString(e));
        return pl.splits;
    }
    CUtensorMap tmX, tmY;
    int rc;
    if ((rc = make_tmap_2d(&tmX, X, M, xcols, 64, what))) return rc;
    if ((rc = make_tmap_2d(&tmY, Y, M, ycols, 64, what))) return rc;
    const size_t smem = (size_t)4 * (kFcWgradXChunks + kFcWgradYChunks) * 64 * 128 + 1024;
    static SmemAttrCache attr;
    if ((rc = attr.ensure(tc_wgrad_tma, smem, what))) return rc;
    const dim3 grid(pl.splits, xcols / (64 * kFcWgradXChunks), (unsigned)ceil_div(ycols, 64 * kFcWgradYChunks));
    tc_wgrad_tma<<<grid, kWgradTmaThreads, smem, s>>>(tmX, tmY, M, pl.rows_per_cta, ws);
    if ((rc = check_launch(what))) return rc;
    return pl.splits;
}

}  // namespace b200rl
