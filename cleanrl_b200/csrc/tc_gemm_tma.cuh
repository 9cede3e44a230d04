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
};

// ------------------------------------------------------------------ kernel 1d: TMA-fed GEMM (fc forward / data-gradient)
// Plain row-major operands => the tiles are rectangular boxes: ONE thread issues cp.async.bulk.tensor (TMA,
// SWIZZLE_128B) loads for the A chunk [128 x 64] and the weight chunk [BN x 64]; the hardware does the address
// generation, zero-fills out-of-range rows and signals the stage's mbarrier with complete_tx.  Warpgroup 0 = TMA
// producer (warp 0), warpgroups 1 and 2 = wgmma on rows 0-63 / 64-127 of the tile, then the epilogue (one thread per row
// and 32-column group) from a shared-memory copy of the accumulators.
constexpr int kGemmThreads = 384;
template <int BN>
__host__ __device__ constexpr size_t gemm_acc_bytes() { return (size_t)128 * (BN + 4) * sizeof(float); }
template <int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1) tc_gemm_tma(const __grid_constant__ CUtensorMap tmA,
                                                               const __grid_constant__ CUtensorMap tmB,
                                                               const KGemmParams p, int total_tiles, int ntiles_n) {
    constexpr int A_BYTES = 128 * 128;
    constexpr int B_BYTES = BN * 128;
    constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    constexpr int LDA = BN + 4;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float* sAcc = reinterpret_cast<float*>(smem + (size_t)STAGES * STAGE_BYTES);
    const int tid = threadIdx.x, warp = tid >> 5;
    const int nch = p.nchunks;
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 256); }   // every consumer thread
        fence_barrier_init();
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
    }
    __syncthreads();

    if (warp == 0) {
        if ((tid & 31) == 0) {
            uint32_t q = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int mt = tile / ntiles_n, n0 = (tile - mt * ntiles_n) * BN;
                for (int j = 0; j < nch; ++j, ++q) {
                    const uint32_t s = q % STAGES;
                    if (q >= (uint32_t)STAGES) mbar_wait(&empty_bar[s], ((q / STAGES) - 1) & 1);
                    const uint32_t dst = smem_u32(smem + (size_t)s * STAGE_BYTES);
                    mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
                    tma_load_2d(dst, &tmA, j * 64, mt * 128, &full_bar[s]);
                    tma_load_2d(dst + A_BYTES, &tmB, j * 64, n0, &full_bar[s]);
                }
            }
        }
    } else if (warp >= 4) {
        const int wg = (warp - 4) >> 2, wt = tid & 127;
        float* st = sAcc + wg * 64 * LDA;
        const int lr = wt & 63, half = wt >> 6;
        const int nwords = p.N >> 5;                         // mask words per row (N is a multiple of 32)
        constexpr int NW = BN / 32;
        float d[BN / 2];
#pragma unroll
        for (int e = 0; e < BN / 2; ++e) d[e] = 0.f;
        uint32_t q = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int mt = tile / ntiles_n, n0 = (tile - mt * ntiles_n) * BN;
            for (int j = 0; j < nch; ++j, ++q) {
                const uint32_t s = q % STAGES;
                mbar_wait(&full_bar[s], (q / STAGES) & 1);
                wgmma_fence();
                const uint32_t stage_addr = smem_u32(smem + (size_t)s * STAGE_BYTES);
                const uint64_t a = desc_kmajor(stage_addr + wg * 64 * 128), b = desc_kmajor(stage_addr + A_BYTES);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) WgmmaBf16<BN, 0, 0>::mma(d, a + 2 * kk, b + 2 * kk, (j | kk) != 0 ? 1u : 0u);
                wgmma_commit();
                // Complete the chunk before its stage is released: TMA keeps STAGES - 1 chunks ahead, and the other warpgroup's
                // MMAs fill the tensor cores meanwhile.  (ptxas reports these MMAs as serialised, C7520; keeping a group in
                // flight across the next stage wait did not avoid that either.)
                wgmma_wait<0>();
                mbar_arrive(&empty_bar[s]);
            }
            wgmma_fence_operands(d);
            const int r = mt * 128 + wg * 64 + lr;
            const bool rvalid = r < (int)p.M;
            const int64_t wb = (int64_t)r * nwords + (n0 >> 5);
            named_bar(1 + wg, 128);                          // the previous tile's rows have been read
            stage_acc(st, LDA, wt, d);
            named_bar(1 + wg, 128);
#pragma unroll
            for (int g = 0; g < NW; ++g) {
                const int col = n0 + g * 32;
                if (!rvalid || (g & 1) != half || col >= p.N) continue;     // rows past M, the ragged last column tile
                uint32_t v[32];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float4 f = *reinterpret_cast<const float4*>(st + lr * LDA + g * 32 + 4 * e);
                    v[4 * e] = __float_as_uint(f.x); v[4 * e + 1] = __float_as_uint(f.y);
                    v[4 * e + 2] = __float_as_uint(f.z); v[4 * e + 3] = __float_as_uint(f.w);
                }
                const uint32_t mbw = p.mask_bits != nullptr ? __ldg(p.mask_bits + wb + g) : 0xFFFFFFFFu;
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
                    if (p.mask_out) p.mask_out[wb + g] = bits;
                }
                if (p.mask_bits) {
#pragma unroll
                    for (int e = 0; e < 32; ++e) if (!((mbw >> e) & 1u)) v[e] = 0u;
                }
                int4 w[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    w[e].x = (int)pack_bf16x2(__uint_as_float(v[8 * e]), __uint_as_float(v[8 * e + 1]));
                    w[e].y = (int)pack_bf16x2(__uint_as_float(v[8 * e + 2]), __uint_as_float(v[8 * e + 3]));
                    w[e].z = (int)pack_bf16x2(__uint_as_float(v[8 * e + 4]), __uint_as_float(v[8 * e + 5]));
                    w[e].w = (int)pack_bf16x2(__uint_as_float(v[8 * e + 6]), __uint_as_float(v[8 * e + 7]));
                }
                if (p.dual_dact3) {
                    // a 64-column group is one 7x7 position of act3 (64 channels); g & 1 = which half of it
                    const int px = col >> 6;
                    const int oy = px / 7, ox = px - oy * 7;
                    bf16* dst = p.out + ((int64_t)r * 81 + oy * 9 + ox) * 64 + (g & 1) * 32;
                    bf16* dst2 = p.out2 + ((int64_t)r * 121 + (oy + 2) * 11 + ox + 2) * 64 + (g & 1) * 32;
                    st_global_32b(dst, w[0], w[1]); st_global_32b(dst + 16, w[2], w[3]);
                    st_global_32b(dst2, w[0], w[1]); st_global_32b(dst2 + 16, w[2], w[3]);
                } else {
                    bf16* dst = p.out + (int64_t)r * p.ldo + col;
                    st_global_32b(dst, w[0], w[1]); st_global_32b(dst + 16, w[2], w[3]);
                }
            }
        }
    }
}

// ------------------------------------------------------------------ kernel 2d: TMA-fed weight gradient (fc)
// D[o, k] = sum_m dhid[m, o] * act3[m, k]: both operands are row-major, so each 64-row x 64-column chunk image is
// one TMA box; they are consumed as MN-major operands.  grid = (row splits, X groups of 2 chunks, Y groups of 4).
// Consumer warpgroup w accumulates X chunk w against all kFcWgradYChunks Y chunks (N = 256, 64-element MN atoms chunk_img
// apart); the geometry is fixed: 2 X chunks (one per consumer warpgroup) x 4 Y chunks per CTA.
constexpr int kWgradTmaThreads = 384;
constexpr int kFcWgradXChunks = 2, kFcWgradYChunks = 4;
__global__ void __launch_bounds__(kWgradTmaThreads, 1) tc_wgrad_tma(const __grid_constant__ CUtensorMap tmX,
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
        for (int it = 0; it < nsteps; ++it) {
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
            wgmma_wait<0>();
            if ((tid & 31) == 0) mbar_arrive(&empty_bar[s]);
        }
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

// A: row-major [M, 64*nchunks] bf16 (p.A), weights p.Bw [N, 64*nchunks]; epilogue fields as KGemmParams
template <int BN, int STAGES>
static int launch_gemm_tma(const KGemmParams& p, cudaStream_t s, const char* what) {
    const size_t smem = (size_t)STAGES * (128 * 128 + BN * 128) + gemm_acc_bytes<BN>() + 1024;
    static SmemAttrCache attr;
    int rc;
    if (p.N % 64 != 0 || BN % 64 != 0) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: N must be a multiple of 64", what);
    if ((rc = attr.ensure(tc_gemm_tma<BN, STAGES>, smem, what))) return rc;
    CUtensorMap tmA, tmB;
    const int64_t K = (int64_t)p.nchunks * 64;
    if ((rc = make_tmap_2d(&tmA, p.A, p.M, K, 128, what))) return rc;
    if ((rc = make_tmap_2d(&tmB, p.Bw, p.N, K, BN, what))) return rc;
    const int ntn = (int)ceil_div(p.N, BN);
    const int total = (int)ceil_div(p.M, 128) * ntn;
    int grid = num_sms();
    if (grid > total) grid = total;
    tc_gemm_tma<BN, STAGES><<<grid, kGemmThreads, smem, s>>>(tmA, tmB, p, total, ntn);
    return check_launch(what);
}

}  // namespace b200rl
