// wgmma window weight-gradient kernel (conv layers).
#pragma once
#include "tc_base.cuh"

namespace b200rl {
using namespace tc;

// ------------------------------------------------------------------ kernel 2c: window weight gradient
// dW^T[(tap,channel), co] = sum over grid rows r of X[r + shift_tap, channel] * dY[r, co] with X and dY on the
// SAME linear grid (dY is zero at positions that are not valid outputs).  Per step of 128 rows the CTA
// stages one X window (128 + max shift rows) and 128 dY rows; every tap is an MN-major descriptor shifted by
// whole rows.  Output tile t pairs the 64-channel chunks slot[2t], slot[2t+1].
constexpr int kWgradWinStages = 3;       // stage = X window (<= 37 KB) + 16 KB of dY rows
struct WGradWinParams {
    const bf16* X; const int64_t* rows; int64_t M; int n, G;
    int tpi_shift;           // > 0: image-aligned steps (2^tpi_shift steps of 128 rows per image, M = n << (7 + tpi_shift))
    int64_t n_images;        // images addressable through `rows`
    int cpr;                 // 64-channel column chunks per X row
    int nslots;              // even; chunk of slot s = (tap slot_tap[s], column chunk slot_cc[s])
    int slot_tap[16], slot_cc[16];
    int shift[16];           // per tap
    int WRX;                 // X window rows
    const bf16* Y; int ldy, ncolsY;
    int64_t rows_per_cta;    // multiple of 128
    float* ws;               // [gridDim.y][nslots*64][64]
    float* wsb;              // [gridDim.y][64] bias-gradient partials: sum_r dY[r, co]
};

// 512 threads: warps 0-3 = dY warps (bias sums; in image-aligned mode they also stage dY with cp.async), warp 4 = TMA
// producer (warps 5-7 only keep the consumers warpgroup-aligned), warpgroups 2 and 3 = wgmma: warpgroup w accumulates slot
// 2 t + w of every output tile t this CTA owns.  A CTA owns at most kWgradWinTilesPerCta output tiles (64 accumulator
// registers per thread); blockIdx.x selects them and blockIdx.y is the row split, so the gridDim.x CTAs that stream the
// same rows are adjacent in launch order and run in the same wave: the first one to read a step's rows pulls them into
// L2 and the others hit there, instead of every y-slice re-reading the whole split from HBM in a wave of its own.
constexpr int kWgradWinThreads = 512;
constexpr int kWgradWinTilesPerCta = 2;

// One wgmma warpgroup's main loop over NT (compile-time) output tiles: every step is one straight-line batch of
// NT x 8 MMAs and one commit group.  The indices of the accumulators must be fixed at compile time: with a runtime tile
// count ptxas moves the accumulators between the tiles' MMAs and injects warpgroup.wait / warpgroup.arrive around them.
template <int NT>
__device__ __forceinline__ void wgrad_win_mma(const WGradWinParams& p, uint8_t* smem, int stage_bytes, int XBYTES, int IMGX,
                                              uint64_t* full_bar, uint64_t* empty_bar, int nsteps, int t0, int w, int tid) {
    constexpr int R = 128, STAGES = kWgradWinStages, NY = 64;
    const int wt = tid & 127;
    uint32_t arel[NT];
#pragma unroll
    for (int tt = 0; tt < NT; ++tt) {
        const int slot = 2 * (t0 + tt) + w;
        arel[tt] = (uint32_t)(p.slot_cc[slot] * IMGX + p.shift[p.slot_tap[slot]] * 128);
    }
    float d[NT][NY / 2];
#pragma unroll
    for (int tt = 0; tt < NT; ++tt)
#pragma unroll
        for (int e = 0; e < NY / 2; ++e) d[tt][e] = 0.f;
    auto step = [&](int it) {                            // one batch of NT x 8 MMAs on the stage of step it, one commit group
        const int s = it % STAGES;
        mbar_wait(&full_bar[s], (it / STAGES) & 1);
        wgmma_fence();
        const uint32_t xa = smem_u32(smem + (size_t)s * stage_bytes), ya = xa + XBYTES;
        // K-step kk starts 2048 bytes further on: + 128 in the descriptor's address field (addresses stay below 2^18)
        const uint64_t yd = desc_mnmajor(ya, 0);
#pragma unroll
        for (int tt = 0; tt < NT; ++tt) {
            const uint64_t xd = desc_mnmajor(xa + arel[tt], 0);
#pragma unroll
            for (int kk = 0; kk < R / 16; ++kk)
                WgmmaBf16<NY, 1, 1>::mma(d[tt], xd + kk * 128, yd + kk * 128, (it | kk) != 0 ? 1u : 0u);
        }
        wgmma_commit();
    };
    // Step it-1's stage is released once step it's batch has been issued (wgmma_wait<1>), so the tensor pipe does not
    // drain between steps; the producer only needs step it-STAGES released to refill for step it.  The last step is
    // peeled: its MMAs, the final wait and the accumulator stores then share one basic block, which keeps ptxas from
    // scheduling the stores above the wait.  Every split has at least one step (launch_wgrad_win checks it).
    for (int it = 0; it + 1 < nsteps; ++it) {
        step(it);
        wgmma_wait<1>();
        if (it > 0 && (tid & 31) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    step(nsteps - 1);
    wgmma_wait<0>();
    const int row = ((wt >> 5) << 4) + ((wt & 31) >> 2), col = (wt & 3) * 2;
    float* wsb = p.ws + (int64_t)blockIdx.y * (p.nslots * 64) * NY;
#pragma unroll
    for (int tt = 0; tt < NT; ++tt) {
        wgmma_fence_operands(d[tt]);
        float* d0 = wsb + (int64_t)((2 * (t0 + tt) + w) * 64 + row) * NY + col;
#pragma unroll
        for (int j = 0; j < NY / 8; ++j) {
            *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(d[tt][4 * j], d[tt][4 * j + 1]);
            *reinterpret_cast<float2*>(d0 + 8 * NY + 8 * j) = make_float2(d[tt][4 * j + 2], d[tt][4 * j + 3]);
        }
    }
}

static __global__ void __launch_bounds__(kWgradWinThreads, 1) tc_wgrad_win(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                                                       const WGradWinParams p, int use_tma) {
    constexpr int R = 128, STAGES = kWgradWinStages, LOOKAHEAD = 1, NY = 64, TT = kWgradWinTilesPerCta;
    static_assert(TT == 2, "the wgmma warpgroups dispatch on 1 or 2 tiles per CTA");
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, warp = tid >> 5;
    const int IMGX = p.WRX * 128;
    const int XBYTES = IMGX * p.cpr;
    const int stage_bytes = XBYTES + R * 128;
    const int xt = p.nslots / 2;
    const int t0 = blockIdx.x * TT;                       // first output tile of this CTA
    float* sRed = reinterpret_cast<float*>(smem + (size_t)STAGES * stage_bytes);     // [16][64] bias partials (4 KB)
    if (tid == 0) {
        // full:  one expect_tx arrival (TMA) [+ the four cp.async warps that stage dY in image-aligned mode]
        // empty: the eight wgmma warps [+ the four dY-summing warps when they read the stage after the TMA landed]
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], use_tma ? 1 : 5); mbar_init(&empty_bar[s], (use_tma ? 4 : 0) + 8); }
        fence_barrier_init();
        tma_prefetch_desc(&tmX);
        if (use_tma) tma_prefetch_desc(&tmY);
    }
    __syncthreads();
    const int64_t m_begin = (int64_t)blockIdx.y * p.rows_per_cta;
    int64_t m_end = m_begin + p.rows_per_cta;
    if (m_end > p.M) m_end = p.M;
    const int nsteps = m_end > m_begin ? (int)((m_end - m_begin + R - 1) / R) : 0;
    const int tmask = (1 << p.tpi_shift) - 1;
    const int64_t g0 = m_begin / R;                       // first global step of this CTA (image-aligned mode)

    if (warp == 4) {
        // ======================= TMA producer (one lane): X window [+ dY rows when they are 128 bytes wide] =========
        if ((tid & 31) == 0) {
            int z_next = 0;
            if (!use_tma && nsteps > 0) {
                const int64_t img = g0 >> p.tpi_shift;
                z_next = p.rows ? (int)__ldg(p.rows + (img < p.n ? img : 0)) : (int)img;
            }
            for (int it = 0; it < nsteps; ++it) {
                const int s = it % STAGES;
                const int z = z_next;
                if (!use_tma && it + 1 < nsteps) {        // gather index of the next step, one step ahead
                    const int64_t img1 = (g0 + it + 1) >> p.tpi_shift;
                    z_next = p.rows ? (int)__ldg(p.rows + (img1 < p.n ? img1 : 0)) : (int)img1;
                }
                if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
                const uint32_t dst = smem_u32(smem + (size_t)s * stage_bytes);
                if (use_tma) {
                    const int m0 = (int)(m_begin + (int64_t)it * R);
                    mbar_arrive_expect_tx(&full_bar[s], (uint32_t)stage_bytes);
                    for (int c = 0; c < p.cpr; ++c) tma_load_2d(dst + c * IMGX, &tmX, c * 64, m0, &full_bar[s]);
                    tma_load_2d(dst + XBYTES, &tmY, 0, m0, &full_bar[s]);
                } else {
                    const int t_in = (int)((g0 + it) & tmask);
                    mbar_arrive_expect_tx(&full_bar[s], (uint32_t)XBYTES);
                    for (int c = 0; c < p.cpr; ++c) tma_load_3d(dst + c * IMGX, &tmX, c * 64, t_in * 128, z, &full_bar[s]);
                }
            }
        }
    } else if (warp < 4) {
        // ======================= dY warps: bias gradient = column sums of dY, taken from the staged tile ==========
        // Thread (tid>>3, tid&7) owns rows ps*16 + (tid>>3) and the 16-byte chunk (tid&7) = 8 channels of every step;
        // it adds them up in fp32 (fixed order).  This replaces an all-ones MMA per 16 rows, which cost a quarter to a
        // third of the kernel's shared-memory operand bandwidth.  In image-aligned mode (conv1: dY rows are 64 bytes,
        // no 128-byte TMA box) the same threads first copy those chunks in with cp.async.
        const int rq = tid >> 3, c16 = tid & 7;
        float bsum[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) bsum[e] = 0.f;
        auto add_step = [&](const uint8_t* sYp) {
#pragma unroll
            for (int ps = 0; ps < R / 16; ++ps) {
                const int rr = ps * 16 + rq;
                const int4 v = *reinterpret_cast<const int4*>(sYp + img_off(rr, c16));
                const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    bsum[2 * e] += __uint_as_float(w[e] << 16);
                    bsum[2 * e + 1] += __uint_as_float(w[e] & 0xFFFF0000u);
                }
            }
        };
        if (use_tma) {
            for (int it = 0; it < nsteps; ++it) {
                const int s = it % STAGES;
                mbar_wait(&full_bar[s], (it / STAGES) & 1);
                add_step(smem + (size_t)s * stage_bytes + XBYTES);
                __syncwarp();
                if ((tid & 31) == 0) mbar_arrive(&empty_bar[s]);
            }
        } else {
            for (int it = 0; it < nsteps; ++it) {
                const int s = it % STAGES;
                const int64_t g = g0 + it;
                const int64_t img = g >> p.tpi_shift;
                const int t_in = (int)(g & tmask);
                if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
                const uint32_t sY = smem_u32(smem + (size_t)s * stage_bytes + XBYTES);
                // dY rows of this step (zero past the image's G rows: those grid positions are padding)
#pragma unroll
                for (int ps = 0; ps < R / 16; ++ps) {
                    const int rr = ps * 16 + rq;
                    const int rl = t_in * 128 + rr;
                    const int col = c16 * 8;
                    const bool ok = rl < p.G && img < p.n && col < p.ncolsY;
                    cp_async16(sY + img_off(rr, c16), p.Y + (ok ? (img * p.G + rl) * (int64_t)p.ldy + col : 0), ok ? 16u : 0u);
                }
                cp_async_commit();
                if (it >= LOOKAHEAD) {
                    cp_async_wait<LOOKAHEAD>();
                    const int sd = (it - LOOKAHEAD) % STAGES;
                    add_step(smem + (size_t)sd * stage_bytes + XBYTES);      // this thread's own chunks have landed
                    fence_proxy_async_smem();
                    __syncwarp();
                    if ((tid & 31) == 0) mbar_arrive(&full_bar[sd]);
                }
            }
            cp_async_wait<0>();
            for (int d = (nsteps >= LOOKAHEAD ? nsteps - LOOKAHEAD : 0); d < nsteps; ++d)
                add_step(smem + (size_t)(d % STAGES) * stage_bytes + XBYTES);
            fence_proxy_async_smem();
            __syncwarp();
            if ((tid & 31) == 0)
                for (int d = (nsteps >= LOOKAHEAD ? nsteps - LOOKAHEAD : 0); d < nsteps; ++d) mbar_arrive(&full_bar[d % STAGES]);
        }
        // fold the 16 row lanes of every column chunk in fixed order -> 64 bias partials of this CTA
#pragma unroll
        for (int e = 0; e < 8; ++e) sRed[rq * 64 + c16 * 8 + e] = bsum[e];
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (tid < 64) {
            float t = 0.f;
#pragma unroll
            for (int l = 0; l < 16; ++l) t += sRed[l * 64 + tid];
            if (blockIdx.x == 0) p.wsb[(int64_t)blockIdx.y * NY + tid] = t;
        }
    } else if (warp >= 8) {
        // ======================= wgmma warpgroups: X slot (MN-major, rows = reduction index, shifted by whole rows per tap)
        // x dY rows (MN-major); 8 K-steps of 16 rows per step
        const int w = (warp - 8) >> 2;
        if (xt - t0 >= TT) wgrad_win_mma<TT>(p, smem, stage_bytes, XBYTES, IMGX, full_bar, empty_bar, nsteps, t0, w, tid);
        else wgrad_win_mma<1>(p, smem, stage_bytes, XBYTES, IMGX, full_bar, empty_bar, nsteps, t0, w, tid);
    }
}

}  // namespace b200rl
