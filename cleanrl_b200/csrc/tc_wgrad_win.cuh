// wgmma window weight-gradient kernels (conv layers).
#pragma once
#include "tc_base.cuh"

namespace b200rl {
using namespace tc;

// Bias gradient = column sums of dY, taken from a staged 128-row tile by the four dY warps (128 threads): thread
// (tid>>3, tid&7) owns rows ps*16 + (tid>>3) and the 16-byte chunk (tid&7) = 8 channels of every step and adds them up in
// fp32 (fixed order).  This replaces an all-ones MMA per 16 rows, which cost a quarter to a third of the kernels'
// shared-memory operand bandwidth.
__device__ __forceinline__ void wgrad_bias_add_step(float (&bsum)[8], const uint8_t* sYp, int tid) {
    const int rq = tid >> 3, c16 = tid & 7;
#pragma unroll
    for (int ps = 0; ps < 128 / 16; ++ps) {
        const int rr = ps * 16 + rq;
        const int4 v = *reinterpret_cast<const int4*>(sYp + img_off(rr, c16));
        const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            bsum[2 * e] += __uint_as_float(w[e] << 16);
            bsum[2 * e + 1] += __uint_as_float(w[e] & 0xFFFF0000u);
        }
    }
}
// fold the 16 row lanes of every column chunk in fixed order -> the 64 bias partials of this CTA (named barrier 1)
__device__ __forceinline__ void wgrad_bias_store(const float (&bsum)[8], float* sRed /* [16][64] */, float* wsb, int tid) {
    const int rq = tid >> 3, c16 = tid & 7;
#pragma unroll
    for (int e = 0; e < 8; ++e) sRed[rq * 64 + c16 * 8 + e] = bsum[e];
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (tid < 64) {
        float t = 0.f;
#pragma unroll
        for (int l = 0; l < 16; ++l) t += sRed[l * 64 + tid];
        wsb[tid] = t;
    }
}

// ------------------------------------------------------------------ kernel 2c: conv1 weight gradient on bf16 frames
// dW^T[(tap,channel), co] = sum over grid rows r of X[r + shift_tap, channel] * dY[r, co] with X and dY on the
// SAME grid (dY is zero at positions that are not valid outputs).  Steps are image-aligned: 2^tpi_shift steps of 128 rows
// per image, the X window a 3-D TMA box whose image coordinate is the minibatch gather, dY rows (64 bytes wide) copied
// in with cp.async.  Every tap is an MN-major descriptor shifted by whole rows.  Output tile t pairs slots 2t, 2t+1.
constexpr int kWgradWinStages = 3;       // stage = X window (<= 37 KB) + 16 KB of dY rows
struct WGradWinParams {
    const bf16* X; const int64_t* rows; int64_t M; int n, G;
    int tpi_shift;           // image-aligned steps (2^tpi_shift steps of 128 rows per image, M = n << (7 + tpi_shift))
    int64_t n_images;        // images addressable through `rows`
    int cpr;                 // 64-channel column chunks per X row
    int nslots;              // 4; chunk of slot s = (tap slot_tap[s], column chunk slot_cc[s])
    int slot_tap[16], slot_cc[16];
    int shift[16];           // per tap
    int WRX;                 // X window rows
    const bf16* Y; int ldy, ncolsY;
    int64_t rows_per_cta;    // multiple of 128
    float* ws;               // [gridDim.x][nslots*64][64]
    float* wsb;              // [gridDim.x][64] bias-gradient partials: sum_r dY[r, co]
};

// 512 threads: warps 0-3 = dY warps (stage dY with cp.async, bias sums), warp 4 = TMA producer (warps 5-7 only keep the
// consumers warpgroup-aligned), warpgroups 2 and 3 = wgmma: warpgroup w accumulates slot 2 t + w of output tiles t = 0, 1
// (64 accumulator registers per thread).  blockIdx.x is the row split.
constexpr int kWgradWinThreads = 512;

// One wgmma warpgroup's main loop over NT (compile-time) output tiles: every step is one straight-line batch of
// NT x 8 MMAs and one commit group.  The indices of the accumulators must be fixed at compile time: with a runtime tile
// count ptxas moves the accumulators between the tiles' MMAs and injects warpgroup.wait / warpgroup.arrive around them.
template <int NT>
__device__ __forceinline__ void wgrad_win_mma(const WGradWinParams& p, uint8_t* smem, int stage_bytes, int XBYTES, int IMGX,
                                              uint64_t* full_bar, uint64_t* empty_bar, int nsteps, int w, int tid) {
    constexpr int R = 128, STAGES = kWgradWinStages, NY = 64;
    const int wt = tid & 127;
    uint32_t arel[NT];
#pragma unroll
    for (int tt = 0; tt < NT; ++tt) {
        const int slot = 2 * tt + w;
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
    float* wsb = p.ws + (int64_t)blockIdx.x * (p.nslots * 64) * NY;
#pragma unroll
    for (int tt = 0; tt < NT; ++tt) {
        wgmma_fence_operands(d[tt]);
        float* d0 = wsb + (int64_t)((2 * tt + w) * 64 + row) * NY + col;
#pragma unroll
        for (int j = 0; j < NY / 8; ++j) {
            *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(d[tt][4 * j], d[tt][4 * j + 1]);
            *reinterpret_cast<float2*>(d0 + 8 * NY + 8 * j) = make_float2(d[tt][4 * j + 2], d[tt][4 * j + 3]);
        }
    }
}

static __global__ void __launch_bounds__(kWgradWinThreads, 1) tc_wgrad_win(const __grid_constant__ CUtensorMap tmX, const WGradWinParams p) {
    constexpr int R = 128, STAGES = kWgradWinStages, LOOKAHEAD = 1;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, warp = tid >> 5;
    const int IMGX = p.WRX * 128;
    const int XBYTES = IMGX * p.cpr;
    const int stage_bytes = XBYTES + R * 128;
    float* sRed = reinterpret_cast<float*>(smem + (size_t)STAGES * stage_bytes);     // [16][64] bias partials (4 KB)
    if (tid == 0) {
        // full: one expect_tx arrival (TMA) + the four cp.async warps that stage dY; empty: the eight wgmma warps
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 5); mbar_init(&empty_bar[s], 8); }
        fence_barrier_init();
        tma_prefetch_desc(&tmX);
    }
    __syncthreads();
    const int64_t m_begin = (int64_t)blockIdx.x * p.rows_per_cta;
    int64_t m_end = m_begin + p.rows_per_cta;
    if (m_end > p.M) m_end = p.M;
    const int nsteps = m_end > m_begin ? (int)((m_end - m_begin + R - 1) / R) : 0;
    const int tmask = (1 << p.tpi_shift) - 1;
    const int64_t g0 = m_begin / R;                       // first global step of this CTA

    if (warp == 4) {
        // ======================= TMA producer (one lane): the X window, a 3-D box at the gathered image ===============
        if ((tid & 31) == 0) {
            int z_next = 0;
            if (nsteps > 0) {
                const int64_t img = g0 >> p.tpi_shift;
                z_next = p.rows ? (int)__ldg(p.rows + (img < p.n ? img : 0)) : (int)img;
            }
            for (int it = 0; it < nsteps; ++it) {
                const int s = it % STAGES;
                const int z = z_next;
                if (it + 1 < nsteps) {                    // gather index of the next step, one step ahead
                    const int64_t img1 = (g0 + it + 1) >> p.tpi_shift;
                    z_next = p.rows ? (int)__ldg(p.rows + (img1 < p.n ? img1 : 0)) : (int)img1;
                }
                if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
                const uint32_t dst = smem_u32(smem + (size_t)s * stage_bytes);
                const int t_in = (int)((g0 + it) & tmask);
                mbar_arrive_expect_tx(&full_bar[s], (uint32_t)XBYTES);
                for (int c = 0; c < p.cpr; ++c) tma_load_3d(dst + c * IMGX, &tmX, c * 64, t_in * 128, z, &full_bar[s]);
            }
        }
    } else if (warp < 4) {
        // ======================= dY warps: copy this thread's dY chunks in (cp.async), then add them to the bias sums ====
        const int rq = tid >> 3, c16 = tid & 7;
        float bsum[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) bsum[e] = 0.f;
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
                wgrad_bias_add_step(bsum, smem + (size_t)sd * stage_bytes + XBYTES, tid);   // this thread's own chunks have landed
                fence_proxy_async_smem();
                __syncwarp();
                if ((tid & 31) == 0) mbar_arrive(&full_bar[sd]);
            }
        }
        cp_async_wait<0>();
        for (int d = (nsteps >= LOOKAHEAD ? nsteps - LOOKAHEAD : 0); d < nsteps; ++d)
            wgrad_bias_add_step(bsum, smem + (size_t)(d % STAGES) * stage_bytes + XBYTES, tid);
        fence_proxy_async_smem();
        __syncwarp();
        if ((tid & 31) == 0)
            for (int d = (nsteps >= LOOKAHEAD ? nsteps - LOOKAHEAD : 0); d < nsteps; ++d) mbar_arrive(&full_bar[d % STAGES]);
        wgrad_bias_store(bsum, sRed, p.wsb + (int64_t)blockIdx.x * 64, tid);
    } else if (warp >= 8) {
        // ======================= wgmma warpgroups: X slot (MN-major, rows = reduction index, shifted by whole rows per tap)
        // x dY rows (MN-major); 8 K-steps of 16 rows per step
        wgrad_win_mma<2>(p, smem, stage_bytes, XBYTES, IMGX, full_bar, empty_bar, nsteps, (warp - 8) >> 2, tid);
    }
}

// ------------------------------------------------------------------ kernel 2d: conv2 / conv3 weight gradients (linear grid)
// dW^T[(tap, c), co] = sum over grid rows r of X[r + shift_tap, c] * dY[r, co], X and dY on the same linear grid of WP
// columns (dY is zero at positions that are not valid outputs), taps (ky, kx) at shift ky * WP + kx.  One CTA per row
// split.  Per step of 128 rows the TMA lane stages one X window (WRX rows x CPR 64-channel chunks) and the 128 dY rows.
// The MMAs put dY^T on the A side (M = the 64 output channels; MN-major: co is contiguous in a dY row) and the TPR taps of
// one kernel row on the N side: those taps start one grid row (128 B) apart, so one MN-major descriptor with LBO = 128 B,
// started at the kernel row's first tap, addresses TPR atoms of 64 channels.  A unit = one (kernel row, channel chunk):
// one m64n(64 TPR)k16 per 16 rows.  Per step that reads 2 + 2 TPR KB of operands per 32 TPR tensor-core cycles, within
// the SM's 128 B/clk of shared memory even with the TMA writes and the bias reads (one m64n64k16 per tap would read 4 KB
// per 32 cycles, all of it).
//
// Every dW element gets the products of the same 128-row steps in the same k16 groups as with one tap per MMA, and
// scale-d 0 only on the split's first MMA, so the partials do not depend on which MMA side the channels are on.
constexpr int kWgradRowsStages = 4;
struct WGradRowsParams {
    int64_t M;                 // grid rows
    int64_t rows_per_cta;      // multiple of 128
    float* ws;                 // [gridDim.x][nslots*64][64]: slot = tap * CPR + chunk, row = channel, column = co
    float* wsb;                // [gridDim.x][64] bias-gradient partials: sum_r dY[r, co]
};
template <int CPR, int KROWS, int TPR, int WP, int NCW>
struct WgradRowsCfg {
    static constexpr int kUnits = KROWS * CPR, kUnitsPerWg = kUnits / NCW, kN = 64 * TPR;
    static constexpr int kSlots = KROWS * TPR * CPR;
    static constexpr int kThreads = 128 + 128 * NCW;      // dY warps (one lane is the TMA producer), NCW wgmma warpgroups
    static constexpr int kWRX = (128 + (KROWS - 1) * WP + TPR - 1 + 7) & ~7;
    static constexpr int kImgX = kWRX * 128, kXBytes = kImgX * CPR, kStageBytes = kXBytes + 128 * 128;
    static constexpr size_t kSmem = (size_t)kWgradRowsStages * kStageBytes + 4096 + 1024;
    static_assert(kUnits % NCW == 0, "every wgmma warpgroup owns the same number of units");
    // ptxas compiles the whole kernel within the launch's register budget (65536 / kThreads per thread)
    static_assert(kUnitsPerWg * kN / 2 + 24 <= ((65536 / kThreads) & ~7), "accumulators exceed the registers of a thread");
    static_assert(kSmem <= 227 * 1024, "stages exceed shared memory");
};

template <int CPR, int KROWS, int TPR, int WP, int NCW>
static __global__ void __launch_bounds__(WgradRowsCfg<CPR, KROWS, TPR, WP, NCW>::kThreads, 1)
tc_wgrad_rows(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY, const WGradRowsParams p) {
    using C = WgradRowsCfg<CPR, KROWS, TPR, WP, NCW>;
    constexpr int R = 128, STAGES = kWgradRowsStages, U = C::kUnitsPerWg, NACC = C::kN / 2;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, warp = tid >> 5;
    float* sRed = reinterpret_cast<float*>(smem + (size_t)STAGES * C::kStageBytes);     // [16][64] bias partials (4 KB)
    if (tid == 0) {
        // full: one expect_tx arrival (TMA); empty: the four dY warps and the wgmma warps
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4 + 4 * NCW); }
        fence_barrier_init();
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmY);
    }
    __syncthreads();
    const int64_t m_begin = (int64_t)blockIdx.x * p.rows_per_cta;
    int64_t m_end = m_begin + p.rows_per_cta;
    if (m_end > p.M) m_end = p.M;
    const int nsteps = (int)((m_end - m_begin + R - 1) / R);     // >= 1: launch_wgrad_rows checks every split owns a row

    if (warp < 4) {
        // ======================= dY warps: bias gradient from the staged dY rows; thread 0 also keeps the ring full ====
        // (X window chunks + 128 dY rows per step; a warpgroup of its own for one lane would cost the wgmma warpgroups
        // the registers their accumulators need)
        auto issue = [&](int j) {
            const int s = j % STAGES;
            if (j >= STAGES) mbar_wait(&empty_bar[s], ((j / STAGES) - 1) & 1);
            const uint32_t dst = smem_u32(smem + (size_t)s * C::kStageBytes);
            const int m0 = (int)(m_begin + (int64_t)j * R);
            // rows past M are zero-filled by the TMA and still count towards complete_tx
            mbar_arrive_expect_tx(&full_bar[s], (uint32_t)C::kStageBytes);
#pragma unroll
            for (int c = 0; c < CPR; ++c) tma_load_2d(dst + c * C::kImgX, &tmX, c * 64, m0, &full_bar[s]);
            tma_load_2d(dst + C::kXBytes, &tmY, 0, m0, &full_bar[s]);
        };
        if (tid == 0)
            for (int j = 0; j < STAGES - 1 && j < nsteps; ++j) issue(j);
        float bsum[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) bsum[e] = 0.f;
        for (int it = 0; it < nsteps; ++it) {
            // step it + STAGES - 1 reuses the stage of step it - 1, released once the wgmma warpgroups have issued step it
            if (tid == 0 && it + STAGES - 1 < nsteps) issue(it + STAGES - 1);
            const int s = it % STAGES;
            mbar_wait(&full_bar[s], (it / STAGES) & 1);
            wgrad_bias_add_step(bsum, smem + (size_t)s * C::kStageBytes + C::kXBytes, tid);
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(&empty_bar[s]);
        }
        wgrad_bias_store(bsum, sRed, p.wsb + (int64_t)blockIdx.x * 64, tid);
    } else {
        // ======================= wgmma warpgroup w: units w*U .. w*U+U-1, 8 K-steps of 16 rows per step ===============
        const int w = (warp >> 2) - 1, wt = tid & 127;
        float d[U][NACC];
#pragma unroll
        for (int uu = 0; uu < U; ++uu)
#pragma unroll
            for (int e = 0; e < NACC; ++e) d[uu][e] = 0.f;
        // byte offset of unit u's first tap inside the stage: its channel chunk's window, shifted by ky * WP rows
        auto brel = [&](int uu) { const int u = w * U + uu; return (uint32_t)((u % CPR) * C::kImgX + (u / CPR) * WP * 128); };
        // one batch of U x 8 MMAs on the stage of step it, one commit group; K-step kk starts 2048 bytes further on:
        // + 128 in the descriptors' address fields (addresses stay below 2^18)
        auto step = [&](int it) {
            const int s = it % STAGES;
            mbar_wait(&full_bar[s], (it / STAGES) & 1);
            wgmma_fence();
            const uint32_t xa = smem_u32(smem + (size_t)s * C::kStageBytes), ya = xa + C::kXBytes;
            const uint64_t yd = desc_mnmajor(ya, 0);
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
                const uint64_t xd = desc_mnmajor(xa + brel(uu), 128);
#pragma unroll
                for (int kk = 0; kk < R / 16; ++kk)
                    WgmmaBf16<C::kN, 1, 1>::mma(d[uu], yd + kk * 128, xd + kk * 128, (it | kk) != 0 ? 1u : 0u);
            }
            wgmma_commit();
        };
        // Step it-1's stage is released once step it's batch has been issued (wgmma_wait<1>), so the tensor pipe does not
        // drain between steps.  The last step is peeled: its MMAs, the final wait and the accumulator stores then share
        // one basic block, which keeps ptxas from scheduling the stores above the wait.
        for (int it = 0; it + 1 < nsteps; ++it) {
            step(it);
            wgmma_wait<1>();
            if (it > 0 && (tid & 31) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
        }
        step(nsteps - 1);
        wgmma_wait<0>();
        // accumulator element (co, n = tap-in-row * 64 + c) -> ws[split][slot * 64 + c][co]: the layout of one tap per MMA
        // with the channels on M, which tc_fold_win folds over the splits
        const int co = ((wt >> 5) << 4) + ((wt & 31) >> 2), col = (wt & 3) * 2;
        float* wsp = p.ws + (int64_t)blockIdx.x * (C::kSlots * 64 * 64);
#pragma unroll
        for (int uu = 0; uu < U; ++uu) {
            wgmma_fence_operands(d[uu]);
            const int u = w * U + uu;
#pragma unroll
            for (int j = 0; j < NACC / 4; ++j) {
                const int slot = ((u / CPR) * TPR + (j >> 3)) * CPR + u % CPR;
                float* q = wsp + (int64_t)(slot * 64 + (8 * j & 63) + col) * 64 + co;
                q[0] = d[uu][4 * j];
                q[64] = d[uu][4 * j + 1];
                q[8] = d[uu][4 * j + 2];
                q[64 + 8] = d[uu][4 * j + 3];
            }
        }
    }
}

}  // namespace b200rl
