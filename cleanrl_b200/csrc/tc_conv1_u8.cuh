// conv1 straight from the uint8 rollout (no 16-bit copy of the frames anywhere).
//
// The rollout keeps every frame as uint8 space-to-depth(4) pixels, 28 224 B per frame (the algorithmic minimum;
// reference: a 14.8 GB fp32 buffer, ppo_atari_envpool.py:203):
//     frames    u8 [img][441 grid rows][64 ch]   row-major    -> forward and weight gradient
//     frames_t  u8 [img][64 ch][448 grid rows]   channel-major (still written by tc_frames_to_s2d_u8; no kernel reads it)
//
// Forward  tc_conv1_i8: integer tensor cores (wgmma u8 x s8 -> s32, accumulators in registers).  The
//   pixels are EXACT (0..255 are integers); the fp32 master weights are split per output channel into two signed
//   8-bit limbs  w ~= s_co * (l1 / 2^7 + l2 / 2^14)  (|error| <= s_co * 2^-15, i.e. 15 bits relative to the row
//   maximum -- tighter than the 8 bits of a bf16 weight), the two limbs are 2 x 32 = 64 GEMM columns, and the
//   epilogue recombines  y = acc1 * s/2^7/255 + acc2 * s/2^14/255 + bias.  Integer accumulation is exact, so the
//   result does not depend on the order of the 256-term dot products.  A 1-byte operand also halves the
//   shared-memory operand traffic that bounded the bf16 kernel (N = 32 is too narrow to amortise the 128-row A tile).
//   Same window scheme as tc_conv_win: one TMA box of 128 + 22 rows per tile, the four 2x2 taps are descriptors
//   shifted by whole 64-byte rows of a SWIZZLE_64B image.
//
// Weight gradient  tc_conv21_bwd_u8 (which first computes dY, the conv2 data gradient, into shared memory):
//   dW[tap, c, co] = sum_p X[p + off_tap, c] * dY[p, co].  The row-major pixels go
//   uint8 (shared memory, TMA boxes of pair rows) -> fp16 1024 + x (one PRMT per two pixels, by a warpgroup of their
//   own, into a SWIZZLE_128B shared-memory image one step ahead of the MMAs; the offset is removed once per CTA through
//   the bias partial), and are consumed as the MN-major B operand (N = 128: both pixel streams X[k], X[k + 1] through
//   LBO = one row); the A operand is the dY image, read at two row offsets (0 and -21) so that one MMA serves all four
//   taps.  Both operands come from shared memory, so the MMAs of one step run while the next step is expanded.
#pragma once
#include "tc_base.cuh"
#include <cuda_fp16.h>
#include "tc_conv_win.cuh"

namespace b200rl {
using namespace tc;

// ------------------------------------------------------------------------------------------------ descriptors
// K-major SWIZZLE_64B operand: rows 64 B apart, 8-row atoms 512 B apart (SBO)
__device__ __forceinline__ uint64_t desc_kmajor_sw64(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (32ull << 32) | kDescSwizzle64;
}
// MN-major SWIZZLE_64B operand of 32-element (64-byte) MN atoms: rows = K index, 8-row K groups 512 B apart (SBO), MN atom
// i (columns 32 i .. 32 i + 31) at smem_addr + i * lbo (LBO; any multiple of 64 B: the swizzle is applied to the absolute
// address bits, as for start addresses shifted by whole rows)
__device__ __forceinline__ uint64_t desc_mnmajor_sw64(uint32_t smem_addr, uint32_t lbo) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) | (32ull << 32) | kDescSwizzle64;
}
// byte offset of 16-byte chunk c (0..3) of row r in a SWIZZLE_64B image (address bits [4,6) ^= bits [7,9))
__device__ __forceinline__ uint32_t img64_off(int r, int c) { return (uint32_t)(r * 64 + ((c ^ ((r >> 1) & 3)) << 4)); }
// ------------------------------------------------------------------------------------ frame conversion (once per env step)
// uint8 frames [n,4,84,84] (NCHW, as the env delivers them) -> row-major u8 [n,441,64] and channel-major u8 [n,64,448]
// space-to-depth(4) pixels: channel = c*16 + sy*4 + sx of source pixel (4Y+sy, 4X+sx), grid row = Y*21 + X.
// One block per frame: the whole 4 x 84 x 84 frame is staged in shared memory with 16-byte loads (7 per thread, all in
// flight before the barrier).  Both outputs are then written as whole lines: a 32-bit word of a plane row holds the 4
// sx pixels of one position, so a row-major position is 16 such words (4 consecutive threads store its 64 bytes), and
// 4 positions x 4 sx of a channel-major (c, sy) group are a 4 x 4 byte transpose of 4 words (one PRMT pair per output
// word, each stored with the neighbouring threads' words of the same channel row).
constexpr int kS2dThreads = 256;
__global__ void __launch_bounds__(kS2dThreads) tc_frames_to_s2d_u8(const uint8_t* __restrict__ obs, const int64_t* __restrict__ rows,
                                                                   int64_t n, uint8_t* __restrict__ out_rm, uint8_t* __restrict__ out_cm) {
    __shared__ __align__(16) uint8_t frame[28224];
    const int64_t i = blockIdx.x;
    const int64_t img = rows ? rows[i] : i;
    const int4* src = reinterpret_cast<const int4*>(obs + img * 28224);
#pragma unroll
    for (int k = 0; k < 7; ++k) {
        const int t = threadIdx.x + k * kS2dThreads;
        if (t < 1764) reinterpret_cast<int4*>(frame)[t] = __ldg(src + t);
    }
    __syncthreads();
    // row-major [441][64]: 16-byte chunk c of position pos = rows 4Y .. 4Y+3 of plane c at column 4X
    int4* rm = reinterpret_cast<int4*>(out_rm + i * 441 * 64);
    for (int t = threadIdx.x; t < 441 * 4; t += kS2dThreads) {
        const int pos = t >> 2, c = t & 3;
        const int Y = (pos * 3121) >> 16, X = pos - Y * 21;                   // pos / 21 for pos < 512
        const uint8_t* p = frame + c * 7056 + (Y * 4) * 84 + X * 4;
        int4 v;
        v.x = *reinterpret_cast<const int*>(p); v.y = *reinterpret_cast<const int*>(p + 84);
        v.z = *reinterpret_cast<const int*>(p + 168); v.w = *reinterpret_cast<const int*>(p + 252);
        rm[t] = v;
    }
    // channel-major [64][448]: group (c, sy, q) = positions 4q .. 4q+3 of the 4 channels c*16 + sy*4 + sx (zero past 441)
    uint8_t* cm = out_cm + i * 64 * 448;
    for (int t = threadIdx.x; t < 16 * 112; t += kS2dThreads) {
        const int g = t / 112, q = t - g * 112;                                // g = c * 4 + sy
        const uint8_t* prow = frame + (g >> 2) * 7056 + (g & 3) * 84;
        uint32_t w[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int pos = q * 4 + e, pc = pos < 441 ? pos : 440;           // the tail reads a valid word, stores 0
            const int Y = (pc * 3121) >> 16, X = pc - Y * 21;
            const uint32_t v = *reinterpret_cast<const uint32_t*>(prow + (Y * 4) * 84 + X * 4);
            w[e] = pos < 441 ? v : 0u;
        }
        const uint32_t lo01 = __byte_perm(w[0], w[1], 0x5140), hi01 = __byte_perm(w[0], w[1], 0x7362);
        const uint32_t lo23 = __byte_perm(w[2], w[3], 0x5140), hi23 = __byte_perm(w[2], w[3], 0x7362);
        uint32_t* dst = reinterpret_cast<uint32_t*>(cm + (g * 4) * 448) + q;
        dst[0] = __byte_perm(lo01, lo23, 0x5410);                             // sx = 0: byte e = position 4q + e
        dst[112] = __byte_perm(lo01, lo23, 0x7632);
        dst[224] = __byte_perm(hi01, hi23, 0x5410);
        dst[336] = __byte_perm(hi01, hi23, 0x7632);
    }
}

// ------------------------------------------------------------------------------------ conv1 weight limbs
// w[co][c][ky][kx] (fp32) -> s8 limbs L[(limb, co)][tap (a,b)][c*16 + sy*4 + sx] with ky = 4a+sy, kx = 4b+sx, and the
// per-column output scales sc[limb*32 + co] = s_co / 2^(7*(limb+1)) / 255 (the /255 of ppo_atari_envpool.py:144).
__global__ void __launch_bounds__(256) tc_pack_conv1_i8(const float* __restrict__ w, int8_t* __restrict__ limbs, float* __restrict__ sc) {
    __shared__ float red[32];
    const int co = blockIdx.x, idx = threadIdx.x;                  // idx = (c, ky, kx)
    const float v = w[co * 256 + idx];
    float m = fabsf(v);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((idx & 31) == 0) red[idx >> 5] = m;
    __syncthreads();
    float mx = red[0];
#pragma unroll
    for (int k = 1; k < 8; ++k) mx = fmaxf(mx, red[k]);
    const float s = mx > 0.f ? mx * (128.0f / 127.0f) : 1.0f;
    const float u = v / s * 128.0f;                                // |u| <= 127
    float l1 = rintf(u);
    l1 = fminf(fmaxf(l1, -127.f), 127.f);
    float l2 = rintf((u - l1) * 128.0f);
    l2 = fminf(fmaxf(l2, -127.f), 127.f);
    const int kx = idx & 7, ky = (idx >> 3) & 7, c = idx >> 6;
    const int a = ky >> 2, sy = ky & 3, b = kx >> 2, sx = kx & 3;
    const int k = (a * 2 + b) * 64 + c * 16 + sy * 4 + sx;
    limbs[co * 256 + k] = (int8_t)l1;
    limbs[(32 + co) * 256 + k] = (int8_t)l2;
    if (idx == 0) {
        sc[co] = s / 128.0f / 255.0f;
        sc[32 + co] = s / 16384.0f / 255.0f;
    }
}

// ------------------------------------------------------------------------------------ conv1 forward (kind::i8)
struct Conv1U8Params {
    const int64_t* rows;     // optional image gather (minibatch rows of the rollout)
    int n;                   // images in this launch
    int64_t n_images;        // images addressable through `rows`
    const int8_t* limbs;     // [64][256] s8 (tc_pack_conv1_i8)
    const float* sc;         // [64] column scales
    const float* bias;       // [32]
    bf16* out;               // act1 as 2x2 cells [n,100,128]
    uint32_t* mask_out;      // act1 > 0 bits: [n,100 cells] x 4 words
};

// Pair rows: TMA delivers one shared-memory row (<= 128 B) per request at ~5.5 cycles per request and SM -- the rate at
// which 128-byte rows saturate HBM -- so a box of 64-byte rows moves half the bytes in the same time (measured: the first
// version of this kernel, boxes of 152 x 64 B, sat at 44 % DRAM with its MMA issuer waiting on the TMA barrier).  The
// row-major image [441][64 B] is therefore read as 221 rows of 128 B = PAIRS of grid positions (2q, 2q+1): one box of
// 139 pair rows per 256 output positions.  GEMM rows are pair rows; the even and the odd position of each pair get their own
// accumulator, and a tap (dy, dx) of position p = 2q + e is the 64-byte half ((e + dx + dy) & 1) of pair row
// q + (e + 21 dy + dx) / 2 -- a K-major SWIZZLE_128B descriptor shifted by whole rows plus a 64-byte K offset.
// Thread roles (384 threads): warpgroup 0 = TMA producer (warp 0), warpgroups 1 and 2 = wgmma on pair rows 0-63 / 64-127
// of the tile, both parities, and the epilogue straight from the accumulator fragments.
constexpr int kConv1I8Threads = 384;
template <int STAGES>
__global__ void __launch_bounds__(kConv1I8Threads, 1) tc_conv1_i8(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                                                                   const Conv1U8Params p, int total_tiles) {
    constexpr int BN = 64, WR = 144, NTAPS = 4;
    constexpr int STAGE_BYTES = WR * 128;           // 18432 = 18 x 1024
    constexpr int B_CHUNK = BN * 64;                // one tap of the limb image: 64 rows x 64 B (SWIZZLE_64B)
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES], w_bar;
    __shared__ __align__(16) float s_sc[32], s_bias[32];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, warp = tid >> 5;
    uint8_t* sW = smem;                             // 4 taps x 4096 B
    uint8_t* sRing = smem + NTAPS * B_CHUNK;        // 16384: 1024-aligned

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // 8 consumer warps
        mbar_init(&w_bar, 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmW);
    }
    if (tid < 32) { s_sc[tid] = p.sc[32 + tid]; s_bias[tid] = p.bias[tid]; }      // sc[32 + co] = s_co / 2^14 / 255
    __syncthreads();
    // a tile = 128 pair rows = 256 grid positions; 2 tiles per image (441 positions used)
    const int tile_begin = (int)(((int64_t)total_tiles * blockIdx.x) / gridDim.x);
    const int tile_end = (int)(((int64_t)total_tiles * (blockIdx.x + 1)) / gridDim.x);

    if (warp == 0) {
        // ======================= TMA producer: one [139 (144) pair rows x 128 B] box of one image per tile; the image
        // coordinate is the minibatch gather, fetched one tile ahead
        if (tid == 0) {
            uint32_t q = 0;
            int z_next = 0;
            if (tile_begin < tile_end) {
                const int img = tile_begin >> 1;
                z_next = p.rows ? (int)__ldg(p.rows + img) : img;
            }
            for (int tile = tile_begin; tile < tile_end; ++tile, ++q) {
                const uint32_t s = q % STAGES;
                const int z = z_next;
                if (tile + 1 < tile_end) {
                    const int img = (tile + 1) >> 1;
                    z_next = p.rows ? (int)__ldg(p.rows + img) : img;
                }
                if (q >= (uint32_t)STAGES) mbar_wait(&empty_bar[s], ((q / STAGES) - 1) & 1);
                mbar_arrive_expect_tx(&full_bar[s], (uint32_t)STAGE_BYTES);
                tma_load_3d(smem_u32(sRing + (size_t)s * STAGE_BYTES), &tmA, 0, (tile & 1) * 128, z, &full_bar[s]);
                if (q == 0) {       // the limb image, one [64 rows x 64 B] SWIZZLE_64B box per tap, behind the first window
                    mbar_arrive_expect_tx(&w_bar, (uint32_t)(NTAPS * B_CHUNK));
#pragma unroll
                    for (int t = 0; t < NTAPS; ++t) tma_load_3d(smem_u32(sW + t * B_CHUNK), &tmW, t * 64, 0, 0, &w_bar);
                }
            }
        }
    } else if (warp >= 4) {
        // ======================= wgmma warpgroup wg: pair rows 64 wg .. 64 wg + 63; per parity e 4 taps x 2 K-steps of 32
        // bytes.  A: K-major SWIZZLE_128B pair rows (row shift + 64-byte half); B: K-major SWIZZLE_64B limb rows.
        const int wg = (warp - 4) >> 2, wt = tid & 127, lane = tid & 31, qd = lane & 3;
        const uint32_t w_base = smem_u32(sW);
        // tap t = (dy, dx): position offset 21 dy + dx; for parity e the operand is half (e + off) & 1 of pair row + (e + off) >> 1
        constexpr int off[4] = {0, 1, 21, 22};
        int acc[2][32];
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int c = 0; c < 32; ++c) acc[e][c] = 0;
        if (tile_begin < tile_end) mbar_wait(&w_bar, 0);
        for (int tile = tile_begin; tile < tile_end; ++tile) {
            const uint32_t q = (uint32_t)(tile - tile_begin), s = q % STAGES;
            mbar_wait(&full_bar[s], (q / STAGES) & 1);
            wgmma_fence();
            const uint32_t win = smem_u32(sRing + (size_t)s * STAGE_BYTES) + (uint32_t)(wg * 64 * 128);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
#pragma unroll
                for (int t = 0; t < NTAPS; ++t) {
                    const int po = e + off[t];
                    const uint64_t a = desc_kmajor(win + (uint32_t)((po >> 1) * 128 + (po & 1) * 64));     // rows of 128 B, halves of 64 B
                    const uint64_t b = desc_kmajor_sw64(w_base + (uint32_t)(t * B_CHUNK));
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) wgmma_u8s8_n64(acc[e], a + 2 * kk, b + 2 * kk, (t | kk) != 0 ? 1u : 0u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_operands(acc[0]);
            wgmma_fence_operands(acc[1]);
            if (lane == 0) mbar_arrive(&empty_bar[s]);
            // epilogue: this thread holds rows lr and lr + 8 of both parities, channels 8 j + 2 qd (+1) of both limbs (column
            // co of limb 1 and column 32 + co of limb 2 are in the same thread).
            // y = (128 acc1 + acc2) * (s / 2^14 / 255) + bias: the limb recombination is exact in int32 (|128 acc1| < 2^31)
            const int i = tile >> 1;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int lrow = wg * 64 + ((wt >> 5) << 4) + (lane >> 2) + 8 * hr;
                    const int rem = 2 * (((tile & 1) << 7) + lrow) + e;
                    const int Y = (rem * 3121) >> 16, X = rem - Y * 21;          // rem / 21 for rem < 512
                    const bool valid = rem < 441 && Y < 20 && X < 20;
                    const int64_t cell = ((int64_t)i * 10 + (Y >> 1)) * 10 + (X >> 1);
                    const int cls = (Y & 1) * 2 + (X & 1);
                    uint32_t bits = 0u, pk[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int co = 8 * j + 2 * qd;
                        const float f0 = fmaf((float)(acc[e][4 * j + 2 * hr] * 128 + acc[e][4 * (j + 4) + 2 * hr]), s_sc[co], s_bias[co]);
                        const float f1 = fmaf((float)(acc[e][4 * j + 2 * hr + 1] * 128 + acc[e][4 * (j + 4) + 2 * hr + 1]), s_sc[co + 1],
                                              s_bias[co + 1]);
                        bits |= (f0 > 0.f ? 1u : 0u) << co;
                        bits |= (f1 > 0.f ? 1u : 0u) << (co + 1);
                        pk[j] = pack_bf16x2_relu(f0, f1);
                    }
                    bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
                    bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
                    if (valid) {
                        if (qd == 0) p.mask_out[cell * 4 + cls] = bits;
                        uint32_t* dst = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.out) + (cell * 4 + cls) * 64);
#pragma unroll
                        for (int j = 0; j < 4; ++j) dst[4 * j + qd] = pk[j];
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------ conv2 data gradient + conv1 weight gradient
// One kernel computes d(act1) (the conv2 data gradient) and, from it, the conv1 weight and bias gradients, so that d(act1)
// is written to HBM once and never read back.
//
// conv2 data gradient (warpgroup 1), per image: d(act1) = the full correlation of the zero-padded 11x11 d(act2) grid
//   with the four stride-parity classes of W2 (one N = 128 GEMM, K = 4 taps x 64 channels), exactly as the window
//   convolution tc_conv_win runs it: a TMA window of 140 rows of the image's d(act2) rows (128 GEMM rows + the largest tap
//   shift of 12 rows) and, with it, one bulk copy of the image's act1 > 0 mask bits (1600 B; read from HBM by the
//   epilogue itself, they stalled it), resident weights, m64n128k16 MMAs in the same tap and K order.  The epilogue (act1 > 0 mask, x
//   kDact1Scale, saturating fp16) writes the image as the dY operand of the weight gradient straight into shared memory,
//   and one TMA store per 128 rows copies it to d(act1) in HBM.
// conv1 weight gradient (warpgroups 2 and 3): dW[tap, c, co] = sum_p X[p + off_tap, c] * dY[p, co] over the grid
//   positions p of an image, off = {0, 1, 21, 22} (taps (dy, dx) of the 2x2 window on the 21-wide grid).  Written over
//   k = p + s_b with s_b = {0, 21}:
//       D[(b, co), (h, c)] = sum_k dY[k - s_b, co] * X16[k + h, c],    tap = 2 b + h,
//   one m64n128k16 per 16 positions, both operands in shared memory:
//   A  (M = 64, MN-major SWIZZLE_64B): the dY rows of the step, rows [k0 - 21, k0 + 107) for b = 1 (MN atom 0, co 0-31)
//       and rows [k0, k0 + 128) for b = 0 (atom 1, 21 rows = LBO later).  A dY image is [24-row zero halo | 512 rows] of
//       64 B: rows of positions that are not conv2 outputs (x = 20 or y = 20) and rows 441..511 stay zero, so the b = 1
//       operand of an image's first step and the padding rows of its last step read zeros.  Two dY images alternate, so
//       the data gradient of image j + 1 runs under the weight gradient of image j.
//   B  (N = 128, MN-major SWIZZLE_128B): X16, an fp16 image of the step's pixels, one 128-byte row (64 channels) per
//       position k0 .. k0 + 128.  The h = 1 atom is the same rows one position on: LBO = 128 B.
//   X  : the row-major frames [img][441][64] u8 that conv1 forward reads, as pair rows of 128 B: per step two TMA boxes
//        of 33 pair rows (positions k0 + 64 hb .. k0 + 64 hb + 65).  Position 441 of an image is the first pixel of the
//        next one (the second half of pair row 220) and pair rows >= 221 are zero-filled: both meet zero dY rows.
//   dY : d(act1) on the 21x21 grid, fp16 [img][441][32] scaled by 2^12 (saturating conversion).
//   Warpgroup 3 expands the bytes to X16 with PRMTs (bytes (x, 0x64) = fp16 1024 + x; the offset is taken out again
//   through the bias partial) one step ahead of the MMAs, which warpgroup 2 issues.  After publishing an image, warpgroup
//   1 accumulates the bias gradient (column sums of dY) from it.  Partial tiles go to ws[cta][256][64] / wsb[cta][64]
//   (first 32 columns used; row = tap * 64 + c) and are folded in fixed order by tc_fold_win.
// Every output is bit-identical to the conv2 data gradient on tc_conv_win followed by a conv1 weight gradient that reads
// d(act1) back: the same bf16 / fp16 products, the same fp32 accumulation order, the same CTA row ranges.
struct Conv21BwdU8Params {
    const int64_t* rows;       // optional image gather (minibatch rows of the rollout)
    int n;                     // images of the minibatch
    int64_t rows_per_cta;      // multiple of 512 grid rows = whole images (M = n * 512)
    const bf16* w2dg;          // conv2 data-gradient weights [128][4 taps x 64] (tc_pack_conv_s2_classes)
    const uint32_t* m1;        // act1 > 0 bits: [n,100 cells] x 4 words
    float* ws;
    float* wsb;
};
// u8 blocks of 33 pair rows (half a step and the h = 1 halo) in flight, and two fp16 pixel images of 129 rows (136: the
// 1 KB swizzle period); with the resident conv2 weights (64 KB), two d(act2) windows and two dY images they fill the 227 KB
// of shared memory
constexpr int kC1WXStages = 4, kC21WinStages = 2;
constexpr int kC1WXRows = 33, kC1WXBytes = kC1WXRows * 128, kC1WF16Bytes = 136 * 128;
constexpr int kC1WYBytes = 128 * 64, kC1WYPadRows = 24, kC1WYPad = kC1WYPadRows * 64;
constexpr int kC1WShift = 21;                     // grid rows between the two tap groups
constexpr int kC21WinRows = 140, kC21WinBytes = 18 * 1024;      // 128 rows + the largest tap shift (12), 1 KB aligned
constexpr int kC21W2Bytes = 4 * 128 * 128;                       // 4 taps x 128 output columns x 64 channels (bf16)
constexpr int kC21ImgBytes = kC1WYPad + 4 * kC1WYBytes;          // zero halo + 512 rows of 64 B
constexpr int kC21MaskBytes = 100 * 16;                           // act1 > 0 bits of one image: 100 cells x 4 words
constexpr size_t kC21Smem = (size_t)kC21W2Bytes + (size_t)kC21WinStages * (kC21WinBytes + kC21MaskBytes) + 2 * (size_t)kC21ImgBytes +
                            2 * (size_t)kC1WF16Bytes + (size_t)kC1WXStages * kC1WXBytes + 1024;
static_assert(kC21Smem + 4608 <= 227 * 1024, "conv21_bwd: shared memory exceeds 227 KB");
static_assert((kC21W2Bytes + kC21WinStages * kC21WinBytes + 2 * kC21ImgBytes) % 1024 == 0, "the fp16 images need 1 KB alignment");
constexpr float kDact1Scale = 4096.0f;

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
}
// uint8 x -> fp16 1024 + x: 0..255 stay exact; sum_k (1024 + x) dY = dW + 1024 sum_k dY, and sum_k dY is the bias partial
// the same CTA computes anyway, so the drain subtracts 1024 x it (fp32; the offset costs < 1e-5 relative accuracy).
constexpr float kU8Bias = 1024.0f;
// 16 pixels -> two 16-byte chunks of fp16 1024 + x (pixels 0-7, 8-15): one PRMT per two pixels
__device__ __forceinline__ void u8x16_to_f16_biased(const uint4& v, uint4& lo, uint4& hi) {
    constexpr uint32_t k64 = 0x64646464u;
    lo = make_uint4(prmt(v.x, k64, 0x5140u), prmt(v.x, k64, 0x7362u), prmt(v.y, k64, 0x5140u), prmt(v.y, k64, 0x7362u));
    hi = make_uint4(prmt(v.z, k64, 0x5140u), prmt(v.z, k64, 0x7362u), prmt(v.w, k64, 0x5140u), prmt(v.w, k64, 0x7362u));
}
// 16 bytes at a shared-memory address.  The staging pointers come from the 1 KB-aligned dynamic shared memory through an
// integer cast, so plain dereferences compile to generic 64-bit loads; these are LDS.128 / STS.128 with 32-bit addresses.
// volatile + memory: the accesses stay between the mbarrier wait that publishes a buffer and the arrive that releases it.
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// fp32 pair -> fp16x2, saturating to +-65504 (d(act1) x kDact1Scale never becomes inf)
__device__ __forceinline__ uint32_t pack_f16x2_sat(float lo, float hi) {
    uint32_t d;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}

__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
// TMA store of a shared-memory box (bulk-group completion); wait_read<N>: at most N groups may still be reading shared memory
__device__ __forceinline__ void tma_store_3d(const void* tmap, uint32_t smem_src, int x, int y, int z) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];"
                 ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(x), "r"(y), "r"(z), "r"(smem_src) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// bulk copy global -> shared (16-byte aligned, a multiple of 16 bytes); completion is signalled on `bar` (complete_tx)
__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// 512 threads: warp 0 = pixel producer, warp 1 = d(act2) window producer (warps 2-3 idle: warpgroup alignment), warpgroup
// 1 = conv2 data gradient + bias sums, warpgroup 2 = weight-gradient wgmma, warpgroup 3 = uint8 -> fp16 pixel expansion.
// Every warpgroup keeps the 128 registers per thread the launch gives it (the wgmma warpgroups hold 64 accumulators each).
constexpr int kC1WThreads = 512;
__global__ void __launch_bounds__(kC1WThreads, 1) tc_conv21_bwd_u8(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmWin,
                                                                 const __grid_constant__ CUtensorMap tmY, const Conv21BwdU8Params p) {
    constexpr int XS = kC1WXStages, WS = kC21WinStages;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t xfull[XS], xempty[XS], wfull[WS], wempty[WS], yfull[2], yempty[2], ffull[2], fempty[2];
    __shared__ float sRed[32 * 32], sBias[32];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sW2 = smem;                                       // conv2 data-gradient weights, 4 taps x 16 KB
    uint8_t* sWin = sW2 + kC21W2Bytes;                         // WS d(act2) windows
    uint8_t* sImg = sWin + (size_t)WS * kC21WinBytes;          // 2 dY images (512-B aligned: the SWIZZLE_64B pattern)
    uint8_t* sF = sImg + 2 * (size_t)kC21ImgBytes;             // 2 fp16 pixel images (1 KB aligned: SWIZZLE_128B)
    uint8_t* sX = sF + 2 * (size_t)kC1WF16Bytes;               // XS u8 blocks of 33 pair rows (unswizzled)
    uint8_t* sM = sX + (size_t)XS * kC1WXBytes;                // WS images of act1 mask bits, one per d(act2) window
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        // a u8 block is released by the four expansion warps, a window by the four data-gradient warps, an fp16 image and
        // a dY image by the four wgmma warps once the MMAs that read them have completed
        for (int s = 0; s < XS; ++s) { mbar_init(&xfull[s], 1); mbar_init(&xempty[s], 4); }
        for (int s = 0; s < WS; ++s) { mbar_init(&wfull[s], 1); mbar_init(&wempty[s], 4); }
        for (int s = 0; s < 2; ++s) {
            mbar_init(&yfull[s], 1); mbar_init(&yempty[s], 4);
            mbar_init(&ffull[s], 4); mbar_init(&fempty[s], 4);
        }
        fence_barrier_init();
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmWin);
        tma_prefetch_desc(&tmY);
    }
    for (int idx = tid; idx < 4 * 128 * 8; idx += blockDim.x) {          // W2dg [128][256] -> 4 K-major SWIZZLE_128B taps
        const int c16 = idx & 7, r = (idx >> 3) & 127, t = idx >> 10;
        *reinterpret_cast<int4*>(sW2 + t * (128 * 128) + img_off(r, c16)) = ldg16(p.w2dg + r * 256 + t * 64 + c16 * 8);
    }
    for (int idx = tid; idx < 2 * kC21ImgBytes / 16; idx += blockDim.x) reinterpret_cast<int4*>(sImg)[idx] = make_int4(0, 0, 0, 0);
    fence_proxy_async_smem();
    __syncthreads();
    // every CTA owns at least one whole image (launch_conv21_bwd_u8 checks it): nsteps >= 4
    const int64_t M = (int64_t)p.n * 512;
    const int64_t m_begin = (int64_t)blockIdx.x * p.rows_per_cta;
    int64_t m_end = m_begin + p.rows_per_cta;
    if (m_end > M) m_end = M;
    const int nsteps = (int)((m_end - m_begin) >> 7);
    const int nimg = nsteps >> 2;
    const int img0 = (int)(m_begin >> 9);

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            // =================== TMA producer 1: the pixels of step k (image-aligned: step k & 3 of its image) as two
            // blocks of 33 pair rows, positions 128 (k & 3) + 64 hb .. + 65 (rows >= 221 are zero-filled)
            auto image_of = [&](int j) -> int { return p.rows ? (int)__ldg(p.rows + img0 + j) : img0 + j; };
            int z = 0, z_next = image_of(0);                   // the gather index is fetched one image ahead
            for (int k = 0; k < nsteps; ++k) {
                if ((k & 3) == 0) {
                    z = z_next;
                    if ((k >> 2) + 1 < nimg) z_next = image_of((k >> 2) + 1);
                }
#pragma unroll
                for (int hb = 0; hb < 2; ++hb) {
                    const int j = 2 * k + hb, xs = j % XS;
                    if (j >= XS) mbar_wait(&xempty[xs], ((j / XS) - 1) & 1);
                    mbar_arrive_expect_tx(&xfull[xs], (uint32_t)kC1WXBytes);
                    tma_load_3d(smem_u32(sX + (size_t)xs * kC1WXBytes), &tmX, 0, (k & 3) * 64 + hb * 32, z, &xfull[xs]);
                }
            }
        } else if (warp == 1 && lane == 0) {
            // =================== TMA producer 2: the d(act2) window of image j (rows 121 i .. 121 i + 139 of the padded
            // 11x11 grids; rows past the last image are zero-filled) and the image's act1 mask bits, which the epilogue
            // would otherwise wait for from HBM
            for (int j = 0; j < nimg; ++j) {
                const int s = j % WS;
                if (j >= WS) mbar_wait(&wempty[s], ((j / WS) - 1) & 1);
                mbar_arrive_expect_tx(&wfull[s], (uint32_t)(kC21WinRows * 128 + kC21MaskBytes));
                tma_load_2d(smem_u32(sWin + (size_t)s * kC21WinBytes), &tmWin, 0, (img0 + j) * 121, &wfull[s]);
                bulk_load(smem_u32(sM + (size_t)s * kC21MaskBytes), p.m1 + (int64_t)(img0 + j) * 100 * 4, (uint32_t)kC21MaskBytes, &wfull[s]);
            }
        }
    } else if (warp < 8) {
        // ======================= conv2 data gradient of image j into dY image j & 1, then the bias sums of that image
        const int wt = tid - 128, lane4 = lane >> 2, qd = lane & 3;
        const uint32_t w_base = smem_u32(sW2);
        const int rq = wt >> 2, c16 = wt & 3;                // bias sums: row group and 16-byte chunk of a 64-byte row
        float bsum[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) bsum[e] = 0.f;
        for (int j = 0; j < nimg; ++j) {
            const int i = img0 + j, buf = j & 1, s = j % WS;
            const uint32_t img = smem_u32(sImg + (size_t)buf * kC21ImgBytes) + kC1WYPad;     // row 0 of the image
            const uint32_t masks = smem_u32(sM + (size_t)s * kC21MaskBytes);
            mbar_wait(&wfull[s], (j / WS) & 1);
            // image j - 2 has left dY image `buf`: the weight gradient consumed it and its TMA store has read it
            if (j >= 2) mbar_wait(&yempty[buf], ((j >> 1) - 1) & 1);
            if (wt == 0) bulk_wait_read<1>();
            named_bar(1, 128);
#pragma unroll 1
            for (int h2 = 0; h2 < 2; ++h2) {
                float d[64];
                wgmma_fence();
                const uint32_t win = smem_u32(sWin + (size_t)s * kC21WinBytes) + (uint32_t)(h2 * 64 * 128);
                // taps t = (a, b): row shift (1 - a) * 11 + (1 - b), the order of tc_conv_win
                constexpr int shift[4] = {12, 11, 1, 0};
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const uint64_t a = desc_kmajor(win + (uint32_t)shift[t] * 128u);
                    const uint64_t b = desc_kmajor(w_base + (uint32_t)(t * 128 * 128));
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) WgmmaBf16<128, 0, 0>::mma(d, a + 2 * kk, b + 2 * kk, (t | kk) != 0 ? 1u : 0u);
                }
                wgmma_commit();
                // this thread's rows r and r + 8 of the 11x11 grid: cell (Y, X) and its mask words
                int pos[2];
                uint4 mb[2];
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const int r = h2 * 64 + ((wt >> 5) << 4) + lane4 + 8 * hr;
                    const int Y = (r * 5958) >> 16, X = r - Y * 11;           // r / 11 for r < 128
                    const bool valid = Y < 10 && X < 10;
                    pos[hr] = valid ? 2 * Y * 21 + 2 * X : -1;
                    mb[hr] = make_uint4(0u, 0u, 0u, 0u);
                    if (valid) mb[hr] = lds128(masks + (uint32_t)(Y * 10 + X) * 16u);
                }
                wgmma_wait<0>();
                wgmma_fence_operands(d);
                // epilogue on the accumulator fragment: column 8 jj + 2 qd (+1) = channel 8 (jj & 3) + 2 qd of class
                // g = jj >> 2 = (py, px), stored at grid position (2 Y + py, 2 X + px) of the dY image
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    if (pos[hr] < 0) continue;
                    const uint32_t mw[4] = {mb[hr].x, mb[hr].y, mb[hr].z, mb[hr].w};
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) {
                        const int g = jj >> 2, c = 8 * (jj & 3) + 2 * qd;
                        float f0 = d[4 * jj + 2 * hr] * kDact1Scale, f1 = d[4 * jj + 2 * hr + 1] * kDact1Scale;
                        if (!((mw[g] >> c) & 1u)) f0 = 0.f;
                        if (!((mw[g] >> (c + 1)) & 1u)) f1 = 0.f;
                        const int q = pos[hr] + (g >> 1) * 21 + (g & 1);
                        sts32(img + img64_off(q, c >> 3) + (uint32_t)((c & 7) * 2), pack_f16x2_sat(f0, f1));
                    }
                }
                // the window and the mask bits of this image have been read
                __syncwarp();
                if (h2 == 1 && lane == 0) mbar_arrive(&wempty[s]);
            }
            // publish: the wgmma operand reads and the TMA store are async-proxy reads of what this warpgroup just wrote
            fence_proxy_async_smem();
            named_bar(1, 128);
            if (wt == 0) {
                mbar_arrive(&yfull[buf]);
#pragma unroll
                for (int k = 0; k < 4; ++k) tma_store_3d(&tmY, img + (uint32_t)(k * kC1WYBytes), 0, k * 128, i);
                bulk_commit();
            }
            // bias gradient = column sums of dY (fp32, fixed order: step by step, 32 rows apart per thread)
#pragma unroll 1
            for (int st = 0; st < 4; ++st) {
#pragma unroll
                for (int ps = 0; ps < 4; ++ps) {
                    const uint4 v = lds128(img + (uint32_t)(st * kC1WYBytes) + img64_off(ps * 32 + rq, c16));
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[e]));
                        bsum[2 * e] += f.x;
                        bsum[2 * e + 1] += f.y;
                    }
                }
            }
        }
        if (wt == 0) bulk_wait<0>();
#pragma unroll
        for (int e = 0; e < 8; ++e) sRed[rq * 32 + c16 * 8 + e] = bsum[e];
        named_bar(1, 128);
        if (wt < 32) {
            float t = 0.f;
#pragma unroll
            for (int l = 0; l < 32; ++l) t += sRed[l * 32 + wt];
            p.wsb[(int64_t)blockIdx.x * 64 + wt] = t;
            // what the 1024 offset of every pixel added to each (tap, c) row: the CTA owns whole images, so the rows of the
            // b = 1 operand (shifted by 21, zero outside the image) sum to the same value as the rows of the b = 0 operand
            sBias[wt] = t * kU8Bias;
        }
        named_bar(2, 256);                                  // sBias is ready for the wgmma warpgroup's drain
    } else if (warp < 12) {
        // ======================= wgmma warpgroup: 8 K-steps of 16 positions per step, m64n128k16 with A = the dY rows of
        // both tap groups, B = X16 of both pixel streams.  Every dW element gets the products of the same steps and K16
        // groups as with the pixels on the A side, and scale-d 0 only on the first MMA.
        //   d[4 j + e]: (b, co) = row 16 (wt >> 5) + lane / 4 (+ 8 for e >= 2), (h, c) = column 8 j + 2 qd (+ 1 for odd e)
        const int wt = tid & 127, qd = lane & 3;
        float d[64];
#pragma unroll
        for (int e = 0; e < 64; ++e) d[e] = 0.f;
        auto step = [&](int it) {                            // one batch of 8 MMAs on the images of step it, one commit group
            const int fs = it & 1, buf = (it >> 2) & 1;
            if ((it & 3) == 0) mbar_wait(&yfull[buf], (it >> 3) & 1);
            mbar_wait(&ffull[fs], (it >> 1) & 1);
            wgmma_fence();
            const uint32_t ystep = smem_u32(sImg + (size_t)buf * kC21ImgBytes) + (uint32_t)(kC1WYPad + (it & 3) * kC1WYBytes);
            const uint64_t ad = desc_mnmajor_sw64(ystep - kC1WShift * 64, kC1WShift * 64);
            const uint64_t bd = desc_mnmajor(smem_u32(sF + (size_t)fs * kC1WF16Bytes), 128);
            // K-step kk: 16 dY rows (1 KB, + 64 in the address field) and 16 X16 rows (2 KB, + 128)
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) WgmmaF16N128<1, 1>::mma(d, ad + 64 * kk, bd + 128 * kk, (it | kk) != 0 ? 1u : 0u);
            wgmma_commit();
        };
        // Step it-1's fp16 image (and, after an image's last step, its dY image) is released once step it's batch has been
        // issued and step it-1's MMAs have completed (wgmma_wait<1>), so the tensor pipe does not drain between steps.  The
        // last step is peeled: its MMAs, the final wait and the accumulator stores then share one basic block.
        for (int it = 0; it + 1 < nsteps; ++it) {
            step(it);
            wgmma_wait<1>();
            if (it > 0 && lane == 0) {
                mbar_arrive(&fempty[(it - 1) & 1]);
                if (((it - 1) & 3) == 3) mbar_arrive(&yempty[((it - 1) >> 2) & 1]);
            }
        }
        step(nsteps - 1);
        wgmma_wait<0>();
        wgmma_fence_operands(d);
        named_bar(2, 256);
        // accumulator element ((b, co), (h, c)) -> ws[cta][(2 b + h) * 64 + c][co], the layout of the channels on M; rows
        // 0-31 of the tile are b = 1, rows 32-63 b = 0
        const int m = ((wt >> 5) << 4) + (lane >> 2), b = m < 32 ? 1 : 0, co = m & 31;
        const float bias0 = sBias[co], bias8 = sBias[co + 8];
        float* wsc = p.ws + (int64_t)blockIdx.x * 256 * 64;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int h = j >> 3, c = 8 * (j & 7) + 2 * qd;
            float* q = wsc + (int64_t)((2 * b + h) * 64 + c) * 64 + co;
            q[0] = d[4 * j] - bias0;
            q[64] = d[4 * j + 1] - bias0;
            q[8] = d[4 * j + 2] - bias8;
            q[64 + 8] = d[4 * j + 3] - bias8;
        }
    } else {
        // ======================= pixel expansion, one step ahead of the MMAs: X16 row r = position k0 + r, r = 0 .. 128,
        // from block hb = r / 64 (row 128, the h = 1 halo, is position 64 of the second block).  Thread wt expands the
        // 16-byte chunks t = wt + 128 i (position t / 4 of the block, channels 16 (t & 3) ..) into chunks 2 (t & 3) and
        // 2 (t & 3) + 1 of the row; 8 consecutive threads read 128 contiguous bytes and write two whole rows.
        const int wt = tid & 127;
        for (int it = 0; it < nsteps; ++it) {
            const int fs = it & 1;
            const uint32_t img = smem_u32(sF + (size_t)fs * kC1WF16Bytes);
            if (it >= 2) mbar_wait(&fempty[fs], ((it >> 1) - 1) & 1);
#pragma unroll
            for (int hb = 0; hb < 2; ++hb) {
                const int j = 2 * it + hb, xs = j % XS;
                const uint32_t blk = smem_u32(sX + (size_t)xs * kC1WXBytes);
                const int nch = (64 + hb) * 4;               // 16-byte chunks used from this block
                mbar_wait(&xfull[xs], (j / XS) & 1);
                uint4 v[3];
#pragma unroll
                for (int i = 0; i < 2 + hb; ++i)
                    if (wt + 128 * i < nch) v[i] = lds128(blk + (uint32_t)(wt + 128 * i) * 16u);
#pragma unroll
                for (int i = 0; i < 2 + hb; ++i) {
                    const int t = wt + 128 * i;
                    if (t < nch) {
                        const int r = 64 * hb + (t >> 2), c = t & 3;
                        uint4 lo, hi;
                        u8x16_to_f16_biased(v[i], lo, hi);
                        sts128(img + (uint32_t)(r * 128 + (((2 * c) ^ (r & 7)) << 4)), lo);
                        sts128(img + (uint32_t)(r * 128 + (((2 * c + 1) ^ (r & 7)) << 4)), hi);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&xempty[xs]);
            }
            // publish: the wgmma operand reads are async-proxy reads of what this warp just wrote
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(&ffull[fs]);
        }
    }
}

// dact2b: d(act2) on the zero-padded 11x11 grids [n,121,64] bf16; dact1: fp16 x kDact1Scale [n,441,32] (written here);
// frames_rm: the row-major uint8 frames [n_images][441][64] (conv1 forward's input)
static int launch_conv21_bwd_u8(const Conv21BwdU8Params& p, const void* frames_rm, int64_t n_images, const bf16* dact2b, void* dact1_f16,
                                int ctas, cudaStream_t s, const char* what) {
    int rc;
    if (p.rows_per_cta % 512 != 0) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: a CTA must own whole images (512 grid rows)", what);
    if (ctas < 1 || (int64_t)(ctas - 1) * p.rows_per_cta >= (int64_t)p.n * 512)
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: every CTA must own at least one image", what);
    CUtensorMap tmX, tmWin, tmY;
    memset(&tmX, 0, sizeof(tmX)); memset(&tmWin, 0, sizeof(tmWin)); memset(&tmY, 0, sizeof(tmY));
    // frames as pair rows [img][221][128 B]: box = 33 pair rows, unswizzled; d(act2) rows [n * 121][64 ch] bf16: box = 140
    // rows, SWIZZLE_128B; dY [img][441 rows][32 co] fp16 = 64-byte rows: box [128 rows][64 B], SWIZZLE_64B (stores; rows
    // >= 441 of a box are not written)
    if ((rc = make_tmap_pairs_u8(&tmX, frames_rm, n_images, kC1WXRows, false, what))) return rc;
    if ((rc = make_tmap_2d(&tmWin, dact2b, (int64_t)p.n * 121, 64, kC21WinRows, what))) return rc;
    if ((rc = make_tmap_3d_u8(&tmY, dact1_f16, p.n, 441, 64, 64, 128, 64, what))) return rc;
    static SmemAttrCache attr;
    if ((rc = attr.ensure(tc_conv21_bwd_u8, kC21Smem, what))) return rc;
    tc_conv21_bwd_u8<<<ctas, kC1WThreads, kC21Smem, s>>>(tmX, tmWin, tmY, p);
    return check_launch(what);
}

constexpr int kConv1I8Stages = 8;
static int launch_conv1_i8(const Conv1U8Params& p, const void* frames_rm, cudaStream_t s, const char* what) {
    constexpr int STAGES = kConv1I8Stages;
    const size_t smem = (size_t)4 * 64 * 64 + (size_t)STAGES * 144 * 128 + 1024;
    const int total = p.n * 2;                     // 2 tiles of 128 pair rows (256 grid positions) per image (441 used)
    int grid = num_sms();
    if (grid > total) grid = total;
    CUtensorMap tmA, tmW;
    memset(&tmA, 0, sizeof(tmA));
    memset(&tmW, 0, sizeof(tmW));
    // the row-major image [441][64 B] viewed as 221 pair rows of 128 B (image stride 28 224 B = 220.5 rows: the second
    // half of row 220 belongs to the next image and only ever feeds invalid positions); SWIZZLE_128B boxes of 144 rows
    int rc = make_tmap_pairs_u8(&tmA, frames_rm, p.n_images, 144, true, what);
    if (rc) return rc;
    // the limbs [64 rows][4 taps x 64 B]: one SWIZZLE_64B box [64 rows][64 B] per tap
    if ((rc = make_tmap_3d_u8(&tmW, p.limbs, 1, 64, 256, 256, 64, 64, what))) return rc;
    static SmemAttrCache attr;
    if ((rc = attr.ensure(tc_conv1_i8<STAGES>, smem, what))) return rc;
    tc_conv1_i8<STAGES><<<grid, kConv1I8Threads, smem, s>>>(tmA, tmW, p, total);
    return check_launch(what);
}

}  // namespace b200rl
