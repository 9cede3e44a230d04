// conv1 straight from the uint8 rollout (no 16-bit copy of the frames anywhere).
//
// The rollout keeps every frame ONCE as uint8 space-to-depth(4) pixels, 28 224 B per frame (the algorithmic
// minimum; reference: a 14.8 GB fp32 buffer, ppo_atari_envpool.py:203):
//     frames    u8 [img][441 grid rows][64 ch]   row-major    -> forward  (K-major operand rows)
//     frames_t  u8 [img][64 ch][448 grid rows]   channel-major -> weight gradient (lanes = channels, K = rows)
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
// Weight gradient  tc_conv1_wgrad_u8: dW[tap, c, co] = sum_p X[p + off_tap, c] * dY[p, co].  The pixels go
//   uint8 (shared memory, channel-major TMA box) -> fp16 pairs in REGISTERS (one PRMT per two pixels builds
//   1024 + x; the offset is removed once per CTA through the bias partial), and are consumed as the A operand straight
//   from registers (wgmma with A in registers); dY rows are SWIZZLE_64B TMA boxes used as an MN-major B operand with
//   N = 32, read at two row offsets (0 and -21) so that one A fragment serves all four taps.  No 16-bit image of the
//   frames ever exists in shared or global memory.
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
// MN-major SWIZZLE_64B operand with ONE 32-element (64-byte) MN atom: rows = K index, 8-row K groups 512 B apart
__device__ __forceinline__ uint64_t desc_mnmajor_sw64(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (32ull << 32) | kDescSwizzle64;
}
// byte offset of 16-byte chunk c (0..3) of row r in a SWIZZLE_64B image (address bits [4,6) ^= bits [7,9))
__device__ __forceinline__ uint32_t img64_off(int r, int c) { return (uint32_t)(r * 64 + ((c ^ ((r >> 1) & 3)) << 4)); }
// ------------------------------------------------------------------------------------ frame conversion (once per env step)
// uint8 frames [n,4,84,84] (NCHW, as the env delivers them) -> row-major u8 [n,441,64] and channel-major u8 [n,64,448]
// space-to-depth(4) pixels: channel = c*16 + sy*4 + sx of source pixel (4Y+sy, 4X+sx), grid row = Y*21 + X.
// One block per (frame, colour plane c): the 84x84 plane is staged in shared memory (coalesced 16-byte reads).
__global__ void __launch_bounds__(256) tc_frames_to_s2d_u8(const uint8_t* __restrict__ obs, const int64_t* __restrict__ rows, int64_t n,
                                                           uint8_t* __restrict__ out_rm, uint8_t* __restrict__ out_cm) {
    __shared__ __align__(16) uint8_t plane[7056];
    const int64_t i = blockIdx.x >> 2;
    const int c = blockIdx.x & 3;
    const int64_t img = rows ? rows[i] : i;
    const int4* src = reinterpret_cast<const int4*>(obs + img * 28224 + c * 7056);
    for (int t = threadIdx.x; t < 441; t += 256) reinterpret_cast<int4*>(plane)[t] = __ldg(src + t);
    __syncthreads();
    // row-major: 16 bytes (4 rows of 4 pixels) per grid position
    for (int pos = threadIdx.x; pos < 441; pos += 256) {
        const int Y = pos / 21, X = pos - Y * 21;
        const uint8_t* p = plane + (Y * 4) * 84 + X * 4;
        int4 v;
        v.x = *reinterpret_cast<const int*>(p); v.y = *reinterpret_cast<const int*>(p + 84);
        v.z = *reinterpret_cast<const int*>(p + 168); v.w = *reinterpret_cast<const int*>(p + 252);
        *reinterpret_cast<int4*>(out_rm + (i * 441 + pos) * 64 + c * 16) = v;
    }
    // channel-major: channel (sy, sx) of this plane, 4 consecutive grid rows per 32-bit store (448-byte rows, zero tail)
    for (int t = threadIdx.x; t < 16 * 112; t += 256) {
        const int ch = t / 112, q = t - ch * 112;
        const int sy = ch >> 2, sx = ch & 3;
        uint32_t w = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int pos = q * 4 + e;
            if (pos < 441) {
                const int Y = pos / 21, X = pos - Y * 21;
                w |= (uint32_t)plane[(Y * 4 + sy) * 84 + X * 4 + sx] << (8 * e);
            }
        }
        *reinterpret_cast<uint32_t*>(out_cm + (i * 64 + c * 16 + ch) * 448 + q * 4) = w;
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
__global__ void __launch_bounds__(kConv1I8Threads, 1) tc_conv1_i8(const __grid_constant__ CUtensorMap tmA, const Conv1U8Params p, int total_tiles) {
    constexpr int BN = 64, WR = 144, NTAPS = 4;
    constexpr int STAGE_BYTES = WR * 128;           // 18432 = 18 x 1024
    constexpr int B_CHUNK = BN * 64;                // one tap of the limb image: 64 rows x 64 B (SWIZZLE_64B)
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
    __shared__ __align__(16) float s_sc[32], s_bias[32];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, warp = tid >> 5;
    uint8_t* sW = smem;                             // 4 taps x 4096 B
    uint8_t* sRing = smem + NTAPS * B_CHUNK;        // 16384: 1024-aligned

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // 8 consumer warps
        fence_barrier_init();
        tma_prefetch_desc(&tmA);
    }
    for (int idx = tid; idx < NTAPS * BN * 4; idx += blockDim.x) {          // 16-byte chunks of the limb image
        const int c16 = idx & 3;
        const int t = (idx >> 2) & 3;
        const int r = idx >> 4;
        *reinterpret_cast<int4*>(sW + t * B_CHUNK + img64_off(r, c16)) = ldg16(p.limbs + r * 256 + t * 64 + c16 * 16);
    }
    if (tid < 32) { s_sc[tid] = p.sc[32 + tid]; s_bias[tid] = p.bias[tid]; }      // sc[32 + co] = s_co / 2^14 / 255
    fence_proxy_async_smem();
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

// ------------------------------------------------------------------------------------ conv1 weight gradient (uint8 frames -> registers)
// dW[tap, c, co] = sum_p X[p + off_tap, c] * dY[p, co] over the grid positions p of an image, off = {0, 1, 21, 22}
// (taps (dy, dx) of the 2x2 window on the 21-wide grid).  Written over k = p + s_b with s_b = {0, 21}:
//       D_b[(h, c), co] = sum_k X[k + h, c] * dY[k - s_b, co],    tap = 2 b + h.
//   A  (registers, 64 rows x 16 K per wgmma): warpgroup h holds channel c of the pixel stream X[k + h] as fp16 fragments;
//       one fragment per K-step serves both tap groups b.
//   B  (shared memory, MN-major SWIZZLE_64B, N = 32): the dY rows of the step, rows [k0, k0 + 128) for b = 0 and rows
//       [k0 - 21, k0 + 107) for b = 1.  The stages form one contiguous ring, so the b = 1 operand is the same tile with its
//       descriptor start moved 21 rows back into the previous stage (the swizzle is a function of the address bits);
//       stage 0 is preceded by a 24-row pad that receives the previous rows by a second small TMA box.  Negative rows and
//       rows >= 441 are zero-filled by the TMA unit: images are independent and occupy 512-row slots, and a CTA owns whole
//       images.
//   X  : channel-major frames [img][64 ch][448 rows] u8, staged in blocks of 128 positions (SWIZZLE_128B boxes of 64 full
//        lines).  The h = 1 stream needs one pixel of the next block.
//   dY : d(act1) on the 21x21 grid, fp16 [img][441][32] scaled by 2^12 (written by conv2's data gradient with a
//        saturating conversion); rows of invalid positions (x = 20 or y = 20) are zero.
//   The wgmma warps read their channel rows with 16-byte loads and expand uint8 -> fp16 with PRMTs (bytes (x, 0x64) =
//   fp16 1024 + x; the offset is taken out again through the bias partial).  Four more warps accumulate the bias gradient
//   (column sums of dY) from the staged tiles.  Partial tiles go to ws[cta][256][64] / wsb[cta][64] (first 32 columns
//   used; row = tap * 64 + c) and are folded in fixed order by tc_fold_win.
struct Conv1WgradU8Params {
    const int64_t* rows;       // optional image gather (minibatch rows of the rollout)
    int n;                     // images of the minibatch
    int64_t rows_per_cta;      // multiple of 512 grid rows = whole images (M = n * 512)
    float* ws;
    float* wsb;
};
// X blocks (8 KB: 64 channels x 128 positions) and dY steps (8 KB) in flight: 210 KB per SM, enough loads in flight to
// cover the latency of the gathered reads.
constexpr int kC1WXStages = 12, kC1WYStages = 14;
constexpr int kC1WBlock = 64 * 128, kC1WYBytes = 128 * 64, kC1WYPadRows = 24, kC1WYPad = kC1WYPadRows * 64;
constexpr int kC1WShift = 21;                     // grid rows between the two tap groups
constexpr float kDact1Scale = 4096.0f;

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
}
// uint8 x -> fp16 1024 + x: 0..255 stay exact; sum_k (1024 + x) dY = dW + 1024 sum_k dY, and sum_k dY is the bias partial
// the same CTA computes anyway, so the drain subtracts 1024 x it (fp32; the offset costs < 1e-5 relative accuracy).
constexpr float kU8Bias = 1024.0f;


// fp16 pair (1024 + x[pos], 1024 + x[pos + 1]) from the 20-byte window w[0..4] (pos in 0..15); pos is lane-dependent, so
// the word is picked with selects rather than a (local-memory) indexed array
__device__ __forceinline__ uint32_t pair_f16_biased(const uint32_t (&w)[5], int pos) {
    const int wi = pos >> 2, b = pos & 3;
    const uint32_t lo = wi == 0 ? w[0] : wi == 1 ? w[1] : wi == 2 ? w[2] : w[3];
    const uint32_t hi = wi == 0 ? w[1] : wi == 1 ? w[2] : wi == 2 ? w[3] : w[4];
    const uint32_t x = prmt(lo, hi, (uint32_t)(b | ((b + 1) << 4)));
    return prmt(x, 0x64646464u, 0x5140u);
}

// 512 threads: warp 0 = X producer, warp 1 = dY producer (warps 2-3 idle: warpgroup alignment), warpgroup 1 = bias sums,
// warpgroups 2 and 3 = wgmma for the pixel streams h = 0 and h = 1
constexpr int kC1WThreads = 512;
__global__ void __launch_bounds__(kC1WThreads, 1) tc_conv1_wgrad_u8(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                                                                  const __grid_constant__ CUtensorMap tmYpad, const Conv1WgradU8Params p) {
    constexpr int XS = kC1WXStages, YS = kC1WYStages;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t xfull[XS], xempty[XS], yfull[YS], yempty[YS];
    __shared__ float sRed[32 * 32], sBias[32];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sX = smem;                                 // XS blocks of 8 KB
    uint8_t* sYpad = smem + (size_t)XS * kC1WBlock;     // 24 rows in front of stage 0 (the ring's wrap-around halo)
    uint8_t* sYb = sYpad + kC1WYPad;                    // YS stages of 8 KB, contiguous
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        // X block k is read by all eight wgmma warps as step k's main block and by the four h = 1 warps as step k - 1's halo;
        // a dY stage is released by the eight wgmma warps and the bias group
        for (int s = 0; s < XS; ++s) { mbar_init(&xfull[s], 1); mbar_init(&xempty[s], 12); }
        for (int s = 0; s < YS; ++s) { mbar_init(&yfull[s], 1); mbar_init(&yempty[s], 8 + 1); }
        fence_barrier_init();
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmY);
        tma_prefetch_desc(&tmYpad);
    }
    __syncthreads();
    const int64_t M = (int64_t)p.n * 512;
    const int64_t m_begin = (int64_t)blockIdx.x * p.rows_per_cta;
    int64_t m_end = m_begin + p.rows_per_cta;
    if (m_end > M) m_end = M;
    const int nsteps = m_end > m_begin ? (int)((m_end - m_begin) >> 7) : 0;
    const int64_t g0 = m_begin >> 7;                       // first global step (4 steps per image)

    if (warp == 0) {
        // ======================= TMA producer 1: X block k (k = 0 .. nsteps, the last one only feeds the one-pixel halo)
        if (lane == 0 && nsteps > 0) {
            auto image_of = [&](int64_t g) -> int {
                int64_t img = g >> 2;
                if (img >= p.n) img = p.n - 1;             // the halo block after the very last step: any mapped block will do
                return p.rows ? (int)__ldg(p.rows + img) : (int)img;
            };
            // the gather index is fetched one IMAGE (four steps) ahead
            int z = image_of(g0), z_next = image_of(g0 + 4);        // g0 is image-aligned (whole images per CTA)
            for (int k = 0; k <= nsteps; ++k) {
                const int64_t g = g0 + k;
                if (k > 0 && (g & 3) == 0) { z = z_next; z_next = image_of(g + 4); }
                const int xs = k % XS;
                if (k >= XS) mbar_wait(&xempty[xs], ((k / XS) - 1) & 1);
                mbar_arrive_expect_tx(&xfull[xs], (uint32_t)kC1WBlock);
                tma_load_3d(smem_u32(sX + (size_t)xs * kC1WBlock), &tmX, (int)(g & 3) * 128, 0, z, &xfull[xs]);
            }
        }
    } else if (warp == 1) {
        // ======================= TMA producer 2: the dY rows of step k.  The tail of stage s is read by step k + 1 (b = 1), so
        // stage s is reloaded (step k + YS) once steps k and k + 1 have both been consumed: the ring is YS - 1 steps deep.
        if (lane == 0) {
            for (int k = 0; k < nsteps; ++k) {
                const int64_t g = g0 + k;
                const int ys = k % YS;
                if (k >= YS) mbar_wait2(&yempty[ys], ((k / YS) - 1) & 1, &yempty[(k + 1) % YS], ((k - YS + 1) / YS) & 1);
                mbar_arrive_expect_tx(&yfull[ys], (uint32_t)(kC1WYBytes + (ys == 0 ? kC1WYPad : 0)));
                tma_load_3d(smem_u32(sYb + (size_t)ys * kC1WYBytes), &tmY, 0, (int)(g & 3) * 128, (int)(g >> 2), &yfull[ys]);
                if (ys == 0) tma_load_3d(smem_u32(sYpad), &tmYpad, 0, (int)(g & 3) * 128 - kC1WYPadRows, (int)(g >> 2), &yfull[ys]);
            }
        }
    } else if (warp >= 4 && warp < 8) {
        // ======================= bias warps: bias gradient = column sums of dY from the staged tiles (fp32, fixed order)
        const int tb = tid - 128;
        const int rq = tb >> 2, c16 = tb & 3;
        float bsum[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) bsum[e] = 0.f;
        for (int it = 0; it < nsteps; ++it) {
            const int ys = it % YS;
            if (tb < 32) mbar_wait(&yfull[ys], (it / YS) & 1);
            named_bar(1, 128);
            const uint8_t* sY = sYb + (size_t)ys * kC1WYBytes;          // the step's own rows
#pragma unroll
            for (int ps = 0; ps < 4; ++ps) {
                const int rr = ps * 32 + rq;
                const int4 v = *reinterpret_cast<const int4*>(sY + img64_off(rr, c16));
                const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[e]));
                    bsum[2 * e] += f.x;
                    bsum[2 * e + 1] += f.y;
                }
            }
            named_bar(1, 128);
            if (tb == 0) mbar_arrive(&yempty[ys]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) sRed[rq * 32 + c16 * 8 + e] = bsum[e];
        named_bar(1, 128);
        if (tb < 32) {
            float t = 0.f;
#pragma unroll
            for (int l = 0; l < 32; ++l) t += sRed[l * 32 + tb];
            p.wsb[(int64_t)blockIdx.x * 64 + tb] = t;
            // what the 1024 offset of every pixel added to each (tap, c) row: the CTA owns whole images, so the rows of the
            // b = 1 operand (shifted by 21, zero outside the image) sum to the same value as the rows of the b = 0 operand
            sBias[tb] = t * kU8Bias;
        }
        named_bar(2, 384);                                  // sBias is ready for the wgmma warpgroups' drain
    } else if (warp >= 8) {
        // ======================= wgmma warpgroup h: A = fp16 fragments of the pixel stream X[k + h] built in registers,
        // B = the step's dY rows at offsets 0 (b = 0) and -21 (b = 1); 8 K-steps of 16 positions per step
        const int h = (warp - 8) >> 2, wt = tid & 127, qd = lane & 3;
        const int c0 = ((wt >> 5) << 4) + (lane >> 2);     // fragment rows c0 and c0 + 8 = channels
        float d[2][16];
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int e = 0; e < 16; ++e) d[b][e] = 0.f;
        for (int it = 0; it < nsteps; ++it) {
            const int xm = it % XS, xh = (it + 1) % XS, ys = it % YS;
            mbar_wait(&xfull[xm], (it / XS) & 1);
            if (h == 1) mbar_wait(&xfull[xh], ((it + 1) / XS) & 1);
            uint32_t a[8][4];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int c = c0 + 8 * r;
                const uint8_t* bm = sX + (size_t)xm * kC1WBlock + c * 128;
                const uint8_t* bh = sX + (size_t)xh * kC1WBlock + c * 128;
                const uint32_t sw = (uint32_t)(c & 7);
                int4 cur = *reinterpret_cast<const int4*>(bm + ((0u ^ sw) << 4));
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) {
                    int4 nxt = make_int4(0, 0, 0, 0);
                    if (h == 1) nxt = *reinterpret_cast<const int4*>((kk < 7 ? bm : bh) + ((((uint32_t)(kk + 1) & 7u) ^ sw) << 4));
                    const uint32_t w[5] = {(uint32_t)cur.x, (uint32_t)cur.y, (uint32_t)cur.z, (uint32_t)cur.w, (uint32_t)nxt.x};
                    a[kk][r] = pair_f16_biased(w, 2 * qd + h);              // K 2 qd, 2 qd + 1
                    a[kk][2 + r] = pair_f16_biased(w, 8 + 2 * qd + h);      // K 8 + 2 qd, 9 + 2 qd
                    if (kk < 7) cur = h == 1 ? nxt : *reinterpret_cast<const int4*>(bm + ((((uint32_t)(kk + 1)) ^ sw) << 4));
                }
            }
            // the pixels are in registers: release the X blocks (block 0 has no halo reader, so its h = 1 readers arrive twice)
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&xempty[xm]);
                if (h == 1) { mbar_arrive(&xempty[xh]); if (it == 0) mbar_arrive(&xempty[xm]); }
            }
            mbar_wait(&yfull[ys], (it / YS) & 1);
            wgmma_fence();                                   // the A fragments were just written by ordinary instructions
            const uint32_t y0 = smem_u32(sYb + (size_t)ys * kC1WYBytes);
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
                for (int b = 0; b < 2; ++b)
                    wgmma_f16_rs_n32_tb(d[b], a[kk], desc_mnmajor_sw64(y0 - (uint32_t)(b * kC1WShift * 64)) + 64 * kk,
                                        (it | kk) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&yempty[ys]);
        }
        wgmma_fence_operands(d[0]);
        wgmma_fence_operands(d[1]);
        named_bar(2, 384);
        float* wsc = p.ws + (int64_t)blockIdx.x * 256 * 64;
#pragma unroll
        for (int b = 0; b < 2; ++b) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float* dst = wsc + (int64_t)((2 * b + h) * 64 + c0 + 8 * r) * 64;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int co = 8 * j + 2 * qd;
                    *reinterpret_cast<float2*>(dst + co) =
                        make_float2(d[b][4 * j + 2 * r] - sBias[co], d[b][4 * j + 2 * r + 1] - sBias[co + 1]);
                }
            }
        }
    }
}

static int launch_conv1_wgrad_u8(const Conv1WgradU8Params& p, const void* frames_cm, int64_t n_images, const void* dact1_f16, int ctas,
                                 cudaStream_t s, const char* what) {
    const size_t smem = (size_t)kC1WXStages * kC1WBlock + kC1WYPad + (size_t)kC1WYStages * kC1WYBytes + 1024;
    int rc;
    if (p.rows_per_cta % 512 != 0) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: a CTA must own whole images (512 grid rows)", what);
    CUtensorMap tmX, tmY, tmYpad;
    memset(&tmX, 0, sizeof(tmX)); memset(&tmY, 0, sizeof(tmY)); memset(&tmYpad, 0, sizeof(tmYpad));
    // frames [img][64 ch][448 positions] u8: box = [64 ch][128 positions], SWIZZLE_128B; dY [img][441 rows][32 co] fp16 = 64-byte
    // rows: box [128 rows][64 B], SWIZZLE_64B
    if ((rc = make_tmap_3d_u8(&tmX, frames_cm, n_images, 64, 448, 448, 64, 128, what))) return rc;
    if ((rc = make_tmap_3d_u8(&tmY, dact1_f16, p.n, 441, 64, 64, 128, 64, what))) return rc;
    if ((rc = make_tmap_3d_u8(&tmYpad, dact1_f16, p.n, 441, 64, 64, kC1WYPadRows, 64, what))) return rc;
    static SmemAttrCache attr;
    if ((rc = attr.ensure(tc_conv1_wgrad_u8, smem, what))) return rc;
    tc_conv1_wgrad_u8<<<ctas, kC1WThreads, smem, s>>>(tmX, tmY, tmYpad, p);
    return check_launch(what);
}

constexpr int kConv1I8Stages = 8;
static int launch_conv1_i8(const Conv1U8Params& p, const void* frames_rm, cudaStream_t s, const char* what) {
    constexpr int STAGES = kConv1I8Stages;
    const size_t smem = (size_t)4 * 64 * 64 + (size_t)STAGES * 144 * 128 + 1024;
    const int total = p.n * 2;                     // 2 tiles of 128 pair rows (256 grid positions) per image (441 used)
    int grid = num_sms();
    if (grid > total) grid = total;
    CUtensorMap tmA;
    memset(&tmA, 0, sizeof(tmA));
    // the row-major image [441][64 B] viewed as 221 pair rows of 128 B (image stride 28 224 B = 220.5 rows: the second
    // half of row 220 belongs to the next image and only ever feeds invalid positions); SWIZZLE_128B boxes of 144 rows
    int rc = make_tmap_pairs_u8(&tmA, frames_rm, p.n_images, what);
    if (rc) return rc;
    static SmemAttrCache attr;
    if ((rc = attr.ensure(tc_conv1_i8<STAGES>, smem, what))) return rc;
    tc_conv1_i8<STAGES><<<grid, kConv1I8Threads, smem, s>>>(tmA, p, total);
    return check_launch(what);
}

}  // namespace b200rl
