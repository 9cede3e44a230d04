// wgmma "window" convolution kernel + launcher (see net_tc.cu for the layer plan).
#pragma once
#include "tc_base.cuh"

namespace b200rl {
using namespace tc;

// ------------------------------------------------------------------ kernel 1c: "window" convolution
// Stride-1 convolutions over activations stored as a LINEAR pixel grid [n*G rows, CPR*64 channels]
// (G = Hp*Wp grid positions per image).  GEMM rows enumerate grid positions, so tap (dy,dx) of a row is
// simply the row `dy*Wp+dx` further down: the CTA stages ONE window of 128+maxshift rows per tile and
// every tap is a wgmma operand descriptor whose start address is shifted by whole 128-byte rows
// (the SWIZZLE_128B pattern is a function of the shared-memory address bits, so any row shift is legal).  Each activation row is therefore read from L2 once per tile
// instead of once per tap, and the producers do no im2col index arithmetic at all.  Grid positions whose
// window would leave the image (X >= vW or Y >= vH) are computed but not stored.
enum { WOUT_DENSE = 0, WOUT_S2D2 = 1, WOUT_DACT2 = 2, WOUT_DACT1 = 3 };
struct WinParams {
    const bf16* A;           // [n*G, CPR*64]
    const int64_t* rows;     // optional image gather (conv1 reads the rollout through mb_inds)
    int64_t M;               // n*G
    int n, G, Wp;
    // image-aligned tiling (conv1): every image owns 2^tpi_shift tiles of 128 grid rows (rows >= G are padding),
    // so a window never spans two images and the minibatch gather is just the TMA box's image coordinate.
    // 0 = tiles walk the linear grid [n*G] (activations produced by this library, always contiguous).
    int tpi_shift;
    int64_t n_images;        // images addressable through `rows` (size of the tensor map's outer dimension)
    int ntaps;
    int shift[16];           // dy*Wp + dx per tap (non-negative)
    int WR;                  // window rows: 128 + max shift, rounded up to 8
    const bf16* Bw;          // packed weights [N][ntaps*CPR*64]
    int N;
    int vH, vW;              // valid outputs: Y < vH && X < vW
    int out_mode;
    bf16* out;               // primary output
    bf16* out2;              // WOUT_DACT2: padded 11x11 copy
    // ReLU masks travel as BITS (1 = the forward activation was > 0), one 32-bit word per 32 channels, in the row
    // order of the tensor they describe: 16x fewer bytes than re-reading the bf16 activation
    const uint32_t* mask_bits;   // input mask (data-gradient kernels): words of the row this thread writes
    uint32_t* mask_out;          // output mask (forward kernels with relu)
    const float* bias;
    float scale;
    int relu;
};

// Thread roles (384 threads): warpgroup 0 = TMA producer (warp 0; warps 1-3 only hold the warpgroup alignment that wgmma
// requires); warpgroups 1 and 2 each run wgmma on 64 rows of every 128-row tile (accumulators in registers), hand the
// accumulators to a row-major shared-memory tile and run the epilogue with one thread per row (a second thread per row
// takes the odd 32-column groups).
// The resident weight image arrives by TMA on a barrier of its own, issued right behind the first window: a CTA's first
// MMAs wait for both copies in flight together, not for every thread's share of a load of the whole image first.  At
// the rollout's n = 1024 a CTA runs only a few tiles, so that wait is a visible part of the launch.
constexpr int kConvWinThreads = 384;
template <int BN>
__host__ __device__ constexpr size_t conv_win_acc_bytes() { return (size_t)128 * (BN + 4) * sizeof(float); }
template <int BN, int CPR, int STAGES, int NTAPS>
__global__ void __launch_bounds__(kConvWinThreads, 1) tc_conv_win(const __grid_constant__ CUtensorMap tmA,
                                                                  const __grid_constant__ CUtensorMap tmW, const WinParams p,
                                                                  int total_tiles) {
    constexpr int B_CHUNK = BN * 128;
    constexpr int LDA = BN + 4;                          // fp32 accumulator tile row pitch (conflict-free row reads)
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES], w_bar;
    // aligned by an offset from smem_raw (not through an integer): the accumulator tile's accesses stay shared-memory
    // instructions instead of generic ones
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5;
    const int nchunks = p.ntaps * CPR;
    const int IMG = p.WR * 128;                 // one 64-channel column image of the window
    const int STAGE_BYTES = IMG * CPR;
    uint8_t* sW = smem;
    uint8_t* sRing = smem + (size_t)nchunks * B_CHUNK;
    float* sAcc = reinterpret_cast<float*>(sRing + (size_t)STAGES * STAGE_BYTES);

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // 8 consumer warps
        mbar_init(&w_bar, 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmW);
    }
    __syncthreads();
    // each CTA walks a CONTIGUOUS range of tiles: with the minibatch gather every image (3-4 tiles) is then
    // touched by one SM only (TLB / L2 locality), and the image indices of tile+1 can be prefetched
    const int tile_begin = (int)(((int64_t)total_tiles * blockIdx.x) / gridDim.x);
    const int tile_end = (int)(((int64_t)total_tiles * (blockIdx.x + 1)) / gridDim.x);

    if (warp == 0) {
        // ======================= TMA producer: the window is one rectangular box per 64-channel column chunk ====
        if (tid == 0) {
            uint32_t q = 0;
            const int tmask = (1 << p.tpi_shift) - 1;
            // image-aligned mode: the box's image coordinate is the (optional) minibatch gather; the index of the
            // NEXT tile's image is fetched one tile ahead so the dependent load never delays a TMA issue
            int z_next = 0;
            if (p.tpi_shift && tile_begin < tile_end) {
                const int img = tile_begin >> p.tpi_shift;
                z_next = p.rows ? (int)__ldg(p.rows + img) : img;
            }
            for (int tile = tile_begin; tile < tile_end; ++tile, ++q) {
                const uint32_t s = q % STAGES;
                const int z = z_next;
                if (p.tpi_shift && tile + 1 < tile_end) {
                    const int img = (tile + 1) >> p.tpi_shift;
                    z_next = p.rows ? (int)__ldg(p.rows + img) : img;
                }
                if (q >= (uint32_t)STAGES) mbar_wait(&empty_bar[s], ((q / STAGES) - 1) & 1);
                const uint32_t dst = smem_u32(sRing + (size_t)s * STAGE_BYTES);
                mbar_arrive_expect_tx(&full_bar[s], (uint32_t)STAGE_BYTES);
                if (p.tpi_shift) {
#pragma unroll
                    for (int c = 0; c < CPR; ++c) tma_load_3d(dst + c * IMG, &tmA, c * 64, (tile & tmask) * 128, z, &full_bar[s]);
                } else {
#pragma unroll
                    for (int c = 0; c < CPR; ++c) tma_load_2d(dst + c * IMG, &tmA, c * 64, tile * 128, &full_bar[s]);
                }
                if (q == 0) {       // the weight image, one [BN rows x 64 channels] box per K chunk (rows >= N zero-filled)
                    mbar_arrive_expect_tx(&w_bar, (uint32_t)(nchunks * B_CHUNK));
                    for (int j = 0; j < nchunks; ++j) tma_load_2d(smem_u32(sW + (size_t)j * B_CHUNK), &tmW, j * 64, 0, &w_bar);
                }
            }
        }
    } else if (warp >= 4) {
        // ======================= consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of every tile.  Every tap is a descriptor
        // of the staged window whose start address is shifted by whole 128-byte rows.
        const int wg = (warp - 4) >> 2, wt = tid & 127;
        float* st = sAcc + wg * 64 * LDA;
        const uint32_t w_base = smem_u32(sW);
        const int lr = wt & 63, half = wt >> 6;
        const int lrow = wg * 64 + lr;
        const uint32_t mW = (65536u + (uint32_t)p.Wp - 1u) / (uint32_t)p.Wp;
        const int tmask = (1 << p.tpi_shift) - 1;
        constexpr int NW = BN / 32;                          // 32-column groups = mask words per row
        float d[BN / 2];
#pragma unroll
        for (int e = 0; e < BN / 2; ++e) d[e] = 0.f;
        if (tile_begin < tile_end) mbar_wait(&w_bar, 0);
        for (int tile = tile_begin; tile < tile_end; ++tile) {
            const uint32_t q = (uint32_t)(tile - tile_begin), s = q % STAGES;
            // the row -> (image, Y, X) -> output offset arithmetic, done while the tile's MMAs run
            const int64_t r = (int64_t)tile * 128 + lrow;
            int i = (int)(r / p.G);
            int rem = (int)(r - (int64_t)i * p.G);
            bool inside = r < p.M;
            if (p.tpi_shift) {                               // image-aligned tiles: rows >= G of an image are padding
                i = tile >> p.tpi_shift;
                rem = ((tile & tmask) << 7) + lrow;
                inside = rem < p.G;
            }
            mbar_wait(&full_bar[s], (q / STAGES) & 1);
            wgmma_fence();
            const uint32_t win = smem_u32(sRing + (size_t)s * STAGE_BYTES) + (uint32_t)(wg * 64 * 128);
#pragma unroll
            for (int t = 0; t < NTAPS; ++t) {
#pragma unroll
                for (int c = 0; c < CPR; ++c) {
                    const uint64_t a = desc_kmajor(win + (uint32_t)(c * IMG) + (uint32_t)p.shift[t] * 128u);
                    const uint64_t b = desc_kmajor(w_base + (uint32_t)((t * CPR + c) * B_CHUNK));
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)
                        WgmmaBf16<BN, 0, 0>::mma(d, a + 2 * kk, b + 2 * kk, (t | c | kk) != 0 ? 1u : 0u);
                }
            }
            wgmma_commit();
            const int Y = (int)(((uint32_t)rem * mW) >> 16), X = rem - Y * p.Wp;
            const bool valid = inside && (Y < p.vH) && (X < p.vW);
            int64_t o1 = 0, ob = 0;
            if (p.out_mode == WOUT_S2D2) {
                const int64_t cell = ((int64_t)i * 10 + (Y >> 1)) * 10 + (X >> 1);
                const int cls = (Y & 1) * 2 + (X & 1);
                o1 = cell * 128 + cls * 32; ob = cell * 4 + cls;
            } else {
                ob = ((int64_t)i * 100 + Y * 10 + X) * 4;                  // act1 (2x2 cells) mask words
            }
            // the row's mask words are requested BEFORE waiting for the accumulator (latency overlaps the MMAs)
            uint32_t mb[NW];
#pragma unroll
            for (int g = 0; g < NW; ++g) mb[g] = 0xFFFFFFFFu;
            if (p.mask_bits != nullptr && valid) {
                if (NW == 4) {
                    const int4 t = ldg16(p.mask_bits + ob);
                    mb[0] = (uint32_t)t.x; mb[1 % NW] = (uint32_t)t.y; mb[2 % NW] = (uint32_t)t.z; mb[3 % NW] = (uint32_t)t.w;
                } else if (NW == 2) {
                    const uint2 t = __ldg(reinterpret_cast<const uint2*>(p.mask_bits + ob));
                    mb[0] = t.x; mb[1 % NW] = t.y;
                } else {
                    mb[0] = __ldg(p.mask_bits + ob);
                }
            }
            wgmma_wait<0>();
            wgmma_fence_operands(d);
            if ((tid & 31) == 0) mbar_arrive(&empty_bar[s]);              // this warp's operand reads are complete
            named_bar(1 + wg, 128);                                         // the previous tile's rows have been read
            stage_acc(st, LDA, wt, d);
            named_bar(1 + wg, 128);
#pragma unroll
            for (int g = 0; g < NW; ++g) {
                if ((g & 1) != half) continue;
                if (!valid || g * 32 >= p.N) continue;
                uint32_t v[32];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float4 f = *reinterpret_cast<const float4*>(st + lr * LDA + g * 32 + 4 * e);
                    v[4 * e] = __float_as_uint(f.x); v[4 * e + 1] = __float_as_uint(f.y);
                    v[4 * e + 2] = __float_as_uint(f.z); v[4 * e + 3] = __float_as_uint(f.w);
                }
                if (p.bias) {
                    const float4* bp = reinterpret_cast<const float4*>(p.bias + g * 32);
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
                        const float f = __uint_as_float(v[e]);
                        bits |= (f > 0.f ? 1u : 0u) << e;           // the clamp itself is folded into the bf16 conversion below
                    }
                    if (p.mask_out) p.mask_out[ob + g] = bits;
                }
                if (p.mask_bits) {
#pragma unroll
                    for (int e = 0; e < 32; ++e) if (!((mb[g] >> e) & 1u)) v[e] = 0u;
                }
                int4 w[4];
                if (p.relu) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        w[e].x = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e]), __uint_as_float(v[8 * e + 1]));
                        w[e].y = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e + 2]), __uint_as_float(v[8 * e + 3]));
                        w[e].z = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e + 4]), __uint_as_float(v[8 * e + 5]));
                        w[e].w = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e + 6]), __uint_as_float(v[8 * e + 7]));
                    }
                } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    w[e].x = (int)pack_bf16x2(__uint_as_float(v[8 * e]), __uint_as_float(v[8 * e + 1]));
                    w[e].y = (int)pack_bf16x2(__uint_as_float(v[8 * e + 2]), __uint_as_float(v[8 * e + 3]));
                    w[e].z = (int)pack_bf16x2(__uint_as_float(v[8 * e + 4]), __uint_as_float(v[8 * e + 5]));
                    w[e].w = (int)pack_bf16x2(__uint_as_float(v[8 * e + 6]), __uint_as_float(v[8 * e + 7]));
                }
                }
                if (p.out_mode == WOUT_DACT1) {
                    // packed into the group's own fp32 bytes (already read), at 128 g + 64 (g & 1): the copy below then
                    // reads groups g and g ^ 1 from different bank halves
                    int4* brow = reinterpret_cast<int4*>(st + lr * LDA) + 8 * g + 4 * (g & 1);
#pragma unroll
                    for (int e = 0; e < 4; ++e) brow[e] = w[e];
                } else {
                    // a thread owns one output row: 64 contiguous bytes per 32-column group
                    bf16* dst = p.out + o1 + g * 32;
                    st_global_32b(dst, w[0], w[1]);
                    st_global_32b(dst + 16, w[2], w[3]);
                }
            }
            if (p.out_mode == WOUT_DACT1) {
                // column group g = (py,px) of the cell -> input pixel (2Y+py, 2X+px) of the 21-grid, 32 channels: a cell's
                // groups (py,0) and (py,1) are 128 contiguous bytes.  The row's pixel offset goes in its padding bytes
                // (-1: not stored), then 16 lanes per row store whole 128-byte lines (4 per warp store instead of 32).
                if (half == 0)
                    *reinterpret_cast<int64_t*>(st + lr * LDA + BN) = valid ? ((int64_t)i * 441 + 2 * Y * 21 + 2 * X) * 32 : -1;
                named_bar(1 + wg, 128);
#pragma unroll
                for (int m = 0; m < 8; ++m) {
                    const int k = m * 128 + wt, g = (k >> 2) & 3, e = k & 3;
                    const float* srow = st + (k >> 4) * LDA;
                    const int64_t o = *reinterpret_cast<const int64_t*>(srow + BN);
                    if (o < 0) continue;
                    const int4 val = reinterpret_cast<const int4*>(srow)[8 * g + 4 * (g & 1) + e];
                    *reinterpret_cast<int4*>(p.out + o + (g >> 1) * 21 * 32 + (g & 1) * 32 + e * 8) = val;
                }
            }
        }
    }
}

// conv1 over space-to-depth frames (WOUT_S2D2, Cout 32) and the conv2 data gradient (WOUT_DACT1, Cout 128)
template <int BN, int CPR, int STAGES, int NTAPS>
static int launch_conv_win(const WinParams& p, cudaStream_t s, const char* what) {
    if (p.ntaps != NTAPS) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: %d taps, kernel instance has %d", what, p.ntaps, NTAPS);
    if (p.out_mode != WOUT_S2D2 && p.out_mode != WOUT_DACT1)
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: dense and conv3 data-gradient outputs run on tc_conv_win_t", what);
    if (p.out_mode == WOUT_DACT1 && (BN != 128 || p.N != 128))
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: the conv2 data gradient stores 4 groups of 32 channels per cell", what);
    const size_t smem = (size_t)p.ntaps * CPR * BN * 128 + (size_t)STAGES * p.WR * 128 * CPR + conv_win_acc_bytes<BN>() + 1024;
    static SmemAttrCache attr;
    if (int rc = attr.ensure(tc_conv_win<BN, CPR, STAGES, NTAPS>, smem, what)) return rc;
    if ((int64_t)p.G * p.Wp >= 65536 || p.G < 1 || p.N % 32 != 0)
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: grid %d x width %d outside the epilogue's multiply-shift range, or N %% 32 != 0", what, p.G, p.Wp);
    if (p.rows && !p.tpi_shift) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: the image gather needs image-aligned tiling", what);
    if (p.tpi_shift && (128 << p.tpi_shift) < p.G) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: tiles per image too small", what);
    const int total = p.tpi_shift ? (int)((int64_t)p.n << p.tpi_shift) : (int)ceil_div(p.M, 128);
    int grid = num_sms();
    if (grid > total) grid = total;
    CUtensorMap tmA, tmW;
    memset(&tmA, 0, sizeof(tmA));
    memset(&tmW, 0, sizeof(tmW));
    int rc;
    // the window is a TMA box [WR rows x 64 channels] per column chunk: of the linear grid, or of one image
    if (p.tpi_shift) rc = make_tmap_3d(&tmA, p.A, p.n_images, p.G, (int64_t)CPR * 64, p.WR, what);
    else rc = make_tmap_2d(&tmA, p.A, p.M, (int64_t)CPR * 64, p.WR, what);
    if (rc) return rc;
    if ((rc = make_tmap_2d(&tmW, p.Bw, p.N, (int64_t)NTAPS * CPR * 64, BN, what))) return rc;      // packed [N][K] weights
    tc_conv_win<BN, CPR, STAGES, NTAPS><<<grid, kConvWinThreads, smem, s>>>(tmA, tmW, p, total);
    return check_launch(what);
}

// ------------------------------------------------------------------ kernel 1d: window convolution, channels on the MMA's M side
// The same window convolution with the operand roles swapped, for Cout = 64 (the conv3 data gradient; conv2 and conv3
// forward run fused in tc_conv23_fwd, tc_conv23.cuh, which keeps this kernel's MMA layout and epilogue).  A is the
// resident weight image (M = Cout); B is the staged pixel window, a K-major operand whose descriptor start moves by whole 128-byte rows per tap (N = BP grid positions), so every wgmma is m64nBPk16.  Per
// 64 x BP x 16 step that is 2 KB of weights and BP x 32 B of window from shared memory, against 2 KB + 2 KB per
// 64 x 64 x 16 with positions on M and Cout on N: at BP = 128 the operand traffic drops from 128 B to 96 B per
// tensor-core cycle, under the 128 B per cycle an SM's shared memory delivers.
// The two consumer warpgroups take alternate tiles, each with its own accumulators and stages, so one warpgroup's
// epilogue runs under the other's MMAs; a stage is released as soon as its MMAs have completed.  The epilogue
// transposes the accumulators (rows = channels) through shared memory into position rows and applies exactly the fp32
// operations of tc_conv_win, one thread per position; the packed rows are then stored as whole 128-byte lines by 8 lanes
// per position (DESIGN.md section 4).  Every output is the same bf16 products summed over the same K sequence (taps,
// column chunks, k16 steps in order; the first MMA with scale-d = 0), and the results are bit-identical to tc_conv_win.
// The conv2 data gradient (Cout = 128, K = 256) stays on tc_conv_win: with two m64 halves per warpgroup, its epilogue
// (128 channels per position) outlasts the other warpgroup's MMAs, and it measured about 3 % slower.
constexpr int kConvWinTThreads = 384;
constexpr int kConvWinTLds = 64 + 4;                     // staging pitch (fp32): conflict-free transposed writes and row reads
template <int BP>
__host__ __device__ constexpr size_t conv_win_t_stage_bytes() { return (size_t)2 * BP * kConvWinTLds * sizeof(float); }

// a warpgroup's 64 x BP accumulator fragment (tc_wgmma.cuh) -> st[position][channel]
template <int R>
__device__ __forceinline__ void stage_acc_transposed(float* st, int wg_tid, const float (&d)[R]) {
    const int co = ((wg_tid >> 5) << 4) + ((wg_tid & 31) >> 2), pos = (wg_tid & 3) * 2;
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
        float* p0 = st + (8 * j + pos) * kConvWinTLds + co;
        p0[0] = d[4 * j];
        p0[kConvWinTLds] = d[4 * j + 1];
        p0[8] = d[4 * j + 2];
        p0[kConvWinTLds + 8] = d[4 * j + 3];
    }
}

template <int BP, int CPR, int STAGES, int NTAPS>
__global__ void __launch_bounds__(kConvWinTThreads, 1) tc_conv_win_t(const __grid_constant__ CUtensorMap tmA,
                                                                     const __grid_constant__ CUtensorMap tmW, const WinParams p,
                                                                     int total_tiles) {
    static_assert(BP % 128 == 0, "the epilogue's 128 threads per warpgroup cover whole position rows");
    static_assert(STAGES % 2 == 0, "each consumer warpgroup owns every other stage");
    constexpr int PPR = 128;                             // positions per pass of the warpgroup (one thread per position)
    constexpr int RPT = BP / 128;                        // passes (position rows per epilogue thread)
    constexpr int A_CHUNK = 64 * 128;                    // one 64-channel K chunk of the 64 weight rows
    constexpr int LDS = kConvWinTLds;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES], w_bar;
    // aligned by an offset from smem_raw (not through an integer): the staging tile's accesses stay shared-memory
    // instructions instead of generic ones
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5;
    const int nchunks = NTAPS * CPR;
    const int IMG = p.WR * 128;
    const int STAGE_BYTES = IMG * CPR;
    uint8_t* sW = smem;
    uint8_t* sRing = smem + (size_t)nchunks * A_CHUNK;
    float* sAcc = reinterpret_cast<float*>(sRing + (size_t)STAGES * STAGE_BYTES);

    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // the consuming warpgroup's 4 warps
        mbar_init(&w_bar, 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmW);
    }
    __syncthreads();
    const int tile_begin = (int)(((int64_t)total_tiles * blockIdx.x) / gridDim.x);
    const int tile_end = (int)(((int64_t)total_tiles * (blockIdx.x + 1)) / gridDim.x);

    if (warp == 0) {
        // ======================= TMA producer: one [WR rows x 64 channels] box per column chunk, tiles in order.  The
        // weight image (one [64 rows x 64 channels] box per K chunk, on a barrier of its own) goes out right after the
        // first window, so both are in flight together instead of the window waiting for a load of the whole image.
        if (tid == 0) {
            uint32_t q = 0;
            for (int tile = tile_begin; tile < tile_end; ++tile, ++q) {
                const uint32_t s = q % STAGES;
                if (q >= (uint32_t)STAGES) mbar_wait(&empty_bar[s], ((q / STAGES) - 1) & 1);
                const uint32_t dst = smem_u32(sRing + (size_t)s * STAGE_BYTES);
                mbar_arrive_expect_tx(&full_bar[s], (uint32_t)STAGE_BYTES);
#pragma unroll
                for (int c = 0; c < CPR; ++c) tma_load_2d(dst + c * IMG, &tmA, c * 64, tile * BP, &full_bar[s]);
                if (q == 0) {
                    mbar_arrive_expect_tx(&w_bar, (uint32_t)(nchunks * A_CHUNK));
                    for (int j = 0; j < nchunks; ++j) tma_load_2d(smem_u32(sW + (size_t)j * A_CHUNK), &tmW, j * 64, 0, &w_bar);
                }
            }
        }
    } else if (warp >= 4) {
        // ======================= consumer warpgroup wg: tiles tile_begin + wg, + 2, ...; every tap is a B descriptor of the
        // staged window whose start address is shifted by whole 128-byte rows
        const int wg = (warp - 4) >> 2, wt = tid & 127;
        float* st = sAcc + wg * BP * LDS;
        const uint32_t w_base = smem_u32(sW);
        const uint32_t mW = (65536u + (uint32_t)p.Wp - 1u) / (uint32_t)p.Wp;
        constexpr int NW = 2;                                // 32-channel groups = mask words per position
        const int pw = wt;                                   // this thread's position in a pass
        float d[BP / 2];
#pragma unroll
        for (int e = 0; e < BP / 2; ++e) d[e] = 0.f;
        if (tile_begin + wg < tile_end) mbar_wait(&w_bar, 0);
        for (int tile = tile_begin + wg; tile < tile_end; tile += 2) {
            const uint32_t q = (uint32_t)(tile - tile_begin), s = q % STAGES;
            mbar_wait(&full_bar[s], (q / STAGES) & 1);
            wgmma_fence();
            const uint32_t win = smem_u32(sRing + (size_t)s * STAGE_BYTES);
#pragma unroll
            for (int t = 0; t < NTAPS; ++t) {
#pragma unroll
                for (int c = 0; c < CPR; ++c) {
                    const uint64_t b = desc_kmajor(win + (uint32_t)(c * IMG) + (uint32_t)p.shift[t] * 128u);
                    const uint64_t a = desc_kmajor(w_base + (uint32_t)((t * CPR + c) * A_CHUNK));
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)
                        WgmmaBf16<BP, 0, 0>::mma(d, a + 2 * kk, b + 2 * kk, (t | c | kk) != 0 ? 1u : 0u);
                }
            }
            wgmma_commit();
            // the position -> (image, Y, X) -> output offset arithmetic and the input mask words, while the MMAs run
            bool valid[RPT];
            int64_t o1[RPT], o2[RPT], ob[RPT];
            uint32_t mb[RPT][NW];
#pragma unroll
            for (int rr = 0; rr < RPT; ++rr) {
                const int64_t r = (int64_t)tile * BP + rr * PPR + pw;
                const int i = (int)(r / p.G);
                const int rem = (int)(r - (int64_t)i * p.G);
                const int Y = (int)(((uint32_t)rem * mW) >> 16), X = rem - Y * p.Wp;
                valid[rr] = r < p.M && (Y < p.vH) && (X < p.vW);
                o2[rr] = 0;
                if (p.out_mode == WOUT_DENSE) {
                    const int64_t orow = ((int64_t)i * p.vH + Y) * p.vW + X;
                    o1[rr] = orow * p.N; ob[rr] = orow * (p.N >> 5);
                } else {
                    o1[rr] = ((int64_t)i * 100 + Y * 10 + X) * 64;                 // 10-grid linear (conv2 wgrad)
                    o2[rr] = ((int64_t)i * 121 + (Y + 1) * 11 + (X + 1)) * 64;     // zero-padded 11x11 (conv2 dgrad)
                    ob[rr] = ((int64_t)i * 81 + Y * 9 + X) * 2;                    // act2 mask words
                }
                mb[rr][0] = mb[rr][1] = 0xFFFFFFFFu;
                if (p.mask_bits != nullptr && valid[rr]) {
                    const uint2 t = __ldg(reinterpret_cast<const uint2*>(p.mask_bits + ob[rr]));
                    mb[rr][0] = t.x; mb[rr][1] = t.y;
                }
            }
            wgmma_wait<0>();
            wgmma_fence_operands(d);
            if ((tid & 31) == 0) mbar_arrive(&empty_bar[s]);              // this warp's operand reads are complete
            named_bar(1 + wg, 128);                                     // the previous tile's rows have been read
            stage_acc_transposed(st, wt, d);
            named_bar(1 + wg, 128);
#pragma unroll
            for (int rr = 0; rr < RPT; ++rr) {
                float* srow = st + (rr * PPR + pw) * LDS;
#pragma unroll
                for (int g = 0; g < NW; ++g) {
                    if (!valid[rr] || g * 32 >= p.N) continue;
                    uint32_t v[32];
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const float4 f = *reinterpret_cast<const float4*>(srow + g * 32 + 4 * e);
                        v[4 * e] = __float_as_uint(f.x); v[4 * e + 1] = __float_as_uint(f.y);
                        v[4 * e + 2] = __float_as_uint(f.z); v[4 * e + 3] = __float_as_uint(f.w);
                    }
                    if (p.bias) {
                        const float4* bp = reinterpret_cast<const float4*>(p.bias + g * 32);
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
                        for (int e = 0; e < 32; ++e) bits |= (__uint_as_float(v[e]) > 0.f ? 1u : 0u) << e;   // from the fp32 value
                        if (p.mask_out) p.mask_out[ob[rr] + g] = bits;
                    }
                    if (p.mask_bits) {
#pragma unroll
                        for (int e = 0; e < 32; ++e) if (!((mb[rr][g] >> e) & 1u)) v[e] = 0u;
                    }
                    int4 w[4];
                    if (p.relu) {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            w[e].x = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e]), __uint_as_float(v[8 * e + 1]));
                            w[e].y = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e + 2]), __uint_as_float(v[8 * e + 3]));
                            w[e].z = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e + 4]), __uint_as_float(v[8 * e + 5]));
                            w[e].w = (int)pack_bf16x2_relu(__uint_as_float(v[8 * e + 6]), __uint_as_float(v[8 * e + 7]));
                        }
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            w[e].x = (int)pack_bf16x2(__uint_as_float(v[8 * e]), __uint_as_float(v[8 * e + 1]));
                            w[e].y = (int)pack_bf16x2(__uint_as_float(v[8 * e + 2]), __uint_as_float(v[8 * e + 3]));
                            w[e].z = (int)pack_bf16x2(__uint_as_float(v[8 * e + 4]), __uint_as_float(v[8 * e + 5]));
                            w[e].w = (int)pack_bf16x2(__uint_as_float(v[8 * e + 6]), __uint_as_float(v[8 * e + 7]));
                        }
                    }
                    // the packed 64 bytes go back into the row's own bytes [64 g, 64 g + 64), whose fp32 values this
                    // thread has already read (group g reads bytes [128 g, 128 g + 128))
                    int4* brow = reinterpret_cast<int4*>(srow) + 4 * g;
#pragma unroll
                    for (int e = 0; e < 4; ++e) brow[e] = w[e];
                }
                // the row's output offsets in its 16 padding bytes (-1: the position is not stored)
                *reinterpret_cast<longlong2*>(srow + 64) = make_longlong2(valid[rr] ? o1[rr] : -1, o2[rr]);
            }
            named_bar(1 + wg, 128);
            // coalesced stores: 8 lanes per position row, so a warp store writes 4 whole 128-byte rows (512 contiguous
            // bytes of a dense output) instead of 16 bytes in each of 32 rows
#pragma unroll
            for (int m = 0; m < BP / 16; ++m) {
                const int k = m * 128 + wt, part = k & 7;
                const float* srow = st + (k >> 3) * LDS;
                const longlong2 off = *reinterpret_cast<const longlong2*>(srow + 64);
                if (off.x < 0) continue;
                const int4 val = reinterpret_cast<const int4*>(srow)[part];
                *reinterpret_cast<int4*>(p.out + off.x + part * 8) = val;
                if (p.out_mode == WOUT_DACT2) *reinterpret_cast<int4*>(p.out2 + off.y + part * 8) = val;
            }
        }
    }
}

// linear-grid window convolutions with Cout = 64 on the MMA's M side, BP grid positions per tile
template <int BP, int CPR, int STAGES, int NTAPS>
static int launch_conv_win_t(WinParams p, cudaStream_t s, const char* what) {
    if (p.ntaps != NTAPS) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: %d taps, kernel instance has %d", what, p.ntaps, NTAPS);
    if (p.N != 64) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: N = %d, the kernel computes 64 output channels", what, p.N);
    if ((int64_t)p.G * p.Wp >= 65536 || p.G < 1)
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: grid %d x width %d outside the epilogue's multiply-shift range", what, p.G, p.Wp);
    if (p.rows || p.tpi_shift) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: the channel-major kernel walks a contiguous linear grid", what);
    if (p.out_mode != WOUT_DENSE && p.out_mode != WOUT_DACT2)
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: only bf16 dense and conv3 data-gradient outputs in this kernel", what);
    int maxs = 0;
    for (int t = 0; t < NTAPS; ++t) maxs = p.shift[t] > maxs ? p.shift[t] : maxs;
    p.WR = (BP + maxs + 7) & ~7;                        // the window: a tile's positions plus the largest tap shift
    if (p.WR > 256) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: window of %d rows exceeds a TMA box", what, p.WR);
    const size_t smem = (size_t)NTAPS * CPR * 64 * 128 + (size_t)STAGES * p.WR * 128 * CPR + conv_win_t_stage_bytes<BP>() + 1024;
    static SmemAttrCache attr;
    if (int rc = attr.ensure(tc_conv_win_t<BP, CPR, STAGES, NTAPS>, smem, what)) return rc;
    const int total = (int)ceil_div(p.M, BP);
    int grid = num_sms();
    if (grid > total) grid = total;
    CUtensorMap tmA, tmW;
    memset(&tmA, 0, sizeof(tmA));
    memset(&tmW, 0, sizeof(tmW));
    if (int rc = make_tmap_2d(&tmA, p.A, p.M, (int64_t)CPR * 64, p.WR, what)) return rc;
    if (int rc = make_tmap_2d(&tmW, p.Bw, 64, (int64_t)NTAPS * CPR * 64, 64, what)) return rc;     // packed [64][K] weights
    tc_conv_win_t<BP, CPR, STAGES, NTAPS><<<grid, kConvWinTThreads, smem, s>>>(tmA, tmW, p, total);
    return check_launch(what);
}

}  // namespace b200rl
