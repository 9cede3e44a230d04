// conv2 -> conv3 forward of the NatureCNN trunk in one persistent kernel (see net_tc.cu for the layer plan).
#pragma once
#include "tc_conv_win.cuh"

namespace b200rl {
using namespace tc;

// ------------------------------------------------------------------ kernel 1e: conv2 + conv3 forward, one image per tile
// act1 (2x2 cells [n,100,128]) -> act2 [n,81,64] + m2, act3 [n,49,64] + m3.  A tile is one image.  conv2 is the window
// convolution of tc_conv_win_t over the image's 10x10 cell grid (channels on M, positions on N: m64n96k16 over cell
// positions 0..95, which hold every valid output Y, X < 9); its epilogue writes the act2 rows into an act2 image in
// shared memory, the SWIZZLE_128B K-major operand conv3 reads, and from there to HBM.  conv3 is the window convolution
// over that image's 9x9 grid (m64n64k16 over positions 0..63, which hold every output y*9 + x with y, x < 7), so act2 is
// never read back from HBM and no MMA runs on positions that cross into the next image.
// The two consumer warpgroups take alternate images, each with its own window stage and act2 image, so one
// warpgroup's epilogues run under the other's MMAs.  Warp 0 is the TMA producer (one 3-D box per 64-channel column
// chunk: image, 112 rows, 64 channels; rows >= 100 zero-filled).  The resident weights arrive on two barriers: W2 right
// behind the first window, W3 behind the second, so W3 lands while the first conv2 MMAs run.
// Every output is the same bf16 products summed over the same K sequence as tc_conv_win_t (conv2: taps in shift order,
// column chunks, k16 steps; conv3: taps ky*3 + kx, k16 steps; the first MMA with scale-d = 0) and the epilogues apply the
// same fp32 operations (bias, mask bit from the fp32 value, ReLU folded into the bf16 conversion): act2, act3, m2 and m3
// are bit-identical to the two window-convolution launches this kernel replaces.
//
// Shared memory (227 KB per CTA):
//   W2 + W3 resident                    8 x 8 KB + 9 x 8 KB              136 KB
//   act1 window stages (one per wg)     2 chunks x 112 rows x 128 B       2 x 28 KB
//     after its conv2 MMAs a stage holds the fp32 transpose of the accumulators (96 x 68 floats = 25.5 KB)
//   act2 image (one per wg)             88 rows x 128 B (rows 81..87 zero)  2 x 16 KB
//     after its conv3 MMAs the same 16 KB hold the fp32 transpose of conv3's accumulators (64 x 64 floats, XOR-swizzled
//     in float4 units instead of padded: 64 x 68 floats would not fit)
//   alignment slack                                                       1 KB        = 225 KB + 48 B of barriers
struct Conv23Params {
    int n;
    const float* b2;
    const float* b3;
    bf16* act2;
    bf16* act3;
    uint32_t* m2;
    uint32_t* m3;
};

constexpr int kConv23Threads = 384;
constexpr int kC23WinRows = 112;                         // 96 positions + 11 rows of tap shift, rounded up to 8
constexpr int kC23Chunk = 64 * 128;                      // one 64-channel K chunk of the 64 weight rows
constexpr int kC23StageBytes = 2 * kC23WinRows * 128;
constexpr int kC23ImgBytes = 64 * 64 * 4;
constexpr size_t kC23Smem = (size_t)(8 + 9) * kC23Chunk + 2 * kC23StageBytes + 2 * kC23ImgBytes + 1024;
static_assert(96 * kConvWinTLds * 4 <= kC23StageBytes, "conv2's fp32 staging fits its window stage");
static_assert(88 * 128 <= kC23ImgBytes, "the act2 image and its zero tail fit the conv3 staging");

// the window-convolution epilogue of one 32-channel group, with the fp32 operations of tc_conv_win_t (scale 1, bias,
// ReLU): the mask word from the fp32 values and the packed bf16 values.  Float4 k of the group is read at index k ^ sw.
__device__ __forceinline__ uint32_t conv23_group(const float* srow, int g, int sw, const float* bias, int4 (&w)[4]) {
    float v[32];
    const float4* bp = reinterpret_cast<const float4*>(bias + g * 32);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const float4 f = reinterpret_cast<const float4*>(srow)[(8 * g + e) ^ sw];
        const float4 bv = __ldg(bp + e);
        v[4 * e] = fmaf(f.x, 1.f, bv.x); v[4 * e + 1] = fmaf(f.y, 1.f, bv.y);
        v[4 * e + 2] = fmaf(f.z, 1.f, bv.z); v[4 * e + 3] = fmaf(f.w, 1.f, bv.w);
    }
    uint32_t bits = 0u;
#pragma unroll
    for (int e = 0; e < 32; ++e) bits |= (v[e] > 0.f ? 1u : 0u) << e;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        w[e].x = (int)pack_bf16x2_relu(v[8 * e], v[8 * e + 1]);
        w[e].y = (int)pack_bf16x2_relu(v[8 * e + 2], v[8 * e + 3]);
        w[e].z = (int)pack_bf16x2_relu(v[8 * e + 4], v[8 * e + 5]);
        w[e].w = (int)pack_bf16x2_relu(v[8 * e + 6], v[8 * e + 7]);
    }
    return bits;
}

// a warpgroup's 64 x 64 accumulator fragment -> st[position][channel], 64 floats per row, float4 k of row r at k ^ (r & 7)
__device__ __forceinline__ void stage_acc_transposed_sw(float* st, int wg_tid, const float (&d)[32]) {
    const int co = ((wg_tid >> 5) << 4) + ((wg_tid & 31) >> 2), pos = (wg_tid & 3) * 2;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int r0 = 8 * j + pos, r1 = r0 + 1;
        st[r0 * 64 + (co ^ ((r0 & 7) << 2))] = d[4 * j];
        st[r1 * 64 + (co ^ ((r1 & 7) << 2))] = d[4 * j + 1];
        st[r0 * 64 + ((co + 8) ^ ((r0 & 7) << 2))] = d[4 * j + 2];
        st[r1 * 64 + ((co + 8) ^ ((r1 & 7) << 2))] = d[4 * j + 3];
    }
}

__global__ void __launch_bounds__(kConv23Threads, 1) tc_conv23_fwd(const __grid_constant__ CUtensorMap tmA,
                                                                   const __grid_constant__ CUtensorMap tmW2,
                                                                   const __grid_constant__ CUtensorMap tmW3, const Conv23Params p) {
    constexpr int IMG = kC23WinRows * 128;               // one 64-channel column chunk of the window
    constexpr int LDS = kConvWinTLds;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[2], empty_bar[2], w2_bar, w3_bar;
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5;
    uint8_t* sW2 = smem;
    uint8_t* sW3 = sW2 + 8 * kC23Chunk;
    uint8_t* sRing = sW3 + 9 * kC23Chunk;
    uint8_t* sImg = sRing + 2 * kC23StageBytes;

    if (tid == 0) {
        for (int s = 0; s < 2; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // the consuming warpgroup's 4 warps
        mbar_init(&w2_bar, 1);
        mbar_init(&w3_bar, 1);
        fence_barrier_init();
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmW2);
        tma_prefetch_desc(&tmW3);
    }
    __syncthreads();
    // each CTA walks a contiguous range of images
    const int img_begin = (int)(((int64_t)p.n * blockIdx.x) / gridDim.x);
    const int img_end = (int)(((int64_t)p.n * (blockIdx.x + 1)) / gridDim.x);

    if (warp == 0) {
        // ======================= TMA producer: image q goes to stage q % 2 (= the warpgroup that owns it)
        if (tid == 0) {
            bool w3_sent = false;
            uint32_t q = 0;
            for (int img = img_begin; img < img_end; ++img, ++q) {
                const uint32_t s = q & 1;
                if (q >= 2) mbar_wait(&empty_bar[s], ((q >> 1) - 1) & 1);
                const uint32_t dst = smem_u32(sRing + (size_t)s * kC23StageBytes);
                mbar_arrive_expect_tx(&full_bar[s], (uint32_t)kC23StageBytes);
                tma_load_3d(dst, &tmA, 0, 0, img, &full_bar[s]);
                tma_load_3d(dst + IMG, &tmA, 64, 0, img, &full_bar[s]);
                if (q == 0) {
                    mbar_arrive_expect_tx(&w2_bar, (uint32_t)(8 * kC23Chunk));
                    for (int j = 0; j < 8; ++j) tma_load_2d(smem_u32(sW2 + (size_t)j * kC23Chunk), &tmW2, j * 64, 0, &w2_bar);
                }
                if (!w3_sent && (q == 1 || img + 1 == img_end)) {
                    mbar_arrive_expect_tx(&w3_bar, (uint32_t)(9 * kC23Chunk));
                    for (int j = 0; j < 9; ++j) tma_load_2d(smem_u32(sW3 + (size_t)j * kC23Chunk), &tmW3, j * 64, 0, &w3_bar);
                    w3_sent = true;
                }
            }
        }
    } else if (warp >= 4) {
        // ======================= consumer warpgroup wg: images img_begin + wg, + 2, ...
        const int wg = (warp - 4) >> 2, wt = tid & 127;
        uint8_t* img2 = sImg + (size_t)wg * kC23ImgBytes;    // act2 image, then conv3's fp32 staging
        float* st3 = reinterpret_cast<float*>(img2);
        const uint32_t w2_base = smem_u32(sW2), w3_base = smem_u32(sW3), img2_base = smem_u32(img2);
        const int shift2[4] = {0, 1, 10, 11};
        float d2[48], d3[32];
#pragma unroll
        for (int e = 0; e < 48; ++e) d2[e] = 0.f;
#pragma unroll
        for (int e = 0; e < 32; ++e) d3[e] = 0.f;
        if (img_begin + wg < img_end) mbar_wait(&w2_bar, 0);
        for (int img = img_begin + wg; img < img_end; img += 2) {
            const uint32_t q = (uint32_t)(img - img_begin), s = q & 1;
            const int64_t i = img;
            // ---- conv2: 4 taps x 2 column chunks x 4 k16 steps over cell positions 0..95
            mbar_wait(&full_bar[s], (q >> 1) & 1);
            wgmma_fence();
            uint8_t* stage = sRing + (size_t)s * kC23StageBytes;
            const uint32_t win = smem_u32(stage);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const uint64_t b = desc_kmajor(win + (uint32_t)(c * IMG) + (uint32_t)shift2[t] * 128u);
                    const uint64_t a = desc_kmajor(w2_base + (uint32_t)((t * 2 + c) * kC23Chunk));
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) WgmmaBf16<96, 0, 0>::mma(d2, a + 2 * kk, b + 2 * kk, (t | c | kk) != 0 ? 1u : 0u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_operands(d2);
            // ---- conv2 epilogue: the accumulators are transposed into the window stage (its operand reads are complete);
            //      192 (position, 32-channel group) items, position = item % 96 so that a quarter warp reads 8 rows
            float* st2 = reinterpret_cast<float*>(stage);
            stage_acc_transposed(st2, wt, d2);
            named_bar(1 + wg, 128);
#pragma unroll
            for (int pass = 0; pass < 2; ++pass) {
                const int k = pass * 128 + wt;
                if (k >= 192) continue;
                const int pos = k % 96, g = k / 96;
                const int Y = pos / 10, X = pos - 10 * Y;
                if (Y >= 9 || X >= 9) continue;
                const int r = Y * 9 + X;
                int4 w[4];
                p.m2[(i * 81 + r) * 2 + g] = conv23_group(st2 + pos * LDS, g, 0, p.b2, w);
#pragma unroll
                for (int e = 0; e < 4; ++e) *reinterpret_cast<int4*>(img2 + img_off(r, 4 * g + e)) = w[e];
            }
            // rows 81..87: reached only by the tap shifts of positions that are not conv3 outputs (the staging of the
            // previous image's conv3 overwrote them)
            if (wt < 56) *reinterpret_cast<int4*>(img2 + 81 * 128 + wt * 16) = make_int4(0, 0, 0, 0);
            // the image (and the staging writes) -> the async proxy: conv3's wgmma reads the image, TMA refills the stage
            fence_proxy_async_smem();
            named_bar(1 + wg, 128);
            if ((tid & 31) == 0) mbar_arrive(&empty_bar[s]);
            // ---- conv3: 9 taps x 4 k16 steps over positions 0..63 of the act2 image
            if (q < 2) mbar_wait(&w3_bar, 0);
            wgmma_fence();
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const uint64_t b = desc_kmajor(img2_base + (uint32_t)((t / 3) * 9 + t % 3) * 128u);
                const uint64_t a = desc_kmajor(w3_base + (uint32_t)(t * kC23Chunk));
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) WgmmaBf16<64, 0, 0>::mma(d3, a + 2 * kk, b + 2 * kk, (t | kk) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            // act2 -> HBM from the image while the MMAs run: 81 rows = 648 whole 16-byte pieces, contiguous per image
            int4* a2 = reinterpret_cast<int4*>(p.act2 + i * 5184);
#pragma unroll
            for (int m = 0; m < 6; ++m) {
                const int k = m * 128 + wt;
                if (k < 648) a2[k] = *reinterpret_cast<const int4*>(img2 + img_off(k >> 3, k & 7));
            }
            wgmma_wait<0>();
            wgmma_fence_operands(d3);
            named_bar(1 + wg, 128);                                  // every read of the image is complete
            stage_acc_transposed_sw(st3, wt, d3);
            named_bar(1 + wg, 128);
            // ---- conv3 epilogue: thread = (position, 32-channel group); act3 rows are 64 contiguous bytes per group
            {
                const int pw = wt & 63, g = wt >> 6;
                const int y = pw / 9, x = pw - 9 * y;
                if (y < 7 && x < 7) {
                    const int64_t orow = i * 49 + y * 7 + x;
                    int4 w[4];
                    p.m3[orow * 2 + g] = conv23_group(st3 + pw * 64, g, pw & 7, p.b3, w);
                    bf16* dst = p.act3 + orow * 64 + g * 32;
                    st_global_32b(dst, w[0], w[1]);
                    st_global_32b(dst + 16, w[2], w[3]);
                }
            }
        }
    }
}

// act1 [n,100,128] -> act2 [n,81,64] + m2, act3 [n,49,64] + m3 with the packed conv2 / conv3 weights ([64][512], [64][576])
static int launch_conv23_fwd(const bf16* act1, const bf16* w2, const bf16* w3, const Conv23Params& p, cudaStream_t s,
                             const char* what) {
    if (p.n < 1) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: n = %d", what, p.n);
    static SmemAttrCache attr;
    if (int rc = attr.ensure(tc_conv23_fwd, kC23Smem, what)) return rc;
    int grid = num_sms();
    if (grid > p.n) grid = p.n;
    CUtensorMap tmA, tmW2, tmW3;
    memset(&tmA, 0, sizeof(tmA));
    memset(&tmW2, 0, sizeof(tmW2));
    memset(&tmW3, 0, sizeof(tmW3));
    int rc;
    if ((rc = make_tmap_3d(&tmA, act1, p.n, 100, 128, kC23WinRows, what))) return rc;
    if ((rc = make_tmap_2d(&tmW2, w2, 64, 512, 64, what))) return rc;
    if ((rc = make_tmap_2d(&tmW3, w3, 64, 576, 64, what))) return rc;
    tc_conv23_fwd<<<grid, kConv23Threads, kC23Smem, s>>>(tmA, tmW2, tmW3, p);
    return check_launch(what);
}

}  // namespace b200rl
