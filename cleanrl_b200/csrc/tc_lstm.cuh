// Recurrent agent (cleanrl/ppo_atari_lstm.py:117-160) on the tensor cores: the two kernels its NatureCNN trunk and
// LSTM need beyond the 4-frame NatureCNN ones.  Both use ldmatrix + mma.sync m16n8k16 (bf16 in, fp32 accumulate).
//
//   conv1 on single frames  uint8 [*, 1, 84, 84] read through the minibatch gather `rows`.  A CTA stages one frame as a
//       bf16 space-to-depth(4) grid in shared memory: 21 x 21 positions x 16 channels (channel sy*4 + sx of pixel
//       (4Y+sy, 4X+sx)), 32-byte rows plus 16 bytes of padding, zero past position 441.  conv1 (8x8, stride 4) is then a
//       2x2 stride-1 convolution: tap (a, b) is the row shift 21a + b and one k16 step.  0..255 is exact in bf16; the /255
//       is applied to the fp32 accumulator.  The forward writes act1 in the 2x2-cell layout [n, 10, 10, 128] and the
//       ReLU bits of the 4-frame path, so conv2 onwards run unchanged.  The weight gradient reads the same staged frames
//       and d(act1) on the 21x21 grid; per-CTA partials over a fixed image range are folded in order (bitwise
//       repeatable).
//   recurrence              one launch runs all S steps of a sequence: a CTA owns 16 env rows (env rows are independent
//       and the state is reset per row by (1 - done)), W_hh bf16 [512][128] stays resident in shared memory, and the
//       backward reads it transposed (ldmatrix .trans) from the same image.  Warp w owns hidden units [16w, 16w + 16) of
//       all four gates, so each thread holds the i, f, g, o pre-activations of its (row, unit) pairs in registers and the
//       cell runs there in fp32; c never leaves fp32.  Rounding points: the masked state h' and dgates are rounded to
//       bf16 as MMA operands, h_t is stored in bf16 for the heads.
#pragma once
#include "tc_base.cuh"
#include "tc_mma_sync.cuh"

namespace b200rl {
namespace lstm {
using namespace tc;

constexpr int kH = 128, kG = 4 * kH;        // hidden units, gate pre-activations (i, f, g, o as torch.nn.LSTM)
constexpr int kThreads = 256;
constexpr int kRows = 16;                   // env rows per CTA of the recurrence (one m16 tile)
constexpr int kWPitch = kH * 2 + 16;        // W_hh row / h' row in shared memory (bytes): 8 ldmatrix rows on distinct banks
constexpr int kGPitch = kG * 2 + 16;        // dgates row in shared memory
constexpr int kMaxA1 = 24;                  // head outputs (A + 1) the recurrence backward folds in

__host__ __device__ constexpr size_t rec_fwd_smem() { return (size_t)kG * kWPitch + 2 * kRows * kWPitch; }
__host__ __device__ constexpr size_t rec_bwd_smem() { return (size_t)kG * kWPitch + 2 * kRows * kGPitch + kMaxA1 * kH * 4; }

// ---------------------------------------------------------------- conv1 on single frames
constexpr int kFramePos = 441;              // 21 x 21 space-to-depth positions
constexpr int kFrameRows = 448;             // GEMM rows: 28 m16 tiles
constexpr int kFrameStage = kFrameRows + 22;    // + the largest tap shift
constexpr int kXPitch = 48, kC1WPitch = 64 * 2 + 16, kDyPitch = 32 * 2 + 16;
constexpr size_t conv1_fwd_smem() { return (size_t)32 * kC1WPitch + (size_t)kFrameStage * kXPitch; }
constexpr size_t conv1_wgrad_smem() { return (size_t)kFrameStage * kXPitch + (size_t)kFrameRows * kDyPitch; }

__device__ __forceinline__ int tap_shift(int t) { return (t >> 1) * 21 + (t & 1); }

__device__ __forceinline__ void stage_frame(uint8_t* sX, const uint8_t* frames, int64_t img) {
    const uint8_t* f = frames + img * 7056;
    for (int q = threadIdx.x; q < kFrameStage; q += blockDim.x) {
        uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (q < kFramePos) {
            const int Y = q / 21, X = q - Y * 21;
            const uint8_t* src = f + (4 * Y) * 84 + 4 * X;
#pragma unroll
            for (int sy = 0; sy < 4; ++sy) {
                const uint32_t w = __ldg(reinterpret_cast<const unsigned int*>(src + sy * 84));
                v[2 * sy] = pack_bf16x2((float)(w & 255u), (float)((w >> 8) & 255u));
                v[2 * sy + 1] = pack_bf16x2((float)((w >> 16) & 255u), (float)(w >> 24));
            }
        }
        int4* d = reinterpret_cast<int4*>(sX + (size_t)q * kXPitch);
        d[0] = make_int4((int)v[0], (int)v[1], (int)v[2], (int)v[3]);
        d[1] = make_int4((int)v[4], (int)v[5], (int)v[6], (int)v[7]);
    }
}

struct Conv1P {
    const uint8_t* obs;        // [*, 1, 84, 84]
    const int64_t* rows;       // frame of batch row i (null = i)
    int64_t n;
    const bf16* w;             // packed [32][tap*16 + sy*4 + sx]
    const float* bias;
    bf16* out;                 // act1 [n, 10, 10, 128] (2x2 cells)
    uint32_t* mask_out;        // [n, 100 cells, 4 classes] words, bit co = act1 > 0
};

__global__ void __launch_bounds__(kThreads) lstm_conv1_fwd(const Conv1P p) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* sW = smem;
    uint8_t* sX = smem + 32 * kC1WPitch;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gq = lane >> 2, tq = lane & 3;
    for (int idx = tid; idx < 32 * 8; idx += blockDim.x)
        *reinterpret_cast<int4*>(sW + (idx >> 3) * kC1WPitch + (idx & 7) * 16) = ldg16(p.w + idx * 8);
    const uint32_t sWa = smem_u32(sW), sXa = smem_u32(sX);
    const uint32_t brow = sWa + (uint32_t)(((lane & 7) + ((lane >> 4) << 3)) * kC1WPitch + ((lane >> 3) & 1) * 16);
    for (int64_t img = blockIdx.x; img < p.n; img += gridDim.x) {
        __syncthreads();                                       // the previous frame's reads of sX are done
        stage_frame(sX, p.obs, p.rows ? __ldg(p.rows + img) : img);
        __syncthreads();
        for (int m = warp; m < kFrameRows / 16; m += kThreads / 32) {
            float acc[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
            const uint32_t arow = sXa + (uint32_t)((m * 16 + (lane & 15)) * kXPitch + (lane >> 4) * 16);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                uint32_t a0, a1, a2, a3;
                ldsm_x4(arow + tap_shift(t) * kXPitch, a0, a1, a2, a3);
#pragma unroll
                for (int np = 0; np < 2; ++np) {
                    uint32_t b0, b1, b2, b3;
                    ldsm_x4(brow + t * 32 + np * 16 * kC1WPitch, b0, b1, b2, b3);
                    mma16816(acc[2 * np], a0, a1, a2, a3, b0, b1);
                    mma16816(acc[2 * np + 1], a0, a1, a2, a3, b2, b3);
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int q = m * 16 + gq + 8 * h, Y = q / 21, X = q - Y * 21;
                const bool valid = q < kFramePos && Y < 20 && X < 20;
                const int64_t cell = (img * 10 + (Y >> 1)) * 10 + (X >> 1);
                const int cls = (Y & 1) * 2 + (X & 1);
                uint32_t bits = 0;
                if (valid) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int co = 8 * j + 2 * tq;
                        const float v0 = fmaf(acc[j][2 * h], 1.0f / 255.0f, __ldg(p.bias + co));
                        const float v1 = fmaf(acc[j][2 * h + 1], 1.0f / 255.0f, __ldg(p.bias + co + 1));
                        bits |= (v0 > 0.f ? 1u : 0u) << co;
                        bits |= (v1 > 0.f ? 1u : 0u) << (co + 1);
                        *reinterpret_cast<unsigned int*>(p.out + cell * 128 + cls * 32 + co) = pack_bf16x2_relu(v0, v1);
                    }
                }
                bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
                bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
                if (valid && tq == 0) p.mask_out[cell * 4 + cls] = bits;
            }
        }
    }
}

struct Conv1WgradP {
    const uint8_t* obs;
    const int64_t* rows;
    int64_t n;
    const bf16* dy;            // d(act1) on the 21x21 grid [n, 441, 32] (zero at row / column 20)
    int64_t imgs_per_cta;
    float* ws;                 // [gridDim.x][32][64]
    float* wsb;                // [gridDim.x][32]
};

// dW^T[co][tap*16 + ch] = sum over the CTA's frames and grid positions q of dY[q][co] * X[q + shift_tap][ch]
__global__ void __launch_bounds__(kThreads) lstm_conv1_wgrad(const Conv1WgradP p) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float red[kThreads];
    uint8_t* sX = smem;
    uint8_t* sY = smem + (size_t)kFrameStage * kXPitch;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gq = lane >> 2, tq = lane & 3;
    const uint32_t sXa = smem_u32(sX), sYa = smem_u32(sY);
    float acc[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const int bco = tid & 31, brl = tid >> 5;                  // bias column sums: 8 row lanes x 32 channels
    float bacc = 0.f;
    const int64_t i0 = (int64_t)blockIdx.x * p.imgs_per_cta;
    const int64_t i1 = i0 + p.imgs_per_cta < p.n ? i0 + p.imgs_per_cta : p.n;
    for (int64_t img = i0; img < i1; ++img) {
        __syncthreads();
        stage_frame(sX, p.obs, p.rows ? __ldg(p.rows + img) : img);
        for (int idx = tid; idx < kFrameRows * 4; idx += blockDim.x) {
            const int q = idx >> 2, ch = idx & 3;
            const int4 v = q < kFramePos ? ldg16(p.dy + (img * kFramePos + q) * 32 + ch * 8) : make_int4(0, 0, 0, 0);
            *reinterpret_cast<int4*>(sY + (size_t)q * kDyPitch + ch * 16) = v;
        }
        __syncthreads();
        for (int q = brl; q < kFramePos; q += kThreads / 32)
            bacc += __bfloat162float(*reinterpret_cast<const bf16*>(sY + (size_t)q * kDyPitch + bco * 2));
        for (int kt = 0; kt < kFrameRows / 16; ++kt) {
#pragma unroll
            for (int ii = 0; ii < 2; ++ii) {
                const int it = warp + 8 * ii, mtile = it >> 3, nt = it & 7;
                uint32_t a0, a1, a2, a3, b0, b1;
                // A = dY^T (m = co, k = position): stored [position][co] -> transposed ldmatrix
                ldsm_x4_t(sYa + (uint32_t)((kt * 16 + (lane & 7) + (lane >> 4) * 8) * kDyPitch + (mtile * 16 + ((lane >> 3) & 1) * 8) * 2),
                          a0, a1, a2, a3);
                // B = X shifted by the tap (k = position, n = channel)
                ldsm_x2_t(sXa + (uint32_t)((kt * 16 + tap_shift(nt >> 1) + (lane & 7) + ((lane >> 3) & 1) * 8) * kXPitch + (nt & 1) * 16),
                          b0, b1);
                mma16816(acc[ii], a0, a1, a2, a3, b0, b1);
            }
        }
    }
    float* wsc = p.ws + (size_t)blockIdx.x * 32 * 64;
#pragma unroll
    for (int ii = 0; ii < 2; ++ii) {
        const int it = warp + 8 * ii, mtile = it >> 3, nt = it & 7;
        const int col = nt * 8 + 2 * tq, co = mtile * 16 + gq;
        *reinterpret_cast<float2*>(wsc + co * 64 + col) = make_float2(acc[ii][0], acc[ii][1]);
        *reinterpret_cast<float2*>(wsc + (co + 8) * 64 + col) = make_float2(acc[ii][2], acc[ii][3]);
    }
    red[tid] = bacc;
    __syncthreads();
    if (tid < 32) {
        float s = 0.f;
        for (int l = 0; l < kThreads / 32; ++l) s += red[l * 32 + tid];
        p.wsb[(size_t)blockIdx.x * 32 + tid] = s;
    }
}

// fixed-order fold of the partials into torch's w[co][0][ky][kx] (x 1/255) and the bias
__global__ void __launch_bounds__(256) lstm_conv1_fold(const float* __restrict__ ws, const float* __restrict__ wsb, int S,
                                                       float* __restrict__ dw, float* __restrict__ db) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < 32 * 64) {
        const int co = idx >> 6, k = idx & 63, tap = k >> 4, sy = (k >> 2) & 3, sx = k & 3;
        float s = 0.f;
        for (int z = 0; z < S; ++z) s += ws[((size_t)z * 32 + co) * 64 + k];
        dw[co * 64 + ((tap >> 1) * 4 + sy) * 8 + (tap & 1) * 4 + sx] = s * (1.0f / 255.0f);
    } else if (idx < 32 * 64 + 32) {
        const int co = idx - 32 * 64;
        float s = 0.f;
        for (int z = 0; z < S; ++z) s += wsb[(size_t)z * 32 + co];
        db[co] = s;
    }
}

// conv1 w[co][0][ky][kx] -> [co][(a*2 + b)*16 + sy*4 + sx], ky = 4a + sy, kx = 4b + sx
__global__ void lstm_pack_conv1(const float* __restrict__ w, bf16* __restrict__ fwd) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 32 * 64) return;
    const int kx = idx & 7, ky = (idx >> 3) & 7, co = idx >> 6;
    fwd[co * 64 + ((ky >> 2) * 2 + (kx >> 2)) * 16 + (ky & 3) * 4 + (kx & 3)] = __float2bfloat16(w[idx]);
}

// ---------------------------------------------------------------- recurrence
__device__ __forceinline__ float sigm(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ void load_whh(uint8_t* sW, const bf16* whh) {
    for (int idx = threadIdx.x; idx < kG * (kH / 8); idx += blockDim.x) {
        const int r = idx / (kH / 8), c = idx - r * (kH / 8);
        *reinterpret_cast<int4*>(sW + (size_t)r * kWPitch + c * 16) = ldg16(whh + (size_t)r * kH + c * 8);
    }
}

struct RecFwdP {
    int S;
    int64_t n;                 // env rows; row (t, e) of the sequence tensors is t*n + e
    const bf16* whh;           // bf16 [512][128] (torch layout)
    const float* bhh;          // [512]
    const float* gx;           // [S*n, 512] = feats W_ih^T + b_ih
    const float* done;         // [S*n]
    const float* h0;           // [n, 128]
    const float* c0;
    bf16* hseq;                // [S*n, 128] h_t (heads input)
    bf16* hm;                  // [S*n, 128] masked state h' of step t (dW_hh operand)
    float* save;               // [S*n, 5, 128] i, f, g, o, tanh(c)
    float* cm;                 // [S*n, 128] masked cell state c'
    float* h_out;              // [n, 128] h_S, c_S
    float* c_out;
};

// Thread (warp w, lane gq*4 + tq) owns rows gq, gq + 8 of the CTA's tile and units u = 16w + 8hf + 2tq + e (hf, e in {0,1}):
// exactly the accumulator positions of n8 tile (gate*2 + hf) of the m16n8 MMAs.
__global__ void __launch_bounds__(kThreads, 1) lstm_rec_fwd(const RecFwdP p) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* sW = smem;
    uint8_t* sH = smem + (size_t)kG * kWPitch;                 // two h' buffers [16][128] (step parity)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gq = lane >> 2, tq = lane & 3;
    load_whh(sW, p.whh);
    const int64_t n = p.n;
    int64_t row[2];
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) { row[h] = (int64_t)blockIdx.x * kRows + gq + 8 * h; valid[h] = row[h] < n; }
    float hr[2][2][2], cr[2][2][2], bh[4][2][2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        const int u = 16 * warp + 8 * hf + 2 * tq;
#pragma unroll
        for (int g = 0; g < 4; ++g) { bh[g][hf][0] = __ldg(p.bhh + g * kH + u); bh[g][hf][1] = __ldg(p.bhh + g * kH + u + 1); }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float2 hv = make_float2(0.f, 0.f), cv = make_float2(0.f, 0.f);
            if (valid[h]) {
                hv = *reinterpret_cast<const float2*>(p.h0 + row[h] * kH + u);
                cv = *reinterpret_cast<const float2*>(p.c0 + row[h] * kH + u);
            }
            hr[h][hf][0] = hv.x; hr[h][hf][1] = hv.y; cr[h][hf][0] = cv.x; cr[h][hf][1] = cv.y;
        }
    }
    const uint32_t sWa = smem_u32(sW), sHa = smem_u32(sH);
    const uint32_t brow = sWa + (uint32_t)(((lane & 7) + ((lane >> 4) << 3) + 16 * warp) * kWPitch + ((lane >> 3) & 1) * 16);
    for (int t = 0; t < p.S; ++t) {
        uint8_t* buf = sH + (size_t)(t & 1) * kRows * kWPitch;
        float gxv[2][4][2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t r = (int64_t)t * n + row[h];
            const float keep = valid[h] ? 1.0f - __ldg(p.done + r) : 0.f;
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int u = 16 * warp + 8 * hf + 2 * tq;
                const float m0 = keep * hr[h][hf][0], m1 = keep * hr[h][hf][1];
                cr[h][hf][0] *= keep; cr[h][hf][1] *= keep;
                const uint32_t hb = pack_bf16x2(m0, m1);
                *reinterpret_cast<uint32_t*>(buf + (gq + 8 * h) * kWPitch + u * 2) = hb;
                if (valid[h]) {
                    *reinterpret_cast<uint32_t*>(p.hm + r * kH + u) = hb;
                    *reinterpret_cast<float2*>(p.cm + r * kH + u) = make_float2(cr[h][hf][0], cr[h][hf][1]);
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const float2 v = __ldg(reinterpret_cast<const float2*>(p.gx + r * kG + g * kH + u));
                        gxv[h][g][hf][0] = v.x; gxv[h][g][hf][1] = v.y;
                    }
                } else {
#pragma unroll
                    for (int g = 0; g < 4; ++g) gxv[h][g][hf][0] = gxv[h][g][hf][1] = 0.f;
                }
            }
        }
        __syncthreads();                                        // h' of this step is staged (the other buffer is free)
        float acc[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        const uint32_t arow = sHa + (uint32_t)((t & 1) * kRows * kWPitch + (lane & 15) * kWPitch + (lane >> 4) * 16);
#pragma unroll
        for (int kc = 0; kc < kH / 16; ++kc) {
            uint32_t a0, a1, a2, a3;
            ldsm_x4(arow + kc * 32, a0, a1, a2, a3);
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                uint32_t b0, b1, b2, b3;
                ldsm_x4(brow + g * kH * kWPitch + kc * 32, b0, b1, b2, b3);
                mma16816(acc[2 * g], a0, a1, a2, a3, b0, b1);
                mma16816(acc[2 * g + 1], a0, a1, a2, a3, b2, b3);
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t r = (int64_t)t * n + row[h];
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int u = 16 * warp + 8 * hf + 2 * tq;
                float sv[5][2], hn[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pi = acc[hf][2 * h + e] + bh[0][hf][e] + gxv[h][0][hf][e];
                    const float pf = acc[2 + hf][2 * h + e] + bh[1][hf][e] + gxv[h][1][hf][e];
                    const float pg = acc[4 + hf][2 * h + e] + bh[2][hf][e] + gxv[h][2][hf][e];
                    const float po = acc[6 + hf][2 * h + e] + bh[3][hf][e] + gxv[h][3][hf][e];
                    const float i = sigm(pi), f = sigm(pf), g = tanhf(pg), o = sigm(po);
                    const float c = f * cr[h][hf][e] + i * g;
                    const float tc = tanhf(c);
                    cr[h][hf][e] = c;
                    hn[e] = o * tc;
                    hr[h][hf][e] = hn[e];
                    sv[0][e] = i; sv[1][e] = f; sv[2][e] = g; sv[3][e] = o; sv[4][e] = tc;
                }
                if (valid[h]) {
#pragma unroll
                    for (int k = 0; k < 5; ++k)
                        *reinterpret_cast<float2*>(p.save + (r * 5 + k) * kH + u) = make_float2(sv[k][0], sv[k][1]);
                    *reinterpret_cast<uint32_t*>(p.hseq + r * kH + u) = pack_bf16x2(hn[0], hn[1]);
                }
            }
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (!valid[h]) continue;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int u = 16 * warp + 8 * hf + 2 * tq;
            *reinterpret_cast<float2*>(p.h_out + row[h] * kH + u) = make_float2(hr[h][hf][0], hr[h][hf][1]);
            *reinterpret_cast<float2*>(p.c_out + row[h] * kH + u) = make_float2(cr[h][hf][0], cr[h][hf][1]);
        }
    }
}

struct RecBwdP {
    int S;
    int64_t n;
    int A1;                    // head outputs (A + 1 <= kMaxA1)
    const bf16* whh;
    const float* wh;           // head weights fp32 [A1][128] (actor rows, then the critic row)
    const float* dhead;        // [S*n, A1]
    const float* done;
    const float* save;
    const float* cm;
    float* dgates;             // [S*n, 512] pre-activation gate gradients
};

// Back-propagation through time.  Step t (descending): dh = dhead[t] . Wh + (1 - done[t+1]) dh_rec; the cell backward of
// lstm_cell_bwd_kernel; dh_rec for step t-1 = dgates[t] . W_hh on the tensor cores (dgates rounded to bf16).
__global__ void __launch_bounds__(kThreads, 1) lstm_rec_bwd(const RecBwdP p) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* sW = smem;
    uint8_t* sG = smem + (size_t)kG * kWPitch;                 // two dgates buffers [16][512] (step parity)
    float* sWh = reinterpret_cast<float*>(sG + 2 * kRows * kGPitch);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gq = lane >> 2, tq = lane & 3;
    load_whh(sW, p.whh);
    for (int i = tid; i < p.A1 * kH; i += blockDim.x) sWh[i] = __ldg(p.wh + i);
    const int64_t n = p.n;
    int64_t row[2];
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) { row[h] = (int64_t)blockIdx.x * kRows + gq + 8 * h; valid[h] = row[h] < n; }
    float dhr[2][2][2], dcr[2][2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) dhr[h][hf][0] = dhr[h][hf][1] = dcr[h][hf][0] = dcr[h][hf][1] = 0.f;
    __syncthreads();
    const uint32_t sWa = smem_u32(sW), sGa = smem_u32(sG);
    const uint32_t bcol = sWa + (uint32_t)(((lane & 7) + ((lane >> 3) & 1) * 8) * kWPitch + (16 * warp + (lane >> 4) * 8) * 2);
    for (int t = p.S - 1; t >= 0; --t) {
        uint8_t* buf = sG + (size_t)(t & 1) * kRows * kGPitch;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t r = (int64_t)t * n + row[h];
            float keep_next = 0.f, keep = 0.f;
            if (valid[h]) {
                keep = 1.0f - __ldg(p.done + r);
                if (t + 1 < p.S) keep_next = 1.0f - __ldg(p.done + r + n);
            }
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int u = 16 * warp + 8 * hf + 2 * tq;
                float dg[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
                if (valid[h]) {
                    float dh0 = 0.f, dh1 = 0.f;
                    for (int a = 0; a < p.A1; ++a) {
                        const float d = __ldg(p.dhead + r * p.A1 + a);
                        const float2 w = *reinterpret_cast<const float2*>(sWh + a * kH + u);
                        dh0 = fmaf(d, w.x, dh0); dh1 = fmaf(d, w.y, dh1);
                    }
                    const float dhv[2] = {dh0 + keep_next * dhr[h][hf][0], dh1 + keep_next * dhr[h][hf][1]};
                    float s[5][2];
#pragma unroll
                    for (int k = 0; k < 5; ++k) {
                        const float2 v = __ldg(reinterpret_cast<const float2*>(p.save + (r * 5 + k) * kH + u));
                        s[k][0] = v.x; s[k][1] = v.y;
                    }
                    const float2 cmv = __ldg(reinterpret_cast<const float2*>(p.cm + r * kH + u));
                    const float cmx[2] = {cmv.x, cmv.y};
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float i = s[0][e], f = s[1][e], g = s[2][e], o = s[3][e], tc = s[4][e];
                        const float dh = dhv[e];
                        const float dc = dh * o * (1.0f - tc * tc) + dcr[h][hf][e];
                        dg[0][e] = dc * g * i * (1.0f - i);
                        dg[1][e] = dc * cmx[e] * f * (1.0f - f);
                        dg[2][e] = dc * i * (1.0f - g * g);
                        dg[3][e] = dh * tc * o * (1.0f - o);
                        dcr[h][hf][e] = keep * dc * f;
                    }
#pragma unroll
                    for (int g = 0; g < 4; ++g)
                        *reinterpret_cast<float2*>(p.dgates + r * kG + g * kH + u) = make_float2(dg[g][0], dg[g][1]);
                }
#pragma unroll
                for (int g = 0; g < 4; ++g)
                    *reinterpret_cast<uint32_t*>(buf + (gq + 8 * h) * kGPitch + (g * kH + u) * 2) = pack_bf16x2(dg[g][0], dg[g][1]);
            }
        }
        __syncthreads();                                        // dgates of this step are staged
        if (t == 0) break;
        float acc[2][4];
#pragma unroll
        for (int j = 0; j < 2; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        const uint32_t arow = sGa + (uint32_t)((t & 1) * kRows * kGPitch + (lane & 15) * kGPitch + (lane >> 4) * 16);
#pragma unroll 8
        for (int kc = 0; kc < kG / 16; ++kc) {
            uint32_t a0, a1, a2, a3, b0, b1, b2, b3;
            ldsm_x4(arow + kc * 32, a0, a1, a2, a3);
            ldsm_x4_t(bcol + kc * 16 * kWPitch, b0, b1, b2, b3);
            mma16816(acc[0], a0, a1, a2, a3, b0, b1);
            mma16816(acc[1], a0, a1, a2, a3, b2, b3);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) { dhr[h][hf][0] = acc[hf][2 * h]; dhr[h][hf][1] = acc[hf][2 * h + 1]; }
    }
}

}  // namespace lstm
}  // namespace b200rl
