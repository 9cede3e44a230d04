// IMPALA-CNN (cleanrl/ppo_procgen.py:89-150) on the Hopper tensor cores: bf16 operands, fp32 accumulation.
//
// Activations are dense channel-last bf16 tensors [n, H, W, C] (C = 16 or 32: 32- or 64-byte pixels).  Every 3x3, pad-1
// convolution stages a band of TR output rows plus its two halo rows into shared memory as a ZERO-BORDERED linear
// pixel grid (row width Ws = W + 2, pitch C*2 + 16 bytes): tap (dy, dx) of grid position q is position q + dy*Ws + dx,
// so the convolution is a GEMM whose A rows are read at 9 shifted start positions.  The A fragments are loaded with
// ldmatrix, whose eight row addresses are arbitrary 16-byte-aligned shared-memory addresses: any row shift is legal,
// the 16-byte padding of the pitch keeps the 8 rows of an 8x8 matrix on distinct banks, and no swizzle constraint
// applies (DESIGN §4).  The MMAs are mma.sync m16n8k16 (bf16 -> fp32).
//
//   seq0 conv     Cin = 3 on uint8 NHWC frames [*, 64, 64, 3] read through the minibatch gather `rows`: the staging loop
//                 builds 16-channel rows j = dx*3 + c (9 used) of the three horizontal taps, so the conv is 3 vertical taps
//                 with K = 16.  0..255 is exact in bf16; the /255 is applied to the fp32 accumulator.
//   max-pool      3x3, stride 2, pad 1 (-inf padding), first maximum in row-major window order; arg-max kept (0..8).
//   residual      x + conv1(relu(conv0(relu(x)))): conv0 stages relu(x) (ReLU applied while staging), its epilogue writes
//                 y0 = bf16(relu(acc + b0)); conv1's epilogue writes the stream bf16(x + acc + b1) in fp32 before the
//                 one rounding.  The last block writes relu(stream) (the fc input, = torch's Flatten/ReLU in the fc's
//                 packed K order (y*8 + x)*32 + c) and its (> 0) bits.
//   backward      data gradient = the same window conv over dY with flipped, transposed weights; its epilogue applies the
//                 ReLU mask of the forward input (from the stored bf16 tensor: value > 0) and adds the skip gradient.
//                 Weight gradient: dW^T[co, (tap, ci)] = sum_q dY[q, co] X[q + shift_tap, ci] over the staged bands of a
//                 CTA's fixed band range, per-CTA partials folded in a fixed order (deterministic), bias = column sums.
//   fc / heads    fc 2048 -> 256 on tc_gemm_tma (forward and data gradient) and tc_wgrad_tma (folded by tc_fold_fc, bias by
//                 tc_colsum_*); heads (A+1 <= kMaxHeads) on CUDA cores in fp32 (tc_heads_* with 256 hidden units).
//   PPG variant   cleanrl/ppg_procgen.py:168-211: the same trunk with a third head, [logits | value | aux_value] = A + 2
//                 outputs.  `critic` (column A) reads a detached copy of the hidden layer: its dhead column reaches its own
//                 weight and bias only, never the hidden layer's data gradient.  b200rl_impala_ppg_*.
#include <cuda.h>
#include <algorithm>
#include <cstring>
#include "tc_base.cuh"
#include "tc_gemm_tma.cuh"
#include "tc_reduce.cuh"
#include "tc_heads.cuh"
#include "tc_mma_sync.cuh"

namespace b200rl {
using namespace tc;

namespace imp {

constexpr int kThreads = 256;
constexpr int kWgradCtas = 264;           // row splits of the conv weight gradients: two waves on 132 SMs

__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
// ReLU of 2 packed bf16 (sign bit set -> +0)
__device__ __forceinline__ uint32_t relu2(uint32_t w) {
    const uint32_t neg = ((w >> 15) & 0x00010001u) * 0xFFFFu;
    return w & ~neg;
}

// ---------------------------------------------------------------- band geometry (shared by host and device)
// A CTA processes groups of NB bands; band b = (image b / (H/TR), output rows [y0, y0 + TR)).  Staged band bl occupies
// grid positions [bl*PB, (bl+1)*PB), PB = (TR+2)*Ws; staged row r is image row y0 - 1 + r, column c is image column
// c - 1 (or c for the folded seq0 frames).  GEMM rows run over all NB*PB positions (rounded up to 16); only positions with
// r < TR and c < W are outputs.  Positions past NB*PB (the shifted reads of the last rows) are zero.
struct Geo {
    int H, W, TR, NB, fold;
    __host__ __device__ int Ws() const { return fold ? W : W + 2; }
    __host__ __device__ int PB() const { return (TR + 2) * Ws(); }
    __host__ __device__ int mtiles() const { return (NB * PB() + 15) / 16; }
    __host__ __device__ int spos() const { return mtiles() * 16 + 2 * Ws() + 2; }
    __host__ __device__ int ntaps() const { return fold ? 3 : 9; }
    __host__ __device__ int shift(int t) const { return fold ? t * Ws() : (t / 3) * Ws() + (t % 3); }
    __host__ __device__ int bands_per_image() const { return H / TR; }
};

enum Epi { E_BIAS = 0, E_RELU = 1, E_SKIP = 2, E_DGRAD = 3 };

struct ConvP {
    Geo g;
    const void* in;            // bf16 [n, H, W, CIN] (or uint8 frames [*, 64, 64, 3] when g.fold)
    const int64_t* rows;       // fold only: frame index of batch row i (null = i)
    int relu_in;               // stage relu(in)
    int64_t nbands;            // n * H / TR
    const bf16* w;             // packed [COUT][ntaps*CIN]
    const float* bias;
    float scale;
    int epi;
    bf16* out;                 // [n, H, W, COUT]
    const bf16* aux;           // E_SKIP: the residual input x; E_DGRAD: ReLU-mask reference (null = no mask)
    const bf16* skipg;         // E_DGRAD: gradient added after the mask (null = none)
    int relu_out;              // E_SKIP: write relu(stream) and its bits (fc input)
    uint32_t* mask_out;        // [n, H*W] words, bit c = (relu(stream)[.., c] > 0) (COUT = 32)
};

// stage NB bands of the input into the zero-bordered shared grid [spos][CIN] (pitch CIN*2 + 16 bytes)
template <int CIN>
__device__ __forceinline__ void stage_bands(uint8_t* sX, const Geo& g, const void* in, const int64_t* rows, int relu_in,
                                            int64_t band0, int64_t nbands) {
    constexpr int PITCH = CIN * 2 + 16, CH = CIN / 8;
    const int Ws = g.Ws(), PB = g.PB(), S = g.spos(), bpi = g.bands_per_image();
    if (g.fold) {
        // folded seq0 frames: row j = dx*3 + c of pixel (y, x) = frame[y][x + dx - 1][c], j < 9; uint8 -> bf16
        const uint8_t* fr = reinterpret_cast<const uint8_t*>(in);
        for (int q = threadIdx.x; q < S; q += blockDim.x) {
            uint32_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            const int bl = q / PB;
            const int64_t b = band0 + bl;
            if (bl < g.NB && b < nbands) {
                const int rem = q - bl * PB, r = rem / Ws, c = rem - r * Ws;
                const int64_t i = b / bpi;
                const int y = (int)(b - i * bpi) * g.TR - 1 + r;
                if (y >= 0 && y < g.H) {
                    const int64_t img = rows ? __ldg(rows + i) : i;
                    const uint8_t* src = fr + ((img * g.H + y) * g.W) * 3;
                    float f[10];
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        const int x = c + dx - 1;
                        const bool ok = x >= 0 && x < g.W;
#pragma unroll
                        for (int ch = 0; ch < 3; ++ch) f[dx * 3 + ch] = ok ? (float)__ldg(src + x * 3 + ch) : 0.f;
                    }
                    f[9] = 0.f;
#pragma unroll
                    for (int e = 0; e < 5; ++e) v[e] = pack_bf16x2(f[2 * e], f[2 * e + 1]);
                }
            }
            int4* d = reinterpret_cast<int4*>(sX + (size_t)q * PITCH);
            d[0] = make_int4((int)v[0], (int)v[1], (int)v[2], (int)v[3]);
            d[1] = make_int4((int)v[4], (int)v[5], (int)v[6], (int)v[7]);
        }
        return;
    }
    const bf16* x = reinterpret_cast<const bf16*>(in);
    for (int idx = threadIdx.x; idx < S * CH; idx += blockDim.x) {
        const int q = idx / CH, ch = idx - q * CH;
        int4 v = make_int4(0, 0, 0, 0);
        const int bl = q / PB;
        const int64_t b = band0 + bl;
        if (bl < g.NB && b < nbands) {
            const int rem = q - bl * PB, r = rem / Ws, c = rem - r * Ws;
            const int64_t i = b / bpi;
            const int y = (int)(b - i * bpi) * g.TR - 1 + r, xx = c - 1;
            if (y >= 0 && y < g.H && xx >= 0 && xx < g.W) {
                v = ldg16(x + (((i * g.H + y) * g.W + xx) * CIN + ch * 8));
                if (relu_in) {
                    v.x = (int)relu2((uint32_t)v.x); v.y = (int)relu2((uint32_t)v.y);
                    v.z = (int)relu2((uint32_t)v.z); v.w = (int)relu2((uint32_t)v.w);
                }
            }
        }
        *reinterpret_cast<int4*>(sX + (size_t)q * PITCH + ch * 16) = v;
    }
}

// output pixel of GEMM row q of the group starting at band0; returns the element offset of (i, y, x, 0) / C or -1
__device__ __forceinline__ int64_t out_pixel(const Geo& g, int64_t band0, int64_t nbands, int q) {
    const int Ws = g.Ws(), PB = g.PB();
    const int bl = q / PB;
    const int64_t b = band0 + bl;
    if (bl >= g.NB || b >= nbands) return -1;
    const int rem = q - bl * PB, r = rem / Ws, c = rem - r * Ws;
    if (r >= g.TR || c >= g.W) return -1;
    const int bpi = g.bands_per_image();
    const int64_t i = b / bpi;
    const int y = (int)(b - i * bpi) * g.TR + r;
    return (i * g.H + y) * g.W + c;
}

// ---------------------------------------------------------------- window convolution (forward and data gradient)
template <int CIN, int COUT>
__global__ void __launch_bounds__(kThreads) conv_win(const ConvP p) {
    constexpr int PA = CIN * 2 + 16;
    constexpr int NT8 = COUT / 8;
    extern __shared__ __align__(16) uint8_t smem[];
    const Geo g = p.g;
    const int NTAPS = g.ntaps(), K = NTAPS * CIN, PW = K * 2 + 16;
    uint8_t* sW = smem;
    uint8_t* sX = smem + (size_t)COUT * PW;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // resident weights [COUT][K] (pitch PW)
    for (int idx = tid; idx < COUT * (K / 8); idx += blockDim.x) {
        const int co = idx / (K / 8), k8 = idx - co * (K / 8);
        *reinterpret_cast<int4*>(sW + (size_t)co * PW + k8 * 16) = ldg16(p.w + (size_t)co * K + k8 * 8);
    }
    const int mt = g.mtiles();
    const int64_t ngroups = (p.nbands + g.NB - 1) / g.NB;
    const uint32_t sWa = smem_u32(sW), sXa = smem_u32(sX);
    const int gq = lane >> 2, tq = lane & 3;
    for (int64_t grp = blockIdx.x; grp < ngroups; grp += gridDim.x) {
        const int64_t band0 = grp * g.NB;
        __syncthreads();                                       // previous group's reads of sX are done
        stage_bands<CIN>(sX, g, p.in, p.rows, p.relu_in, band0, p.nbands);
        __syncthreads();
        for (int m = warp; m < mt; m += kThreads / 32) {
            float acc[NT8][4];
#pragma unroll
            for (int j = 0; j < NT8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
            const uint32_t arow = sXa + (uint32_t)((m * 16 + (lane & 15)) * PA + (lane >> 4) * 16);
            const uint32_t brow = sWa + (uint32_t)(((lane & 7) + ((lane >> 4) << 3)) * PW + ((lane >> 3) & 1) * 16);
            for (int t = 0; t < NTAPS; ++t) {
                const uint32_t at = arow + (uint32_t)(g.shift(t) * PA);
#pragma unroll
                for (int kc = 0; kc < CIN / 16; ++kc) {
                    uint32_t a0, a1, a2, a3;
                    ldsm_x4(at + kc * 32, a0, a1, a2, a3);
                    const uint32_t bk = brow + (uint32_t)((t * CIN + kc * 16) * 2);
#pragma unroll
                    for (int np = 0; np < COUT / 16; ++np) {
                        uint32_t b0, b1, b2, b3;
                        ldsm_x4(bk + np * 16 * PW, b0, b1, b2, b3);
                        mma16816(acc[2 * np], a0, a1, a2, a3, b0, b1);
                        mma16816(acc[2 * np + 1], a0, a1, a2, a3, b2, b3);
                    }
                }
            }
            // epilogue: lane holds rows m*16 + gq (+8), channels 8j + 2tq (+1)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t pix = out_pixel(g, band0, p.nbands, m * 16 + gq + 8 * h);
                uint32_t bits = 0;
                if (pix >= 0) {
                    const int64_t base = pix * COUT;
#pragma unroll
                    for (int j = 0; j < NT8; ++j) {
                        const int co = 8 * j + 2 * tq;
                        float v0 = acc[j][2 * h], v1 = acc[j][2 * h + 1];
                        uint32_t o;
                        if (p.epi == E_DGRAD) {
                            if (p.aux) {
                                const uint32_t r = __ldg(reinterpret_cast<const unsigned int*>(p.aux + base + co));
                                if (!(bf_lo(r) > 0.f)) v0 = 0.f;
                                if (!(bf_hi(r) > 0.f)) v1 = 0.f;
                            }
                            if (p.skipg) {
                                const uint32_t sg = __ldg(reinterpret_cast<const unsigned int*>(p.skipg + base + co));
                                v0 += bf_lo(sg); v1 += bf_hi(sg);
                            }
                            o = pack_bf16x2(v0, v1);
                        } else {
                            v0 = fmaf(v0, p.scale, p.bias[co]); v1 = fmaf(v1, p.scale, p.bias[co + 1]);
                            if (p.epi == E_RELU) {
                                o = pack_bf16x2_relu(v0, v1);
                            } else if (p.epi == E_SKIP) {
                                const uint32_t x = __ldg(reinterpret_cast<const unsigned int*>(p.aux + base + co));
                                v0 += bf_lo(x); v1 += bf_hi(x);
                                if (p.relu_out) {
                                    o = pack_bf16x2_relu(v0, v1);
                                    bits |= (bf_lo(o) > 0.f ? 1u : 0u) << co;
                                    bits |= (bf_hi(o) > 0.f ? 1u : 0u) << (co + 1);
                                } else {
                                    o = pack_bf16x2(v0, v1);
                                }
                            } else {
                                o = pack_bf16x2(v0, v1);
                            }
                        }
                        *reinterpret_cast<unsigned int*>(p.out + base + co) = o;
                    }
                }
                if (p.mask_out) {                              // OR the quad's bits: one word per pixel (COUT = 32)
                    bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
                    bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
                    if (pix >= 0 && tq == 0) p.mask_out[pix] = bits;
                }
            }
        }
    }
}

// ---------------------------------------------------------------- weight gradient
struct WgradP {
    Geo g;
    const void* x;             // forward input (bf16 [n,H,W,CIN] or uint8 frames when g.fold)
    const int64_t* rows;
    int relu_in;
    const bf16* dy;            // [n, H, W, COUT]
    int64_t nbands;
    int64_t groups_per_cta;
    float* ws;                 // [gridDim.x][COUT][ntaps*CIN]
    float* wsb;                // [gridDim.x][COUT]
};

template <int CIN, int COUT, int FOLD>
__global__ void __launch_bounds__(kThreads) wgrad_win(const WgradP p) {
    constexpr int PX = CIN * 2 + 16, PY = COUT * 2 + 16;
    constexpr int MT = COUT / 16;
    constexpr int CC = CIN / 8;                               // n8 tiles per tap
    constexpr int NTAPS = FOLD ? 3 : 9;
    constexpr int NIT = MT * NTAPS * CC;                      // items (m16 x n8 tiles)
    constexpr int MAXI = (NIT + 7) / 8;                       // items per warp
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float red[kThreads];
    const Geo g = p.g;
    const int S = g.spos(), KT = g.mtiles();
    uint8_t* sX = smem;
    uint8_t* sY = smem + (size_t)S * PX;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t sXa = smem_u32(sX), sYa = smem_u32(sY);
    float acc[MAXI][4];
#pragma unroll
    for (int i = 0; i < MAXI; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const int bco = tid % COUT, brl = tid / COUT;              // bias column sums: row lanes x channels
    constexpr int BRL = kThreads / COUT;
    float bacc = 0.f;
    const int64_t ngroups = (p.nbands + g.NB - 1) / g.NB;
    const int64_t g0 = (int64_t)blockIdx.x * p.groups_per_cta;
    int64_t g1 = g0 + p.groups_per_cta;
    if (g1 > ngroups) g1 = ngroups;
    const int PB = g.PB();
    for (int64_t grp = g0; grp < g1; ++grp) {
        const int64_t band0 = grp * g.NB;
        __syncthreads();
        stage_bands<CIN>(sX, g, p.x, p.rows, p.relu_in, band0, p.nbands);
        // dY on the same grid positions (zero where q is not an output)
        for (int idx = tid; idx < S * (COUT / 8); idx += blockDim.x) {
            const int q = idx / (COUT / 8), ch = idx - q * (COUT / 8);
            int4 v = make_int4(0, 0, 0, 0);
            const int64_t pix = q < g.NB * PB ? out_pixel(g, band0, p.nbands, q) : -1;
            if (pix >= 0) v = ldg16(p.dy + pix * COUT + ch * 8);
            *reinterpret_cast<int4*>(sY + (size_t)q * PY + ch * 16) = v;
        }
        __syncthreads();
        for (int q = brl; q < KT * 16; q += BRL) {
            const bf16 v = *reinterpret_cast<const bf16*>(sY + (size_t)q * PY + bco * 2);
            bacc += __bfloat162float(v);
        }
        for (int kt = 0; kt < KT; ++kt) {
#pragma unroll
            for (int ii = 0; ii < MAXI; ++ii) {
                const int it = warp + 8 * ii;
                if (it >= NIT) break;
                const int mtile = it / (NTAPS * CC), nt = it - mtile * (NTAPS * CC);
                const int tap = nt / CC, c8 = nt - tap * CC;
                uint32_t a0, a1, a2, a3, b0, b1;
                // A = dY^T (m = co, k = position): stored [position][co] -> transposed ldmatrix
                ldsm_x4_t(sYa + (uint32_t)((kt * 16 + (lane & 7) + (lane >> 4) * 8) * PY + (mtile * 16 + ((lane >> 3) & 1) * 8) * 2),
                          a0, a1, a2, a3);
                // B = shifted X (k = position, n = ci): stored [position][ci] -> transposed ldmatrix
                ldsm_x2_t(sXa + (uint32_t)((kt * 16 + g.shift(tap) + (lane & 7) + ((lane >> 3) & 1) * 8) * PX + c8 * 16), b0, b1);
                mma16816(acc[ii], a0, a1, a2, a3, b0, b1);
            }
        }
    }
    // partials: ws[cta][co][tap*CIN + ci]
    const int K = NTAPS * CIN;
    float* wsc = p.ws + (size_t)blockIdx.x * COUT * K;
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int ii = 0; ii < MAXI; ++ii) {
        const int it = warp + 8 * ii;
        if (it >= NIT) break;
        const int mtile = it / (NTAPS * CC), nt = it - mtile * (NTAPS * CC);
        const int col = nt * 8 + 2 * tq, co = mtile * 16 + gq;
        *reinterpret_cast<float2*>(wsc + (size_t)co * K + col) = make_float2(acc[ii][0], acc[ii][1]);
        *reinterpret_cast<float2*>(wsc + (size_t)(co + 8) * K + col) = make_float2(acc[ii][2], acc[ii][3]);
    }
    red[tid] = bacc;
    __syncthreads();
    if (tid < COUT) {
        float s = 0.f;
        for (int l = 0; l < BRL; ++l) s += red[l * COUT + tid];
        p.wsb[(size_t)blockIdx.x * COUT + tid] = s;
    }
}

// fixed-order fold of the per-CTA partials into torch's layout w[co][ci][ky][kx] (and the bias)
__global__ void __launch_bounds__(256) fold_conv(const float* __restrict__ ws, const float* __restrict__ wsb, int S, int Cout,
                                                 int Cin, int fold, float scale, float* __restrict__ dw, float* __restrict__ db) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int nw = Cout * Cin * 9;
    if (idx < nw) {
        const int kx = idx % 3, ky = (idx / 3) % 3, ci = (idx / 9) % Cin, co = idx / (9 * Cin);
        const int K = fold ? 48 : 9 * Cin;
        const int col = fold ? ky * 16 + kx * 3 + ci : (ky * 3 + kx) * Cin + ci;
        float s = 0.f;
        for (int z = 0; z < S; ++z) s += ws[((size_t)z * Cout + co) * K + col];
        dw[idx] = s * scale;
    } else if (idx < nw + Cout) {
        const int co = idx - nw;
        float s = 0.f;
        for (int z = 0; z < S; ++z) s += wsb[(size_t)z * Cout + co];
        db[co] = s;
    }
}

// ---------------------------------------------------------------- max-pool 3x3 / stride 2 / pad 1 (channel-last bf16)
__global__ void __launch_bounds__(256) maxpool_fwd(const bf16* __restrict__ x, int64_t n, int H, int W, int C,
                                                   bf16* __restrict__ y, uint8_t* __restrict__ arg) {
    const int OH = (H + 1) / 2, OW = (W + 1) / 2;
    const int64_t total = n * OH * OW * C;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        int64_t t = idx / C;
        const int ox = (int)(t % OW); t /= OW;
        const int oy = (int)(t % OH);
        const int64_t i = t / OH;
        float best = -INFINITY;
        int bi = 0;
        bf16 bv = __float2bfloat16(-INFINITY);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int iy = oy * 2 + ky - 1, ix = ox * 2 + kx - 1;
                if (iy < 0 || ix < 0 || iy >= H || ix >= W) continue;
                const bf16 e = x[((i * H + iy) * W + ix) * C + c];
                const float v = __bfloat162float(e);
                if (v > best || (v != v && !(best != best))) { best = v; bi = ky * 3 + kx; bv = e; }   // first maximum
            }
        y[idx] = bv;
        arg[idx] = (uint8_t)bi;
    }
}
// dx[i][iy][ix][c] = sum of dy over the (<= 4) windows whose arg-max is (iy, ix), in window order (deterministic)
__global__ void __launch_bounds__(256) maxpool_bwd(const bf16* __restrict__ dy, const uint8_t* __restrict__ arg, int64_t n, int H,
                                                   int W, int C, bf16* __restrict__ dx) {
    const int OH = (H + 1) / 2, OW = (W + 1) / 2;
    const int64_t total = n * H * W * C;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        int64_t t = idx / C;
        const int ix = (int)(t % W); t /= W;
        const int iy = (int)(t % H);
        const int64_t i = t / H;
        float s = 0.f;
        for (int oy = iy / 2; oy <= (iy + 1) / 2; ++oy) {
            if (oy >= OH) continue;
            const int ky = iy - (oy * 2 - 1);
            if (ky < 0 || ky > 2) continue;
            for (int ox = ix / 2; ox <= (ix + 1) / 2; ++ox) {
                if (ox >= OW) continue;
                const int kx = ix - (ox * 2 - 1);
                if (kx < 0 || kx > 2) continue;
                const int64_t o = ((i * OH + oy) * OW + ox) * C + c;
                if (arg[o] == ky * 3 + kx) s += __bfloat162float(dy[o]);
            }
        }
        dx[idx] = __float2bfloat16(s);
    }
}

// ---------------------------------------------------------------- weight packing
// conv w[co][ci][ky][kx] -> fwd [co][(ky*3+kx)*Cin + ci]; dgrad [ci][(ky'*3+kx')*Cout + co] = w[co][ci][2-ky'][2-kx']
__global__ void pack_conv(const float* __restrict__ w, int Cout, int Cin, bf16* __restrict__ fwd, bf16* __restrict__ dg) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= Cout * Cin * 9) return;
    const int kx = idx % 3, ky = (idx / 3) % 3, ci = (idx / 9) % Cin, co = idx / (9 * Cin);
    const bf16 v = __float2bfloat16(w[idx]);
    fwd[co * 9 * Cin + (ky * 3 + kx) * Cin + ci] = v;
    dg[ci * 9 * Cout + ((2 - ky) * 3 + (2 - kx)) * Cout + co] = v;
}
// seq0 conv w[co][c][dy][dx] (Cin = 3) -> [co][dy*16 + dx*3 + c], zero for j >= 9
__global__ void pack_conv_fold(const float* __restrict__ w, bf16* __restrict__ fwd) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 16 * 48) return;
    const int co = idx / 48, k = idx % 48, dy = k / 16, j = k % 16;
    float v = 0.f;
    if (j < 9) v = w[((co * 3 + j % 3) * 3 + dy) * 3 + j / 3];
    fwd[idx] = __float2bfloat16(v);
}
// fc w[o][c*64 + p] -> fwd [o][p*32 + c] (K order of the dense 8x8x32 stream); dgrad [p*32 + c][o]
__global__ void pack_fc(const float* __restrict__ w, bf16* __restrict__ fwd, bf16* __restrict__ dg) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 256 * 2048) return;
    const int o = idx >> 11, k = idx & 2047, c = k >> 6, pp = k & 63;
    const bf16 v = __float2bfloat16(w[idx]);
    fwd[(size_t)o * 2048 + pp * 32 + c] = v;
    dg[(size_t)(pp * 32 + c) * 256 + o] = v;
}
// ---------------------------------------------------------------- host plan
struct ImpalaLayout {       // flat fp32 parameter offsets (ImpalaAgent / PPGAgent._param_order) and packed bf16 offsets
    int A1;                 // head outputs: A + 1 (actor | critic) or A + 2 (actor | critic | aux_critic)
    int64_t cw[15], cb[15], fcw, fcb, hw, hb, total;
    int64_t pf[15], pd[15], pfc, pfcd, packed_total;
    explicit ImpalaLayout(int A1_) : A1(A1_) {
        int64_t o = 0, q = 0;
        const int cin[3] = {3, 16, 32}, cout[3] = {16, 32, 32};
        for (int s = 0; s < 3; ++s)
            for (int l = 0; l < 5; ++l) {
                const int k = s * 5 + l, ci = l == 0 ? cin[s] : cout[s], co = cout[s];
                cw[k] = o; o += (int64_t)co * ci * 9;
                cb[k] = o; o += co;
                pf[k] = q; q += k == 0 ? 16 * 48 : (int64_t)co * ci * 9;
                pd[k] = q; q += k == 0 ? 0 : (int64_t)co * ci * 9;
            }
        fcw = o; o += 256 * 2048;
        fcb = o; o += 256;
        hw = o; o += (int64_t)A1 * 256;
        hb = o; o += A1;
        total = o;
        pfc = q; q += 256 * 2048;
        pfcd = q; q += 256 * 2048;
        packed_total = q;
    }
};

struct ImpalaActs {         // byte offsets in the (zero-initialised) activation workspace for batch n
    int64_t c0, s[3][3], y[3][2], arg[3], c1, c2, h0, mh0, hid, mhid, dc, ga, gb, gy, dhid, total;
    explicit ImpalaActs(int64_t n) {
        int64_t o = 0;
        auto take = [&](int64_t bytes) { const int64_t r = o; o += (bytes + 255) & ~int64_t(255); return r; };
        const int64_t HWC[3] = {32 * 32 * 16, 16 * 16 * 32, 8 * 8 * 32};     // per-sample stream elements of each sequence
        c0 = take(n * 65536 * 2);
        c1 = take(n * 32768 * 2);
        c2 = take(n * 8192 * 2);
        for (int q = 0; q < 3; ++q) {
            for (int j = 0; j < 3; ++j) s[q][j] = (q == 2 && j == 2) ? -1 : take(n * HWC[q] * 2);
            for (int j = 0; j < 2; ++j) y[q][j] = take(n * HWC[q] * 2);
            arg[q] = take(n * HWC[q]);
        }
        h0 = take(n * 2048 * 2);
        mh0 = take(n * 64 * 4);
        hid = take(n * 256 * 2);
        mhid = take(n * 8 * 4);
        dc = take(n * 65536 * 2);
        ga = take(n * 16384 * 2);
        gb = take(n * 16384 * 2);
        gy = take(n * 16384 * 2);
        dhid = take(n * 256 * 2);
        total = o;
    }
};

// A actions plus `values` value heads (1: actor-critic, 2: PPG's critic and aux_critic)
static bool heads_ok(int A, int values = 1) { return A >= 1 && A + values <= kMaxHeads; }
constexpr int64_t kMaxN = (int64_t)1 << 17;

static Geo geo(int H, int fold = 0) {
    Geo g;
    g.H = H; g.W = H; g.fold = fold;
    if (fold) { g.TR = 4; g.NB = 1; }                      // 64x64 frames: 6 x 64 staged positions
    else if (H == 32) { g.TR = 8; g.NB = 1; }              // 10 x 34
    else if (H == 16) { g.TR = 16; g.NB = 1; }             // 18 x 18
    else { g.TR = 8; g.NB = 3; }                           // 3 images of 10 x 10
    return g;
}

template <int CIN, int COUT>
static int run_conv(ConvP p, int64_t n, cudaStream_t s, const char* what) {
    const Geo& g = p.g;
    p.nbands = n * g.bands_per_image();
    const size_t smem = (size_t)COUT * (g.ntaps() * CIN * 2 + 16) + (size_t)g.spos() * (CIN * 2 + 16);
    static SmemAttrCache attr;
    if (int rc = attr.ensure(conv_win<CIN, COUT>, smem, what)) return rc;
    const int64_t groups = (p.nbands + g.NB - 1) / g.NB;
    const int per_sm = (int)(200 * 1024 / (smem + 1024)) < 1 ? 1 : (int)(200 * 1024 / (smem + 1024));
    int64_t grid = (int64_t)num_sms() * (per_sm > 8 ? 8 : per_sm);
    if (grid > groups) grid = groups;
    conv_win<CIN, COUT><<<(unsigned)grid, kThreads, smem, s>>>(p);
    return check_launch(what);
}

static int64_t wgrad_ctas(int64_t groups) { return groups < kWgradCtas ? groups : kWgradCtas; }

template <int CIN, int COUT, int FOLD = 0>
static int run_wgrad(WgradP p, int64_t n, float scale, float* dw, float* db, cudaStream_t s, const char* what) {
    const Geo& g = p.g;
    p.nbands = n * g.bands_per_image();
    const int64_t groups = (p.nbands + g.NB - 1) / g.NB;
    const int64_t ctas = wgrad_ctas(groups);
    p.groups_per_cta = (groups + ctas - 1) / ctas;
    const int64_t used = (groups + p.groups_per_cta - 1) / p.groups_per_cta;
    const size_t smem = (size_t)g.spos() * (CIN * 2 + 16 + COUT * 2 + 16);
    static SmemAttrCache attr;
    if (g.fold != FOLD) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: geometry does not match the kernel", what);
    if (int rc = attr.ensure(wgrad_win<CIN, COUT, FOLD>, smem, what)) return rc;
    wgrad_win<CIN, COUT, FOLD><<<(unsigned)used, kThreads, smem, s>>>(p);
    const int cin = g.fold ? 3 : CIN;
    fold_conv<<<(unsigned)ceil_div(COUT * cin * 9 + COUT, 256), 256, 0, s>>>(p.ws, p.wsb, (int)used, COUT, cin, g.fold, scale, dw, db);
    return check_launch(what, 2);
}

static size_t wgrad_ws_floats() { return (size_t)kWgradCtas * 32 * 288; }

}  // namespace imp
}  // namespace b200rl

using namespace b200rl;
using namespace b200rl::imp;

extern "C" int64_t b200rl_impala_param_count(int A) { return A >= 1 ? ImpalaLayout(A + 1).total : -1; }
extern "C" size_t b200rl_impala_bf16_packed_bytes(int A) { return heads_ok(A) ? (size_t)ImpalaLayout(A + 1).packed_total * 2 : 0; }
extern "C" int64_t b200rl_impala_ppg_param_count(int A) { return A >= 1 ? ImpalaLayout(A + 2).total : -1; }
extern "C" size_t b200rl_impala_ppg_bf16_packed_bytes(int A) {
    return heads_ok(A, 2) ? (size_t)ImpalaLayout(A + 2).packed_total * 2 : 0;
}
extern "C" size_t b200rl_impala_bf16_acts_bytes(int64_t n) { return n >= 0 && n <= kMaxN ? (size_t)ImpalaActs(n).total : 0; }
extern "C" int b200rl_impala_bf16_acts_layout(int64_t n, int64_t* offsets) {
    B200RL_REQUIRE(offsets, "impala_acts_layout: null pointer");
    B200RL_REQUIRE(n >= 0 && n <= kMaxN, "impala_acts_layout: n=%lld out of range", (long long)n);
    const ImpalaActs Q(n);
    int k = 0;
    offsets[k++] = Q.c0; offsets[k++] = Q.c1; offsets[k++] = Q.c2;
    for (int q = 0; q < 3; ++q) {
        for (int j = 0; j < 3; ++j) offsets[k++] = Q.s[q][j];
        for (int j = 0; j < 2; ++j) offsets[k++] = Q.y[q][j];
        offsets[k++] = Q.arg[q];
    }
    const int64_t tail[9] = {Q.h0, Q.mh0, Q.hid, Q.mhid, Q.dc, Q.ga, Q.gb, Q.gy, Q.dhid};
    for (int j = 0; j < 9; ++j) offsets[k++] = tail[j];
    return B200RL_OK;
}
// the backward workspace = [big part: weight-gradient partials, sized for the largest n | small part], each the largest
// its launches need: heads, fc, convolutions
static size_t impala_big_bytes() { return std::max(wgrad_tma_bytes(kMaxN, 256, 2048), wgrad_ws_floats() * 4); }
static size_t impala_workspace_bytes(int64_t n, int A1) {
    const size_t small = std::max({heads_partial_bytes(n, A1, 256), colsum_ws(n, 256), (size_t)kWgradCtas * 32 * 4});
    return impala_big_bytes() + small + 512;
}
extern "C" size_t b200rl_impala_bf16_workspace_bytes(int64_t n, int A) {
    return n < 1 || n > kMaxN || !heads_ok(A) ? 0 : impala_workspace_bytes(n, A + 1);
}
extern "C" size_t b200rl_impala_ppg_bf16_workspace_bytes(int64_t n, int A) {
    return n < 1 || n > kMaxN || !heads_ok(A, 2) ? 0 : impala_workspace_bytes(n, A + 2);
}

// `values` = 1 (actor | critic) or 2 (the PPG variant's actor | critic | aux_critic)
static int impala_pack(const float* params, int A, int values, void* packed, void* stream) {
    B200RL_REQUIRE(params && packed, "impala_pack: null pointer");
    B200RL_REQUIRE(heads_ok(A, values), "impala_pack: A=%d outside [1,%d]", A, kMaxHeads - values);
    B200RL_REQUIRE(aligned(params, 16) && aligned(packed, 16), "impala_pack: misaligned buffer");
    const ImpalaLayout L(A + values);
    bf16* P = reinterpret_cast<bf16*>(packed);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "pack_weights", 0, (double)L.total * 4 + (double)L.packed_total * 2);
    pack_conv_fold<<<3, 256, 0, s>>>(params + L.cw[0], P + L.pf[0]);
    const int cin[3] = {3, 16, 32}, cout[3] = {16, 32, 32};
    for (int k = 1; k < 15; ++k) {
        const int q = k / 5, ci = k % 5 == 0 ? cin[q] : cout[q], co = cout[q];
        pack_conv<<<(unsigned)ceil_div(co * ci * 9, 256), 256, 0, s>>>(params + L.cw[k], co, ci, P + L.pf[k], P + L.pd[k]);
    }
    pack_fc<<<2048, 256, 0, s>>>(params + L.fcw, P + L.pfc, P + L.pfcd);
    return check_launch("impala_pack", 16);
}
extern "C" int b200rl_impala_bf16_pack(const float* params, int A, void* packed, void* stream) {
    return impala_pack(params, A, 1, packed, stream);
}
extern "C" int b200rl_impala_ppg_bf16_pack(const float* params, int A, void* packed, void* stream) {
    return impala_pack(params, A, 2, packed, stream);
}

namespace {
ConvP conv_defaults(const Geo& g) { ConvP p; memset(&p, 0, sizeof(p)); p.g = g; p.scale = 1.f; return p; }
WgradP wgrad_defaults(const Geo& g, float* ws, float* wsb) {
    WgradP p; memset(&p, 0, sizeof(p)); p.g = g; p.ws = ws; p.wsb = wsb; return p;
}
const int kH[3] = {64, 32, 16};           // conv input size of each sequence
}  // namespace

static int impala_forward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, int values, const float* params,
                          const void* packed, void* acts, float* head_out, void* stream) {
    B200RL_REQUIRE(n >= 0, "impala_forward: negative n");
    B200RL_REQUIRE(obs && params && packed && acts && head_out, "impala_forward: null pointer");
    B200RL_REQUIRE(heads_ok(A, values), "impala_forward: A=%d outside [1,%d]", A, kMaxHeads - values);
    B200RL_REQUIRE(n <= kMaxN, "impala_forward: n=%lld above %lld", (long long)n, (long long)kMaxN);
    B200RL_REQUIRE(aligned(params, 16) && aligned(packed, 16) && aligned(acts, 256) && aligned(head_out, 4) &&
                   aligned(rows, 8), "impala_forward: misaligned buffer");
    if (n == 0) return B200RL_OK;
    const int A1 = A + values;
    const ImpalaLayout L(A1);
    const ImpalaActs Q(n);
    const bf16* P = reinterpret_cast<const bf16*>(packed);
    uint8_t* ab = reinterpret_cast<uint8_t*>(acts);
    auto T = [&](int64_t off) { return reinterpret_cast<bf16*>(ab + off); };
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    const int cout[3] = {16, 32, 32};
    for (int q = 0; q < 3; ++q) {
        const int H = kH[q], C = cout[q], k0 = q * 5;
        bf16* c = T(q == 0 ? Q.c0 : q == 1 ? Q.c1 : Q.c2);
        ConvP p = conv_defaults(geo(H, q == 0));
        p.w = P + L.pf[k0]; p.bias = params + L.cb[k0]; p.epi = E_BIAS; p.out = c;
        {
            ProfScope ps(s, "impala_conv_fwd", 2.0 * n * H * H * C * 9 * (q == 0 ? 3 : kH[q] == 32 ? 16 : 32), 0);
            if (q == 0) { p.in = obs; p.rows = rows; p.scale = 1.0f / 255.0f; rc = run_conv<16, 16>(p, n, s, "impala/seq0_conv"); }
            else if (q == 1) { p.in = T(Q.s[0][2]); rc = run_conv<16, 32>(p, n, s, "impala/seq1_conv"); }
            else { p.in = T(Q.s[1][2]); rc = run_conv<32, 32>(p, n, s, "impala/seq2_conv"); }
            if (rc) return rc;
        }
        const int OH = H / 2;
        {
            ProfScope ps(s, "impala_maxpool", 0, (double)n * H * H * C * 2 + (double)n * OH * OH * C * 3);
            const int64_t tot = n * OH * OH * C;
            maxpool_fwd<<<(unsigned)std::min<int64_t>(ceil_div(tot, 256), (int64_t)num_sms() * 16), 256, 0, s>>>(
                c, n, H, H, C, T(Q.s[q][0]), ab + Q.arg[q]);
            if ((rc = check_launch("impala/maxpool"))) return rc;
        }
        for (int blk = 0; blk < 2; ++blk) {
            const int kc0 = k0 + 1 + 2 * blk, kc1 = kc0 + 1;
            const bool last = q == 2 && blk == 1;
            ProfScope ps(s, "impala_res_fwd", 2 * 2.0 * n * OH * OH * C * 9 * C, 0);
            ConvP a = conv_defaults(geo(OH));
            a.in = T(Q.s[q][blk]); a.relu_in = 1; a.w = P + L.pf[kc0]; a.bias = params + L.cb[kc0]; a.epi = E_RELU;
            a.out = T(Q.y[q][blk]);
            ConvP b = conv_defaults(geo(OH));
            b.in = T(Q.y[q][blk]); b.w = P + L.pf[kc1]; b.bias = params + L.cb[kc1]; b.epi = E_SKIP; b.aux = T(Q.s[q][blk]);
            if (last) { b.out = T(Q.h0); b.relu_out = 1; b.mask_out = reinterpret_cast<uint32_t*>(ab + Q.mh0); }
            else b.out = T(Q.s[q][blk + 1]);
            if (C == 16) {
                if ((rc = run_conv<16, 16>(a, n, s, "impala/res_conv0"))) return rc;
                if ((rc = run_conv<16, 16>(b, n, s, "impala/res_conv1"))) return rc;
            } else {
                if ((rc = run_conv<32, 32>(a, n, s, "impala/res_conv0"))) return rc;
                if ((rc = run_conv<32, 32>(b, n, s, "impala/res_conv1"))) return rc;
            }
        }
    }
    // fc 2048 -> 256 + ReLU (bits of hid > 0 for the heads' data gradient)
    KGemmParams g;
    memset(&g, 0, sizeof(g));
    g.scale = 1.f; g.A = T(Q.h0); g.M = n; g.nchunks = 32;
    g.Bw = P + L.pfc; g.N = 256; g.out = T(Q.hid); g.ldo = 256; g.bias = params + L.fcb; g.relu = 1;
    g.mask_out = reinterpret_cast<uint32_t*>(ab + Q.mhid);
    { ProfScope ps(s, "fc_fwd", 2.0 * n * 256 * 2048, (double)n * (2048 + 256) * 2 + 256.0 * 2048 * 2);
      if ((rc = launch_gemm_tma<64, 6>(g, s, "impala/fc"))) return rc; }
    ProfScope ps(s, "heads_fwd", 2.0 * n * 256 * A1, (double)n * (512 + 4 * A1));
    return heads_fwd<256>(T(Q.hid), params + L.hw, params + L.hb, n, A1, head_out, s, "impala/heads");
}
extern "C" int b200rl_impala_bf16_forward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                                          const void* packed, void* acts, float* head_out, void* stream) {
    return impala_forward(obs, rows, n, A, 1, params, packed, acts, head_out, stream);
}
extern "C" int b200rl_impala_ppg_bf16_forward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                                              const void* packed, void* acts, float* head_out, void* stream) {
    return impala_forward(obs, rows, n, A, 2, params, packed, acts, head_out, stream);
}

// values == 2: head column A (PPG's critic) read a detached hidden layer, so it stays out of the hidden layer's gradient
static int impala_backward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, int values, const float* params,
                           const void* packed, void* acts, const float* dhead, float* grads,
                           void* workspace, size_t workspace_bytes, void* stream) {
    B200RL_REQUIRE(n >= 1, "impala_backward: n must be >= 1");
    B200RL_REQUIRE(obs && params && packed && acts && dhead && grads && workspace, "impala_backward: null pointer");
    B200RL_REQUIRE(heads_ok(A, values), "impala_backward: A=%d outside [1,%d]", A, kMaxHeads - values);
    B200RL_REQUIRE(n <= kMaxN, "impala_backward: n=%lld above %lld", (long long)n, (long long)kMaxN);
    B200RL_REQUIRE(aligned(params, 16) && aligned(packed, 16) && aligned(acts, 256) && aligned(workspace, 256) &&
                   aligned(dhead, 4) && aligned(grads, 16) && aligned(rows, 8), "impala_backward: misaligned buffer");
    const int A1 = A + values;
    const size_t need = impala_workspace_bytes(n, A1);
    if (workspace_bytes < need) return fail(B200RL_ERR_WORKSPACE, "impala_backward: workspace %zu < %zu", workspace_bytes, need);
    const ImpalaLayout L(A1);
    const ImpalaActs Q(n);
    const bf16* P = reinterpret_cast<const bf16*>(packed);
    uint8_t* ab = reinterpret_cast<uint8_t*>(acts);
    auto T = [&](int64_t off) { return reinterpret_cast<bf16*>(ab + off); };
    cudaStream_t s = (cudaStream_t)stream;
    float* wsbig = reinterpret_cast<float*>(workspace);
    float* wssmall = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + impala_big_bytes());
    int rc;
    // ---- heads
    {
        ProfScope ps(s, "heads_bwd", 4.0 * n * 256 * A1, (double)n * (1024 + 8 * A1));
        if ((rc = heads_bwd_weight<256>(dhead, T(Q.hid), n, A1, wssmall, grads + L.hw, grads + L.hb, s, "impala/heads_bwd"))) return rc;
        if ((rc = heads_bwd_data<256>(dhead, params + L.hw, ab + Q.mhid, n, A1, T(Q.dhid), s, "impala/heads_bwd",
                                      values == 2 ? A : -1))) return rc;
    }
    // ---- fc: dW = dhid^T . h0 (row splits folded in order), db = column sums, dh0 = (dhid . Wfc) * (h0 > 0)
    {
        ProfScope ps(s, "fc_wgrad", 2.0 * n * 256 * 2048, (double)n * (2048 + 256) * 2 + 256.0 * 2048 * 4);
        const int splits = launch_wgrad_tma(T(Q.dhid), 256, T(Q.h0), 2048, n, wsbig, s, "impala/fc_wgrad");
        if (splits < 0) return splits;
        tc_fold_fc<<<2048, 256, 0, s>>>(wsbig, splits, 256, 2048, 256, 2048, 32, 64, 1.f, grads + L.fcw);
        if ((rc = check_launch("impala/fc_fold"))) return rc;
        if ((rc = colsum(T(Q.dhid), n, 256, 256, wssmall, grads + L.fcb, s))) return rc;
    }
    {
        KGemmParams g;
        memset(&g, 0, sizeof(g));
        g.scale = 1.f; g.A = T(Q.dhid); g.M = n; g.nchunks = 4;
        g.Bw = P + L.pfcd; g.N = 2048; g.out = T(Q.ga); g.ldo = 2048;
        g.mask_bits = reinterpret_cast<const uint32_t*>(ab + Q.mh0);
        ProfScope ps(s, "fc_dgrad", 2.0 * n * 256 * 2048, (double)n * (2048 + 256) * 2 + 256.0 * 2048 * 2);
        if ((rc = launch_gemm_tma<128, 3>(g, s, "impala/fc_dgrad"))) return rc;
    }
    // ---- sequences in reverse; G = gradient of the current stream tensor (ping-pong ga / gb), gy = d(y0)
    bf16* G = T(Q.ga);
    bf16* Gn = T(Q.gb);
    const int cin[3] = {3, 16, 32}, cout[3] = {16, 32, 32};
    for (int q = 2; q >= 0; --q) {
        const int H = kH[q], OH = H / 2, C = cout[q], k0 = q * 5;
        for (int blk = 1; blk >= 0; --blk) {
            const int kc0 = k0 + 1 + 2 * blk, kc1 = kc0 + 1;
            bf16* x = T(Q.s[q][blk]);
            bf16* y0 = T(Q.y[q][blk]);
            ProfScope ps(s, "impala_res_bwd", 4 * 2.0 * n * OH * OH * C * 9 * C, 0);
            WgradP w1 = wgrad_defaults(geo(OH), wsbig, wssmall);
            w1.x = y0; w1.dy = G;
            ConvP d1 = conv_defaults(geo(OH));
            d1.in = G; d1.w = P + L.pd[kc1]; d1.epi = E_DGRAD; d1.aux = y0; d1.out = T(Q.gy);
            WgradP w0 = wgrad_defaults(geo(OH), wsbig, wssmall);
            w0.x = x; w0.relu_in = 1; w0.dy = T(Q.gy);
            ConvP d0 = conv_defaults(geo(OH));
            d0.in = T(Q.gy); d0.w = P + L.pd[kc0]; d0.epi = E_DGRAD; d0.aux = x; d0.skipg = G; d0.out = Gn;
            if (C == 16) {
                if ((rc = run_wgrad<16, 16>(w1, n, 1.f, grads + L.cw[kc1], grads + L.cb[kc1], s, "impala/res_wgrad1"))) return rc;
                if ((rc = run_conv<16, 16>(d1, n, s, "impala/res_dgrad1"))) return rc;
                if ((rc = run_wgrad<16, 16>(w0, n, 1.f, grads + L.cw[kc0], grads + L.cb[kc0], s, "impala/res_wgrad0"))) return rc;
                if ((rc = run_conv<16, 16>(d0, n, s, "impala/res_dgrad0"))) return rc;
            } else {
                if ((rc = run_wgrad<32, 32>(w1, n, 1.f, grads + L.cw[kc1], grads + L.cb[kc1], s, "impala/res_wgrad1"))) return rc;
                if ((rc = run_conv<32, 32>(d1, n, s, "impala/res_dgrad1"))) return rc;
                if ((rc = run_wgrad<32, 32>(w0, n, 1.f, grads + L.cw[kc0], grads + L.cb[kc0], s, "impala/res_wgrad0"))) return rc;
                if ((rc = run_conv<32, 32>(d0, n, s, "impala/res_dgrad0"))) return rc;
            }
            bf16* t = G; G = Gn; Gn = t;
        }
        // max-pool: G = d(pooled) -> d(conv output) in dc
        bf16* dc = T(Q.dc);
        {
            ProfScope ps(s, "impala_maxpool", 0, (double)n * H * H * C * 2 + (double)n * OH * OH * C * 3);
            const int64_t tot = n * H * H * C;
            maxpool_bwd<<<(unsigned)std::min<int64_t>(ceil_div(tot, 256), (int64_t)num_sms() * 16), 256, 0, s>>>(
                G, ab + Q.arg[q], n, H, H, C, dc);
            if ((rc = check_launch("impala/maxpool_bwd"))) return rc;
        }
        ProfScope ps(s, "impala_conv_bwd", (q == 0 ? 1.0 : 2.0) * 2.0 * n * H * H * C * 9 * cin[q], 0);
        WgradP w = wgrad_defaults(geo(H, q == 0), wsbig, wssmall);
        w.dy = dc;
        if (q == 0) {
            w.x = obs; w.rows = rows;
            if ((rc = run_wgrad<16, 16, 1>(w, n, 1.0f / 255.0f, grads + L.cw[0], grads + L.cb[0], s, "impala/seq0_wgrad"))) return rc;
            break;                                            // no gradient for the observations
        }
        w.x = T(Q.s[q - 1][2]);
        ConvP d = conv_defaults(geo(H));
        d.in = dc; d.w = P + L.pd[k0]; d.epi = E_DGRAD; d.out = G == T(Q.ga) ? T(Q.gb) : T(Q.ga);
        if (q == 1) {
            if ((rc = run_wgrad<16, 32>(w, n, 1.f, grads + L.cw[k0], grads + L.cb[k0], s, "impala/seq1_wgrad"))) return rc;
            if ((rc = run_conv<32, 16>(d, n, s, "impala/seq1_dgrad"))) return rc;
        } else {
            if ((rc = run_wgrad<32, 32>(w, n, 1.f, grads + L.cw[k0], grads + L.cb[k0], s, "impala/seq2_wgrad"))) return rc;
            if ((rc = run_conv<32, 32>(d, n, s, "impala/seq2_dgrad"))) return rc;
        }
        Gn = G; G = d.out;
    }
    return B200RL_OK;
}
extern "C" int b200rl_impala_bf16_backward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                                           const void* packed, void* acts, const float* dhead, float* grads,
                                           void* workspace, size_t workspace_bytes, void* stream) {
    return impala_backward(obs, rows, n, A, 1, params, packed, acts, dhead, grads, workspace, workspace_bytes, stream);
}
extern "C" int b200rl_impala_ppg_bf16_backward(const uint8_t* obs, const int64_t* rows, int64_t n, int A, const float* params,
                                               const void* packed, void* acts, const float* dhead, float* grads,
                                               void* workspace, size_t workspace_bytes, void* stream) {
    return impala_backward(obs, rows, n, A, 2, params, packed, acts, dhead, grads, workspace, workspace_bytes, stream);
}
