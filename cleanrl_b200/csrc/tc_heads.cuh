// Policy / value heads on CUDA cores (fp32 math).
#pragma once
#include "tc_base.cuh"
#include "tc_reduce.cuh"

namespace b200rl {
using namespace tc;

// ------------------------------------------------------------------ policy/value heads (tiny: CUDA cores, fp32 math)
// A1 = A + 1 head outputs (logits | value), 1 <= A1 <= kMaxHeads.  Head weights live in dynamic shared memory.
constexpr int kMaxHeads = 24;              // (A+1) * 2 KB of head weights must fit the 48 KB default dynamic shared memory
constexpr int kHeadsPartialBlocks = 264;     // 2 x 132 SMs: row blocks of the head weight gradient (x2 row lanes = partial slabs)
// rows per block of tc_heads_bwd_weight: its dhead rows are staged in (static-limit) shared memory, <= 256 x 32 floats
static inline int64_t heads_rows_per_block(int64_t n) {
    int64_t rpb = (n + kHeadsPartialBlocks - 1) / kHeadsPartialBlocks;
    if (rpb < 16) rpb = 16;
    if (rpb > 256) rpb = 256;
    return rpb;
}

// out[n][A1] = hidden[n][HT](bf16) . Wh[A1][HT]^T + bh (HT = 512: NatureCNN, 256: IMPALA-CNN, 128: the LSTM agent's
// recurrent state; H == HT).  One warp per row: lane l holds hidden units [256q + 8l, 256q + 8l + 8) (one 16-byte load
// per q; lanes past HT / 8 hold zeros), weights are read as float4 from shared memory.
template <int HT = 512>
__global__ void __launch_bounds__(256) tc_heads_fwd(const bf16* __restrict__ hid, const float* __restrict__ Wh,
                                                    const float* __restrict__ bh, int64_t n, int A1, int H,
                                                    float* __restrict__ out) {
    constexpr int NQ = (HT + 255) / 256;
    extern __shared__ float sW[];                       // [A1][HT]
    for (int i = threadIdx.x; i < A1 * HT; i += blockDim.x) sW[i] = Wh[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    for (int64_t row = (int64_t)blockIdx.x * wpb + (threadIdx.x >> 5); row < n; row += (int64_t)gridDim.x * wpb) {
        float hv[8 * NQ];
        const bf16* hp = hid + row * HT;
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
            const bool own = HT % 256 == 0 || lane * 8 < HT;
            const int4 v = own ? ldg16(hp + q * 256 + lane * 8) : make_int4(0, 0, 0, 0);
            const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                hv[q * 8 + 2 * e] = __uint_as_float(w[e] << 16);
                hv[q * 8 + 2 * e + 1] = __uint_as_float(w[e] & 0xFFFF0000u);
            }
        }
        float mine = 0.f;                               // lane a keeps output a
        for (int a = 0; a < A1; ++a) {
            float s = 0.f;
#pragma unroll
            for (int q = 0; q < NQ; ++q) {
                if (HT % 256 != 0 && lane * 8 >= HT) continue;
                const float4 w0 = *reinterpret_cast<const float4*>(sW + a * HT + q * 256 + lane * 8);
                const float4 w1 = *reinterpret_cast<const float4*>(sW + a * HT + q * 256 + lane * 8 + 4);
                s = fmaf(hv[q * 8 + 0], w0.x, s); s = fmaf(hv[q * 8 + 1], w0.y, s);
                s = fmaf(hv[q * 8 + 2], w0.z, s); s = fmaf(hv[q * 8 + 3], w0.w, s);
                s = fmaf(hv[q * 8 + 4], w1.x, s); s = fmaf(hv[q * 8 + 5], w1.y, s);
                s = fmaf(hv[q * 8 + 6], w1.z, s); s = fmaf(hv[q * 8 + 7], w1.w, s);
            }
            s = warp_sum(s);
            if (lane == a) mine = s + bh[a];
        }
        if (lane < A1) out[row * A1 + lane] = mine;     // one coalesced store per row
    }
}
// dhid_pre[n][HT] (bf16) = (dhead[n][A1] . Wh[A1][HT]) * (hid > 0), leaving head `skip_col` out of the product (-1 = none:
// a head that reads a detached copy of the hidden layer).  Thread = 8 consecutive hidden units of one
// row (one mask byte in, one 16-byte store out).  Weights are staged transposed, sWt[a][e][group], so the 32 lanes
// of a warp (consecutive groups) hit 32 different banks.
template <int HT = 512>
__global__ void __launch_bounds__(256) tc_heads_bwd_data(const float* __restrict__ dhead, const float* __restrict__ Wh,
                                                         const uint8_t* __restrict__ hid_bits, int64_t n, int A1, int H,
                                                         int skip_col, bf16* __restrict__ dhid) {
    constexpr int G = HT / 8;                           // groups of 8 per row
    extern __shared__ float sWt[];                      // [A1][8][G]
    for (int i = threadIdx.x; i < A1 * HT; i += blockDim.x) {
        const int a = i / HT, h = i % HT;
        sWt[a * HT + (h & 7) * G + (h >> 3)] = Wh[i];
    }
    __syncthreads();
    const int64_t total = n * G;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = idx / G;
        const int g = (int)(idx % G);
        const uint32_t m = hid_bits[idx];               // bit e: hid[row][8g + e] > 0
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = 0.f;
        for (int a = 0; a < A1; ++a) {
            if (a == skip_col) continue;
            const float d = __ldg(dhead + row * A1 + a);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = fmaf(d, sWt[a * HT + e * G + g], o[e]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) if (!((m >> e) & 1u)) o[e] = 0.f;
        int4 w;
        w.x = (int)pack_bf16x2(o[0], o[1]); w.y = (int)pack_bf16x2(o[2], o[3]);
        w.z = (int)pack_bf16x2(o[4], o[5]); w.w = (int)pack_bf16x2(o[6], o[7]);
        *reinterpret_cast<int4*>(dhid + row * HT + g * 8) = w;
    }
}
// dWh[a][h] = sum_m dhead[m][a] * hid[m][h]; dbh[a] = sum_m dhead[m][a]  (partial slabs per (row block, row lane),
// folded by tc_heads_fold).  Block = HT threads = 2 row lanes x HT/2 hidden pairs; the block's dhead rows are staged
// in shared memory once, 8 rows of hidden values are in flight per thread.
template <int MAXA, int HT = 512>
__global__ void __launch_bounds__(512) tc_heads_bwd_weight(const float* __restrict__ dhead, const bf16* __restrict__ hid,
                                                           int64_t n, int A1, int H, int64_t rows_per_block,
                                                           float* __restrict__ part) {
    extern __shared__ float sD[];                       // [rows_per_block][A1]
    const int hp = threadIdx.x % (HT / 2), rl = threadIdx.x / (HT / 2);
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    int64_t r1 = r0 + rows_per_block;
    if (r1 > n) r1 = n;
    const int nrows = (int)(r1 > r0 ? r1 - r0 : 0);
    for (int i = threadIdx.x; i < nrows * A1; i += blockDim.x) sD[i] = dhead[r0 * A1 + i];
    __syncthreads();
    float acc0[MAXA], acc1[MAXA], bacc[MAXA];
#pragma unroll
    for (int a = 0; a < MAXA; ++a) { acc0[a] = 0.f; acc1[a] = 0.f; bacc[a] = 0.f; }
    const uint32_t* h2 = reinterpret_cast<const uint32_t*>(hid);      // bf16 pairs
    int r = rl;
    for (; r + 14 < nrows; r += 16) {                   // 8 rows (stride 2) in flight
        uint32_t hv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) hv[u] = __ldg(h2 + (r0 + r + 2 * u) * (HT / 2) + hp);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const float x0 = __uint_as_float(hv[u] << 16), x1 = __uint_as_float(hv[u] & 0xFFFF0000u);
            const float* dr = sD + (r + 2 * u) * A1;
#pragma unroll
            for (int a = 0; a < MAXA; ++a) {
                if (a < A1) {
                    const float d = dr[a];
                    acc0[a] = fmaf(d, x0, acc0[a]); acc1[a] = fmaf(d, x1, acc1[a]); bacc[a] += d;
                }
            }
        }
    }
    for (; r < nrows; r += 2) {
        const uint32_t hv = __ldg(h2 + (r0 + r) * (HT / 2) + hp);
        const float x0 = __uint_as_float(hv << 16), x1 = __uint_as_float(hv & 0xFFFF0000u);
        const float* dr = sD + r * A1;
#pragma unroll
        for (int a = 0; a < MAXA; ++a) {
            if (a < A1) {
                const float d = dr[a];
                acc0[a] = fmaf(d, x0, acc0[a]); acc1[a] = fmaf(d, x1, acc1[a]); bacc[a] += d;
            }
        }
    }
    float* pb = part + ((int64_t)blockIdx.x * 2 + rl) * A1 * (H + 2);      // slab rows: H weights, bias, pad
#pragma unroll
    for (int a = 0; a < MAXA; ++a) {
        if (a < A1) {
            *reinterpret_cast<float2*>(pb + (int64_t)a * (H + 2) + 2 * hp) = make_float2(acc0[a], acc1[a]);
            if (hp == 0) pb[(int64_t)a * (H + 2) + H] = bacc[a];
        }
    }
}
static __global__ void __launch_bounds__(256) tc_heads_fold(const float* __restrict__ part, int nslabs, int A1, int H,
                                                     float* __restrict__ dW, float* __restrict__ db) {
    __shared__ float red[256];
    const int idx = blockIdx.x * 32 + (threadIdx.x & 31);
    const int a = idx / (H + 2), h = idx - a * (H + 2);
    const bool valid = a < A1 && h <= H;                // h == H: bias; h == H + 1: padding
    const float s = zlane_sum(part, (int64_t)A1 * (H + 2), nslabs, idx, valid, red);
    if (!valid || threadIdx.x >= 32) return;
    if (h == H) db[a] = s; else dW[(int64_t)a * H + h] = s;
}

// ---- launchers over H hidden units (128: the LSTM agent, 256: IMPALA-CNN, 512: NatureCNN); Wh, bh, dW, db fp32 [A1][H]
template <int H>
static int heads_fwd(const bf16* hid, const float* Wh, const float* bh, int64_t n, int A1, float* out, cudaStream_t s,
                     const char* what) {
    static_assert(H == 128 || H == 256 || H == 512, "head input width");
    const int grid = (int)(ceil_div(n, 8) < (int64_t)num_sms() * 8 ? ceil_div(n, 8) : (int64_t)num_sms() * 8);
    tc_heads_fwd<H><<<grid, 256, (size_t)A1 * H * sizeof(float), s>>>(hid, Wh, bh, n, A1, H, out);
    return check_launch(what);
}
// scratch of heads_bwd_weight: 2 partial slabs of A1 x (H + 2) floats per row block
static size_t heads_partial_bytes(int64_t n, int A1, int H) {
    return (size_t)2 * ceil_div(n, heads_rows_per_block(n)) * A1 * (H + 2) * sizeof(float);
}
// dW = dhead^T . hid, db = column sums of dhead, through the partial slabs `part` (heads_partial_bytes)
template <int H>
static int heads_bwd_weight(const float* dhead, const bf16* hid, int64_t n, int A1, float* part, float* dW, float* db,
                            cudaStream_t s, const char* what) {
    static_assert(H == 128 || H == 256 || H == 512, "head input width");
    const int64_t rpb = heads_rows_per_block(n);
    const int nb = (int)ceil_div(n, rpb);
    const size_t sd = (size_t)rpb * A1 * sizeof(float);
    if (A1 <= 8) tc_heads_bwd_weight<8, H><<<nb, H, sd, s>>>(dhead, hid, n, A1, H, rpb, part);
    else tc_heads_bwd_weight<kMaxHeads, H><<<nb, H, sd, s>>>(dhead, hid, n, A1, H, rpb, part);
    tc_heads_fold<<<(unsigned)ceil_div(A1 * (H + 2), 32), 256, 0, s>>>(part, 2 * nb, A1, H, dW, db);
    return check_launch(what, 2);
}
// dhid = (dhead . Wh) * (hid > 0) without head `skip_col` (-1 = all heads), hid_bits = one mask byte per 8 hidden units
template <int H>
static int heads_bwd_data(const float* dhead, const float* Wh, const uint8_t* hid_bits, int64_t n, int A1, bf16* dhid,
                          cudaStream_t s, const char* what, int skip_col = -1) {
    static_assert(H == 128 || H == 256 || H == 512, "head input width");
    const int grid = (int)(ceil_div(n * H, 2048) < (int64_t)num_sms() * 8 ? ceil_div(n * H, 2048) : (int64_t)num_sms() * 8);
    tc_heads_bwd_data<H><<<grid, 256, (size_t)A1 * H * sizeof(float), s>>>(dhead, Wh, hid_bits, n, A1, H, skip_col, dhid);
    return check_launch(what);
}

}  // namespace b200rl
