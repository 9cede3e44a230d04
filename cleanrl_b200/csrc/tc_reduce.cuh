// Deterministic fold / column-sum kernels for the split weight-gradient reductions.
#pragma once
#include "tc_base.cuh"
#include "tc_wgrad_win.cuh"

namespace b200rl {
using namespace tc;

// out[idx] = sum_z part[z][idx], z < nslabs: block = 8 z-lanes x 32 consecutive outputs; every z-lane sums its
// slabs (z = lane, lane+8, ...) in ascending order, lane 0 then adds the 8 lane sums in order (deterministic).
__device__ __forceinline__ float zlane_sum(const float* __restrict__ part, int64_t slab, int nslabs, int64_t idx, bool valid,
                                           float* red /* [256] */) {
    const int zl = threadIdx.x >> 5, ol = threadIdx.x & 31;
    float s = 0.f;
    if (valid) {
        int z = zl;
        for (; z + 24 < nslabs; z += 32) {
            const float v0 = part[(int64_t)z * slab + idx], v1 = part[(int64_t)(z + 8) * slab + idx];
            const float v2 = part[(int64_t)(z + 16) * slab + idx], v3 = part[(int64_t)(z + 24) * slab + idx];
            s += v0; s += v1; s += v2; s += v3;
        }
        for (; z < nslabs; z += 8) s += part[(int64_t)z * slab + idx];
    }
    red[threadIdx.x] = s;
    __syncthreads();
    float t = 0.f;
    if (zl == 0) {
#pragma unroll
        for (int l = 0; l < 8; ++l) t += red[l * 32 + ol];
    }
    return t;                                           // meaningful for zl == 0
}

// fold for the window weight gradients: ws[S][nslots*64][64] -> torch layout dst[co][c][ky][kx].
//   layer 1: slot = tap (a,b); row channel q = c*16 + sy*4 + sx; ky = 4a+sy, kx = 4b+sx; 32 outputs, Cin 4, 8x8
//   layer 2: slot = (tap (a,b), cc); q = cc*64 + row = (py*2+px)*32 + c; ky = 2a+py, kx = 2b+px; Cin 32, 4x4
//   layer 3: slot -> tap (ky,kx) via slot_tap; q = c; Cin 64, 3x3
struct FoldWin { int layer, S, nslots, Cout; int slot_tap[16], slot_cc[16]; float scale;
                 float bscale;     // scale of the bias gradient (1, or 1 / kDact1Scale when dY was stored scaled)
                 const float* wsb; float* db; };
static __global__ void __launch_bounds__(256) tc_fold_win(const float* __restrict__ ws, const FoldWin f, float* __restrict__ dst) {
    __shared__ float red[256];
    const int idx = blockIdx.x * 32 + (threadIdx.x & 31);            // (slot*64 + row) * Cout + co
    const int KX = f.nslots * 64;
    if (idx >= KX * f.Cout) {                                        // trailing blocks fold the bias partials
        const int co = idx - KX * f.Cout;
        const bool valid = co < f.Cout && f.db != nullptr;
        const float s = zlane_sum(f.wsb, 64, f.S, co, valid, red);
        if (valid && threadIdx.x < 32) f.db[co] = s * f.bscale;
        return;
    }
    const int xi = idx / f.Cout, co = idx - xi * f.Cout;
    const int slot = xi >> 6, row = xi & 63;
    float s = zlane_sum(ws, (int64_t)KX * 64, f.S, (int64_t)xi * 64 + co, true, red);
    if (threadIdx.x >= 32) return;
    s *= f.scale;
    const int tap = f.slot_tap[slot];
    int64_t o;
    if (f.layer == 1) {
        const int c = row >> 4, sy = (row >> 2) & 3, sx = row & 3;
        o = (((int64_t)co * 4 + c) * 8 + ((tap >> 1) * 4 + sy)) * 8 + (tap & 1) * 4 + sx;
    } else if (f.layer == 2) {
        const int q = f.slot_cc[slot] * 64 + row;
        const int g = q >> 5, c = q & 31;
        o = (((int64_t)co * 32 + c) * 4 + (2 * (tap >> 1) + (g >> 1))) * 4 + 2 * (tap & 1) + (g & 1);
    } else {
        o = ((int64_t)co * 64 + row) * 9 + tap;
    }
    dst[o] = s;
}

// fold the fc weight-gradient partials ws[S][KX rows = o][NY cols = k], k = p*64 + c, into the REFERENCE's layout
// dst[o][c*49 + p] (torch flattens NCHW activations channel-major); partial slabs are added in ascending order.
static __global__ void tc_fold_fc(const float* __restrict__ ws, int S, int KX, int NY, int validX, int validY,
                           int C, int KK, float scale, float* __restrict__ dst) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)validX * validY;
    if (idx >= total) return;
    const int xi = (int)(idx / validY), yi = (int)(idx - (int64_t)xi * validY);
    float s = 0.f;
    const int64_t slab = (int64_t)KX * NY;
    for (int z = 0; z < S; ++z) s += ws[z * slab + (int64_t)xi * NY + yi];
    const int pp = yi / C, c = yi - pp * C;
    dst[(int64_t)xi * validY + (int64_t)c * KK + pp] = s * scale;
}

// column sums of a bf16 matrix [M, ld] (bias gradients): two-level deterministic reduction.
// Block = 256 threads = (256 / (ncols/8)) row lanes x (ncols/8) column groups; every thread streams
// 16-byte vectors (8 columns) down its rows, then the row lanes are folded through shared memory.
static __global__ void __launch_bounds__(256) tc_colsum_partial(const bf16* __restrict__ Y, int64_t M, int ld, int ncols,
                                                         int64_t rows_per_block, float* __restrict__ part) {
    __shared__ float red[256 * 8];
    const int cg = ncols >> 3;                 // column groups of 8
    const int lanes = 256 / cg;                // row lanes per block
    const int tx = threadIdx.x % cg, ty = threadIdx.x / cg;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    int64_t r1 = r0 + rows_per_block;
    if (r1 > M) r1 = M;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    if (ty < lanes) {
        for (int64_t r = r0 + ty; r < r1; r += lanes) {
            const int4 v = ldg16(Y + r * ld + tx * 8);
            const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                acc[2 * e] += __uint_as_float(w[e] << 16);
                acc[2 * e + 1] += __uint_as_float(w[e] & 0xFFFF0000u);
            }
        }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) red[threadIdx.x * 8 + e] = acc[e];
    __syncthreads();
    for (int c = threadIdx.x; c < ncols; c += blockDim.x) {
        const int g = c >> 3, e = c & 7;
        float s = 0.f;
        for (int l = 0; l < lanes; ++l) s += red[(l * cg + g) * 8 + e];
        part[(int64_t)blockIdx.x * ncols + c] = s;
    }
}
static __global__ void __launch_bounds__(256) tc_colsum_final(const float* __restrict__ part, int nblocks, int ncols,
                                                       float* __restrict__ db) {
    __shared__ float red[256];
    const int c = blockIdx.x * 32 + (threadIdx.x & 31);
    const float s = zlane_sum(part, ncols, nblocks, c, c < ncols, red);
    if (c < ncols && threadIdx.x < 32) db[c] = s;
}

// db = column sums of bf16 Y [M, ld] (first ncols columns), through per-block partials `part` (colsum_ws bytes)
static int64_t colsum_rows(int64_t M) {
    const int64_t rpb = ceil_div(M, 132 * 3);
    return rpb < 64 ? 64 : rpb;
}
static int colsum(const bf16* Y, int64_t M, int ld, int ncols, float* part, float* db, cudaStream_t s) {
    const int64_t rpb = colsum_rows(M);
    const int nb = (int)ceil_div(M, rpb);
    tc_colsum_partial<<<nb, 256, 0, s>>>(Y, M, ld, ncols, rpb, part);
    tc_colsum_final<<<(unsigned)ceil_div(ncols, 32), 256, 0, s>>>(part, nb, ncols, db);
    return check_launch("colsum", 2);
}
static size_t colsum_ws(int64_t M, int ncols) { return (size_t)ceil_div(M, colsum_rows(M)) * ncols * sizeof(float); }

}  // namespace b200rl
