// Wide heads (A1 = A + 1 > kMaxHeads outputs, e.g. C51's A * n_atoms logits): the GEMMs run on wgmma through
// tc_gemm_tma / tc_wgrad_tma; these are the small glue kernels around them.
#pragma once
#include "tc_base.cuh"

namespace b200rl {
using namespace tc;

constexpr int kMaxWideHeads = 2048;
constexpr int kWideHeadPad = 128;          // N granularity of the head GEMMs (2 x 64-column chunks of tc_wgrad_tma)

// Wh [A1][512] f32 -> whf [G][512] bf16 (forward B operand), whdg [512][G] bf16 (data-gradient B operand),
// bias [A1] f32 -> bpad [G] f32; rows / columns / entries >= A1 are zero.
__global__ void __launch_bounds__(256) tc_pack_head_wide(const float* __restrict__ Wh, const float* __restrict__ bh, int A1, int G,
                                                         bf16* __restrict__ whf, bf16* __restrict__ whdg, float* __restrict__ bpad) {
    const int64_t total = (int64_t)G * 512;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int g = (int)(i >> 9), h = (int)(i & 511);
        const bf16 w = __float2bfloat16_rn(g < A1 ? Wh[i] : 0.f);
        whf[i] = w;
        whdg[(int64_t)h * G + g] = w;
        if (h == 0) bpad[g] = g < A1 ? bh[g] : 0.f;
    }
}

// dhead f32 [n][A1] -> bf16 [n][G] (zero columns >= A1): the A operand of the dhid GEMM and the X operand of dWh
__global__ void __launch_bounds__(256) tc_head_dhead_bf16(const float* __restrict__ dhead, int64_t n, int A1, int G,
                                                          bf16* __restrict__ out) {
    const int64_t total = n * G;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / G;
        const int c = (int)(i - r * G);
        out[i] = __float2bfloat16_rn(c < A1 ? dhead[r * A1 + c] : 0.f);
    }
}

// dbh = column sums of dhead f32 [n][A1] in fp32: per row block (rows in order) -> part[nb][A1], then blocks in order
static inline int64_t wide_colsum_rows(int64_t n) {
    int64_t rpb = ceil_div(n, 256);
    return rpb < 64 ? 64 : rpb;
}
__global__ void __launch_bounds__(128) tc_colsum_f32_partial(const float* __restrict__ x, int64_t n, int cols, int64_t rpb,
                                                             float* __restrict__ part) {
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    const int64_t r0 = (int64_t)blockIdx.x * rpb;
    const int64_t r1 = r0 + rpb < n ? r0 + rpb : n;
    float s = 0.f;
    for (int64_t r = r0; r < r1; ++r) s += __ldg(x + r * cols + c);
    part[(int64_t)blockIdx.x * cols + c] = s;
}
__global__ void __launch_bounds__(128) tc_colsum_f32_final(const float* __restrict__ part, int nb, int cols, float* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float s = 0.f;
    for (int b = 0; b < nb; ++b) s += part[(int64_t)b * cols + c];
    out[c] = s;
}
static int colsum_f32(const float* x, int64_t n, int cols, float* part, float* out, cudaStream_t s) {
    const int64_t rpb = wide_colsum_rows(n);
    const int nb = (int)ceil_div(n, rpb);
    tc_colsum_f32_partial<<<dim3(nb, (unsigned)ceil_div(cols, 128)), 128, 0, s>>>(x, n, cols, rpb, part);
    tc_colsum_f32_final<<<(unsigned)ceil_div(cols, 128), 128, 0, s>>>(part, nb, cols, out);
    return check_launch("colsum_f32", 2);
}
static size_t colsum_f32_ws(int64_t n, int cols) { return (size_t)ceil_div(n, wide_colsum_rows(n)) * cols * sizeof(float); }

}  // namespace b200rl
