// Parallel Q-learning (cleanrl/pqn.py): fp32 kernels for the reference's LayerNorm Q-network and its Q(lambda) targets.
//
//   QNetwork  obs (d) -> Linear 120 -> LayerNorm -> ReLU -> Linear 84 -> LayerNorm -> ReLU -> Linear A
//
// Flat parameter layout: nn.Module order (network.0.weight [120, d], network.0.bias, network.1.weight / .bias = LN1
// gamma / beta, network.3.*, network.4.* = LN2, network.6.weight [A, 84], network.6.bias).
//
// The network has ~11 k parameters at CartPole shapes, so an update is bound by its chain of dependent launches, not by
// arithmetic: the kernels keep the reference's fp32 on the CUDA cores and make the chain short.  Every forward /
// data-backward CTA owns kPqnRows rows and the whole hidden width (thread j = hidden unit j), with the input and every
// activation in shared memory; LayerNorm row means and variances are warp reductions in a fixed lane order.  Dot
// products run sequentially over their inner index, weight gradients sequentially over rows, the minibatch means go
// through per-block partials folded by the last block in block order (no float atomics): every result is bitwise
// repeatable.  Q(lambda) is one thread per env with every operation separately rounded (the reference loop's bits).
#include "common.cuh"

namespace b200rl {

constexpr int kP1 = 120;           // hidden widths (the reference's constants)
constexpr int kP2 = 84;
constexpr int kPqnThreads = 128;
constexpr int kPqnRows = 8;        // rows per forward / data-backward CTA
constexpr int kPqnMaxIn = 512;
constexpr int kPqnMaxA = 64;
constexpr int kPqnWgThreads = 256;
constexpr int kPqnWT = 32;
constexpr float kLnEps = 1e-5f;    // nn.LayerNorm's default

struct PqnOff {
    int64_t w1, b1, g1, be1, w2, b2, g2, be2, w3, b3, total;
    __host__ __device__ PqnOff(int d, int A) {
        w1 = 0; b1 = w1 + (int64_t)kP1 * d; g1 = b1 + kP1; be1 = g1 + kP1; w2 = be1 + kP1; b2 = w2 + kP2 * kP1;
        g2 = b2 + kP2; be2 = g2 + kP2; w3 = be2 + kP2; b3 = w3 + (int64_t)A * kP2; total = b3 + A;
    }
};

constexpr int kPqnMaxTiles = 100;     // weight-gradient tiles at obs_dim 512, A 64
constexpr int kPqnSplitRows = 512;    // rows per weight-gradient CTA of a split tile
constexpr int kPqnMaxSplits = 64;

// Row splits of the weight gradient at M rows: one CTA per tile up to 512 rows, then up to 64 per tile.
__host__ __device__ inline int pqn_splits(int64_t M) {
    const int64_t s = (M + kPqnSplitRows - 1) / kPqnSplitRows;
    return (int)(s < 1 ? 1 : (s > kPqnMaxSplits ? kPqnMaxSplits : s));
}

// The update workspace: [loss ticket | weight-gradient tile tickets] (a fixed 512-byte head, zero at rest), the loss
// partials (2 floats per loss block), the kept activations and gradients of M rows that the weight gradient reads, and
// the weight gradient's per-split tile partials.  One layout for loss_bwd and wgrad.
struct PqnWs {
    unsigned int* ticket; unsigned int* tile_tickets; float* partials;
    float *h1, *dz1, *dy1, *gx1;       // [M, 120] each: post-ReLU h1, d z1, d LN1-output (post mask), d * xhat1
    float *h2, *dz2, *dy2, *gx2;       // [M, 84] each
    float* dq;                         // [M]
    float* tile_partials;              // [kPqnMaxTiles][splits][32 x 32] when splits > 1
    static constexpr size_t kHead = 512;
    __host__ __device__ static int64_t pad4(int64_t n) { return (n + 3) & ~(int64_t)3; }
    __host__ __device__ PqnWs(void* ws, int64_t M) {
        char* c = reinterpret_cast<char*>(ws);
        ticket = reinterpret_cast<unsigned int*>(c);
        tile_tickets = ticket + 4;
        partials = reinterpret_cast<float*>(c + kHead);
        float* f = partials + pad4(2 * ((M + kPqnRows - 1) / kPqnRows));
        h1 = f; f += M * kP1; dz1 = f; f += M * kP1; dy1 = f; f += M * kP1; gx1 = f; f += M * kP1;
        h2 = f; f += M * kP2; dz2 = f; f += M * kP2; dy2 = f; f += M * kP2; gx2 = f; f += M * kP2;
        dq = f; f += pad4(M);
        tile_partials = f;
    }
    static size_t bytes(int64_t M) {
        const int S = pqn_splits(M);
        return kHead + 4 * (size_t)(pad4(2 * ((M + kPqnRows - 1) / kPqnRows)) + M * (4 * kP1 + 4 * kP2) + pad4(M) +
                                    (S > 1 ? (int64_t)kPqnMaxTiles * S * kPqnWT * kPqnWT : 0));
    }
};

struct PqnSmem {
    float x[kPqnRows][kPqnMaxIn];  // the input rows; in the backward d h2, dz2, d h1 and dz1
    float z1[kPqnRows][kP1];       // pre-LN, then xhat1
    float h1[kPqnRows][kP1];       // post-ReLU
    float z2[kPqnRows][kP2];
    float h2[kPqnRows][kP2];
    float q[kPqnRows][kPqnMaxA];
    float mean[kPqnRows], rstd1[kPqnRows], rstd2[kPqnRows], m1[kPqnRows], m2[kPqnRows];
    float dq[kPqnRows];
    int act[kPqnRows];
};

// torch.relu: NaN stays NaN.
__device__ __forceinline__ float relu_nan(float y) { return y < 0.f ? 0.f : y; }

// z[r][j] = b[j] + sum_k in[r][k] W[j][k] for thread j < N (sequential over k).
template <int N, int LD>
__device__ __forceinline__ void pqn_dense(const float* __restrict__ W, const float* __restrict__ b, const float (*in)[LD],
                                          int K, float (*z)[N]) {
    const int j = threadIdx.x;
    if (j >= N) return;
    float acc[kPqnRows];
#pragma unroll
    for (int r = 0; r < kPqnRows; ++r) acc[r] = 0.f;
    const float* w = W + (int64_t)j * K;
    for (int k = 0; k < K; ++k) {
        const float wk = __ldg(w + k);
#pragma unroll
        for (int r = 0; r < kPqnRows; ++r) acc[r] = fmaf(wk, in[r][k], acc[r]);
    }
    const float bj = __ldg(b + j);
#pragma unroll
    for (int r = 0; r < kPqnRows; ++r) z[r][j] = __fadd_rn(acc[r], bj);
}

// Row means of a[r][:] and (optionally) of a[r][:] * b[r][:] over H columns: warp w takes rows w, w + 4, lanes stride
// the columns, then a fixed xor tree.
template <int H>
__device__ __forceinline__ void pqn_row_means(const float (*a)[H], const float (*b)[H], float* ma, float* mab) {
    const int lane = threadIdx.x & 31;
    for (int r = threadIdx.x >> 5; r < kPqnRows; r += kPqnThreads / 32) {
        float s = 0.f, t = 0.f;
        for (int j = lane; j < H; j += 32) {
            s = __fadd_rn(s, a[r][j]);
            if (b) t = fmaf(a[r][j], b[r][j], t);
        }
        s = warp_sum(s);
        if (b) t = warp_sum(t);
        if (lane == 0) {
            ma[r] = __fdiv_rn(s, (float)H);
            if (b) mab[r] = __fdiv_rn(t, (float)H);
        }
    }
}

// LayerNorm + ReLU in place over z[r][:] (H wide): z becomes xhat = (z - mean) * rstd, h = relu(xhat * gamma + beta).
template <int H>
__device__ __forceinline__ void pqn_ln_relu(float (*z)[H], float (*h)[H], const float* __restrict__ gamma,
                                            const float* __restrict__ beta, float* mean, float* rstd) {
    pqn_row_means<H>(z, nullptr, mean, nullptr);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int r = threadIdx.x >> 5; r < kPqnRows; r += kPqnThreads / 32) {       // biased variance, two-pass
        float v = 0.f;
        for (int j = lane; j < H; j += 32) {
            const float d = __fsub_rn(z[r][j], mean[r]);
            v = fmaf(d, d, v);
        }
        v = warp_sum(v);
        if (lane == 0) rstd[r] = __frcp_rn(__fsqrt_rn(__fadd_rn(__fdiv_rn(v, (float)H), kLnEps)));
    }
    __syncthreads();
    const int j = threadIdx.x;
    if (j < H) {
        const float g = __ldg(gamma + j), be = __ldg(beta + j);
#pragma unroll
        for (int r = 0; r < kPqnRows; ++r) {
            const float xh = __fmul_rn(__fsub_rn(z[r][j], mean[r]), rstd[r]);
            z[r][j] = xh;
            h[r][j] = relu_nan(__fadd_rn(__fmul_rn(xh, g), be));
        }
    }
    __syncthreads();
}

// The forward of the CTA's rows obs[rows[r0 + r]] (rows NULL: r0 + r) to Q in s.q; rows past n are zeros.
__device__ __forceinline__ void pqn_forward_rows(PqnSmem& s, const float* __restrict__ p, const PqnOff& o,
                                                 const float* __restrict__ obs, int64_t ld_obs,
                                                 const int64_t* __restrict__ rows, int64_t n, int d, int A, int64_t r0) {
    for (int i = threadIdx.x; i < kPqnRows * d; i += kPqnThreads) {
        const int r = i / d, k = i - r * d;
        const int64_t b = r0 + r;
        s.x[r][k] = b < n ? obs[(rows ? rows[b] : b) * ld_obs + k] : 0.f;
    }
    __syncthreads();
    pqn_dense<kP1, kPqnMaxIn>(p + o.w1, p + o.b1, s.x, d, s.z1);
    __syncthreads();
    pqn_ln_relu<kP1>(s.z1, s.h1, p + o.g1, p + o.be1, s.mean, s.rstd1);
    pqn_dense<kP2, kP1>(p + o.w2, p + o.b2, s.h1, kP1, s.z2);
    __syncthreads();
    pqn_ln_relu<kP2>(s.z2, s.h2, p + o.g2, p + o.be2, s.mean, s.rstd2);
    for (int i = threadIdx.x; i < kPqnRows * A; i += kPqnThreads) {
        const int r = i / A, c = i - r * A;
        const float* w = p + o.w3 + (int64_t)c * kP2;
        float acc = 0.f;
        for (int k = 0; k < kP2; ++k) acc = fmaf(__ldg(w + k), s.h2[r][k], acc);
        s.q[r][c] = __fadd_rn(acc, __ldg(p + o.b3 + c));
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------ forward / rollout step
struct PqnActParams {
    const float* params; const float* obs; int64_t ld_obs; int64_t n; int d, A;
    const int64_t* rand_act; const float* u; float eps;
    float* obs_slot; int64_t* act_slot; float* val_slot; float* q_out;
    const float* copy_in; float* copy_out; int64_t copy_n;
};

__global__ void __launch_bounds__(kPqnThreads) pqn_act_kernel(const PqnActParams P) {
    __shared__ PqnSmem s;
    const int64_t r0 = (int64_t)blockIdx.x * kPqnRows;
    const PqnOff o(P.d, P.A);
    pqn_forward_rows(s, P.params, o, P.obs, P.ld_obs, nullptr, P.n, P.d, P.A, r0);
    if (P.obs_slot)
        for (int i = threadIdx.x; i < kPqnRows * P.d; i += kPqnThreads) {
            const int r = i / P.d, k = i - r * P.d;
            if (r0 + r < P.n) P.obs_slot[(r0 + r) * P.d + k] = s.x[r][k];
        }
    if (P.q_out)
        for (int i = threadIdx.x; i < kPqnRows * P.A; i += kPqnThreads) {
            const int r = i / P.A, c = i - r * P.A;
            if (r0 + r < P.n) P.q_out[(r0 + r) * P.A + c] = s.q[r][c];
        }
    if (P.copy_in)
        for (int64_t i = (int64_t)blockIdx.x * kPqnThreads + threadIdx.x; i < P.copy_n; i += (int64_t)gridDim.x * kPqnThreads)
            P.copy_out[i] = P.copy_in[i];
    if (threadIdx.x >= kPqnRows || r0 + threadIdx.x >= P.n) return;
    const int r = threadIdx.x;
    const int64_t b = r0 + r;
    // torch.argmax: the first maximum, a NaN counts as the maximum (the first NaN wins)
    int best = 0;
    float bv = s.q[r][0];
    for (int c = 1; c < P.A; ++c) {
        const float v = s.q[r][c];
        if (bv != bv) break;
        if (v != v || v > bv) { best = c; bv = v; }
    }
    if (P.val_slot) P.val_slot[b] = bv;
    if (P.act_slot) {
        int64_t a = best;
        if (P.rand_act && P.u[b] < P.eps) a = P.rand_act[b];       // torch.where(rand < epsilon, random, greedy)
        P.act_slot[b] = a;
    }
}

// ------------------------------------------------------------------------------- minibatch loss + data backward
struct PqnLossParams {
    const float* params; const float* obs; int64_t ld_obs; const int64_t* rows; const int64_t* actions;
    const float* returns; int64_t M; int d, A; float two_over_m;
    float* stats; void* ws;
};

// LayerNorm + ReLU backward of the CTA's rows, H wide: dh (d post-ReLU output) in dh[r][j] -> dz[r][j]; keeps dy
// (post-mask) and dy * xhat per row for the gamma / beta gradients.  dz = rstd (dxhat - mean(dxhat) - xhat
// mean(dxhat xhat)), dxhat = dy gamma.
template <int H>
__device__ __forceinline__ void pqn_ln_relu_bwd(PqnSmem& s, float (*dh)[H], const float (*xh)[H], const float (*h)[H],
                                                const float* __restrict__ gamma, const float* rstd, float* keep_dy,
                                                float* keep_gx, float* keep_dz, float (*dz)[H], int64_t M, int64_t r0) {
    const int j = threadIdx.x;
    if (j < H) {
        const float g = __ldg(gamma + j);
#pragma unroll
        for (int r = 0; r < kPqnRows; ++r) {
            const int64_t b = r0 + r;
            const float dy = h[r][j] > 0.f ? dh[r][j] : 0.f;
            const float gx = __fmul_rn(dy, xh[r][j]);
            if (b < M) { keep_dy[b * H + j] = dy; keep_gx[b * H + j] = gx; }
            dh[r][j] = __fmul_rn(dy, g);
        }
    }
    __syncthreads();
    pqn_row_means<H>(dh, xh, s.m1, s.m2);
    __syncthreads();
    if (j < H) {
#pragma unroll
        for (int r = 0; r < kPqnRows; ++r) {
            const int64_t b = r0 + r;
            const float v = __fmul_rn(rstd[r], __fsub_rn(__fsub_rn(dh[r][j], s.m1[r]), __fmul_rn(xh[r][j], s.m2[r])));
            dz[r][j] = v;
            if (b < M) keep_dz[b * H + j] = v;
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kPqnThreads) pqn_loss_bwd_kernel(const PqnLossParams P) {
    __shared__ PqnSmem s;
    __shared__ float red[32];
    __shared__ bool is_last;
    const int64_t r0 = (int64_t)blockIdx.x * kPqnRows;
    const PqnOff o(P.d, P.A);
    const float* p = P.params;
    PqnWs W(P.ws, P.M);
    pqn_forward_rows(s, p, o, P.obs, P.ld_obs, P.rows, P.M, P.d, P.A, r0);
    float v[2] = {0.f, 0.f};
    if (threadIdx.x < kPqnRows) {
        const int r = threadIdx.x;
        const int64_t b = r0 + r;
        float dq = 0.f;
        int a = 0;
        if (b < P.M) {
            const int64_t row = P.rows ? P.rows[b] : b;
            const int64_t ai = P.actions[row];
            a = ai < 0 ? 0 : (ai >= P.A ? P.A - 1 : (int)ai);
            const float q = s.q[r][a];
            const float e = __fsub_rn(P.returns[row], q);            // F.mse_loss(b_returns[mb], Q[a])
            v[0] = __fmul_rn(e, e);
            v[1] = q;
            dq = -__fmul_rn(P.two_over_m, e);                        // its backward for the target argument
            W.dq[b] = dq;
        }
        s.dq[r] = dq;
        s.act[r] = a;
    }
    // keep h1 / h2 for the weight gradient; s.x is free now and holds d h2, dz2, d h1 and dz1
    const int j = threadIdx.x;
    for (int r = 0; r < kPqnRows && r0 + r < P.M; ++r) {
        if (j < kP1) W.h1[(r0 + r) * kP1 + j] = s.h1[r][j];
        if (j < kP2) W.h2[(r0 + r) * kP2 + j] = s.h2[r][j];
    }
    float (*dh2)[kP2] = reinterpret_cast<float (*)[kP2]>(&s.x[0][0]);
    float (*dz2)[kP2] = dh2 + kPqnRows;
    float (*dh1)[kP1] = reinterpret_cast<float (*)[kP1]>(&s.x[0][0] + 2 * kPqnRows * kP2);
    float (*dz1)[kP1] = dh1 + kPqnRows;
    __syncthreads();
    if (j < kP2)                                                     // d h2 = dq W3[a]
        for (int r = 0; r < kPqnRows; ++r) dh2[r][j] = __fmul_rn(s.dq[r], __ldg(p + o.w3 + (int64_t)s.act[r] * kP2 + j));
    __syncthreads();
    pqn_ln_relu_bwd<kP2>(s, dh2, s.z2, s.h2, p + o.g2, s.rstd2, W.dy2, W.gx2, W.dz2, dz2, P.M, r0);
    if (j < kP1) {                                                   // d h1 = W2^T dz2, sequential over the 84 outputs
        float acc[kPqnRows];
#pragma unroll
        for (int r = 0; r < kPqnRows; ++r) acc[r] = 0.f;
        for (int k = 0; k < kP2; ++k) {
            const float w = __ldg(p + o.w2 + (int64_t)k * kP1 + j);
#pragma unroll
            for (int r = 0; r < kPqnRows; ++r) acc[r] = fmaf(w, dz2[r][k], acc[r]);
        }
#pragma unroll
        for (int r = 0; r < kPqnRows; ++r) dh1[r][j] = acc[r];
    }
    __syncthreads();
    pqn_ln_relu_bwd<kP1>(s, dh1, s.z1, s.h1, p + o.g1, s.rstd1, W.dy1, W.gx1, W.dz1, dz1, P.M, r0);
    // stats: td_loss and mean(q), folded in block order
    for (int k = 0; k < 2; ++k) v[k] = block_sum(v[k], red);
    if (threadIdx.x == 0) {
        W.partials[2 * blockIdx.x] = v[0];
        W.partials[2 * blockIdx.x + 1] = v[1];
        __threadfence();
        is_last = (atomicAdd(W.ticket, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last || threadIdx.x != 0) return;
    __threadfence();
    float a0 = 0.f, a1 = 0.f;
    for (unsigned bk = 0; bk < gridDim.x; ++bk) {
        a0 = __fadd_rn(a0, __ldcg(W.partials + 2 * bk));
        a1 = __fadd_rn(a1, __ldcg(W.partials + 2 * bk + 1));
    }
    *W.ticket = 0;
    const float m = (float)P.M;
    P.stats[0] = __fdiv_rn(a0, m);                                   // losses/td_loss
    P.stats[1] = __fdiv_rn(a1, m);                                   // losses/q_values
}

// ------------------------------------------------------------------------------------------- weight gradients
// Seven jobs: dW[n][k] = sum_b dz[b][n] x[b][k] and db[n] = sum_b dz[b][n] (the bias is the column k = K with x = 1).
// K = 0 jobs are column sums (LayerNorm gamma from dy * xhat, beta from dy).  x may be gathered through rows (the
// minibatch's obs); dz NULL is the head's one-hot gradient, dz[b][n] = (a_b == n) dq[b].  A CTA owns a 32 x 32 tile of
// [dW | db] and one of gridDim.y row splits, walked in chunks of 32 rows in row order; with more than one split each CTA
// stores its partial tile and the last CTA of the tile to arrive adds the partials in split order (no float atomics:
// the result is bitwise repeatable).
constexpr int kPqnJobs = 7;
struct PqnWgradJob {
    const float* dz; int ld_dz; const float* x; int64_t ld_x; const int64_t* x_rows; int N, K; float* dw; float* db;
    int tiles_k, tile0;
};
struct PqnWgradParams {
    PqnWgradJob job[kPqnJobs]; int njobs; int64_t M, rows_per_split; const int64_t* rows; const int64_t* actions;
    const float* dq; int A; float* tile_partials; unsigned int* tile_tickets;
};

__global__ void __launch_bounds__(kPqnWgThreads) pqn_wgrad_kernel(const PqnWgradParams P) {
    __shared__ float zs[kPqnWT][kPqnWT + 1];
    __shared__ float xs[kPqnWT][kPqnWT + 1];
    __shared__ int as[kPqnWT];
    __shared__ bool is_last;
    int jb = 0;
    while (jb + 1 < P.njobs && (int)blockIdx.x >= P.job[jb + 1].tile0) ++jb;
    const PqnWgradJob& J = P.job[jb];
    const int tile = blockIdx.x - J.tile0;
    const int n0 = (tile / J.tiles_k) * kPqnWT, k0 = (tile % J.tiles_k) * kPqnWT;
    const int tn = threadIdx.x >> 3, tk = (threadIdx.x & 7) * 4;
    const int64_t lo = (int64_t)blockIdx.y * P.rows_per_split;
    const int64_t hi = lo + P.rows_per_split < P.M ? lo + P.rows_per_split : P.M;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int64_t b0 = lo; b0 < hi; b0 += kPqnWT) {
        if (!J.dz && threadIdx.x < kPqnWT) {
            const int64_t b = b0 + threadIdx.x;
            as[threadIdx.x] = b < hi ? (int)P.actions[P.rows ? P.rows[b] : b] : -1;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < kPqnWT * kPqnWT; i += kPqnWgThreads) {
            const int r = i / kPqnWT, c = i - r * kPqnWT;
            const int64_t b = b0 + r;
            const bool ok = b < hi;
            float z = 0.f;
            if (ok && n0 + c < J.N) z = J.dz ? J.dz[b * J.ld_dz + n0 + c] : (as[r] == n0 + c ? P.dq[b] : 0.f);
            zs[r][c] = z;
            const int k = k0 + c;
            xs[r][c] = !ok || k > J.K ? 0.f : (k == J.K ? 1.f : J.x[(J.x_rows ? J.x_rows[b] : b) * J.ld_x + k]);
        }
        __syncthreads();
        const int rn = (int)(hi - b0 < kPqnWT ? hi - b0 : kPqnWT);
        for (int r = 0; r < rn; ++r) {
            const float z = zs[r][tn];
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[c] = fmaf(z, xs[r][tk + c], acc[c]);
        }
        __syncthreads();
    }
    const int S = gridDim.y;
    if (S > 1) {
        float* part = P.tile_partials + (int64_t)blockIdx.x * S * kPqnWT * kPqnWT;
#pragma unroll
        for (int c = 0; c < 4; ++c) part[(int64_t)blockIdx.y * kPqnWT * kPqnWT + tn * kPqnWT + tk + c] = acc[c];
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) is_last = atomicAdd(P.tile_tickets + blockIdx.x, 1u) == (unsigned)S - 1;
        __syncthreads();
        if (!is_last) return;
        __threadfence();
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float sum = 0.f;
            for (int sp = 0; sp < S; ++sp) sum = __fadd_rn(sum, __ldcg(part + (int64_t)sp * kPqnWT * kPqnWT + tn * kPqnWT + tk + c));
            acc[c] = sum;
        }
        if (threadIdx.x == 0) P.tile_tickets[blockIdx.x] = 0;
    }
    const int n = n0 + tn;
    if (n >= J.N) return;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int k = k0 + tk + c;
        if (k < J.K) J.dw[(int64_t)n * J.K + k] = acc[c];
        else if (k == J.K) J.db[n] = acc[c];
    }
}

// ------------------------------------------------------------------------------------------------- Q(lambda)
__global__ void qlambda_kernel(const float* __restrict__ rewards, const float* __restrict__ values,
                               const float* __restrict__ dones, const float* __restrict__ next_value,
                               const float* __restrict__ next_done, float* __restrict__ returns, int64_t T, int64_t N,
                               float gamma, float ql, float one_minus_ql) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    // returns[T-1] = r + ((gamma * next_value) * (1 - next_done))
    int64_t i = (T - 1) * N + n;
    float R = __fadd_rn(rewards[i], __fmul_rn(__fmul_rn(gamma, next_value[n]), __fsub_rn(1.f, next_done[n])));
    returns[i] = R;
    for (int64_t t = T - 2; t >= 0; --t) {
        const int64_t nx = i;
        i -= N;
        // r + ((gamma * ((ql * R') + ((1 - ql) * v'))) * (1 - d'))
        const float inner = __fadd_rn(__fmul_rn(ql, R), __fmul_rn(one_minus_ql, values[nx]));
        R = __fadd_rn(rewards[i], __fmul_rn(__fmul_rn(gamma, inner), __fsub_rn(1.f, dones[nx])));
        returns[i] = R;
    }
}

}  // namespace b200rl

#define PQN_SHAPES(what)                                                                                               \
    B200RL_REQUIRE(obs_dim >= 1 && obs_dim <= b200rl::kPqnMaxIn, what ": obs_dim=%d outside [1, %d]", obs_dim,         \
                   b200rl::kPqnMaxIn);                                                                                  \
    B200RL_REQUIRE(A >= 2 && A <= b200rl::kPqnMaxA, what ": A=%d outside [2, %d]", A, b200rl::kPqnMaxA)

#define PQN_ALIGNED(what, ...)                                                                                         \
    do {                                                                                                               \
        const void* ps_[] = {__VA_ARGS__};                                                                             \
        for (const void* p_ : ps_) B200RL_REQUIRE(b200rl::aligned(p_, 4), what ": misaligned pointer");               \
    } while (0)

extern "C" int64_t b200rl_pqn_param_count(int obs_dim, int A) {
    if (obs_dim < 1 || obs_dim > b200rl::kPqnMaxIn || A < 2 || A > b200rl::kPqnMaxA) return -1;
    return b200rl::PqnOff(obs_dim, A).total;
}

extern "C" size_t b200rl_pqn_workspace_bytes(int64_t M) {
    if (M < 1) return 0;
    return b200rl::PqnWs::bytes(M);
}

extern "C" int b200rl_pqn_act_f32(const float* params, const float* obs, int64_t ld_obs, int64_t n, int obs_dim, int A,
                                  const int64_t* random_actions, const float* u, double eps, float* obs_slot,
                                  int64_t* actions_slot, float* values_slot, const float* copy_in, float* copy_out,
                                  int64_t copy_n, void* stream) {
    using namespace b200rl;
    PQN_SHAPES("pqn_act");
    B200RL_REQUIRE(n >= 1, "pqn_act: n=%lld must be >= 1", (long long)n);
    B200RL_REQUIRE(params && obs && values_slot, "pqn_act: null pointer");
    B200RL_REQUIRE(ld_obs >= obs_dim, "pqn_act: ld_obs=%lld < obs_dim=%d", (long long)ld_obs, obs_dim);
    B200RL_REQUIRE((random_actions == nullptr) == (u == nullptr), "pqn_act: random_actions and u go together");
    B200RL_REQUIRE(!random_actions || actions_slot, "pqn_act: the epsilon-greedy step needs actions_slot");
    B200RL_REQUIRE(copy_n >= 0 && (copy_n == 0 || (copy_in && copy_out)), "pqn_act: copy_n=%lld without buffers",
                   (long long)copy_n);
    PQN_ALIGNED("pqn_act", params, obs, u, obs_slot, values_slot, copy_in, copy_out);
    B200RL_REQUIRE(aligned(random_actions, 8) && aligned(actions_slot, 8), "pqn_act: misaligned action buffer");
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "pqn_act", 2.0 * n * (kP1 * obs_dim + kP2 * kP1 + A * kP2), 0);
    PqnActParams P{params, obs, ld_obs, n, obs_dim, A, random_actions, u, (float)eps, obs_slot, actions_slot,
                   values_slot, nullptr, copy_n ? copy_in : nullptr, copy_out, copy_n};
    pqn_act_kernel<<<(unsigned)ceil_div(n, kPqnRows), kPqnThreads, 0, s>>>(P);
    return check_launch("pqn_act");
}

extern "C" int b200rl_pqn_forward_f32(const float* params, const float* obs, int64_t ld_obs, int64_t n, int obs_dim,
                                      int A, float* q, void* stream) {
    using namespace b200rl;
    PQN_SHAPES("pqn_forward");
    B200RL_REQUIRE(n >= 1, "pqn_forward: n=%lld must be >= 1", (long long)n);
    B200RL_REQUIRE(params && obs && q, "pqn_forward: null pointer");
    B200RL_REQUIRE(ld_obs >= obs_dim, "pqn_forward: ld_obs=%lld < obs_dim=%d", (long long)ld_obs, obs_dim);
    PQN_ALIGNED("pqn_forward", params, obs, q);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "pqn_forward", 2.0 * n * (kP1 * obs_dim + kP2 * kP1 + A * kP2), 0);
    PqnActParams P{params, obs, ld_obs, n, obs_dim, A, nullptr, nullptr, 0.f, nullptr, nullptr, nullptr, q, nullptr,
                   nullptr, 0};
    pqn_act_kernel<<<(unsigned)ceil_div(n, kPqnRows), kPqnThreads, 0, s>>>(P);
    return check_launch("pqn_forward");
}

extern "C" int b200rl_pqn_loss_bwd_f32(const float* params, const float* obs, int64_t ld_obs, const int64_t* mb_inds,
                                       const int64_t* b_actions, const float* b_returns, int64_t M, int obs_dim, int A,
                                       float* stats, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    PQN_SHAPES("pqn_loss_bwd");
    B200RL_REQUIRE(M >= 1, "pqn_loss_bwd: M=%lld must be >= 1", (long long)M);
    B200RL_REQUIRE(params && obs && b_actions && b_returns && stats, "pqn_loss_bwd: null pointer");
    B200RL_REQUIRE(ld_obs >= obs_dim, "pqn_loss_bwd: ld_obs=%lld < obs_dim=%d", (long long)ld_obs, obs_dim);
    PQN_ALIGNED("pqn_loss_bwd", params, obs, b_returns, stats);
    B200RL_REQUIRE(aligned(mb_inds, 8) && aligned(b_actions, 8), "pqn_loss_bwd: misaligned index buffer");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "pqn_loss_bwd: workspace null or misaligned");
    if (workspace_bytes < b200rl_pqn_workspace_bytes(M))
        return fail(B200RL_ERR_WORKSPACE, "pqn_loss_bwd: workspace %zu < %zu", workspace_bytes,
                    b200rl_pqn_workspace_bytes(M));
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "pqn_loss_bwd", 4.0 * M * (kP1 * obs_dim + kP2 * kP1 + kP2), 0);
    PqnLossParams P{params, obs, ld_obs, mb_inds, b_actions, b_returns, M, obs_dim, A, (float)(2.0 / (double)M), stats,
                    workspace};
    pqn_loss_bwd_kernel<<<(unsigned)ceil_div(M, kPqnRows), kPqnThreads, 0, s>>>(P);
    return check_launch("pqn_loss_bwd");
}

extern "C" int b200rl_pqn_wgrad_f32(const float* obs, int64_t ld_obs, const int64_t* mb_inds, const int64_t* b_actions,
                                    int64_t M, int obs_dim, int A, const void* workspace, size_t workspace_bytes,
                                    float* grad, void* stream) {
    using namespace b200rl;
    PQN_SHAPES("pqn_wgrad");
    B200RL_REQUIRE(M >= 1, "pqn_wgrad: M=%lld must be >= 1", (long long)M);
    B200RL_REQUIRE(obs && b_actions && grad, "pqn_wgrad: null pointer");
    B200RL_REQUIRE(ld_obs >= obs_dim, "pqn_wgrad: ld_obs=%lld < obs_dim=%d", (long long)ld_obs, obs_dim);
    PQN_ALIGNED("pqn_wgrad", obs, grad);
    B200RL_REQUIRE(aligned(mb_inds, 8) && aligned(b_actions, 8), "pqn_wgrad: misaligned index buffer");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "pqn_wgrad: workspace null or misaligned");
    if (workspace_bytes < b200rl_pqn_workspace_bytes(M))
        return fail(B200RL_ERR_WORKSPACE, "pqn_wgrad: workspace %zu < %zu", workspace_bytes,
                    b200rl_pqn_workspace_bytes(M));
    const PqnWs W(const_cast<void*>(workspace), M);
    const PqnOff o(obs_dim, A);
    PqnWgradParams P{};
    const int S = pqn_splits(M);
    P.M = M; P.rows = mb_inds; P.actions = b_actions; P.dq = W.dq; P.A = A;
    P.rows_per_split = ceil_div(ceil_div(M, S), kPqnWT) * kPqnWT;
    P.tile_partials = W.tile_partials; P.tile_tickets = W.tile_tickets;
    int t = 0;
    auto add = [&](const float* dz, int ld_dz, const float* x, int64_t ld_x, const int64_t* x_rows, int N, int K,
                   float* dw, float* db) {
        PqnWgradJob& J = P.job[P.njobs++];
        J = PqnWgradJob{dz, ld_dz, x, ld_x, x_rows, N, K, dw, db, (int)ceil_div(K + 1, kPqnWT), t};
        t += (int)ceil_div(N, kPqnWT) * J.tiles_k;
    };
    add(W.dz1, kP1, obs, ld_obs, mb_inds, kP1, obs_dim, grad + o.w1, grad + o.b1);
    add(W.gx1, kP1, nullptr, 0, nullptr, kP1, 0, nullptr, grad + o.g1);
    add(W.dy1, kP1, nullptr, 0, nullptr, kP1, 0, nullptr, grad + o.be1);
    add(W.dz2, kP2, W.h1, kP1, nullptr, kP2, kP1, grad + o.w2, grad + o.b2);
    add(W.gx2, kP2, nullptr, 0, nullptr, kP2, 0, nullptr, grad + o.g2);
    add(W.dy2, kP2, nullptr, 0, nullptr, kP2, 0, nullptr, grad + o.be2);
    add(nullptr, 0, W.h2, kP2, nullptr, A, kP2, grad + o.w3, grad + o.b3);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "pqn_wgrad", 2.0 * M * (kP1 * (obs_dim + 3) + kP2 * (kP1 + 3) + A * (kP2 + 1)), 0);
    if (t > kPqnMaxTiles) return fail(B200RL_ERR_UNSUPPORTED, "pqn_wgrad: %d tiles > %d", t, kPqnMaxTiles);
    pqn_wgrad_kernel<<<dim3((unsigned)t, (unsigned)ceil_div(M, P.rows_per_split)), kPqnWgThreads, 0, s>>>(P);
    return check_launch("pqn_wgrad");
}

extern "C" int b200rl_qlambda_f32(const float* rewards, const float* values, const float* dones, const float* next_value,
                                  const float* next_done, float* returns, int64_t T, int64_t N, double gamma,
                                  double q_lambda, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(T >= 1 && N >= 1, "qlambda: T=%lld, N=%lld must be >= 1", (long long)T, (long long)N);
    B200RL_REQUIRE(rewards && values && dones && next_value && next_done && returns, "qlambda: null pointer");
    PQN_ALIGNED("qlambda", rewards, values, dones, next_value, next_done, returns);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "qlambda", 8.0 * T * N, 20.0 * T * N);
    qlambda_kernel<<<(unsigned)ceil_div(N, 128), 128, 0, s>>>(rewards, values, dones, next_value, next_done, returns, T,
                                                               N, (float)gamma, (float)q_lambda,
                                                               (float)(1.0 - q_lambda));
    return check_launch("qlambda");
}
