// Phasic policy gradient: the auxiliary-phase loss with its gradient (cleanrl/ppg_procgen.py:449-461).
//
//   kl_loss         = mean_i KL(Categorical(old_logits_i) || Categorical(logits_i))
//   aux_value_loss  = 0.5 mean_i (aux_value_i - R_i)^2
//   real_value_loss = 0.5 mean_i (value_i - R_i)^2
//   loss            = (aux_value_loss + beta_clone kl_loss + real_value_loss) / n_aux_grad_accum
//
// The network's joint head gives [logits | value | aux_value] per row; the kernel writes d(loss)/d(head) for all A + 2
// columns.  Row i of the minibatch is row rows[i] of the auxiliary buffer (the gather the forward used).  Both logit sets
// are normalised inside the kernel; the KL follows torch.distributions.kl._kl_categorical_categorical at the edges: a
// term with p_old == 0 is 0, a term with p_new == 0 < p_old is +inf.
// Launch pair: one thread per row with per-block partial sums, then one block folds the partials in a fixed order.
#include "common.cuh"

namespace b200rl {

constexpr int kAuxThreads = 128;
constexpr int kAuxMaxA = 22;               // A + 2 head outputs <= kMaxHeads of the tensor-core plans

struct AuxLossParams {
    const float* head; int64_t ld;         // [n][A + 2], row stride ld
    const int64_t* rows;                   // null = identity
    const float* old_logits;               // [*][A]
    const float* returns;                  // [*]
    int64_t n; int A;
    float beta, inv_accum;
    float* dhead; int64_t ldd;
    float* partials;                       // [gridDim.x][3]
};

// x lives in registers: fixed trip counts, entries past A masked
__device__ __forceinline__ float log_sum_exp(const float (&x)[kAuxMaxA], int A) {
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < kAuxMaxA; ++k) if (k < A) m = fmaxf(m, x[k]);
    if (m == -INFINITY || m == INFINITY) m = 0.f;          // as torch.logsumexp: no inf - inf
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kAuxMaxA; ++k) if (k < A) s += expf(x[k] - m);
    return logf(s) + m;
}

__global__ void __launch_bounds__(kAuxThreads) ppg_aux_rows_kernel(AuxLossParams P) {
    __shared__ float red[32];
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float kl = 0.f, sq_aux = 0.f, sq_val = 0.f;
    if (i < P.n) {
        const int A = P.A;
        const int64_t j = P.rows ? P.rows[i] : i;
        const float* x = P.head + i * P.ld;
        float xn[kAuxMaxA], xo[kAuxMaxA];
#pragma unroll
        for (int k = 0; k < kAuxMaxA; ++k)
            if (k < A) { xn[k] = x[k]; xo[k] = __ldg(P.old_logits + j * A + k); }
        const float lse_n = log_sum_exp(xn, A), lse_o = log_sum_exp(xo, A);
        const float scale = P.inv_accum / (float)P.n;
        float* d = P.dhead + i * P.ldd;
#pragma unroll
        for (int k = 0; k < kAuxMaxA; ++k) {
            if (k < A) {
                const float lp_n = xn[k] - lse_n, lp_o = xo[k] - lse_o;
                const float p_n = expf(lp_n), p_o = expf(lp_o);
                float t = p_o * (lp_o - lp_n);
                if (p_n == 0.f) t = INFINITY;
                if (p_o == 0.f) t = 0.f;
                kl += t;
                d[k] = P.beta * (p_n - p_o) * scale;
            }
        }
        const float R = __ldg(P.returns + j);
        const float dv = x[A] - R, da = x[A + 1] - R;
        d[A] = dv * scale;
        d[A + 1] = da * scale;
        sq_val = dv * dv;
        sq_aux = da * da;
    }
    const float s0 = block_sum(kl, red), s1 = block_sum(sq_aux, red), s2 = block_sum(sq_val, red);
    if (threadIdx.x == 0) {
        float* p = P.partials + (int64_t)blockIdx.x * 3;
        p[0] = s0; p[1] = s1; p[2] = s2;
    }
}

// stats[0..2] = kl_loss, aux_value_loss, real_value_loss: thread t sums partials t, t + 128, ...; then the block in order
__global__ void __launch_bounds__(kAuxThreads) ppg_aux_fold_kernel(const float* __restrict__ partials, int nblocks, int64_t n,
                                                                   float* __restrict__ stats) {
    __shared__ float red[32];
    float tot[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float s = 0.f;
        for (int b = threadIdx.x; b < nblocks; b += blockDim.x) s += partials[(int64_t)b * 3 + k];
        tot[k] = block_sum(s, red);
    }
    if (threadIdx.x == 0) {
        const float inv = 1.0f / (float)n;
        stats[0] = tot[0] * inv;
        stats[1] = 0.5f * (tot[1] * inv);
        stats[2] = 0.5f * (tot[2] * inv);
    }
}

constexpr int64_t kAuxMaxN = (int64_t)1 << 22;

}  // namespace b200rl

using namespace b200rl;

extern "C" size_t b200rl_ppg_aux_loss_workspace_bytes(int64_t n) {
    return n >= 1 && n <= kAuxMaxN ? (size_t)ceil_div(n, kAuxThreads) * 3 * sizeof(float) : 0;
}

extern "C" int b200rl_ppg_aux_loss_f32(const float* head_out, int64_t ld_head, const int64_t* rows, const float* old_logits,
                                       const float* returns, int64_t n, int A, double beta_clone, double inv_accum,
                                       float* dhead, int64_t ld_dhead, float* stats, void* workspace, size_t workspace_bytes,
                                       void* stream) {
    B200RL_REQUIRE(n >= 1 && n <= kAuxMaxN, "ppg_aux_loss: n=%lld outside [1,%lld]", (long long)n, (long long)kAuxMaxN);
    B200RL_REQUIRE(A >= 1 && A <= kAuxMaxA, "ppg_aux_loss: A=%d outside [1,%d]", A, kAuxMaxA);
    B200RL_REQUIRE(head_out && old_logits && returns, "ppg_aux_loss: null input pointer");
    B200RL_REQUIRE(dhead && stats, "ppg_aux_loss: null output pointer");
    B200RL_REQUIRE(ld_head >= A + 2 && ld_dhead >= A + 2, "ppg_aux_loss: bad strides");
    B200RL_REQUIRE(aligned(head_out, 4) && aligned(old_logits, 4) && aligned(returns, 4) && aligned(dhead, 4) &&
                   aligned(stats, 4) && aligned(rows, 8), "ppg_aux_loss: misaligned buffer");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "ppg_aux_loss: workspace null or not 16-B aligned");
    const size_t need = b200rl_ppg_aux_loss_workspace_bytes(n);
    if (workspace_bytes < need) return fail(B200RL_ERR_WORKSPACE, "ppg_aux_loss: workspace %zu < %zu bytes", workspace_bytes, need);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "ppg_aux_loss", 0, (double)n * (12.0 + 4.0 * (3 * A + 4)));
    AuxLossParams P;
    P.head = head_out; P.ld = ld_head; P.rows = rows; P.old_logits = old_logits; P.returns = returns;
    P.n = n; P.A = A; P.beta = (float)beta_clone; P.inv_accum = (float)inv_accum;
    P.dhead = dhead; P.ldd = ld_dhead; P.partials = reinterpret_cast<float*>(workspace);
    const int blocks = (int)ceil_div(n, kAuxThreads);
    ppg_aux_rows_kernel<<<blocks, kAuxThreads, 0, s>>>(P);
    ppg_aux_fold_kernel<<<1, kAuxThreads, 0, s>>>(P.partials, blocks, n, stats);
    return check_launch("ppg_aux_loss", 2);
}
