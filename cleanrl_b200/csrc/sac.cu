// Discrete soft actor-critic (cleanrl/sac_atari.py): the policy's log-probabilities and probabilities, the soft-Q target
// and critic loss with both Q heads' gradients, and the actor loss with its gradient and the temperature step -- one
// thread per row, A <= 32 actions.
//
// Numerics follow the reference's fp32 torch expressions where their order is visible (separately rounded, no fused
// multiply-adds where torch rounds twice), e.g. y = r + ((1 - d) * gamma) * v.  Reductions over rows go through
// per-block partials that the last block folds in a fixed order (no float atomics): results are bitwise repeatable.
//
// The temperature lives in device memory: the critic reads alpha, the actor-loss kernel reads alpha and log_alpha and,
// with autotune, its last block takes the Adam step of log_alpha and rewrites alpha = exp(log_alpha) after every block
// has read the old values (the ticket orders them).  The host never reads alpha inside an update.
#include "common.cuh"

namespace b200rl {

constexpr int kSacThreads = 128;
constexpr int kSacMaxA = 32;

// log_softmax and softmax of one row of logits: the row's max and sum of exp(x - max); each action's terms are then
// recomputed from its logit (no per-row arrays: nothing goes to local memory).
struct PolicyRow {
    float mx, s, lse;
    __device__ __forceinline__ PolicyRow(const float* __restrict__ x, int A) {
        mx = x[0];
        for (int a = 1; a < A; ++a) mx = fmaxf(mx, x[a]);
        s = 0.f;
        for (int a = 0; a < A; ++a) s = __fadd_rn(s, expf(__fsub_rn(x[a], mx)));
        lse = logf(s);
    }
    __device__ __forceinline__ float logp(float xa) const { return __fsub_rn(__fsub_rn(xa, mx), lse); }   // F.log_softmax
    __device__ __forceinline__ float prob(float xa) const { return __fdiv_rn(expf(__fsub_rn(xa, mx)), s); }  // .probs
};

// Last-block fold of K per-block partials: sums[k] = sum over blocks in block order (fixed), valid in thread 0.
template <int K>
__device__ __forceinline__ bool fold_partials(float (&v)[K], float* partials, unsigned int* ticket, float* red,
                                              bool* is_last) {
    for (int k = 0; k < K; ++k) v[k] = block_sum(v[k], red);
    if (threadIdx.x == 0) {
        for (int k = 0; k < K; ++k) partials[K * blockIdx.x + k] = v[k];
        __threadfence();
        *is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!*is_last) return false;
    __threadfence();
    float acc[K];
    for (int k = 0; k < K; ++k) acc[k] = 0.f;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x)
        for (int k = 0; k < K; ++k) acc[k] += __ldcg(partials + K * b + k);
    for (int k = 0; k < K; ++k) v[k] = block_sum(acc[k], red);
    return true;
}

__global__ void __launch_bounds__(kSacThreads) sac_policy_kernel(const float* __restrict__ logits, int64_t ld, int64_t n,
                                                                 int A, float* __restrict__ logp, int64_t ldl,
                                                                 float* __restrict__ probs, int64_t ldp) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* x = logits + i * ld;
    const PolicyRow r(x, A);
    for (int a = 0; a < A; ++a) {
        if (logp) logp[i * ldl + a] = r.logp(x[a]);
        if (probs) probs[i * ldp + a] = r.prob(x[a]);
    }
}

struct SacCriticParams {
    const float* nl; int64_t ldnl;             // actor logits on next_obs
    const float* q1t; int64_t ldq1t;
    const float* q2t; int64_t ldq2t;
    const float* q1; int64_t ldq1;
    const float* q2; int64_t ldq2;
    const int64_t* actions; const float* rewards; const float* dones; const float* alpha;
    int64_t B; int A; float gamma; float two_over_b;
    float* y; float* dq1; int64_t lddq1; float* dq2; int64_t lddq2;
    float* stats; float* partials; unsigned int* ticket;
};

__global__ void __launch_bounds__(kSacThreads) sac_critic_loss_kernel(SacCriticParams P) {
    __shared__ float red[32];
    __shared__ bool is_last;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float v[4] = {0.f, 0.f, 0.f, 0.f};          // qf1_a, qf2_a, (qf1_a - y)^2, (qf2_a - y)^2
    if (i < P.B) {
        const float alpha = __ldg(P.alpha);
        const float* x = P.nl + i * P.ldnl;
        const PolicyRow r(x, P.A);
        const float* q1t = P.q1t + i * P.ldq1t;
        const float* q2t = P.q2t + i * P.ldq2t;
        // (probs * (min(q1t, q2t) - alpha * logp)).sum(1)   (sac_atari.py:279-284)
        float m = 0.f;
        for (int a = 0; a < P.A; ++a)
            m = __fadd_rn(m, __fmul_rn(r.prob(x[a]), __fsub_rn(fminf(q1t[a], q2t[a]), __fmul_rn(alpha, r.logp(x[a])))));
        const float y = __fadd_rn(P.rewards[i], __fmul_rn(__fmul_rn(__fsub_rn(1.f, P.dones[i]), P.gamma), m));
        int a = (int)P.actions[i];
        a = a < 0 ? 0 : (a >= P.A ? P.A - 1 : a);
        const float q1a = P.q1[i * P.ldq1 + a], q2a = P.q2[i * P.ldq2 + a];
        const float d1 = __fsub_rn(q1a, y), d2 = __fsub_rn(q2a, y);
        v[0] = q1a; v[1] = q2a; v[2] = __fmul_rn(d1, d1); v[3] = __fmul_rn(d2, d2);
        if (P.y) P.y[i] = y;
        float* g1 = P.dq1 + i * P.lddq1;
        float* g2 = P.dq2 + i * P.lddq2;
        // F.mse_loss backward: (2 / B) * (input - target), scattered to the taken action by gather's backward
        for (int k = 0; k < P.A; ++k) {
            g1[k] = k == a ? __fmul_rn(P.two_over_b, d1) : 0.f;
            g2[k] = k == a ? __fmul_rn(P.two_over_b, d2) : 0.f;
        }
    }
    if (!fold_partials<4>(v, P.partials, P.ticket, red, &is_last)) return;
    if (threadIdx.x == 0) {
        const float b = (float)P.B;
        P.stats[0] = v[0] / b;     // losses/qf1_values
        P.stats[1] = v[1] / b;     // losses/qf2_values
        P.stats[2] = v[2] / b;     // losses/qf1_loss
        P.stats[3] = v[3] / b;     // losses/qf2_loss
        *P.ticket = 0;
    }
}

struct SacActorParams {
    const float* logits; int64_t ld;
    const float* q1; int64_t ldq1;
    const float* q2; int64_t ldq2;
    int64_t B; int A; float inv_ba; float target_entropy;
    float* alpha; float* log_alpha; float* m; float* v; const float* step_scalars;
    float w1, beta2, w2, eps; int autotune;
    float* dlogits; int64_t ldd; float* stats; float* partials; unsigned int* ticket;
};

__global__ void __launch_bounds__(kSacThreads) sac_actor_loss_kernel(SacActorParams P) {
    __shared__ float red[32];
    __shared__ bool is_last;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float alpha = __ldcg(P.alpha);
    const float ea = P.autotune ? expf(__ldcg(P.log_alpha)) : 0.f;
    float s[3] = {0.f, 0.f, 0.f};                // sum p * f, sum p * (-ea * (logp + te)), sum (p / (B A)) * (logp + te)
    if (i < P.B) {
        const float* x = P.logits + i * P.ld;
        const PolicyRow r(x, P.A);
        const float* q1 = P.q1 + i * P.ldq1;
        const float* q2 = P.q2 + i * P.ldq2;
        // action_probs * ((alpha * log_pi) - min_qf_values)   (sac_atari.py:301)
        auto f = [&](int a) { return __fsub_rn(__fmul_rn(alpha, r.logp(x[a])), fminf(q1[a], q2[a])); };
        float dot = 0.f;
        for (int a = 0; a < P.A; ++a) dot = __fadd_rn(dot, __fmul_rn(r.prob(x[a]), f(a)));
        s[0] = dot;
        float* d = P.dlogits + i * P.ldd;
        for (int a = 0; a < P.A; ++a) d[a] = __fmul_rn(__fmul_rn(r.prob(x[a]), __fsub_rn(f(a), dot)), P.inv_ba);
        if (P.autotune) {
            // alpha_loss = (probs * (-exp(log_alpha) * (log_pi + target_entropy))).mean()   (sac_atari.py:309)
            for (int a = 0; a < P.A; ++a) {
                const float p = r.prob(x[a]), t = __fadd_rn(r.logp(x[a]), P.target_entropy);
                s[1] = __fadd_rn(s[1], __fmul_rn(p, __fmul_rn(-ea, t)));
                s[2] = __fadd_rn(s[2], __fmul_rn(__fmul_rn(P.inv_ba, p), t));
            }
        }
    }
    if (!fold_partials<3>(s, P.partials, P.ticket, red, &is_last)) return;
    if (threadIdx.x == 0) {
        const float ba = (float)(P.B * P.A);
        P.stats[0] = s[0] / ba;                  // losses/actor_loss
        if (P.autotune) {
            P.stats[1] = s[1] / ba;              // losses/alpha_loss
            // d alpha_loss / d log_alpha: the mean's gradient summed over the broadcast, negated, times exp(log_alpha)
            const float g = __fmul_rn(-s[2], ea);
            float m = *P.m, v = *P.v, la = *P.log_alpha;
            m = fmaf(P.w1, g - m, m);                                     // exp_avg.lerp_(grad, 1 - beta1)
            v = v * P.beta2;
            v = __fadd_rn(v, __fmul_rn(__fmul_rn(P.w2, g), g));
            const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), P.step_scalars[0]), P.eps);
            la = __fadd_rn(la, __fmul_rn(P.step_scalars[1], __fdiv_rn(m, denom)));
            *P.m = m; *P.v = v; *P.log_alpha = la;
            *P.alpha = expf(la);                 // alpha = log_alpha.exp().item()
        } else {
            P.stats[1] = 0.f;
        }
        P.stats[2] = *P.alpha;
        P.stats[3] = P.autotune ? *P.log_alpha : 0.f;
        *P.ticket = 0;
    }
}

static size_t sac_ws_bytes(int64_t B, int K) {
    return 16 + (size_t)ceil_div(B > 0 ? B : 1, kSacThreads) * K * sizeof(float);
}

}  // namespace b200rl

extern "C" int b200rl_sac_policy_f32(const float* logits, int64_t ld, int64_t n, int A, float* logp, int64_t ld_logp,
                                     float* probs, int64_t ld_probs, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(n >= 0 && n <= 0x7fffffff, "sac_policy: n outside [0, 2^31)");
    B200RL_REQUIRE(A >= 2 && A <= kSacMaxA, "sac_policy: A=%d outside [2,%d]", A, kSacMaxA);
    B200RL_REQUIRE(logits && (logp || probs), "sac_policy: null pointer");
    B200RL_REQUIRE(ld >= A && (!logp || ld_logp >= A) && (!probs || ld_probs >= A), "sac_policy: bad strides");
    B200RL_REQUIRE(aligned(logits, 4) && (!logp || aligned(logp, 4)) && (!probs || aligned(probs, 4)),
                   "sac_policy: misaligned pointer");
    if (n == 0) return B200RL_OK;
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "sac_policy", 0, (double)n * 12.0 * A);
    sac_policy_kernel<<<(unsigned)ceil_div(n, kSacThreads), kSacThreads, 0, s>>>(logits, ld, n, A, logp, ld_logp, probs,
                                                                                ld_probs);
    return check_launch("sac_policy");
}

extern "C" size_t b200rl_sac_critic_loss_workspace_bytes(int64_t B) {
    return B < 0 ? 0 : b200rl::sac_ws_bytes(B, 4);
}

extern "C" int b200rl_sac_critic_loss_f32(const float* next_logits, int64_t ld_next, const float* q1_target,
                                          int64_t ld_q1t, const float* q2_target, int64_t ld_q2t, const float* q1,
                                          int64_t ld_q1, const float* q2, int64_t ld_q2, const int64_t* actions,
                                          const float* rewards, const float* dones, const float* alpha, int64_t B, int A,
                                          double gamma, float* y, float* dq1, int64_t ld_dq1, float* dq2, int64_t ld_dq2,
                                          float* stats, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(B >= 1 && B <= 0x7fffffff, "sac_critic_loss: B must be in [1, 2^31)");
    B200RL_REQUIRE(A >= 2 && A <= kSacMaxA, "sac_critic_loss: A=%d outside [2,%d]", A, kSacMaxA);
    B200RL_REQUIRE(ld_next >= A && ld_q1t >= A && ld_q2t >= A && ld_q1 >= A && ld_q2 >= A && ld_dq1 >= A && ld_dq2 >= A,
                   "sac_critic_loss: bad strides");
    B200RL_REQUIRE(next_logits && q1_target && q2_target && q1 && q2 && actions && rewards && dones && alpha && dq1 && dq2 &&
                   stats, "sac_critic_loss: null pointer");
    B200RL_REQUIRE(aligned(next_logits, 4) && aligned(q1_target, 4) && aligned(q2_target, 4) && aligned(q1, 4) &&
                   aligned(q2, 4) && aligned(actions, 8) && aligned(rewards, 4) && aligned(dones, 4) && aligned(alpha, 4) &&
                   (!y || aligned(y, 4)) && aligned(dq1, 4) && aligned(dq2, 4) && aligned(stats, 4),
                   "sac_critic_loss: misaligned pointer");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "sac_critic_loss: workspace null or misaligned");
    if (workspace_bytes < b200rl_sac_critic_loss_workspace_bytes(B))
        return fail(B200RL_ERR_WORKSPACE, "sac_critic_loss: workspace %zu < %zu", workspace_bytes,
                    b200rl_sac_critic_loss_workspace_bytes(B));
    cudaStream_t s = (cudaStream_t)stream;
    unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
    float* partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16);
    ProfScope ps(s, "sac_critic_loss", 0, (double)B * (28.0 * A + 24));
    cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int), s);
    if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "sac_critic_loss: memset: %s", cudaGetErrorString(e));
    SacCriticParams P{next_logits, ld_next, q1_target, ld_q1t, q2_target, ld_q2t, q1, ld_q1, q2, ld_q2, actions, rewards,
                      dones, alpha, B, A, (float)gamma, (float)(2.0 / (double)B), y, dq1, ld_dq1, dq2, ld_dq2, stats,
                      partials, ticket};
    sac_critic_loss_kernel<<<(unsigned)ceil_div(B, kSacThreads), kSacThreads, 0, s>>>(P);
    return check_launch("sac_critic_loss");
}

extern "C" size_t b200rl_sac_actor_loss_workspace_bytes(int64_t B) {
    return B < 0 ? 0 : b200rl::sac_ws_bytes(B, 3);
}

extern "C" int b200rl_sac_actor_loss_f32(const float* logits, int64_t ld, const float* q1, int64_t ld_q1, const float* q2,
                                         int64_t ld_q2, int64_t B, int A, float* alpha, int autotune, float* log_alpha,
                                         float* exp_avg, float* exp_avg_sq, const float* step_scalars, double target_entropy,
                                         double beta1, double beta2, double eps, float* dlogits, int64_t ld_d, float* stats,
                                         void* workspace, size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(B >= 1 && B <= 0x7fffffff, "sac_actor_loss: B must be in [1, 2^31)");
    B200RL_REQUIRE(A >= 2 && A <= kSacMaxA, "sac_actor_loss: A=%d outside [2,%d]", A, kSacMaxA);
    B200RL_REQUIRE(ld >= A && ld_q1 >= A && ld_q2 >= A && ld_d >= A, "sac_actor_loss: bad strides");
    B200RL_REQUIRE(logits && q1 && q2 && alpha && dlogits && stats, "sac_actor_loss: null pointer");
    B200RL_REQUIRE(!autotune || (log_alpha && exp_avg && exp_avg_sq && step_scalars),
                   "sac_actor_loss: autotune needs log_alpha, its Adam moments and the step scalars");
    B200RL_REQUIRE(aligned(logits, 4) && aligned(q1, 4) && aligned(q2, 4) && aligned(alpha, 4) && aligned(dlogits, 4) &&
                   aligned(stats, 4) && (!log_alpha || aligned(log_alpha, 4)) && (!exp_avg || aligned(exp_avg, 4)) &&
                   (!exp_avg_sq || aligned(exp_avg_sq, 4)) && (!step_scalars || aligned(step_scalars, 4)),
                   "sac_actor_loss: misaligned pointer");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "sac_actor_loss: workspace null or misaligned");
    if (workspace_bytes < b200rl_sac_actor_loss_workspace_bytes(B))
        return fail(B200RL_ERR_WORKSPACE, "sac_actor_loss: workspace %zu < %zu", workspace_bytes,
                    b200rl_sac_actor_loss_workspace_bytes(B));
    cudaStream_t s = (cudaStream_t)stream;
    unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
    float* partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16);
    ProfScope ps(s, "sac_actor_loss", 0, (double)B * 16.0 * A);
    cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int), s);
    if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "sac_actor_loss: memset: %s", cudaGetErrorString(e));
    SacActorParams P{logits, ld, q1, ld_q1, q2, ld_q2, B, A, (float)(1.0 / ((double)B * A)), (float)target_entropy,
                     alpha, log_alpha, exp_avg, exp_avg_sq, step_scalars,
                     (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, autotune != 0,
                     dlogits, ld_d, stats, partials, ticket};
    sac_actor_loss_kernel<<<(unsigned)ceil_div(B, kSacThreads), kSacThreads, 0, s>>>(P);
    return check_launch("sac_actor_loss");
}
