// Continuous soft actor-critic (cleanrl/sac_continuous_action.py): fp32 kernels for the reference's 256-wide MLPs.
//
//   critic  SoftQNetwork  [obs | act] (K = obs_dim + act_dim) -> 256 -> ReLU -> 256 -> ReLU -> 1
//   actor   Actor         obs -> 256 -> ReLU -> 256 -> ReLU -> fc_mean (D) and fc_logstd (D), tanh-Gaussian head
//
// The twin delayed DDPG of cleanrl/td3_continuous_action.py uses the same critics and trunk with a deterministic head:
//   actor   Actor         obs -> 256 -> ReLU -> 256 -> ReLU -> fc_mu (D), tanh(z) * scale + bias
// and cleanrl/ddpg_continuous_action.py the same actor with one critic (net_stride 0) instead of two.
//
// Flat parameter layout: each network's parameters in nn.Module order (fc1.weight [256, in], fc1.bias, fc2.weight, fc2.bias,
// head weight(s) and bias(es)); the twin critics are two such blocks ``net_stride`` floats apart (q_optimizer's one flat
// buffer, and the two targets' one flat buffer).
//
// Every forward / data-backward CTA owns kRows rows and the whole hidden width (thread j = hidden unit j), with the
// input, h1 and h2 (or their gradients) staged in shared memory; the input [obs[rows] | act] is assembled while it is
// loaded.  Dot products run sequentially over their inner index, weight gradients sequentially over rows, row means go
// through per-block partials folded by the last block in block order (no float atomics): every result is bitwise
// repeatable.  The tanh-Gaussian head, the losses and the temperature step follow the reference's visible operation
// order with separately rounded operations (__fadd_rn / __fmul_rn / __fdiv_rn keep nvcc from contracting them).
#include "common.cuh"

namespace b200rl {

constexpr int kH = 256;          // hidden width (the reference's)
constexpr int kRows = 8;         // rows per forward / data-backward CTA
constexpr int kSacMaxIn = 1024;  // obs_dim + act_dim
constexpr int kSacMaxD = 32;     // act_dim
constexpr int kLossThreads = 128;

// Parameter offsets of one network: fc1.w, fc1.b, fc2.w, fc2.b, then the head.
struct MlpOff {
    int64_t w1, b1, w2, b2, w3, b3, w4, b4;     // w4 / b4: fc_logstd (actor only)
    __host__ __device__ MlpOff(int64_t in, int out_per_head) {
        w1 = 0; b1 = w1 + (int64_t)kH * in; w2 = b1 + kH; b2 = w2 + (int64_t)kH * kH; w3 = b2 + kH;
        b3 = w3 + (int64_t)out_per_head * kH; w4 = b3 + out_per_head; b4 = w4 + (int64_t)out_per_head * kH;
    }
};

// torch.min / torch.minimum: NaN if either operand is NaN (fminf would drop it).
__device__ __forceinline__ float min_nan(float a, float b) {
    return (a != a || b != b) ? __int_as_float(0x7fc00000) : fminf(a, b);
}

// Last-block fold of K per-block partials in block order (as sac.cu); valid in thread 0 of the last block.
template <int K>
__device__ __forceinline__ bool fold(float (&v)[K], float* partials, unsigned int* ticket, float* red, bool* is_last) {
    for (int k = 0; k < K; ++k) v[k] = block_sum(v[k], red);
    if (threadIdx.x == 0) {
        for (int k = 0; k < K; ++k) partials[K * blockIdx.x + k] = v[k];
        __threadfence();
        *is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!*is_last) return false;
    __threadfence();
    if (threadIdx.x == 0) {
        for (int k = 0; k < K; ++k) {
            float acc = 0.f;
            for (unsigned b = 0; b < gridDim.x; ++b) acc = __fadd_rn(acc, __ldcg(partials + K * b + k));
            v[k] = acc;
        }
        *ticket = 0;
    }
    return true;
}

// out[r][j] = relu(b[j] + sum_k in[r][k] W[j][k]) for the CTA's rows; thread j = hidden unit j.
__device__ __forceinline__ void dense_relu(const float* __restrict__ W, const float* __restrict__ b, const float* in,
                                           int K, float* out) {
    const int j = threadIdx.x;
    float acc[kRows];
#pragma unroll
    for (int r = 0; r < kRows; ++r) acc[r] = 0.f;
    const float* w = W + (int64_t)j * K;
    for (int k = 0; k < K; ++k) {
        const float wk = __ldg(w + k);
#pragma unroll
        for (int r = 0; r < kRows; ++r) acc[r] = fmaf(wk, in[r * K + k], acc[r]);
    }
    const float bj = __ldg(b + j);
#pragma unroll
    for (int r = 0; r < kRows; ++r) out[r * kH + j] = fmaxf(__fadd_rn(acc[r], bj), 0.f);
}

// ---------------------------------------------------------------------------------------------- twin critic forward
struct CriticFwdParams {
    const float* params; int64_t net_stride;
    const float* obs; int64_t ld_obs; const int64_t* obs_rows;
    const float* act; int64_t ld_act; const int64_t* act_rows;
    int64_t B; int obs_dim, D;
    float* q;                                   // [2, B]
    float* keep_x; float* keep_h1; float* keep_h2;   // [B, K], [2, B, 256] x2 (optional)
};

__global__ void __launch_bounds__(kH) sacc_critic_fwd_kernel(CriticFwdParams P) {
    extern __shared__ float sm[];
    const int K = P.obs_dim + P.D;
    float* xs = sm;                       // [kRows][K]
    float* h1 = xs + kRows * K;           // [kRows][256]
    float* h2 = h1 + kRows * kH;
    const int net = blockIdx.y;
    const int64_t r0 = (int64_t)blockIdx.x * kRows;
    for (int i = threadIdx.x; i < kRows * K; i += kH) {
        const int r = i / K, k = i - r * K;
        const int64_t b = r0 + r;
        float v = 0.f;
        if (b < P.B) {
            if (k < P.obs_dim) v = P.obs[(P.obs_rows ? P.obs_rows[b] : b) * P.ld_obs + k];
            else v = P.act[(P.act_rows ? P.act_rows[b] : b) * P.ld_act + (k - P.obs_dim)];
            if (P.keep_x && net == 0) P.keep_x[b * K + k] = v;
        }
        xs[i] = v;
    }
    __syncthreads();
    const float* p = P.params + net * P.net_stride;
    const MlpOff o(K, 1);
    dense_relu(p + o.w1, p + o.b1, xs, K, h1);
    __syncthreads();
    dense_relu(p + o.w2, p + o.b2, h1, kH, h2);
    __syncthreads();
    if (P.keep_h1)
        for (int r = 0; r < kRows && r0 + r < P.B; ++r) {
            P.keep_h1[((int64_t)net * P.B + r0 + r) * kH + threadIdx.x] = h1[r * kH + threadIdx.x];
            P.keep_h2[((int64_t)net * P.B + r0 + r) * kH + threadIdx.x] = h2[r * kH + threadIdx.x];
        }
    // fc3: warp r reduces row r (lane-strided partial sums, then a fixed xor tree)
    const int lane = threadIdx.x & 31, r = threadIdx.x >> 5;
    float s = 0.f;
    for (int j = lane; j < kH; j += 32) s = fmaf(h2[r * kH + j], __ldg(p + o.w3 + j), s);
    s = warp_sum(s);
    if (lane == 0 && r0 + r < P.B) P.q[(int64_t)net * P.B + r0 + r] = __fadd_rn(s, __ldg(p + o.b3));
}

// --------------------------------------------------------------------------------------- actor forward + head
// Normal(mean, std).log_prob(x) - log(scale (1 - y^2) + 1e-6) of one element, as the reference evaluates it.
__device__ __forceinline__ float tanh_gauss_logp(float m, float std_, float x, float y, float scale) {
    const float u = __fsub_rn(x, m);
    const float var = __fmul_rn(std_, std_);
    const float q = __fdiv_rn(-__fmul_rn(u, u), __fmul_rn(2.f, var));
    const float lp = __fsub_rn(__fsub_rn(q, logf(std_)), 0.91893853320467274178f);   // math.log(math.sqrt(2 pi))
    const float w = __fadd_rn(__fmul_rn(scale, __fsub_rn(1.f, __fmul_rn(y, y))), 1e-6f);
    return __fsub_rn(lp, logf(w));
}

__device__ __forceinline__ float log_std_of(float raw) {
    // LOG_STD_MIN + 0.5 * (LOG_STD_MAX - LOG_STD_MIN) * (tanh(raw) + 1)
    return __fadd_rn(-5.f, __fmul_rn(3.5f, __fadd_rn(tanhf(raw), 1.f)));
}

// The actor's trunk for the CTA's rows: [obs[rows]] gathered into shared memory, h1 = relu(fc1), h2 = relu(fc2), each
// kept when asked.  ``sm`` holds [kRows][K + 512] floats; returns h2 there.
__device__ __forceinline__ const float* actor_trunk(const float* p, const MlpOff& o, const float* obs, int64_t ld_obs,
                                                    const int64_t* rows, int64_t B, int K, float* keep_x, float* keep_h1,
                                                    float* keep_h2, float* sm, int64_t r0) {
    float* xs = sm;
    float* h1 = xs + kRows * K;
    float* h2 = h1 + kRows * kH;
    for (int i = threadIdx.x; i < kRows * K; i += kH) {
        const int r = i / K, k = i - r * K;
        const int64_t b = r0 + r;
        float v = 0.f;
        if (b < B) {
            v = obs[(rows ? rows[b] : b) * ld_obs + k];
            if (keep_x) keep_x[b * K + k] = v;
        }
        xs[i] = v;
    }
    __syncthreads();
    dense_relu(p + o.w1, p + o.b1, xs, K, h1);
    __syncthreads();
    dense_relu(p + o.w2, p + o.b2, h1, kH, h2);
    __syncthreads();
    if (keep_h1)
        for (int r = 0; r < kRows && r0 + r < B; ++r) {
            keep_h1[(r0 + r) * kH + threadIdx.x] = h1[r * kH + threadIdx.x];
            keep_h2[(r0 + r) * kH + threadIdx.x] = h2[r * kH + threadIdx.x];
        }
    return h2;
}

struct ActorFwdParams {
    const float* params;
    const float* obs; int64_t ld_obs; const int64_t* rows;
    int64_t B; int obs_dim, D;
    const float* eps; const float* scale; const float* bias;
    float* action; float* log_pi; float* mean_out; float* mean_logstd;     // [B,D], [B], [B,D], [B,2D] (optional each)
    float* keep_x; float* keep_h1; float* keep_h2; float* keep_head;     // [B,obs], [B,256] x2, [B,2D] (optional)
    // temperature step (autotune re-evaluation): alpha_loss, the Adam step of log_alpha, alpha = exp(log_alpha)
    int temperature; float target_entropy, inv_b, w1, beta2, w2, adam_eps;
    float* alpha; float* log_alpha; float* m; float* v; const float* step_scalars;
    float* stats; float* partials; unsigned int* ticket;
};

__global__ void __launch_bounds__(kH) sacc_actor_fwd_kernel(ActorFwdParams P) {
    extern __shared__ float sm[];
    __shared__ float head[kRows][2 * kSacMaxD];
    __shared__ float lps[kRows][kSacMaxD];
    __shared__ float red[32];
    __shared__ bool is_last;
    const int K = P.obs_dim, D = P.D;
    const int64_t r0 = (int64_t)blockIdx.x * kRows;
    const MlpOff o(K, D);
    const float* p = P.params;
    const float* h2 = actor_trunk(p, o, P.obs, P.ld_obs, P.rows, P.B, K, P.keep_x, P.keep_h1, P.keep_h2, sm, r0);
    // joint [2D, 256] head: outputs 0..D-1 fc_mean, D..2D-1 fc_logstd
    for (int i = threadIdx.x; i < kRows * 2 * D; i += kH) {
        const int r = i / (2 * D), c = i - r * 2 * D;
        const float* w = c < D ? p + o.w3 + (int64_t)c * kH : p + o.w4 + (int64_t)(c - D) * kH;
        float s = 0.f;
        for (int j = 0; j < kH; ++j) s = fmaf(__ldg(w + j), h2[r * kH + j], s);
        s = __fadd_rn(s, c < D ? __ldg(p + o.b3 + c) : __ldg(p + o.b4 + c - D));
        head[r][c] = s;
        if (P.keep_head && r0 + r < P.B) P.keep_head[(r0 + r) * 2 * D + c] = s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kRows * D; i += kH) {
        const int r = i / D, d = i - r * D;
        const int64_t b = r0 + r;
        float lp = 0.f;
        if (b < P.B) {
            const float m = head[r][d];
            const float ls = log_std_of(head[r][D + d]);
            const float sc = P.scale[d], bi = P.bias[d];
            if (P.mean_out) P.mean_out[b * D + d] = __fadd_rn(__fmul_rn(tanhf(m), sc), bi);
            if (P.mean_logstd) { P.mean_logstd[b * 2 * D + d] = m; P.mean_logstd[b * 2 * D + D + d] = ls; }
            if (P.eps) {                                                        // Actor.forward alone draws nothing
                const float sd = expf(ls);
                const float x = __fadd_rn(m, __fmul_rn(P.eps[b * D + d], sd));  // rsample: loc + eps * scale
                const float y = tanhf(x);
                if (P.action) P.action[b * D + d] = __fadd_rn(__fmul_rn(y, sc), bi);
                lp = tanh_gauss_logp(m, sd, x, y, sc);
            }
        }
        lps[r][d] = lp;
    }
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < kRows && r0 + threadIdx.x < P.B) {
        float s = 0.f;
        for (int d = 0; d < D; ++d) s = __fadd_rn(s, lps[threadIdx.x][d]);        // log_prob.sum(1)
        if (P.log_pi) P.log_pi[r0 + threadIdx.x] = s;
        t = __fadd_rn(s, P.target_entropy);
    }
    if (!P.temperature) return;
    // alpha_loss = (-log_alpha.exp() * (log_pi + target_entropy)).mean() and its gradient w.r.t. log_alpha
    const float ea = expf(__ldcg(P.log_alpha));
    float s[2] = {0.f, 0.f};
    if (threadIdx.x < kRows && r0 + threadIdx.x < P.B) {
        s[0] = __fmul_rn(-ea, t);
        s[1] = __fmul_rn(P.inv_b, t);
    }
    if (!fold<2>(s, P.partials, P.ticket, red, &is_last)) return;
    if (threadIdx.x == 0) {
        P.stats[1] = __fdiv_rn(s[0], (float)P.B);                  // losses/alpha_loss
        const float g = __fmul_rn(-s[1], ea);
        float m = *P.m, v = *P.v, la = *P.log_alpha;
        m = fmaf(P.w1, g - m, m);                                   // exp_avg.lerp_(grad, 1 - beta1)
        v = v * P.beta2;
        v = __fadd_rn(v, __fmul_rn(__fmul_rn(P.w2, g), g));
        const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), P.step_scalars[0]), P.adam_eps);
        la = __fadd_rn(la, __fmul_rn(P.step_scalars[1], __fdiv_rn(m, denom)));
        *P.m = m; *P.v = v; *P.log_alpha = la;
        const float a = expf(la);                                  // alpha = log_alpha.exp().item()
        *P.alpha = a;
        P.stats[2] = a;
        P.stats[3] = la;
    }
}

// ------------------------------------------------------------------------- deterministic actor forward (TD3)
// torch.clamp: NaN stays NaN.
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

struct Td3ActorFwdParams {
    const float* params;
    const float* obs; int64_t ld_obs; const int64_t* rows;
    int64_t B; int obs_dim, D;
    const float* scale; const float* bias;
    float* mu; float* keep_y;                                            // [B, D] each (optional)
    float* keep_x; float* keep_h1; float* keep_h2;                       // [B, obs], [B, 256] x2 (optional)
    const float* eps; float policy_noise, noise_clip, lo, hi; float* smoothed;   // target policy smoothing (optional)
};

__global__ void __launch_bounds__(kH, 1) td3_actor_fwd_kernel(Td3ActorFwdParams P) {
    extern __shared__ float sm[];
    const int K = P.obs_dim, D = P.D;
    const int64_t r0 = (int64_t)blockIdx.x * kRows;
    const MlpOff o(K, D);
    const float* p = P.params;
    const float* h2 = actor_trunk(p, o, P.obs, P.ld_obs, P.rows, P.B, K, P.keep_x, P.keep_h1, P.keep_h2, sm, r0);
    // fc_mu, then x = tanh(z); x * action_scale + action_bias, each rounded
    for (int i = threadIdx.x; i < kRows * D; i += kH) {
        const int r = i / D, c = i - r * D;
        const int64_t b = r0 + r;
        if (b >= P.B) continue;
        const float* w = p + o.w3 + (int64_t)c * kH;
        float s = 0.f;
        for (int j = 0; j < kH; ++j) s = fmaf(__ldg(w + j), h2[r * kH + j], s);
        const float y = tanhf(__fadd_rn(s, __ldg(p + o.b3 + c)));
        const float sc = P.scale[c];
        const float mu = __fadd_rn(__fmul_rn(y, sc), P.bias[c]);
        if (P.keep_y) P.keep_y[b * D + c] = y;
        if (P.mu) P.mu[b * D + c] = mu;
        if (P.smoothed) {
            // clipped_noise = (eps * policy_noise).clamp(-noise_clip, noise_clip) * action_scale;
            // (mu + clipped_noise).clamp(low[0], high[0])
            const float n = __fmul_rn(clamp_nan(__fmul_rn(P.eps[b * D + c], P.policy_noise), -P.noise_clip, P.noise_clip), sc);
            P.smoothed[b * D + c] = clamp_nan(__fadd_rn(mu, n), P.lo, P.hi);
        }
    }
}

// ------------------------------------------------------------------------------------------------ critic loss
struct CriticLossParams {
    const float* q_next; const float* next_logpi; const float* q;        // [2,B], [B], [2,B]
    const float* rewards; const float* dones; int64_t ld_rd; const int64_t* rows; const float* alpha;
    int64_t B; float gamma, two_over_b;
    float* y; float* dq; float* stats; float* partials; unsigned int* ticket;
};

__global__ void __launch_bounds__(kLossThreads) sacc_critic_loss_kernel(CriticLossParams P) {
    __shared__ float red[32];
    __shared__ bool is_last;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (i < P.B) {
        const int64_t ri = (P.rows ? P.rows[i] : i) * P.ld_rd;
        // min(qf1_next_target, qf2_next_target) - alpha * next_state_log_pi; r + ((1 - d) * gamma) * that.  Without
        // next_logpi (TD3) the entropy term is absent: the min itself.
        float m = min_nan(P.q_next[i], P.q_next[P.B + i]);
        if (P.next_logpi) m = __fsub_rn(m, __fmul_rn(__ldg(P.alpha), P.next_logpi[i]));
        const float y = __fadd_rn(P.rewards[ri], __fmul_rn(__fmul_rn(__fsub_rn(1.f, P.dones[ri]), P.gamma), m));
        const float q1 = P.q[i], q2 = P.q[P.B + i];
        const float d1 = __fsub_rn(q1, y), d2 = __fsub_rn(q2, y);
        v[0] = q1; v[1] = q2; v[2] = __fmul_rn(d1, d1); v[3] = __fmul_rn(d2, d2);
        if (P.y) P.y[i] = y;
        P.dq[i] = __fmul_rn(P.two_over_b, d1);                     // F.mse_loss backward: (2 / B) (input - target)
        P.dq[P.B + i] = __fmul_rn(P.two_over_b, d2);
    }
    if (!fold<4>(v, P.partials, P.ticket, red, &is_last)) return;
    if (threadIdx.x == 0) {
        const float b = (float)P.B;
        for (int k = 0; k < 4; ++k) P.stats[k] = __fdiv_rn(v[k], b);    // qf1_values, qf2_values, qf1_loss, qf2_loss
    }
}

// ------------------------------------------------------------------------------------- twin critic data backward
// Critic step (dq given): dz2 = relu'(h2) * w3 dq, dz1 = relu'(h1) * W2^T dz2, kept for the weight gradients.
// Actor step (dq null): dq from actor_loss = mean(alpha log_pi - min(q1, q2)) -- -1/B to the smaller Q, half of it to each
// at a tie (autograd's binary min) -- and the gradient is carried to the action columns only: dact = W1[:, obs:]^T dz1.
// Single-network actor step (dq and q null, TD3): actor_loss = -mean(q1), dq = -1/B into the one network.
struct CriticBwdParams {
    const float* params; int64_t net_stride;
    int64_t B; int obs_dim, D;
    const float* dq; const float* q; float inv_b;
    const float* h1; const float* h2;
    float* dz1; float* dz2; float* dact;                  // [2,B,256] x2, [2,B,D]
};

// From dq of the CTA's rows (dq[r], row r0 + r) back through one critic's trunk: dz2 = relu'(h2) * w3 dq, then
// dz1 = relu'(h1) * W2^T dz2, into z2 / z1 in shared memory and, when dz1 is given, into dz1 / dz2 [B, 256].  h1, h2,
// dz1 and dz2 point at the network's own [B, 256] block.  The twin critic backward and the one-critic DDPG step share it.
__device__ __forceinline__ void critic_trunk_bwd(const float* p, const MlpOff& o, const float (&dq)[kRows],
                                                 const float* h1, const float* h2, float* dz1, float* dz2,
                                                 float (*z2)[kH], float (*z1)[kH], int64_t B, int64_t r0) {
    const int j = threadIdx.x;
    const float w3 = __ldg(p + o.w3 + j);
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
        const int64_t b = r0 + r;
        float g = 0.f;
        if (b < B) g = h2[b * kH + j] > 0.f ? __fmul_rn(dq[r], w3) : 0.f;
        z2[r][j] = g;
    }
    __syncthreads();
    float acc[kRows];
#pragma unroll
    for (int r = 0; r < kRows; ++r) acc[r] = 0.f;
    for (int i = 0; i < kH; ++i) {
        const float w = __ldg(p + o.w2 + (int64_t)i * kH + j);
#pragma unroll
        for (int r = 0; r < kRows; ++r) acc[r] = fmaf(w, z2[r][i], acc[r]);
    }
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
        const int64_t b = r0 + r;
        float g = 0.f;
        if (b < B) {
            g = h1[b * kH + j] > 0.f ? acc[r] : 0.f;
            if (dz1) { dz1[b * kH + j] = g; dz2[b * kH + j] = z2[r][j]; }
        }
        z1[r][j] = g;
    }
}

__global__ void __launch_bounds__(kH) sacc_critic_bwd_kernel(CriticBwdParams P) {
    __shared__ float z2[kRows][kH];
    __shared__ float z1[kRows][kH];
    const int net = blockIdx.y;
    const int K = P.obs_dim + P.D;
    const int64_t r0 = (int64_t)blockIdx.x * kRows;
    const float* p = P.params + net * P.net_stride;
    const MlpOff o(K, 1);
    float dq[kRows];
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
        const int64_t b = r0 + r;
        float d = 0.f;
        if (b < P.B) {
            if (P.dq) {
                d = P.dq[net * P.B + b];
            } else if (!P.q) {
                d = -P.inv_b;
            } else {
                const float q1 = P.q[b], q2 = P.q[P.B + b];
                const float mine = net == 0 ? q1 : q2, other = net == 0 ? q2 : q1;
                const float gm = -P.inv_b;
                d = mine == other ? __fmul_rn(gm, 0.5f) : (mine > other ? 0.f : gm);   // minimum's backward
            }
        }
        dq[r] = d;
    }
    const int64_t at = (int64_t)net * P.B * kH;
    critic_trunk_bwd(p, o, dq, P.h1 + at, P.h2 + at, P.dz1 ? P.dz1 + at : nullptr, P.dz1 ? P.dz2 + at : nullptr, z2,
                     z1, P.B, r0);
    if (!P.dact) return;
    __syncthreads();
    for (int i = threadIdx.x; i < kRows * P.D; i += kH) {
        const int r = i / P.D, c = i - r * P.D;
        const int64_t b = r0 + r;
        if (b >= P.B) continue;
        const float* w = p + o.w1 + P.obs_dim + c;
        float s = 0.f;
        for (int k = 0; k < kH; ++k) s = fmaf(__ldg(w + (int64_t)k * K), z1[r][k], s);
        P.dact[((int64_t)net * P.B + b) * P.D + c] = s;
    }
}

// ------------------------------------------------------------ one-critic loss + critic data backward (DDPG)
// y = r + ((1 - d) gamma) q_next and dq = (2 / B)(q - y) for the CTA's rows (threads 0..kRows-1, in the twin loss's
// rounding order), then the critic trunk backward of critic_trunk_bwd on the one network.  The last block writes
// stats[0..1] = mean q (losses/qf1_values) and qf1_loss.
struct DdpgLossBwdParams {
    const float* params;
    int64_t B; int obs_dim, D;
    const float* q_next; const float* q;                                   // [B] each
    const float* rewards; const float* dones; int64_t ld_rd; const int64_t* rows;
    float gamma, two_over_b;
    const float* h1; const float* h2;                                      // [B, 256] each
    float* y; float* dq; float* dz1; float* dz2;                           // [B], [B], [B, 256] x2
    float* stats; float* partials; unsigned int* ticket;
};

__global__ void __launch_bounds__(kH) ddpg_critic_loss_bwd_kernel(DdpgLossBwdParams P) {
    __shared__ float z2[kRows][kH];
    __shared__ float z1[kRows][kH];
    __shared__ float dqs[kRows];
    __shared__ float red[32];
    __shared__ bool is_last;
    const int64_t r0 = (int64_t)blockIdx.x * kRows;
    float v[2] = {0.f, 0.f};
    if (threadIdx.x < kRows) {
        const int64_t b = r0 + threadIdx.x;
        float d = 0.f;
        if (b < P.B) {
            const int64_t ri = (P.rows ? P.rows[b] : b) * P.ld_rd;
            const float y = __fadd_rn(P.rewards[ri], __fmul_rn(__fmul_rn(__fsub_rn(1.f, P.dones[ri]), P.gamma), P.q_next[b]));
            const float q = P.q[b];
            const float e = __fsub_rn(q, y);
            v[0] = q;
            v[1] = __fmul_rn(e, e);
            if (P.y) P.y[b] = y;
            d = __fmul_rn(P.two_over_b, e);                             // F.mse_loss backward: (2 / B) (input - target)
            P.dq[b] = d;
        }
        dqs[threadIdx.x] = d;
    }
    __syncthreads();
    float dq[kRows];
#pragma unroll
    for (int r = 0; r < kRows; ++r) dq[r] = dqs[r];
    critic_trunk_bwd(P.params, MlpOff(P.obs_dim + P.D, 1), dq, P.h1, P.h2, P.dz1, P.dz2, z2, z1, P.B, r0);
    if (!fold<2>(v, P.partials, P.ticket, red, &is_last)) return;
    if (threadIdx.x == 0) {
        const float b = (float)P.B;
        P.stats[0] = __fdiv_rn(v[0], b);                                // losses/qf1_values
        P.stats[1] = __fdiv_rn(v[1], b);                                // losses/qf1_loss
    }
}

// ------------------------------------------------------------------------------ actor loss + actor data backward
// The gradient of actor_loss = mean(alpha * log_pi - min(q1_pi, q2_pi)) through the tanh-Gaussian head to d mean and
// d raw_logstd (dhead [B, 2D]), restating autograd's chain through Normal.rsample / Normal.log_prob / tanh / log step by
// step, then back through fc2 and fc1 to dz2 and dz1.  The last block writes losses/actor_loss.
struct ActorBwdParams {
    const float* params;
    int64_t B; int obs_dim, D;
    const float* head; const float* eps; const float* scale; const float* dact;   // [B,2D], [B,D], [D], [2,B,D]
    const float* q; const float* log_pi; const float* alpha; float inv_b;
    const float* h1; const float* h2;
    float* dhead; float* dz1; float* dz2;
    float* stats; float* partials; unsigned int* ticket;
};

__device__ __forceinline__ void tanh_gauss_bwd(float m, float raw, float e, float sc, float g, float dpi, float* dm,
                                               float* draw) {
    // forward, as in sacc_actor_fwd_kernel
    const float t = tanhf(raw);
    const float ls = __fadd_rn(-5.f, __fmul_rn(3.5f, __fadd_rn(t, 1.f)));
    const float sd = expf(ls);
    const float x = __fadd_rn(m, __fmul_rn(e, sd));
    const float y = tanhf(x);
    const float u = __fsub_rn(x, m);
    const float nn = -__fmul_rn(u, u);
    const float var = __fmul_rn(sd, sd);
    const float den = __fmul_rn(2.f, var);
    const float qv = __fdiv_rn(nn, den);
    const float w2 = __fadd_rn(__fmul_rn(sc, __fsub_rn(1.f, __fmul_rn(y, y))), 1e-6f);
    // log_prob -= log(scale * (1 - y^2) + 1e-6): the correction's path to y
    const float g_w = __fdiv_rn(-g, w2);
    const float g_ysq = -__fmul_rn(g_w, sc);
    const float g_y = __fadd_rn(__fmul_rn(dpi, sc), __fmul_rn(g_ysq, __fmul_rn(2.f, y)));
    // Normal.log_prob: -(u^2) / (2 var) - log(scale) - c
    const float g_nn = __fdiv_rn(g, den);
    const float g_den = -__fmul_rn(g, __fdiv_rn(qv, den));
    const float g_u = __fmul_rn(-g_nn, __fmul_rn(2.f, u));
    const float g_std_var = __fmul_rn(__fmul_rn(g_den, 2.f), __fmul_rn(2.f, sd));
    const float g_std_log = __fdiv_rn(-g, sd);
    // x = loc + eps * scale, y = tanh(x), u = x - loc
    const float g_x = __fadd_rn(__fmul_rn(g_y, __fsub_rn(1.f, __fmul_rn(y, y))), g_u);
    *dm = __fsub_rn(g_x, g_u);
    const float g_std = __fadd_rn(__fadd_rn(__fmul_rn(g_x, e), g_std_var), g_std_log);
    const float g_t = __fmul_rn(__fmul_rn(g_std, sd), 3.5f);
    *draw = __fmul_rn(g_t, __fsub_rn(1.f, __fmul_rn(t, t)));
}

// From the head gradient dh [kRows][ncols] of the CTA's rows back through the trunk: dz2 = relu'(h2) * W_head^T dh, then
// dz1 = relu'(h1) * W2^T dz2 (both [B, 256]); head column c < D is row c of w3, c >= D row c - D of w4.
__device__ __forceinline__ void actor_trunk_bwd(const float* p, const MlpOff& o, int D, int ncols,
                                                const float (*dh)[2 * kSacMaxD], float (*z2)[kH], const float* h1,
                                                const float* h2, float* dz1, float* dz2, int64_t B, int64_t r0) {
    const int j = threadIdx.x;
    for (int r = 0; r < kRows; ++r) {
        const int64_t b = r0 + r;
        float s = 0.f;
        if (b < B) {
            for (int c = 0; c < ncols; ++c) {
                const float w = c < D ? __ldg(p + o.w3 + (int64_t)c * kH + j) : __ldg(p + o.w4 + (int64_t)(c - D) * kH + j);
                s = fmaf(w, dh[r][c], s);
            }
            s = h2[b * kH + j] > 0.f ? s : 0.f;
            dz2[b * kH + j] = s;
        }
        z2[r][j] = s;
    }
    __syncthreads();
    float acc[kRows];
#pragma unroll
    for (int r = 0; r < kRows; ++r) acc[r] = 0.f;
    for (int i = 0; i < kH; ++i) {
        const float w = __ldg(p + o.w2 + (int64_t)i * kH + j);
#pragma unroll
        for (int r = 0; r < kRows; ++r) acc[r] = fmaf(w, z2[r][i], acc[r]);
    }
    for (int r = 0; r < kRows; ++r) {
        const int64_t b = r0 + r;
        if (b < B) dz1[b * kH + j] = h1[b * kH + j] > 0.f ? acc[r] : 0.f;
    }
}

__global__ void __launch_bounds__(kH) sacc_actor_bwd_kernel(ActorBwdParams P) {
    __shared__ float dh[kRows][2 * kSacMaxD];
    __shared__ float z2[kRows][kH];
    __shared__ float red[32];
    __shared__ bool is_last;
    const int D = P.D;
    const int64_t r0 = (int64_t)blockIdx.x * kRows;
    const float alpha = __ldg(P.alpha);
    const float g = __fmul_rn(P.inv_b, alpha);                  // d actor_loss / d log_pi
    for (int i = threadIdx.x; i < kRows * D; i += kH) {
        const int r = i / D, d = i - r * D;
        const int64_t b = r0 + r;
        float dm = 0.f, dr = 0.f;
        if (b < P.B) {
            const float dpi = __fadd_rn(P.dact[b * D + d], P.dact[(P.B + b) * D + d]);
            tanh_gauss_bwd(P.head[b * 2 * D + d], P.head[b * 2 * D + D + d], P.eps[b * D + d], P.scale[d], g, dpi, &dm,
                           &dr);
            P.dhead[b * 2 * D + d] = dm;
            P.dhead[b * 2 * D + D + d] = dr;
        }
        dh[r][d] = dm;
        dh[r][D + d] = dr;
    }
    __syncthreads();
    actor_trunk_bwd(P.params, MlpOff(P.obs_dim, D), D, 2 * D, dh, z2, P.h1, P.h2, P.dz1, P.dz2, P.B, r0);
    // losses/actor_loss = ((alpha * log_pi) - min_qf_pi).mean()
    float v[1] = {0.f};
    if (threadIdx.x < kRows && r0 + threadIdx.x < P.B) {
        const int64_t b = r0 + threadIdx.x;
        v[0] = __fsub_rn(__fmul_rn(alpha, P.log_pi[b]), min_nan(P.q[b], P.q[P.B + b]));
    }
    if (!fold<1>(v, P.partials, P.ticket, red, &is_last)) return;
    if (threadIdx.x == 0) P.stats[0] = __fdiv_rn(v[0], (float)P.B);
}

// ----------------------------------------------------------- deterministic actor loss + data backward (TD3)
// actor_loss = -mean(qf1(obs, actor(obs))): dact [B, D] is qf1's gradient w.r.t. the action (dq = -1/B).  Through
// x * action_scale + action_bias and tanh: dz = (dact * scale) * (1 - y^2), autograd's mul backward then tanh_backward;
// then fc_mu, fc2 and fc1 backward.  The last block writes losses/actor_loss.
struct Td3ActorBwdParams {
    const float* params;
    int64_t B; int obs_dim, D;
    const float* y; const float* scale; const float* dact; const float* q;    // [B,D], [D], [B,D], [B]
    const float* h1; const float* h2;
    float* dhead; float* dz1; float* dz2;                                     // [B,D], [B,256] x2
    float* stats; float* partials; unsigned int* ticket;
};

__global__ void __launch_bounds__(kH) td3_actor_bwd_kernel(Td3ActorBwdParams P) {
    __shared__ float dh[kRows][2 * kSacMaxD];
    __shared__ float z2[kRows][kH];
    __shared__ float red[32];
    __shared__ bool is_last;
    const int D = P.D;
    const int64_t r0 = (int64_t)blockIdx.x * kRows;
    for (int i = threadIdx.x; i < kRows * D; i += kH) {
        const int r = i / D, d = i - r * D;
        const int64_t b = r0 + r;
        float dz = 0.f;
        if (b < P.B) {
            const float y = P.y[b * D + d];
            dz = __fmul_rn(__fmul_rn(P.dact[b * D + d], P.scale[d]), __fsub_rn(1.f, __fmul_rn(y, y)));
            P.dhead[b * D + d] = dz;
        }
        dh[r][d] = dz;
    }
    __syncthreads();
    actor_trunk_bwd(P.params, MlpOff(P.obs_dim, D), D, D, dh, z2, P.h1, P.h2, P.dz1, P.dz2, P.B, r0);
    // losses/actor_loss = -qf1(...).mean()
    float v[1] = {0.f};
    if (threadIdx.x < kRows && r0 + threadIdx.x < P.B) v[0] = P.q[r0 + threadIdx.x];
    if (!fold<1>(v, P.partials, P.ticket, red, &is_last)) return;
    if (threadIdx.x == 0) P.stats[0] = -__fdiv_rn(v[0], (float)P.B);
}

// ------------------------------------------------------------------------------------------- weight gradients
// Up to kMaxJobs layers: dW[n][k] = sum_b dz[b][n] x[b][k], db[n] = sum_b dz[b][n], sequentially over b.  A CTA owns
// a 32 x 32 tile of [dW | db] (the bias is the column k = K with x = 1) and walks the rows in chunks of 32.
constexpr int kMaxJobs = 8;
constexpr int kWT = 32;

struct WgradJob {
    const float* dz; int64_t ld_dz; const float* x; int64_t ld_x; int N, K; float* dw; float* db; int tiles_k, tile0;
};
struct WgradParams { WgradJob job[kMaxJobs]; int njobs; int64_t B; };

__global__ void __launch_bounds__(kH) sacc_wgrad_kernel(const WgradParams P) {
    __shared__ float zs[kWT][kWT + 1];
    __shared__ float xs[kWT][kWT + 1];
    int jb = 0;
    while (jb + 1 < P.njobs && (int)blockIdx.x >= P.job[jb + 1].tile0) ++jb;
    const WgradJob& J = P.job[jb];
    const int tile = blockIdx.x - J.tile0;
    const int n0 = (tile / J.tiles_k) * kWT, k0 = (tile % J.tiles_k) * kWT;
    const int tn = threadIdx.x >> 3, tk = (threadIdx.x & 7) * 4;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int64_t b0 = 0; b0 < P.B; b0 += kWT) {
        for (int i = threadIdx.x; i < kWT * kWT; i += kH) {
            const int r = i / kWT, c = i - r * kWT;
            const int64_t b = b0 + r;
            const bool ok = b < P.B;
            zs[r][c] = ok && n0 + c < J.N ? J.dz[b * J.ld_dz + n0 + c] : 0.f;
            const int k = k0 + c;
            xs[r][c] = !ok || k > J.K ? 0.f : (k == J.K ? 1.f : J.x[b * J.ld_x + k]);
        }
        __syncthreads();
        const int rn = (int)(P.B - b0 < kWT ? P.B - b0 : kWT);
        for (int r = 0; r < rn; ++r) {
            const float z = zs[r][tn];
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[c] = fmaf(z, xs[r][tk + c], acc[c]);
        }
        __syncthreads();
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

// ------------------------------------------------------------------------------------------------ soft update
__global__ void sacc_soft_update_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t n, float tau,
                                        float one_minus_tau) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = __fadd_rn(__fmul_rn(tau, src[i]), __fmul_rn(one_minus_tau, dst[i]));
}

// The forward kernels stage [kRows][in + 512] floats: up to 49152 B of dynamic shared memory at in = 1024, which with
// the actor's static arrays exceeds the default 48 KB window.  Opt the three kernels in once per device.
static int sacc_opt_in_smem() {
    static bool done[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64)
        return fail(B200RL_ERR_CUDA, "sac_continuous: cudaGetDevice failed");
    if (done[dev]) return 0;
    const int bytes = kRows * (kSacMaxIn + 2 * kH) * (int)sizeof(float);
    if (cudaFuncSetAttribute(sacc_critic_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess ||
        cudaFuncSetAttribute(sacc_actor_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess ||
        cudaFuncSetAttribute(td3_actor_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess)
        return fail(B200RL_ERR_CUDA, "sac_continuous: cudaFuncSetAttribute(MaxDynamicSharedMemorySize, %d)", bytes);
    done[dev] = true;
    return 0;
}

}  // namespace b200rl

#define SACC_SHAPES(what, in)                                                                                          \
    B200RL_REQUIRE(B >= 1 && B <= 8192, what ": B=%lld outside [1, 8192]", (long long)B);                               \
    B200RL_REQUIRE(act_dim >= 1 && act_dim <= b200rl::kSacMaxD, what ": act_dim=%d outside [1, %d]", act_dim,           \
                   b200rl::kSacMaxD);                                                                                   \
    B200RL_REQUIRE(obs_dim >= 1 && obs_dim + act_dim <= b200rl::kSacMaxIn,                                              \
                   what ": obs_dim + act_dim = %d outside [2, %d]", obs_dim + act_dim, b200rl::kSacMaxIn)

#define SACC_ALIGNED(what, ...)                                                                                        \
    do {                                                                                                               \
        const void* ps_[] = {__VA_ARGS__};                                                                             \
        for (const void* p_ : ps_) B200RL_REQUIRE(b200rl::aligned(p_, 4), what ": misaligned pointer");               \
    } while (0)

// Network kinds of b200rl_sacc_param_count / b200rl_sacc_wgrad_f32 (include/b200rl.h).
enum { kSaccActor = 0, kSaccCritic = 1, kTd3Actor = 2 };

extern "C" int64_t b200rl_sacc_param_count(int obs_dim, int act_dim, int critic) {
    if (obs_dim < 1 || act_dim < 1 || act_dim > b200rl::kSacMaxD || obs_dim + act_dim > b200rl::kSacMaxIn) return -1;
    if (critic < kSaccActor || critic > kTd3Actor) return -1;
    const int64_t in = critic == kSaccCritic ? obs_dim + act_dim : obs_dim;
    const int64_t H = b200rl::kH, D = act_dim;
    const int64_t head = critic == kSaccCritic ? H + 1 : critic == kTd3Actor ? D * H + D : 2 * (D * H + D);
    return H * in + H + H * H + H + head;
}

extern "C" size_t b200rl_sacc_workspace_bytes(int64_t B) {
    if (B < 1) return 0;
    return 16 + (size_t)b200rl::ceil_div(B, b200rl::kRows) * 4 * sizeof(float);
}

extern "C" int b200rl_sacc_critic_fwd_f32(const float* params, int64_t net_stride, const float* obs, int64_t ld_obs,
                                          const int64_t* obs_rows, const float* act, int64_t ld_act, const int64_t* act_rows,
                                          int64_t B, int obs_dim, int act_dim, float* q, float* keep_x, float* keep_h1,
                                          float* keep_h2, void* stream) {
    using namespace b200rl;
    SACC_SHAPES("sacc_critic_fwd", obs_dim + act_dim);
    B200RL_REQUIRE(params && obs && act && q, "sacc_critic_fwd: null pointer");
    B200RL_REQUIRE((keep_h1 == nullptr) == (keep_h2 == nullptr), "sacc_critic_fwd: keep_h1 and keep_h2 go together");
    B200RL_REQUIRE(ld_obs >= obs_dim && ld_act >= act_dim, "sacc_critic_fwd: bad strides");
    B200RL_REQUIRE(net_stride == 0 || net_stride >= b200rl_sacc_param_count(obs_dim, act_dim, 1),
                   "sacc_critic_fwd: net_stride too small");
    SACC_ALIGNED("sacc_critic_fwd", params, obs, act, q, keep_x, keep_h1, keep_h2);
    B200RL_REQUIRE(aligned(obs_rows, 8) && aligned(act_rows, 8), "sacc_critic_fwd: misaligned rows");
    cudaStream_t s = (cudaStream_t)stream;
    const int K = obs_dim + act_dim;
    ProfScope ps(s, "sacc_critic_fwd", 4.0 * B * kH * (K + kH + 1), 0);
    CriticFwdParams P{params, net_stride, obs, ld_obs, obs_rows, act, ld_act, act_rows, B, obs_dim, act_dim, q, keep_x,
                      keep_h1, keep_h2};
    if (int rc = sacc_opt_in_smem()) return rc;
    const size_t smem = (size_t)kRows * (K + 2 * kH) * sizeof(float);
    sacc_critic_fwd_kernel<<<dim3((unsigned)ceil_div(B, kRows), net_stride ? 2 : 1), kH, smem, s>>>(P);
    return check_launch("sacc_critic_fwd");
}

extern "C" int b200rl_sacc_actor_fwd_f32(const float* params, const float* obs, int64_t ld_obs, const int64_t* rows,
                                         int64_t B, int obs_dim, int act_dim, const float* eps, const float* scale,
                                         const float* bias, float* action, float* log_pi, float* mean_out,
                                         float* mean_logstd, float* keep_x, float* keep_h1, float* keep_h2,
                                         float* keep_head, int temperature, double target_entropy, float* alpha,
                                         float* log_alpha, float* exp_avg, float* exp_avg_sq, const float* step_scalars,
                                         double beta1, double beta2, double adam_eps, float* stats, void* workspace,
                                         size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    SACC_SHAPES("sacc_actor_fwd", obs_dim);
    B200RL_REQUIRE(params && obs && scale && bias, "sacc_actor_fwd: null pointer");
    B200RL_REQUIRE(!(action || log_pi || temperature) || eps, "sacc_actor_fwd: sampling needs eps");
    B200RL_REQUIRE((keep_h1 == nullptr) == (keep_h2 == nullptr), "sacc_actor_fwd: keep_h1 and keep_h2 go together");
    B200RL_REQUIRE(ld_obs >= obs_dim, "sacc_actor_fwd: bad strides");
    SACC_ALIGNED("sacc_actor_fwd", params, obs, eps, scale, bias, action, log_pi, mean_out, mean_logstd, keep_x, keep_h1,
                 keep_h2, keep_head, alpha, log_alpha, exp_avg, exp_avg_sq, step_scalars, stats);
    B200RL_REQUIRE(aligned(rows, 8), "sacc_actor_fwd: misaligned rows");
    if (temperature) {
        B200RL_REQUIRE(alpha && log_alpha && exp_avg && exp_avg_sq && step_scalars && stats,
                       "sacc_actor_fwd: the temperature step needs alpha, log_alpha, its Adam moments, the step scalars "
                       "and stats");
        B200RL_REQUIRE(workspace && aligned(workspace, 16), "sacc_actor_fwd: workspace null or misaligned");
        if (workspace_bytes < b200rl_sacc_workspace_bytes(B))
            return fail(B200RL_ERR_WORKSPACE, "sacc_actor_fwd: workspace %zu < %zu", workspace_bytes,
                        b200rl_sacc_workspace_bytes(B));
    }
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "sacc_actor_fwd", 2.0 * B * kH * (obs_dim + kH + 2 * act_dim), 0);
    unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
    float* partials = workspace ? reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16) : nullptr;
    ActorFwdParams P{params, obs, ld_obs, rows, B, obs_dim, act_dim, eps, scale, bias, action, log_pi, mean_out,
                     mean_logstd, keep_x, keep_h1, keep_h2, keep_head, temperature != 0, (float)target_entropy,
                     (float)(1.0 / (double)B), (float)(1.0 - beta1), (float)beta2,
                     (float)(1.0 - beta2), (float)adam_eps, alpha, log_alpha, exp_avg, exp_avg_sq, step_scalars, stats,
                     partials, ticket};
    if (int rc = sacc_opt_in_smem()) return rc;
    const size_t smem = (size_t)kRows * (obs_dim + 2 * kH) * sizeof(float);
    sacc_actor_fwd_kernel<<<(unsigned)ceil_div(B, kRows), kH, smem, s>>>(P);
    return check_launch("sacc_actor_fwd");
}

extern "C" int b200rl_sacc_critic_loss_f32(const float* q_next, const float* next_logpi, const float* q,
                                           const float* rewards, const float* dones, int64_t ld_rd, const int64_t* rows,
                                           const float* alpha, int64_t B, double gamma, float* y, float* dq, float* stats,
                                           void* workspace, size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(B >= 1 && B <= 8192, "sacc_critic_loss: B=%lld outside [1, 8192]", (long long)B);
    B200RL_REQUIRE(q_next && q && rewards && dones && dq && stats, "sacc_critic_loss: null pointer");
    B200RL_REQUIRE(!next_logpi || alpha, "sacc_critic_loss: next_logpi needs alpha");
    B200RL_REQUIRE(ld_rd >= 1, "sacc_critic_loss: bad strides");
    SACC_ALIGNED("sacc_critic_loss", q_next, next_logpi, q, rewards, dones, alpha, y, dq, stats);
    B200RL_REQUIRE(aligned(rows, 8), "sacc_critic_loss: misaligned rows");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "sacc_critic_loss: workspace null or misaligned");
    if (workspace_bytes < b200rl_sacc_workspace_bytes(B))
        return fail(B200RL_ERR_WORKSPACE, "sacc_critic_loss: workspace %zu < %zu", workspace_bytes,
                    b200rl_sacc_workspace_bytes(B));
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "sacc_critic_loss", 20.0 * B, 0);
    CriticLossParams P{q_next, next_logpi, q, rewards, dones, ld_rd, rows, alpha, B, (float)gamma, (float)(2.0 / (double)B), y,
                       dq, stats, reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16),
                       reinterpret_cast<unsigned int*>(workspace)};
    sacc_critic_loss_kernel<<<(unsigned)ceil_div(B, kLossThreads), kLossThreads, 0, s>>>(P);
    return check_launch("sacc_critic_loss");
}

extern "C" int b200rl_sacc_critic_bwd_f32(const float* params, int64_t net_stride, int64_t B, int obs_dim, int act_dim,
                                          const float* dq, const float* q, const float* h1, const float* h2, float* dz1,
                                          float* dz2, float* dact, void* stream) {
    using namespace b200rl;
    SACC_SHAPES("sacc_critic_bwd", obs_dim + act_dim);
    B200RL_REQUIRE(params && h1 && h2, "sacc_critic_bwd: null pointer");
    // single: the one-network actor step (net_stride 0, neither dq nor q)
    const bool single = !dq && !q && net_stride == 0;
    B200RL_REQUIRE(dq ? (dz1 && dz2 && !dact) : ((q || single) && dact && !dz1 && !dz2),
                   "sacc_critic_bwd: give dq with dz1 / dz2 (critic step), q with dact (actor step) or, with "
                   "net_stride 0, dact alone (single-network actor step)");
    B200RL_REQUIRE(net_stride == 0 || net_stride >= b200rl_sacc_param_count(obs_dim, act_dim, 1),
                   "sacc_critic_bwd: net_stride too small");
    SACC_ALIGNED("sacc_critic_bwd", params, dq, q, h1, h2, dz1, dz2, dact);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "sacc_critic_bwd", 4.0 * B * kH * (kH + 1 + (dact ? act_dim : 0)), 0);
    CriticBwdParams P{params, net_stride, B, obs_dim, act_dim, dq, q, (float)(1.0 / (double)B), h1, h2, dz1, dz2, dact};
    sacc_critic_bwd_kernel<<<dim3((unsigned)ceil_div(B, kRows), single ? 1 : 2), kH, 0, s>>>(P);
    return check_launch("sacc_critic_bwd");
}

extern "C" int b200rl_ddpg_critic_loss_bwd_f32(const float* params, int64_t B, int obs_dim, int act_dim,
                                               const float* q_next, const float* q, const float* rewards,
                                               const float* dones, int64_t ld_rd, const int64_t* rows, double gamma,
                                               const float* h1, const float* h2, float* y, float* dq, float* dz1,
                                               float* dz2, float* stats, void* workspace, size_t workspace_bytes,
                                               void* stream) {
    using namespace b200rl;
    SACC_SHAPES("ddpg_critic_loss_bwd", obs_dim + act_dim);
    B200RL_REQUIRE(params && q_next && q && rewards && dones && h1 && h2 && dq && dz1 && dz2 && stats,
                   "ddpg_critic_loss_bwd: null pointer");
    B200RL_REQUIRE(ld_rd >= 1, "ddpg_critic_loss_bwd: bad strides");
    SACC_ALIGNED("ddpg_critic_loss_bwd", params, q_next, q, rewards, dones, h1, h2, y, dq, dz1, dz2, stats);
    B200RL_REQUIRE(aligned(rows, 8), "ddpg_critic_loss_bwd: misaligned rows");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "ddpg_critic_loss_bwd: workspace null or misaligned");
    if (workspace_bytes < b200rl_sacc_workspace_bytes(B))
        return fail(B200RL_ERR_WORKSPACE, "ddpg_critic_loss_bwd: workspace %zu < %zu", workspace_bytes,
                    b200rl_sacc_workspace_bytes(B));
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "ddpg_critic_loss_bwd", 20.0 * B + 2.0 * B * kH * (kH + 1), 0);
    DdpgLossBwdParams P{params, B, obs_dim, act_dim, q_next, q, rewards, dones, ld_rd, rows, (float)gamma,
                        (float)(2.0 / (double)B), h1, h2, y, dq, dz1, dz2, stats,
                        reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16),
                        reinterpret_cast<unsigned int*>(workspace)};
    ddpg_critic_loss_bwd_kernel<<<(unsigned)ceil_div(B, kRows), kH, 0, s>>>(P);
    return check_launch("ddpg_critic_loss_bwd");
}

extern "C" int b200rl_sacc_actor_bwd_f32(const float* params, int64_t B, int obs_dim, int act_dim, const float* head,
                                         const float* eps, const float* scale, const float* dact, const float* q,
                                         const float* log_pi, const float* alpha, const float* h1, const float* h2,
                                         float* dhead, float* dz1, float* dz2, float* stats, void* workspace,
                                         size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    SACC_SHAPES("sacc_actor_bwd", obs_dim);
    B200RL_REQUIRE(params && head && eps && scale && dact && q && log_pi && alpha && h1 && h2 && dhead && dz1 && dz2 &&
                   stats, "sacc_actor_bwd: null pointer");
    SACC_ALIGNED("sacc_actor_bwd", params, head, eps, scale, dact, q, log_pi, alpha, h1, h2, dhead, dz1, dz2, stats);
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "sacc_actor_bwd: workspace null or misaligned");
    if (workspace_bytes < b200rl_sacc_workspace_bytes(B))
        return fail(B200RL_ERR_WORKSPACE, "sacc_actor_bwd: workspace %zu < %zu", workspace_bytes,
                    b200rl_sacc_workspace_bytes(B));
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "sacc_actor_bwd", 2.0 * B * kH * (kH + 2 * act_dim), 0);
    ActorBwdParams P{params, B, obs_dim, act_dim, head, eps, scale, dact, q, log_pi, alpha, (float)(1.0 / (double)B), h1,
                     h2, dhead, dz1, dz2, stats, reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16),
                     reinterpret_cast<unsigned int*>(workspace)};
    sacc_actor_bwd_kernel<<<(unsigned)ceil_div(B, kRows), kH, 0, s>>>(P);
    return check_launch("sacc_actor_bwd");
}

extern "C" int b200rl_sacc_wgrad_f32(int critic, int64_t B, int obs_dim, int act_dim, const float* x, const float* h1,
                                     const float* h2, const float* dz1, const float* dz2, const float* dout, float* grad,
                                     int64_t net_stride, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(critic >= kSaccActor && critic <= kTd3Actor, "sacc_wgrad: network kind %d outside [0, 2]", critic);
    SACC_SHAPES("sacc_wgrad", critic == kSaccCritic ? obs_dim + act_dim : obs_dim);
    B200RL_REQUIRE(x && h1 && h2 && dz1 && dz2 && dout && grad, "sacc_wgrad: null pointer");
    B200RL_REQUIRE(critic != kSaccCritic || net_stride == 0 ||
                   net_stride >= b200rl_sacc_param_count(obs_dim, act_dim, 1), "sacc_wgrad: net_stride too small");
    SACC_ALIGNED("sacc_wgrad", x, h1, h2, dz1, dz2, dout, grad);
    WgradParams P{};
    P.B = B;
    int t = 0;
    auto add = [&](const float* dz, int64_t ld_dz, const float* xx, int64_t ld_x, int N, int K, float* dw, float* db) {
        WgradJob& J = P.job[P.njobs++];
        J = WgradJob{dz, ld_dz, xx, ld_x, N, K, dw, db, (int)ceil_div(K + 1, kWT), t};
        t += (int)ceil_div(N, kWT) * J.tiles_k;
    };
    if (critic == kSaccCritic) {
        const int K = obs_dim + act_dim;
        const MlpOff o(K, 1);
        for (int n = 0; n < (net_stride ? 2 : 1); ++n) {              // net_stride 0: one critic (DDPG)
            float* g = grad + n * net_stride;
            const int64_t a = (int64_t)n * B * kH;
            add(dz1 + a, kH, x, K, kH, K, g + o.w1, g + o.b1);
            add(dz2 + a, kH, h1 + a, kH, kH, kH, g + o.w2, g + o.b2);
            add(dout + (int64_t)n * B, 1, h2 + a, kH, 1, kH, g + o.w3, g + o.b3);
        }
    } else if (critic == kSaccActor) {
        const MlpOff o(obs_dim, act_dim);
        add(dz1, kH, x, obs_dim, kH, obs_dim, grad + o.w1, grad + o.b1);
        add(dz2, kH, h1, kH, kH, kH, grad + o.w2, grad + o.b2);
        add(dout, 2 * act_dim, h2, kH, act_dim, kH, grad + o.w3, grad + o.b3);
        add(dout + act_dim, 2 * act_dim, h2, kH, act_dim, kH, grad + o.w4, grad + o.b4);
    } else {
        const MlpOff o(obs_dim, act_dim);
        add(dz1, kH, x, obs_dim, kH, obs_dim, grad + o.w1, grad + o.b1);
        add(dz2, kH, h1, kH, kH, kH, grad + o.w2, grad + o.b2);
        add(dout, act_dim, h2, kH, act_dim, kH, grad + o.w3, grad + o.b3);
    }
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "sacc_wgrad", 0, 0);
    sacc_wgrad_kernel<<<(unsigned)t, kH, 0, s>>>(P);
    return check_launch("sacc_wgrad");
}

extern "C" int b200rl_td3_actor_fwd_f32(const float* params, const float* obs, int64_t ld_obs, const int64_t* rows,
                                        int64_t B, int obs_dim, int act_dim, const float* scale, const float* bias,
                                        float* mu, float* keep_y, float* keep_x, float* keep_h1, float* keep_h2,
                                        const float* eps, double policy_noise, double noise_clip, double low,
                                        double high, float* smoothed, void* stream) {
    using namespace b200rl;
    SACC_SHAPES("td3_actor_fwd", obs_dim);
    B200RL_REQUIRE(params && obs && scale && bias, "td3_actor_fwd: null pointer");
    B200RL_REQUIRE((eps == nullptr) == (smoothed == nullptr), "td3_actor_fwd: eps and smoothed go together");
    B200RL_REQUIRE((keep_h1 == nullptr) == (keep_h2 == nullptr), "td3_actor_fwd: keep_h1 and keep_h2 go together");
    B200RL_REQUIRE(ld_obs >= obs_dim, "td3_actor_fwd: bad strides");
    B200RL_REQUIRE(!smoothed || (noise_clip >= 0.0 && low <= high), "td3_actor_fwd: noise_clip < 0 or low > high");
    SACC_ALIGNED("td3_actor_fwd", params, obs, scale, bias, mu, keep_y, keep_x, keep_h1, keep_h2, eps, smoothed);
    B200RL_REQUIRE(aligned(rows, 8), "td3_actor_fwd: misaligned rows");
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "td3_actor_fwd", 2.0 * B * kH * (obs_dim + kH + act_dim), 0);
    Td3ActorFwdParams P{params, obs, ld_obs, rows, B, obs_dim, act_dim, scale, bias, mu, keep_y, keep_x, keep_h1,
                        keep_h2, eps, (float)policy_noise, (float)noise_clip, (float)low, (float)high, smoothed};
    if (int rc = sacc_opt_in_smem()) return rc;
    const size_t smem = (size_t)kRows * (obs_dim + 2 * kH) * sizeof(float);
    td3_actor_fwd_kernel<<<(unsigned)ceil_div(B, kRows), kH, smem, s>>>(P);
    return check_launch("td3_actor_fwd");
}

extern "C" int b200rl_td3_actor_bwd_f32(const float* params, int64_t B, int obs_dim, int act_dim, const float* y,
                                        const float* scale, const float* dact, const float* q, const float* h1,
                                        const float* h2, float* dhead, float* dz1, float* dz2, float* stats,
                                        void* workspace, size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    SACC_SHAPES("td3_actor_bwd", obs_dim);
    B200RL_REQUIRE(params && y && scale && dact && q && h1 && h2 && dhead && dz1 && dz2 && stats,
                   "td3_actor_bwd: null pointer");
    SACC_ALIGNED("td3_actor_bwd", params, y, scale, dact, q, h1, h2, dhead, dz1, dz2, stats);
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "td3_actor_bwd: workspace null or misaligned");
    if (workspace_bytes < b200rl_sacc_workspace_bytes(B))
        return fail(B200RL_ERR_WORKSPACE, "td3_actor_bwd: workspace %zu < %zu", workspace_bytes,
                    b200rl_sacc_workspace_bytes(B));
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "td3_actor_bwd", 2.0 * B * kH * (kH + act_dim), 0);
    Td3ActorBwdParams P{params, B, obs_dim, act_dim, y, scale, dact, q, h1, h2, dhead, dz1, dz2, stats,
                        reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16),
                        reinterpret_cast<unsigned int*>(workspace)};
    td3_actor_bwd_kernel<<<(unsigned)ceil_div(B, kRows), kH, 0, s>>>(P);
    return check_launch("td3_actor_bwd");
}

extern "C" int b200rl_sacc_soft_update_f32(const float* src, float* dst, int64_t n, double tau, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(n >= 1, "sacc_soft_update: n must be >= 1");
    B200RL_REQUIRE(src && dst, "sacc_soft_update: null pointer");
    SACC_ALIGNED("sacc_soft_update", src, dst);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "sacc_soft_update", 3.0 * n, 12.0 * n);
    const int64_t blocks = ceil_div(n, 256) < 1184 ? ceil_div(n, 256) : 1184;
    sacc_soft_update_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dst, n, (float)tau, (float)(1.0 - tau));
    return check_launch("sacc_soft_update");
}
