// C51 distributional heads (cleanrl/c51_atari.py): the per-action softmax over atoms, the greedy action, and the
// categorical-projection cross-entropy loss with its gradient -- one block per row, one pass each.
//
// Numerics follow the reference's fp32 torch expressions operation by operation (separately rounded, no fused
// multiply-adds where torch rounds twice).  The projection accumulates target_pmfs exactly as CPU index_add_ does:
// every d_m_l in atom order, then every d_m_u in atom order.  Reductions are fixed-order (no float atomics).
#include "common.cuh"

namespace b200rl {

constexpr int kC51Threads = 256;          // 8 warps; one thread per atom in the loss (n_atoms <= 256)
constexpr int kC51MaxAtoms = 256;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Softmax statistics of one action's atom logits, computed by one warp: max and sum of exp(x - max).
__device__ __forceinline__ void warp_softmax_stats(const float* __restrict__ x, int Z, float& mx, float& sum) {
    const int lane = threadIdx.x & 31;
    float m = -INFINITY;
    for (int j = lane; j < Z; j += 32) m = fmaxf(m, x[j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < Z; j += 32) s += expf(x[j] - m);
    mx = m;
    sum = warp_sum(s);
}

// q[a] = sum_j softmax(x_a)_j * atoms_j for every action (one warp per action), then the first-max argmax.
// Returns the greedy action in *best (valid after the trailing __syncthreads).
__device__ void c51_q_row(const float* __restrict__ row, const float* __restrict__ atoms, int A, int Z, float* sq,
                          int* best) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int a = warp; a < A; a += nw) {
        const float* x = row + (int64_t)a * Z;
        float mx, sum;
        warp_softmax_stats(x, Z, mx, sum);
        float q = 0.f;
        for (int j = lane; j < Z; j += 32) q += __fmul_rn(__fdiv_rn(expf(x[j] - mx), sum), atoms[j]);
        q = warp_sum(q);
        if (lane == 0) sq[a] = q;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int b = 0; float bv = sq[0];
        for (int a = 1; a < A; ++a) if (sq[a] > bv) { bv = sq[a]; b = a; }
        *best = b;
    }
    __syncthreads();
}

struct C51ActParams {
    const float* logits; int64_t ld;
    const float* atoms; int64_t n; int A, Z;
    const int64_t* action_in;
    int64_t* action_out; float* q_out; float* pmf_out;
};

__global__ void __launch_bounds__(kC51Threads) c51_act_kernel(C51ActParams P) {
    extern __shared__ float sq[];              // [A]
    __shared__ int best;
    __shared__ float st[2];
    const int64_t i = blockIdx.x;
    const float* row = P.logits + i * P.ld;
    c51_q_row(row, P.atoms, P.A, P.Z, sq, &best);
    int a = best;
    if (P.action_in) {
        a = (int)P.action_in[i];
        a = a < 0 ? 0 : (a >= P.A ? P.A - 1 : a);
    }
    if (P.q_out) for (int k = threadIdx.x; k < P.A; k += blockDim.x) P.q_out[i * P.A + k] = sq[k];
    if (threadIdx.x == 0) P.action_out[i] = a;
    if (!P.pmf_out) return;
    const float* x = row + (int64_t)a * P.Z;
    if (threadIdx.x < 32) {
        float mx, sum;
        warp_softmax_stats(x, P.Z, mx, sum);
        if (threadIdx.x == 0) { st[0] = mx; st[1] = sum; }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < P.Z; j += blockDim.x)
        P.pmf_out[i * P.Z + j] = __fdiv_rn(expf(x[j] - st[0]), st[1]);
}

struct C51LossParams {
    const float* logits; int64_t ld;
    const float* next_logits; int64_t ldn;
    const float* atoms; const int64_t* actions; const float* rewards; const float* dones;
    int64_t B; int A, Z; float gamma, v_min, v_max;
    float* dlogits; int64_t ldd; float* stats; float* partials; unsigned int* ticket;
};

__global__ void __launch_bounds__(kC51Threads) c51_loss_kernel(C51LossParams P) {
    extern __shared__ float sq[];              // [A]
    __shared__ float tgt[kC51MaxAtoms], dml[kC51MaxAtoms], dmu[kC51MaxAtoms];
    __shared__ int sl[kC51MaxAtoms], su[kC51MaxAtoms];
    __shared__ float red[32], st[2];
    __shared__ int best;
    __shared__ bool is_last;
    const int64_t i = blockIdx.x;
    const int Z = P.Z, j = threadIdx.x;
    // ---- target network: greedy action and its pmf (c51_atari.py:234)
    const float* trow = P.next_logits + i * P.ldn;
    c51_q_row(trow, P.atoms, P.A, Z, sq, &best);
    const float* tx = trow + (int64_t)best * Z;
    if (threadIdx.x < 32) {
        float mx, sum;
        warp_softmax_stats(tx, Z, mx, sum);
        if (threadIdx.x == 0) { st[0] = mx; st[1] = sum; }
    }
    __syncthreads();
    // ---- projection terms (c51_atari.py:235-246)
    if (j < Z) {
        const float p = __fdiv_rn(expf(tx[j] - st[0]), st[1]);
        const float r = P.rewards[i], d = P.dones[i];
        const float atom = P.atoms[j];
        const float next_atom = __fadd_rn(r, __fmul_rn(__fmul_rn(P.gamma, atom), __fsub_rn(1.f, d)));
        const float tz = fminf(fmaxf(next_atom, P.v_min), P.v_max);
        const float delta_z = __fsub_rn(P.atoms[1], P.atoms[0]);
        const float b = __fdiv_rn(__fsub_rn(tz, P.v_min), delta_z);
        const float zmax = (float)(Z - 1);
        const float l = fminf(fmaxf(floorf(b), 0.f), zmax), u = fminf(fmaxf(ceilf(b), 0.f), zmax);
        dml[j] = __fmul_rn(__fsub_rn(__fadd_rn(u, l == u ? 1.f : 0.f), b), p);
        dmu[j] = __fmul_rn(__fsub_rn(b, l), p);
        sl[j] = (int)l; su[j] = (int)u;
        tgt[j] = 0.f;
    }
    __syncthreads();
    // index_add_ order: all lower neighbours, then all upper neighbours (c51_atari.py:248-250)
    if (threadIdx.x == 0) {
        for (int k = 0; k < Z; ++k) tgt[sl[k]] = __fadd_rn(tgt[sl[k]], dml[k]);
        for (int k = 0; k < Z; ++k) tgt[su[k]] = __fadd_rn(tgt[su[k]], dmu[k]);
    }
    // ---- online network: chosen action's pmf, clamped cross-entropy and its gradient (c51_atari.py:252-253)
    int a = (int)P.actions[i];
    a = a < 0 ? 0 : (a >= P.A ? P.A - 1 : a);
    const float* ox = P.logits + i * P.ld + (int64_t)a * Z;
    if (threadIdx.x < 32) {
        float mx, sum;
        warp_softmax_stats(ox, Z, mx, sum);
        if (threadIdx.x == 0) { st[0] = mx; st[1] = sum; }
    }
    __syncthreads();
    const float lo = 1e-5f, hi = (float)(1.0 - 1e-5);
    const float invB = __fdiv_rn(1.f, (float)P.B);
    float p = 0.f, term = 0.f, qv = 0.f, g = 0.f;
    if (j < Z) {
        p = __fdiv_rn(expf(ox[j] - st[0]), st[1]);
        const float pc = fminf(fmaxf(p, lo), hi);
        term = __fmul_rn(tgt[j], logf(pc));
        qv = __fmul_rn(p, P.atoms[j]);
        // d/dp of -(target * log(clamp(p))).sum() / B; clamp passes the gradient on its closed interval
        g = (p >= lo && p <= hi) ? __fdiv_rn(__fmul_rn(-invB, tgt[j]), pc) : 0.f;
    }
    const float row_loss = -block_sum(term, red);
    const float row_q = block_sum(qv, red);
    const float dot = block_sum(__fmul_rn(g, p), red);
    float* drow = P.dlogits + i * P.ldd;
    for (int k = threadIdx.x; k < P.A * Z; k += blockDim.x) {
        if (k / Z != a) drow[k] = 0.f;
    }
    if (j < Z) drow[(int64_t)a * Z + j] = __fmul_rn(p, __fsub_rn(g, dot));
    // ---- stats: fixed-order fold of the per-row partials by the last block (ticket)
    if (threadIdx.x == 0) {
        P.partials[2 * i] = row_loss;
        P.partials[2 * i + 1] = row_q;
        __threadfence();
        is_last = (atomicAdd(P.ticket, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    float s0 = 0.f, s1 = 0.f;
    for (int64_t b = threadIdx.x; b < P.B; b += blockDim.x) { s0 += __ldcg(P.partials + 2 * b); s1 += __ldcg(P.partials + 2 * b + 1); }
    s0 = block_sum(s0, red);
    s1 = block_sum(s1, red);
    if (threadIdx.x == 0) {
        P.stats[0] = s0 / (float)P.B;      // losses/loss
        P.stats[1] = s1 / (float)P.B;      // losses/q_values: mean of (old_pmfs * atoms).sum(1)
        *P.ticket = 0;
    }
}

static size_t c51_q_smem(int A) { return (size_t)A * sizeof(float); }

}  // namespace b200rl

extern "C" int b200rl_c51_act_f32(const float* logits, int64_t ld, const float* atoms, int64_t n, int A, int n_atoms,
                                  const int64_t* action_in, int64_t* action_out, float* q_out, float* pmf_out,
                                  void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(n >= 0, "c51_act: negative n");
    B200RL_REQUIRE(n_atoms >= 2 && n_atoms <= kC51MaxAtoms, "c51_act: n_atoms=%d outside [2,%d]", n_atoms, kC51MaxAtoms);
    B200RL_REQUIRE(A >= 1 && A <= 4096, "c51_act: A=%d outside [1,4096]", A);
    B200RL_REQUIRE(ld >= (int64_t)A * n_atoms, "c51_act: ld %lld < A * n_atoms", (long long)ld);
    B200RL_REQUIRE(logits && atoms && action_out, "c51_act: null pointer");
    B200RL_REQUIRE(aligned(logits, 4) && aligned(atoms, 4) && aligned(action_out, 8) &&
                   (!action_in || aligned(action_in, 8)) && (!q_out || aligned(q_out, 4)) && (!pmf_out || aligned(pmf_out, 4)),
                   "c51_act: misaligned pointer");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(n <= 0x7fffffff, "c51_act: n too large");
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "c51_act", 0, (double)n * ((double)A * n_atoms * 4 + 4 * A + 4 * n_atoms + 8));
    C51ActParams P{logits, ld, atoms, n, A, n_atoms, action_in, action_out, q_out, pmf_out};
    c51_act_kernel<<<(unsigned)n, kC51Threads, c51_q_smem(A), s>>>(P);
    return check_launch("c51_act");
}

extern "C" size_t b200rl_c51_loss_workspace_bytes(int64_t B) {
    if (B < 0) return 0;
    return 16 + (size_t)(B > 0 ? B : 1) * 2 * sizeof(float);
}

extern "C" int b200rl_c51_loss_f32(const float* logits, int64_t ld, const float* next_logits, int64_t ld_next,
                                   const float* atoms, const int64_t* actions, const float* rewards, const float* dones,
                                   int64_t B, int A, int n_atoms, double gamma, double v_min, double v_max,
                                   float* dlogits, int64_t ld_d, float* stats,
                                   void* workspace, size_t workspace_bytes, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(B >= 1 && B <= 0x7fffffff, "c51_loss: B must be in [1, 2^31)");
    B200RL_REQUIRE(n_atoms >= 2 && n_atoms <= kC51MaxAtoms, "c51_loss: n_atoms=%d outside [2,%d]", n_atoms, kC51MaxAtoms);
    B200RL_REQUIRE(A >= 1 && A <= 4096, "c51_loss: A=%d outside [1,4096]", A);
    const int64_t w = (int64_t)A * n_atoms;
    B200RL_REQUIRE(ld >= w && ld_next >= w && ld_d >= w, "c51_loss: bad strides");
    B200RL_REQUIRE(logits && next_logits && atoms && actions && rewards && dones && dlogits && stats, "c51_loss: null pointer");
    B200RL_REQUIRE(aligned(logits, 4) && aligned(next_logits, 4) && aligned(atoms, 4) && aligned(actions, 8) &&
                   aligned(rewards, 4) && aligned(dones, 4) && aligned(dlogits, 4) && aligned(stats, 4),
                   "c51_loss: misaligned pointer");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "c51_loss: workspace null or misaligned");
    if (workspace_bytes < b200rl_c51_loss_workspace_bytes(B))
        return fail(B200RL_ERR_WORKSPACE, "c51_loss: workspace %zu < %zu", workspace_bytes, b200rl_c51_loss_workspace_bytes(B));
    cudaStream_t s = (cudaStream_t)stream;
    unsigned int* ticket = reinterpret_cast<unsigned int*>(workspace);
    float* partials = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 16);
    ProfScope ps(s, "c51_loss", 0, (double)B * (12.0 * w + 24));
    cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int), s);
    if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "c51_loss: memset: %s", cudaGetErrorString(e));
    C51LossParams P{logits, ld, next_logits, ld_next, atoms, actions, rewards, dones, B, A, n_atoms,
                    (float)gamma, (float)v_min, (float)v_max, dlogits, ld_d, stats, partials, ticket};
    c51_loss_kernel<<<(unsigned)B, kC51Threads, c51_q_smem(A), s>>>(P);
    return check_launch("c51_loss");
}
