// GAE reverse scan -- replaces the python loop cleanrl/ppo.py:218-231.
//
// Layout: rewards/values/dones/advantages/returns are f32 [T, N] with N (envs)
// contiguous, so consecutive threads = consecutive envs => every global access
// of a warp is one fully coalesced 128-B line.  Algorithmic traffic per launch:
// 3 reads + 2 writes of [T,N] f32 + next_value/next_done = 20*T*N + 8*N bytes.
//
// mode 0 (bit-exact): one thread per env walks t = T-1..0.  All loads of a time
// chunk are issued before the dependent recurrence runs (software prefetch,
// UNROLL deep), and every arithmetic op is an explicit *_rn intrinsic so nvcc
// cannot contract a*b+c into an FMA: the result is bit-identical to the
// reference's torch loop (separately rounded mul/add, ppo.py:229-230).
//
// mode 1 (chunked scan): the recurrence A[t] = delta[t] + c[t]*A[t+1] is affine,
// so a time chunk composes to A_first = B + P*A_in.  Thread (chunk c, env n)
// reduces its chunk to (P,B), the chunk carries are chained through shared
// memory (<= 31 steps), then every chunk re-walks its steps with the right
// carry-in.  Dependent chain: L + C + L instead of T.
#include "common.cuh"

namespace b200rl {

template <int UNROLL>
__global__ void __launch_bounds__(64) gae_seq_kernel(
    const float* __restrict__ rewards, const float* __restrict__ values, const float* __restrict__ dones,
    const float* __restrict__ next_value, const float* __restrict__ next_done,
    float* __restrict__ advantages, float* __restrict__ returns,
    int64_t T, int64_t N, float gamma, float gl) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float nv = next_value[n];
    float nd = next_done[n];
    float last = 0.f;
    int64_t t = T - 1;
    for (; t >= UNROLL - 1; t -= UNROLL) {
        float r[UNROLL], v[UNROLL], d[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int64_t o = (t - u) * N + n;
            r[u] = __ldg(rewards + o);
            v[u] = __ldg(values + o);
            d[u] = __ldg(dones + o);
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const float nnt = __fsub_rn(1.0f, nd);
            const float delta = __fsub_rn(__fadd_rn(r[u], __fmul_rn(__fmul_rn(gamma, nv), nnt)), v[u]);
            last = __fadd_rn(delta, __fmul_rn(__fmul_rn(gl, nnt), last));
            const int64_t o = (t - u) * N + n;
            advantages[o] = last;
            returns[o] = __fadd_rn(last, v[u]);
            nv = v[u];
            nd = d[u];
        }
    }
    for (; t >= 0; --t) {
        const int64_t o = t * N + n;
        const float r = rewards[o], v = values[o], d = dones[o];
        const float nnt = __fsub_rn(1.0f, nd);
        const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(__fmul_rn(gamma, nv), nnt)), v);
        last = __fadd_rn(delta, __fmul_rn(__fmul_rn(gl, nnt), last));
        advantages[o] = last;
        returns[o] = __fadd_rn(last, v);
        nv = v;
        nd = d;
    }
}

// blockDim = (32 envs, C chunks).  Chunk c covers t in [c*L, min(T,(c+1)*L)).
__global__ void gae_chunk_kernel(
    const float* __restrict__ rewards, const float* __restrict__ values, const float* __restrict__ dones,
    const float* __restrict__ next_value, const float* __restrict__ next_done,
    float* __restrict__ advantages, float* __restrict__ returns,
    int64_t T, int64_t N, int L, float gamma, float gl) {
    extern __shared__ float sm[];  // [C][32] P then [C][32] B
    const int C = blockDim.y;
    float* sP = sm;
    float* sB = sm + C * 32;
    const int c = threadIdx.y;
    const int64_t n = (int64_t)blockIdx.x * 32 + threadIdx.x;
    const bool live = n < N;
    const int64_t t0 = (int64_t)c * L;
    const int64_t t1 = (t0 + L < T) ? (t0 + L) : T;  // exclusive
    float P = 1.f, B = 0.f;
    if (live && t0 < T) {
        float nv, nd;
        if (t1 == T) { nv = next_value[n]; nd = next_done[n]; }
        else { nv = __ldg(values + t1 * N + n); nd = __ldg(dones + t1 * N + n); }
        for (int64_t t = t1 - 1; t >= t0; --t) {
            const int64_t o = t * N + n;
            const float r = __ldg(rewards + o), v = __ldg(values + o), d = __ldg(dones + o);
            const float nnt = 1.0f - nd;
            const float delta = r + gamma * nv * nnt - v;
            const float coef = gl * nnt;
            B = delta + coef * B;
            P = coef * P;
            nv = v;
            nd = d;
        }
    }
    sP[c * 32 + threadIdx.x] = P;
    sB[c * 32 + threadIdx.x] = B;
    __syncthreads();
    if (!live || t0 >= T) return;
    float last = 0.f;  // carry-in: advantage at t1 (0 beyond the rollout)
    for (int cc = C - 1; cc > c; --cc) last = sB[cc * 32 + threadIdx.x] + sP[cc * 32 + threadIdx.x] * last;
    float nv, nd;
    if (t1 == T) { nv = next_value[n]; nd = next_done[n]; }
    else { nv = __ldg(values + t1 * N + n); nd = __ldg(dones + t1 * N + n); }
    for (int64_t t = t1 - 1; t >= t0; --t) {
        const int64_t o = t * N + n;
        const float r = __ldg(rewards + o), v = __ldg(values + o), d = __ldg(dones + o);
        const float nnt = 1.0f - nd;
        const float delta = r + gamma * nv * nnt - v;
        last = delta + gl * nnt * last;
        advantages[o] = last;
        returns[o] = last + v;
        nv = v;
        nd = d;
    }
}

}  // namespace b200rl

extern "C" int b200rl_gae_f32(const float* rewards, const float* values, const float* dones,
                              const float* next_value, const float* next_done,
                              float* advantages, float* returns,
                              int64_t T, int64_t N, double gamma, double gae_lambda,
                              int mode, void* stream) {
    using namespace b200rl;
    B200RL_REQUIRE(T >= 0 && N >= 0, "gae: negative shape T=%lld N=%lld", (long long)T, (long long)N);
    if (T == 0 || N == 0) return B200RL_OK;
    B200RL_REQUIRE(rewards && values && dones && next_value && next_done && advantages && returns,
                   "gae: null pointer");
    B200RL_REQUIRE(mode == 0 || mode == 1, "gae: mode must be 0 (sequential) or 1 (chunked scan)");
    B200RL_REQUIRE(N <= (int64_t)2147483647 * 32, "gae: N too large");
    const float g = (float)gamma;
    const float gl = (float)(gamma * gae_lambda);  // double product rounded once (ppo.py:230)
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, mode == 0 ? "gae_seq" : "gae_scan", 0, 20.0 * T * N + 8.0 * N);
    if (mode == 0) {
        const int threads = (N >= 132 * 64) ? 64 : 32;
        const unsigned blocks = (unsigned)ceil_div(N, threads);
        gae_seq_kernel<8><<<blocks, threads, 0, s>>>(rewards, values, dones, next_value, next_done,
                                                     advantages, returns, T, N, g, gl);
    } else {
        // up to 32 time chunks per env (block = 32 envs x C chunks): the dependent chain is L + C + L steps
        int C = (int)ceil_div(T, 4);
        if (C > 32) C = 32;
        if (C < 1) C = 1;
        const int L = (int)ceil_div(T, C);
        dim3 block(32, C);
        const unsigned blocks = (unsigned)ceil_div(N, 32);
        gae_chunk_kernel<<<blocks, block, 2 * C * 32 * sizeof(float), s>>>(
            rewards, values, dones, next_value, next_done, advantages, returns, T, N, L, g, gl);
    }
    return check_launch("gae");
}
