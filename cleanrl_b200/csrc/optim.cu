// Fused grad-clip + Adam over one flat fp32 parameter vector.
//
// Replaces clip_grad_norm_ + optimizer.step() (cleanrl/ppo.py:289-290) and the
// `/ world_size` copy-back of the DP path (ppo_atari_multigpu.py:369-373).
// HBM-bound: algorithmic traffic = read g,p,m,v + write p,m,v = 7 * 4 B * P
// (+ one extra read of g for the norm pass: the norm must be complete before
// any element is updated, so it is a separate grid-wide phase).
// Phase 1 (sumsq): float4 loads, per-block partials, last block (ticket)
// folds them in fixed order in double and stores norm + clip coefficient.
// Phase 2 (adam): float4 elementwise update in torch's op order.
#include "common.cuh"

namespace b200rl {

constexpr int kOptThreads = 256;
constexpr int kOptMaxBlocks = 132 * 8;

struct OptScratch {      // lives at the head of the caller's workspace
    float norm;          // pre-clip global L2 norm
    float coef;          // clamp(max_norm / (norm + 1e-6), max=1)
    unsigned int ticket;
    unsigned int pad;
};

__global__ void __launch_bounds__(kOptThreads) grad_sumsq_kernel(
    const float* __restrict__ g, int64_t P, float inv_world_is_div, float world,
    float max_norm, OptScratch* sc, double* partials, float* norm_out) {
    __shared__ float red[32];
    __shared__ bool is_last;
    float s = 0.f;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t P4 = P >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int64_t i = tid; i < P4; i += stride) {
        float4 v = __ldg(g4 + i);
        if (inv_world_is_div != 0.f) { v.x /= world; v.y /= world; v.z /= world; v.w /= world; }
        s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    for (int64_t i = (P4 << 2) + tid; i < P; i += stride) {
        float v = g[i];
        if (inv_world_is_div != 0.f) v /= world;
        s += v * v;
    }
    const float bs = block_sum(s, red);
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = (double)bs;
        __threadfence();
        is_last = (atomicAdd(&sc->ticket, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // last block: fixed-order two-level sum of the block partials (thread t takes t, t+256, ...; then lanes in order)
    __shared__ double dred[kOptThreads];
    double mine = 0.0;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) mine += __ldcg(partials + b);
    dred[threadIdx.x] = mine;
    __syncthreads();
    for (unsigned off = kOptThreads / 2; off > 0; off >>= 1) {
        if (threadIdx.x < off) dred[threadIdx.x] += dred[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double tot = dred[0];
        const float norm = (float)sqrt(tot);
        sc->norm = norm;
        float coef = 1.f;
        if (max_norm >= 0.f) coef = fminf(max_norm / (norm + 1e-6f), 1.0f);
        sc->coef = coef;
        if (norm_out) *norm_out = norm;
        sc->ticket = 0;
    }
}

struct AdamScalars {
    float w1;        // 1 - beta1
    float beta2;
    float w2;        // 1 - beta2
    float bc2_sqrt;  // sqrt(1 - beta2^step)
    float eps;
    float neg_step_size;  // -(lr / (1 - beta1^step))
    float world;
    int divide_world;
    int do_clip;
};

// The moment updates Adam and RAdam share (torch/optim/adam.py and radam.py, the same two lines).  CPU torch's
// addcmul_ is one fused multiply-add, fma(value * t1, t2, self), which RAdam follows (kFmaAddcmul) to stay bitwise
// equal to CPU torch.optim.RAdam; Adam keeps its separately rounded sum.
template <bool kFmaAddcmul>
__device__ __forceinline__ void adam_moments(float g, float& m, float& v, float w1, float beta2, float w2) {
    m = fmaf(w1, g - m, m);                         // exp_avg.lerp_(grad, 1-beta1)
    v = v * beta2;                                  // exp_avg_sq.mul_(beta2)
    if (kFmaAddcmul) v = fmaf(__fmul_rn(w2, g), g, v);     // .addcmul_(grad, grad, value=1-beta2)
    else v = __fadd_rn(v, __fmul_rn(__fmul_rn(w2, g), g));
}

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, const AdamScalars& a, float coef) {
    if (a.divide_world) g = g / a.world;
    if (a.do_clip) g = g * coef;
    adam_moments<false>(g, m, v, a.w1, a.beta2, a.w2);
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), a.bc2_sqrt), a.eps);
    p = __fadd_rn(p, __fmul_rn(a.neg_step_size, __fdiv_rn(m, denom)));   // addcdiv_(m, denom, -step_size)
}

__global__ void __launch_bounds__(kOptThreads) adam_kernel(
    float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
    int64_t P, AdamScalars a, const OptScratch* sc, const float* __restrict__ dyn) {
    if (dyn) { a.bc2_sqrt = __ldg(dyn); a.neg_step_size = __ldg(dyn + 1); }     // step / lr dependent scalars from device memory
    const float coef = a.do_clip ? sc->coef : 1.f;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t P4 = P >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(m);
    float4* v4 = reinterpret_cast<float4*>(v);
    for (int64_t i = tid; i < P4; i += stride) {
        float4 pp = p4[i], gg = __ldg(g4 + i), mm = m4[i], vv = v4[i];
        adam_one(pp.x, gg.x, mm.x, vv.x, a, coef);
        adam_one(pp.y, gg.y, mm.y, vv.y, a, coef);
        adam_one(pp.z, gg.z, mm.z, vv.z, a, coef);
        adam_one(pp.w, gg.w, mm.w, vv.w, a, coef);
        p4[i] = pp; m4[i] = mm; v4[i] = vv;
    }
    for (int64_t i = (P4 << 2) + tid; i < P; i += stride) {
        float pp = p[i], mm = m[i], vv = v[i];
        adam_one(pp, g[i], mm, vv, a, coef);
        p[i] = pp; m[i] = mm; v[i] = vv;
    }
}

// ---- the same update with a few element ranges treated apart (torch.optim.Adam keeps a `step` per tensor and skips a
// tensor whose grad is None; so does clip_grad_norm_).  frozen: the ranges take no part in the norm and are not touched
// (parameters, both moments).  Otherwise they are updated with their own step-dependent scalars.
constexpr int kOptMaxRanges = 4;
struct OptRanges {
    int n;
    int frozen;
    int64_t lo[kOptMaxRanges], hi[kOptMaxRanges];
    float bc2_sqrt, neg_step_size;         // of the ranges' own (step, lr)
    __device__ __forceinline__ bool has(int64_t i) const {
        bool in = false;
#pragma unroll
        for (int r = 0; r < kOptMaxRanges; ++r) in = in || (r < n && i >= lo[r] && i < hi[r]);
        return in;
    }
};

__global__ void __launch_bounds__(kOptThreads) grad_sumsq_ranges_kernel(const float* __restrict__ g, int64_t P, OptRanges R,
                                                                        double* __restrict__ partials) {
    __shared__ float red[32];
    float s = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = g[i];
        if (!(R.frozen && R.has(i))) s += v * v;
    }
    const float bs = block_sum(s, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = (double)bs;
}

// one block: the per-block partials in a fixed order (as the last block of grad_sumsq_kernel), then the Adam pass reads coef
__global__ void __launch_bounds__(kOptThreads) grad_norm_fold_kernel(const double* __restrict__ partials, int nblocks,
                                                                     float max_norm, OptScratch* sc, float* norm_out) {
    __shared__ double dred[kOptThreads];
    double mine = 0.0;
    for (int b = threadIdx.x; b < nblocks; b += blockDim.x) mine += partials[b];
    dred[threadIdx.x] = mine;
    __syncthreads();
    for (unsigned off = kOptThreads / 2; off > 0; off >>= 1) {
        if (threadIdx.x < off) dred[threadIdx.x] += dred[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float norm = (float)sqrt(dred[0]);
        sc->norm = norm;
        sc->coef = max_norm >= 0.f ? fminf(max_norm / (norm + 1e-6f), 1.0f) : 1.f;
        if (norm_out) *norm_out = norm;
    }
}

__global__ void __launch_bounds__(kOptThreads) adam_ranges_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                                  float* __restrict__ m, float* __restrict__ v, int64_t P,
                                                                  AdamScalars a, OptRanges R, const OptScratch* sc,
                                                                  const float* __restrict__ dyn) {
    if (dyn) {      // step / lr dependent scalars from device memory: [0..1] every element, [2..3] the ranges
        a.bc2_sqrt = __ldg(dyn); a.neg_step_size = __ldg(dyn + 1);
        R.bc2_sqrt = __ldg(dyn + 2); R.neg_step_size = __ldg(dyn + 3);
    }
    const float coef = a.do_clip ? sc->coef : 1.f;
    AdamScalars b = a;
    b.bc2_sqrt = R.bc2_sqrt; b.neg_step_size = R.neg_step_size;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x) {
        const bool in = R.has(i);
        if (in && R.frozen) continue;
        float pp = p[i], mm = m[i], vv = v[i];
        adam_one(pp, g[i], mm, vv, in ? b : a, coef);
        p[i] = pp; m[i] = mm; v[i] = vv;
    }
}

static inline unsigned opt_blocks(int64_t P) {
    int64_t b = ceil_div(ceil_div(P, 4), kOptThreads);
    if (b < 1) b = 1;
    if (b > kOptMaxBlocks) b = kOptMaxBlocks;
    return (unsigned)b;
}

}  // namespace b200rl

extern "C" size_t b200rl_clip_adam_workspace_bytes(int64_t P) {
    (void)P;
    return sizeof(b200rl::OptScratch) + sizeof(double) * b200rl::kOptMaxBlocks;
}

namespace b200rl {
static void adam_step_scalars(int64_t step, double lr, double beta1, double beta2, float* bc2_sqrt, float* neg_step_size) {
    // scalar algebra in double exactly as torch/optim/adam.py does it in python
    const double bc1 = 1.0 - pow(beta1, (double)step);
    const double bc2 = 1.0 - pow(beta2, (double)step);
    const double step_size = lr / bc1;
    *bc2_sqrt = (float)sqrt(bc2);
    *neg_step_size = (float)(-step_size);
}

// dyn == nullptr: (step, lr) by value; else the two step-dependent scalars are read from device memory (CUDA-graph replays)
static int clip_adam_impl(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P, int64_t step, double lr,
                          const float* dyn, double beta1, double beta2, double eps, double max_norm, int world_size, float* norm_out,
                          void* workspace, size_t workspace_bytes, void* stream) {
    B200RL_REQUIRE(P >= 0, "clip_adam: negative P");
    if (P == 0) return B200RL_OK;
    B200RL_REQUIRE(params && grads && exp_avg && exp_avg_sq, "clip_adam: null pointer");
    B200RL_REQUIRE(aligned(params, 16) && aligned(grads, 16) && aligned(exp_avg, 16) && aligned(exp_avg_sq, 16),
                   "clip_adam: buffers must be 16-B aligned (float4 path)");
    B200RL_REQUIRE(dyn || step >= 1, "clip_adam: step is 1-based (got %lld)", (long long)step);
    B200RL_REQUIRE(!dyn || aligned(dyn, 4), "clip_adam: misaligned scalar table");
    B200RL_REQUIRE(world_size >= 1, "clip_adam: world_size must be >= 1");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "clip_adam: workspace null or misaligned");
    if (workspace_bytes < b200rl_clip_adam_workspace_bytes(P))
        return fail(B200RL_ERR_WORKSPACE, "clip_adam: workspace %zu < %zu bytes", workspace_bytes,
                    b200rl_clip_adam_workspace_bytes(P));
    cudaStream_t s = (cudaStream_t)stream;
    OptScratch* sc = reinterpret_cast<OptScratch*>(workspace);
    double* partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + sizeof(OptScratch));
    const unsigned blocks = opt_blocks(P);
    ProfScope ps(s, "clip_adam", 0, 32.0 * P);
    const bool need_norm = (max_norm >= 0.0) || (norm_out != nullptr);
    if (need_norm) {
        cudaError_t e = cudaMemsetAsync(&sc->ticket, 0, sizeof(unsigned int), s);
        if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "clip_adam: memset: %s", cudaGetErrorString(e));
        grad_sumsq_kernel<<<blocks, kOptThreads, 0, s>>>(grads, P, world_size > 1 ? 1.f : 0.f, (float)world_size,
                                                        (float)max_norm, sc, partials, norm_out);
        int rc = check_launch("clip_adam/sumsq");
        if (rc) return rc;
    }
    AdamScalars a;
    a.w1 = (float)(1.0 - beta1);
    a.beta2 = (float)beta2;
    a.w2 = (float)(1.0 - beta2);
    a.bc2_sqrt = 1.f;
    a.neg_step_size = 0.f;
    if (!dyn) adam_step_scalars(step, lr, beta1, beta2, &a.bc2_sqrt, &a.neg_step_size);
    a.eps = (float)eps;
    a.world = (float)world_size;
    a.divide_world = world_size > 1;
    a.do_clip = max_norm >= 0.0;
    adam_kernel<<<blocks, kOptThreads, 0, s>>>(params, grads, exp_avg, exp_avg_sq, P, a, sc, dyn);
    return check_launch("clip_adam/adam");
}
}  // namespace b200rl

extern "C" int b200rl_clip_adam_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                                    int64_t P, int64_t step, double lr, double beta1, double beta2, double eps,
                                    double max_norm, int world_size, float* norm_out,
                                    void* workspace, size_t workspace_bytes, void* stream) {
    return b200rl::clip_adam_impl(params, grads, exp_avg, exp_avg_sq, P, step, lr, nullptr, beta1, beta2, eps, max_norm, world_size,
                                  norm_out, workspace, workspace_bytes, stream);
}

extern "C" int b200rl_adam_step_scalars(int64_t step, double lr, double beta1, double beta2, float* out2) {
    B200RL_REQUIRE(out2 && step >= 1, "adam_step_scalars: bad arguments");
    b200rl::adam_step_scalars(step, lr, beta1, beta2, out2, out2 + 1);
    return B200RL_OK;
}

extern "C" int b200rl_clip_adam_dyn_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                                        int64_t P, const float* step_scalars, double beta1, double beta2, double eps,
                                        double max_norm, int world_size, float* norm_out,
                                        void* workspace, size_t workspace_bytes, void* stream) {
    B200RL_REQUIRE(step_scalars, "clip_adam_dyn: null scalar table");
    return b200rl::clip_adam_impl(params, grads, exp_avg, exp_avg_sq, P, 0, 0.0, step_scalars, beta1, beta2, eps, max_norm, world_size,
                                  norm_out, workspace, workspace_bytes, stream);
}

namespace b200rl {
// dyn == nullptr: (step, lr) and (range_step, range_lr) by value; else the four step-dependent scalars are read from device
// memory (CUDA-graph replays) and `frozen` says whether the ranges are skipped
static int clip_adam_ranges_impl(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P, int64_t step,
                                 double lr, const int64_t* ranges, int nranges, int64_t range_step, double range_lr,
                                 const float* dyn, int frozen, double beta1, double beta2, double eps, double max_norm,
                                 float* norm_out, void* workspace, size_t workspace_bytes, void* stream) {
    B200RL_REQUIRE(P >= 1, "clip_adam_ranges: P must be >= 1");
    B200RL_REQUIRE(params && grads && exp_avg && exp_avg_sq, "clip_adam_ranges: null pointer");
    B200RL_REQUIRE(aligned(params, 4) && aligned(grads, 4) && aligned(exp_avg, 4) && aligned(exp_avg_sq, 4) && aligned(dyn, 4),
                   "clip_adam_ranges: misaligned buffer");
    B200RL_REQUIRE(dyn || (step >= 1 && range_step >= 0), "clip_adam_ranges: steps are 1-based (got %lld, %lld)",
                   (long long)step, (long long)range_step);
    B200RL_REQUIRE(nranges >= 0 && nranges <= kOptMaxRanges && (nranges == 0 || ranges), "clip_adam_ranges: %d ranges outside [0,%d]",
                   nranges, kOptMaxRanges);
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "clip_adam_ranges: workspace null or misaligned");
    if (workspace_bytes < b200rl_clip_adam_workspace_bytes(P))
        return fail(B200RL_ERR_WORKSPACE, "clip_adam_ranges: workspace %zu < %zu bytes", workspace_bytes,
                    b200rl_clip_adam_workspace_bytes(P));
    OptRanges R;
    R.n = nranges; R.frozen = dyn ? frozen != 0 : range_step == 0; R.bc2_sqrt = 1.f; R.neg_step_size = 0.f;
    for (int r = 0; r < kOptMaxRanges; ++r) {
        R.lo[r] = r < nranges ? ranges[2 * r] : 0;
        R.hi[r] = r < nranges ? ranges[2 * r + 1] : 0;
        B200RL_REQUIRE(R.lo[r] >= 0 && R.lo[r] <= R.hi[r] && R.hi[r] <= P, "clip_adam_ranges: range %d outside [0,%lld]", r, (long long)P);
    }
    if (!dyn && !R.frozen) adam_step_scalars(range_step, range_lr, beta1, beta2, &R.bc2_sqrt, &R.neg_step_size);
    cudaStream_t s = (cudaStream_t)stream;
    OptScratch* sc = reinterpret_cast<OptScratch*>(workspace);
    double* partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + sizeof(OptScratch));
    const unsigned blocks = opt_blocks(P);
    ProfScope ps(s, "clip_adam_ranges", 0, 32.0 * P);
    int launches = 1;
    if (max_norm >= 0.0 || norm_out) {
        grad_sumsq_ranges_kernel<<<blocks, kOptThreads, 0, s>>>(grads, P, R, partials);
        grad_norm_fold_kernel<<<1, kOptThreads, 0, s>>>(partials, (int)blocks, (float)max_norm, sc, norm_out);
        launches = 3;
    }
    AdamScalars a;
    a.w1 = (float)(1.0 - beta1);
    a.beta2 = (float)beta2;
    a.w2 = (float)(1.0 - beta2);
    a.bc2_sqrt = 1.f;
    a.neg_step_size = 0.f;
    if (!dyn) adam_step_scalars(step, lr, beta1, beta2, &a.bc2_sqrt, &a.neg_step_size);
    a.eps = (float)eps;
    a.world = 1.f;
    a.divide_world = 0;
    a.do_clip = max_norm >= 0.0;
    adam_ranges_kernel<<<blocks, kOptThreads, 0, s>>>(params, grads, exp_avg, exp_avg_sq, P, a, R, sc, dyn);
    return check_launch("clip_adam_ranges", launches);
}
}  // namespace b200rl

// clip + Adam with `nranges` element ranges [ranges[2r], ranges[2r+1]) (host array) treated apart: range_step == 0 freezes
// them (no part in the clip norm, parameters and moments untouched); range_step >= 1 updates them with (range_step,
// range_lr) while every other element uses (step, lr).  The clip norm is over the elements that are updated.
extern "C" int b200rl_clip_adam_ranges_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                                           int64_t step, double lr, const int64_t* ranges, int nranges, int64_t range_step,
                                           double range_lr, double beta1, double beta2, double eps, double max_norm,
                                           float* norm_out, void* workspace, size_t workspace_bytes, void* stream) {
    return b200rl::clip_adam_ranges_impl(params, grads, exp_avg, exp_avg_sq, P, step, lr, ranges, nranges, range_step, range_lr,
                                         nullptr, 0, beta1, beta2, eps, max_norm, norm_out, workspace, workspace_bytes, stream);
}

// the same with the step-dependent scalars in device memory: step_scalars[0..1] = b200rl_adam_step_scalars(step, lr) for
// every element, [2..3] = those of (range_step, range_lr) for the ranges (unused when `frozen`)
extern "C" int b200rl_clip_adam_ranges_dyn_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                                               const float* step_scalars, const int64_t* ranges, int nranges, int frozen,
                                               double beta1, double beta2, double eps, double max_norm, float* norm_out,
                                               void* workspace, size_t workspace_bytes, void* stream) {
    B200RL_REQUIRE(step_scalars, "clip_adam_ranges_dyn: null scalar table");
    return b200rl::clip_adam_ranges_impl(params, grads, exp_avg, exp_avg_sq, P, 0, 0.0, ranges, nranges, 0, 0.0, step_scalars,
                                         frozen, beta1, beta2, eps, max_norm, norm_out, workspace, workspace_bytes, stream);
}

// ---- clip + RAdam (torch/optim/radam.py _single_tensor_radam, no weight decay).  The four step-dependent scalars stay
// separate, each rounded to f32 where the tensor operation that uses it rounds it:
//   rho_t <= 5: p -= (m / bc1) * lr
//   rho_t >  5: p -= (((m / bc1) * lr) * (reciprocal(sqrt(v) + eps) * sqrt(bc2))) * rect
namespace b200rl {
struct RAdamScalars {
    float w1, beta2, w2, eps;
    float bc1, lr, bc2_sqrt, rect;   // rect <= 0: rho_t <= 5 (no rectification)
    int do_clip;
};

__device__ __forceinline__ void radam_one(float& p, float g, float& m, float& v, const RAdamScalars& a, float coef) {
    if (a.do_clip) g = g * coef;
    adam_moments<true>(g, m, v, a.w1, a.beta2, a.w2);
    const float u = __fmul_rn(__fdiv_rn(m, a.bc1), a.lr);                 // bias_corrected_exp_avg * lr
    if (a.rect > 0.f) {
        const float adaptive = __fmul_rn(__frcp_rn(__fadd_rn(sqrtf(v), a.eps)), a.bc2_sqrt);   // bc2**0.5 / (sqrt(v)+eps)
        p = __fsub_rn(p, __fmul_rn(__fmul_rn(u, adaptive), a.rect));
    } else {
        p = __fsub_rn(p, u);
    }
}

__global__ void __launch_bounds__(kOptThreads) radam_kernel(
    float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
    int64_t P, RAdamScalars a, const OptScratch* sc, const float* __restrict__ dyn) {
    if (dyn) { a.bc1 = __ldg(dyn); a.lr = __ldg(dyn + 1); a.bc2_sqrt = __ldg(dyn + 2); a.rect = __ldg(dyn + 3); }
    const float coef = a.do_clip ? sc->coef : 1.f;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t P4 = P >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(m);
    float4* v4 = reinterpret_cast<float4*>(v);
    for (int64_t i = tid; i < P4; i += stride) {
        float4 pp = p4[i], gg = __ldg(g4 + i), mm = m4[i], vv = v4[i];
        radam_one(pp.x, gg.x, mm.x, vv.x, a, coef);
        radam_one(pp.y, gg.y, mm.y, vv.y, a, coef);
        radam_one(pp.z, gg.z, mm.z, vv.z, a, coef);
        radam_one(pp.w, gg.w, mm.w, vv.w, a, coef);
        p4[i] = pp; m4[i] = mm; v4[i] = vv;
    }
    for (int64_t i = (P4 << 2) + tid; i < P; i += stride) {
        float pp = p[i], mm = m[i], vv = v[i];
        radam_one(pp, g[i], mm, vv, a, coef);
        p[i] = pp; m[i] = mm; v[i] = vv;
    }
}

// the scalar algebra of _single_tensor_radam in double, as python runs it (x ** 0.5 is C pow)
static void radam_step_scalars(int64_t step, double lr, double beta1, double beta2, float* out4) {
    const double st = (double)step;
    const double bc1 = 1.0 - pow(beta1, st);
    const double bc2 = 1.0 - pow(beta2, st);
    const double rho_inf = 2.0 / (1.0 - beta2) - 1.0;
    const double rho_t = rho_inf - 2.0 * st * pow(beta2, st) / bc2;
    out4[0] = (float)bc1;
    out4[1] = (float)lr;
    out4[2] = (float)pow(bc2, 0.5);
    out4[3] = rho_t > 5.0 ? (float)pow((rho_t - 4.0) * (rho_t - 2.0) * rho_inf / ((rho_inf - 4.0) * (rho_inf - 2.0) * rho_t), 0.5)
                          : 0.f;
}

// dyn == nullptr: (step, lr) by value; else the four step-dependent scalars are read from device memory
static int clip_radam_impl(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P, int64_t step,
                           double lr, const float* dyn, double beta1, double beta2, double eps, double max_norm,
                           float* norm_out, void* workspace, size_t workspace_bytes, void* stream) {
    B200RL_REQUIRE(P >= 0, "clip_radam: negative P");
    if (P == 0) return B200RL_OK;
    B200RL_REQUIRE(params && grads && exp_avg && exp_avg_sq, "clip_radam: null pointer");
    B200RL_REQUIRE(aligned(params, 16) && aligned(grads, 16) && aligned(exp_avg, 16) && aligned(exp_avg_sq, 16),
                   "clip_radam: buffers must be 16-B aligned (float4 path)");
    B200RL_REQUIRE(dyn || step >= 1, "clip_radam: step is 1-based (got %lld)", (long long)step);
    B200RL_REQUIRE(!dyn || aligned(dyn, 4), "clip_radam: misaligned scalar table");
    B200RL_REQUIRE(workspace && aligned(workspace, 16), "clip_radam: workspace null or misaligned");
    if (workspace_bytes < b200rl_clip_adam_workspace_bytes(P))
        return fail(B200RL_ERR_WORKSPACE, "clip_radam: workspace %zu < %zu bytes", workspace_bytes,
                    b200rl_clip_adam_workspace_bytes(P));
    cudaStream_t s = (cudaStream_t)stream;
    OptScratch* sc = reinterpret_cast<OptScratch*>(workspace);
    double* partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + sizeof(OptScratch));
    const unsigned blocks = opt_blocks(P);
    ProfScope ps(s, "clip_radam", 0, 32.0 * P);
    if (max_norm >= 0.0 || norm_out) {
        cudaError_t e = cudaMemsetAsync(&sc->ticket, 0, sizeof(unsigned int), s);
        if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "clip_radam: memset: %s", cudaGetErrorString(e));
        grad_sumsq_kernel<<<blocks, kOptThreads, 0, s>>>(grads, P, 0.f, 1.f, (float)max_norm, sc, partials, norm_out);
        int rc = check_launch("clip_radam/sumsq");
        if (rc) return rc;
    }
    RAdamScalars a;
    a.w1 = (float)(1.0 - beta1);
    a.beta2 = (float)beta2;
    a.w2 = (float)(1.0 - beta2);
    a.eps = (float)eps;
    float s4[4] = {1.f, 0.f, 1.f, 0.f};
    if (!dyn) radam_step_scalars(step, lr, beta1, beta2, s4);
    a.bc1 = s4[0]; a.lr = s4[1]; a.bc2_sqrt = s4[2]; a.rect = s4[3];
    a.do_clip = max_norm >= 0.0;
    radam_kernel<<<blocks, kOptThreads, 0, s>>>(params, grads, exp_avg, exp_avg_sq, P, a, sc, dyn);
    return check_launch("clip_radam/radam");
}
}  // namespace b200rl

extern "C" int b200rl_radam_step_scalars(int64_t step, double lr, double beta1, double beta2, float* out4) {
    B200RL_REQUIRE(out4 && step >= 1, "radam_step_scalars: bad arguments");
    b200rl::radam_step_scalars(step, lr, beta1, beta2, out4);
    return B200RL_OK;
}

extern "C" int b200rl_clip_radam_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                                     int64_t step, double lr, double beta1, double beta2, double eps, double max_norm,
                                     float* norm_out, void* workspace, size_t workspace_bytes, void* stream) {
    return b200rl::clip_radam_impl(params, grads, exp_avg, exp_avg_sq, P, step, lr, nullptr, beta1, beta2, eps, max_norm,
                                   norm_out, workspace, workspace_bytes, stream);
}

extern "C" int b200rl_clip_radam_dyn_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t P,
                                         const float* step_scalars, double beta1, double beta2, double eps,
                                         double max_norm, float* norm_out, void* workspace, size_t workspace_bytes,
                                         void* stream) {
    B200RL_REQUIRE(step_scalars, "clip_radam_dyn: null scalar table");
    return b200rl::clip_radam_impl(params, grads, exp_avg, exp_avg_sq, P, 0, 0.0, step_scalars, beta1, beta2, eps,
                                   max_norm, norm_out, workspace, workspace_bytes, stream);
}
