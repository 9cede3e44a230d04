// Shared host/device helpers for libb200rl.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include "../../include/b200rl.h"

namespace b200rl {

// thread-local message for b200rl_last_error()
char* err_buf();
int fail(int code, const char* fmt, ...);

void note_launches(int n);
inline int check_launch(const char* what, int kernels = 1) {
    note_launches(kernels);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
    return B200RL_OK;
}

#define B200RL_REQUIRE(cond, ...) \
    do { if (!(cond)) return ::b200rl::fail(B200RL_ERR_INVALID_ARGUMENT, __VA_ARGS__); } while (0)

inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }
inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- optional per-kernel timing (b200rl_profile_*): CUDA events on the launching stream
bool prof_enabled();
void prof_begin(cudaStream_t s, const char* name, double flops, double bytes);
void prof_end(cudaStream_t s);
struct ProfScope {
    cudaStream_t s; bool on;
    ProfScope(cudaStream_t s_, const char* name, double flops, double bytes) : s(s_), on(prof_enabled()) {
        if (on) prof_begin(s, name, flops, bytes);
    }
    ~ProfScope() { if (on) prof_end(s); }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum (fixed order => deterministic).  `red` must hold >= 32 floats.
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
    if (wid == 0) r = warp_sum(r);
    if (threadIdx.x == 0) red[0] = r;
    __syncthreads();
    r = red[0];
    return r;
}

}  // namespace b200rl
