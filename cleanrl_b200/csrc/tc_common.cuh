// wgmma / TMA / mbarrier primitives for sm_90a (inline PTX; no CUTLASS dependency).
//
// Shared-memory operand images follow the wgmma canonical SWIZZLE_128B layouts
// (bit fields as in the PTX ISA's matrix-descriptor format, restated here):
//   one "row" = 128 bytes = 64 bf16, rows 128 B apart, 8 rows = one 1024-B swizzle atom,
//   the 16-byte chunk c of row r is stored at chunk position (c ^ (r & 7)).
// The SAME image serves as
//   * a K-major operand   (row = M/N index, the 64 elements = 64 consecutive K), and
//   * an MN-major operand (row = K index,   the 64 elements = 64 consecutive M/N),
// only the descriptor differs.  That is what lets the weight-gradient GEMM
// (reduction over rows) reuse the forward im2col staging code unchanged.
#pragma once
#include <cuda_bf16.h>
#include <cstdint>
#include "tc_wgmma.cuh"

namespace b200rl { namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must surface as a launch failure (trap), never as a hung GPU.  The bound is counted on the
// SM's own cycle counter: reading %globaltimer inside the spin loop costs several hundred cycles per poll, which would
// become the period of every tight producer/consumer handshake.
#ifndef B200RL_WAIT_MODE
#define B200RL_WAIT_MODE 0
#endif
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
#if B200RL_WAIT_MODE == 1
    while (!mbar_try_wait_hint(bar, parity, 1000000u)) {
#elif B200RL_WAIT_MODE == 2
    while (!mbar_try_wait(bar, parity)) {
        __nanosleep(40);
#else
    while (!mbar_try_wait(bar, parity)) {
#endif
        if (clock64() - t0 > (1ll << 33)) __trap();      // ~4 s without progress
    }
}

// Two barriers at once: both polls are in flight together (a try_wait costs ~90 cycles even when the phase is complete)
__device__ __forceinline__ void mbar_wait2(uint64_t* bar_a, uint32_t parity_a, uint64_t* bar_b, uint32_t parity_b) {
    const bool a = mbar_try_wait(bar_a, parity_a), b = mbar_try_wait(bar_b, parity_b);
    if (a && b) return;
    if (!a) mbar_wait(bar_a, parity_a);
    if (!b) mbar_wait(bar_b, parity_b);
}

// 32 bytes to global memory as two 16-byte stores
__device__ __forceinline__ void st_global_32b(void* p, const int4& a, const int4& b) {
    reinterpret_cast<int4*>(p)[0] = a;
    reinterpret_cast<int4*>(p)[1] = b;
}

// generic-proxy smem writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor: start address >> 4 (bits 0-13), leading byte offset >> 4 (16-29), stride byte
// offset >> 4 (32-45), base offset 0 (the swizzle is applied to absolute address bits, so a start address shifted by whole
// rows inside a swizzled image addresses the shifted rows), layout type in bits 62-63.
constexpr uint64_t kDescSwizzle128 = 1ull << 62;     // SWIZZLE_128B
constexpr uint64_t kDescSwizzle64 = 2ull << 62;      // SWIZZLE_64B

// K-major SW128 operand: rows (M or N index) 128 B apart, 8-row atoms 1024 B apart (SBO), LBO unused (=1)
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | kDescSwizzle128;
}
// MN-major SW128 operand: 64-element MN atoms `lbo_bytes` apart, 8-row K groups 1024 B apart (SBO)
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t smem_addr, uint32_t lbo_bytes) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | (64ull << 32) |
           kDescSwizzle128;
}

// Accumulator hand-off from a warpgroup's 64 x N fp32 fragment (tc_wgmma.cuh) to a row-major shared-memory tile
// st[64][ld] (ld = N + 4: conflict-free row-wise float4 reads), so that an epilogue thread can own a whole row.
template <int R>
__device__ __forceinline__ void stage_acc(float* st, int ld, int wg_tid, const float (&d)[R]) {
    const int row = ((wg_tid >> 5) << 4) + ((wg_tid & 31) >> 2), col = (wg_tid & 3) * 2;
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
        *reinterpret_cast<float2*>(st + row * ld + 8 * j + col) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2*>(st + (row + 8) * ld + 8 * j + col) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}
// named barrier over `n` threads (warpgroups synchronise among themselves without stalling the producer warps)
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// byte offset of 16-byte chunk `c` of row `r` inside an operand image (rows stacked 128 B apart)
__device__ __forceinline__ uint32_t img_off(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

// max(x, 0) folded into the fp32 -> bf16x2 conversion (one F2FP instead of two FMNMX + one F2FP)
__device__ __forceinline__ uint32_t pack_bf16x2_relu(float lo, float hi) {
    uint32_t d;
    asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

}}  // namespace b200rl::tc

namespace b200rl { namespace tc {
// ---------------------------------------------------------------- cp.async (LDGSTS) + mbarrier arrive
// 16-byte global -> shared copy that bypasses registers; src_bytes = 0 zero-fills the destination.
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(gptr), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
}}  // namespace b200rl::tc

namespace b200rl { namespace tc {
// ---------------------------------------------------------------- TMA (cp.async.bulk.tensor) 2-D tile loads
// dst: 1024-B aligned smem (SWIZZLE_128B box image), tmap: address of a __grid_constant__ CUtensorMap,
// (x, y) = (element column, row) of the box origin; completion is signalled on `bar` with complete_tx bytes.
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, int x, int y, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(x), "r"(y), "r"(smem_u32(bar))
                 : "memory");
}
// 3-D variant: (x, y, z) = (element column, row inside the image, image index); rows past the image end are
// zero-filled by the hardware and still count towards complete_tx
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const void* tmap, int x, int y, int z, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
}}  // namespace b200rl::tc
