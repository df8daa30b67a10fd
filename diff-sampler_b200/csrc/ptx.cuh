// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma.
// Everything here is hand-written PTX; there is no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "wgmma.cuh"

namespace dsb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() {
    uint32_t l;
    asm("mov.u32 %0, %%laneid;" : "=r"(l));          // not volatile: the lane id is loop-invariant, let the compiler hoist it
    return l;
}

// One elected lane of a fully converged warp (elect.sync over all 32 lanes): the TMA producer loop runs with the whole warp converged
// and only the copies elected.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .pred px;\n\t"
        "elect.sync _|px, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, px;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok;
}
// Bounded spin: a protocol bug traps (-> CUDA error) instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}

// The same for a fully converged warp: lane 0 polls, the other lanes wait at the warp barrier (one poller per barrier instead of 32;
// __syncwarp orders lane 0's acquire before the other lanes' subsequent accesses).
__device__ __forceinline__ void mbar_wait_warp(uint64_t* bar, uint32_t parity) {
    if (lane_id() == 0) mbar_wait(bar, parity);
    __syncwarp();
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, fp32 accumulators in registers)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Keeps the compiler from moving accumulator accesses across the asynchronous MMAs that own those registers.
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128-byte-swizzled operand tile: rows of 128 B (64 x 16-bit or 128 x 8-bit), 8-row groups 1024 B apart.  The tile base
// must be 1024-byte aligned; a K step of 32 bytes inside the swizzle row adds 2 to the descriptor (16-byte units).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);      // start address, 16-byte units
    d |= static_cast<uint64_t>(1) << 16;                         // leading byte offset (unused: one swizzle atom along K)
    d |= static_cast<uint64_t>(1024 >> 4) << 32;                 // stride byte offset between 8-row groups
    d |= static_cast<uint64_t>(1) << 62;                         // SWIZZLE_128B
    return d;
}

// D[64 x N] (+)= A * B^T for any N that is a multiple of 16 up to 256: one instruction per set bit of N / 16.  The accumulator
// of the part starting at column n0 sits at d[n0 / 2 ..], so the register layout is that of a single m64nN instruction; the B part
// starts n0 rows (n0 * 128 bytes: whole 1024-byte swizzle atoms) further into the tile.
template <int N, bool F8>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    static_assert(N % 16 == 0 && N >= 16 && N <= 256, "N");
    constexpr int n256 = N & 256, n128 = N & 128, n64 = N & 64, n32 = N & 32, n16 = N & 16;
    auto part = [&](auto nc, int n0) {
        constexpr int NC = decltype(nc)::value;
        if (F8) Wgmma<NC>::e4m3(d + n0 / 2, da, db + (uint64_t)(n0 * 128 / 16), scale_d);
        else Wgmma<NC>::f16(d + n0 / 2, da, db + (uint64_t)(n0 * 128 / 16), scale_d);
    };
    if constexpr (n256 != 0) part(std::integral_constant<int, 256>{}, 0);
    if constexpr (n128 != 0) part(std::integral_constant<int, 128>{}, n256);
    if constexpr (n64 != 0) part(std::integral_constant<int, 64>{}, n256 + n128);
    if constexpr (n32 != 0) part(std::integral_constant<int, 32>{}, n256 + n128 + n64);
    if constexpr (n16 != 0) part(std::integral_constant<int, 16>{}, n256 + n128 + n64 + n32);
}

// named barrier over the 128 threads of one warpgroup (ids 1..; 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

}  // namespace dsb
