// pbs_plus_b200/csrc/device.cuh -- device-only primitives shared by the kernels: shared-memory mbarriers, TMA copies,
// the warp's TMA staging rule, the "which range owns work unit g" search and the device-count clamp.
// Included by the kernel .cu files only (not by internal.cuh / host.hpp), so the C ABI units see no inline asm.
#pragma once
#include <cuda.h>   // CUtensorMap
#include <stdint.h>

namespace pbsgpu {

// The range that owns work unit g: the largest i < n with first[i] <= g.  `first` is a non-decreasing prefix with
// first[0] <= g < first[n] (first[n] is never read), so ranges without units (first[i] == first[i + 1]) are skipped.
__device__ __forceinline__ uint32_t owner_of(const uint64_t *first, uint32_t n, uint64_t g) {
    uint32_t lo = 0, hi = n;   // invariant: first[lo] <= g < first[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (first[mid] <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// A count the device wrote (`n`, read from device memory), bounded by `cap`: the capacity a launch was sized for, or
// an enclosing count.
__device__ __forceinline__ unsigned long long live_count(unsigned long long n, unsigned long long cap) { return n < cap ? n : cap; }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarriers in shared memory (`bar` = smem_u32 address) -------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// after the mbar_init calls and before the __syncthreads that publishes them
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n .reg .pred P1;\n LAB_WAIT:\n"
        " mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        " @P1 bra DONE;\n bra LAB_WAIT;\n DONE:\n }" ::"r"(bar), "r"(parity) : "memory");
}

// ---- TMA copies, completing as transaction bytes on `bar` ------------------------------------------------------
// generic-proxy accesses of shared memory before this are ordered before later async-proxy (TMA) ones
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// `bytes` contiguous bytes; dst, src and bytes are multiples of 16
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// one box of a 4-D tensor map at coordinates {c0, c1, c2, c3}
__device__ __forceinline__ void tma_tensor4d_g2s(uint32_t dst, const CUtensorMap *map, int c0, int c1, int c2, int c3,
                                                 uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}

// ---- per-warp double buffering -----------------------------------------------------------------------------------
// Lane 0 of every warp sets up the warp's two single-arrival barriers.  Ends in the CTA's __syncthreads, so every
// thread calls it, after the shared-memory set-up that sync must also publish.
__device__ __forceinline__ void warp_bars_init(const uint32_t (&bar)[2], uint32_t lane) {
    if (lane == 0) {
        mbar_init(bar[0], 1);
        mbar_init(bar[1], 1);
        mbar_init_fence();
    }
    __syncthreads();
}

// The warp's staging rule for `bytes` from a 16 B aligned `src` to a 16 B aligned shared `dst`, completing on a
// single-arrival `bar`: the lanes copy the tail below 16 B (bulk = bytes & ~15 onwards), __syncwarp, then lane 0
// calls this.  It makes the tail stores visible to the async proxy, arrives expecting `bulk` bytes and brings them
// as ONE bulk copy.  (The tail loop stays in the callers: as part of a shared function it changes their register
// allocation.)
__device__ __forceinline__ void stage_bulk(uint8_t *dst, const uint8_t *src, uint32_t bulk, uint32_t bar) {
    fence_proxy_async();
    mbar_arrive_expect_tx(bar, bulk);
    if (bulk) tma_bulk_g2s(smem_u32(dst), src, bulk, bar);
}

}  // namespace pbsgpu
