// tma_ring.cuh — mbarrier + 1-D bulk-copy (TMA) helpers shared by the row-streaming kernels (sm_90a).
//
// Pattern (resize_rows.cu, warp_stream.cu; the same scheme as fused_rows in resize_fused.cu): a producer lane issues
// `cp.async.bulk` global -> shared copies (SASS UBLKCP) of row spans into a ring of stages, completion is counted on the
// stage's `full` mbarrier (expect_tx), consumer warps wait on `full`, read the taps from shared memory, and arrive on the
// stage's `empty` mbarrier when done.  Copies need 16-byte aligned source, destination and size.
#pragma once

#include <stdint.h>

namespace kb200 {
namespace tma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "TMA_WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra TMA_WAIT_DONE;\n"
        "bra TMA_WAIT_LOOP;\n"
        "TMA_WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// Producer-side wait: the producer is normally far ahead and blocked on a full ring, so it must not burn issue slots —
// try_wait with a suspend-time hint (the warp sleeps until the phase completes or the hint expires).
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    for (;;) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(2000u) : "memory");
        if (ok) return;
    }
}
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// 1-D bulk copy global -> shared::cta through the TMA engine; bytes % 16 == 0, both addresses 16-B aligned.
__device__ __forceinline__ void load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// 1-D bulk copy shared::cta -> global through the TMA engine (SASS UBLKCP with the S2G flavour): whole, byte-exact sectors
// reach L2 however the threads filled the shared buffer.  bytes % 16 == 0, both addresses 16-B aligned.  The writers make
// their shared-memory stores visible to the async proxy first (fence_proxy_async, then a warp / block sync), one thread
// issues the copy, commits the group and — before the buffer is reused or the CTA exits — waits until it has been READ.
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
// one lane of `mask` (the same lane for every call with that mask): lets the compiler issue the uniform-datapath TMA
// instructions straight-line instead of a per-lane waterfall loop
__device__ __forceinline__ bool elect_one(unsigned mask) {
    uint32_t p;
    asm volatile("{\n.reg .pred p;\nelect.sync _|p, %1;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(p) : "r"(mask));
    return p != 0;
}
__device__ __forceinline__ void store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// A warp has filled `bytes` (a multiple of 16) of its 16-byte aligned shared buffer with results: one TMA copy writes them
// to global memory as whole sectors.  Used by the kernels whose threads own 3-, 12- or C-byte pixels: their direct stores
// (lanes a pixel apart, one channel per instruction) send every destination sector to L2 once per channel, a third full.
__device__ __forceinline__ void warp_store_span(void* gmem_dst, const void* smem_src, uint32_t bytes, unsigned mask = 0xFFFFFFFFu) {
    fence_proxy_async();
    __syncwarp(mask);
    if (elect_one(mask)) {
        store_1d(gmem_dst, smem_src, bytes);
        store_commit();
        store_wait_read<0>();       // before the CTA (and its shared memory) goes away
    }
}
// named barrier among `count` threads of the CTA (consumer warps only; the producer warp never joins)
__device__ __forceinline__ void named_barrier(uint32_t id, uint32_t count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

}  // namespace tma
}  // namespace kb200
