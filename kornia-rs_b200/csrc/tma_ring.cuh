// tma_ring.cuh — mbarrier, bulk-copy (TMA) and persistent unit-walk helpers shared by the TMA-staged kernels (sm_90a).
//
// Users: fused_rows_kernel and fused_point_rows_kernel (resize_fused.cu), resize_rows_f32_kernel (resize_rows.cu),
// sep_filter_stream2_kernel (filter.cu), blur_u8_stream_kernel (filter_u8.cu), warp_tiled_kernel and the lean warp
// kernel's tile stores (warp.cu), warp_stream_kernel and warp_stream2_kernel (warp_stream.cuh, warp_stream*.cu).
//
// Pattern: a producer lane issues `cp.async.bulk` global -> shared copies (SASS UBLKCP) of row spans into a ring of
// stages, completion is counted on the stage's `full` mbarrier (expect_tx), consumer warps wait on `full`, read the taps
// from shared memory, and arrive on the stage's `empty` mbarrier when done.  Copies need 16-byte aligned source,
// destination and size.
#pragma once

#include <cuda.h>
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
// Tensor-map box global -> shared::cta through the TMA engine (SASS UTMALDG.3D); c0 is the innermost coordinate.  The box
// must start on a 16-byte boundary; parts outside the tensor are zero-filled.
__device__ __forceinline__ void load_3d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
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
// Tensor-map box shared::cta -> global (SASS UTMASTG.4D), same protocol as store_1d; the map clips the box at the tensor's
// edges.  c0 is the innermost coordinate.
__device__ __forceinline__ void store_4d(const CUtensorMap* tmap, int c0, int c1, int c2, int c3, const void* smem_src) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%1, %2, %3, %4}], [%5];" ::"l"(tmap), "r"(c0), "r"(c1), "r"(c2),
                 "r"(c3), "r"(smem_u32(smem_src))
                 : "memory");
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

// Persistent-CTA walk over units (column tile tx, row chunk cy, image img), unit u = (img * chunks_y + cy) * tiles_x + tx.
// A CTA starts at unit blockIdx.x and steps by gridDim.x: init divides once, advance adds the stride's digits
// (dtx, dcy, dimg from carry_strides) with carries instead of dividing.  P has tiles_x, chunks_y, dtx, dcy and dimg.
template <typename P>
struct UnitWalk {
    uint32_t tx, cy, img;
    __device__ __forceinline__ void init(uint32_t u, const P& p) {
        const uint32_t per_img = p.tiles_x * p.chunks_y;
        img = u / per_img;
        const uint32_t t = u - img * per_img;
        cy = t / p.tiles_x;
        tx = t - cy * p.tiles_x;
    }
    __device__ __forceinline__ void advance(const P& p) {
        tx += p.dtx; cy += p.dcy; img += p.dimg;
        if (tx >= p.tiles_x) { tx -= p.tiles_x; ++cy; }
        if (cy >= p.chunks_y) { cy -= p.chunks_y; ++img; }
        if (cy >= p.chunks_y) { cy -= p.chunks_y; ++img; }
    }
};

// Host side of UnitWalk: decompose the CTA stride `grid` so that grid = (dimg * chunks_y + dcy) * tiles_x + dtx.
template <typename P>
inline void carry_strides(uint32_t grid, P& p) {
    p.dtx = grid % p.tiles_x;
    const uint32_t g = grid / p.tiles_x;
    p.dcy = g % p.chunks_y;
    p.dimg = g / p.chunks_y;
}

}  // namespace tma
}  // namespace kb200
