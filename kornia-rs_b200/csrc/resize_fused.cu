// resize_fused.cu — fused u8 HWC → f32 / f16 / bf16 CHW bilinear resize + normalize (a2; BASELINE config 2).
//
// Reference: resize/fused.rs:147-228 (general bilinear, half-pixel, non-antialiased), scalar leaf
// :273-318, AVX2+FMA leaf :414-497 (FMA form on the dst_w&~7 bulk, scalar form on the tail),
// exact-2x box path :57-127 with leaves :528-559 (scalar) / fused_row_avx2 (FMA on dst_w&~15).
//
// `fma_bulk` = number of leading destination columns whose arithmetic is the reference's FMA leaf;
// columns ≥ fma_bulk use the scalar (mul, add) leaf — so the output is bit-identical to what the
// reference produces on the chosen CPU (x86 AVX2+FMA: bulk = dst_w & ~7, or & ~15 on the 2x path).
//
// 16-bit outputs (an extension: the reference writes f32 only): every kernel is templated on the output element type
// and computes the f32 value exactly as the f32 instantiation does; only the store differs, one round-to-nearest-even
// conversion (fused_out) of that value.  So out16 == RNE(out_f32) for every mode, leaf and column.
#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "kb200_common.cuh"
#include "resize_fused.cuh"

namespace kb200 {

__device__ __forceinline__ float fused_lerp(float a, float b, float c, float d, float wx, float wy, float sc, float bi,
                                            bool fused) {
    if (fused) {  // resize/fused.rs:475-478
        const float top = fmaf(b - a, wx, a);
        const float bot = fmaf(d - c, wx, c);
        const float val = fmaf(bot - top, wy, top);
        return fmaf(val, sc, bi);
    }
    const float top = a + wx * (b - a);  // resize/fused.rs:286-317
    const float bot = c + wx * (d - c);
    const float val = top + wy * (bot - top);
    return val * sc + bi;
}

// The one place the output type enters the arithmetic: f32 is stored as computed, a 16-bit type is the hardware RNE
// conversion of it (overflow -> inf, subnormals and the sign of zero kept, NaN -> NaN).
template <typename T> __device__ __forceinline__ T fused_out(float v);
template <> __device__ __forceinline__ float fused_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __half fused_out<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 fused_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// Generic path: any size / alignment.  One thread per destination pixel, batch = grid.z.
template <typename T, bool BOX2X>
__global__ void __launch_bounds__(256) fused_resize_gather_kernel(const uint8_t* __restrict__ src, T* __restrict__ dst,
                                                                  const __grid_constant__ FusedParams p) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= p.dw || y >= p.dh) return;
    const uint8_t* s = src + (size_t)blockIdx.z * p.sw * p.src_rows * 3;
    const size_t plane = (size_t)p.dw * p.dh;
    T* d = dst + (size_t)blockIdx.z * plane * 3 + (size_t)y * p.dw + x;
    const bool fused = x < p.fma_bulk;
    if (BOX2X) {  // resize/fused.rs:528-559
        const uint8_t* r0 = s + ((size_t)(2 * y) * p.sw + 2 * x) * 3;
        const uint8_t* r1 = r0 + (size_t)p.sw * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const uint32_t sum = (uint32_t)r0[c] + r0[3 + c] + r1[c] + r1[3 + c];
            const float s4 = p.scale[c] * 0.25f;
            d[c * plane] = fused_out<T>(fused ? fmaf((float)sum, s4, p.bias[c]) : (float)sum * s4 + p.bias[c]);
        }
        return;
    }
    const float fx = fmaxf(((float)x + 0.5f) * p.scale_x - 0.5f, 0.0f);
    const float fy = fmaxf(((float)y + 0.5f) * p.scale_y - 0.5f, 0.0f);
    const uint32_t x0 = min((uint32_t)fx, p.sw - 1u), y0 = min((uint32_t)fy, p.sh - 1u);
    const uint32_t x1 = min(x0 + 1u, p.sw - 1u);
    const float wx = fx - (float)x0, wy = fy - (float)y0;
    // a zero vertical weight drops the y1 row exactly (see fs_row<SINGLE>): alias it to y0, which a compacted source
    // (row map) is guaranteed to hold
    const uint32_t y1 = (wy == 0.0f) ? y0 : min(y0 + 1u, p.sh - 1u);
    const uint8_t* row0 = s + (size_t)fused_row_slot(p, y0) * p.sw * 3;
    const uint8_t* row1 = s + (size_t)fused_row_slot(p, y1) * p.sw * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float a = (float)row0[x0 * 3 + c], b = (float)row0[x1 * 3 + c];
        const float cc = (float)row1[x0 * 3 + c], dd = (float)row1[x1 * 3 + c];
        d[c * plane] = fused_out<T>(fused_lerp(a, b, cc, dd, wx, wy, p.scale[c], p.bias[c], fused));
    }
}

template <typename T>
int launch_fused_resize_rows(cudaStream_t s, const uint8_t* src, T* dst, const FusedParams& p, uint32_t batch, bool* handled);

FusedParams make_fused_params(uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, const float scale[3], const float bias[3], int leaf) {
    FusedParams p;
    p.sw = sw; p.sh = sh; p.dw = dw; p.dh = dh;
    p.scale_x = (float)sw / (float)dw;
    p.scale_y = (float)sh / (float)dh;
    for (int c = 0; c < 3; ++c) { p.scale[c] = scale[c]; p.bias[c] = bias[c]; }
    const bool box2x = (sw == 2 * dw && sh == 2 * dh);
    if (leaf == KB200_LEAF_SCALAR) p.fma_bulk = 0;
    else if (box2x) p.fma_bulk = dw & ~15u;                          // fused_row_avx2 / fused_row_neon: 16 px per iter
    else p.fma_bulk = (leaf == KB200_LEAF_X86_AVX2_FMA) ? (dw & ~7u) : (dw & ~3u);  // :448 / :355
    p.row_p = 1; p.row_f = 0; p.row_k = 1; p.src_rows = sh;
    return p;
}

// Which source rows does this vertical geometry tap?  Walks every destination row with the sampler's own f32
// expression (identical on host and device: mul, add, no contraction) and fits the tapped set to a periodic window
// "rows y with first <= y mod period < first + keep".  Integer downscales fit exactly (3:1 -> period 3, first 1,
// keep 1; 4:1 -> period 4, first 1, keep 2); anything else reports the dense map (1, 0, 1).
void resize_row_plan(uint32_t sh, uint32_t dh, uint32_t* period, uint32_t* first, uint32_t* keep) {
    *period = 1; *first = 0; *keep = 1;
    if (dh == 0 || sh % dh != 0) return;
    const uint32_t P = sh / dh;
    if (P < 3 || (sh == 2 * dh)) return;
    const float scale_y = (float)sh / (float)dh;
    uint32_t lo = P, hi = 0;
    for (uint32_t d = 0; d < dh; ++d) {
        const float f = std::max(((float)d + 0.5f) * scale_y - 0.5f, 0.0f);
        const uint32_t y0 = std::min((uint32_t)f, sh - 1u);
        const float wy = f - (float)y0;
        const uint32_t y1 = (wy == 0.0f) ? y0 : std::min(y0 + 1u, sh - 1u);
        if (y0 / P != d || y1 / P != d) return;  // a tap leaves its own period: no compact window
        lo = std::min(lo, y0 % P); hi = std::max(hi, y1 % P);
    }
    if (hi - lo + 1 >= P) return;
    *period = P; *first = lo; *keep = hi - lo + 1;
}

template <typename T>
int launch_fused_resize(cudaStream_t s, const uint8_t* src, T* dst, const FusedParams& p, uint32_t batch) {
    const bool box2x = (p.sw == 2 * p.dw && p.sh == 2 * p.dh);
    {
        bool handled = false;
        KB200_TRY(launch_fused_resize_rows(s, src, dst, p, batch, &handled));
        if (handled) return KB200_OK;
    }
    dim3 block(32, 8), grid(div_up(p.dw, 32), div_up(p.dh, 8), batch);
    if (box2x) fused_resize_gather_kernel<T, true><<<grid, block, 0, s>>>(src, dst, p);
    else fused_resize_gather_kernel<T, false><<<grid, block, 0, s>>>(src, dst, p);
    return check_launch("fused_resize_gather_kernel");
}
template int launch_fused_resize<float>(cudaStream_t, const uint8_t*, float*, const FusedParams&, uint32_t);
template int launch_fused_resize<__half>(cudaStream_t, const uint8_t*, __half*, const FusedParams&, uint32_t);
template int launch_fused_resize<__nv_bfloat16>(cudaStream_t, const uint8_t*, __nv_bfloat16*, const FusedParams&, uint32_t);

}  // namespace kb200

using namespace kb200;

// Device-buffer entry points: one validation for every output type (dst_len counts elements).
template <typename T>
static int resize_normalize_chw(kb200_stream_t stream, const uint8_t* src, size_t src_len, T* dst, size_t dst_len, uint32_t sw,
                                uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch, const float scale[3], const float bias[3],
                                int leaf) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_ptr("scale", scale)); KB200_TRY(check_ptr("bias", bias));
    if (leaf < 0 || leaf > 2) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown cpu leaf %d", leaf);
    if (batch == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "batch must be non-zero");
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    // InvalidChannelShape checks of resize/fused.rs:156-167 (lengths must cover the images)
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * 3 * batch));
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * 3 * batch));
    if (dw == 0 || dh == 0 || sw == 0 || sh == 0) return KB200_OK;  // resize/fused.rs:184-186: empty is a no-op
    FusedParams p = make_fused_params(sw, sh, dw, dh, scale, bias, leaf);
    return launch_fused_resize(as_stream(stream), src, dst, p, batch);
}

extern "C" {

KB200_API int kb200_resize_normalize_chw_u8_f32(kb200_stream_t stream, const uint8_t* src, size_t src_len,
                                                float* dst, size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw,
                                                uint32_t dh, uint32_t batch, const float scale[3],
                                                const float bias[3], int leaf) {
    return resize_normalize_chw(stream, src, src_len, dst, dst_len, sw, sh, dw, dh, batch, scale, bias, leaf);
}

KB200_API int kb200_resize_normalize_chw_u8_f16(kb200_stream_t stream, const uint8_t* src, size_t src_len,
                                                uint16_t* dst, size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw,
                                                uint32_t dh, uint32_t batch, const float scale[3],
                                                const float bias[3], int leaf) {
    return resize_normalize_chw(stream, src, src_len, reinterpret_cast<__half*>(dst), dst_len, sw, sh, dw, dh, batch, scale, bias, leaf);
}

KB200_API int kb200_resize_normalize_chw_u8_bf16(kb200_stream_t stream, const uint8_t* src, size_t src_len,
                                                 uint16_t* dst, size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw,
                                                 uint32_t dh, uint32_t batch, const float scale[3],
                                                 const float bias[3], int leaf) {
    return resize_normalize_chw(stream, src, src_len, reinterpret_cast<__nv_bfloat16*>(dst), dst_len, sw, sh, dw, dh, batch, scale,
                                bias, leaf);
}

KB200_API int kb200_resize_normalize_chw_u8_f32_rows(kb200_stream_t stream, const uint8_t* src, size_t src_len,
                                                     float* dst, size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw,
                                                     uint32_t dh, uint32_t batch, const float scale[3],
                                                     const float bias[3], int leaf, uint32_t row_period,
                                                     uint32_t row_first, uint32_t row_keep) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_ptr("scale", scale)); KB200_TRY(check_ptr("bias", bias));
    if (leaf < 0 || leaf > 2) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown cpu leaf %d", leaf);
    if (batch == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "batch must be non-zero");
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    if (dw == 0 || dh == 0 || sw == 0 || sh == 0) return KB200_OK;
    uint32_t P = 1, F = 0, K = 1;
    resize_row_plan(sh, dh, &P, &F, &K);
    if (row_period == 0 || row_keep == 0 || row_first + row_keep > row_period || sh % row_period != 0)
        return fail(KB200_ERR_INVALID_ARGUMENT, "row map (period %u, first %u, keep %u) is not a partition of %u rows",
                    row_period, row_first, row_keep, sh);
    // the supplied map must hold every row this geometry taps: either dense, or exactly the plan
    const bool dense = (row_first == 0 && row_keep == row_period);
    if (!dense && !(row_period == P && row_first == F && row_keep == K))
        return fail(KB200_ERR_INVALID_ARGUMENT, "row map (period %u, first %u, keep %u) does not hold the rows %ux%u -> %ux%u taps (plan: %u, %u, %u)",
                    row_period, row_first, row_keep, sw, sh, dw, dh, P, F, K);
    FusedParams p = make_fused_params(sw, sh, dw, dh, scale, bias, leaf);
    if (!dense) { p.row_p = row_period; p.row_f = row_first; p.row_k = row_keep; p.src_rows = sh / row_period * row_keep; }
    KB200_TRY(check_slice("src", src_len, (size_t)sw * p.src_rows * 3 * batch));
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * 3 * batch));
    return launch_fused_resize(as_stream(stream), src, dst, p, batch);
}

KB200_API void kb200_resize_row_plan(uint32_t src_h, uint32_t dst_h, uint32_t* period, uint32_t* first, uint32_t* keep) {
    uint32_t P = 1, F = 0, K = 1;
    if (src_h && dst_h) resize_row_plan(src_h, dst_h, &P, &F, &K);
    if (period) *period = P;
    if (first) *first = F;
    if (keep) *keep = K;
}

}  // extern "C"

// ─────────────────────────────────────────────────────────────────────────────────────────────
// Row-span staged kernel (the config-2 fast path).
//
// ncu history: the gather kernel above is instruction-bound.  A first staged kernel (TMA row spans, one destination
// column per thread) cut the instructions per pixel but was still issue-bound: ~45 of those instructions were per-ROW bookkeeping repeated for a single pixel.  The kernel below keeps
// the staging scheme and spreads that bookkeeping over several pixels per thread (point mode is
// DRAM-bound):
//
//   * work unit = (image, column tile of TW destination columns, chunk of RC destination rows); CTAs are
//     persistent and walk their units with carry arithmetic (no integer division in the loop).
//   * per destination row, the source rows it taps are copied — only the byte span [x0(first col), x1(last col)]
//     the column tile touches, rounded out to 16 B — global -> shared by the TMA engine (cp.async.bulk 1-D, SASS
//     UBLKCP), completion counted on an mbarrier (expect_tx).  Source rows with no (or a zero) weight are never
//     addressed: 2 of every 3 at scale 3.
//   * a short ring (3 stages), one destination row per stage, running continuously across units.  Warp 4 is the
//     producer (one elected lane: wait `empty`, publish the row's y-weight, issue the copies); warps 0-3 are
//     consumers (wait `full`, compute one row, arrive on `empty`).  No __syncthreads in the loop.
//   * the x-side of the sampler (fx, x0, wx, smem byte offset, funnel shift) is computed once per unit per column
//     and lives in registers.
//   * taps are read as three aligned 32-bit words per source row and funnel-shifted into place; a byte becomes a
//     float with one PRMT into the mantissa of 2^23; `b - a` is formed on the biased values (exact) and only the
//     base taps are unbiased (one FADD).
//   * stores: a warp writes 32 consecutive values of one channel plane = one full 128-B line (f32), or two full
//     32-B sectors (f16 / bf16: element alignment is all a store needs).
//
// Arithmetic is identical to the gather kernel (and therefore to the reference leaf selected).
namespace kb200 {

struct FusedStagedParams {
    FusedParams p;
    uint32_t tiles_x, chunks_y, rows_per_chunk, nunits;
    uint32_t slot_bytes;   // bytes reserved per staged source-row span (multiple of 128)
    uint32_t row_bytes;    // sw * 3
    // CTA stride decomposed for the carry walk: gridDim.x = (dimg*chunks_y + dcy)*tiles_x + dtx
    uint32_t dtx, dcy, dimg;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
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
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D bulk copy global -> shared::cta through the TMA engine; bytes % 16 == 0, both addresses 16-B aligned.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// half-pixel source coordinate of the fused path — resize/fused.rs:196-201 (unfused mul/add)
__device__ __forceinline__ void fused_axis(uint32_t d, float scale, uint32_t src_len, uint32_t* i0, uint32_t* i1, float* w) {
    const float f = fmaxf(((float)d + 0.5f) * scale - 0.5f, 0.0f);
    const uint32_t a = min((uint32_t)f, src_len - 1u);
    *i0 = a;
    *i1 = min(a + 1u, src_len - 1u);
    *w = f - (float)a;
}

// (tx, chunk, img) walk: advance by one CTA stride without dividing.
struct UnitWalk {
    uint32_t tx, cy, img;
    __device__ __forceinline__ void init(uint32_t u, const FusedStagedParams& P) {
        const uint32_t per_img = P.tiles_x * P.chunks_y;
        img = u / per_img;
        const uint32_t t = u - img * per_img;
        cy = t / P.tiles_x;
        tx = t - cy * P.tiles_x;
    }
    __device__ __forceinline__ void advance(const FusedStagedParams& P) {
        tx += P.dtx; cy += P.dcy; img += P.dimg;
        if (tx >= P.tiles_x) { tx -= P.tiles_x; ++cy; }
        if (cy >= P.chunks_y) { cy -= P.chunks_y; ++img; }
        if (cy >= P.chunks_y) { cy -= P.chunks_y; ++img; }
    }
};

// Several destination columns per thread + per-launch specialisation.
//
// A consumer thread owns NPX columns (t, t+128, ..., all lane-contiguous), so the per-row bookkeeping (mbarrier
// wait/arrive, ring index, pointer bumps) is paid once per NPX pixels, and the sampler is specialised per LAUNCH on
// what the geometry makes exactly zero:
//
//   FR_GENERAL  two source rows per destination row (the y1 row is skipped by the producer when its weight is 0;
//               the consumer then multiplies stale-but-finite bytes by 0, which is exact).
//   FR_YZERO    every destination row has wy == 0 (odd integer vertical ratio, or 1:1): one source row per stage.
//   FR_POINT    additionally every column has wx == 0: out = byte * scale + bias — three byte loads per pixel.
//   FR_BOX      exact 2x downscale (resize/fused.rs:57-127): the integer sum of the 2x2 block times scale/4.  The
//               half-pixel sampler at scale 2 taps exactly the block's rows and columns (x0 = 2d, y0 = 2d), so the
//               staging is the general one; the four byte sums per channel are IDP4A dot products with 0/1 masks.
//
// A right-edge column (x1 == x0) is folded into the general arithmetic by forcing wx = 0: b == a there, so
// a + wx*(b-a) == a for any wx, and with wx = 0 the (finite) neighbour byte that is read instead contributes ±0.
static constexpr int FR_CT = 128;               // consumer threads per CTA
static constexpr int FR_THREADS = FR_CT + 32;   // + producer warp
static constexpr int FR_MAX_STAGES = 16;
enum { FR_GENERAL = 0, FR_YZERO = 1, FR_POINT = 2, FR_BOX = 3 };

struct FusedRowsParams {
    FusedStagedParams g;   // geometry + unit walk (tiles_x counts tiles of FR_CT*NPX columns)
    uint32_t stages;       // ring depth
    uint32_t stage_bytes;  // slot_bytes * (rows staged per destination row)
};

template <int MODE>
__device__ __forceinline__ void fr_pixel(const uint8_t* __restrict__ rp, uint32_t slot_bytes, uint32_t shft, float wx, float wy, bool fma_leaf,
                                         float s0, float s1, float s2, float o0, float o1, float o2, float& q0, float& q1, float& q2) {
    float v[3];
    if (MODE == FR_BOX) {
        const uint32_t* r0 = reinterpret_cast<const uint32_t*>(rp);
        const uint32_t* r1 = reinterpret_cast<const uint32_t*>(rp + slot_bytes);
        const uint32_t a0 = r0[0], a1 = r0[1], a2 = r0[2], c0 = r1[0], c1 = r1[1], c2 = r1[2];
        const uint32_t lo0 = __funnelshift_r(a0, a1, shft), hi0 = __funnelshift_r(a1, a2, shft);  // r0 g0 b0 r1 | g1 b1 . .
        const uint32_t lo1 = __funnelshift_r(c0, c1, shft), hi1 = __funnelshift_r(c1, c2, shft);
        // sums of resize/fused.rs:543-548: u32 adds of four bytes — exact, order-free
        const uint32_t sr = __dp4a(lo0, 0x01000001u, __dp4a(lo1, 0x01000001u, 0u));
        const uint32_t sg = __dp4a(lo0, 0x00000100u, __dp4a(hi0, 0x00000001u, __dp4a(lo1, 0x00000100u, __dp4a(hi1, 0x00000001u, 0u))));
        const uint32_t sb = __dp4a(lo0, 0x00010000u, __dp4a(hi0, 0x00000100u, __dp4a(lo1, 0x00010000u, __dp4a(hi1, 0x00000100u, 0u))));
        // s0..s2 carry scale[c] * 0.25f here (formed once per thread, the reference forms it once per row)
        const float fr = (float)sr, fg = (float)sg, fb = (float)sb;
        if (fma_leaf) { q0 = fmaf(fr, s0, o0); q1 = fmaf(fg, s1, o1); q2 = fmaf(fb, s2, o2); }
        else          { q0 = fr * s0 + o0;     q1 = fg * s1 + o1;     q2 = fb * s2 + o2; }
        return;
    }
    if (MODE == FR_POINT) {
        v[0] = (float)rp[0]; v[1] = (float)rp[1]; v[2] = (float)rp[2];
    } else {
        const uint32_t* r0 = reinterpret_cast<const uint32_t*>(rp);
        const uint32_t a0 = r0[0], a1 = r0[1], a2 = r0[2];
        const uint32_t lo0 = __funnelshift_r(a0, a1, shft), hi0 = __funnelshift_r(a1, a2, shft);  // bytes off..off+3 | off+4..off+7
        uint32_t lo1 = 0, hi1 = 0;
        if (MODE == FR_GENERAL) {
            const uint32_t* r1 = reinterpret_cast<const uint32_t*>(rp + slot_bytes);
            const uint32_t c0 = r1[0], c1 = r1[1], c2 = r1[2];
            lo1 = __funnelshift_r(c0, c1, shft); hi1 = __funnelshift_r(c1, c2, shft);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            // biased floats 2^23 + byte: a = tap(x0,y0), b = tap(x1,y0), c = tap(x0,y1), d = tap(x1,y1)
            const float ab = __uint_as_float(__byte_perm(lo0, 0x4B000000u, 0x7650u + (uint32_t)c));
            const float bb = __uint_as_float(c == 0 ? __byte_perm(lo0, 0x4B000000u, 0x7653u) : __byte_perm(hi0, 0x4B000000u, 0x7650u + (uint32_t)(c - 1)));
            const float a = ab - 8388608.0f;  // exact
            const float dba = bb - ab;        // exact: (2^23+b) - (2^23+a) = b - a
            const float top = fma_leaf ? fmaf(dba, wx, a) : a + wx * dba;   // resize/fused.rs:475 | :286
            if (MODE == FR_YZERO) { v[c] = top; continue; }
            const float cb = __uint_as_float(__byte_perm(lo1, 0x4B000000u, 0x7650u + (uint32_t)c));
            const float db = __uint_as_float(c == 0 ? __byte_perm(lo1, 0x4B000000u, 0x7653u) : __byte_perm(hi1, 0x4B000000u, 0x7650u + (uint32_t)(c - 1)));
            const float cc = cb - 8388608.0f, ddc = db - cb;
            const float bot = fma_leaf ? fmaf(ddc, wx, cc) : cc + wx * ddc;
            v[c] = fma_leaf ? fmaf(bot - top, wy, top) : top + wy * (bot - top);
        }
    }
    if (fma_leaf) { q0 = fmaf(v[0], s0, o0); q1 = fmaf(v[1], s1, o1); q2 = fmaf(v[2], s2, o2); }   // resize/fused.rs:478
    else          { q0 = v[0] * s0 + o0;     q1 = v[1] * s1 + o1;     q2 = v[2] * s2 + o2; }       // :317
}

template <typename T, int NPX, int MODE, bool ALLFMA>
__global__ void __launch_bounds__(FR_THREADS) fused_rows_kernel(const uint8_t* __restrict__ src, T* __restrict__ dst,
                                                                const __grid_constant__ FusedRowsParams R) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[FR_MAX_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[FR_MAX_STAGES];
    __shared__ float wy_s[FR_MAX_STAGES];
    constexpr uint32_t TW = FR_CT * NPX;
    const FusedStagedParams& P = R.g;
    const FusedParams& p = P.p;
    const uint32_t tid = threadIdx.x;
    const uint32_t nst = R.stages;
    const size_t frame_bytes = (size_t)P.row_bytes * p.src_rows;
    const size_t plane = (size_t)p.dw * p.dh;

    if (tid == 0) {
        for (uint32_t s = 0; s < nst; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], FR_CT / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    UnitWalk w;
    w.init(blockIdx.x, P);
    uint32_t stage = 0, phase = 0;  // ring position, running continuously across units

    if (tid >= FR_CT) {
        // ── producer warp: one elected lane ──
        if (tid != FR_CT) return;
        bool first_lap = true;
        for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x, w.advance(P)) {
            const uint32_t dx0 = w.tx * TW, dx1 = min(dx0 + TW, p.dw) - 1u;
            uint32_t xa, xb, tmp;
            float wtmp;
            fused_axis(dx0, p.scale_x, p.sw, &xa, &tmp, &wtmp);
            fused_axis(dx1, p.scale_x, p.sw, &tmp, &xb, &wtmp);
            const uint32_t b0 = (xa * 3u) & ~15u;                                 // span start, 16-B aligned
            const uint32_t b1 = min(((xb * 3u + 3u) + 15u) & ~15u, P.row_bytes);  // span end (row_bytes % 16 == 0)
            const uint32_t bytes = b1 - b0;
            const uint8_t* frame = src + (size_t)w.img * frame_bytes + b0;
            const uint32_t y_first = w.cy * P.rows_per_chunk, y_end = min(y_first + P.rows_per_chunk, p.dh);
            for (uint32_t dy = y_first; dy < y_end; ++dy) {
                if (!first_lap) mbar_wait(&empty_bar[stage], phase ^ 1u);  // consumers drained the previous tenant
                uint32_t y0, y1;
                float wy;
                fused_axis(dy, p.scale_y, p.sh, &y0, &y1, &wy);
                uint8_t* sbase = smem_raw + (size_t)stage * R.stage_bytes;
                const bool two = (MODE == FR_BOX) || ((MODE == FR_GENERAL) && (wy != 0.0f));  // a zero-weight y1 row is never fetched
                if (MODE == FR_GENERAL) wy_s[stage] = wy;  // before the arrive(release): covered by the consumers' acquire on `full`
                mbar_expect_tx(&full_bar[stage], two ? bytes * 2u : bytes);
                tma_load_1d(sbase, frame + (size_t)fused_row_slot(p, y0) * P.row_bytes, bytes, &full_bar[stage]);
                if (two) tma_load_1d(sbase + P.slot_bytes, frame + (size_t)fused_row_slot(p, y1) * P.row_bytes, bytes, &full_bar[stage]);
                if (++stage == nst) { stage = 0; phase ^= 1u; first_lap = false; }
            }
        }
        return;
    }

    // ── consumer warps ──
    const float qs = (MODE == FR_BOX) ? 0.25f : 1.0f;   // box: scale[c] * 0.25f (resize/fused.rs:541); x * 1.0f is exact
    const float s0 = p.scale[0] * qs, s1 = p.scale[1] * qs, s2 = p.scale[2] * qs;
    const float o0 = p.bias[0], o1 = p.bias[1], o2 = p.bias[2];
    const bool lane0 = (tid & 31u) == 0;
    for (uint32_t u = blockIdx.x; u < P.nunits; u += gridDim.x, w.advance(P)) {
        const uint32_t dx0 = w.tx * TW;
        uint32_t xa, tmp;
        float wtmp;
        fused_axis(dx0, p.scale_x, p.sw, &xa, &tmp, &wtmp);
        const uint32_t b0 = (xa * 3u) & ~15u;
        // x-side of the sampler, once per unit, for this thread's NPX columns
        uint32_t off[NPX], shft[NPX];
        float wx[NPX];
        uint32_t act = 0, fm = 0;
#pragma unroll
        for (int j = 0; j < NPX; ++j) {
            const uint32_t x = dx0 + tid + (uint32_t)j * FR_CT;
            uint32_t x0, x1;
            fused_axis(min(x, p.dw - 1u), p.scale_x, p.sw, &x0, &x1, &wx[j]);
            if (x1 == x0) wx[j] = 0.0f;                      // right edge: b == a, any weight gives a — use the exact one
            const uint32_t ob = x0 * 3u - b0;                // byte offset of tap x0 inside the staged span
            if (MODE == FR_POINT) { off[j] = ob; shft[j] = 0; }
            else { off[j] = ob & ~3u; shft[j] = (ob & 3u) * 8u; }
            act |= (x < p.dw ? 1u : 0u) << j;
            fm |= (x < p.fma_bulk ? 1u : 0u) << j;
        }
        const uint32_t y_first = w.cy * P.rows_per_chunk, y_end = min(y_first + P.rows_per_chunk, p.dh);
        T* out0 = dst + (size_t)w.img * plane * 3 + (size_t)y_first * p.dw + dx0 + tid;
        T* out1 = out0 + plane;
        T* out2 = out1 + plane;
        for (uint32_t dy = y_first; dy < y_end; ++dy) {
            mbar_wait(&full_bar[stage], phase);
            const uint8_t* sbase = smem_raw + (size_t)stage * R.stage_bytes;
            const float wy = (MODE == FR_GENERAL) ? wy_s[stage] : 0.0f;
#pragma unroll
            for (int j = 0; j < NPX; ++j) {
                float q0, q1, q2;
                fr_pixel<MODE>(sbase + off[j], P.slot_bytes, shft[j], wx[j], wy, ALLFMA || ((fm >> j) & 1u), s0, s1, s2, o0, o1, o2, q0, q1, q2);
                if ((act >> j) & 1u) { out0[j * FR_CT] = fused_out<T>(q0); out1[j * FR_CT] = fused_out<T>(q1); out2[j * FR_CT] = fused_out<T>(q2); }
            }
            out0 += p.dw; out1 += p.dw; out2 += p.dw;
            __syncwarp();
            if (lane0) mbar_arrive(&empty_bar[stage]);
            if (++stage == nst) { stage = 0; phase ^= 1u; }
        }
    }
}

// Are all the sampler's weights along one axis exactly zero (with the right-edge rule above)?  Same f32 expression
// as the device (mul, add; no contraction), evaluated on the host once per launch.
static bool axis_weights_all_zero(uint32_t dst_len, uint32_t src_len, float scale) {
    for (uint32_t d = 0; d < dst_len; ++d) {
        const float f = std::max(((float)d + 0.5f) * scale - 0.5f, 0.0f);
        const uint32_t a = std::min((uint32_t)f, src_len - 1u);
        const uint32_t b = std::min(a + 1u, src_len - 1u);
        if (b != a && f - (float)a != 0.0f) return false;
    }
    return true;
}

template <typename T, int NPX, int MODE>
static cudaError_t fr_launch(bool allfma, unsigned grid, size_t smem, cudaStream_t s, const uint8_t* src, T* dst, const FusedRowsParams& R) {
    auto go = [&](auto kern) -> cudaError_t {
        if (smem > 40 * 1024) {
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
        }
        kern<<<grid, FR_THREADS, smem, s>>>(src, dst, R);
        return cudaSuccess;
    };
    return allfma ? go(fused_rows_kernel<T, NPX, MODE, true>) : go(fused_rows_kernel<T, NPX, MODE, false>);
}

template <typename T, int MODE>
static cudaError_t fr_launch_npx(int npx, bool allfma, unsigned grid, size_t smem, cudaStream_t s, const uint8_t* src, T* dst, const FusedRowsParams& R) {
    switch (npx) {
        case 1: return fr_launch<T, 1, MODE>(allfma, grid, smem, s, src, dst, R);
        case 2: return fr_launch<T, 2, MODE>(allfma, grid, smem, s, src, dst, R);
        case 3: return fr_launch<T, 3, MODE>(allfma, grid, smem, s, src, dst, R);
        case 4: return fr_launch<T, 4, MODE>(allfma, grid, smem, s, src, dst, R);
        default: return fr_launch<T, 5, MODE>(allfma, grid, smem, s, src, dst, R);
    }
}

// Geometry, mode, npx, ring depth and CTA count depend on the source side only: the same for every output type.
template <typename T>
int launch_fused_resize_rows(cudaStream_t s, const uint8_t* src, T* dst, const FusedParams& p, uint32_t batch, bool* handled) {
    *handled = false;
    const uint32_t row_bytes = p.sw * 3u;
    // TMA 1-D bulk copies need 16-B aligned rows; very strong downscales have sparse taps (the span would be
    // mostly unused bytes) and stay on the gather kernel.
    if ((row_bytes & 15u) || !aligned16(src) || p.scale_x > 6.0f || p.sw < 16u) return KB200_OK;
    // developer knobs (tuning sweeps only, kb200_debug_set_knob): fr.npx, fr.stages, fr.ctas
    const int tune_npx = knob(KNOB_FR_NPX), tune_stages = knob(KNOB_FR_STAGES), tune_ctas = knob(KNOB_FR_CTAS);
    const bool yz = axis_weights_all_zero(p.dh, p.sh, p.scale_y);
    const bool xz = yz && axis_weights_all_zero(p.dw, p.sw, p.scale_x);
    const bool box2x = (p.sw == 2 * p.dw && p.sh == 2 * p.dh);
    const int mode = box2x ? FR_BOX : (xz ? FR_POINT : (yz ? FR_YZERO : FR_GENERAL));
    // columns per thread: least padding in the last tile; among near-equals prefer 2, then 3, 1, 4, 5 — 2 columns/thread
    // give enough amortisation and many producers.  The general mode (two source rows and a full lerp per pixel) is
    // heavier per pixel: it accepts up to 10 % tile padding to keep >= 2 columns per thread.
    int npx = 1;
    {
        static const int order[5] = {2, 3, 1, 4, 5};
        const double tol = mode == FR_GENERAL ? 0.10 : 0.02;
        double best = 1e30;
        for (int i = 0; i < 5; ++i) {
            const uint32_t tw = FR_CT * order[i];
            const double waste = (double)((p.dw + tw - 1) / tw) * tw / (double)p.dw;
            if (waste < best - tol) { best = waste; npx = order[i]; }
        }
        if (tune_npx >= 1 && tune_npx <= 5) npx = tune_npx;
    }
    const uint32_t TW = FR_CT * (uint32_t)npx;
    // span bound: x0(last) - x0(first) <= ceil((TW-1)*scale_x) + 1 pixels, + the +1 tap, + 16-B rounding both ends
    const double span_px = (double)(TW - 1) * (double)p.scale_x + 4.0;
    uint32_t slot = (uint32_t)(span_px * 3.0) + 32u;
    slot = (slot + 127u) & ~127u;
    slot = std::min(slot, (row_bytes + 16u + 127u) & ~127u);  // +16: the 3-word tap read may run 8 B past the span
    const uint32_t stage_bytes = slot * ((mode == FR_GENERAL || mode == FR_BOX) ? 2u : 1u);
    // Ring sizing: ~36 KB of source rows in flight per SM (about bandwidth x latency for the whole GPU); the general mode
    // runs 4 CTAs x 3 stages.  H100 sweep (npx 1..3 x stages 3/4/6 x CTAs 2..8): the point / box / general defaults are
    // within 3 % of the best configuration (general: 4 stages was 5 % slower than 3).  Knobs fr.* re-sweep them.
    uint32_t stages = tune_stages >= 2 && tune_stages <= FR_MAX_STAGES ? (uint32_t)tune_stages : 3u;
    int per_sm = tune_ctas > 0 ? tune_ctas : (mode == FR_GENERAL ? 4 : (int)std::lround(36.0 * 1024.0 / ((double)stages * stage_bytes)));
    per_sm = std::max(2, std::min(per_sm, 8));
    while (per_sm > 2 && (size_t)per_sm * ((size_t)stages * stage_bytes + 1024) > 200 * 1024) --per_sm;
    if (tune_ctas <= 0 && tune_stages <= 0 && per_sm == 2) stages = std::min<uint32_t>(FR_MAX_STAGES, std::max<uint32_t>(3u, (uint32_t)(18.0 * 1024.0 / stage_bytes)));
    if (stages < 3) return KB200_OK;
    const size_t smem = (size_t)stage_bytes * stages;
    if (smem > 200 * 1024) return KB200_OK;

    FusedRowsParams R;
    FusedStagedParams& P = R.g;
    P.p = p;
    P.tiles_x = (p.dw + TW - 1) / TW;
    const size_t ctas = (size_t)device_info().sm_count * per_sm;
    // chunk height: enough units for ~16 per CTA (load balance) but at least 8 rows (amortise the x-side)
    const size_t total_rows = (size_t)p.dh * batch * P.tiles_x;
    uint32_t rc = (uint32_t)std::max<size_t>(8, total_rows / (ctas * 16));
    rc = std::min(rc, p.dh);
    P.rows_per_chunk = rc;
    P.chunks_y = (p.dh + rc - 1) / rc;
    const size_t nunits = (size_t)P.tiles_x * P.chunks_y * batch;
    if (nunits > 0x7FFFFFFFull) return KB200_OK;
    P.nunits = (uint32_t)nunits;
    P.slot_bytes = slot;
    P.row_bytes = row_bytes;
    R.stages = stages;
    R.stage_bytes = stage_bytes;
    const unsigned grid = (unsigned)std::min<size_t>(nunits, ctas);
    P.dtx = grid % P.tiles_x;
    const uint32_t g = grid / P.tiles_x;
    P.dcy = g % P.chunks_y;
    P.dimg = g / P.chunks_y;
    const bool allfma = p.fma_bulk >= p.dw;
    cudaError_t e;
    if (mode == FR_POINT) e = fr_launch_npx<T, FR_POINT>(npx, allfma, grid, smem, s, src, dst, R);
    else if (mode == FR_YZERO) e = fr_launch_npx<T, FR_YZERO>(npx, allfma, grid, smem, s, src, dst, R);
    else if (mode == FR_BOX) e = fr_launch_npx<T, FR_BOX>(npx, allfma, grid, smem, s, src, dst, R);
    else e = fr_launch_npx<T, FR_GENERAL>(npx, allfma, grid, smem, s, src, dst, R);
    if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    KB200_TRY(check_launch("fused_rows_kernel"));
    *handled = true;
    return KB200_OK;
}
template int launch_fused_resize_rows<float>(cudaStream_t, const uint8_t*, float*, const FusedParams&, uint32_t, bool*);
template int launch_fused_resize_rows<__half>(cudaStream_t, const uint8_t*, __half*, const FusedParams&, uint32_t, bool*);
template int launch_fused_resize_rows<__nv_bfloat16>(cudaStream_t, const uint8_t*, __nv_bfloat16*, const FusedParams&, uint32_t, bool*);

}  // namespace kb200
