// color.cu — gray_from_rgb (f32, u8), the Q20 video decoders (4:2:0: NV12, NV21, I420, YV12; 4:2:2: YUYV, UYVY, YVYU;
// 4:4:4: I444; BT.601 or BT.709, limited or full range: kb200_yuv_matrix), their Q16 forms for 10- and 12-bit codes
// (P010, P012, I010, I012; I410, I412 and their MSB-aligned forms) and the bilinear Bayer demosaic (RGGB, BGGR, GRBG, GBRG; bayer.cuh).
//
// Reference: color/gray/kernels.rs (CPU), cuda/color/gray.rs:17-68 (GPU twin, 1 px or 4 px per
// thread, scalar 4-byte accesses); color/yuv/kernels.rs:707-1069 (CPU), cuda/color/video.rs:33-130
// (GPU twin, 1 thread per 2x2 block, byte stores).
//
// Design: these are pure streaming ops (16 B/px, 4 B/px, 4.5 B/px, 5 B/px).  Every thread
// moves whole 16-byte vectors in both directions (LDG.128 / STG.128, streaming cache hints),
// de-interleaving the stride-3 pixels in registers; grids are sized so each SM holds several
// CTAs with ≥ 4 independent 16-byte loads in flight per thread.
#include "bayer.cuh"
#include "kb200_common.cuh"

namespace kb200 {

static constexpr float RW = 0.299f, GW = 0.587f, BW = 0.114f;  // color/gray/kernels.rs:2-4

// scalar leaf: rw*r + gw*g + bw*b, left to right, unfused  (kernels.rs:405-410, cuda/color/gray.rs:55-68)
// x86 AVX2+FMA leaf: fma(r,rw, fma(g,gw, b*bw)) on the npixels&~7 bulk (kernels.rs:338-402)
__device__ __forceinline__ float gray_px(float r, float g, float b, bool fused) {
    if (fused) return fmaf(r, RW, fmaf(g, GW, b * BW));
    return RW * r + GW * g + BW * b;
}

// 4 px per thread: 3 x LDG.128 in, 1 x STG.128 out.
__global__ void __launch_bounds__(256) gray_from_rgb_f32_vec4(const float4* __restrict__ src, float4* __restrict__ dst,
                                                              size_t nquads, size_t bulk_px) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < nquads; q += stride) {
        // L1-allocating loads: the three vectors of a thread interleave with its neighbours' (48-B lane stride), so the
        // second and third instruction hit the sectors the first one brought in
        const float4 a = __ldg(src + 3 * q);      // r0 g0 b0 r1
        const float4 b = __ldg(src + 3 * q + 1);  // g1 b1 r2 g2
        const float4 c = __ldg(src + 3 * q + 2);  // b2 r3 g3 b3
        const size_t p = 4 * q;
        float4 o;
        // bulk_px is a multiple of 8, so the 4 px of a quad are all on one side of it.
        const bool fused = p < bulk_px;
        o.x = gray_px(a.x, a.y, a.z, fused);
        o.y = gray_px(a.w, b.x, b.y, fused);
        o.z = gray_px(b.z, b.w, c.x, fused);
        o.w = gray_px(c.y, c.z, c.w, fused);
        stg_stream_f4(dst + q, o);
    }
}

__global__ void gray_from_rgb_f32_scalar(const float* __restrict__ src, float* __restrict__ dst, size_t first,
                                         size_t npixels, size_t bulk_px) {
    const size_t i = first + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npixels) return;
    dst[i] = gray_px(__ldg(src + 3 * i), __ldg(src + 3 * i + 1), __ldg(src + 3 * i + 2), i < bulk_px);
}

// Q14: (4899 R + 9617 G + 1868 B + 8192) >> 14 — color/gray/kernels.rs:229-238
__device__ __forceinline__ uint32_t gray_q14(uint32_t r, uint32_t g, uint32_t b) {
    return (4899u * r + 9617u * g + 1868u * b + 8192u) >> 14;
}
__device__ __forceinline__ uint32_t byte_of(uint32_t w, int i) { return (w >> (8 * i)) & 0xFFu; }

// 16 px per thread: 3 x LDG.128 (48 B) in, 1 x STG.128 (16 B) out.
__global__ void __launch_bounds__(256) gray_from_rgb_u8_vec16(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                                              size_t ngroups) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < ngroups; q += stride) {
        const uint4 A = __ldg(src + 3 * q), B = __ldg(src + 3 * q + 1), C = __ldg(src + 3 * q + 2);  // L1-allocating (48-B lane stride)
        const uint32_t w[12] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w, C.x, C.y, C.z, C.w};
        uint32_t out[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // 4 px = 12 bytes = 3 words: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
            const uint32_t w0 = w[3 * k], w1 = w[3 * k + 1], w2 = w[3 * k + 2];
            const uint32_t g0 = gray_q14(byte_of(w0, 0), byte_of(w0, 1), byte_of(w0, 2));
            const uint32_t g1 = gray_q14(byte_of(w0, 3), byte_of(w1, 0), byte_of(w1, 1));
            const uint32_t g2 = gray_q14(byte_of(w1, 2), byte_of(w1, 3), byte_of(w2, 0));
            const uint32_t g3 = gray_q14(byte_of(w2, 1), byte_of(w2, 2), byte_of(w2, 3));
            out[k] = g0 | (g1 << 8) | (g2 << 16) | (g3 << 24);
        }
        stg_stream_u4(dst + q, make_uint4(out[0], out[1], out[2], out[3]));
    }
}

__global__ void gray_from_rgb_u8_scalar(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t first,
                                        size_t npixels) {
    const size_t i = first + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npixels) return;
    dst[i] = (uint8_t)gray_q14(src[3 * i], src[3 * i + 1], src[3 * i + 2]);
}

// ── NV12 → RGB8 ─────────────────────────────────────────────────────────────────────────────
// One thread: 16 luma columns x 2 rows (one chroma row).  Loads 16 B Y (top), 16 B Y (bottom),
// 16 B UV; stores 2 x 48 B as 3 x STG.128 each.  Requires width % 16 == 0 and 16-B aligned bases.
// Saturate-and-pack (I2IP): d = (c << 16) | (sat_u8(a) << 8) | sat_u8(b) — one instruction replaces two min/max
// pairs and the byte insertion.  ncu on the min/max version: math-pipe throttled,
// below the HBM roofline.
__device__ __forceinline__ uint32_t pack_sat2(int hi, int lo, uint32_t upper) {
    uint32_t d;
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(hi), "r"(lo), "r"(upper));
    return d;
}
// four saturated bytes, b0 in the low byte
__device__ __forceinline__ uint32_t pack_sat4(int b0, int b1, int b2, int b3) { return pack_sat2(b1, b0, pack_sat2(b3, b2, 0u)); }

// 48 bytes of interleaved 16-bit RGB, r0 g0 b0 r1 ..., two samples per 32-bit word, from rgb[channel][pixel] of 8 pixels.
__device__ __forceinline__ void pack_rgb48_u16(const int (&rgb)[3][8], uint4 o[3]) {
    uint32_t w[12];
#pragma unroll
    for (int m = 0; m < 12; ++m) w[m] = (uint32_t)rgb[(2 * m) % 3][(2 * m) / 3] | ((uint32_t)rgb[(2 * m + 1) % 3][(2 * m + 1) / 3] << 16);
    o[0] = make_uint4(w[0], w[1], w[2], w[3]);
    o[1] = make_uint4(w[4], w[5], w[6], w[7]);
    o[2] = make_uint4(w[8], w[9], w[10], w[11]);
}

__device__ __forceinline__ void pack_rgb16(const uint32_t yw[4], const ChromaTerms ct[8], const YuvCoeffs& yc, uint4 out[3]) {
    uint32_t w[12];
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // 4 px -> 12 bytes = 3 words: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
        int r[4], g[4], b[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int yy = yy_term((int)((yw[k] >> (8 * j)) & 0xFFu), yc);
            const ChromaTerms& t = ct[2 * k + (j >> 1)];
            b[j] = (yy + t.b) >> 20; g[j] = (yy + t.g) >> 20; r[j] = (yy + t.r) >> 20;   // saturated by the pack below
        }
        w[3 * k] = pack_sat4(r[0], g[0], b[0], r[1]);
        w[3 * k + 1] = pack_sat4(g[1], b[1], r[2], g[2]);
        w[3 * k + 2] = pack_sat4(b[2], r[3], g[3], b[3]);
    }
    out[0] = make_uint4(w[0], w[1], w[2], w[3]);
    out[1] = make_uint4(w[4], w[5], w[6], w[7]);
    out[2] = make_uint4(w[8], w[9], w[10], w[11]);
}

// A thread's 48 output bytes are three 16-B chunks at a 48-B lane stride: stored directly, every STG.128 of the warp
// half-fills its sectors (ncu: 2x the L2 write sectors).  The warp's 1536 B are contiguous, so they are transposed
// through shared memory (STS.128 at 48-B stride is conflict-free per quarter-warp) and written as three
// lane-contiguous STG.128.  `stage` = this warp's 1536-B scratch; all 32 lanes must call.
__device__ __forceinline__ void store_rgb48_coalesced(uint4* __restrict__ warp_dst, uint4* __restrict__ stage, uint32_t lane, const uint4 o[3]) {
    stage[3 * lane] = o[0]; stage[3 * lane + 1] = o[1]; stage[3 * lane + 2] = o[2];
    __syncwarp();
    const uint4 a = stage[lane], b = stage[32 + lane], c = stage[64 + lane];
    __syncwarp();
    stg_stream_u4(warp_dst + lane, a); stg_stream_u4(warp_dst + 32 + lane, b); stg_stream_u4(warp_dst + 64 + lane, c);
}

// The warp runs of the row-wise vector decoders: thread gx of a grid row owns COLS columns, so a warp owns 32 * COLS
// contiguous columns of one row and 1536 contiguous output bytes.  A kernel returns when its warp is past the row
// (gx0 * COLS >= width); a ragged last warp of a row stores its active threads' 48 B directly.
template <uint32_t COLS>
struct WarpRun {
    uint32_t gx, lane, gx0;   // the thread's column group, its lane and its warp's first group
    bool full_warp, active;
    __device__ __forceinline__ explicit WarpRun(uint32_t width)
        : gx(blockIdx.x * blockDim.x + threadIdx.x), lane(threadIdx.x & 31u), gx0(gx - lane),
          full_warp((gx0 + 32) * COLS <= width), active(gx * COLS < width) {}
    // d: the warp's run; stage: the warp's 1536-B scratch (store_rgb48_coalesced)
    __device__ __forceinline__ void store(uint4* __restrict__ d, uint4* __restrict__ stage, const uint4 o[3]) const {
        if (full_warp) store_rgb48_coalesced(d, stage, lane, o);
        else if (active) { stg_stream_u4(d + 3 * lane, o[0]); stg_stream_u4(d + 3 * lane + 1, o[1]); stg_stream_u4(d + 3 * lane + 2, o[2]); }
    }
};

// One thread: 16 luma columns x 2 rows (one chroma row) — 16 B Y (top), 16 B Y (bottom) and the 8 chroma pairs: one
// 16-B load of the interleaved row (NV12 / NV21), or 8 B of the U plane and 8 B of the V plane (I420 / YV12; with
// width % 16 == 0 both planes and every thread's offset in them are 8-B aligned).
template <int L>
__global__ void __launch_bounds__(128) rgb_from_yuv420_vec16(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                             uint32_t width, uint32_t height, size_t frame_bytes, const YuvCoeffs yc) {
    __shared__ uint4 stage[4][96];
    const uint32_t gx = blockIdx.x * blockDim.x + threadIdx.x;  // 16-column group
    const uint32_t cy = blockIdx.y;                             // chroma row
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const uint32_t gx0 = gx - lane;                             // first group of this warp
    if (gx0 * 16 >= width) return;                              // whole warp out of the row
    const bool full_warp = (gx0 + 32) * 16 <= width;
    const bool active = gx * 16 < width;
    const uint8_t* frame = src + (size_t)blockIdx.z * frame_bytes;
    uint8_t* out = dst + (size_t)blockIdx.z * (size_t)width * height * 3;
    const size_t x = (size_t)gx * 16;
    uint4 yt = make_uint4(0, 0, 0, 0), yb = yt, uv = yt;   // planar layouts: uv = {U bytes 0-7, V bytes 0-7}
    if (active) {
        yt = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)(2 * cy) * width + x));
        yb = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)(2 * cy + 1) * width + x));
        if (yuv420_planar(L)) {
            const size_t c = (size_t)cy * (width / 2) + x / 2;
            const uint2 u = ldg_stream_u2(reinterpret_cast<const uint2*>(frame + yuv420_u_plane(L, width, height) + c));
            const uint2 v = ldg_stream_u2(reinterpret_cast<const uint2*>(frame + yuv420_v_plane(L, width, height) + c));
            uv = make_uint4(u.x, u.y, v.x, v.y);
        } else {
            uv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)width * height + (size_t)cy * width + x));
        }
    }
    const uint32_t uvw[4] = {uv.x, uv.y, uv.z, uv.w};
    ChromaTerms ct[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (yuv420_planar(L)) {
            ct[k] = chroma_terms((int)((uvw[k >> 2] >> (8 * (k & 3))) & 0xFFu), (int)((uvw[2 + (k >> 2)] >> (8 * (k & 3))) & 0xFFu), yc);
        } else {
            const uint32_t pair = (uvw[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
            if (L == YUV420_NV21) ct[k] = chroma_terms((int)(pair >> 8), (int)(pair & 0xFFu), yc);
            else ct[k] = chroma_terms((int)(pair & 0xFFu), (int)(pair >> 8), yc);
        }
    }
    uint4 o[3];
    const uint32_t ytw[4] = {yt.x, yt.y, yt.z, yt.w};
    const uint32_t ybw[4] = {yb.x, yb.y, yb.z, yb.w};
    uint4* d0 = reinterpret_cast<uint4*>(out + ((size_t)(2 * cy) * width + (size_t)gx0 * 16) * 3);       // this warp's 1536-B run, top row
    uint4* d1 = reinterpret_cast<uint4*>(out + ((size_t)(2 * cy + 1) * width + (size_t)gx0 * 16) * 3);   // bottom row
    if (full_warp) {
        pack_rgb16(ytw, ct, yc, o);
        store_rgb48_coalesced(d0, stage[wid], lane, o);
        pack_rgb16(ybw, ct, yc, o);
        store_rgb48_coalesced(d1, stage[wid], lane, o);
    } else if (active) {   // ragged last warp of a row: direct 48-B stores
        pack_rgb16(ytw, ct, yc, o);
        stg_stream_u4(d0 + 3 * lane, o[0]); stg_stream_u4(d0 + 3 * lane + 1, o[1]); stg_stream_u4(d0 + 3 * lane + 2, o[2]);
        pack_rgb16(ybw, ct, yc, o);
        stg_stream_u4(d1 + 3 * lane, o[0]); stg_stream_u4(d1 + 3 * lane + 1, o[1]); stg_stream_u4(d1 + 3 * lane + 2, o[2]);
    }
}

// Generic fallback (any even width / unaligned buffers): one thread per 2x2 block.
template <int L>
__global__ void rgb_from_yuv420_generic(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t width,
                                        uint32_t height, size_t frame_bytes, const YuvCoeffs yc) {
    const uint32_t cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y;
    if (cx >= width / 2 || cy >= height / 2) return;
    const uint8_t* frame = src + (size_t)blockIdx.z * frame_bytes;
    uint8_t* out = dst + (size_t)blockIdx.z * (size_t)width * height * 3;
    ChromaTerms ct;
    if (yuv420_planar(L)) {
        const size_t c = (size_t)cy * (width / 2) + cx;
        ct = chroma_terms(frame[yuv420_u_plane(L, width, height) + c], frame[yuv420_v_plane(L, width, height) + c], yc);
    } else {
        const uint8_t* uvp = frame + (size_t)width * height + (size_t)cy * width + 2 * cx;
        ct = L == YUV420_NV21 ? chroma_terms(uvp[1], uvp[0], yc) : chroma_terms(uvp[0], uvp[1], yc);
    }
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const size_t p = (size_t)(2 * cy + dy) * width + 2 * cx + dx;
            int r, g, b;
            decode_rgb(yy_term(frame[p], yc), ct, r, g, b);
            out[3 * p] = (uint8_t)r; out[3 * p + 1] = (uint8_t)g; out[3 * p + 2] = (uint8_t)b;
        }
}

// ── 10- and 12-bit 4:2:0 (P010, P012, I010, I012) → RGB16 ─────────────────────────────────────────────
// L = kb200_yuv420_u16_layout; the depth and matrix arrive in Yuv16Coeffs (code extraction and Q16 set), so one kernel
// serves both depths of a layout.  One thread: 8 luma columns x 2 rows (one chroma row) — 16 B of Y words per row, and
// the 4 chroma pairs: one 16-B load of the interleaved row (P01x), or 8 B of the U plane and 8 B of the V plane (I01x;
// with width % 8 == 0 both planes and every thread's offset in them are 8-B aligned).  8 pixels of 16-bit RGB are 48 B
// per row, stored through store_rgb48_coalesced like the 8-bit kernels' 16 pixels.
template <int L>
__global__ void __launch_bounds__(128) rgb_from_yuv420_u16_vec(const uint16_t* __restrict__ src, uint16_t* __restrict__ dst,
                                                               uint32_t width, uint32_t height, const Yuv16Coeffs k) {
    __shared__ uint4 stage[4][96];
    const uint32_t gx = blockIdx.x * blockDim.x + threadIdx.x;  // 8-column group
    const uint32_t cy = blockIdx.y;                             // chroma row
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const uint32_t gx0 = gx - lane;                             // first group of this warp
    if (gx0 * 8 >= width) return;                               // whole warp out of the row
    const bool full_warp = (gx0 + 32) * 8 <= width;
    const bool active = gx * 8 < width;
    const size_t plane = (size_t)width * height;
    const uint16_t* frame = src + (size_t)blockIdx.z * (plane * 3 / 2);
    uint16_t* out = dst + (size_t)blockIdx.z * plane * 3;
    const size_t x = (size_t)gx * 8;
    uint4 yt = make_uint4(0, 0, 0, 0), yb = yt, uv = yt;   // I01x: uv = {U words 0-3, V words 0-3}; P01x: 4 (U, V) word pairs
    if (active) {
        yt = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)(2 * cy) * width + x));
        yb = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)(2 * cy + 1) * width + x));
        if (L == KB200_YUV420_I01X) {
            const size_t c = (size_t)cy * (width / 2) + x / 2;
            const uint2 u = ldg_stream_u2(reinterpret_cast<const uint2*>(frame + plane + c));
            const uint2 v = ldg_stream_u2(reinterpret_cast<const uint2*>(frame + plane + plane / 4 + c));
            uv = make_uint4(u.x, u.y, v.x, v.y);
        } else {
            uv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + plane + (size_t)cy * width + x));
        }
    }
    const uint32_t uvw[4] = {uv.x, uv.y, uv.z, uv.w};
    ChromaTerms ct[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {   // yuv16_code keeps the n code bits of the low half-word it is shifted to
        if (L == KB200_YUV420_I01X)
            ct[j] = chroma_terms16(yuv16_code(uvw[j >> 1] >> (16 * (j & 1)), k), yuv16_code(uvw[2 + (j >> 1)] >> (16 * (j & 1)), k), k);
        else
            ct[j] = chroma_terms16(yuv16_code(uvw[j], k), yuv16_code(uvw[j] >> 16, k), k);
    }
    auto pack = [&](const uint4& yv, uint4 o[3]) {   // 8 pixels -> 24 samples r0 g0 b0 r1 ..., two per 32-bit word
        const uint32_t yw[4] = {yv.x, yv.y, yv.z, yv.w};
        int rgb[3][8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
            decode_rgb16(yy_term16(yuv16_code(yw[j >> 1] >> (16 * (j & 1)), k), k), ct[j >> 1], k.white, rgb[0][j], rgb[1][j], rgb[2][j]);
        pack_rgb48_u16(rgb, o);
    };
    uint4 o[3];
    uint4* d0 = reinterpret_cast<uint4*>(out + ((size_t)(2 * cy) * width + (size_t)gx0 * 8) * 3);       // this warp's 1536-B run, top row
    uint4* d1 = reinterpret_cast<uint4*>(out + ((size_t)(2 * cy + 1) * width + (size_t)gx0 * 8) * 3);   // bottom row
    if (full_warp) {
        pack(yt, o);
        store_rgb48_coalesced(d0, stage[wid], lane, o);
        pack(yb, o);
        store_rgb48_coalesced(d1, stage[wid], lane, o);
    } else if (active) {   // ragged last warp of a row: direct 48-B stores
        pack(yt, o);
        stg_stream_u4(d0 + 3 * lane, o[0]); stg_stream_u4(d0 + 3 * lane + 1, o[1]); stg_stream_u4(d0 + 3 * lane + 2, o[2]);
        pack(yb, o);
        stg_stream_u4(d1 + 3 * lane, o[0]); stg_stream_u4(d1 + 3 * lane + 1, o[1]); stg_stream_u4(d1 + 3 * lane + 2, o[2]);
    }
}

// Generic fallback (any even width, 2-B aligned buffers): one thread per pixel.
template <int L>
__global__ void rgb_from_yuv420_u16_generic(const uint16_t* __restrict__ src, uint16_t* __restrict__ dst, uint32_t width,
                                            uint32_t height, const Yuv16Coeffs k) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t plane = (size_t)width * height;
    const uint16_t* frame = src + (size_t)blockIdx.z * (plane * 3 / 2);
    size_t cu, cv;
    if (L == KB200_YUV420_I01X) {
        cu = plane + (size_t)(y >> 1) * (width / 2) + (x >> 1);
        cv = cu + plane / 4;
    } else {
        cu = plane + (size_t)(y >> 1) * width + (x & ~1u);
        cv = cu + 1;
    }
    const ChromaTerms ct = chroma_terms16(yuv16_code(frame[cu], k), yuv16_code(frame[cv], k), k);
    int r, g, b;
    decode_rgb16(yy_term16(yuv16_code(frame[(size_t)y * width + x], k), k), ct, k.white, r, g, b);
    uint16_t* o = dst + ((size_t)blockIdx.z * plane + (size_t)y * width + x) * 3;
    o[0] = (uint16_t)r; o[1] = (uint16_t)g; o[2] = (uint16_t)b;
}

// ── 4:4:4 (I444 bytes; I410, I412 and their MSB-aligned forms in 16-bit words) → RGB8 / RGB16 ──────────────────────
// Three full-resolution planes Y, U, V: every pixel decodes from its own chroma.  One thread: one row's 16 pixels of bytes
// or 8 pixels of words, i.e. one 16-B load from each plane (lane-contiguous over the warp), and 48 B of RGB stored through
// store_rgb48_coalesced.  Requires width % 16 == 0 (bytes) / width % 8 == 0 (words) and 16-B aligned bases: then every
// row of every plane starts 16-B aligned.  grid = (groups of a row, rows, frames).
__global__ void __launch_bounds__(128) rgb_from_i444_vec16(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t width,
                                                           uint32_t height, const YuvCoeffs yc) {
    __shared__ uint4 stage[4][96];
    const WarpRun<16> run(width);
    if (run.gx0 * 16 >= width) return;   // whole warp out of the row
    const size_t plane = (size_t)width * height;
    const uint8_t* frame = src + (size_t)blockIdx.z * plane * 3;
    const size_t row = (size_t)blockIdx.y * width;
    uint4 yv = make_uint4(0, 0, 0, 0), uv = yv, vv = yv;
    if (run.active) {
        const size_t p = row + (size_t)run.gx * 16;
        yv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + p));
        uv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + plane + p));
        vv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + 2 * plane + p));
    }
    const uint32_t yw[4] = {yv.x, yv.y, yv.z, yv.w}, uw[4] = {uv.x, uv.y, uv.z, uv.w}, vw[4] = {vv.x, vv.y, vv.z, vv.w};
    uint32_t w[12];
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // 4 px -> 12 bytes = 3 words: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
        int r[4], g[4], b[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const ChromaTerms t = chroma_terms((int)byte_of(uw[k], j), (int)byte_of(vw[k], j), yc);
            const int yy = yy_term((int)byte_of(yw[k], j), yc);
            b[j] = (yy + t.b) >> 20; g[j] = (yy + t.g) >> 20; r[j] = (yy + t.r) >> 20;   // saturated by the pack below
        }
        w[3 * k] = pack_sat4(r[0], g[0], b[0], r[1]);
        w[3 * k + 1] = pack_sat4(g[1], b[1], r[2], g[2]);
        w[3 * k + 2] = pack_sat4(b[2], r[3], g[3], b[3]);
    }
    const uint4 o[3] = {make_uint4(w[0], w[1], w[2], w[3]), make_uint4(w[4], w[5], w[6], w[7]), make_uint4(w[8], w[9], w[10], w[11])};
    run.store(reinterpret_cast<uint4*>(dst + (size_t)blockIdx.z * plane * 3 + (row + (size_t)run.gx0 * 16) * 3), stage[threadIdx.x >> 5], o);
}

// The depth, code position and matrix arrive in Yuv16Coeffs, so one kernel serves I410, I412, I410Msb and I412Msb.
__global__ void __launch_bounds__(128) rgb_from_i41x_vec(const uint16_t* __restrict__ src, uint16_t* __restrict__ dst, uint32_t width,
                                                         uint32_t height, const Yuv16Coeffs k) {
    __shared__ uint4 stage[4][96];
    const WarpRun<8> run(width);
    if (run.gx0 * 8 >= width) return;   // whole warp out of the row
    const size_t plane = (size_t)width * height;
    const uint16_t* frame = src + (size_t)blockIdx.z * plane * 3;
    const size_t row = (size_t)blockIdx.y * width;
    uint4 yv = make_uint4(0, 0, 0, 0), uv = yv, vv = yv;
    if (run.active) {
        const size_t p = row + (size_t)run.gx * 8;
        yv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + p));
        uv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + plane + p));
        vv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + 2 * plane + p));
    }
    const uint32_t yw[4] = {yv.x, yv.y, yv.z, yv.w}, uw[4] = {uv.x, uv.y, uv.z, uv.w}, vw[4] = {vv.x, vv.y, vv.z, vv.w};
    int rgb[3][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {   // yuv16_code keeps the n code bits of the low half-word it is shifted to
        const int sh = 16 * (j & 1);
        const ChromaTerms t = chroma_terms16(yuv16_code(uw[j >> 1] >> sh, k), yuv16_code(vw[j >> 1] >> sh, k), k);
        decode_rgb16(yy_term16(yuv16_code(yw[j >> 1] >> sh, k), k), t, k.white, rgb[0][j], rgb[1][j], rgb[2][j]);
    }
    uint4 o[3];
    pack_rgb48_u16(rgb, o);
    run.store(reinterpret_cast<uint4*>(dst + (size_t)blockIdx.z * plane * 3 + (row + (size_t)run.gx0 * 8) * 3), stage[threadIdx.x >> 5], o);
}

// Generic fallbacks (any width, unaligned bases; words 2-B aligned): one thread per pixel.
__global__ void rgb_from_i444_generic(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t width, uint32_t height,
                                      const YuvCoeffs yc) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t plane = (size_t)width * height, p = (size_t)y * width + x;
    const uint8_t* frame = src + (size_t)blockIdx.z * plane * 3;
    int r, g, b;
    decode_rgb(yy_term(frame[p], yc), chroma_terms(frame[plane + p], frame[2 * plane + p], yc), r, g, b);
    uint8_t* o = dst + ((size_t)blockIdx.z * plane + p) * 3;
    o[0] = (uint8_t)r; o[1] = (uint8_t)g; o[2] = (uint8_t)b;
}

__global__ void rgb_from_i41x_generic(const uint16_t* __restrict__ src, uint16_t* __restrict__ dst, uint32_t width, uint32_t height,
                                      const Yuv16Coeffs k) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t plane = (size_t)width * height, p = (size_t)y * width + x;
    const uint16_t* frame = src + (size_t)blockIdx.z * plane * 3;
    int r, g, b;
    decode_rgb16(yy_term16(yuv16_code(frame[p], k), k), chroma_terms16(yuv16_code(frame[plane + p], k), yuv16_code(frame[2 * plane + p], k), k),
                 k.white, r, g, b);
    uint16_t* o = dst + ((size_t)blockIdx.z * plane + p) * 3;
    o[0] = (uint16_t)r; o[1] = (uint16_t)g; o[2] = (uint16_t)b;
}

// ── YUYV → RGB8 ─────────────────────────────────────────────────────────────────────────────
// One thread: 16 px = 32 B in (2 x LDG.128), 48 B out (3 x STG.128).  Flat over the whole batch
// (rows are independent and tight), requires total px % 16 == 0 and aligned bases.  The byte places of the 4:2:2
// layouts are Yuv422Bytes<L> (kb200_common.cuh).

template <int L>
__device__ __forceinline__ void yuv422_decode16(const uint4& A, const uint4& B, const YuvCoeffs& yc, uint4 o[3]) {
    using P = Yuv422Bytes<L>;
    const uint32_t g4[8] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w};  // each word: one 2-px group
    uint32_t yw[4];
    ChromaTerms ct[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t w = g4[k];
        ct[k] = chroma_terms((int)((w >> (8 * P::u)) & 0xFFu), (int)((w >> (8 * P::v)) & 0xFFu), yc);
        const uint32_t ypair = __byte_perm(w, 0, 0x4400 | (P::y1 << 4) | P::y0);   // {Y0, Y1, 0, 0}
        if (k & 1) yw[k >> 1] |= ypair << 16; else yw[k >> 1] = ypair;
    }
    pack_rgb16(yw, ct, yc, o);
}

// A warp owns 32 consecutive 16-px groups = 1024 B in, 1536 B out, both contiguous: the loads are issued
// lane-contiguous (2 x LDG.128 per lane over the warp's run) and handed to their owners through shared memory, the
// stores go back through it (store_rgb48_coalesced) — every global access instruction covers whole 128-B lines.
template <int L>
__global__ void __launch_bounds__(256) rgb_from_yuv422_vec16(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                                             size_t ngroups, const YuvCoeffs yc) {
    __shared__ uint4 stage[8][96];
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t q0 = (size_t)blockIdx.x * blockDim.x + wid * 32u; q0 < ngroups; q0 += stride) {
        uint4 o[3];
        if (q0 + 32 <= ngroups) {
            uint4* st = stage[wid];
            st[lane] = ldg_stream_u4(src + 2 * q0 + lane);
            st[32 + lane] = ldg_stream_u4(src + 2 * q0 + 32 + lane);
            __syncwarp();
            const uint4 A = st[2 * lane], B = st[2 * lane + 1];
            __syncwarp();
            yuv422_decode16<L>(A, B, yc, o);
            store_rgb48_coalesced(dst + 3 * q0, st, lane, o);
        } else if (q0 + lane < ngroups) {   // ragged tail warp
            const size_t q = q0 + lane;
            yuv422_decode16<L>(ldg_stream_u4(src + 2 * q), ldg_stream_u4(src + 2 * q + 1), yc, o);
            stg_stream_u4(dst + 3 * q, o[0]); stg_stream_u4(dst + 3 * q + 1, o[1]); stg_stream_u4(dst + 3 * q + 2, o[2]);
        }
    }
}

template <int L>
__global__ void rgb_from_yuv422_generic(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t first_group,
                                        size_t ngroups, const YuvCoeffs yc) {
    using P = Yuv422Bytes<L>;
    const size_t g = first_group + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ngroups) return;
    const uint8_t* s = src + 4 * g;
    const ChromaTerms ct = chroma_terms(s[P::u], s[P::v], yc);
    int r, gg, b;
    decode_rgb(yy_term(s[P::y0], yc), ct, r, gg, b);
    dst[6 * g] = (uint8_t)r; dst[6 * g + 1] = (uint8_t)gg; dst[6 * g + 2] = (uint8_t)b;
    decode_rgb(yy_term(s[P::y1], yc), ct, r, gg, b);
    dst[6 * g + 3] = (uint8_t)r; dst[6 * g + 4] = (uint8_t)gg; dst[6 * g + 5] = (uint8_t)b;
}

// ── Bayer → RGB (bilinear demosaic, bayer.cuh): 8-bit mosaics to RGB8, 10- to 16-bit ones to RGB16 ───────────────
// The S = BayerSample<T>::VEC_COLS demosaiced pixels of one row (bayer_row) -> 48 RGB bytes, the interleaved samples
// r0 g0 b0 r1 g1 b1 ...: 16 pixels as saturated bytes, or 8 pixels as 16-bit words (every result is <= 65535: no
// saturation).  Either way a thread stores 48 B per row, so the same coalesced store serves both.
template <typename T, int P, int PY>
__device__ __forceinline__ void bayer_row48(const uint32_t n[4], const uint32_t c[4], const uint32_t s[4], const int hl[3], const int hr[3],
                                            bool left_edge, bool right_edge, uint4 o[3]) {
    int rgb[3][BayerSample<T>::VEC_COLS];
    bayer_row<P, PY, 4, T>(n, c, s, hl, hr, left_edge, right_edge, rgb[0], rgb[1], rgb[2]);
    auto sample = [&](int a) { return rgb[a % 3][a / 3]; };   // output sample a of the row
    uint32_t w[12];
#pragma unroll
    for (int m = 0; m < 12; ++m) {
        if constexpr (sizeof(T) == 1) w[m] = pack_sat4(sample(4 * m), sample(4 * m + 1), sample(4 * m + 2), sample(4 * m + 3));
        else w[m] = (uint32_t)sample(2 * m) | ((uint32_t)sample(2 * m + 1) << 16);
    }
    o[0] = make_uint4(w[0], w[1], w[2], w[3]);
    o[1] = make_uint4(w[4], w[5], w[6], w[7]);
    o[2] = make_uint4(w[8], w[9], w[10], w[11]);
}

// One thread: S = BayerSample<T>::VEC_COLS columns (one 16-B vector per row) x 2 output rows, ya = 1 + 2 * blockIdx.y
// and ya + 1 (bayer_row_pairs).  Loads the rows ya-1 .. ya+2 of its S columns as four lane-contiguous LDG.128 plus
// shuffled halos (bayer_load_rows) and stores 48 B per row through store_rgb48_coalesced (three lane-contiguous STG.128
// per warp and row).  Requires width % S == 0 and 16-B aligned bases, so every row of source and output starts 16-B aligned.
// Packed samples (T = BayerPacked<BITS>): a warp's 32 * 8 columns are 32 * BITS contiguous bytes of a row (320, 384 or
// 448), loaded as lane-contiguous LDG.128 into shared memory; each lane then unpacks its BITS bytes into the uint16_t
// words of the 16-bit kernel.  Requires width * BITS % 128 == 0 (every row 16-B aligned) and 16-B aligned bases.
template <typename T, int P>
__global__ void __launch_bounds__(128) rgb_from_bayer_vec(const T* __restrict__ src, typename BayerSample<T>::Word* __restrict__ dst,
                                                          uint32_t width, uint32_t height) {
    using W = typename BayerSample<T>::Word;
    constexpr int PB = BayerSample<T>::PACKED_BITS;
    constexpr uint32_t S = BayerSample<T>::VEC_COLS;
    __shared__ uint4 stage[4][96];
    const uint32_t gx = blockIdx.x * blockDim.x + threadIdx.x;  // S-column group
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const uint32_t gx0 = gx - lane;                             // first group of this warp
    if (gx0 * S >= width) return;                               // whole warp out of the row
    const bool full_warp = (gx0 + 32) * S <= width;
    const bool active = gx * S < width;
    const uint32_t x = gx * S;
    const uint32_t ya = 1 + 2 * blockIdx.y, yb = ya + 1;
    uint32_t rows[4][4];
    int hl[4], hr[4];
    if constexpr (PB == 0) {
        const T* frame = src + (size_t)blockIdx.z * width * height;
        bayer_load_rows<4>(frame, width, width, height, x, ya, lane, [&](const T* p, uint32_t v[4]) {
            const uint4 q = active ? ldg_stream_u4(reinterpret_cast<const uint4*>(p)) : make_uint4(0, 0, 0, 0);
            v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        }, rows, hl, hr);
    } else {
        __shared__ uint4 packed[4][4][33];   // per warp and row: the warp's <= 448 bytes, and room for the last lane's over-read
        const size_t pitch = (size_t)width * PB / 8;
        const uint8_t* frame = reinterpret_cast<const uint8_t*>(src) + (size_t)blockIdx.z * pitch * height;
        const uint32_t seg_bytes = (min(width - gx0 * S, 32u * S) * PB) / 8;   // this warp's bytes of a row
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint8_t* seg = frame + (size_t)min(ya - 1 + k, height - 1) * pitch + (size_t)gx0 * PB;
            if (16u * lane < seg_bytes) packed[wid][k][lane] = ldg_stream_u4(reinterpret_cast<const uint4*>(seg) + lane);
        }
        __syncwarp();
        bayer_load_rows_packed<4, PB>(frame, pitch, width, height, x, ya, lane, [&](int k, const uint8_t*, uint32_t v[4]) {
            const uint32_t o = lane * PB;   // the lane's first byte in the warp's segment
            const uint32_t* wds = reinterpret_cast<const uint32_t*>(packed[wid][k]) + (o >> 2);
            const uint32_t sh = 8u * (o & 3u);
            uint32_t bytes[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) bytes[i] = __funnelshift_r(wds[i], wds[i + 1], sh);
            bayer_unpack<PB, 8>(bytes, v);
            if (!active) { v[0] = 0; v[1] = 0; v[2] = 0; v[3] = 0; }
        }, rows, hl, hr);
    }
    W* out = dst + (size_t)blockIdx.z * width * height * 3;
    const bool left_edge = x == 0, right_edge = x + S == width;
    auto store_row = [&](uint32_t y, const uint4 o[3]) {
        uint4* d = reinterpret_cast<uint4*>(out + ((size_t)y * width + (size_t)gx0 * S) * 3);   // this warp's run of row y
        if (full_warp) store_rgb48_coalesced(d, stage[wid], lane, o);
        else if (active) { stg_stream_u4(d + 3 * lane, o[0]); stg_stream_u4(d + 3 * lane + 1, o[1]); stg_stream_u4(d + 3 * lane + 2, o[2]); }
    };
    uint4 oa[3];
    bayer_row48<W, P, 1>(rows[0], rows[1], rows[2], hl, hr, left_edge, right_edge, oa);   // ya is odd
    store_row(ya, oa);
    if (ya == 1) store_row(0, oa);
    if (yb == height - 1) {
        store_row(yb, oa);
    } else {
        uint4 ob[3];
        bayer_row48<W, P, 0>(rows[1], rows[2], rows[3], hl + 1, hr + 1, left_edge, right_edge, ob);
        store_row(yb, ob);
        if (yb == height - 2) store_row(height - 1, ob);
    }
}

// Generic fallback (any width, any base aligned to T; packed: any base): one thread per pixel, nine sample loads.
template <typename T, int P>
__global__ void rgb_from_bayer_generic(const T* __restrict__ src, typename BayerSample<T>::Word* __restrict__ dst, uint32_t width,
                                       uint32_t height) {
    using W = typename BayerSample<T>::Word;
    constexpr int PB = BayerSample<T>::PACKED_BITS;
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= width || y >= height) return;
    const size_t frame = (size_t)width * height;
    int rgb[3];
    if constexpr (PB == 0) {
        bayer_px(src + blockIdx.z * frame, width, (int)width, (int)height, (int)x, (int)y, P, rgb);
    } else {
        const size_t pitch = (size_t)width * PB / 8;
        bayer_px_packed(reinterpret_cast<const uint8_t*>(src) + blockIdx.z * pitch * height, pitch, (int)width, (int)height, (int)x, (int)y, P,
                        PB, rgb);
    }
    W* o = dst + (blockIdx.z * frame + (size_t)y * width + x) * 3;
    o[0] = (W)rgb[0]; o[1] = (W)rgb[1]; o[2] = (W)rgb[2];
}

static inline unsigned stream_grid(size_t items, unsigned block, unsigned ctas_per_sm) {
    const size_t want = (items + block - 1) / block;
    const size_t cap = (size_t)device_info().sm_count * ctas_per_sm;
    return (unsigned)std::max<size_t>(1, std::min(want, cap));
}

// The argument checks the decoders share.
static int check_matrix(int matrix) {
    if (matrix < KB200_YUV_BT601_LIMITED || matrix > KB200_YUV_BT709_FULL) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown YUV matrix %d", matrix);
    return KB200_OK;
}
static int check_words(const char* what, const void* p) {   // a buffer of 16-bit samples
    if (reinterpret_cast<uintptr_t>(p) & 1u) return fail(KB200_ERR_INVALID_ARGUMENT, "'%s' is not 2-byte aligned (16-bit samples)", what);
    return KB200_OK;
}
static int check_batch(uint32_t batch) {   // one frame per gridDim.z
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535", batch);
    return KB200_OK;
}

// The kernels of one decoder that has a vector kernel, and the names they report through kb200_last_kernel().  Both
// take (src, dst, width, height, A...).
template <typename S, typename D, typename... A>
struct DecodeKernels {
    void (*vec)(const S*, D*, uint32_t, uint32_t, A...);
    void (*generic)(const S*, D*, uint32_t, uint32_t, A...);
    const char *vec_name, *generic_name;
};

// The launch of a DecodeKernels row (arguments already checked).  The vector kernel when the format's gate `fits` holds,
// both bases are 16-B aligned and its `rows` grid rows fit gridDim.y: each thread owns `cols` columns of a grid row, the
// threads of a row are CTAs of up to 128.  The fallback otherwise, one thread per `step` x `step` pixels (1, or 2 for the
// 8-bit 4:2:0 kernel's 2x2 blocks) over a (width, height, batch) grid of 32 x 8 CTAs.
template <typename S, typename D, typename... A>
static int launch_decoder(const DecodeKernels<S, D, A...>& k, kb200_stream_t stream, bool fits, uint32_t cols, uint32_t rows, uint32_t step,
                          const S* src, D* dst, uint32_t width, uint32_t height, uint32_t batch, A... args) {
    cudaStream_t s = as_stream(stream);
    if (fits && aligned16(src) && aligned16(dst) && rows <= 65535u) {
        const unsigned groups = width / cols;
        const unsigned bx = groups >= 128 ? 128 : 32 * ((groups + 31) / 32);
        dim3 grid(div_up(groups, bx), rows, batch);
        k.vec<<<grid, bx, 0, s>>>(src, dst, width, height, args...);
        return check_launch(k.vec_name);
    }
    dim3 block(32, 8), grid(div_up(width / step, 32), div_up(height / step, 8), batch);
    k.generic<<<grid, block, 0, s>>>(src, dst, width, height, args...);
    return check_launch(k.generic_name);
}

// 8-bit 4:2:0, indexed by kb200_yuv420_layout.
static const char* const YUV420_LAYOUTS[4] = {"NV12", "NV21", "I420", "YV12"};
static const DecodeKernels<uint8_t, uint8_t, size_t, YuvCoeffs> YUV420_KERNELS[4] = {
    {rgb_from_yuv420_vec16<YUV420_NV12>, rgb_from_yuv420_generic<YUV420_NV12>, "rgb_from_nv12_vec16", "rgb_from_nv12_generic"},
    {rgb_from_yuv420_vec16<YUV420_NV21>, rgb_from_yuv420_generic<YUV420_NV21>, "rgb_from_nv21_vec16", "rgb_from_nv21_generic"},
    {rgb_from_yuv420_vec16<YUV420_I420>, rgb_from_yuv420_generic<YUV420_I420>, "rgb_from_i420_vec16", "rgb_from_i420_generic"},
    {rgb_from_yuv420_vec16<YUV420_YV12>, rgb_from_yuv420_generic<YUV420_YV12>, "rgb_from_yv12_vec16", "rgb_from_yv12_generic"},
};
// 16-bit 4:2:0, indexed by kb200_yuv420_u16_layout.
static const DecodeKernels<uint16_t, uint16_t, Yuv16Coeffs> YUV420_U16_KERNELS[2] = {
    {rgb_from_yuv420_u16_vec<KB200_YUV420_P01X>, rgb_from_yuv420_u16_generic<KB200_YUV420_P01X>, "rgb_from_p01x_vec", "rgb_from_p01x_generic"},
    {rgb_from_yuv420_u16_vec<KB200_YUV420_I01X>, rgb_from_yuv420_u16_generic<KB200_YUV420_I01X>, "rgb_from_i01x_vec", "rgb_from_i01x_generic"},
};
static const DecodeKernels<uint8_t, uint8_t, YuvCoeffs> YUV444_KERNELS = {rgb_from_i444_vec16, rgb_from_i444_generic,
                                                                          "rgb_from_i444_vec16", "rgb_from_i444_generic"};
static const DecodeKernels<uint16_t, uint16_t, Yuv16Coeffs> YUV444_U16_KERNELS = {rgb_from_i41x_vec, rgb_from_i41x_generic,
                                                                                  "rgb_from_i41x_vec", "rgb_from_i41x_generic"};

// 4:2:2, indexed by kb200_yuv422_layout.  These kernels walk the batch flat in 2-pixel groups, so they have a row of their own.
struct Yuv422Kernels {
    const char* layout;
    void (*vec16)(const uint4*, uint4*, size_t, YuvCoeffs);
    void (*generic)(const uint8_t*, uint8_t*, size_t, size_t, YuvCoeffs);
    const char *vec16_name, *generic_name;
};
static const Yuv422Kernels YUV422_KERNELS[3] = {
    {"YUYV", rgb_from_yuv422_vec16<YUV422_YUYV>, rgb_from_yuv422_generic<YUV422_YUYV>, "rgb_from_yuyv_vec16", "rgb_from_yuyv_generic"},
    {"UYVY", rgb_from_yuv422_vec16<YUV422_UYVY>, rgb_from_yuv422_generic<YUV422_UYVY>, "rgb_from_uyvy_vec16", "rgb_from_uyvy_generic"},
    {"YVYU", rgb_from_yuv422_vec16<YUV422_YVYU>, rgb_from_yuv422_generic<YUV422_YVYU>, "rgb_from_yvyu_vec16", "rgb_from_yvyu_generic"},
};
// The Bayer kernels of each sample type, indexed by kb200_bayer_pattern.
static const char* const BAYER_PATTERNS[4] = {"RGGB", "BGGR", "GRBG", "GBRG"};
template <typename T> using BayerKernels = DecodeKernels<T, typename BayerSample<T>::Word>;
static const BayerKernels<uint8_t> BAYER_KERNELS_U8[4] = {
    {rgb_from_bayer_vec<uint8_t, KB200_BAYER_RGGB>, rgb_from_bayer_generic<uint8_t, KB200_BAYER_RGGB>, "rgb_from_bayer_rggb_vec16", "rgb_from_bayer_rggb_generic"},
    {rgb_from_bayer_vec<uint8_t, KB200_BAYER_BGGR>, rgb_from_bayer_generic<uint8_t, KB200_BAYER_BGGR>, "rgb_from_bayer_bggr_vec16", "rgb_from_bayer_bggr_generic"},
    {rgb_from_bayer_vec<uint8_t, KB200_BAYER_GRBG>, rgb_from_bayer_generic<uint8_t, KB200_BAYER_GRBG>, "rgb_from_bayer_grbg_vec16", "rgb_from_bayer_grbg_generic"},
    {rgb_from_bayer_vec<uint8_t, KB200_BAYER_GBRG>, rgb_from_bayer_generic<uint8_t, KB200_BAYER_GBRG>, "rgb_from_bayer_gbrg_vec16", "rgb_from_bayer_gbrg_generic"},
};
static const BayerKernels<uint16_t> BAYER_KERNELS_U16[4] = {
    {rgb_from_bayer_vec<uint16_t, KB200_BAYER_RGGB>, rgb_from_bayer_generic<uint16_t, KB200_BAYER_RGGB>, "rgb_from_bayer16_rggb_vec", "rgb_from_bayer16_rggb_generic"},
    {rgb_from_bayer_vec<uint16_t, KB200_BAYER_BGGR>, rgb_from_bayer_generic<uint16_t, KB200_BAYER_BGGR>, "rgb_from_bayer16_bggr_vec", "rgb_from_bayer16_bggr_generic"},
    {rgb_from_bayer_vec<uint16_t, KB200_BAYER_GRBG>, rgb_from_bayer_generic<uint16_t, KB200_BAYER_GRBG>, "rgb_from_bayer16_grbg_vec", "rgb_from_bayer16_grbg_generic"},
    {rgb_from_bayer_vec<uint16_t, KB200_BAYER_GBRG>, rgb_from_bayer_generic<uint16_t, KB200_BAYER_GBRG>, "rgb_from_bayer16_gbrg_vec", "rgb_from_bayer16_gbrg_generic"},
};

// The demosaic behind kb200_rgb_from_bayer_u8 / _u16 (pointers already checked): the fast kernel when every row is whole
// 16-B vectors, the one-thread-per-pixel kernel otherwise.  Lengths are in samples.
template <typename T>
static int launch_rgb_from_bayer(const BayerKernels<T> (&table)[4], kb200_stream_t stream, const T* src, size_t src_len, T* dst,
                                 size_t dst_len, uint32_t width, uint32_t height, uint32_t batch, int pattern) {
    if (pattern < KB200_BAYER_RGGB || pattern > KB200_BAYER_GBRG) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown Bayer pattern %d", pattern);
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if (width < 3 || height < 3) return fail(KB200_ERR_INVALID_ARGUMENT, "Bayer %s needs at least 3x3 pixels, got %ux%u", BAYER_PATTERNS[pattern], width, height);
    KB200_TRY(check_batch(batch));
    const size_t frame = (size_t)width * height;
    KB200_TRY(check_slice("src", src_len, frame * batch)); KB200_TRY(check_slice("dst", dst_len, frame * 3 * batch));
    constexpr uint32_t S = BayerSample<T>::VEC_COLS;
    return launch_decoder(table[pattern], stream, width % S == 0, S, bayer_row_pairs(height), 1, src, dst, width, height, batch);
}

// The packed decoders, by depth (10, 12, 14 bits) and pattern.
#define KB200_BAYER_PACKED_KERNELS(B, p, P)                                                                            \
    {rgb_from_bayer_vec<BayerPacked<B>, P>, rgb_from_bayer_generic<BayerPacked<B>, P>, "rgb_from_bayer" #B "p_" #p "_vec", \
     "rgb_from_bayer" #B "p_" #p "_generic"}
#define KB200_BAYER_PACKED_TABLE(B)                                                                                     \
    static const BayerKernels<BayerPacked<B>> BAYER_KERNELS_##B##P[4] = {                                               \
        KB200_BAYER_PACKED_KERNELS(B, rggb, KB200_BAYER_RGGB), KB200_BAYER_PACKED_KERNELS(B, bggr, KB200_BAYER_BGGR),   \
        KB200_BAYER_PACKED_KERNELS(B, grbg, KB200_BAYER_GRBG), KB200_BAYER_PACKED_KERNELS(B, gbrg, KB200_BAYER_GBRG)};
KB200_BAYER_PACKED_TABLE(10)
KB200_BAYER_PACKED_TABLE(12)
KB200_BAYER_PACKED_TABLE(14)
#undef KB200_BAYER_PACKED_TABLE
#undef KB200_BAYER_PACKED_KERNELS

// The demosaic behind kb200_rgb_from_bayer_packed (pointers, pattern and bits already checked): `batch` tight frames of
// h rows of width * BITS / 8 bytes.  The fast kernel when every row and both bases are 16-B aligned, the
// one-thread-per-pixel kernel otherwise.  src_len in bytes, dst_len in elements.
template <int BITS>
static int launch_rgb_from_bayer_packed(const BayerKernels<BayerPacked<BITS>> (&table)[4], kb200_stream_t stream, const uint8_t* src,
                                        size_t src_len, uint16_t* dst, size_t dst_len, uint32_t width, uint32_t height, uint32_t batch,
                                        int pattern) {
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if (width < 3 || height < 3)
        return fail(KB200_ERR_INVALID_ARGUMENT, "Bayer %s%dP needs at least 3x3 pixels, got %ux%u", BAYER_PATTERNS[pattern], BITS, width, height);
    constexpr uint32_t G = bayer_packed_group(BITS);
    if (width % G)
        return fail(KB200_ERR_INVALID_ARGUMENT, "Bayer %s%dP needs a width that is a multiple of %u (whole %d-byte groups), got %u",
                    BAYER_PATTERNS[pattern], BITS, G, bayer_packed_group_bytes(BITS), width);
    KB200_TRY(check_batch(batch));
    const size_t frame = (size_t)width * BITS / 8 * height;
    KB200_TRY(check_slice("src", src_len, frame * batch)); KB200_TRY(check_slice("dst", dst_len, (size_t)width * height * 3 * batch));
    return launch_decoder(table[pattern], stream, ((size_t)width * BITS) % 128 == 0, 8, bayer_row_pairs(height), 1,
                          reinterpret_cast<const BayerPacked<BITS>*>(src), dst, width, height, batch);
}

// ── RGB8 → YUYV / NV12 encode (SURVEY §8(f) #4) ─────────────────────────────────────────────
// color/yuv/kernels.rs:1223-1252: Q8 BT.601 limited — Y = ((66R + 129G + 25B + 128) >> 8) + 16,
// U = ((-38R - 74G + 112B + 128) >> 8) + 128, V = ((112R - 94G - 18B + 128) >> 8) + 128, clamped to 0..255.
__device__ __forceinline__ uint32_t enc_y(int r, int g, int b) { return (uint32_t)min(max(((66 * r + 129 * g + 25 * b + 128) >> 8) + 16, 0), 255); }
__device__ __forceinline__ uint32_t enc_u(int r, int g, int b) { return (uint32_t)min(max(((-38 * r - 74 * g + 112 * b + 128) >> 8) + 128, 0), 255); }
__device__ __forceinline__ uint32_t enc_v(int r, int g, int b) { return (uint32_t)min(max(((112 * r - 94 * g - 18 * b + 128) >> 8) + 128, 0), 255); }

// One thread per pixel pair: 6 bytes in, one 32-bit word `Y0 U Y1 V` out (lane-contiguous stores).  kernels.rs:1301-1322.
__global__ void __launch_bounds__(256) yuyv_from_rgb_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t npairs) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < npairs; g += stride) {
        const uint8_t* s = src + g * 6;
        const int r0 = s[0], g0 = s[1], b0 = s[2], r1 = s[3], g1 = s[4], b1 = s[5];
        const int ra = (r0 + r1 + 1) >> 1, ga = (g0 + g1 + 1) >> 1, ba = (b0 + b1 + 1) >> 1;   // shared chroma: rounded pair average
        const uint32_t w = enc_y(r0, g0, b0) | (enc_u(ra, ga, ba) << 8) | (enc_y(r1, g1, b1) << 16) | (enc_v(ra, ga, ba) << 24);
        uint8_t* d = dst + g * 4;
        if ((reinterpret_cast<uintptr_t>(d) & 3u) == 0) *reinterpret_cast<uint32_t*>(d) = w;
        else { d[0] = (uint8_t)w; d[1] = (uint8_t)(w >> 8); d[2] = (uint8_t)(w >> 16); d[3] = (uint8_t)(w >> 24); }
    }
}

// One thread per 2x2 block: 4 luma bytes (two 16-bit stores) + one UV pair.  kernels.rs:1480-1516, :1563-1576.
__global__ void __launch_bounds__(256) nv12_from_rgb_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t width,
                                                            uint32_t height, size_t frame_bytes) {
    const uint32_t cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y;
    if (cx >= width / 2 || cy >= height / 2) return;
    const uint8_t* s = src + (size_t)blockIdx.z * width * height * 3;
    uint8_t* frame = dst + (size_t)blockIdx.z * frame_bytes;
    const uint8_t* t = s + ((size_t)(2 * cy) * width + 2 * cx) * 3;
    const uint8_t* b = t + (size_t)width * 3;
    const int r00 = t[0], g00 = t[1], b00 = t[2], r01 = t[3], g01 = t[4], b01 = t[5];
    const int r10 = b[0], g10 = b[1], b10 = b[2], r11 = b[3], g11 = b[4], b11 = b[5];
    uint8_t* y0 = frame + (size_t)(2 * cy) * width + 2 * cx;
    uint8_t* y1 = y0 + width;
    y0[0] = (uint8_t)enc_y(r00, g00, b00); y0[1] = (uint8_t)enc_y(r01, g01, b01);
    y1[0] = (uint8_t)enc_y(r10, g10, b10); y1[1] = (uint8_t)enc_y(r11, g11, b11);
    const int ra = (r00 + r01 + r10 + r11 + 2) >> 2, ga = (g00 + g01 + g10 + g11 + 2) >> 2, ba = (b00 + b01 + b10 + b11 + 2) >> 2;
    uint8_t* uv = frame + (size_t)width * height + (size_t)cy * width + 2 * cx;
    uv[0] = (uint8_t)enc_u(ra, ga, ba); uv[1] = (uint8_t)enc_v(ra, ga, ba);
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_gray_from_rgb_f32(kb200_stream_t stream, const float* src, size_t src_len, float* dst,
                                      size_t dst_len, size_t npixels, int leaf) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    if (leaf < 0 || leaf > 2) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown cpu leaf %d", leaf);
    KB200_TRY(check_slice("src", src_len, npixels * 3)); KB200_TRY(check_slice("dst", dst_len, npixels));
    if (npixels == 0) return KB200_OK;
    const size_t bulk_px = (leaf == KB200_LEAF_SCALAR) ? 0 : (npixels & ~(size_t)7);
    cudaStream_t s = as_stream(stream);
    size_t done = 0;
    if (aligned16(src) && aligned16(dst)) {
        const size_t nquads = npixels / 4;
        if (nquads) {
            gray_from_rgb_f32_vec4<<<stream_grid(nquads, 256, 8), 256, 0, s>>>(
                reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst), nquads, bulk_px);
            KB200_TRY(check_launch("gray_from_rgb_f32_vec4"));
        }
        done = nquads * 4;
    }
    if (done < npixels) {
        const size_t rest = npixels - done;
        gray_from_rgb_f32_scalar<<<div_up(rest, 256), 256, 0, s>>>(src, dst, done, npixels, bulk_px);
        KB200_TRY(check_launch("gray_from_rgb_f32_scalar"));
    }
    return KB200_OK;
}

KB200_API int kb200_gray_from_rgb_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                     size_t dst_len, size_t npixels) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_slice("src", src_len, npixels * 3)); KB200_TRY(check_slice("dst", dst_len, npixels));
    if (npixels == 0) return KB200_OK;
    cudaStream_t s = as_stream(stream);
    size_t done = 0;
    if (aligned16(src) && aligned16(dst)) {
        const size_t ngroups = npixels / 16;
        if (ngroups) {
            gray_from_rgb_u8_vec16<<<stream_grid(ngroups, 256, 8), 256, 0, s>>>(
                reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), ngroups);
            KB200_TRY(check_launch("gray_from_rgb_u8_vec16"));
        }
        done = ngroups * 16;
    }
    if (done < npixels) {
        gray_from_rgb_u8_scalar<<<div_up(npixels - done, 256), 256, 0, s>>>(src, dst, done, npixels);
        KB200_TRY(check_launch("gray_from_rgb_u8_scalar"));
    }
    return KB200_OK;
}

KB200_API int kb200_rgb_from_yuv420_u8_matrix(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                              size_t dst_len, uint32_t width, uint32_t height, uint32_t batch, int layout, int matrix) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    if (layout < KB200_YUV420_NV12 || layout > KB200_YUV420_YV12) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown 4:2:0 layout %d", layout);
    KB200_TRY(check_matrix(matrix));
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if ((width & 1u) || (height & 1u)) return fail(KB200_ERR_INVALID_ARGUMENT, "%s needs even dimensions, got %ux%u", YUV420_LAYOUTS[layout], width, height);
    KB200_TRY(check_batch(batch));
    const size_t frame = (size_t)width * height * 3 / 2;
    KB200_TRY(check_slice("src", src_len, frame * batch)); KB200_TRY(check_slice("dst", dst_len, (size_t)width * height * 3 * batch));
    // w % 16 == 0, h even: every frame is a multiple of 16 B
    return launch_decoder(YUV420_KERNELS[layout], stream, width % 16u == 0, 16, height / 2, 2, src, dst, width, height, batch, frame, YUV_COEFFS[matrix]);
}

KB200_API int kb200_rgb_from_yuv420_u16(kb200_stream_t stream, const uint16_t* src, size_t src_len, uint16_t* dst, size_t dst_len,
                                        uint32_t width, uint32_t height, uint32_t batch, int layout, int bits, int matrix) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_words("src", src)); KB200_TRY(check_words("dst", dst));
    if (layout != KB200_YUV420_P01X && layout != KB200_YUV420_I01X) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown 16-bit 4:2:0 layout %d", layout);
    if (bits != 10 && bits != 12) return fail(KB200_ERR_INVALID_ARGUMENT, "16-bit 4:2:0 samples are 10 or 12 bits, got %d", bits);
    KB200_TRY(check_matrix(matrix));
    const bool planar = layout == KB200_YUV420_I01X;
    char name[8];
    snprintf(name, sizeof name, "%c01%d", planar ? 'I' : 'P', bits - 10);
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if ((width & 1u) || (height & 1u)) return fail(KB200_ERR_INVALID_ARGUMENT, "%s needs even dimensions, got %ux%u", name, width, height);
    KB200_TRY(check_batch(batch));
    const size_t plane = (size_t)width * height;
    KB200_TRY(check_slice("src", src_len, plane * 3 / 2 * batch)); KB200_TRY(check_slice("dst", dst_len, plane * 3 * batch));
    // w % 8 == 0, h even: every frame 16-B aligned
    return launch_decoder(YUV420_U16_KERNELS[layout], stream, width % 8u == 0, 8, height / 2, 1, src, dst, width, height, batch,
                          yuv16_coeffs(matrix, bits, !planar));
}

KB200_API int kb200_rgb_from_yuv444_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len,
                                       uint32_t width, uint32_t height, uint32_t batch, int matrix) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_matrix(matrix));
    KB200_TRY(check_geometry(width, height, width, height, batch));
    KB200_TRY(check_batch(batch));
    const size_t plane = (size_t)width * height;
    KB200_TRY(check_slice("src", src_len, plane * 3 * batch)); KB200_TRY(check_slice("dst", dst_len, plane * 3 * batch));
    return launch_decoder(YUV444_KERNELS, stream, width % 16u == 0, 16, height, 1, src, dst, width, height, batch, YUV_COEFFS[matrix]);
}

KB200_API int kb200_rgb_from_yuv444_u16(kb200_stream_t stream, const uint16_t* src, size_t src_len, uint16_t* dst, size_t dst_len,
                                        uint32_t width, uint32_t height, uint32_t batch, int layout, int bits, int matrix) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_words("src", src)); KB200_TRY(check_words("dst", dst));
    if (layout != KB200_YUV444_I41X && layout != KB200_YUV444_I41X_MSB) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown 16-bit 4:4:4 layout %d", layout);
    if (bits != 10 && bits != 12) return fail(KB200_ERR_INVALID_ARGUMENT, "16-bit 4:4:4 samples are 10 or 12 bits, got %d", bits);
    KB200_TRY(check_matrix(matrix));
    KB200_TRY(check_geometry(width, height, width, height, batch));
    KB200_TRY(check_batch(batch));
    const size_t plane = (size_t)width * height;
    KB200_TRY(check_slice("src", src_len, plane * 3 * batch)); KB200_TRY(check_slice("dst", dst_len, plane * 3 * batch));
    return launch_decoder(YUV444_U16_KERNELS, stream, width % 8u == 0, 8, height, 1, src, dst, width, height, batch,
                          yuv16_coeffs(matrix, bits, layout == KB200_YUV444_I41X_MSB));
}

KB200_API int kb200_rgb_from_yuv422_u8_matrix(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                              size_t dst_len, uint32_t width, uint32_t height, uint32_t batch, int layout, int matrix) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    if (layout < KB200_YUV422_YUYV || layout > KB200_YUV422_YVYU) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown 4:2:2 layout %d", layout);
    KB200_TRY(check_matrix(matrix));
    const YuvCoeffs& yc = YUV_COEFFS[matrix];
    const Yuv422Kernels& k = YUV422_KERNELS[layout];
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if (width & 1u) return fail(KB200_ERR_INVALID_ARGUMENT, "%s needs an even width, got %u", k.layout, width);
    const size_t npx = (size_t)width * height * batch;
    KB200_TRY(check_slice("src", src_len, npx * 2)); KB200_TRY(check_slice("dst", dst_len, npx * 3));
    cudaStream_t s = as_stream(stream);
    const size_t ngroups2 = npx / 2;  // 2-px groups
    size_t done = 0;
    if (aligned16(src) && aligned16(dst)) {
        const size_t n16 = npx / 16;
        if (n16) {
            k.vec16<<<stream_grid(n16, 256, 8), 256, 0, s>>>(reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), n16, yc);
            KB200_TRY(check_launch(k.vec16_name));
        }
        done = n16 * 8;
    }
    if (done < ngroups2) {
        k.generic<<<div_up(ngroups2 - done, 256), 256, 0, s>>>(src, dst, done, ngroups2, yc);
        KB200_TRY(check_launch(k.generic_name));
    }
    return KB200_OK;
}

KB200_API int kb200_rgb_from_yuv420_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                       size_t dst_len, uint32_t width, uint32_t height, uint32_t batch, int layout) {
    return kb200_rgb_from_yuv420_u8_matrix(stream, src, src_len, dst, dst_len, width, height, batch, layout, KB200_YUV_BT601_LIMITED);
}

KB200_API int kb200_rgb_from_yuv422_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                       size_t dst_len, uint32_t width, uint32_t height, uint32_t batch, int layout) {
    return kb200_rgb_from_yuv422_u8_matrix(stream, src, src_len, dst, dst_len, width, height, batch, layout, KB200_YUV_BT601_LIMITED);
}

KB200_API int kb200_rgb_from_nv12_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                     size_t dst_len, uint32_t width, uint32_t height, uint32_t batch) {
    return kb200_rgb_from_yuv420_u8(stream, src, src_len, dst, dst_len, width, height, batch, KB200_YUV420_NV12);
}

KB200_API int kb200_rgb_from_yuyv_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                     size_t dst_len, uint32_t width, uint32_t height, uint32_t batch) {
    return kb200_rgb_from_yuv422_u8(stream, src, src_len, dst, dst_len, width, height, batch, KB200_YUV422_YUYV);
}

KB200_API int kb200_rgb_from_bayer_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                      size_t dst_len, uint32_t width, uint32_t height, uint32_t batch, int pattern) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    return launch_rgb_from_bayer(BAYER_KERNELS_U8, stream, src, src_len, dst, dst_len, width, height, batch, pattern);
}

KB200_API int kb200_rgb_from_bayer_u16(kb200_stream_t stream, const uint16_t* src, size_t src_len, uint16_t* dst,
                                       size_t dst_len, uint32_t width, uint32_t height, uint32_t batch, int pattern) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_words("src", src)); KB200_TRY(check_words("dst", dst));
    return launch_rgb_from_bayer(BAYER_KERNELS_U16, stream, src, src_len, dst, dst_len, width, height, batch, pattern);
}

KB200_API int kb200_rgb_from_bayer_packed(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint16_t* dst, size_t dst_len,
                                          uint32_t width, uint32_t height, uint32_t batch, int pattern, int bits) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_words("dst", dst));
    if (pattern < KB200_BAYER_RGGB || pattern > KB200_BAYER_GBRG) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown Bayer pattern %d", pattern);
    switch (bits) {
        case 10: return launch_rgb_from_bayer_packed<10>(BAYER_KERNELS_10P, stream, src, src_len, dst, dst_len, width, height, batch, pattern);
        case 12: return launch_rgb_from_bayer_packed<12>(BAYER_KERNELS_12P, stream, src, src_len, dst, dst_len, width, height, batch, pattern);
        case 14: return launch_rgb_from_bayer_packed<14>(BAYER_KERNELS_14P, stream, src, src_len, dst, dst_len, width, height, batch, pattern);
        default: return fail(KB200_ERR_INVALID_ARGUMENT, "packed Bayer samples are 10, 12 or 14 bits, got %d", bits);
    }
}


KB200_API int kb200_yuyv_from_rgb_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len,
                                     uint32_t width, uint32_t height, uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if (width & 1u) return fail(KB200_ERR_INVALID_ARGUMENT, "YUYV needs an even width, got %u", width);   // color/yuv/mod.rs:282-284
    const size_t npx = (size_t)width * height * batch;
    KB200_TRY(check_slice("src", src_len, npx * 3)); KB200_TRY(check_slice("dst", dst_len, npx * 2));
    const size_t npairs = npx / 2;
    yuyv_from_rgb_kernel<<<stream_grid(npairs, 256, 16), 256, 0, as_stream(stream)>>>(src, dst, npairs);
    return check_launch("yuyv_from_rgb_kernel");
}

KB200_API int kb200_nv12_from_rgb_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len,
                                     uint32_t width, uint32_t height, uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if ((width & 1u) || (height & 1u)) return fail(KB200_ERR_INVALID_ARGUMENT, "NV12 needs even dimensions, got %ux%u", width, height);   // color/yuv/mod.rs:298-300
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    const size_t frame = (size_t)width * height * 3 / 2;
    KB200_TRY(check_slice("src", src_len, (size_t)width * height * 3 * batch)); KB200_TRY(check_slice("dst", dst_len, frame * batch));
    dim3 block(32, 8), grid(div_up(width / 2, 32), div_up(height / 2, 8), batch);
    nv12_from_rgb_kernel<<<grid, block, 0, as_stream(stream)>>>(src, dst, width, height, frame);
    return check_launch("nv12_from_rgb_kernel");
}

}  // extern "C"
