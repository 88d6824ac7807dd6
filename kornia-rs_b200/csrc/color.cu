// color.cu — gray_from_rgb (f32, u8) and the BT.601-limited Q20 video decoders (NV12, YUYV).
//
// Reference: color/gray/kernels.rs (CPU), cuda/color/gray.rs:17-68 (GPU twin, 1 px or 4 px per
// thread, scalar 4-byte accesses); color/yuv/kernels.rs:707-1069 (CPU), cuda/color/video.rs:33-130
// (GPU twin, 1 thread per 2x2 block, byte stores).
//
// Design: these are pure streaming ops (16 B/px, 4 B/px, 4.5 B/px, 5 B/px).  Every thread
// moves whole 16-byte vectors in both directions (LDG.128 / STG.128, streaming cache hints),
// de-interleaving the stride-3 pixels in registers; grids are sized so each SM holds several
// CTAs with ≥ 4 independent 16-byte loads in flight per thread.
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

__device__ __forceinline__ void pack_rgb16(const uint32_t yw[4], const ChromaTerms ct[8], uint4 out[3]) {
    uint32_t w[12];
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // 4 px -> 12 bytes = 3 words: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
        int r[4], g[4], b[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int yy = yy_term((int)((yw[k] >> (8 * j)) & 0xFFu));
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

__global__ void __launch_bounds__(128) rgb_from_nv12_vec16(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                           uint32_t width, uint32_t height, size_t frame_bytes) {
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
    uint4 yt = make_uint4(0, 0, 0, 0), yb = yt, uv = yt;
    if (active) {
        yt = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)(2 * cy) * width + x));
        yb = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)(2 * cy + 1) * width + x));
        uv = ldg_stream_u4(reinterpret_cast<const uint4*>(frame + (size_t)width * height + (size_t)cy * width + x));
    }
    const uint32_t uvw[4] = {uv.x, uv.y, uv.z, uv.w};
    ChromaTerms ct[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t pair = (uvw[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
        ct[k] = chroma_terms((int)(pair & 0xFFu), (int)(pair >> 8));
    }
    uint4 o[3];
    const uint32_t ytw[4] = {yt.x, yt.y, yt.z, yt.w};
    const uint32_t ybw[4] = {yb.x, yb.y, yb.z, yb.w};
    uint4* d0 = reinterpret_cast<uint4*>(out + ((size_t)(2 * cy) * width + (size_t)gx0 * 16) * 3);       // this warp's 1536-B run, top row
    uint4* d1 = reinterpret_cast<uint4*>(out + ((size_t)(2 * cy + 1) * width + (size_t)gx0 * 16) * 3);   // bottom row
    if (full_warp) {
        pack_rgb16(ytw, ct, o);
        store_rgb48_coalesced(d0, stage[wid], lane, o);
        pack_rgb16(ybw, ct, o);
        store_rgb48_coalesced(d1, stage[wid], lane, o);
    } else if (active) {   // ragged last warp of a row: direct 48-B stores
        pack_rgb16(ytw, ct, o);
        stg_stream_u4(d0 + 3 * lane, o[0]); stg_stream_u4(d0 + 3 * lane + 1, o[1]); stg_stream_u4(d0 + 3 * lane + 2, o[2]);
        pack_rgb16(ybw, ct, o);
        stg_stream_u4(d1 + 3 * lane, o[0]); stg_stream_u4(d1 + 3 * lane + 1, o[1]); stg_stream_u4(d1 + 3 * lane + 2, o[2]);
    }
}

// Generic fallback (any even width / unaligned buffers): one thread per 2x2 block.
__global__ void rgb_from_nv12_generic(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t width,
                                      uint32_t height, size_t frame_bytes) {
    const uint32_t cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y;
    if (cx >= width / 2 || cy >= height / 2) return;
    const uint8_t* frame = src + (size_t)blockIdx.z * frame_bytes;
    uint8_t* out = dst + (size_t)blockIdx.z * (size_t)width * height * 3;
    const uint8_t* uvp = frame + (size_t)width * height + (size_t)cy * width + 2 * cx;
    const ChromaTerms ct = chroma_terms(uvp[0], uvp[1]);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const size_t p = (size_t)(2 * cy + dy) * width + 2 * cx + dx;
            int r, g, b;
            decode_rgb(yy_term(frame[p]), ct, r, g, b);
            out[3 * p] = (uint8_t)r; out[3 * p + 1] = (uint8_t)g; out[3 * p + 2] = (uint8_t)b;
        }
}

// ── YUYV → RGB8 ─────────────────────────────────────────────────────────────────────────────
// One thread: 16 px = 32 B in (2 x LDG.128), 48 B out (3 x STG.128).  Flat over the whole batch
// (rows are independent and tight), requires total px % 16 == 0 and aligned bases.
__device__ __forceinline__ void yuyv_decode16(const uint4& A, const uint4& B, uint4 o[3]) {
    const uint32_t g4[8] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w};  // each word: Y0 U Y1 V
    uint32_t yw[4];
    ChromaTerms ct[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t w = g4[k];
        ct[k] = chroma_terms((int)((w >> 8) & 0xFFu), (int)(w >> 24));
        const uint32_t ypair = __byte_perm(w, 0, 0x4420);   // {Y0, Y1, 0, 0}
        if (k & 1) yw[k >> 1] |= ypair << 16; else yw[k >> 1] = ypair;
    }
    pack_rgb16(yw, ct, o);
}

// A warp owns 32 consecutive 16-px groups = 1024 B in, 1536 B out, both contiguous: the loads are issued
// lane-contiguous (2 x LDG.128 per lane over the warp's run) and handed to their owners through shared memory, the
// stores go back through it (store_rgb48_coalesced) — every global access instruction covers whole 128-B lines.
__global__ void __launch_bounds__(256) rgb_from_yuyv_vec16(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                                           size_t ngroups) {
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
            yuyv_decode16(A, B, o);
            store_rgb48_coalesced(dst + 3 * q0, st, lane, o);
        } else if (q0 + lane < ngroups) {   // ragged tail warp
            const size_t q = q0 + lane;
            yuyv_decode16(ldg_stream_u4(src + 2 * q), ldg_stream_u4(src + 2 * q + 1), o);
            stg_stream_u4(dst + 3 * q, o[0]); stg_stream_u4(dst + 3 * q + 1, o[1]); stg_stream_u4(dst + 3 * q + 2, o[2]);
        }
    }
}

__global__ void rgb_from_yuyv_generic(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t first_group,
                                      size_t ngroups) {
    const size_t g = first_group + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ngroups) return;
    const uint8_t* s = src + 4 * g;
    const ChromaTerms ct = chroma_terms(s[1], s[3]);
    int r, gg, b;
    decode_rgb(yy_term(s[0]), ct, r, gg, b);
    dst[6 * g] = (uint8_t)r; dst[6 * g + 1] = (uint8_t)gg; dst[6 * g + 2] = (uint8_t)b;
    decode_rgb(yy_term(s[2]), ct, r, gg, b);
    dst[6 * g + 3] = (uint8_t)r; dst[6 * g + 4] = (uint8_t)gg; dst[6 * g + 5] = (uint8_t)b;
}

static inline unsigned stream_grid(size_t items, unsigned block, unsigned ctas_per_sm) {
    const size_t want = (items + block - 1) / block;
    const size_t cap = (size_t)device_info().sm_count * ctas_per_sm;
    return (unsigned)std::max<size_t>(1, std::min(want, cap));
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

KB200_API int kb200_rgb_from_nv12_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                     size_t dst_len, uint32_t width, uint32_t height, uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if ((width & 1u) || (height & 1u)) return fail(KB200_ERR_INVALID_ARGUMENT, "NV12 needs even dimensions, got %ux%u", width, height);
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535", batch);
    const size_t frame = (size_t)width * height * 3 / 2, out_frame = (size_t)width * height * 3;
    KB200_TRY(check_slice("src", src_len, frame * batch)); KB200_TRY(check_slice("dst", dst_len, out_frame * batch));
    cudaStream_t s = as_stream(stream);
    if ((width % 16u) == 0 && aligned16(src) && aligned16(dst) && (frame % 16u) == 0 && height / 2 <= 65535u) {
        const unsigned groups = width / 16;
        const unsigned bx = groups >= 128 ? 128 : 32 * ((groups + 31) / 32);
        dim3 grid(div_up(groups, bx), height / 2, batch);
        rgb_from_nv12_vec16<<<grid, bx, 0, s>>>(src, dst, width, height, frame);
        return check_launch("rgb_from_nv12_vec16");
    }
    dim3 block(32, 8), grid(div_up(width / 2, 32), div_up(height / 2, 8), batch);
    rgb_from_nv12_generic<<<grid, block, 0, s>>>(src, dst, width, height, frame);
    return check_launch("rgb_from_nv12_generic");
}

KB200_API int kb200_rgb_from_yuyv_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                     size_t dst_len, uint32_t width, uint32_t height, uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(width, height, width, height, batch));
    if (width & 1u) return fail(KB200_ERR_INVALID_ARGUMENT, "YUYV needs an even width, got %u", width);
    const size_t npx = (size_t)width * height * batch;
    KB200_TRY(check_slice("src", src_len, npx * 2)); KB200_TRY(check_slice("dst", dst_len, npx * 3));
    cudaStream_t s = as_stream(stream);
    const size_t ngroups2 = npx / 2;  // 2-px groups
    size_t done = 0;
    if (aligned16(src) && aligned16(dst)) {
        const size_t n16 = npx / 16;
        if (n16) {
            rgb_from_yuyv_vec16<<<stream_grid(n16, 256, 8), 256, 0, s>>>(reinterpret_cast<const uint4*>(src),
                                                                        reinterpret_cast<uint4*>(dst), n16);
            KB200_TRY(check_launch("rgb_from_yuyv_vec16"));
        }
        done = n16 * 8;
    }
    if (done < ngroups2) {
        rgb_from_yuyv_generic<<<div_up(ngroups2 - done, 256), 256, 0, s>>>(src, dst, done, ngroups2);
        KB200_TRY(check_launch("rgb_from_yuyv_generic"));
    }
    return KB200_OK;
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
