// resize.cu — f32 HWC bilinear / nearest resize (a1) and the u8 Q14 bilinear resize (a3).
//
// Reference: resize/mod.rs:114-207 (CPU `resize`), interpolation/bilinear.rs:16-66,
// interpolation/nearest.rs:15-30, cuda/resize.rs:97-235 (GPU twins), resize/bilinear.rs:25-104 +
// resize/kernels.rs:1141-1166 (u8 Q14).
//
// Bit-exactness contract (cuda/resize.rs:113-118): the coordinate is `a*x + b` evaluated as an
// unfused multiply-add, weights are formed first and the four terms summed left to right.  This
// file is compiled with -fmad=false, so plain `*` and `+` already round twice.
//
// The f32 bilinear hot kernel is the row-streaming one in resize_rows.cu (TMA row ring, shared-memory taps, STG.128
// rows); the kernels here are its gather fallback (unaligned rows, nearest, generic channel counts) and the u8 family.
// The TMA row-span staged variant for the u8→f32 CHW headline path lives in resize_fused.cu.
#include "kb200_common.cuh"

namespace kb200 {

struct AxisMap {
    float ax, bx, ay, by;
};

// PixelMapping::coeffs — cuda/resize.rs:462-478
static inline void mapping_coeffs(int mapping, uint32_t src_len, uint32_t dst_len, float* a, float* b) {
    if (mapping == KB200_MAP_HALF_PIXEL) {
        *a = (float)src_len / (float)dst_len;
        *b = 0.5f * *a - 0.5f;
    } else {
        if (dst_len > 1) { *a = (float)(src_len - 1) / (float)(dst_len - 1); *b = 0.0f; }
        else { *a = 0.0f; *b = 0.0f; }
    }
}

// Gather fallback of the f32 C=3 resize (the row-streaming kernel of resize_rows.cu takes every geometry whose rows are
// 16-byte aligned; this one takes the rest, and nearest).  MODE: 0 nearest, 1 bilinear, 2 bilinear + (v - mean) * inv_std.
// Per axis the sampler state is (i0, i1, f) from `axis_taps` — the same expression tree as resize_rows.cu's rr_axis
// (cuda/resize.rs:113-125: clamp(a*i + b, 0, len-1), trunc, +1 tap clamped) — and a pixel is the weights-first, four-term
// left-to-right sum of cuda/resize.rs:127-139.  A thread produces one destination pixel; batch = grid.z.
struct AxisTaps { uint32_t i0, i1; float f; };
__device__ __forceinline__ AxisTaps axis_taps(uint32_t i, float a, float b, uint32_t len) {
    const float s = fmaxf(fminf(a * (float)i + b, (float)(len - 1u)), 0.0f);
    AxisTaps t;
    t.i0 = (uint32_t)s;
    t.i1 = min(t.i0 + 1u, len - 1u);
    t.f = s - (float)t.i0;
    return t;
}

template <int MODE>
__global__ void __launch_bounds__(256) resize_f32_c3_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                            uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, AxisMap m,
                                                            float mean0, float mean1, float mean2, float is0, float is1,
                                                            float is2) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const float* s = src + (size_t)blockIdx.z * sw * sh * 3;
    float* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)y * dw + x) * 3;
    if (MODE == 0) {   // cuda/resize.rs:146-175: (a*i + b) + 0.5, truncated, clamped to the last index
        const uint32_t xi = min((uint32_t)((m.ax * (float)x + m.bx) + 0.5f), sw - 1u);
        const uint32_t yi = min((uint32_t)((m.ay * (float)y + m.by) + 0.5f), sh - 1u);
        const float* p = s + ((size_t)yi * sw + xi) * 3;
        d[0] = __ldg(p); d[1] = __ldg(p + 1); d[2] = __ldg(p + 2);
        return;
    }
    const AxisTaps tx = axis_taps(x, m.ax, m.bx, sw), ty = axis_taps(y, m.ay, m.by, sh);
    const float gy = 1.0f - ty.f, gx = 1.0f - tx.f;
    const float w[4] = {gy * gx, gy * tx.f, ty.f * gx, ty.f * tx.f};          // taps (x0,y0) (x1,y0) (x0,y1) (x1,y1)
    const float* r0 = s + (size_t)ty.i0 * sw * 3;
    const float* r1 = s + (size_t)ty.i1 * sw * 3;
    const float* tap[4] = {r0 + tx.i0 * 3u, r0 + tx.i1 * 3u, r1 + tx.i0 * 3u, r1 + tx.i1 * 3u};
    const float mean[3] = {mean0, mean1, mean2}, inv[3] = {is0, is1, is2};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float c = w[0] * __ldg(tap[0] + k) + w[1] * __ldg(tap[1] + k) + w[2] * __ldg(tap[2] + k) + w[3] * __ldg(tap[3] + k);
        if (MODE == 2) c = (c - mean[k]) * inv[k];
        d[k] = c;
    }
}

// Generic channel count, CPU `resize<C>` semantics (val00 replicate, round() for nearest).
__global__ void __launch_bounds__(256) resize_f32_generic_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                 uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                                                                 uint32_t C, AxisMap m, int bilinear) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const float* s = src + (size_t)blockIdx.z * sw * sh * C;
    float* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)y * dw + x) * C;
    // axis_lut: (a*i + b).clamp(0, max)   resize/mod.rs:169-176
    const float u = fminf(fmaxf(m.ax * (float)x + m.bx, 0.0f), (float)(sw - 1u));
    const float v = fminf(fmaxf(m.ay * (float)y + m.by, 0.0f), (float)(sh - 1u));
    if (!bilinear) {
        const uint32_t iu = min((uint32_t)roundf(u), sw - 1u), iv = min((uint32_t)roundf(v), sh - 1u);
        for (uint32_t k = 0; k < C; ++k) d[k] = __ldg(s + ((size_t)iv * sw + iu) * C + k);
        return;
    }
    const uint32_t iu = (uint32_t)u, iv = (uint32_t)v;  // trunc, u,v >= 0
    const float fu = u - truncf(u), fv = v - truncf(v);
    const bool hx = iu + 1u < sw, hy = iv + 1u < sh;
    const size_t b00 = ((size_t)iv * sw + iu) * C;
    const size_t b01 = hx ? b00 + C : b00;
    const size_t b10 = hy ? b00 + (size_t)sw * C : b00;
    const size_t b11 = (hx && hy) ? b00 + (size_t)sw * C + C : b00;
    const float fuu = 1.0f - fu, fvv = 1.0f - fv;
    const float w00 = fvv * fuu, w10 = fvv * fu, w01 = fv * fuu, w11 = fv * fu;
    for (uint32_t k = 0; k < C; ++k)
        d[k] = w00 * __ldg(s + b00 + k) + w10 * __ldg(s + b01 + k) + w01 * __ldg(s + b10 + k) + w11 * __ldg(s + b11 + k);
}

// ── u8 Q14 bilinear ─────────────────────────────────────────────────────────────────────────
// bilinear_tap (resize/bilinear.rs:25-38) in f64 on the device — one per axis per thread; the
// result is identical to the host LUT because it is the same IEEE f64 expression.
__device__ __forceinline__ void bilinear_tap_q14(uint32_t i, double scale, uint32_t src_len, uint32_t* ofs, uint32_t* fq) {
    const double s = __dadd_rn(__dmul_rn((double)i + 0.5, scale), -0.5);
    long long i0 = (long long)floor(s);
    double f = s - (double)i0;
    if (i0 < 0) { i0 = 0; f = 0.0; }
    else if (i0 >= (long long)src_len - 1) { i0 = (long long)src_len - 2; f = 1.0; }
    const double q = round(__dmul_rn(f, 16384.0));
    *fq = min((uint32_t)q, 16384u);
    *ofs = (uint32_t)i0;
}

// ── u8 kernels of resize_fast_u8_aa (resize/mod.rs:283-410) ──────────────────────────────────
// Thread per destination pixel (pyrup: per 2x2 destination block) with byte loads: a warp's pixels read one
// contiguous byte run per source row and L1 turns the byte loads into whole sectors.  A variant that gave each thread
// four consecutive destination BYTES (one STG.32) and re-evaluated the per-pixel setup per byte measured
// slower: these kernels are bound by instructions per pixel, not by the byte stores.

// resize/kernels.rs:64-75: dst = (a + b + c + d + 2) >> 2 per channel
__global__ void __launch_bounds__(256) pyrdown_2x_rgb_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                                uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const uint8_t* s = src + (size_t)blockIdx.z * sw * sh * 3;
    uint8_t* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)y * dw + x) * 3;
    const uint8_t* r0 = s + ((size_t)(2 * y) * sw + 2 * x) * 3;
    const uint8_t* r1 = r0 + (size_t)sw * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) d[ch] = (uint8_t)(((uint32_t)r0[ch] + r0[3 + ch] + r1[ch] + r1[3 + ch] + 2u) >> 2);
}

// Word-granular pyrdown: a thread produces 4 destination pixels (12 bytes = 3 words) from 2 x 24 source bytes read as
// 6 + 6 aligned words — 15 memory instructions per 4 pixels instead of 60 (the byte version is LSU-bound).  Needs sw % 8 == 0 (row = whole 24-byte groups, 4-byte aligned) and 4-byte aligned bases.
__global__ void __launch_bounds__(256) pyrdown_2x_rgb_u8_w4_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, uint32_t sw,
                                                                   uint32_t sh, uint32_t dw, uint32_t dh) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;   // group of 4 destination pixels
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    const uint32_t groups = dw >> 2;
    if (g >= groups || y >= dh) return;
    const uint32_t srow_w = sw * 3u / 4u, drow_w = dw * 3u / 4u;   // words per row
    const uint32_t* r0 = src + ((size_t)blockIdx.z * sh + 2u * y) * srow_w + 6u * g;
    const uint32_t* r1 = r0 + srow_w;
    uint32_t a[6], b[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { a[k] = __ldg(r0 + k); b[k] = __ldg(r1 + k); }
    auto byte_of_row = [](const uint32_t (&w)[6], int k) -> uint32_t { return (w[k >> 2] >> (8 * (k & 3))) & 0xFFu; };
    uint32_t out[3] = {0u, 0u, 0u};
#pragma unroll
    for (int o = 0; o < 12; ++o) {                 // destination byte o: pixel o / 3, channel o % 3
        const int k = 6 * (o / 3) + (o % 3);       // first source byte; its horizontal neighbour is k + 3
        const uint32_t v = (byte_of_row(a, k) + byte_of_row(a, k + 3) + byte_of_row(b, k) + byte_of_row(b, k + 3) + 2u) >> 2;
        out[o >> 2] |= v << (8 * (o & 3));
    }
    uint32_t* d = dst + ((size_t)blockIdx.z * dh + y) * drow_w + 3u * g;
    d[0] = out[0]; d[1] = out[1]; d[2] = out[2];
}

// resize/kernels.rs:168-181 + :274-281 + resize/pyramid.rs:50-120.
// Horizontal stage H(row)[X]: X = 2j+1 -> (a + avg + 1) >> 1, X = 2j+2 -> (b + avg + 1) >> 1 with a = row[j], b = row[j+1],
// avg = (a + b + 1) >> 1; X = 0 and X = 2sw-1 copy the edge pixel.  Vertical stage: row 2I+1 -> blend(H(I), H(I+1)),
// row 2I+2 -> blend(H(I+1), H(I)), blend(p, q) = (p + ((p + q + 1) >> 1) + 1) >> 1; rows 0 and 2sh-1 are H of the edge row.
// One thread per (j, I) in [-1, sw-1] x [-1, sh-1] produces the 2x2 destination block X in {2j+1, 2j+2}, Y in {2I+1, 2I+2}
// from the four source pixels it shares.  The edges need no special case: with the index clamped, a == b gives
// avg = a and (a + a + 1) >> 1 = a, i.e. exactly the copied edge pixel / edge row of the reference.
__global__ void __launch_bounds__(256) pyrup_2x_rgb_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                              uint32_t sw, uint32_t sh) {
    const int j = (int)(blockIdx.x * blockDim.x + threadIdx.x) - 1;
    const int I = (int)(blockIdx.y * blockDim.y + threadIdx.y) - 1;
    if (j > (int)sw - 1 || I > (int)sh - 1) return;
    const uint32_t dw = 2 * sw;
    const uint8_t* s = src + (size_t)blockIdx.z * sw * sh * 3;
    uint8_t* d = dst + (size_t)blockIdx.z * dw * (2 * sh) * 3;
    const uint32_t ja = (uint32_t)max(j, 0), jb = (uint32_t)min(j + 1, (int)sw - 1);
    const uint32_t Ia = (uint32_t)max(I, 0), Ib = (uint32_t)min(I + 1, (int)sh - 1);
    const uint8_t* ra = s + (size_t)Ia * sw * 3;
    const uint8_t* rb = s + (size_t)Ib * sw * 3;
    const bool x_odd = j >= 0, x_even = j + 1 < (int)sw;     // X = 2j+1 / X = 2j+2 inside the row
    const bool y_top = I >= 0, y_bot = I + 1 < (int)sh;      // Y = 2I+1 / Y = 2I+2 inside the image
    uint8_t* d_top = d + ((size_t)(2 * I + 1) * dw + (size_t)(2 * j + 1)) * 3;   // only dereferenced where valid
    uint8_t* d_bot = d_top + (size_t)dw * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const uint32_t a0 = ra[ja * 3 + ch], b0 = ra[jb * 3 + ch], a1 = rb[ja * 3 + ch], b1 = rb[jb * 3 + ch];
        const uint32_t avg0 = (a0 + b0 + 1u) >> 1, avg1 = (a1 + b1 + 1u) >> 1;
        const uint32_t hao = (a0 + avg0 + 1u) >> 1, hae = (b0 + avg0 + 1u) >> 1;   // H(Ia) at X odd / even
        const uint32_t hbo = (a1 + avg1 + 1u) >> 1, hbe = (b1 + avg1 + 1u) >> 1;   // H(Ib)
        const uint32_t mo = (hao + hbo + 1u) >> 1, me = (hae + hbe + 1u) >> 1;
        if (y_top) {
            if (x_odd) d_top[ch] = (uint8_t)((hao + mo + 1u) >> 1);
            if (x_even) d_top[3 + ch] = (uint8_t)((hae + me + 1u) >> 1);
        }
        if (y_bot) {
            if (x_odd) d_bot[ch] = (uint8_t)((hbo + mo + 1u) >> 1);
            if (x_even) d_bot[3 + ch] = (uint8_t)((hbe + me + 1u) >> 1);
        }
    }
}

// resize/bilinear.rs:70 + resize/kernels.rs:1141-1166 — Q14 bilinear, taps from the f64 expression (bilinear_tap_q14).
template <int C>
__global__ void __launch_bounds__(256) resize_bilinear_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                                 uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                                                                 double scale_x, double scale_y) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const uint8_t* s = src + (size_t)blockIdx.z * sw * sh * C;
    uint8_t* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)y * dw + x) * C;
    uint32_t xi, fx, yi, fy;
    bilinear_tap_q14(x, scale_x, sw, &xi, &fx);
    bilinear_tap_q14(y, scale_y, sh, &yi, &fy);
    const unsigned long long fx1 = 16384u - fx, fy1 = 16384u - fy;
    const uint8_t* r0 = s + ((size_t)yi * sw + xi) * C;
    // fy == 0 (e.g. every row of an odd integer downscale): `bot * 0` contributes exactly nothing in the Q28
    // integer sum, so the y1 row is not addressed at all — one source row in three is read at 2160 -> 720
    const uint8_t* r1 = fy ? r0 + (size_t)sw * C : r0;
#pragma unroll
    for (int ch = 0; ch < C; ++ch) {
        const unsigned long long p00 = r0[ch], p01 = r0[C + ch], p10 = r1[ch], p11 = r1[C + ch];
        const unsigned long long top = p00 * fx1 + p01 * fx;
        const unsigned long long bot = p10 * fx1 + p11 * fx;
        d[ch] = (uint8_t)((top * fy1 + bot * (unsigned long long)fy + (1ull << 27)) >> 28);
    }
}

// Exact 3:1 downscale (2160p -> 720p, 1080p -> 360p): the f64 half-pixel tap is s = 3i + 1 with fraction exactly 0 on
// both axes, so the Q28 blend returns p00 unchanged — the result is the centre pixel of every 3x3 block.  A thread
// copies 4 destination pixels: 36 source bytes read as 9 aligned words, bytes 3..5, 12..14, 21..23, 30..32 packed into
// 3 words (12 memory instructions per 4 pixels instead of 60; one source row in three is read).
__global__ void __launch_bounds__(256) resize_bilinear_u8_c3_3to1_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst,
                                                                         uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;   // group of 4 destination pixels
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (g >= (dw >> 2) || y >= dh) return;
    const uint32_t srow_w = sw * 3u / 4u, drow_w = dw * 3u / 4u;
    const uint32_t* r = src + ((size_t)blockIdx.z * sh + 3u * y + 1u) * srow_w + 9u * g;
    uint32_t w[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) w[k] = __ldg(r + k);
    uint32_t out[3] = {0u, 0u, 0u};
#pragma unroll
    for (int o = 0; o < 12; ++o) {                  // destination byte o: pixel o / 3, channel o % 3
        const int k = 9 * (o / 3) + 3 + (o % 3);    // source pixel 3*px + 1
        out[o >> 2] |= ((w[k >> 2] >> (8 * (k & 3))) & 0xFFu) << (8 * (o & 3));
    }
    uint32_t* d = dst + ((size_t)blockIdx.z * dh + y) * drow_w + 3u * g;
    d[0] = out[0]; d[1] = out[1]; d[2] = out[2];
}

// resize/nearest.rs:18-21: clamp(floor((i + 0.5) * scale)) in f64
__device__ __forceinline__ uint32_t nearest_index_f64(uint32_t i, double scale, uint32_t src_len) {
    const long long v = (long long)floor(__dmul_rn((double)i + 0.5, scale));
    return (uint32_t)min(max(v, 0ll), (long long)src_len - 1);
}
template <int C>
__global__ void __launch_bounds__(256) resize_nearest_u8_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t sw,
                                                                uint32_t sh, uint32_t dw, uint32_t dh, uint32_t Cdyn, double scale_x,
                                                                double scale_y) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const uint32_t Cn = C > 0 ? (uint32_t)C : Cdyn;
    const uint32_t xi = nearest_index_f64(x, scale_x, sw), yi = nearest_index_f64(y, scale_y, sh);
    const uint8_t* p = src + ((size_t)blockIdx.z * sw * sh + (size_t)yi * sw + xi) * Cn;
    uint8_t* d = dst + ((size_t)blockIdx.z * dw * dh + (size_t)y * dw + x) * Cn;
    if (C > 0) {
#pragma unroll
        for (int ch = 0; ch < (C > 0 ? C : 1); ++ch) d[ch] = p[ch];
    } else {
        for (uint32_t ch = 0; ch < Cn; ++ch) d[ch] = p[ch];
    }
}

int launch_resize_rows_f32(int mode, cudaStream_t s, const float* src, float* dst, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                           uint32_t batch, float ax, float bx, float ay, float by, const float* mean, const float* inv_std, bool* handled);   // resize_rows.cu

static inline int check_batch(uint32_t batch) {
    if (batch > 65535u) return fail(KB200_ERR_INVALID_ARGUMENT, "batch %u exceeds 65535 per call", batch);
    return KB200_OK;
}

static int launch_resize_c3(int mode, kb200_stream_t stream, const float* src, size_t src_len, float* dst,
                            size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t batch,
                            int mapping, const float* mean, const float* stdv) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch)); KB200_TRY(check_batch(batch));
    if (mapping != KB200_MAP_HALF_PIXEL && mapping != KB200_MAP_ALIGN_CORNERS)
        return fail(KB200_ERR_INVALID_ARGUMENT, "unknown pixel mapping %d", mapping);
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * 3 * batch));
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * 3 * batch));
    float is[3] = {1, 1, 1}, mn[3] = {0, 0, 0};
    if (mode == 2) {
        if (!mean || !stdv) return fail(KB200_ERR_INVALID_ARGUMENT, "mean/std must not be null");
        if (stdv[0] == 0.0f || stdv[1] == 0.0f || stdv[2] == 0.0f)
            return fail(KB200_ERR_INVALID_ARGUMENT, "std must be non-zero for all channels");  // cuda/resize.rs:606-610
        for (int c = 0; c < 3; ++c) { is[c] = 1.0f / stdv[c]; mn[c] = mean[c]; }
    }
    AxisMap m;
    mapping_coeffs(mapping, sw, dw, &m.ax, &m.bx);
    mapping_coeffs(mapping, sh, dh, &m.ay, &m.by);
    dim3 block(32, 8), grid(div_up(dw, 32), div_up(dh, 8), batch);
    cudaStream_t s = as_stream(stream);
    if (mode != 0) {   // bilinear: the row-streaming kernel (resize_rows.cu) whenever the geometry allows TMA row copies
        bool handled = false;
        KB200_TRY(launch_resize_rows_f32(mode, s, src, dst, sw, sh, dw, dh, batch, m.ax, m.bx, m.ay, m.by, mn, is, &handled));
        if (handled) return KB200_OK;
    }
    if (mode == 0) resize_f32_c3_kernel<0><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, m, 0, 0, 0, 1, 1, 1);
    else if (mode == 1) resize_f32_c3_kernel<1><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, m, 0, 0, 0, 1, 1, 1);
    else resize_f32_c3_kernel<2><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, m, mn[0], mn[1], mn[2], is[0], is[1], is[2]);
    return check_launch("resize_f32_c3_kernel");
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_resize_bilinear_f32_c3(kb200_stream_t stream, const float* src, size_t src_len, float* dst,
                                           size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                                           uint32_t batch, int mapping) {
    return launch_resize_c3(1, stream, src, src_len, dst, dst_len, sw, sh, dw, dh, batch, mapping, nullptr, nullptr);
}

KB200_API int kb200_resize_nearest_f32_c3(kb200_stream_t stream, const float* src, size_t src_len, float* dst,
                                          size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                                          uint32_t batch, int mapping) {
    return launch_resize_c3(0, stream, src, src_len, dst, dst_len, sw, sh, dw, dh, batch, mapping, nullptr, nullptr);
}

KB200_API int kb200_resize_bilinear_normalize_f32_c3(kb200_stream_t stream, const float* src, size_t src_len,
                                                     float* dst, size_t dst_len, uint32_t sw, uint32_t sh,
                                                     uint32_t dw, uint32_t dh, uint32_t batch, const float mean[3],
                                                     const float stdv[3], int mapping) {
    return launch_resize_c3(2, stream, src, src_len, dst, dst_len, sw, sh, dw, dh, batch, mapping, mean, stdv);
}

KB200_API int kb200_resize_f32(kb200_stream_t stream, const float* src, size_t src_len, float* dst, size_t dst_len,
                               uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t C, uint32_t batch,
                               int interp) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch)); KB200_TRY(check_batch(batch));
    if (C == 0 || C > 4) return fail(KB200_ERR_UNSUPPORTED, "CUDA resize supports 1..4 channels only, got %u", C);
    if (interp != KB200_INTERP_NEAREST && interp != KB200_INTERP_BILINEAR)
        return fail(KB200_ERR_UNSUPPORTED, "CUDA resize supports Nearest/Bilinear only (mode %d)", interp);
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * C * batch));
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * C * batch));
    cudaStream_t s = as_stream(stream);
    if (sw == dw && sh == dh) {  // resize/mod.rs:134-137: same size is a copy
        cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)sw * sh * C * batch * sizeof(float), cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaMemcpyAsync failed: %s", cudaGetErrorString(e));
        return KB200_OK;
    }
    AxisMap m;
    mapping_coeffs(KB200_MAP_HALF_PIXEL, sw, dw, &m.ax, &m.bx);
    mapping_coeffs(KB200_MAP_HALF_PIXEL, sh, dh, &m.ay, &m.by);
    dim3 block(32, 8), grid(div_up(dw, 32), div_up(dh, 8), batch);
    resize_f32_generic_kernel<<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, C, m, interp == KB200_INTERP_BILINEAR);
    return check_launch("resize_f32_generic_kernel");
}

KB200_API int kb200_resize_bilinear_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst,
                                       size_t dst_len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh,
                                       uint32_t C, uint32_t batch) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch)); KB200_TRY(check_batch(batch));
    if (!(C == 1 || C == 3 || C == 4)) return fail(KB200_ERR_UNSUPPORTED, "u8 bilinear resize supports 1, 3 or 4 channels, got %u", C);
    if (sw < 2 || sh < 2) return fail(KB200_ERR_INVALID_ARGUMENT, "u8 bilinear resize needs a source of at least 2x2, got %ux%u", sw, sh);  // resize/mod.rs:318-320
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * C * batch));
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * C * batch));
    const double scale_x = (double)sw / (double)dw, scale_y = (double)sh / (double)dh;
    dim3 block(32, 8), grid(div_up(dw, 32), div_up(dh, 8), batch);
    cudaStream_t s = as_stream(stream);
    if (C == 3 && sw == 3 * dw && sh == 3 * dh && (dw & 3u) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3u) == 0) {
        dim3 wgrid(div_up(dw / 4, 32), div_up(dh, 8), batch);
        resize_bilinear_u8_c3_3to1_kernel<<<wgrid, block, 0, s>>>(reinterpret_cast<const uint32_t*>(src), reinterpret_cast<uint32_t*>(dst), sw, sh, dw, dh);
        return check_launch("resize_bilinear_u8_c3_3to1_kernel");
    }
    if (C == 1) resize_bilinear_u8_kernel<1><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, scale_x, scale_y);
    else if (C == 3) resize_bilinear_u8_kernel<3><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, scale_x, scale_y);
    else resize_bilinear_u8_kernel<4><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, scale_x, scale_y);
    return check_launch("resize_bilinear_u8_kernel");
}


/* resize/mod.rs:348 resize_fast_u8_aa for Nearest / Bilinear — the reference's path selection (resize_u8_path, :283-337):
 * exact 2x down / up on RGB take the pyramid arms, Nearest works for any channel count, Bilinear is the Q14 arm. */
KB200_API int kb200_resize_fast_u8(kb200_stream_t stream, const uint8_t* src, size_t src_len, uint8_t* dst, size_t dst_len,
                                   uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t C, uint32_t batch, int interp) {
    KB200_TRY(check_ptr("src", src)); KB200_TRY(check_ptr("dst", dst));
    KB200_TRY(check_geometry(sw, sh, dw, dh, batch)); KB200_TRY(check_batch(batch));
    if (C == 0) return fail(KB200_ERR_UNSUPPORTED, "channel count must be at least 1");
    KB200_TRY(check_slice("dst", dst_len, (size_t)dw * dh * C * batch));
    KB200_TRY(check_slice("src", src_len, (size_t)sw * sh * C * batch));
    cudaStream_t s = as_stream(stream);
    dim3 block(32, 8), grid(div_up(dw, 32), div_up(dh, 8), batch);
    if (interp == KB200_INTERP_BILINEAR && C == 3 && sw == 2 * dw && sh == 2 * dh && sw >= 2 && sh >= 2) {
        if ((sw & 7u) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3u) == 0) {
            dim3 wgrid(div_up(dw / 4, 32), div_up(dh, 8), batch);
            pyrdown_2x_rgb_u8_w4_kernel<<<wgrid, block, 0, s>>>(reinterpret_cast<const uint32_t*>(src), reinterpret_cast<uint32_t*>(dst), sw, sh, dw, dh);
            return check_launch("pyrdown_2x_rgb_u8_w4_kernel");
        }
        pyrdown_2x_rgb_u8_kernel<<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh);
        return check_launch("pyrdown_2x_rgb_u8_kernel");
    }
    if (interp == KB200_INTERP_BILINEAR && C == 3 && dw == 2 * sw && dh == 2 * sh && sw >= 2 && sh >= 2) {
        dim3 ugrid(div_up(sw + 1, 32), div_up(sh + 1, 8), batch);   // (j, I) in [-1, sw-1] x [-1, sh-1]
        pyrup_2x_rgb_u8_kernel<<<ugrid, block, 0, s>>>(src, dst, sw, sh);
        return check_launch("pyrup_2x_rgb_u8_kernel");
    }
    if (interp == KB200_INTERP_NEAREST) {
        // exact 3:1: floor((i + 0.5) * 3) = 3i + 1 — the same centre-pixel gather as the bilinear 3:1 case
        if (C == 3 && sw == 3 * dw && sh == 3 * dh && (dw & 3u) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 3u) == 0) {
            dim3 wgrid(div_up(dw / 4, 32), div_up(dh, 8), batch);
            resize_bilinear_u8_c3_3to1_kernel<<<wgrid, block, 0, s>>>(reinterpret_cast<const uint32_t*>(src), reinterpret_cast<uint32_t*>(dst), sw, sh, dw, dh);
            return check_launch("resize_bilinear_u8_c3_3to1_kernel");
        }
        const double scale_x = (double)sw / (double)dw, scale_y = (double)sh / (double)dh;
        if (C == 1) resize_nearest_u8_kernel<1><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, C, scale_x, scale_y);
        else if (C == 3) resize_nearest_u8_kernel<3><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, C, scale_x, scale_y);
        else if (C == 4) resize_nearest_u8_kernel<4><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, C, scale_x, scale_y);
        else resize_nearest_u8_kernel<0><<<grid, block, 0, s>>>(src, dst, sw, sh, dw, dh, C, scale_x, scale_y);
        return check_launch("resize_nearest_u8_kernel");
    }
    if (interp == KB200_INTERP_BILINEAR) return kb200_resize_bilinear_u8(stream, src, src_len, dst, dst_len, sw, sh, dw, dh, C, batch);
    return fail(KB200_ERR_UNSUPPORTED, "resize_fast_u8: interpolation mode %d is not built (Nearest and Bilinear are)", interp);
}

}  // extern "C"
