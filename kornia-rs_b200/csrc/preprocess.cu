// preprocess.cu — the fused camera preprocess (a12; BASELINE config 3): raw frame (RGB/BGR/RGBA/
// Gray/NV12/YUYV, tight or pitched) → letterbox/stretch resample → (v/255 - mean) * inv_std →
// planar CHW f32 or f16, for a whole batch in ONE launch.
//
// Reference: preprocess.rs:430-647 (the CUDA source string — the specification of this path; there
// is no CPU implementation for the camera formats), launch seam :1324-1372, batch loop :1277-1280
// (one launch per frame), Affine::new :349-370.
//
// Arithmetic is the reference's, op for op (it JIT-compiles with fmad=false, IEEE division):
//   sx = ((float)ox - pad_x) / scale_x                         plan_pixel :437-448
//   bilinear taps x0=floor(sx), x1=min(x0+1,W-1), x0=max(x0,0); decode-in-tap (Q20 → float 0..255)
//   top = t00 + (t10 - t00)*ax ; px = top + (bot - top)*ay     sample_bilinear :534-554
//   o = (px / 255.0f - mean) * inv_std                         BODY :610-612
// One exact shortcut: when ax == 0 the x1 taps are multiplied by zero — `t00 + (t10-t00)*0` is t00
// bit-for-bit for the finite decoded values — so those taps are not fetched (same for ay == 0).  At
// integer scales (1080p NV12 → 1080p CHW, config 3a) that removes 3 of the 4 decodes per pixel.
#include <cuda_fp16.h>

#include "kb200_common.cuh"

namespace kb200 {

struct PreFrames {
    const uint8_t* base;  // strided mode
    size_t stride;
    const uint8_t* ptr[256];  // pointer-table mode
};

// preprocess.rs:461-484 — manual RNE f32 -> binary16 (kept bit-identical, including its rule that
// any exp >= 31 input with a nonzero mantissa gets the quiet bit).
__device__ __forceinline__ unsigned short f2h_ref(float f) {
    const unsigned int x = __float_as_uint(f);
    const unsigned int sign = (x >> 16) & 0x8000u;
    const int exp = (int)((x >> 23) & 0xFFu) - 127 + 15;
    unsigned int man = x & 0x7FFFFFu;
    if (exp >= 31) {
        const unsigned int nan_bit = (man != 0u) ? 0x0200u : 0u;
        return (unsigned short)(sign | 0x7C00u | nan_bit);
    }
    if (exp <= 0) {
        if (exp < -10) return (unsigned short)sign;
        man |= 0x800000u;
        const unsigned int shift = (unsigned int)(14 - exp);
        unsigned short h = (unsigned short)(sign | (man >> shift));
        const unsigned int rem = man & ((1u << shift) - 1u);
        const unsigned int mid = 1u << (shift - 1u);
        if (rem > mid || (rem == mid && (h & 1u))) h++;
        return h;
    }
    unsigned short h = (unsigned short)(sign | ((unsigned int)exp << 10) | (man >> 13));
    const unsigned int rem = man & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) h++;
    return h;
}

// `p / 255.0f`, exactly: q = p*c; e = fma(-q, 255, p); q' = fma(e, c, q) with c = RN(1/255) (Markstein's correction).
// Verified bit-identical to the IEEE division for EVERY float in [0, 256) by kb200_selftest_div255 (1.13e9 inputs,
// tests/test_gpu_parity.py::test_div255_identity_exhaustive); every px here is a decoded or interpolated value in [0, 255].
__device__ __forceinline__ float div255_exact(float p) {
    const float c = 0.00392156885936856269836f;  // 0x3b808081
    const float q = p * c;
    const float e = fmaf(-q, 255.0f, p);
    return fmaf(e, c, q);
}

__device__ __forceinline__ void yuv_to_rgbf(int yv, int u, int v, float px[3]) {  // :501-508
    const ChromaTerms t = chroma_terms(u, v);
    int r, g, b;
    decode_rgb(yy_term(yv), t, r, g, b);
    px[0] = (float)r; px[1] = (float)g; px[2] = (float)b;
}

__device__ __forceinline__ void fetch_px(const uint8_t* __restrict__ src, int x, int y, const kb200_preprocess_desc& d,
                                         float px[3]) {  // :510-530
    if (d.fmt <= 1) {
        const uint8_t* p = src + (long long)y * d.src_pitch + x * d.src_bpp;
        if (d.fmt == 0) { px[0] = (float)p[0]; px[1] = (float)p[1]; px[2] = (float)p[2]; }
        else { px[0] = (float)p[2]; px[1] = (float)p[1]; px[2] = (float)p[0]; }
    } else if (d.fmt == 2) {
        const float v = (float)src[(long long)y * d.src_pitch + x];
        px[0] = v; px[1] = v; px[2] = v;
    } else if (d.fmt == 3) {
        const int yv = src[(long long)y * d.src_w + x];
        const uint8_t* uv = src + (long long)d.src_w * d.src_h + (long long)(y >> 1) * d.src_w + (x >> 1) * 2;
        yuv_to_rgbf(yv, uv[0], uv[1], px);
    } else {
        const uint8_t* grp = src + (long long)y * d.src_pitch + (x >> 1) * 4;
        const int yv = grp[(x & 1) ? 2 : 0];
        yuv_to_rgbf(yv, grp[1], grp[3], px);
    }
}

// preprocess.rs:481-488 (kernel source): 1-D Lanczos-3 weight — the CUDA math library's sinf, like the reference kernel
__device__ __forceinline__ float pre_lanczos_w(float dd) {
    const float ad = fabsf(dd);
    if (ad < 1e-6f) return 1.0f;
    if (ad >= 3.0f) return 0.0f;
    const float pd = 3.14159265358979f * dd;
    return __fdiv_rn(3.0f * sinf(pd) * sinf(__fdiv_rn(pd, 3.0f)), pd * pd);
}

// SAMP: kb200_interp — 0 nearest, 1 bilinear, 3 Lanczos-3 (6x6 taps, clamp-to-edge, weights renormalised by their sum)
template <bool F16, int SAMP, bool PTRS>
__global__ void __launch_bounds__(256) preprocess_generic_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                 const __grid_constant__ PreFrames fr, void* __restrict__ dst,
                                                                 uint32_t frame0) {
    const int pixels = d.dst_w * d.dst_h;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pixels) return;
    const uint32_t f = blockIdx.y;
    const uint8_t* src = PTRS ? fr.ptr[f] : fr.base + (size_t)(frame0 + f) * fr.stride;
    const int ox = i % d.dst_w, oy = i / d.dst_w;
    const float sx = __fdiv_rn((float)ox - d.pad_x, d.scale_x);
    const float sy = __fdiv_rn((float)oy - d.pad_y, d.scale_y);
    const bool inside = !(sx < 0.0f || sy < 0.0f || sx >= (float)d.src_w || sy >= (float)d.src_h);
    float px[3];
    if (inside) {
        if (SAMP == KB200_INTERP_LANCZOS) {   // preprocess.rs:565-590 sample_lanczos: acc += w * t (unfused), one division per channel
            const int x0 = (int)floorf(sx), y0 = (int)floorf(sy);
            float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f, wsum = 0.0f;
            for (int j = -2; j <= 3; ++j) {
                const int yj = y0 + j;
                const float wy = pre_lanczos_w(sy - (float)yj);
                const int yc = min(max(yj, 0), d.src_h - 1);
                for (int ii = -2; ii <= 3; ++ii) {
                    const int xi = x0 + ii;
                    const float w = wy * pre_lanczos_w(sx - (float)xi);
                    const int xc = min(max(xi, 0), d.src_w - 1);
                    float t[3];
                    fetch_px(src, xc, yc, d, t);
                    acc0 += w * t[0]; acc1 += w * t[1]; acc2 += w * t[2];
                    wsum += w;
                }
            }
            px[0] = __fdiv_rn(acc0, wsum); px[1] = __fdiv_rn(acc1, wsum); px[2] = __fdiv_rn(acc2, wsum);
        } else if (SAMP == KB200_INTERP_BILINEAR) {
            int x0 = (int)floorf(sx), y0 = (int)floorf(sy);
            const float ax = sx - (float)x0, ay = sy - (float)y0;
            const int x1 = min(x0 + 1, d.src_w - 1), y1 = min(y0 + 1, d.src_h - 1);
            x0 = max(x0, 0); y0 = max(y0, 0);
            float t00[3], t10[3], t01[3], t11[3];
            fetch_px(src, x0, y0, d, t00);
            const bool need_x = ax != 0.0f, need_y = ay != 0.0f;
            if (need_x) fetch_px(src, x1, y0, d, t10);
            if (need_y) {
                fetch_px(src, x0, y1, d, t01);
                if (need_x) fetch_px(src, x1, y1, d, t11);
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float top = need_x ? t00[c] + (t10[c] - t00[c]) * ax : t00[c];
                if (need_y) {
                    const float bot = need_x ? t01[c] + (t11[c] - t01[c]) * ax : t01[c];
                    px[c] = top + (bot - top) * ay;
                } else {
                    px[c] = top;
                }
            }
        } else {
            const int xn = min(max((int)roundf(sx), 0), d.src_w - 1);
            const int yn = min(max((int)roundf(sy), 0), d.src_h - 1);
            fetch_px(src, xn, yn, d, px);
        }
    } else {
        px[0] = d.pad_value; px[1] = d.pad_value; px[2] = d.pad_value;
    }
    float q0, q1, q2;
    if (inside && SAMP != KB200_INTERP_LANCZOS) { q0 = div255_exact(px[0]); q1 = div255_exact(px[1]); q2 = div255_exact(px[2]); }
    else if (inside) { q0 = __fdiv_rn(px[0], 255.0f); q1 = __fdiv_rn(px[1], 255.0f); q2 = __fdiv_rn(px[2], 255.0f); }  // Lanczos overshoots [0, 255]
    else { q0 = __fdiv_rn(px[0], 255.0f); q1 = q0; q2 = q0; }  // pad_value is caller-supplied: plain IEEE division
    const float o0 = (q0 - d.mean[0]) * d.inv_std[0];
    const float o1 = (q1 - d.mean[1]) * d.inv_std[1];
    const float o2 = (q2 - d.mean[2]) * d.inv_std[2];
    const size_t out = (size_t)(frame0 + f) * 3 * pixels + i;
    if (F16) {
        unsigned short* o = reinterpret_cast<unsigned short*>(dst);
        o[out] = f2h_ref(o0); o[out + pixels] = f2h_ref(o1); o[out + 2 * (size_t)pixels] = f2h_ref(o2);
    } else {
        float* o = reinterpret_cast<float*>(dst);
        o[out] = o0; o[out + pixels] = o1; o[out + 2 * (size_t)pixels] = o2;
    }
}

// ── NV12 identity fast path (config 3a: 1080p NV12 → [N,3,1080,1920], scale 1, no pad) ─────────────────────
// When scale_x == scale_y == 1 and pad == 0, sx = (float)ox / 1.0f = ox exactly, so ax = ay = 0 and the
// bilinear (and the nearest) sample is the decoded tap (ox, oy) itself — bit-for-bit (see the header note).
// The generic kernel is issue-bound here, far below the HBM roofline (ncu).  This kernel is a pure streaming decode:
//   * one thread = 8 luma columns x 2 rows (one chroma row): 3 x LDG.64 in, 12 x STG.128 out (f32) — a warp
//     reads 256 contiguous bytes per plane row and writes 1 KB contiguous per output plane row;
//   * the chroma terms (CUB*u+half, CUG*u+CVG*v+half, CVR*v+half) are computed once per 2x2 block;
//   * `px / 255.0f` for the INTEGER px in [0,255] is evaluated as q = px*c; e = fma(-q,255,px); q' = fma(e,c,q)
//     with c = RN(1/255): Markstein's correction gives the correctly rounded quotient (verified for all 256
//     values, tests/test_abi_and_host.py) — identical bits to the IEEE division the reference performs.
template <bool F16>
__device__ __forceinline__ void nv12_store4(void* __restrict__ dst, size_t idx, const float v[4]) {
    if (F16) {
        unsigned short hbits[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            // hardware RNE == the reference's manual RNE for every finite value below the f16 overflow threshold;
            // beyond it (and for NaN) defer to the reference's own bit rules
            hbits[i] = (fabsf(v[i]) < 65504.0f) ? __half_as_ushort(__float2half_rn(v[i])) : f2h_ref(v[i]);
        }
        uint2 w;
        w.x = hbits[0] | ((uint32_t)hbits[1] << 16); w.y = hbits[2] | ((uint32_t)hbits[3] << 16);
        *reinterpret_cast<uint2*>(reinterpret_cast<unsigned short*>(dst) + idx) = w;
    } else {
        stg_stream_f4(reinterpret_cast<float4*>(reinterpret_cast<float*>(dst) + idx), make_float4(v[0], v[1], v[2], v[3]));
    }
}

__device__ __forceinline__ float norm_int_px(int r, float m, float is) { return (div255_exact((float)r) - m) * is; }

// One thread = 4 luma columns x 2 rows.  Every warp-level access is lane-contiguous: 3 x LDG.32 (128 B per
// warp), 6 x STG.128 (512 contiguous bytes per warp per plane row).  [The first version gave each thread 8
// columns = two STG.128 per plane row; each store instruction then wrote only half of every 32-B sector and
// ncu showed 2x the write sectors at L2 (lts__t_sectors_srcunit_tex_op_write).]
template <bool F16, bool PTRS>
__global__ void __launch_bounds__(128) preprocess_nv12_identity_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                       const __grid_constant__ PreFrames fr, void* __restrict__ dst,
                                                                       uint32_t frame0, uint32_t groups_per_row, uint32_t items) {
    const uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    if (item >= items) return;
    const uint32_t rp = item / groups_per_row, g = item - rp * groups_per_row;
    const uint32_t w = (uint32_t)d.src_w, h = (uint32_t)d.src_h;
    const uint32_t f = blockIdx.y;
    const uint8_t* src = PTRS ? fr.ptr[f] : fr.base + (size_t)(frame0 + f) * fr.stride;
    const uint32_t x = g * 4u;
    const uint32_t y0w = __ldg(reinterpret_cast<const uint32_t*>(src + (size_t)(2u * rp) * w + x));
    const uint32_t y1w = __ldg(reinterpret_cast<const uint32_t*>(src + (size_t)(2u * rp + 1u) * w + x));
    const uint32_t uvw = __ldg(reinterpret_cast<const uint32_t*>(src + (size_t)w * h + (size_t)rp * w + x));
    ChromaTerms ct[2];
    ct[0] = chroma_terms((int)(uvw & 0xFFu), (int)((uvw >> 8) & 0xFFu));
    ct[1] = chroma_terms((int)((uvw >> 16) & 0xFFu), (int)(uvw >> 24));
    const size_t plane = (size_t)w * h;
    const size_t base = (size_t)(frame0 + f) * 3 * plane + (size_t)(2u * rp) * w + x;
    const float m0 = d.mean[0], m1 = d.mean[1], m2 = d.mean[2], i0 = d.inv_std[0], i1 = d.inv_std[1], i2 = d.inv_std[2];
#pragma unroll
    for (int row = 0; row < 2; ++row) {
        const uint32_t yw = row == 0 ? y0w : y1w;
        float r4[4], g4[4], b4[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int yv = (int)((yw >> (8 * i)) & 0xFFu);
            int r, gg, b;
            decode_rgb(yy_term(yv), ct[i >> 1], r, gg, b);
            r4[i] = norm_int_px(r, m0, i0);
            g4[i] = norm_int_px(gg, m1, i1);
            b4[i] = norm_int_px(b, m2, i2);
        }
        const size_t o = base + (size_t)row * w;
        nv12_store4<F16>(dst, o, r4);
        nv12_store4<F16>(dst, o + plane, g4);
        nv12_store4<F16>(dst, o + 2 * plane, b4);
    }
}

// ── NV12 general path (config 3b: 1080p NV12 → letterboxed 640x640, and every other NV12 geometry) ──────────
// ncu on the generic kernel for config 3b: issue-bound (format switch, integer div/mod for (ox, oy), byte-granular
// everything), DRAM mostly idle.  This kernel is NV12-only:
//   * one thread = 4 consecutive destination pixels of one row; the row comes from blockIdx.y (no div/mod);
//     pad rows and pad pixels store a host-precomputed normalised pad value; 3 lane-contiguous STG.128 per thread;
//   * taps are fetched only when their weight is non-zero (exact, see the header) — at integer scale ratios
//     (1080p → 640 letterbox is exactly 3:1) that is ONE decode per pixel;
//   * a pixel that was not interpolated is an integer 0..255, whose `px / 255.0f` is the 3-instruction exact
//     form (norm_int_px); interpolated pixels use the IEEE division.
struct Nv12Args {
    float pad_norm[3];  // ((pad_value / 255) - mean) * inv_std, evaluated on the host in f32
    uint32_t groups;    // ceil(dst_w / 4)
};

__device__ __forceinline__ void nv12_tap(const uint8_t* __restrict__ src, int x, int y, int w, int h, int rgb[3]) {
    const int yv = __ldg(src + (size_t)y * w + x);
    const uint32_t uv = __ldg(reinterpret_cast<const unsigned short*>(src + (size_t)w * h + (size_t)(y >> 1) * w + (x >> 1) * 2));
    const ChromaTerms t = chroma_terms((int)(uv & 0xFFu), (int)(uv >> 8));
    decode_rgb(yy_term(yv), t, rgb[0], rgb[1], rgb[2]);
}

static constexpr int NV12_ROWS = 8;  // destination rows per thread: the x-side of the sampler is computed once for all of them

template <bool F16, bool BILINEAR, bool PTRS>
__global__ void __launch_bounds__(128) preprocess_nv12_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                              const __grid_constant__ PreFrames fr, const __grid_constant__ Nv12Args na,
                                                              void* __restrict__ dst, uint32_t frame0) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= na.groups) return;
    const uint32_t f = blockIdx.z;
    const int ox0 = (int)g * 4;
    const int w = d.src_w, h = d.src_h;
    const uint8_t* src = PTRS ? fr.ptr[f] : fr.base + (size_t)(frame0 + f) * fr.stride;
    const size_t plane = (size_t)d.dst_w * d.dst_h;
    // x-side, once: plan_pixel + sample_* coordinate rules (preprocess.rs:437-448, :534-563)
    int xa[4], xb[4];
    float ax[4];
    bool xin[4];
    bool any_in = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float sx = __fdiv_rn((float)(ox0 + j) - d.pad_x, d.scale_x);
        xin[j] = !(sx < 0.0f || sx >= (float)w);
        any_in = any_in || xin[j];
        if (BILINEAR) {
            const int x0 = (int)floorf(sx);
            ax[j] = sx - (float)x0;
            xb[j] = min(x0 + 1, w - 1);
            xa[j] = max(x0, 0);
        } else {
            xa[j] = min(max((int)roundf(sx), 0), w - 1);
            xb[j] = xa[j]; ax[j] = 0.0f;
        }
    }
    const int oy_first = (int)blockIdx.y * NV12_ROWS;
#pragma unroll 1
    for (int r = 0; r < NV12_ROWS; ++r) {
        const int oy = oy_first + r;
        if (oy >= d.dst_h) break;
        const size_t obase = (size_t)(frame0 + f) * 3 * plane + (size_t)oy * d.dst_w + ox0;
        float o[3][4];
        const float sy = __fdiv_rn((float)oy - d.pad_y, d.scale_y);
        const bool row_in = !(sy < 0.0f || sy >= (float)h);
        if (!(row_in && any_in)) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { o[0][j] = na.pad_norm[0]; o[1][j] = na.pad_norm[1]; o[2][j] = na.pad_norm[2]; }
        } else {
            int y0, y1 = 0;
            float ay = 0.0f;
            if (BILINEAR) {
                y0 = (int)floorf(sy);
                ay = sy - (float)y0;
                y1 = min(y0 + 1, h - 1);
                y0 = max(y0, 0);
            } else {
                y0 = min(max((int)roundf(sy), 0), h - 1);
            }
            const bool need_y = BILINEAR && ay != 0.0f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (!xin[j]) { o[0][j] = na.pad_norm[0]; o[1][j] = na.pad_norm[1]; o[2][j] = na.pad_norm[2]; continue; }
                int t00[3];
                nv12_tap(src, xa[j], y0, w, h, t00);
                const bool need_x = BILINEAR && ax[j] != 0.0f;
                float px[3];
                if (!need_x && !need_y) {  // the sample IS the decoded tap (exact, see header)
                    px[0] = (float)t00[0]; px[1] = (float)t00[1]; px[2] = (float)t00[2];
                } else {
                    int t10[3] = {0, 0, 0}, t01[3] = {0, 0, 0}, t11[3] = {0, 0, 0};
                    if (need_x) nv12_tap(src, xb[j], y0, w, h, t10);
                    if (need_y) {
                        nv12_tap(src, xa[j], y1, w, h, t01);
                        if (need_x) nv12_tap(src, xb[j], y1, w, h, t11);
                    }
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float a = (float)t00[c];
                        const float top = need_x ? a + ((float)t10[c] - a) * ax[j] : a;
                        if (need_y) {
                            const float cc = (float)t01[c];
                            const float bot = need_x ? cc + ((float)t11[c] - cc) * ax[j] : cc;
                            px[c] = top + (bot - top) * ay;
                        } else {
                            px[c] = top;
                        }
                    }
                }
                o[0][j] = (div255_exact(px[0]) - d.mean[0]) * d.inv_std[0];
                o[1][j] = (div255_exact(px[1]) - d.mean[1]) * d.inv_std[1];
                o[2][j] = (div255_exact(px[2]) - d.mean[2]) * d.inv_std[2];
            }
        }
        nv12_store4<F16>(dst, obase, o[0]);
        nv12_store4<F16>(dst, obase + plane, o[1]);
        nv12_store4<F16>(dst, obase + 2 * plane, o[2]);
    }
}

static size_t src_bytes(const kb200_preprocess_desc& d) {
    const size_t chroma = d.fmt == KB200_FMT_NV12 ? (size_t)d.src_w * d.src_h / 2 : 0;
    return (size_t)d.src_pitch * d.src_h + chroma;
}

static int validate_desc(const kb200_preprocess_desc* dp) {
    if (!dp) return fail(KB200_ERR_INVALID_ARGUMENT, "null preprocess descriptor");
    const kb200_preprocess_desc& d = *dp;
    if (d.src_w <= 0 || d.src_h <= 0 || d.dst_w <= 0 || d.dst_h <= 0)
        return fail(KB200_ERR_INVALID_ARGUMENT, "image dimensions must be non-zero");
    if ((long long)d.dst_w * d.dst_h > 0x7FFFFFFFll) return fail(KB200_ERR_DIMS_TOO_LARGE, "dimensions exceed the 32-bit CUDA kernel index limit");  // :1336-1339
    if (d.fmt < 0 || d.fmt > 4) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown source format code %d", d.fmt);
    if (d.sampling != KB200_INTERP_NEAREST && d.sampling != KB200_INTERP_BILINEAR && d.sampling != KB200_INTERP_LANCZOS)
        return fail(KB200_ERR_UNSUPPORTED, "unsupported sampling mode %d (expected Nearest, Bilinear or Lanczos)", d.sampling);  // preprocess.rs:1044-1051
    if (d.fmt <= 1 && d.src_bpp != 3 && d.src_bpp != 4) return fail(KB200_ERR_UNSUPPORTED, "unsupported source channel count %d (expected 3 or 4)", d.src_bpp);
    // SourceFormat::dims_ok :188-195 ; pitch covers a row (PitchedSurface::validate :829-842)
    if (d.fmt == KB200_FMT_NV12 && ((d.src_w | d.src_h) & 1)) return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source for Nv12 at %dx%d (even dimensions required)", d.src_w, d.src_h);
    if (d.fmt == KB200_FMT_YUYV && (d.src_w & 1)) return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source for Yuyv at %dx%d (even width required)", d.src_w, d.src_h);
    const int bpp = d.fmt <= 1 ? d.src_bpp : (d.fmt == KB200_FMT_YUYV ? 2 : 1);
    if ((long long)d.src_pitch < (long long)d.src_w * bpp) return fail(KB200_ERR_INVALID_SOURCE, "invalid pitched surface (need pitch >= width*channels and len >= pitch*height)");
    if (d.fmt == KB200_FMT_NV12 && d.src_pitch != d.src_w) return fail(KB200_ERR_INVALID_SOURCE, "NV12 frames must be tightly packed (pitch == width)");
    if (!(d.scale_x > 0.0f) || !(d.scale_y > 0.0f)) return fail(KB200_ERR_INVALID_ARGUMENT, "scale must be positive");
    return KB200_OK;
}

template <bool F16>
static int launch_preprocess(cudaStream_t s, const kb200_preprocess_desc& d, const uint8_t* const* frames,
                             const uint8_t* base, size_t stride, uint32_t batch, void* dst) {
    const int pixels = d.dst_w * d.dst_h;
    const bool bil = d.sampling == KB200_INTERP_BILINEAR, lanczos = d.sampling == KB200_INTERP_LANCZOS;
    // identity fast path: NV12, scale 1, no pad, same size, 8-column vectors possible
    // (Lanczos always takes the generic kernel: its off-centre weights at integer coordinates are sinf(k*pi) != 0 exactly)
    bool identity = !lanczos && d.fmt == KB200_FMT_NV12 && d.scale_x == 1.0f && d.scale_y == 1.0f && d.pad_x == 0.0f && d.pad_y == 0.0f &&
                    d.dst_w == d.src_w && d.dst_h == d.src_h && (d.src_w % 4) == 0 && aligned16(dst);
    if (identity) {
        if (frames) { for (uint32_t k = 0; k < batch; ++k) identity = identity && ((reinterpret_cast<uintptr_t>(frames[k]) & 3u) == 0); }
        else identity = ((reinterpret_cast<uintptr_t>(base) & 3u) == 0) && (stride % 4 == 0);
    }
    const uint32_t id_groups = (uint32_t)d.src_w / 4u;
    const size_t id_items = (size_t)id_groups * ((size_t)d.src_h / 2);
    if (id_items > 0x7FFFFFFFull) identity = false;
    // NV12 general fast path: vector stores need dst_w % 4 == 0 and a 16-B (f32) / 8-B (f16) aligned destination
    const bool nv12_fast = !lanczos && d.fmt == KB200_FMT_NV12 && (d.dst_w % 4) == 0 && aligned16(dst) && d.dst_h <= 65535 * NV12_ROWS;
    Nv12Args nv{};
    nv.groups = (uint32_t)(d.dst_w + 3) / 4u;
    for (int c = 0; c < 3; ++c) nv.pad_norm[c] = (d.pad_value / 255.0f - d.mean[c]) * d.inv_std[c];  // BODY :610-612 on the host (f32, unfused)
    for (uint32_t f0 = 0; f0 < batch; f0 += 256) {
        const uint32_t nb = std::min<uint32_t>(256, batch - f0);
        PreFrames fr{};
        fr.base = base; fr.stride = stride;
        if (frames) for (uint32_t k = 0; k < nb; ++k) fr.ptr[k] = frames[f0 + k];
        if (identity) {
            dim3 grid(div_up(id_items, 128), nb);
            if (frames) preprocess_nv12_identity_kernel<F16, true><<<grid, 128, 0, s>>>(d, fr, dst, f0, id_groups, (uint32_t)id_items);
            else preprocess_nv12_identity_kernel<F16, false><<<grid, 128, 0, s>>>(d, fr, dst, f0, id_groups, (uint32_t)id_items);
            KB200_TRY(check_launch("preprocess_nv12_identity_kernel"));
            continue;
        }
        if (nv12_fast) {
            dim3 grid(div_up(nv.groups, 128), div_up((size_t)d.dst_h, NV12_ROWS), nb);
#define KB200_NV12_LAUNCH(BIL, PT) preprocess_nv12_kernel<F16, BIL, PT><<<grid, 128, 0, s>>>(d, fr, nv, dst, f0)
            if (bil) { if (frames) KB200_NV12_LAUNCH(true, true); else KB200_NV12_LAUNCH(true, false); }
            else     { if (frames) KB200_NV12_LAUNCH(false, true); else KB200_NV12_LAUNCH(false, false); }
#undef KB200_NV12_LAUNCH
            KB200_TRY(check_launch("preprocess_nv12_kernel"));
            continue;
        }
        dim3 grid(div_up(pixels, 256), nb);
        if (frames) {
            if (lanczos) preprocess_generic_kernel<F16, KB200_INTERP_LANCZOS, true><<<grid, 256, 0, s>>>(d, fr, dst, f0);
            else if (bil) preprocess_generic_kernel<F16, KB200_INTERP_BILINEAR, true><<<grid, 256, 0, s>>>(d, fr, dst, f0);
            else preprocess_generic_kernel<F16, KB200_INTERP_NEAREST, true><<<grid, 256, 0, s>>>(d, fr, dst, f0);
        } else {
            if (lanczos) preprocess_generic_kernel<F16, KB200_INTERP_LANCZOS, false><<<grid, 256, 0, s>>>(d, fr, dst, f0);
            else if (bil) preprocess_generic_kernel<F16, KB200_INTERP_BILINEAR, false><<<grid, 256, 0, s>>>(d, fr, dst, f0);
            else preprocess_generic_kernel<F16, KB200_INTERP_NEAREST, false><<<grid, 256, 0, s>>>(d, fr, dst, f0);
        }
        KB200_TRY(check_launch("preprocess_generic_kernel"));
    }
    return KB200_OK;
}

// used by the host-buffer pipeline (host_pipeline.cu): frames already staged at base + i*stride on the device
int preprocess_validate(const kb200_preprocess_desc* desc) { return validate_desc(desc); }
size_t preprocess_frame_bytes(const kb200_preprocess_desc& d) { return src_bytes(d); }
int preprocess_launch_strided(cudaStream_t s, const kb200_preprocess_desc& d, const uint8_t* base, size_t stride, uint32_t batch, void* dst, bool f16) {
    return f16 ? launch_preprocess<true>(s, d, nullptr, base, stride, batch, dst) : launch_preprocess<false>(s, d, nullptr, base, stride, batch, dst);
}

template <bool F16>
static int preprocess_entry(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames,
                            const size_t* frame_len, const uint8_t* base, size_t base_len, size_t stride,
                            uint32_t batch, void* dst, size_t dst_len) {
    KB200_TRY(validate_desc(desc));
    KB200_TRY(check_ptr("dst", dst));
    if (batch == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "batch must be non-zero");
    const size_t need = src_bytes(*desc);
    if (frames) {
        for (uint32_t i = 0; i < batch; ++i) {
            if (!frames[i]) return fail(KB200_ERR_INVALID_ARGUMENT, "null frame pointer at index %u", i);
            if (frame_len && frame_len[i] < need)  // InvalidRawSource{got,need}, preprocess.rs:1287-1300
                return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source at %dx%d (got %zu bytes, need %zu)", desc->src_w, desc->src_h, frame_len[i], need);
        }
    } else {
        KB200_TRY(check_ptr("base", base));
        if (stride < need && batch > 1) return fail(KB200_ERR_INVALID_SOURCE, "frame stride %zu smaller than a frame (%zu bytes)", stride, need);
        if (base_len < (size_t)(batch - 1) * stride + need)
            return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source at %dx%d (got %zu bytes, need %zu)", desc->src_w, desc->src_h, base_len, (size_t)(batch - 1) * stride + need);
    }
    // BatchMismatch / BadOutputShape: dst must hold [batch,3,H,W]
    KB200_TRY(check_slice("dst", dst_len, (size_t)batch * 3 * desc->dst_w * desc->dst_h));
    return launch_preprocess<F16>(as_stream(stream), *desc, frames, base, stride, batch, dst);
}

__global__ void selftest_div255_kernel(unsigned long long* mismatches) {
    const float c = 0.00392156885936856269836f;
    const uint32_t end = 0x43800000u;  // bits of 256.0f
    unsigned long long bad = 0;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t bits = blockIdx.x * blockDim.x + threadIdx.x; bits < end; bits += stride) {
        const float p = __uint_as_float(bits);
        const float q = p * c;
        const float e = fmaf(-q, 255.0f, p);
        const float q2 = fmaf(e, c, q);
        if (__float_as_uint(q2) != __float_as_uint(__fdiv_rn(p, 255.0f))) ++bad;
        if (bits + stride < bits) break;
    }
    if (bad) atomicAdd(mismatches, bad);
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_selftest_div255(kb200_stream_t stream, uint64_t* mismatches_dev) {
    KB200_TRY(check_ptr("mismatches_dev", mismatches_dev));
    cudaStream_t s = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(mismatches_dev, 0, sizeof(uint64_t), s);
    if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaMemsetAsync failed: %s", cudaGetErrorString(e));
    selftest_div255_kernel<<<device_info().sm_count * 8, 256, 0, s>>>(reinterpret_cast<unsigned long long*>(mismatches_dev));
    return check_launch("selftest_div255_kernel");
}

KB200_API size_t kb200_preprocess_src_bytes(const kb200_preprocess_desc* desc) { return desc ? src_bytes(*desc) : 0; }

KB200_API int kb200_preprocess_f32(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames,
                                   const size_t* frame_len, uint32_t batch, float* dst, size_t dst_len) {
    if (!frames) return fail(KB200_ERR_INVALID_ARGUMENT, "null pointer for 'frames'");
    return preprocess_entry<false>(stream, desc, frames, frame_len, nullptr, 0, 0, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_f16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames,
                                   const size_t* frame_len, uint32_t batch, uint16_t* dst, size_t dst_len) {
    if (!frames) return fail(KB200_ERR_INVALID_ARGUMENT, "null pointer for 'frames'");
    return preprocess_entry<true>(stream, desc, frames, frame_len, nullptr, 0, 0, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_strided_f32(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* base,
                                           size_t base_len, size_t frame_stride, uint32_t batch, float* dst, size_t dst_len) {
    return preprocess_entry<false>(stream, desc, nullptr, nullptr, base, base_len, frame_stride, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_strided_f16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* base,
                                           size_t base_len, size_t frame_stride, uint32_t batch, uint16_t* dst, size_t dst_len) {
    return preprocess_entry<true>(stream, desc, nullptr, nullptr, base, base_len, frame_stride, batch, dst, dst_len);
}

}  // extern "C"
