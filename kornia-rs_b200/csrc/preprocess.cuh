// preprocess.cuh — what the camera preprocess's sources share: preprocess.cu (one affine per frame, the batch entries)
// and the region entries (preprocess_roi.cu, preprocess_warp.cu, preprocess_remap.cu): the source-format facts, the taps
// (fetch_px), the Lanczos weight, the normalising divisions, the stores, the two sampler bodies over a frame's or a
// region's geometry, the fast resampler's arguments and launch rule, the host rules of the descriptor and of a region
// call, and the kernel-selection and output-format switches.  The arithmetic is documented in preprocess.cu's header.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "bayer.cuh"
#include "kb200_common.cuh"
#include "yuv.cuh"

namespace kb200 {

// The frames of one batch launch, by value in the kernel parameter block.  A strided call's frames are written into the
// table by the host (base + i * stride), so every batch kernel reads its frame from ptr[], except the packed-Bayer
// generic kernel of a strided call, which reads base and stride (see launch_preprocess).
struct PreFrames {
    const uint8_t* base;
    size_t stride;
    const uint8_t* ptr[256];
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

// The facts of one source format code (kb200_src_fmt without the matrix bits), from SRC_FORMATS below.  Every host
// function reads them from here; the generic kernel takes its format's as an argument.
enum SrcFamily { SRC_NONE, SRC_RGB, SRC_GRAY, SRC_YUV420, SRC_YUV422, SRC_BAYER, SRC_YUV444 };
struct SrcFormat {
    int code = -1;
    const char* name = nullptr;   // the SourceFormat name in messages; nullptr: the code is not a format
    SrcFamily family = SRC_NONE;
    int layout = 0;    // SRC_RGB: 0 RGB, 1 BGR order; SRC_YUV420: kb200_yuv420_layout (P01x NV12's, I01x I420's); SRC_YUV422: kb200_yuv422_layout;
                       // SRC_YUV444: kb200_yuv444_u16_layout (I41x's code position; 0 for I444)
    int pattern = 0;   // SRC_BAYER: kb200_bayer_pattern
    int bits = 8;      // bits per sample
    bool words = false;    // one little-endian 16-bit word per sample
    bool packed = false;   // MIPI CSI-2 packed samples (bits / 8 bytes each)
    const char* identity_kernel = nullptr;   // kb200_last_kernel() names of the format's fast kernels, nullptr: none
    const char* fast_kernel = nullptr;
    __host__ __device__ float white() const { return (float)((1u << bits) - 1u); }   // the white level W = 2^bits - 1
};

// p / W of a 16-bit YUV tap, bit for bit the IEEE quotient __fdiv_rn(p, W) (W = 1023 or 4095), but the division never sees
// a zero dividend: 0 / W is p itself (+0 or -0, since W > 0), so a zero p is returned as it is and 1 is divided in its
// place.  A zero operand fails the fast-path check (FCHK) of __fdiv_rn and enters its slow-path subroutine, and decoded
// video is full of codes clamped to 0 (blacks, out-of-gamut chroma), so without this most warps took the subroutine on
// some lane.
__device__ __forceinline__ float div_white(float p, float w) {
    const bool zero = p == 0.0f;
    const float q = __fdiv_rn(zero ? 1.0f : p, w);
    return zero ? p : q;
}

// The taps an instantiation of the generic kernel reads: interleaved RGB / BGR or gray bytes, 4:2:2, the 16-bit words of
// P01x / I01x, a Bayer mosaic of bytes, 16-bit words or packed samples, 8-bit 4:2:0 in one layout (TAP_YUV420 +
// kb200_yuv420_layout), 8-bit 4:4:4 (TAP_YUV444, the same tap in the YUV444 layout) or the 16-bit words of I41x
// (TAP_YUV444_16).  Within a kind the format's layout is a uniform branch.  The 4:2:0 layouts get an instantiation
// each: with the four taps in one kernel, its Lanczos loop no longer unrolls and spills; for the same reason 4:4:4 is not
// a branch of TAP_YUV16.  TapCoeffs: the coefficient argument, the Q16 set with its code extraction for the 16-bit words
// (as in the fast kernels), the Q20 set otherwise.
static constexpr int TAP_RGB = 0, TAP_YUV422 = 1, TAP_YUV16 = 2, TAP_BAYER = 3, TAP_BAYER16 = 4, TAP_BAYER_PACKED = 5, TAP_YUV420 = 6;
static constexpr int TAP_YUV444 = TAP_YUV420 + YUV444, TAP_YUV444_16 = TAP_YUV444 + 1;
template <int TAP> constexpr bool tap_words = TAP == TAP_YUV16 || TAP == TAP_YUV444_16;   // YUV taps of 16-bit words
template <int TAP> using TapCoeffs = std::conditional_t<tap_words<TAP>, Yuv16Coeffs, YuvCoeffs>;

template <int TAP>
__device__ __forceinline__ void fetch_px(const uint8_t* __restrict__ src, int x, int y, const kb200_preprocess_desc& d, const SrcFormat& f,
                                         const TapCoeffs<TAP>& yc, float px[3]) {  // :510-530
    if constexpr (TAP == TAP_RGB) {
        if (f.family == SRC_GRAY) {
            const float v = (float)src[(long long)y * d.src_pitch + x];
            px[0] = v; px[1] = v; px[2] = v;
            return;
        }
        const uint8_t* p = src + (long long)y * d.src_pitch + x * d.src_bpp;
        if (f.layout == 0) { px[0] = (float)p[0]; px[1] = (float)p[1]; px[2] = (float)p[2]; }
        else { px[0] = (float)p[2]; px[1] = (float)p[1]; px[2] = (float)p[0]; }
        return;
    }
    int rgb[3];
    if constexpr (TAP == TAP_BAYER || TAP == TAP_BAYER16) {   // src_pitch is in bytes (even for 16-bit samples)
        using T = std::conditional_t<TAP == TAP_BAYER16, uint16_t, uint8_t>;
        bayer_px(reinterpret_cast<const T*>(src), (size_t)d.src_pitch / sizeof(T), d.src_w, d.src_h, x, y, f.pattern, rgb);
    } else if constexpr (TAP == TAP_BAYER_PACKED) {
        bayer_px_packed(src, (size_t)d.src_pitch, d.src_w, d.src_h, x, y, f.pattern, f.bits, rgb);
    } else if constexpr (TAP == TAP_YUV16) {
        if (f.layout == YUV420_I420) yuv_tap<YUV420_I420>(src, x, y, d.src_w, d.src_h, yc, rgb);
        else yuv_tap<YUV420_NV12>(src, x, y, d.src_w, d.src_h, yc, rgb);
    } else if constexpr (TAP == TAP_YUV444_16) {
        yuv_tap<YUV444>(src, x, y, d.src_w, d.src_h, yc, rgb);
    } else if constexpr (TAP >= TAP_YUV420) {
        yuv_tap<TAP - TAP_YUV420, false>(src, x, y, d.src_w, d.src_h, yc, rgb);
    } else {
        switch (f.layout) {
            case YUV422_YUYV: yuv422_tap<YUV422_YUYV>(src, x, y, d.src_pitch, yc, rgb); break;
            case YUV422_UYVY: yuv422_tap<YUV422_UYVY>(src, x, y, d.src_pitch, yc, rgb); break;
            default: yuv422_tap<YUV422_YVYU>(src, x, y, d.src_pitch, yc, rgb); break;
        }
    }
    px[0] = (float)rgb[0]; px[1] = (float)rgb[1]; px[2] = (float)rgb[2];
}

// preprocess.rs:481-488 (kernel source): 1-D Lanczos-3 weight — the CUDA math library's sinf, like the reference kernel
__device__ __forceinline__ float pre_lanczos_w(float dd) {
    const float ad = fabsf(dd);
    if (ad < 1e-6f) return 1.0f;
    if (ad >= 3.0f) return 0.0f;
    const float pd = 3.14159265358979f * dd;
    return __fdiv_rn(3.0f * sinf(pd) * sinf(__fdiv_rn(pd, 3.0f)), pd * pd);
}

// OUT: the kb200_out_format of dst.  A bfloat16 value is the f32 one rounded to nearest even (__floats2bfloat162_rn, two
// values per conversion), stored like binary16 as one 8-byte word.
template <int OUT>
__device__ __forceinline__ void nv12_store4(void* __restrict__ dst, size_t idx, const float v[4]) {
    if constexpr (OUT == KB200_OUT_BF16) {
        const __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
        uint2 w;
        memcpy(&w.x, &lo, 4); memcpy(&w.y, &hi, 4);
        *reinterpret_cast<uint2*>(reinterpret_cast<unsigned short*>(dst) + idx) = w;
    } else if constexpr (OUT == KB200_OUT_F16) {
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

struct Nv12Args {
    float pad_norm[3];  // ((pad_value / 255) - mean) * inv_std, evaluated on the host in f32
    uint32_t groups;    // ceil(dst_w / 4)
};

static constexpr int NV12_ROWS = 8;  // destination rows per thread: the x-side of the sampler is computed once for all of them

// ── the sampler bodies ──────────────────────────────────────────────────────────────────────────────────────────────────
// generic_pixel and yuv_resample sample a source rectangle through a geometry G, which gives the source coordinate of an
// output column / row (sx, sy: IEEE division, plan_pixel :437-448), the rectangle's extent (w, h: the inside test and the
// tap clamps) and its origin in the frame (x0, y0: added to every tap, so that taps decode at frame coordinates), and, for
// yuv_resample's row loop, all three of a row at once (row).  FrameGeom is a whole frame under the descriptor's affine;
// RoiGeom (preprocess_roi.cu) is one region of a frame under its own.

// The row side of yuv_resample: the source row of an output row, the extent it is tested and clamped against, the origin.
struct GeomRow {
    float sy;
    int h, y0;
};

struct FrameGeom {
    const kb200_preprocess_desc& d;
    int rows;   // d.src_h, read once: see row()
    __device__ __forceinline__ explicit FrameGeom(const kb200_preprocess_desc& desc) : d(desc), rows(desc.src_h) {}
    __device__ __forceinline__ float sx(int ox) const { return __fdiv_rn((float)ox - d.pad_x, d.scale_x); }
    __device__ __forceinline__ float sy(int oy) const { return __fdiv_rn((float)oy - d.pad_y, d.scale_y); }
    __device__ __forceinline__ int w() const { return d.src_w; }
    __device__ __forceinline__ int h() const { return d.src_h; }
    __device__ __forceinline__ int x0() const { return 0; }
    __device__ __forceinline__ int y0() const { return 0; }
    // The height comes from the copy taken at construction, so the row loop holds it as one value.  Read through d after
    // each row's stores (whose inline asm clobbers memory), it is reloaded in the body's own optimisation, and every
    // preprocess_yuv_kernel instantiation compiled to a different predicate order and register assignment.
    __device__ __forceinline__ GeomRow row(int oy) const { return {sy(oy), rows, 0}; }
};

// One output pixel's sample point as a geometry for generic_pixel, which then samples and normalises it exactly as it does
// a pixel of a whole frame: the caller's frame coordinate, or (-1, -1) when the caller found it outside, so that
// generic_pixel's inside test (0 <= s < extent) agrees with the caller's; the extent is the frame's and the origin 0.
// generic_pixel's ox / oy arguments are not read.  The warp and remap region entries sample through it.
struct WarpPoint {
    float x, y;
    int fw, fh;
    __device__ __forceinline__ float sx(int) const { return x; }
    __device__ __forceinline__ float sy(int) const { return y; }
    __device__ __forceinline__ int w() const { return fw; }
    __device__ __forceinline__ int h() const { return fh; }
    __device__ __forceinline__ int x0() const { return 0; }
    __device__ __forceinline__ int y0() const { return 0; }
};

// Output pixel (ox, oy) of the rectangle g of the frame at src, sampled with SAMP (kb200_interp — 0 nearest, 1 bilinear,
// 3 Lanczos-3: 6x6 taps, clamp-to-edge, weights renormalised by their sum) and normalised into o.
template <int SAMP, int TAP, class G>
__device__ __forceinline__ void generic_pixel(const uint8_t* __restrict__ src, int ox, int oy, const kb200_preprocess_desc& d, const SrcFormat& sf,
                                              const TapCoeffs<TAP>& yc, const G& g, float o[3]) {
    const float sx = g.sx(ox);
    const float sy = g.sy(oy);
    const bool inside = !(sx < 0.0f || sy < 0.0f || sx >= (float)g.w() || sy >= (float)g.h());
    float px[3];
    if (inside) {
        if (SAMP == KB200_INTERP_LANCZOS) {   // preprocess.rs:565-590 sample_lanczos: acc += w * t (unfused), one division per channel
            const int x0 = (int)floorf(sx), y0 = (int)floorf(sy);
            float acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f, wsum = 0.0f;
            for (int j = -2; j <= 3; ++j) {
                const int yj = y0 + j;
                const float wy = pre_lanczos_w(sy - (float)yj);
                const int ycl = min(max(yj, 0), g.h() - 1);
                for (int ii = -2; ii <= 3; ++ii) {
                    const int xi = x0 + ii;
                    const float w = wy * pre_lanczos_w(sx - (float)xi);
                    const int xc = min(max(xi, 0), g.w() - 1);
                    float t[3];
                    fetch_px<TAP>(src, g.x0() + xc, g.y0() + ycl, d, sf, yc, t);
                    acc0 += w * t[0]; acc1 += w * t[1]; acc2 += w * t[2];
                    wsum += w;
                }
            }
            px[0] = __fdiv_rn(acc0, wsum); px[1] = __fdiv_rn(acc1, wsum); px[2] = __fdiv_rn(acc2, wsum);
        } else if (SAMP == KB200_INTERP_BILINEAR) {
            int x0 = (int)floorf(sx), y0 = (int)floorf(sy);
            const float ax = sx - (float)x0, ay = sy - (float)y0;
            const int x1 = g.x0() + min(x0 + 1, g.w() - 1), y1 = g.y0() + min(y0 + 1, g.h() - 1);
            x0 = g.x0() + max(x0, 0); y0 = g.y0() + max(y0, 0);
            float t00[3], t10[3], t01[3], t11[3];
            fetch_px<TAP>(src, x0, y0, d, sf, yc, t00);
            const bool need_x = ax != 0.0f, need_y = ay != 0.0f;
            if (need_x) fetch_px<TAP>(src, x1, y0, d, sf, yc, t10);
            if (need_y) {
                fetch_px<TAP>(src, x0, y1, d, sf, yc, t01);
                if (need_x) fetch_px<TAP>(src, x1, y1, d, sf, yc, t11);
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
            const int xn = g.x0() + min(max((int)roundf(sx), 0), g.w() - 1);
            const int yn = g.y0() + min(max((int)roundf(sy), 0), g.h() - 1);
            fetch_px<TAP>(src, xn, yn, d, sf, yc, px);
        }
    } else {
        px[0] = d.pad_value; px[1] = d.pad_value; px[2] = d.pad_value;
    }
    float q0, q1, q2;
    if (tap_words<TAP> && inside) {   // px / W, the IEEE quotient (div_white: no zero dividend reaches the division)
        const float wl = sf.white();
        q0 = div_white(px[0], wl); q1 = div_white(px[1], wl); q2 = div_white(px[2], wl);
    } else if ((TAP == TAP_BAYER16 || TAP == TAP_BAYER_PACKED) && inside) {   // px / W: taps up to 65535 and Lanczos overshoot, so the IEEE division
        const float wl = sf.white();
        q0 = __fdiv_rn(px[0], wl); q1 = __fdiv_rn(px[1], wl); q2 = __fdiv_rn(px[2], wl);
    } else if (inside && SAMP != KB200_INTERP_LANCZOS) { q0 = div255_exact(px[0]); q1 = div255_exact(px[1]); q2 = div255_exact(px[2]); }
    else if (inside) { q0 = __fdiv_rn(px[0], 255.0f); q1 = __fdiv_rn(px[1], 255.0f); q2 = __fdiv_rn(px[2], 255.0f); }  // Lanczos overshoots [0, 255]
    else { q0 = __fdiv_rn(px[0], 255.0f); q1 = q0; q2 = q0; }  // pad_value is caller-supplied: plain IEEE division
    o[0] = (q0 - d.mean[0]) * d.inv_std[0];
    o[1] = (q1 - d.mean[1]) * d.inv_std[1];
    o[2] = (q2 - d.mean[2]) * d.inv_std[2];
}

// The three planes of one pixel: element `out` of plane 0 of a CHW image of `pixels` pixels per plane.
template <int OUT>
__device__ __forceinline__ void generic_store(void* __restrict__ dst, size_t out, int pixels, const float o[3]) {
    if constexpr (OUT == KB200_OUT_F16) {
        unsigned short* p = reinterpret_cast<unsigned short*>(dst);
        p[out] = f2h_ref(o[0]); p[out + pixels] = f2h_ref(o[1]); p[out + 2 * (size_t)pixels] = f2h_ref(o[2]);
    } else if constexpr (OUT == KB200_OUT_BF16) {
        __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(dst);
        p[out] = __float2bfloat16_rn(o[0]); p[out + pixels] = __float2bfloat16_rn(o[1]); p[out + 2 * (size_t)pixels] = __float2bfloat16_rn(o[2]);
    } else {
        float* p = reinterpret_cast<float*>(dst);
        p[out] = o[0]; p[out + pixels] = o[1]; p[out + 2 * (size_t)pixels] = o[2];
    }
}

// The fast resampler: the 4 output columns ox0 .. ox0 + 3 of the NV12_ROWS rows from blockIdx.y * NV12_ROWS of output
// image `img`, sampled from the rectangle geo of the frame at src.  The frame's w x h (the descriptor's) address its planes
// in yuv_tap; geo's extent sets the inside test and the clamps.  L: a 4:2:0 layout or YUV444 (yuv_tap); T: the sample type
// (YuvSample).  A pixel of 16-bit words is normalised as (px / W - mean) * inv_std with the IEEE division, interpolated or not.
template <int OUT, bool BILINEAR, int L, typename T, class G>
__device__ __forceinline__ void yuv_resample(const G& geo, const uint8_t* __restrict__ src, const kb200_preprocess_desc& d, const Nv12Args& na,
                                             void* __restrict__ dst, uint32_t img, int ox0, const typename YuvSample<T>::Coeffs& yc) {
    const int w = d.src_w, h = d.src_h;
    const int rw = geo.w();
    const size_t plane = (size_t)d.dst_w * d.dst_h;
    // x-side, once: plan_pixel + sample_* coordinate rules (preprocess.rs:437-448, :534-563)
    int xa[4], xb[4];
    float ax[4];
    bool xin[4];
    bool any_in = false;
    // 16-bit samples and 4:4:4: the four divisions first, so that only their quotients are live across the slow-path calls
    // they may make (the interleaved form spilled in the f16 bilinear instantiations); the 8-bit 4:2:0 kernels keep the
    // interleaved form
    constexpr bool SX_FIRST = sizeof(T) == 2 || L == YUV444;
    [[maybe_unused]] float sx16[4];
    if constexpr (SX_FIRST) {
#pragma unroll
        for (int j = 0; j < 4; ++j) sx16[j] = geo.sx(ox0 + j);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float sx = SX_FIRST ? sx16[j] : geo.sx(ox0 + j);
        xin[j] = !(sx < 0.0f || sx >= (float)rw);
        any_in = any_in || xin[j];
        if (BILINEAR) {
            const int x0 = (int)floorf(sx);
            ax[j] = sx - (float)x0;
            xb[j] = geo.x0() + min(x0 + 1, rw - 1);
            xa[j] = geo.x0() + max(x0, 0);
        } else {
            xa[j] = geo.x0() + min(max((int)roundf(sx), 0), rw - 1);
            xb[j] = xa[j]; ax[j] = 0.0f;
        }
    }
    const int oy_first = (int)blockIdx.y * NV12_ROWS;
#pragma unroll 1
    for (int r = 0; r < NV12_ROWS; ++r) {
        const int oy = oy_first + r;
        if (oy >= d.dst_h) break;
        const size_t obase = (size_t)img * 3 * plane + (size_t)oy * d.dst_w + ox0;
        float o[3][4];
        const GeomRow gr = geo.row(oy);
        const float sy = gr.sy;
        const int rh = gr.h, ry = gr.y0;
        const bool row_in = !(sy < 0.0f || sy >= (float)rh);
        if (!(row_in && any_in)) {
#pragma unroll
            for (int j = 0; j < 4; ++j) { o[0][j] = na.pad_norm[0]; o[1][j] = na.pad_norm[1]; o[2][j] = na.pad_norm[2]; }
        } else {
            int y0, y1 = 0;
            float ay = 0.0f;
            if (BILINEAR) {
                y0 = (int)floorf(sy);
                ay = sy - (float)y0;
                y1 = ry + min(y0 + 1, rh - 1);
                y0 = ry + max(y0, 0);
            } else {
                y0 = ry + min(max((int)roundf(sy), 0), rh - 1);
            }
            const bool need_y = BILINEAR && ay != 0.0f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (!xin[j]) { o[0][j] = na.pad_norm[0]; o[1][j] = na.pad_norm[1]; o[2][j] = na.pad_norm[2]; continue; }
                int t00[3];
                yuv_tap<L>(src, xa[j], y0, w, h, yc, t00);
                const bool need_x = BILINEAR && ax[j] != 0.0f;
                float px[3];
                if (!need_x && !need_y) {  // the sample IS the decoded tap (exact, see preprocess.cu's header)
                    px[0] = (float)t00[0]; px[1] = (float)t00[1]; px[2] = (float)t00[2];
                } else {
                    int t10[3] = {0, 0, 0}, t01[3] = {0, 0, 0}, t11[3] = {0, 0, 0};
                    if (need_x) yuv_tap<L>(src, xb[j], y0, w, h, yc, t10);
                    if (need_y) {
                        yuv_tap<L>(src, xa[j], y1, w, h, yc, t01);
                        if (need_x) yuv_tap<L>(src, xb[j], y1, w, h, yc, t11);
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
                if constexpr (sizeof(T) == 2) {
                    const float wl = (float)yc.white;
                    o[0][j] = (div_white(px[0], wl) - d.mean[0]) * d.inv_std[0];
                    o[1][j] = (div_white(px[1], wl) - d.mean[1]) * d.inv_std[1];
                    o[2][j] = (div_white(px[2], wl) - d.mean[2]) * d.inv_std[2];
                } else {
                    o[0][j] = (div255_exact(px[0]) - d.mean[0]) * d.inv_std[0];
                    o[1][j] = (div255_exact(px[1]) - d.mean[1]) * d.inv_std[1];
                    o[2][j] = (div255_exact(px[2]) - d.mean[2]) * d.inv_std[2];
                }
            }
        }
        nv12_store4<OUT>(dst, obase, o[0]);
        nv12_store4<OUT>(dst, obase + plane, o[1]);
        nv12_store4<OUT>(dst, obase + 2 * plane, o[2]);
    }
}

// ── host side ───────────────────────────────────────────────────────────────────────────────────────────────────────────
// The rules of the descriptor, in preprocess.cu.
SrcFormat src_format(int fmt);   // the facts of a plain format code; name == nullptr: not a format
kb200_preprocess_desc plain_desc(const kb200_preprocess_desc& d);   // the format code without its YUV matrix bits
int yuv_matrix(const kb200_preprocess_desc& raw);
size_t src_bytes(const kb200_preprocess_desc& d);    // d: a plain descriptor
int validate_desc(const kb200_preprocess_desc* dp);  // the raw descriptor an entry was given
// The checks of a table of n frame pointers (frame_len: their lengths, or nullptr): none null, every frame of 16-bit samples
// 2-byte aligned, every length >= src_bytes(d).  d: a plain descriptor.
int check_frame_table(const kb200_preprocess_desc& d, const uint8_t* const* frames, const size_t* frame_len, uint32_t n);
// The checks a region entry (kb200_preprocess_rois, _warps, _remap) starts with, in this order: a descriptor is given; its
// rules hold (validate_desc) with its scale and pad taken as the identity, since each region brings its own geometry; the
// resize mode of the entry that takes one (mode; nullptr for the others) is known; a point-sampled entry refuses Lanczos
// (point: the noun its message names the regions by, "warped regions"; nullptr: Lanczos is sampled); the output format
// is known.  raw: that descriptor; plain: its plain_desc.
int check_region_call(const kb200_preprocess_desc* desc, const int* mode, const char* point, int out_format, kb200_preprocess_desc* raw,
                      kb200_preprocess_desc* plain);
// The first rule of every region entry's per-region loop: region i's frame index names one of the n_frames frames.
int check_region_frame(uint32_t i, int32_t frame, uint32_t n_frames);

// Every frame of a call starts a-byte aligned: the n frames of the pointer table `frames`, or, when it is nullptr, the
// frames at base + k * stride.
inline bool frames_aligned(const uint8_t* const* frames, const uint8_t* base, size_t stride, uint32_t n, uint32_t a) {
    if (!frames) return ((reinterpret_cast<uintptr_t>(base) & (a - 1)) == 0) && (stride % a == 0);
    for (uint32_t k = 0; k < n; ++k)
        if (reinterpret_cast<uintptr_t>(frames[k]) & (a - 1)) return false;
    return true;
}

// Whether the fast resampler (yuv_resample) takes a call of format f (plain descriptor d) into dst: a format with fast
// kernels, not Lanczos, and vector stores, which need dst_w % 4 == 0 and a 16-B (f32) / 8-B (f16, bf16) aligned
// destination.  The NV12 / NV21 tap reads a chroma pair as one 16-bit word (yuv_tap), so those frames must start 2-B
// aligned (frames_even); frames at odd addresses take the generic kernel, which reads the pair's two bytes.
inline bool yuv_resampler_ok(const SrcFormat& f, const kb200_preprocess_desc& d, const void* dst, bool frames_even) {
    const bool pair_loads = f.family == SRC_YUV420 && !f.words && (f.layout == YUV420_NV12 || f.layout == YUV420_NV21);
    return d.sampling != KB200_INTERP_LANCZOS && f.fast_kernel && (d.dst_w % 4) == 0 && aligned16(dst) && d.dst_h <= 65535 * NV12_ROWS &&
           (!pair_loads || frames_even);
}

// Whether the warp and remap region kernels' 4-column stores (nv12_store4) can write dst in output format out: whole
// 4-column groups and a destination 16-B (f32) / 8-B (f16, bf16) aligned.
inline bool vector_dst_ok(const kb200_preprocess_desc& d, const void* dst, int out) {
    const uintptr_t a = out == KB200_OUT_F32 ? 15u : 7u;
    return d.dst_w % 4 == 0 && (reinterpret_cast<uintptr_t>(dst) & a) == 0;
}

// The Q16 coefficient set of a format of 16-bit YUV words (P01x, I01x, I41x) decoded with `matrix`.
inline Yuv16Coeffs yuv16_coeffs_of(const SrcFormat& f, int matrix) {
    const bool msb = f.family == SRC_YUV444 ? f.layout == KB200_YUV444_I41X_MSB : f.layout == YUV420_NV12;   // P01x, I41xMsb
    return yuv16_coeffs(matrix, f.bits, msb);
}

// The fast resampler's arguments: the normalised pad value (BODY :610-612 on the host, f32, unfused) and the 4-column groups of a row.
inline Nv12Args nv12_args(const kb200_preprocess_desc& d) {
    Nv12Args nv{};
    nv.groups = (uint32_t)(d.dst_w + 3) / 4u;
    for (int c = 0; c < 3; ++c) nv.pad_norm[c] = (d.pad_value / 255.0f - d.mean[c]) * d.inv_std[c];
    return nv;
}

template <int V> using IntC = std::integral_constant<int, V>;

// Calls launch(IntC<TAP>{}, coeffs) with the generic kernels' tap kind for format f and that tap's coefficient set.
template <class Launch>
void with_tap(const SrcFormat& f, const YuvCoeffs& yc, const Yuv16Coeffs& yc16, Launch&& launch) {
    if (f.family == SRC_BAYER) {
        if (f.packed) launch(IntC<TAP_BAYER_PACKED>{}, yc);
        else if (f.words) launch(IntC<TAP_BAYER16>{}, yc);
        else launch(IntC<TAP_BAYER>{}, yc);
    } else if (f.family == SRC_YUV444) {
        if (f.words) launch(IntC<TAP_YUV444_16>{}, yc16);
        else launch(IntC<TAP_YUV444>{}, yc);
    } else if (f.words) {
        launch(IntC<TAP_YUV16>{}, yc16);
    } else if (f.family == SRC_YUV420) {
        switch (f.layout) {
            case YUV420_NV12: launch(IntC<TAP_YUV420 + YUV420_NV12>{}, yc); break;
            case YUV420_NV21: launch(IntC<TAP_YUV420 + YUV420_NV21>{}, yc); break;
            case YUV420_I420: launch(IntC<TAP_YUV420 + YUV420_I420>{}, yc); break;
            default: launch(IntC<TAP_YUV420 + YUV420_YV12>{}, yc); break;
        }
    } else if (f.family == SRC_YUV422) {
        launch(IntC<TAP_YUV422>{}, yc);
    } else {
        launch(IntC<TAP_RGB>{}, yc);
    }
}

// Returns launch(IntC<OUT>{}) for the kb200_out_format out, one the caller has checked.
template <class Launch>
int with_out_format(int out, Launch&& launch) {
    if (out == KB200_OUT_F16) return launch(IntC<KB200_OUT_F16>{});
    if (out == KB200_OUT_BF16) return launch(IntC<KB200_OUT_BF16>{});
    return launch(IntC<KB200_OUT_F32>{});
}

// Calls launch(IntC<L>{}, T{}, coeffs) with the fast kernels' layout L (4:2:0, or YUV444) and sample type T for a format
// that has fast kernels (SrcFormat::fast_kernel), and their coefficient set.
template <class Launch>
void with_yuv_layout(const SrcFormat& f, const YuvCoeffs& yc, const Yuv16Coeffs& yc16, Launch&& launch) {
    if (f.family == SRC_YUV444) {
        if (f.words) launch(IntC<YUV444>{}, uint16_t{}, yc16);
        else launch(IntC<YUV444>{}, uint8_t{}, yc);
    } else if (f.words) {
        if (f.layout == YUV420_I420) launch(IntC<YUV420_I420>{}, uint16_t{}, yc16);
        else launch(IntC<YUV420_NV12>{}, uint16_t{}, yc16);
    } else {
        switch (f.layout) {
            case YUV420_NV12: launch(IntC<YUV420_NV12>{}, uint8_t{}, yc); break;
            case YUV420_NV21: launch(IntC<YUV420_NV21>{}, uint8_t{}, yc); break;
            case YUV420_I420: launch(IntC<YUV420_I420>{}, uint8_t{}, yc); break;
            default: launch(IntC<YUV420_YV12>{}, uint8_t{}, yc); break;
        }
    }
}

}  // namespace kb200
