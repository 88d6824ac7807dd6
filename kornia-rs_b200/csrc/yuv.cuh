// yuv.cuh — one decoded pixel of a YUV frame, per layout: the YUV taps of the camera preprocess (preprocess.cu:
// preprocess_yuv_kernel and the YUV instantiations of the generic kernel), kept out of preprocess.cu as bayer.cuh keeps
// the Bayer taps.  The coefficient sets, the decode arithmetic and the layout constants are in kb200_common.cuh.
#pragma once

#include "kb200_common.cuh"

namespace kb200 {

// The sample type T of a 4:2:0 or 4:4:4 frame: bytes (NV12, NV21, I420, YV12, I444), or 16-bit words holding n-bit codes
// — P01x in the NV12 layout, I01x in the I420 layout, I41x in the 4:4:4 one.  Coeffs is the kernels' coefficient argument: the Q20 set for bytes, the Q16
// set with its code extraction (Yuv16Coeffs) for words.
template <typename T> struct YuvSample { using Coeffs = YuvCoeffs; };
template <> struct YuvSample<uint16_t> { using Coeffs = Yuv16Coeffs; };

// One decoded tap of a 4:2:0 frame in layout L (kb200_yuv420_layout), or of a 4:4:4 frame (L = YUV444: the pixel's own
// U and V from the full-resolution planes).  PAIR: an interleaved chroma pair is read as one 16-bit word, which needs a
// 2-B aligned frame (the preprocess fast kernel's); PAIR = false reads its two bytes, so it takes frames at any address.
template <int L, bool PAIR = true>
__device__ __forceinline__ void yuv_tap(const uint8_t* __restrict__ src, int x, int y, int w, int h, const YuvCoeffs& yc, int rgb[3]) {
    if constexpr (L == YUV444) {
        // The same three bytes either way; each kernel gets the addressing with which ptxas allocates it without spills:
        // the fast kernel's f16 bilinear instantiations spill with the row form, the generic Lanczos loop with the other.
        int yv, u, v;
        if constexpr (PAIR) {
            const uint8_t* p = src + (size_t)y * w + x;
            const size_t plane = (size_t)w * h;
            yv = __ldg(p); u = __ldg(p + plane); v = __ldg(p + 2 * plane);
        } else {   // the frame as 3h rows: Y rows, then U rows, then V rows
            yv = __ldg(src + (size_t)y * w + x); u = __ldg(src + (size_t)(y + h) * w + x); v = __ldg(src + (size_t)(y + 2 * h) * w + x);
        }
        decode_rgb(yy_term(yv, yc), chroma_terms(u, v, yc), rgb[0], rgb[1], rgb[2]);
        return;
    }
    const int yv = __ldg(src + (size_t)y * w + x);
    ChromaTerms t;
    if (yuv420_planar(L)) {
        const size_t c = (size_t)(y >> 1) * (w >> 1) + (x >> 1);
        t = chroma_terms(__ldg(src + yuv420_u_plane(L, w, h) + c), __ldg(src + yuv420_v_plane(L, w, h) + c), yc);
    } else {
        const uint8_t* p = src + (size_t)w * h + (size_t)(y >> 1) * w + (x >> 1) * 2;
        uint32_t uv;
        if constexpr (PAIR) uv = __ldg(reinterpret_cast<const unsigned short*>(p));
        else uv = __ldg(p) | (uint32_t)__ldg(p + 1) << 8;
        t = L == YUV420_NV21 ? chroma_terms((int)(uv >> 8), (int)(uv & 0xFFu), yc) : chroma_terms((int)(uv & 0xFFu), (int)(uv >> 8), yc);
    }
    decode_rgb(yy_term(yv, yc), t, rgb[0], rgb[1], rgb[2]);
}
// ... and of a frame of 16-bit words (the coefficient type selects it): P01x in the NV12 layout, I01x in the I420 layout,
// I41x in the 4:4:4 one.  A P01x tap reads its chroma pair as two 16-bit words, since frames are only 2-B aligned.
template <int L>
__device__ __forceinline__ void yuv_tap(const uint8_t* __restrict__ src, int x, int y, int w, int h, const Yuv16Coeffs& k, int rgb[3]) {
    const uint16_t* s = reinterpret_cast<const uint16_t*>(src);
    const size_t plane = (size_t)w * h;
    size_t cu, cv;
    if constexpr (L == YUV444) {
        cu = plane + (size_t)y * w + x;
        cv = cu + plane;
    } else if (yuv420_planar(L)) {
        cu = plane + (size_t)(y >> 1) * (w >> 1) + (x >> 1);
        cv = cu + plane / 4;
    } else {
        cu = plane + (size_t)(y >> 1) * w + (x & ~1);
        cv = cu + 1;
    }
    const ChromaTerms t = chroma_terms16(yuv16_code(__ldg(s + cu), k), yuv16_code(__ldg(s + cv), k), k);
    decode_rgb16(yy_term16(yuv16_code(__ldg(s + (size_t)y * w + x), k), k), t, k.white, rgb[0], rgb[1], rgb[2]);
}

// One decoded tap of a 4:2:2 frame in layout L (kb200_yuv422_layout): the pixel's 2-px group at its byte places.
template <int L>
__device__ __forceinline__ void yuv422_tap(const uint8_t* __restrict__ src, int x, int y, int pitch, const YuvCoeffs& yc, int rgb[3]) {
    using P = Yuv422Bytes<L>;
    const uint8_t* grp = src + (long long)y * pitch + (x >> 1) * 4;
    const ChromaTerms t = chroma_terms(grp[P::u], grp[P::v], yc);
    decode_rgb(yy_term(grp[(x & 1) ? P::y1 : P::y0], yc), t, rgb[0], rgb[1], rgb[2]);
}

}  // namespace kb200
