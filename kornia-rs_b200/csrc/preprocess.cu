// preprocess.cu — the fused camera preprocess (a12; BASELINE config 3): raw frame (RGB/BGR/RGBA/
// Gray/NV12/YUYV, tight or pitched; beyond the reference also NV21/I420/YV12/UYVY/YVYU, the 8- and 16-bit Bayer
// mosaics, the 10- and 12-bit 4:2:0 video P010/P012/I010/I012 and the 4:4:4 video I444/I410/I412/I410Msb/I412Msb) →
// letterbox/stretch resample → (v/255 - mean) * inv_std → planar CHW f32, f16 or bf16, for a whole batch in ONE launch.
// The 4:2:0 formats share the NV12 kernels (templated on the chroma layout); the 4:2:2 formats take the generic kernel.
// A Bayer tap is the demosaiced pixel at the tap's coordinate (bayer.cuh); Bayer frames take the generic kernel, except
// the identity geometry, which has its own fast kernel.  A 16-bit Bayer tap is normalised against the white level
// W = 2^bits - 1 of its format: (px / W - mean) * inv_std, px / W the IEEE quotient.
// A YUV tap decodes with the colour matrix the fmt code carries in bits 8-9 (KB200_FMT_YUV_MATRIX): the entry points
// strip those bits from the descriptor and hand every kernel the matrix's coefficient set (YuvCoeffs) as an argument.
// The 10- and 12-bit 4:2:0 formats (fmt 80-83: P010, P012 in NV12's layout, I010, I012 in I420's, one 16-bit word per
// sample) take the 4:2:0 fast kernels instantiated for 16-bit words, with the Q16 set of their matrix and depth; a tap is
// the decoded n-bit code, normalised like a 16-bit Bayer tap by W = 2^n - 1.
// The 4:4:4 formats (fmt 11: I444 bytes; 85-88: I410, I412, I410Msb, I412Msb words) take their own identity kernel and
// preprocess_yuv_kernel in the YUV444 layout, the 4:2:0 layouts' resampler with a tap that reads the pixel's own chroma.
// The YUV taps (yuv_tap, yuv422_tap) are in yuv.cuh, as the Bayer taps are in bayer.cuh.
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
#include <cctype>

#include "preprocess.cuh"

namespace kb200 {

// One thread per output pixel of frame frame0 + blockIdx.y; SAMP: kb200_interp (generic_pixel).  STRIDED: the frame is
// fr.base + (frame0 + f) * fr.stride rather than fr.ptr[f]; only the packed-Bayer tap is instantiated so (launch_preprocess).
template <int OUT, int SAMP, int TAP, bool STRIDED = false>
__global__ void __launch_bounds__(256) preprocess_generic_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                 const __grid_constant__ PreFrames fr, void* __restrict__ dst,
                                                                 uint32_t frame0, const SrcFormat sf, const TapCoeffs<TAP> yc) {
    const int pixels = d.dst_w * d.dst_h;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pixels) return;
    const uint32_t f = blockIdx.y;
    const uint8_t* src = STRIDED ? fr.base + (size_t)(frame0 + f) * fr.stride : fr.ptr[f];
    const int ox = i % d.dst_w, oy = i / d.dst_w;
    float o[3];
    generic_pixel<SAMP, TAP>(src, ox, oy, d, sf, yc, FrameGeom{d}, o);
    generic_store<OUT>(dst, (size_t)(frame0 + f) * 3 * pixels + i, pixels, o);
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

// One thread = 4 luma columns x 2 rows.  Every warp-level access is lane-contiguous: 3 x LDG.32 (128 B per
// warp), 6 x STG.128 (512 contiguous bytes per warp per plane row).  [The first version gave each thread 8
// columns = two STG.128 per plane row; each store instruction then wrote only half of every 32-B sector and
// ncu showed 2x the write sectors at L2 (lts__t_sectors_srcunit_tex_op_write).]
// The other 4:2:0 layouts (L, kb200_yuv420_layout) take this kernel too: NV21 loads the same 4 chroma bytes and swaps
// each pair; I420 / YV12 load 2 U bytes and 2 V bytes (LDG.16 each; w % 4 == 0 keeps them 2-B aligned).
// 16-bit words (T = uint16_t): LDG.64 of 4 Y words per row; P01x one LDG.64 of the 2 chroma pairs, I01x 2 U words and
// 2 V words (LDG.32 each; w % 4 == 0 and even h keep them 4-B aligned in an 8-B aligned frame).  A pixel is normalised
// as (px / W - mean) * inv_std with the IEEE division, like a 16-bit Bayer tap.
template <int OUT, int L, typename T>
__global__ void __launch_bounds__(128) preprocess_yuv420_identity_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                         const __grid_constant__ PreFrames fr, void* __restrict__ dst,
                                                                         uint32_t frame0, uint32_t groups_per_row, uint32_t items,
                                                                         const typename YuvSample<T>::Coeffs yc) {
    const uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    if (item >= items) return;
    const uint32_t rp = item / groups_per_row, g = item - rp * groups_per_row;
    const uint32_t w = (uint32_t)d.src_w, h = (uint32_t)d.src_h;
    const uint32_t f = blockIdx.y;
    const uint8_t* src = fr.ptr[f];
    const uint32_t x = g * 4u;
    if constexpr (sizeof(T) == 2) {
        const uint16_t* s = reinterpret_cast<const uint16_t*>(src);
        const size_t plane = (size_t)w * h;
        const uint2 y0 = __ldg(reinterpret_cast<const uint2*>(s + (size_t)(2u * rp) * w + x));
        const uint2 y1 = __ldg(reinterpret_cast<const uint2*>(s + (size_t)(2u * rp + 1u) * w + x));
        ChromaTerms ct[2];
        if (yuv420_planar(L)) {
            const size_t c = (size_t)rp * (w / 2u) + x / 2u;
            const uint32_t u2 = __ldg(reinterpret_cast<const uint32_t*>(s + plane + c));
            const uint32_t v2 = __ldg(reinterpret_cast<const uint32_t*>(s + plane + plane / 4 + c));
            ct[0] = chroma_terms16(yuv16_code(u2, yc), yuv16_code(v2, yc), yc);
            ct[1] = chroma_terms16(yuv16_code(u2 >> 16, yc), yuv16_code(v2 >> 16, yc), yc);
        } else {
            const uint2 uv = __ldg(reinterpret_cast<const uint2*>(s + plane + (size_t)rp * w + x));
            ct[0] = chroma_terms16(yuv16_code(uv.x, yc), yuv16_code(uv.x >> 16, yc), yc);
            ct[1] = chroma_terms16(yuv16_code(uv.y, yc), yuv16_code(uv.y >> 16, yc), yc);
        }
        const size_t base = (size_t)(frame0 + f) * 3 * plane + (size_t)(2u * rp) * w + x;
        const float m0 = d.mean[0], m1 = d.mean[1], m2 = d.mean[2], i0 = d.inv_std[0], i1 = d.inv_std[1], i2 = d.inv_std[2];
        const float wl = (float)yc.white;
#pragma unroll
        for (int row = 0; row < 2; ++row) {
            const uint2 yw = row == 0 ? y0 : y1;
            float r4[4], g4[4], b4[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int yv = yuv16_code((i < 2 ? yw.x : yw.y) >> (16 * (i & 1)), yc);
                int r, gg, b;
                decode_rgb16(yy_term16(yv, yc), ct[i >> 1], yc.white, r, gg, b);
                r4[i] = (div_white((float)r, wl) - m0) * i0;
                g4[i] = (div_white((float)gg, wl) - m1) * i1;
                b4[i] = (div_white((float)b, wl) - m2) * i2;
            }
            const size_t o = base + (size_t)row * w;
            nv12_store4<OUT>(dst, o, r4);
            nv12_store4<OUT>(dst, o + plane, g4);
            nv12_store4<OUT>(dst, o + 2 * plane, b4);
        }
    } else {
        const uint32_t y0w = __ldg(reinterpret_cast<const uint32_t*>(src + (size_t)(2u * rp) * w + x));
        const uint32_t y1w = __ldg(reinterpret_cast<const uint32_t*>(src + (size_t)(2u * rp + 1u) * w + x));
        ChromaTerms ct[2];
        if (yuv420_planar(L)) {
            const size_t c = (size_t)rp * (w / 2u) + x / 2u;
            const uint32_t u2 = __ldg(reinterpret_cast<const unsigned short*>(src + yuv420_u_plane(L, w, h) + c));
            const uint32_t v2 = __ldg(reinterpret_cast<const unsigned short*>(src + yuv420_v_plane(L, w, h) + c));
            ct[0] = chroma_terms((int)(u2 & 0xFFu), (int)(v2 & 0xFFu), yc);
            ct[1] = chroma_terms((int)(u2 >> 8), (int)(v2 >> 8), yc);
        } else {
            const uint32_t uvw = __ldg(reinterpret_cast<const uint32_t*>(src + (size_t)w * h + (size_t)rp * w + x));
            if (L == YUV420_NV21) {
                ct[0] = chroma_terms((int)((uvw >> 8) & 0xFFu), (int)(uvw & 0xFFu), yc);
                ct[1] = chroma_terms((int)(uvw >> 24), (int)((uvw >> 16) & 0xFFu), yc);
            } else {
                ct[0] = chroma_terms((int)(uvw & 0xFFu), (int)((uvw >> 8) & 0xFFu), yc);
                ct[1] = chroma_terms((int)((uvw >> 16) & 0xFFu), (int)(uvw >> 24), yc);
            }
        }
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
                decode_rgb(yy_term(yv, yc), ct[i >> 1], r, gg, b);
                r4[i] = norm_int_px(r, m0, i0);
                g4[i] = norm_int_px(gg, m1, i1);
                b4[i] = norm_int_px(b, m2, i2);
            }
            const size_t o = base + (size_t)row * w;
            nv12_store4<OUT>(dst, o, r4);
            nv12_store4<OUT>(dst, o + plane, g4);
            nv12_store4<OUT>(dst, o + 2 * plane, b4);
        }
    }
}

// ── 4:4:4 identity fast path (the config-3a shape from I444 / I41x frames: scale 1, no pad, same size) ──────────────
// Every pixel has its own chroma, so one thread = 4 columns of one row: one lane-contiguous load from each of the Y, U
// and V planes (LDG.32 of 4 bytes, LDG.64 of 4 words: w % 4 == 0 and a frame aligned to that load align every plane's
// rows), 3 x nv12_store4.  Bytes are normalised as in the 4:2:0 kernel (norm_int_px), words by W through div_white.
template <int OUT, typename T>
__global__ void __launch_bounds__(128) preprocess_yuv444_identity_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                         const __grid_constant__ PreFrames fr, void* __restrict__ dst,
                                                                         uint32_t frame0, uint32_t groups_per_row, uint32_t items,
                                                                         const typename YuvSample<T>::Coeffs yc) {
    const uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    if (item >= items) return;
    const uint32_t y = item / groups_per_row, g = item - y * groups_per_row;
    const uint32_t w = (uint32_t)d.src_w, h = (uint32_t)d.src_h;
    const uint32_t f = blockIdx.y;
    const uint8_t* src = fr.ptr[f];
    const size_t plane = (size_t)w * h, p = (size_t)y * w + g * 4u;
    const float m0 = d.mean[0], m1 = d.mean[1], m2 = d.mean[2], i0 = d.inv_std[0], i1 = d.inv_std[1], i2 = d.inv_std[2];
    float r4[4], g4[4], b4[4];
    if constexpr (sizeof(T) == 2) {
        const uint16_t* s = reinterpret_cast<const uint16_t*>(src);
        const uint2 yv = __ldg(reinterpret_cast<const uint2*>(s + p));
        const uint2 uv = __ldg(reinterpret_cast<const uint2*>(s + plane + p));
        const uint2 vv = __ldg(reinterpret_cast<const uint2*>(s + 2 * plane + p));
        const float wl = (float)yc.white;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int sh = 16 * (i & 1);
            const uint32_t yw = i < 2 ? yv.x : yv.y, uw = i < 2 ? uv.x : uv.y, vw = i < 2 ? vv.x : vv.y;
            int r, gg, b;
            decode_rgb16(yy_term16(yuv16_code(yw >> sh, yc), yc), chroma_terms16(yuv16_code(uw >> sh, yc), yuv16_code(vw >> sh, yc), yc),
                         yc.white, r, gg, b);
            r4[i] = (div_white((float)r, wl) - m0) * i0;
            g4[i] = (div_white((float)gg, wl) - m1) * i1;
            b4[i] = (div_white((float)b, wl) - m2) * i2;
        }
    } else {
        const uint32_t yw = __ldg(reinterpret_cast<const uint32_t*>(src + p));
        const uint32_t uw = __ldg(reinterpret_cast<const uint32_t*>(src + plane + p));
        const uint32_t vw = __ldg(reinterpret_cast<const uint32_t*>(src + 2 * plane + p));
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int r, gg, b;
            decode_rgb(yy_term((int)((yw >> (8 * i)) & 0xFFu), yc), chroma_terms((int)((uw >> (8 * i)) & 0xFFu), (int)((vw >> (8 * i)) & 0xFFu), yc),
                       r, gg, b);
            r4[i] = norm_int_px(r, m0, i0);
            g4[i] = norm_int_px(gg, m1, i1);
            b4[i] = norm_int_px(b, m2, i2);
        }
    }
    const size_t o = (size_t)(frame0 + f) * 3 * plane + p;
    nv12_store4<OUT>(dst, o, r4);
    nv12_store4<OUT>(dst, o + plane, g4);
    nv12_store4<OUT>(dst, o + 2 * plane, b4);
}

// ── Bayer identity fast path (the config-3a shape from a Bayer mosaic: scale 1, no pad, same size) ──────────────
// As for 4:2:0, the sample is the demosaiced pixel (ox, oy) itself.  One thread = 4 columns x 2 output rows (the row
// pairs of bayer_row_pairs): 4 lane-contiguous loads of the rows ya-1 .. ya+2 (LDG.32 of 8-bit samples, LDG.64 of 16-bit
// ones: BayerSample<T>::ID_WORDS) plus shuffled halos (bayer_load_rows), 6 to 12 lane-contiguous 4-pixel stores per
// thread (nv12_store4).  Requires w % 4 == 0 and rows aligned to BayerSample<T>::ID_ALIGN.
// Packed samples (T = BayerPacked<BITS>): a thread's 4 columns are BITS / 2 bytes of a row, read as the aligned 8-byte
// word that holds their first byte and, when they run past it, the next one (L1-allocating: the neighbouring lanes read
// the same words), then unpacked into the words of the 16-bit kernel (bayer_unpack).  Rows and frames 16-B aligned.
template <int OUT, typename T, int P>
__global__ void __launch_bounds__(128) preprocess_bayer_identity_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                        const __grid_constant__ PreFrames fr, void* __restrict__ dst,
                                                                        uint32_t frame0, uint32_t groups_per_row, uint32_t items, uint32_t bits) {
    constexpr uint32_t NW = BayerSample<T>::ID_WORDS;
    constexpr int PB = BayerSample<T>::PACKED_BITS;
    const uint32_t item = blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = item < items;                         // the lanes past the end still take part in the shuffles
    const uint32_t it = active ? item : items - 1;
    const uint32_t rp = it / groups_per_row, g = it - rp * groups_per_row;
    const uint32_t w = (uint32_t)d.src_w, h = (uint32_t)d.src_h;
    const uint32_t f = blockIdx.y;
    const T* src = reinterpret_cast<const T*>(fr.ptr[f]);
    const uint32_t x = g * 4u, ya = 1u + 2u * rp, yb = ya + 1u;
    uint32_t rows[4][NW];
    int hl[4], hr[4];
    if constexpr (PB == 0) {
        bayer_load_rows<NW>(src, (size_t)d.src_pitch / sizeof(T), w, h, x, ya, threadIdx.x & 31u, [](const T* p, uint32_t v[NW]) {
            if constexpr (NW == 1) {
                v[0] = __ldg(reinterpret_cast<const uint32_t*>(p));
            } else {
                const uint2 q = __ldg(reinterpret_cast<const uint2*>(p));
                v[0] = q.x; v[1] = q.y;
            }
        }, rows, hl, hr);
    } else {
        const uint32_t off = x * PB / 8, s = off & 7u;   // the thread's first byte in its row, and its place in its 8-byte word
        bayer_load_rows_packed<NW, PB>(reinterpret_cast<const uint8_t*>(src), (size_t)d.src_pitch, w, h, x, ya, threadIdx.x & 31u,
                                       [&](int, const uint8_t* row, uint32_t v[NW]) {
            const uint2* p = reinterpret_cast<const uint2*>(row + (off - s));
            const uint2 a = __ldg(p);
            const uint2 b = s + PB / 2 > 8u ? __ldg(p + 1) : make_uint2(0, 0);
            const uint32_t t0 = s >= 4u ? a.y : a.x, t1 = s >= 4u ? b.x : a.y, t2 = s >= 4u ? b.y : b.x;
            const uint32_t sh = 8u * (s & 3u);
            const uint32_t bytes[2] = {__funnelshift_r(t0, t1, sh), __funnelshift_r(t1, t2, sh)};
            bayer_unpack<PB, 4>(bytes, v);
        }, rows, hl, hr);
    }
    if (!active) return;
    const bool left_edge = x == 0, right_edge = x + 4u == w;
    const size_t plane = (size_t)w * h;
    const size_t base = (size_t)(frame0 + f) * 3 * plane + x;
    // the white level W of a 16-bit (`bits` from the host's SrcFormat) or packed format
    [[maybe_unused]] const float wl = PB == 0 ? (float)((1u << bits) - 1u) : (float)((1u << PB) - 1u);
    const float m0 = d.mean[0], m1 = d.mean[1], m2 = d.mean[2], i0 = d.inv_std[0], i1 = d.inv_std[1], i2 = d.inv_std[2];
    float r4[4], g4[4], b4[4];
    auto store_row = [&](uint32_t y) {
        const size_t o = base + (size_t)y * w;
        nv12_store4<OUT>(dst, o, r4);
        nv12_store4<OUT>(dst, o + plane, g4);
        nv12_store4<OUT>(dst, o + 2 * plane, b4);
    };
    // 8-bit: px / 255 by the exact 3-instruction form (norm_int_px); 16-bit and packed: px / W, the IEEE division
    auto norm = [&](const int r[4], const int gg[4], const int b[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if constexpr (std::is_same_v<T, uint8_t>) {
                r4[i] = norm_int_px(r[i], m0, i0); g4[i] = norm_int_px(gg[i], m1, i1); b4[i] = norm_int_px(b[i], m2, i2);
            } else {
                r4[i] = (__fdiv_rn((float)r[i], wl) - m0) * i0;
                g4[i] = (__fdiv_rn((float)gg[i], wl) - m1) * i1;
                b4[i] = (__fdiv_rn((float)b[i], wl) - m2) * i2;
            }
        }
    };
    using W = typename BayerSample<T>::Word;
    int r[4], gg[4], b[4];
    bayer_row<P, 1, NW, W>(rows[0], rows[1], rows[2], hl, hr, left_edge, right_edge, r, gg, b);   // ya is odd
    norm(r, gg, b);
    store_row(ya);
    if (ya == 1u) store_row(0);
    if (yb == h - 1u) { store_row(yb); return; }
    bayer_row<P, 0, NW, W>(rows[1], rows[2], rows[3], hl + 1, hr + 1, left_edge, right_edge, r, gg, b);
    norm(r, gg, b);
    store_row(yb);
    if (yb == h - 2u) store_row(h - 1u);
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
// The sampler is yuv_resample (preprocess.cuh), here over frame frame0 + blockIdx.z.
template <int OUT, bool BILINEAR, int L, typename T>
__global__ void __launch_bounds__(128) preprocess_yuv_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                             const __grid_constant__ PreFrames fr, const __grid_constant__ Nv12Args na,
                                                             void* __restrict__ dst, uint32_t frame0, const typename YuvSample<T>::Coeffs yc) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= na.groups) return;
    const uint32_t f = blockIdx.z;
    const uint8_t* src = fr.ptr[f];
    yuv_resample<OUT, BILINEAR, L, T>(FrameGeom{d}, src, d, na, dst, frame0 + f, (int)g * 4, yc);
}

// One row per format code.  A Bayer code is 16 + pattern (8-bit samples), 32 + 4*k + pattern (16-bit words, k = 0..3 for
// 10, 12, 14 and 16 bits) or 64 + 4*k + pattern (packed, k = 0..2 for 10, 12 and 14 bits); each sample type has its own
// identity kernel, and the 16-bit one serves every depth.
#define KB200_BAYER_FORMATS(code, suffix, bits, words, packed, kernel)                                                            \
    {code, "BayerRggb" suffix, SRC_BAYER, 0, KB200_BAYER_RGGB, bits, words, packed, "preprocess_" kernel "_rggb_identity_kernel"},     \
    {code + 1, "BayerBggr" suffix, SRC_BAYER, 0, KB200_BAYER_BGGR, bits, words, packed, "preprocess_" kernel "_bggr_identity_kernel"}, \
    {code + 2, "BayerGrbg" suffix, SRC_BAYER, 0, KB200_BAYER_GRBG, bits, words, packed, "preprocess_" kernel "_grbg_identity_kernel"}, \
    {code + 3, "BayerGbrg" suffix, SRC_BAYER, 0, KB200_BAYER_GBRG, bits, words, packed, "preprocess_" kernel "_gbrg_identity_kernel"}
static const SrcFormat SRC_FORMATS[] = {
    {KB200_FMT_RGB, "Rgb8", SRC_RGB, 0},
    {KB200_FMT_BGR, "Bgr8", SRC_RGB, 1},
    {KB200_FMT_GRAY, "Gray8", SRC_GRAY},
    {KB200_FMT_NV12, "Nv12", SRC_YUV420, YUV420_NV12, 0, 8, false, false, "preprocess_nv12_identity_kernel", "preprocess_nv12_kernel"},
    {KB200_FMT_YUYV, "Yuyv", SRC_YUV422, YUV422_YUYV},
    {KB200_FMT_NV21, "Nv21", SRC_YUV420, YUV420_NV21, 0, 8, false, false, "preprocess_nv21_identity_kernel", "preprocess_nv21_kernel"},
    {KB200_FMT_I420, "I420", SRC_YUV420, YUV420_I420, 0, 8, false, false, "preprocess_i420_identity_kernel", "preprocess_i420_kernel"},
    {KB200_FMT_YV12, "Yv12", SRC_YUV420, YUV420_YV12, 0, 8, false, false, "preprocess_yv12_identity_kernel", "preprocess_yv12_kernel"},
    {KB200_FMT_UYVY, "Uyvy", SRC_YUV422, YUV422_UYVY},
    {KB200_FMT_YVYU, "Yvyu", SRC_YUV422, YUV422_YVYU},
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB, "", 8, false, false, "bayer"),
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB10, "10", 10, true, false, "bayer16"),
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB12, "12", 12, true, false, "bayer16"),
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB14, "14", 14, true, false, "bayer16"),
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB16, "16", 16, true, false, "bayer16"),
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB10P, "10p", 10, false, true, "bayer10p"),
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB12P, "12p", 12, false, true, "bayer12p"),
    KB200_BAYER_FORMATS(KB200_FMT_BAYER_RGGB14P, "14p", 14, false, true, "bayer14p"),
    // 10- and 12-bit 4:2:0 video: P01x in NV12's layout with each code in the high bits of its word, I01x in I420's with it
    // in the low bits; the 16-bit instantiations of the 4:2:0 fast kernels serve both depths
    {KB200_FMT_P010, "P010", SRC_YUV420, YUV420_NV12, 0, 10, true, false, "preprocess_p01x_identity_kernel", "preprocess_p01x_kernel"},
    {KB200_FMT_P012, "P012", SRC_YUV420, YUV420_NV12, 0, 12, true, false, "preprocess_p01x_identity_kernel", "preprocess_p01x_kernel"},
    {KB200_FMT_I010, "I010", SRC_YUV420, YUV420_I420, 0, 10, true, false, "preprocess_i01x_identity_kernel", "preprocess_i01x_kernel"},
    {KB200_FMT_I012, "I012", SRC_YUV420, YUV420_I420, 0, 12, true, false, "preprocess_i01x_identity_kernel", "preprocess_i01x_kernel"},
    // 4:4:4 video: three full-resolution planes, of bytes (I444) or of 16-bit words with each code in the low (I41x) or the
    // high bits (I41xMsb); the 4:4:4 identity kernel and the YUV444 instantiations of preprocess_yuv_kernel serve them
    {KB200_FMT_I444, "I444", SRC_YUV444, 0, 0, 8, false, false, "preprocess_i444_identity_kernel", "preprocess_i444_kernel"},
    {KB200_FMT_I410, "I410", SRC_YUV444, KB200_YUV444_I41X, 0, 10, true, false, "preprocess_i41x_identity_kernel", "preprocess_i41x_kernel"},
    {KB200_FMT_I412, "I412", SRC_YUV444, KB200_YUV444_I41X, 0, 12, true, false, "preprocess_i41x_identity_kernel", "preprocess_i41x_kernel"},
    {KB200_FMT_I410_MSB, "I410Msb", SRC_YUV444, KB200_YUV444_I41X_MSB, 0, 10, true, false, "preprocess_i41x_identity_kernel", "preprocess_i41x_kernel"},
    {KB200_FMT_I412_MSB, "I412Msb", SRC_YUV444, KB200_YUV444_I41X_MSB, 0, 12, true, false, "preprocess_i41x_identity_kernel", "preprocess_i41x_kernel"},
};
#undef KB200_BAYER_FORMATS

SrcFormat src_format(int fmt) {
    for (const SrcFormat& f : SRC_FORMATS)
        if (f.code == fmt) return f;
    return {};
}

// kb200_preprocess_desc::fmt = format code (bits 0-7) | KB200_FMT_YUV_MATRIX(m) (bits 8-9).  The entry points strip the
// matrix once, here: every other function sees the plain code and gets the matrix (kb200_yuv_matrix) on its own.
kb200_preprocess_desc plain_desc(const kb200_preprocess_desc& d) {
    kb200_preprocess_desc p = d;
    p.fmt = d.fmt & 0xFF;
    return p;
}
int yuv_matrix(const kb200_preprocess_desc& raw) { return (raw.fmt >> 8) & 3; }

size_t src_bytes(const kb200_preprocess_desc& d) {
    // 4:2:0 chroma after the pitch * h luma bytes: w*h/2 samples, of 1 byte or of 2 (16-bit words); 4:4:4: two more planes
    const SrcFormat f = src_format(d.fmt);
    if (f.family == SRC_YUV444) return (size_t)d.src_pitch * d.src_h * 3;
    const size_t chroma = f.family != SRC_YUV420 ? 0 : f.words ? (size_t)d.src_w * d.src_h : (size_t)d.src_w * d.src_h / 2;
    return (size_t)d.src_pitch * d.src_h + chroma;
}

int validate_desc(const kb200_preprocess_desc* dp) {
    if (!dp) return fail(KB200_ERR_INVALID_ARGUMENT, "null preprocess descriptor");
    if (dp->src_w <= 0 || dp->src_h <= 0 || dp->dst_w <= 0 || dp->dst_h <= 0)
        return fail(KB200_ERR_INVALID_ARGUMENT, "image dimensions must be non-zero");
    if ((long long)dp->dst_w * dp->dst_h > 0x7FFFFFFFll) return fail(KB200_ERR_DIMS_TOO_LARGE, "dimensions exceed the 32-bit CUDA kernel index limit");  // :1336-1339
    const kb200_preprocess_desc d = plain_desc(*dp);
    const SrcFormat f = src_format(d.fmt);
    if (dp->fmt < 0 || !f.name) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown source format code %d", dp->fmt);
    if (dp->fmt >> 10)
        return fail(KB200_ERR_INVALID_ARGUMENT, "source format code %d has bits set above bit 9 (bits 8-9 are the YUV matrix, 0-3)", dp->fmt);
    if ((dp->fmt >> 8) && f.family != SRC_YUV420 && f.family != SRC_YUV422 && f.family != SRC_YUV444)
        return fail(KB200_ERR_INVALID_ARGUMENT, "source format code %d: a YUV matrix (%d) applies only to the YUV formats, not format code %d", dp->fmt,
                    dp->fmt >> 8, d.fmt);
    if (d.sampling != KB200_INTERP_NEAREST && d.sampling != KB200_INTERP_BILINEAR && d.sampling != KB200_INTERP_LANCZOS)
        return fail(KB200_ERR_UNSUPPORTED, "unsupported sampling mode %d (expected Nearest, Bilinear or Lanczos)", d.sampling);  // preprocess.rs:1044-1051
    if (f.family == SRC_RGB && d.src_bpp != 3 && d.src_bpp != 4) return fail(KB200_ERR_UNSUPPORTED, "unsupported source channel count %d (expected 3 or 4)", d.src_bpp);
    // SourceFormat::dims_ok :188-195 ; pitch covers a row (PitchedSurface::validate :829-842)
    if (f.family == SRC_YUV420 && ((d.src_w | d.src_h) & 1)) return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source for %s at %dx%d (even dimensions required)", f.name, d.src_w, d.src_h);
    if (f.family == SRC_YUV422 && (d.src_w & 1)) return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source for %s at %dx%d (even width required)", f.name, d.src_w, d.src_h);
    if (f.family == SRC_BAYER && (d.src_w < 3 || d.src_h < 3))
        return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source for %s at %dx%d (at least 3x3 required)", f.name, d.src_w, d.src_h);
    if (f.family == SRC_BAYER && f.words && (d.src_pitch & 1))
        return fail(KB200_ERR_INVALID_SOURCE, "invalid pitched surface for %s (pitch %d is odd: rows of 16-bit samples must start 2-byte aligned)", f.name, d.src_pitch);
    if (f.packed) {
        const int g = bayer_packed_group(f.bits);
        if (d.src_w % g)
            return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source for %s at %dx%d (the width must be a multiple of %d: whole %d-byte groups)", f.name,
                        d.src_w, d.src_h, g, bayer_packed_group_bytes(f.bits));
        if ((long long)d.src_pitch < (long long)d.src_w * f.bits / 8)
            return fail(KB200_ERR_INVALID_SOURCE, "invalid pitched surface for %s (pitch %d < %lld bytes of a packed row)", f.name, d.src_pitch,
                        (long long)d.src_w * f.bits / 8);
    }
    if ((f.family == SRC_YUV420 || f.family == SRC_YUV444) && f.words && (long long)d.src_pitch != 2ll * d.src_w)
        return fail(KB200_ERR_INVALID_SOURCE, "invalid pitched surface for %s (pitch %d bytes at width %d: frames must be tightly packed, pitch == 2*width)",
                    f.name, d.src_pitch, d.src_w);
    const int bpp = f.family == SRC_RGB ? d.src_bpp : f.family == SRC_YUV422 || f.words ? 2 : 1;
    if (!f.packed && (long long)d.src_pitch < (long long)d.src_w * bpp)
        return fail(KB200_ERR_INVALID_SOURCE, "invalid pitched surface (need pitch >= width*channels and len >= pitch*height)");
    if ((f.family == SRC_YUV420 || f.family == SRC_YUV444) && !f.words && d.src_pitch != d.src_w) {
        char upper[8] = "";   // the layout's own spelling: NV12, NV21, I420, YV12, I444
        for (int i = 0; f.name[i] && i < 7; ++i) upper[i] = (char)toupper((unsigned char)f.name[i]);
        return fail(KB200_ERR_INVALID_SOURCE, "%s frames must be tightly packed (pitch == width)", upper);
    }
    if (!(d.scale_x > 0.0f) || !(d.scale_y > 0.0f)) return fail(KB200_ERR_INVALID_ARGUMENT, "scale must be positive");
    return KB200_OK;
}

int check_frame_table(const kb200_preprocess_desc& d, const uint8_t* const* frames, const size_t* frame_len, uint32_t n) {
    const SrcFormat f = src_format(d.fmt);
    const size_t need = src_bytes(d);
    for (uint32_t i = 0; i < n; ++i) {
        if (!frames[i]) return fail(KB200_ERR_INVALID_ARGUMENT, "null frame pointer at index %u", i);
        if (f.words && (reinterpret_cast<uintptr_t>(frames[i]) & 1u)) return fail(KB200_ERR_INVALID_SOURCE, "%s frame %u is not 2-byte aligned", f.name, i);
        if (frame_len && frame_len[i] < need)  // InvalidRawSource{got,need}, preprocess.rs:1287-1300
            return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source at %dx%d (got %zu bytes, need %zu)", d.src_w, d.src_h, frame_len[i], need);
    }
    return KB200_OK;
}

int check_region_call(const kb200_preprocess_desc* desc, const int* mode, const char* point, int out_format, kb200_preprocess_desc* raw,
                      kb200_preprocess_desc* plain) {
    if (!desc) return fail(KB200_ERR_INVALID_ARGUMENT, "null preprocess descriptor");
    *raw = *desc;   // each region gets its own geometry: the descriptor's scale and pad are not used
    raw->scale_x = raw->scale_y = 1.0f;
    raw->pad_x = raw->pad_y = 0.0f;
    KB200_TRY(validate_desc(raw));
    if (mode && *mode != 0 && *mode != 1) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown resize mode %d (expected 0 Letterbox or 1 Stretch)", *mode);
    if (point && raw->sampling == KB200_INTERP_LANCZOS)
        return fail(KB200_ERR_UNSUPPORTED, "unsupported sampling mode %d for %s (expected Nearest or Bilinear)", raw->sampling, point);
    if (out_format != KB200_OUT_F32 && out_format != KB200_OUT_F16 && out_format != KB200_OUT_BF16)
        return fail(KB200_ERR_INVALID_ARGUMENT, "unknown output format %d (expected 0 f32, 1 f16 or 2 bf16)", out_format);
    *plain = plain_desc(*raw);
    return KB200_OK;
}

int check_region_frame(uint32_t i, int32_t frame, uint32_t n_frames) {
    if (frame < 0 || (uint32_t)frame >= n_frames)
        return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: frame index %d is outside [0, %u)", i, frame, n_frames);
    return KB200_OK;
}

// The fast kernels of layout L (4:2:0, or YUV444) and sample type T, for one launch of <= 256 frames.
template <int OUT, int L, typename T = uint8_t>
static void launch_yuv_fast(cudaStream_t s, bool identity, bool bil, const kb200_preprocess_desc& d, const typename YuvSample<T>::Coeffs& yc,
                            const PreFrames& fr, const Nv12Args& nv, void* dst, uint32_t f0, uint32_t nb, uint32_t id_groups, size_t id_items) {
    if (identity) {
        dim3 grid(div_up(id_items, 128), nb);
        if constexpr (L == YUV444) preprocess_yuv444_identity_kernel<OUT, T><<<grid, 128, 0, s>>>(d, fr, dst, f0, id_groups, (uint32_t)id_items, yc);
        else preprocess_yuv420_identity_kernel<OUT, L, T><<<grid, 128, 0, s>>>(d, fr, dst, f0, id_groups, (uint32_t)id_items, yc);
        return;
    }
    dim3 grid(div_up(nv.groups, 128), div_up((size_t)d.dst_h, NV12_ROWS), nb);
    if (bil) preprocess_yuv_kernel<OUT, true, L, T><<<grid, 128, 0, s>>>(d, fr, nv, dst, f0, yc);
    else preprocess_yuv_kernel<OUT, false, L, T><<<grid, 128, 0, s>>>(d, fr, nv, dst, f0, yc);
}

// The Bayer identity kernel of sample type T and pattern P, for one launch of <= 256 frames.
template <int OUT, typename T, int P>
static void launch_bayer_identity(cudaStream_t s, const kb200_preprocess_desc& d, const PreFrames& fr, void* dst, uint32_t f0, uint32_t nb,
                                  uint32_t id_groups, size_t id_items, uint32_t bits) {
    dim3 grid(div_up(id_items, 128), nb);
    preprocess_bayer_identity_kernel<OUT, T, P><<<grid, 128, 0, s>>>(d, fr, dst, f0, id_groups, (uint32_t)id_items, bits);
}

template <int OUT, int TAP, bool STRIDED = false>
static void launch_generic(cudaStream_t s, dim3 grid, const kb200_preprocess_desc& d, const SrcFormat& f, const TapCoeffs<TAP>& yc,
                           const PreFrames& fr, void* dst, uint32_t f0) {
    if (d.sampling == KB200_INTERP_LANCZOS) preprocess_generic_kernel<OUT, KB200_INTERP_LANCZOS, TAP, STRIDED><<<grid, 256, 0, s>>>(d, fr, dst, f0, f, yc);
    else if (d.sampling == KB200_INTERP_BILINEAR) preprocess_generic_kernel<OUT, KB200_INTERP_BILINEAR, TAP, STRIDED><<<grid, 256, 0, s>>>(d, fr, dst, f0, f, yc);
    else preprocess_generic_kernel<OUT, KB200_INTERP_NEAREST, TAP, STRIDED><<<grid, 256, 0, s>>>(d, fr, dst, f0, f, yc);
}

template <int OUT>
static void launch_generic_for(cudaStream_t s, dim3 grid, const kb200_preprocess_desc& d, const SrcFormat& f, const YuvCoeffs& yc,
                               const Yuv16Coeffs& yc16, const PreFrames& fr, void* dst, uint32_t f0) {
    with_tap(f, yc, yc16, [&](auto tap, const auto& c) { launch_generic<OUT, decltype(tap)::value>(s, grid, d, f, c, fr, dst, f0); });
}

// d: a validated descriptor with the plain format code; matrix: its kb200_yuv_matrix
template <int OUT>
static int launch_preprocess(cudaStream_t s, const kb200_preprocess_desc& d, int matrix, const uint8_t* const* frames, const uint8_t* base,
                             size_t stride, uint32_t batch, void* dst) {
    const SrcFormat f = src_format(d.fmt);
    const int pixels = d.dst_w * d.dst_h;
    const bool bil = d.sampling == KB200_INTERP_BILINEAR, lanczos = d.sampling == KB200_INTERP_LANCZOS;
    const bool bayer = f.family == SRC_BAYER;
    // identity fast path: a format with an identity kernel (4:2:0, 4:4:4 or Bayer), scale 1, no pad, same size, 8-column vectors
    // possible (Lanczos always takes the generic kernel: its off-centre weights at integer coordinates are sinf(k*pi) != 0
    // exactly).  A thread loads 4 samples per row, so rows and frames are aligned to that load: 4 B for bytes, 8 B for
    // 16-bit words, 16 B for packed Bayer.
    const uint32_t row_align = f.packed ? BayerSample<BayerPacked<12>>::ID_ALIGN
                                        : f.words ? BayerSample<uint16_t>::ID_ALIGN : BayerSample<uint8_t>::ID_ALIGN;
    bool identity = !lanczos && f.identity_kernel && d.scale_x == 1.0f && d.scale_y == 1.0f && d.pad_x == 0.0f && d.pad_y == 0.0f &&
                    d.dst_w == d.src_w && d.dst_h == d.src_h && (d.src_w % 4) == 0 && (d.src_pitch % row_align) == 0 && aligned16(dst) &&
                    frames_aligned(frames, base, stride, batch, row_align);
    const uint32_t id_groups = (uint32_t)d.src_w / 4u;
    const size_t id_rows = bayer ? bayer_row_pairs((uint32_t)d.src_h) : f.family == SRC_YUV444 ? (size_t)d.src_h : (size_t)d.src_h / 2;
    const size_t id_items = (size_t)id_groups * id_rows;   // threads of 4 columns x (2 rows, or 1 row of 4:4:4)
    if (id_items > 0x7FFFFFFFull) identity = false;
    const bool yuv420_fast = yuv_resampler_ok(f, d, dst, frames_aligned(frames, base, stride, batch, 2));
    const YuvCoeffs& yc = YUV_COEFFS[matrix];
    const Yuv16Coeffs yc16 = yuv16_coeffs_of(f, matrix);   // used by the 16-bit 4:2:0 and 4:4:4 formats only
    const Nv12Args nv = nv12_args(d);
    for (uint32_t f0 = 0; f0 < batch; f0 += 256) {
        const uint32_t nb = std::min<uint32_t>(256, batch - f0);
        PreFrames fr{};
        fr.base = base; fr.stride = stride;
        for (uint32_t k = 0; k < nb; ++k) fr.ptr[k] = frames ? frames[f0 + k] : base + (size_t)(f0 + k) * stride;
        if (identity && bayer) {
            auto launch = [&](auto sample) {   // the kernel of the format's pattern for samples of the type of `sample`
                using T = decltype(sample);
                switch (f.pattern) {
                    case KB200_BAYER_RGGB: launch_bayer_identity<OUT, T, KB200_BAYER_RGGB>(s, d, fr, dst, f0, nb, id_groups, id_items, f.bits); break;
                    case KB200_BAYER_BGGR: launch_bayer_identity<OUT, T, KB200_BAYER_BGGR>(s, d, fr, dst, f0, nb, id_groups, id_items, f.bits); break;
                    case KB200_BAYER_GRBG: launch_bayer_identity<OUT, T, KB200_BAYER_GRBG>(s, d, fr, dst, f0, nb, id_groups, id_items, f.bits); break;
                    default: launch_bayer_identity<OUT, T, KB200_BAYER_GBRG>(s, d, fr, dst, f0, nb, id_groups, id_items, f.bits); break;
                }
            };
            if (!f.packed && f.words) launch(uint16_t{});
            else if (!f.packed) launch(uint8_t{});
            else if (f.bits == 10) launch(BayerPacked<10>{});
            else if (f.bits == 12) launch(BayerPacked<12>{});
            else launch(BayerPacked<14>{});
            KB200_TRY(check_launch(f.identity_kernel));
            continue;
        }
        if (identity || yuv420_fast) {
            with_yuv_layout(f, yc, yc16, [&](auto l, auto t, const auto& c) {
                launch_yuv_fast<OUT, decltype(l)::value, decltype(t)>(s, identity, bil, d, c, fr, nv, dst, f0, nb, id_groups, id_items);
            });
            KB200_TRY(check_launch(identity ? f.identity_kernel : f.fast_kernel));
            continue;
        }
        dim3 grid(div_up(pixels, 256), nb);
        // The packed-Bayer generic kernel reading base + i * stride compiles shorter than the one reading the table (its
        // tap addresses in 64-bit adds, not IMAD.WIDE) and runs about 1.5 % faster on a strided batch, so it is kept
        if (f.packed && !frames) launch_generic<OUT, TAP_BAYER_PACKED, true>(s, grid, d, f, yc, fr, dst, f0);
        else launch_generic_for<OUT>(s, grid, d, f, yc, yc16, fr, dst, f0);
        KB200_TRY(check_launch("preprocess_generic_kernel"));
    }
    return KB200_OK;
}

// used by the host-buffer pipeline (host_pipeline.cu): frames already staged at base + i*stride on the device
int preprocess_validate(const kb200_preprocess_desc* desc) { return validate_desc(desc); }
size_t preprocess_frame_bytes(const kb200_preprocess_desc& d) { return src_bytes(plain_desc(d)); }
// out: a kb200_out_format the caller has checked
int preprocess_launch_strided(cudaStream_t s, const kb200_preprocess_desc& desc, const uint8_t* base, size_t stride, uint32_t batch, void* dst, int out) {
    return with_out_format(out, [&](auto o) {
        return launch_preprocess<decltype(o)::value>(s, plain_desc(desc), yuv_matrix(desc), nullptr, base, stride, batch, dst);
    });
}

template <int OUT>
static int preprocess_entry(kb200_stream_t stream, const kb200_preprocess_desc* raw_desc, const uint8_t* const* frames,
                            const size_t* frame_len, const uint8_t* base, size_t base_len, size_t stride,
                            uint32_t batch, void* dst, size_t dst_len) {
    KB200_TRY(validate_desc(raw_desc));
    const kb200_preprocess_desc plain = plain_desc(*raw_desc);
    const kb200_preprocess_desc* desc = &plain;
    const SrcFormat f = src_format(desc->fmt);
    KB200_TRY(check_ptr("dst", dst));
    if (batch == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "batch must be non-zero");
    const size_t need = src_bytes(*desc);
    // 16-bit samples: every frame must start 2-byte aligned
    if (f.words && !frames && ((reinterpret_cast<uintptr_t>(base) & 1u) || (batch > 1 && (stride & 1u))))
        return fail(KB200_ERR_INVALID_SOURCE, "%s frames must start 2-byte aligned (base %p, stride %zu)", f.name, (const void*)base, stride);
    if (frames) {
        KB200_TRY(check_frame_table(*desc, frames, frame_len, batch));
    } else {
        KB200_TRY(check_ptr("base", base));
        if (stride < need && batch > 1) return fail(KB200_ERR_INVALID_SOURCE, "frame stride %zu smaller than a frame (%zu bytes)", stride, need);
        if (base_len < (size_t)(batch - 1) * stride + need)
            return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source at %dx%d (got %zu bytes, need %zu)", desc->src_w, desc->src_h, base_len, (size_t)(batch - 1) * stride + need);
    }
    // BatchMismatch / BadOutputShape: dst must hold [batch,3,H,W]
    KB200_TRY(check_slice("dst", dst_len, (size_t)batch * 3 * desc->dst_w * desc->dst_h));
    return launch_preprocess<OUT>(as_stream(stream), *desc, yuv_matrix(*raw_desc), frames, base, stride, batch, dst);
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

KB200_API size_t kb200_preprocess_src_bytes(const kb200_preprocess_desc* desc) { return desc ? src_bytes(plain_desc(*desc)) : 0; }

KB200_API int kb200_preprocess_f32(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames,
                                   const size_t* frame_len, uint32_t batch, float* dst, size_t dst_len) {
    if (!frames) return fail(KB200_ERR_INVALID_ARGUMENT, "null pointer for 'frames'");
    return preprocess_entry<KB200_OUT_F32>(stream, desc, frames, frame_len, nullptr, 0, 0, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_f16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames,
                                   const size_t* frame_len, uint32_t batch, uint16_t* dst, size_t dst_len) {
    if (!frames) return fail(KB200_ERR_INVALID_ARGUMENT, "null pointer for 'frames'");
    return preprocess_entry<KB200_OUT_F16>(stream, desc, frames, frame_len, nullptr, 0, 0, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_bf16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames,
                                    const size_t* frame_len, uint32_t batch, uint16_t* dst, size_t dst_len) {
    if (!frames) return fail(KB200_ERR_INVALID_ARGUMENT, "null pointer for 'frames'");
    return preprocess_entry<KB200_OUT_BF16>(stream, desc, frames, frame_len, nullptr, 0, 0, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_strided_f32(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* base,
                                           size_t base_len, size_t frame_stride, uint32_t batch, float* dst, size_t dst_len) {
    return preprocess_entry<KB200_OUT_F32>(stream, desc, nullptr, nullptr, base, base_len, frame_stride, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_strided_f16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* base,
                                           size_t base_len, size_t frame_stride, uint32_t batch, uint16_t* dst, size_t dst_len) {
    return preprocess_entry<KB200_OUT_F16>(stream, desc, nullptr, nullptr, base, base_len, frame_stride, batch, dst, dst_len);
}
KB200_API int kb200_preprocess_strided_bf16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* base,
                                            size_t base_len, size_t frame_stride, uint32_t batch, uint16_t* dst, size_t dst_len) {
    return preprocess_entry<KB200_OUT_BF16>(stream, desc, nullptr, nullptr, base, base_len, frame_stride, batch, dst, dst_len);
}

}  // extern "C"
