// preprocess_roi.cu — kb200_preprocess_rois: crop-and-resize many regions of interest of a set of frames, for every
// source format, in one launch per ROI_CHUNK regions.  Region i = (frame k, x, y, w, h) is sampled as the batch entries
// (preprocess.cu) sample a w x h frame with kb200_preprocess_affine(mode, w, h, dst_w, dst_h): the inside test and the tap
// clamps are the region's, and every tap is offset by the region's origin, so it decodes at frame coordinates (the
// demosaic neighbourhood and the chroma siting are the frame's, not the crop's).  The taps, the Lanczos weight, the
// divisions and the stores are preprocess.cuh's, shared with preprocess.cu; the two sampler bodies below are
// preprocess_generic_kernel's and preprocess_yuv_kernel's, op for op, with the region's extent and origin.  (Those kernels
// keep their own copies: routing them through these bodies changes ptxas's register assignment in 63 of their
// instantiations, and their SASS is kept identical.)
//
// Kernels: the fast 4:2:0 / 4:4:4 resampler (yuv_resample) as preprocess_{nv12,nv21,i420,yv12,p01x,i01x,i444,i41x}_roi_kernel
// under the batch entries' yuv420_fast rule without its geometry terms, and the generic per-pixel body as
// preprocess_roi_generic_kernel for everything else (Lanczos, Bayer, 4:2:2, RGB / BGR / Gray, unaligned destinations).
#include <cstring>

#include "preprocess.cuh"

namespace kb200 {

// One region as its kernels get it, resolved and checked on the host: its frame, its rectangle in that frame and its affine.
struct PreRoi {
    const uint8_t* src;
    float scale_x, scale_y, pad_x, pad_y;
    int32_t x, y, w, h;
};
// Regions per launch.  They travel by value in the kernel parameter block (as PreFrames carries frame pointers), which stays
// within the classic 4 KB limit with the descriptor and the other arguments.
static constexpr uint32_t ROI_CHUNK = 80;
struct PreRois {
    PreRoi r[ROI_CHUNK];
};
static_assert(sizeof(PreRoi) == 40, "PreRoi is 40 bytes");
static_assert(sizeof(kb200_preprocess_desc) + sizeof(PreRois) + sizeof(Nv12Args) + sizeof(SrcFormat) + sizeof(Yuv16Coeffs) + 16 <= 4096,
              "the region kernels' parameters must fit the classic 4 KB parameter block");

// One region's geometry as the sampler bodies below read it: its affine (sx, sy: the source coordinate of an output column
// / row, IEEE), its extent w x h (the inside test and the tap clamps) and its origin (x0, y0) in the frame, which every tap
// is offset by, so that taps decode at frame coordinates.
struct RoiGeom {
    const PreRoi& r;
    __device__ __forceinline__ float sx(int ox) const { return __fdiv_rn((float)ox - r.pad_x, r.scale_x); }
    __device__ __forceinline__ float sy(int oy) const { return __fdiv_rn((float)oy - r.pad_y, r.scale_y); }
    __device__ __forceinline__ int w() const { return r.w; }
    __device__ __forceinline__ int h() const { return r.h; }
    __device__ __forceinline__ int x0() const { return r.x; }
    __device__ __forceinline__ int y0() const { return r.y; }
};

// The region generic kernel's pixel: output pixel (ox, oy) of region g of the frame at src, sampled with SAMP (kb200_interp —
// 0 nearest, 1 bilinear, 3 Lanczos-3: 6x6 taps, clamp-to-edge, weights renormalised by their sum) and normalised into o.
template <int SAMP, int TAP>
__device__ __forceinline__ void generic_pixel(const uint8_t* __restrict__ src, int ox, int oy, const kb200_preprocess_desc& d, const SrcFormat& sf,
                                              const TapCoeffs<TAP>& yc, const RoiGeom& g, float o[3]) {
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

// preprocess_yuv_kernel's resampler for one region: the 4 output columns ox0 .. ox0 + 3 of the NV12_ROWS rows from
// blockIdx.y * NV12_ROWS of output image `img`, sampled from region geo of the frame at src.  The
// frame's w x h (the descriptor's) address its planes in yuv_tap; geo's extent sets the inside test and the clamps.
// L: a 4:2:0 layout or YUV444 (yuv_tap); T: the sample type (YuvSample).  A pixel of 16-bit words is normalised as
// (px / W - mean) * inv_std with the IEEE division, interpolated or not.
template <int OUT, bool BILINEAR, int L, typename T>
__device__ __forceinline__ void yuv_resample(const RoiGeom& geo, const uint8_t* __restrict__ src, const kb200_preprocess_desc& d, const Nv12Args& na,
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
        // The row side reads the region's pad_y, scale_y, h and y afresh each row, through a pointer the compiler cannot
        // prove loop-invariant, so that none of them is held in a register across the calls the sy and sx divisions may
        // make: held, they were saved to local memory and reloaded on every row (NV12 f32 bilinear: 8 B stores, 12 B loads).
        const PreRoi* rr = &geo.r;
        asm volatile("" : "+l"(rr));
        const float sy = __fdiv_rn((float)oy - rr->pad_y, rr->scale_y);
        const int rh = rr->h, ry = rr->y;
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

// One thread per output pixel of region roi0 + blockIdx.y.
template <int OUT, int SAMP, int TAP>
__global__ void __launch_bounds__(256) preprocess_roi_generic_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                     const __grid_constant__ PreRois rs, void* __restrict__ dst, uint32_t roi0,
                                                                     const SrcFormat sf, const TapCoeffs<TAP> yc) {
    const int pixels = d.dst_w * d.dst_h;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pixels) return;
    const PreRoi& r = rs.r[blockIdx.y];
    const int ox = i % d.dst_w, oy = i / d.dst_w;
    float o[3];
    generic_pixel<SAMP, TAP>(r.src, ox, oy, d, sf, yc, RoiGeom{r}, o);
    generic_store<OUT>(dst, (size_t)(roi0 + blockIdx.y) * 3 * pixels + i, pixels, o);
}

// preprocess_yuv_kernel with per-region geometry: one thread = 4 columns x NV12_ROWS rows of region roi0 + blockIdx.z.
template <int OUT, bool BILINEAR, int L, typename T>
__global__ void __launch_bounds__(128) preprocess_yuv_roi_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                 const __grid_constant__ PreRois rs, const __grid_constant__ Nv12Args na,
                                                                 void* __restrict__ dst, uint32_t roi0, const typename YuvSample<T>::Coeffs yc) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= na.groups) return;
    const PreRoi& r = rs.r[blockIdx.z];
    yuv_resample<OUT, BILINEAR, L, T>(RoiGeom{r}, r.src, d, na, dst, roi0 + blockIdx.z, (int)g * 4, yc);
}

// kb200_last_kernel() name of the fast region kernel of a format with fast kernels (SrcFormat::fast_kernel)
static const char* roi_fast_kernel(const SrcFormat& f) {
    static const char* const names[][2] = {
        {"preprocess_nv12_kernel", "preprocess_nv12_roi_kernel"}, {"preprocess_nv21_kernel", "preprocess_nv21_roi_kernel"},
        {"preprocess_i420_kernel", "preprocess_i420_roi_kernel"}, {"preprocess_yv12_kernel", "preprocess_yv12_roi_kernel"},
        {"preprocess_p01x_kernel", "preprocess_p01x_roi_kernel"}, {"preprocess_i01x_kernel", "preprocess_i01x_roi_kernel"},
        {"preprocess_i444_kernel", "preprocess_i444_roi_kernel"}, {"preprocess_i41x_kernel", "preprocess_i41x_roi_kernel"},
    };
    if (!f.fast_kernel) return nullptr;
    for (const auto& n : names)
        if (!strcmp(n[0], f.fast_kernel)) return n[1];
    return nullptr;
}

// d: a validated descriptor with the plain format code; frames and rois: checked by the entry
template <int OUT>
static int launch_rois(cudaStream_t s, const kb200_preprocess_desc& d, int matrix, int mode, const uint8_t* const* frames, uint32_t n_frames,
                       const kb200_roi* rois, uint32_t n_rois, void* dst) {
    const SrcFormat f = src_format(d.fmt);
    const bool lanczos = d.sampling == KB200_INTERP_LANCZOS, bil = d.sampling == KB200_INTERP_BILINEAR;
    // the batch entries' yuv420_fast rule without its geometry terms: vector stores need dst_w % 4 == 0 and a 16-B aligned
    // destination; the NV12 / NV21 tap reads a chroma pair as one 16-bit word, so their frames must all start 2-B aligned
    const bool pair_loads = f.family == SRC_YUV420 && !f.words && (f.layout == YUV420_NV12 || f.layout == YUV420_NV21);
    bool frames_even = true;
    for (uint32_t k = 0; k < n_frames; ++k) frames_even = frames_even && !(reinterpret_cast<uintptr_t>(frames[k]) & 1u);
    const char* fast = lanczos ? nullptr : roi_fast_kernel(f);
    const bool use_fast = fast && (d.dst_w % 4) == 0 && aligned16(dst) && d.dst_h <= 65535 * NV12_ROWS && (!pair_loads || frames_even);
    const YuvCoeffs& yc = YUV_COEFFS[matrix];
    const Yuv16Coeffs yc16 = yuv16_coeffs_of(f, matrix);   // used by the 16-bit 4:2:0 and 4:4:4 formats only
    const Nv12Args nv = nv12_args(d);
    const int pixels = d.dst_w * d.dst_h;
    for (uint32_t r0 = 0; r0 < n_rois; r0 += ROI_CHUNK) {
        const uint32_t nr = std::min<uint32_t>(ROI_CHUNK, n_rois - r0);
        PreRois rs{};
        for (uint32_t j = 0; j < nr; ++j) {
            const kb200_roi& q = rois[r0 + j];
            float a[4];
            kb200_preprocess_affine(mode, (uint32_t)q.w, (uint32_t)q.h, (uint32_t)d.dst_w, (uint32_t)d.dst_h, a);
            rs.r[j] = PreRoi{frames[q.frame], a[0], a[1], a[2], a[3], q.x, q.y, q.w, q.h};
        }
        if (use_fast) {
            const dim3 grid(div_up(nv.groups, 128), div_up((size_t)d.dst_h, NV12_ROWS), nr);
            with_yuv_layout(f, yc, yc16, [&](auto l, auto t, const auto& c) {
                constexpr int L = decltype(l)::value;
                using T = decltype(t);
                if (bil) preprocess_yuv_roi_kernel<OUT, true, L, T><<<grid, 128, 0, s>>>(d, rs, nv, dst, r0, c);
                else preprocess_yuv_roi_kernel<OUT, false, L, T><<<grid, 128, 0, s>>>(d, rs, nv, dst, r0, c);
            });
            KB200_TRY(check_launch(fast));
            continue;
        }
        const dim3 grid(div_up(pixels, 256), nr);
        with_tap(f, yc, yc16, [&](auto tap, const auto& c) {
            constexpr int TAP = decltype(tap)::value;
            if (lanczos) preprocess_roi_generic_kernel<OUT, KB200_INTERP_LANCZOS, TAP><<<grid, 256, 0, s>>>(d, rs, dst, r0, f, c);
            else if (bil) preprocess_roi_generic_kernel<OUT, KB200_INTERP_BILINEAR, TAP><<<grid, 256, 0, s>>>(d, rs, dst, r0, f, c);
            else preprocess_roi_generic_kernel<OUT, KB200_INTERP_NEAREST, TAP><<<grid, 256, 0, s>>>(d, rs, dst, r0, f, c);
        });
        KB200_TRY(check_launch("preprocess_roi_generic_kernel"));
    }
    return KB200_OK;
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_preprocess_rois(kb200_stream_t stream, const kb200_preprocess_desc* desc, int mode, const uint8_t* const* frames,
                                    const size_t* frame_len, uint32_t n_frames, const kb200_roi* rois, uint32_t n_rois, void* dst,
                                    size_t dst_len, int out_format) {
    if (!desc) return fail(KB200_ERR_INVALID_ARGUMENT, "null preprocess descriptor");
    kb200_preprocess_desc raw = *desc;   // each region gets its own affine: the descriptor's scale and pad are not used
    raw.scale_x = raw.scale_y = 1.0f;
    raw.pad_x = raw.pad_y = 0.0f;
    KB200_TRY(validate_desc(&raw));
    if (mode != 0 && mode != 1) return fail(KB200_ERR_INVALID_ARGUMENT, "unknown resize mode %d (expected 0 Letterbox or 1 Stretch)", mode);
    if (out_format != KB200_OUT_F32 && out_format != KB200_OUT_F16 && out_format != KB200_OUT_BF16)
        return fail(KB200_ERR_INVALID_ARGUMENT, "unknown output format %d (expected 0 f32, 1 f16 or 2 bf16)", out_format);
    KB200_TRY(check_ptr("frames", frames));
    KB200_TRY(check_ptr("rois", rois));
    KB200_TRY(check_ptr("dst", dst));
    if (n_rois == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "n_rois must be non-zero");
    const kb200_preprocess_desc d = plain_desc(raw);
    const SrcFormat f = src_format(d.fmt);
    for (uint32_t i = 0; i < n_rois; ++i) {
        const kb200_roi& q = rois[i];
        if (q.frame < 0 || (uint32_t)q.frame >= n_frames)
            return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: frame index %d is outside [0, %u)", i, q.frame, n_frames);
        if (q.x < 0 || q.y < 0) return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: origin (%d, %d) is negative", i, q.x, q.y);
        if (q.w < 1 || q.h < 1) return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: size %dx%d is empty", i, q.w, q.h);
        if ((int64_t)q.x + q.w > d.src_w || (int64_t)q.y + q.h > d.src_h)
            return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: (%d, %d) + %dx%d reaches outside the %dx%d frame", i, q.x, q.y, q.w, q.h, d.src_w,
                        d.src_h);
    }
    const size_t need = src_bytes(d);
    for (uint32_t k = 0; k < n_frames; ++k) {
        if (!frames[k]) return fail(KB200_ERR_INVALID_ARGUMENT, "null frame pointer at index %u", k);
        if (f.words && (reinterpret_cast<uintptr_t>(frames[k]) & 1u)) return fail(KB200_ERR_INVALID_SOURCE, "%s frame %u is not 2-byte aligned", f.name, k);
        if (frame_len && frame_len[k] < need)
            return fail(KB200_ERR_INVALID_SOURCE, "invalid raw source at %dx%d (got %zu bytes, need %zu)", d.src_w, d.src_h, frame_len[k], need);
    }
    KB200_TRY(check_slice("dst", dst_len, (size_t)n_rois * 3 * d.dst_w * d.dst_h));
    const cudaStream_t s = as_stream(stream);
    const int m = yuv_matrix(raw);
    if (out_format == KB200_OUT_F16) return launch_rois<KB200_OUT_F16>(s, d, m, mode, frames, n_frames, rois, n_rois, dst);
    if (out_format == KB200_OUT_BF16) return launch_rois<KB200_OUT_BF16>(s, d, m, mode, frames, n_frames, rois, n_rois, dst);
    return launch_rois<KB200_OUT_F32>(s, d, m, mode, frames, n_frames, rois, n_rois, dst);
}

}  // extern "C"
