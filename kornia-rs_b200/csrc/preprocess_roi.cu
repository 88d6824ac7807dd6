// preprocess_roi.cu — kb200_preprocess_rois: crop-and-resize many regions of interest of a set of frames, for every
// source format, in one launch per ROI_CHUNK regions.  Region i = (frame k, x, y, w, h) is sampled as the batch entries
// (preprocess.cu) sample a w x h frame with kb200_preprocess_affine(mode, w, h, dst_w, dst_h): the inside test and the tap
// clamps are the region's, and every tap is offset by the region's origin, so it decodes at frame coordinates (the
// demosaic neighbourhood and the chroma siting are the frame's, not the crop's).  The sampler bodies, the taps and the
// stores are preprocess.cuh's, shared with preprocess.cu's kernels; here they read the region's geometry (RoiGeom).
//
// Kernels: the fast 4:2:0 / 4:4:4 resampler (yuv_resample) as preprocess_{nv12,nv21,i420,yv12,p01x,i01x,i444,i41x}_roi_kernel
// under the batch entries' rule (yuv_resampler_ok), and the generic per-pixel body as preprocess_roi_generic_kernel for
// everything else (Lanczos, Bayer, 4:2:2, RGB / BGR / Gray, unaligned destinations).
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

// One region's geometry for the sampler bodies (preprocess.cuh): its affine, its extent w x h and its origin in the frame.
struct RoiGeom {
    const PreRoi& r;
    __device__ __forceinline__ float sx(int ox) const { return __fdiv_rn((float)ox - r.pad_x, r.scale_x); }
    __device__ __forceinline__ float sy(int oy) const { return __fdiv_rn((float)oy - r.pad_y, r.scale_y); }
    __device__ __forceinline__ int w() const { return r.w; }
    __device__ __forceinline__ int h() const { return r.h; }
    __device__ __forceinline__ int x0() const { return r.x; }
    __device__ __forceinline__ int y0() const { return r.y; }
    // yuv_resample's row side reads the region's pad_y, scale_y, h and y afresh each row, through a pointer the compiler
    // cannot prove loop-invariant, so that none of them is held in a register across the calls the sy and sx divisions may
    // make: held, they were saved to local memory and reloaded on every row (NV12 f32 bilinear: 8 B stores, 12 B loads).
    __device__ __forceinline__ GeomRow row(int oy) const {
        const PreRoi* rr = &r;
        asm volatile("" : "+l"(rr));
        return {__fdiv_rn((float)oy - rr->pad_y, rr->scale_y), rr->h, rr->y};
    }
};

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
    const bool use_fast = yuv_resampler_ok(f, d, dst, frames_aligned(frames, nullptr, 0, n_frames, 2));
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
            KB200_TRY(check_launch(roi_fast_kernel(f)));
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
    kb200_preprocess_desc raw, d;
    KB200_TRY(check_region_call(desc, &mode, nullptr, out_format, &raw, &d));
    KB200_TRY(check_ptr("frames", frames));
    KB200_TRY(check_ptr("rois", rois));
    KB200_TRY(check_ptr("dst", dst));
    if (n_rois == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "n_rois must be non-zero");
    for (uint32_t i = 0; i < n_rois; ++i) {
        const kb200_roi& q = rois[i];
        KB200_TRY(check_region_frame(i, q.frame, n_frames));
        if (q.x < 0 || q.y < 0) return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: origin (%d, %d) is negative", i, q.x, q.y);
        if (q.w < 1 || q.h < 1) return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: size %dx%d is empty", i, q.w, q.h);
        if ((int64_t)q.x + q.w > d.src_w || (int64_t)q.y + q.h > d.src_h)
            return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: (%d, %d) + %dx%d reaches outside the %dx%d frame", i, q.x, q.y, q.w, q.h, d.src_w,
                        d.src_h);
    }
    KB200_TRY(check_frame_table(d, frames, frame_len, n_frames));
    KB200_TRY(check_slice("dst", dst_len, (size_t)n_rois * 3 * d.dst_w * d.dst_h));
    return with_out_format(out_format, [&](auto o) {
        return launch_rois<decltype(o)::value>(as_stream(stream), d, yuv_matrix(raw), mode, frames, n_frames, rois, n_rois, dst);
    });
}

}  // extern "C"
