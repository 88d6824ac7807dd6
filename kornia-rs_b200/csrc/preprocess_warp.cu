// preprocess_warp.cu — kb200_preprocess_warps: rotated and perspective crops of a set of frames, one forward 2x3 or 3x3
// map per region, for every source format, in one launch per WARP_CHUNK regions.  Region i = (frame k, M), M a forward
// row-major 3x3 map from frame pixel coordinates to output pixel coordinates (cv2.warpAffine / warpPerspective without
// WARP_INVERSE_MAP; pixel centres at integer coordinates).  Its inverse is computed on the host: affine when
// M[6..8] == (0, 0, 1) (kb200_invert_affine_transform of the first two rows), perspective otherwise
// (kb200_invert_homography).  Output pixel (ox, oy) takes its source coordinate and its inside test from warp_coord
// (warp_common.cuh, the f32 warps' rule) on the region's inverse against the frame's src_w x src_h, and is then sampled and
// normalised by preprocess.cuh's sample_pixel over the whole frame (FrameGeom's extent and origin), the body every
// preprocess kernel shares: taps decode at frame coordinates, so the demosaic neighbourhood and the chroma siting are the
// frame's.  Outside pixels take the normalised pad value.
//
// Kernels: preprocess_warp_kernel (4 adjacent output columns per thread, lane-contiguous nv12_store4 stores) when
// dst_w % 4 == 0 and dst is 16-B (f32) / 8-B (f16, bf16) aligned; preprocess_warp_generic_kernel (one thread per pixel,
// generic_store) for every other destination.  Nearest and Bilinear only.
#include <cmath>

#include "preprocess.cuh"
#include "warp_common.cuh"

namespace kb200 {

// One region as its kernels get it, resolved and checked on the host: its frame and its inverse map (frame coordinates of
// an output pixel), affine in m[0..5] or perspective in m[0..8].
struct PreWarp {
    const uint8_t* src;
    float m[9];
    int32_t perspective;
};
// Regions per launch.  They travel by value in the kernel parameter block (as PreRois does), which stays within the classic
// 4 KB limit with the descriptor and the other arguments.
static constexpr uint32_t WARP_CHUNK = 72;
struct PreWarps {
    PreWarp r[WARP_CHUNK];
};
static_assert(sizeof(PreWarp) == 48, "PreWarp is 48 bytes");
static_assert(sizeof(kb200_preprocess_desc) + sizeof(PreWarps) + sizeof(SrcFormat) + sizeof(Yuv16Coeffs) + 16 <= 4096,
              "the warp kernels' parameters must fit the classic 4 KB parameter block");

// The largest float below the positive integer n.
__device__ __forceinline__ float below(int n) { return __int_as_float(__float_as_int((float)n) - 1); }

// Output pixel (ox, oy) of region r, normalised into o, sampled through WarpPoint (preprocess.cuh) at the coordinate
// warp_coord gives it.  warp_coord's degenerate-axis rule judges an axis whose step is
// below 1e-6 on its row constant, so an inside coordinate can sit a hair outside [0, src_w) x [0, src_h); it is clamped
// into [0, below(src_w)] x [0, below(src_h)] before sampling, which leaves every other inside coordinate as it is.  The
// clamped value samples what its nearest frame pixel holds: x0 = x1 = W - 1 above W - 1, and nearest rounds it to W - 1.
template <int SAMP, int TAP>
__device__ __forceinline__ void warp_pixel(const PreWarp& r, int ox, int oy, const kb200_preprocess_desc& d, const SrcFormat& sf,
                                           const TapCoeffs<TAP>& yc, float o[3]) {
    float sx = 0.0f, sy = 0.0f;
    const bool inside = r.perspective ? warp_coord<true>(r.m, (uint32_t)ox, (uint32_t)oy, (uint32_t)d.src_w, (uint32_t)d.src_h, &sx, &sy)
                                      : warp_coord<false>(r.m, (uint32_t)ox, (uint32_t)oy, (uint32_t)d.src_w, (uint32_t)d.src_h, &sx, &sy);
    const WarpPoint p{inside ? fminf(fmaxf(sx, 0.0f), below(d.src_w)) : -1.0f, inside ? fminf(fmaxf(sy, 0.0f), below(d.src_h)) : -1.0f,
                      d.src_w, d.src_h};
    generic_pixel<SAMP, TAP>(r.src, ox, oy, d, sf, yc, p, o);
}

// Output columns 4g .. 4g + 3 of one row of region w0 + blockIdx.z: thread i of the region is row i / (dst_w / 4), group
// i % (dst_w / 4).
template <int OUT, int SAMP, int TAP>
__global__ void __launch_bounds__(256) preprocess_warp_kernel(const __grid_constant__ kb200_preprocess_desc d, const __grid_constant__ PreWarps ws,
                                                              void* __restrict__ dst, uint32_t w0, const SrcFormat sf, const TapCoeffs<TAP> yc) {
    const uint32_t groups = (uint32_t)d.dst_w / 4u;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= groups * (uint32_t)d.dst_h) return;
    const PreWarp& r = ws.r[blockIdx.z];
    const int oy = (int)(i / groups), ox0 = (int)(i % groups) * 4;
    const size_t plane = (size_t)d.dst_w * d.dst_h;
    const size_t obase = (size_t)(w0 + blockIdx.z) * 3 * plane + (size_t)oy * d.dst_w + ox0;
    float o[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float p[3];
        warp_pixel<SAMP, TAP>(r, ox0 + j, oy, d, sf, yc, p);
        o[0][j] = p[0]; o[1][j] = p[1]; o[2][j] = p[2];
    }
    nv12_store4<OUT>(dst, obase, o[0]);
    nv12_store4<OUT>(dst, obase + plane, o[1]);
    nv12_store4<OUT>(dst, obase + 2 * plane, o[2]);
}

// One thread per output pixel of region w0 + blockIdx.z.
template <int OUT, int SAMP, int TAP>
__global__ void __launch_bounds__(256) preprocess_warp_generic_kernel(const __grid_constant__ kb200_preprocess_desc d,
                                                                      const __grid_constant__ PreWarps ws, void* __restrict__ dst, uint32_t w0,
                                                                      const SrcFormat sf, const TapCoeffs<TAP> yc) {
    const int pixels = d.dst_w * d.dst_h;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= pixels) return;
    float o[3];
    warp_pixel<SAMP, TAP>(ws.r[blockIdx.z], i % d.dst_w, i / d.dst_w, d, sf, yc, o);
    generic_store<OUT>(dst, (size_t)(w0 + blockIdx.z) * 3 * pixels + i, pixels, o);
}

// Region i's inverse map into inv (9 entries; an affine one fills 0..5 and the row 0, 0, 1), perspective or not, or the
// refusal naming the region: non-finite entries (KB200_ERR_INVALID_ARGUMENT), a singular map or a non-finite inverse
// (KB200_ERR_SINGULAR_MATRIX).
static int invert_warp(uint32_t i, const kb200_warp_roi& q, float inv[9], bool* perspective) {
    for (int j = 0; j < 9; ++j)
        if (!std::isfinite(q.m[j])) return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: matrix entry %d is not finite", i, j);
    *perspective = !(q.m[6] == 0.0f && q.m[7] == 0.0f && q.m[8] == 1.0f);
    if (*perspective) {
        if (kb200_invert_homography(q.m, inv) != KB200_OK)
            return fail(KB200_ERR_SINGULAR_MATRIX, "region %u: the perspective map is singular (|det_norm| < 1e-10)", i);
    } else {
        if (q.m[0] * q.m[4] - q.m[1] * q.m[3] == 0.0f)   // kb200_invert_affine_transform's determinant; it returns zeros for 0
            return fail(KB200_ERR_SINGULAR_MATRIX, "region %u: the affine map is singular (zero determinant)", i);
        kb200_invert_affine_transform(q.m, inv);
        inv[6] = 0.0f; inv[7] = 0.0f; inv[8] = 1.0f;
    }
    for (int j = 0; j < 9; ++j)
        if (!std::isfinite(inv[j])) return fail(KB200_ERR_SINGULAR_MATRIX, "region %u: the inverse map has a non-finite entry %d", i, j);
    return KB200_OK;
}

// d: a validated descriptor with the plain format code; frames and warps: checked by the entry
template <int OUT>
static int launch_warps(cudaStream_t s, const kb200_preprocess_desc& d, int matrix, const uint8_t* const* frames, const kb200_warp_roi* warps,
                        uint32_t n_warps, void* dst) {
    const SrcFormat f = src_format(d.fmt);
    const bool bil = d.sampling == KB200_INTERP_BILINEAR;
    const bool vec = vector_dst_ok(d, dst, OUT);
    const YuvCoeffs& yc = YUV_COEFFS[matrix];
    const Yuv16Coeffs yc16 = yuv16_coeffs_of(f, matrix);   // used by the 16-bit YUV formats only
    const size_t items = vec ? (size_t)(d.dst_w / 4) * d.dst_h : (size_t)d.dst_w * d.dst_h;
    for (uint32_t r0 = 0; r0 < n_warps; r0 += WARP_CHUNK) {
        const uint32_t nr = std::min<uint32_t>(WARP_CHUNK, n_warps - r0);
        PreWarps ws{};
        for (uint32_t j = 0; j < nr; ++j) {
            bool persp = false;
            KB200_TRY(invert_warp(r0 + j, warps[r0 + j], ws.r[j].m, &persp));   // checked by the entry: cannot fail here
            ws.r[j].src = frames[warps[r0 + j].frame];
            ws.r[j].perspective = persp;
        }
        const dim3 grid(div_up(items, 256), 1, nr);   // a region's blocks are adjacent: its source footprint stays in L2
        with_tap(f, yc, yc16, [&](auto tap, const auto& c) {
            constexpr int TAP = decltype(tap)::value;
            if (vec) {
                if (bil) preprocess_warp_kernel<OUT, KB200_INTERP_BILINEAR, TAP><<<grid, 256, 0, s>>>(d, ws, dst, r0, f, c);
                else preprocess_warp_kernel<OUT, KB200_INTERP_NEAREST, TAP><<<grid, 256, 0, s>>>(d, ws, dst, r0, f, c);
            } else {
                if (bil) preprocess_warp_generic_kernel<OUT, KB200_INTERP_BILINEAR, TAP><<<grid, 256, 0, s>>>(d, ws, dst, r0, f, c);
                else preprocess_warp_generic_kernel<OUT, KB200_INTERP_NEAREST, TAP><<<grid, 256, 0, s>>>(d, ws, dst, r0, f, c);
            }
        });
        KB200_TRY(check_launch(vec ? "preprocess_warp_kernel" : "preprocess_warp_generic_kernel"));
    }
    return KB200_OK;
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_preprocess_warps(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames, const size_t* frame_len,
                                     uint32_t n_frames, const kb200_warp_roi* warps, uint32_t n_warps, void* dst, size_t dst_len, int out_format) {
    kb200_preprocess_desc raw, d;
    KB200_TRY(check_region_call(desc, nullptr, "warped regions", out_format, &raw, &d));
    KB200_TRY(check_ptr("frames", frames));
    KB200_TRY(check_ptr("warps", warps));
    KB200_TRY(check_ptr("dst", dst));
    if (n_warps == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "n_warps must be non-zero");
    for (uint32_t i = 0; i < n_warps; ++i) {
        KB200_TRY(check_region_frame(i, warps[i].frame, n_frames));
        float inv[9];
        bool persp;
        KB200_TRY(invert_warp(i, warps[i], inv, &persp));
    }
    KB200_TRY(check_frame_table(d, frames, frame_len, n_frames));
    KB200_TRY(check_slice("dst", dst_len, (size_t)n_warps * 3 * d.dst_w * d.dst_h));
    return with_out_format(out_format, [&](auto o) {
        return launch_warps<decltype(o)::value>(as_stream(stream), d, yuv_matrix(raw), frames, warps, n_warps, dst);
    });
}

}  // extern "C"
