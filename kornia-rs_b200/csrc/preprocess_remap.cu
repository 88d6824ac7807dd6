// preprocess_remap.cu — kb200_preprocess_remap: a set of frames resampled through dense per-pixel coordinate maps (lens
// undistortion, rig rectification, fisheye dewarping into pinhole views), for every source format, in one launch per
// REMAP_CHUNK regions.  Region i = (frame k, map j): output pixel (ox, oy) reads x = map_x[j][oy][ox] and
// y = map_y[j][oy][ox], frame coordinates with pixel centres at integers (remap.cu's and cv2.remap's convention).  It is
// inside iff 0 <= x < src_w && 0 <= y < src_h in f32 (NaN and +-inf are outside); an inside pixel is sampled and
// normalised by preprocess.cuh's generic_pixel through a WarpPoint, the body every preprocess kernel shares, so taps decode
// at frame coordinates; an outside pixel takes the normalised pad value.
//
// Kernels: preprocess_remap_kernel (4 adjacent output columns per thread: one 16-B float4 load per map, lane-contiguous
// nv12_store4 stores) when dst_w % 4 == 0, both maps are 16-B aligned and dst is 16-B (f32) / 8-B (f16, bf16) aligned;
// preprocess_remap_generic_kernel (one thread per pixel, generic_store) otherwise.  Nearest and Bilinear only.
//
// Block order: the region is the fastest-varying part of the block index, so consecutive blocks read the same span of a
// map for different regions, and regions that share a map find it in L2 rather than re-reading it from HBM per frame (a
// 1080p map pair is 16.6 MB; the outputs streaming past it would evict it between regions in a region-major order).
#include "preprocess.cuh"

namespace kb200 {

// One region as its kernels get it, resolved on the host: its frame and the element offset of its map in map_x / map_y.
struct PreMap {
    const uint8_t* src;
    uint64_t map;
};
// Regions per launch.  They travel by value in the kernel parameter block, which stays within the classic 4 KB limit with
// the descriptor and the other arguments.
static constexpr uint32_t REMAP_CHUNK = 192;
struct PreMaps {
    PreMap r[REMAP_CHUNK];
};
static_assert(sizeof(PreMap) == 16, "PreMap is 16 bytes");
static_assert(sizeof(kb200_preprocess_desc) + sizeof(PreMaps) + sizeof(SrcFormat) + sizeof(Yuv16Coeffs) + 3 * sizeof(void*) + 8 <= 4096,
              "the remap kernels' parameters must fit the classic 4 KB parameter block");

// Block b of a launch of nr regions: region b % nr, block b / nr of that region's output.
__device__ __forceinline__ uint32_t block_region(uint32_t nr) { return blockIdx.x % nr; }
__device__ __forceinline__ uint32_t region_block(uint32_t nr) { return blockIdx.x / nr; }

// The output pixel whose map entry is (x, y) in frame src, normalised into o.
template <int SAMP, int TAP>
__device__ __forceinline__ void remap_pixel(const uint8_t* __restrict__ src, float x, float y, const kb200_preprocess_desc& d, const SrcFormat& sf,
                                            const TapCoeffs<TAP>& yc, float o[3]) {
    const bool inside = x >= 0.0f && x < (float)d.src_w && y >= 0.0f && y < (float)d.src_h;
    const WarpPoint p{inside ? x : -1.0f, inside ? y : -1.0f, d.src_w, d.src_h};
    generic_pixel<SAMP, TAP>(src, 0, 0, d, sf, yc, p, o);
}

// Output columns 4g .. 4g + 3 of one row: thread i of the region is group i of its plane, whose first element is 4i.
template <int OUT, int SAMP, int TAP>
__global__ void __launch_bounds__(256) preprocess_remap_kernel(const __grid_constant__ kb200_preprocess_desc d, const __grid_constant__ PreMaps ms,
                                                               uint32_t nr, const float* __restrict__ map_x, const float* __restrict__ map_y,
                                                               void* __restrict__ dst, uint32_t r0, const SrcFormat sf, const TapCoeffs<TAP> yc) {
    const uint32_t r = block_region(nr);
    const uint32_t i = region_block(nr) * blockDim.x + threadIdx.x;
    if (i >= (uint32_t)d.dst_w / 4u * (uint32_t)d.dst_h) return;
    const PreMap& m = ms.r[r];
    const size_t e = (size_t)i * 4;
    const float4 mx = __ldg(reinterpret_cast<const float4*>(map_x + m.map + e));
    const float4 my = __ldg(reinterpret_cast<const float4*>(map_y + m.map + e));
    const float xs[4] = {mx.x, mx.y, mx.z, mx.w}, ys[4] = {my.x, my.y, my.z, my.w};
    float o[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float p[3];
        remap_pixel<SAMP, TAP>(m.src, xs[j], ys[j], d, sf, yc, p);
        o[0][j] = p[0]; o[1][j] = p[1]; o[2][j] = p[2];
    }
    const size_t plane = (size_t)d.dst_w * d.dst_h;
    const size_t obase = (size_t)(r0 + r) * 3 * plane + e;
    nv12_store4<OUT>(dst, obase, o[0]);
    nv12_store4<OUT>(dst, obase + plane, o[1]);
    nv12_store4<OUT>(dst, obase + 2 * plane, o[2]);
}

// One thread per output pixel.
template <int OUT, int SAMP, int TAP>
__global__ void __launch_bounds__(256) preprocess_remap_generic_kernel(const __grid_constant__ kb200_preprocess_desc d, const __grid_constant__ PreMaps ms,
                                                                       uint32_t nr, const float* __restrict__ map_x, const float* __restrict__ map_y,
                                                                       void* __restrict__ dst, uint32_t r0, const SrcFormat sf, const TapCoeffs<TAP> yc) {
    const uint32_t r = block_region(nr);
    const int pixels = d.dst_w * d.dst_h;
    const int i = (int)(region_block(nr) * blockDim.x + threadIdx.x);
    if (i >= pixels) return;
    const PreMap& m = ms.r[r];
    float o[3];
    remap_pixel<SAMP, TAP>(m.src, __ldg(map_x + m.map + i), __ldg(map_y + m.map + i), d, sf, yc, o);
    generic_store<OUT>(dst, (size_t)(r0 + r) * 3 * pixels + i, pixels, o);
}

// d: a validated descriptor with the plain format code; frames, maps and regions: checked by the entry
template <int OUT>
static int launch_remap(cudaStream_t s, const kb200_preprocess_desc& d, int matrix, const uint8_t* const* frames, const float* map_x,
                        const float* map_y, const kb200_remap_roi* regions, uint32_t n_regions, void* dst) {
    const SrcFormat f = src_format(d.fmt);
    const bool bil = d.sampling == KB200_INTERP_BILINEAR;
    // the vector kernel's rule: its stores' (vector_dst_ok), and maps its float4 loads can address (every map then starts
    // 16-B aligned too: a map is dst_w * dst_h floats)
    const bool vec = vector_dst_ok(d, dst, OUT) && aligned16(map_x) && aligned16(map_y);
    const YuvCoeffs& yc = YUV_COEFFS[matrix];
    const Yuv16Coeffs yc16 = yuv16_coeffs_of(f, matrix);   // used by the 16-bit YUV formats only
    const size_t plane = (size_t)d.dst_w * d.dst_h;
    const unsigned blocks = div_up(vec ? plane / 4 : plane, 256);   // per region
    for (uint32_t r0 = 0; r0 < n_regions; r0 += REMAP_CHUNK) {
        const uint32_t nr = std::min<uint32_t>(REMAP_CHUNK, n_regions - r0);
        PreMaps ms{};
        for (uint32_t j = 0; j < nr; ++j) {
            ms.r[j].src = frames[regions[r0 + j].frame];
            ms.r[j].map = (uint64_t)regions[r0 + j].map * plane;
        }
        const unsigned grid = nr * blocks;   // < 2^31: plane < 2^31 (validate_desc) and nr <= REMAP_CHUNK
        with_tap(f, yc, yc16, [&](auto tap, const auto& c) {
            constexpr int TAP = decltype(tap)::value;
            if (vec) {
                if (bil) preprocess_remap_kernel<OUT, KB200_INTERP_BILINEAR, TAP><<<grid, 256, 0, s>>>(d, ms, nr, map_x, map_y, dst, r0, f, c);
                else preprocess_remap_kernel<OUT, KB200_INTERP_NEAREST, TAP><<<grid, 256, 0, s>>>(d, ms, nr, map_x, map_y, dst, r0, f, c);
            } else {
                if (bil) preprocess_remap_generic_kernel<OUT, KB200_INTERP_BILINEAR, TAP><<<grid, 256, 0, s>>>(d, ms, nr, map_x, map_y, dst, r0, f, c);
                else preprocess_remap_generic_kernel<OUT, KB200_INTERP_NEAREST, TAP><<<grid, 256, 0, s>>>(d, ms, nr, map_x, map_y, dst, r0, f, c);
            }
        });
        KB200_TRY(check_launch(vec ? "preprocess_remap_kernel" : "preprocess_remap_generic_kernel"));
    }
    return KB200_OK;
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_preprocess_remap(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames, const size_t* frame_len,
                                     uint32_t n_frames, const float* map_x, const float* map_y, size_t map_len, uint32_t n_maps,
                                     const kb200_remap_roi* regions, uint32_t n_regions, void* dst, size_t dst_len, int out_format) {
    kb200_preprocess_desc raw, d;
    KB200_TRY(check_region_call(desc, nullptr, "remapped regions", out_format, &raw, &d));
    KB200_TRY(check_ptr("frames", frames));
    KB200_TRY(check_ptr("regions", regions));
    KB200_TRY(check_ptr("map_x", map_x));
    KB200_TRY(check_ptr("map_y", map_y));
    KB200_TRY(check_ptr("dst", dst));
    if (n_regions == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "n_regions must be non-zero");
    if (n_maps == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "n_maps must be non-zero");
    if (!aligned4(map_x) || !aligned4(map_y)) return fail(KB200_ERR_INVALID_ARGUMENT, "map_x and map_y must be 4-byte aligned float arrays");
    for (uint32_t i = 0; i < n_regions; ++i) {
        const kb200_remap_roi& q = regions[i];
        KB200_TRY(check_region_frame(i, q.frame, n_frames));
        if (q.map < 0 || (uint32_t)q.map >= n_maps)
            return fail(KB200_ERR_INVALID_ARGUMENT, "region %u: map index %d is outside [0, %u)", i, q.map, n_maps);
    }
    KB200_TRY(check_frame_table(d, frames, frame_len, n_frames));
    const size_t plane = (size_t)d.dst_w * d.dst_h;   // < 2^31 (validate_desc), so the products below fit 64 bits
    KB200_TRY(check_slice("map", map_len, (size_t)n_maps * plane));
    KB200_TRY(check_slice("dst", dst_len, (size_t)n_regions * 3 * plane));
    return with_out_format(out_format, [&](auto o) {
        return launch_remap<decltype(o)::value>(as_stream(stream), d, yuv_matrix(raw), frames, map_x, map_y, regions, n_regions, dst);
    });
}

}  // extern "C"
