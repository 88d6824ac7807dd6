// distortion.cu — undistort / rectify map generation on the device (SURVEY §8(f) #2): the producer of the maps `remap`
// consumes, i.e. the real "undistort" caller next to BASELINE config 5.
//
// Reference: calibration/distortion.rs:60-103 `distort_point_polynomial` (Brown-Conrady rational model, f64, plain
// mul/add/div — this file is compiled with -fmad=false, which also forbids f64 contraction), :135-150
// `generate_correction_map_polynomial` (one evaluation per destination pixel, result cast to f32, two H x W x 1 maps).
// The reference builds the maps on the host and uploads them; here they are written in place on the device by one
// kernel, ready for kb200_remap_* on the same stream.  f64 throughput is irrelevant: the map is generated once per
// camera, 2 x 8 bytes of output per pixel.
#include "kb200_common.cuh"

namespace kb200 {

// intr: the camera the map distorts with (fx, fy, cx, cy); out: the camera of the output pixels (fx', fy', cx', cy'), intr
// itself for the reference's map.
struct DistortArgs { double intr[4]; double dist[8]; double out[4]; };

__global__ void __launch_bounds__(256) correction_map_kernel(float* __restrict__ map_x, float* __restrict__ map_y, uint32_t w, uint32_t h,
                                                             const __grid_constant__ DistortArgs A) {
    const uint32_t px = blockIdx.x * 32u + threadIdx.x, py = blockIdx.y * 8u + threadIdx.y;
    if (px >= w || py >= h) return;
    const double fx = A.intr[0], fy = A.intr[1], cx = A.intr[2], cy = A.intr[3];
    const double k1 = A.dist[0], k2 = A.dist[1], k3 = A.dist[2], k4 = A.dist[3], k5 = A.dist[4], k6 = A.dist[5], p1 = A.dist[6], p2 = A.dist[7];
    const double x = __ddiv_rn((double)px - A.out[2], A.out[0]);
    const double y = __ddiv_rn((double)py - A.out[3], A.out[1]);
    const double r2 = x * x + y * y;
    const double r4 = r2 * r2;
    const double r6 = r4 * r2;
    const double kr = __ddiv_rn(1.0 + k1 * r2 + k2 * r4 + k3 * r6, 1.0 + k4 * r2 + k5 * r4 + k6 * r6);
    const double x_2 = 2.0 * x, y_2 = 2.0 * y;
    const double xy_2 = x_2 * y;
    const double xd = x * kr + xy_2 * p1 + p2 * (r2 + x_2 * x);
    const double yd = y * kr + p1 * (r2 + y_2 * y) + xy_2 * p2;
    const size_t o = (size_t)py * w + px;
    map_x[o] = (float)(fx * xd + cx);
    map_y[o] = (float)(fy * yd + cy);
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_generate_correction_map_polynomial_to(kb200_stream_t stream, const double intrinsic[4], const double distortion[8],
                                                          const double new_intrinsic[4], uint32_t width, uint32_t height, float* map_x,
                                                          float* map_y, size_t map_len) {
    KB200_TRY(check_ptr("intrinsic", intrinsic)); KB200_TRY(check_ptr("distortion", distortion)); KB200_TRY(check_ptr("new_intrinsic", new_intrinsic));
    KB200_TRY(check_ptr("map_x", map_x)); KB200_TRY(check_ptr("map_y", map_y));
    if (width == 0 || height == 0) return fail(KB200_ERR_INVALID_ARGUMENT, "image dimensions must be non-zero");
    KB200_TRY(check_slice("map", map_len, (size_t)width * height));
    DistortArgs A;
    for (int i = 0; i < 4; ++i) A.intr[i] = intrinsic[i];
    for (int i = 0; i < 8; ++i) A.dist[i] = distortion[i];
    for (int i = 0; i < 4; ++i) A.out[i] = new_intrinsic[i];
    correction_map_kernel<<<dim3(div_up(width, 32), div_up(height, 8)), dim3(32, 8), 0, as_stream(stream)>>>(map_x, map_y, width, height, A);
    return check_launch("correction_map_kernel");
}

KB200_API int kb200_generate_correction_map_polynomial(kb200_stream_t stream, const double intrinsic[4], const double distortion[8], uint32_t width,
                                                       uint32_t height, float* map_x, float* map_y, size_t map_len) {
    return kb200_generate_correction_map_polynomial_to(stream, intrinsic, distortion, intrinsic, width, height, map_x, map_y, map_len);
}

}  // extern "C"
