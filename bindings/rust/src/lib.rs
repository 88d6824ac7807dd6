//! `kornia-b200-sys`: the Rust side of the drop-in boundary.
//!
//! * `ffi` — the `extern "C"` block, 1:1 with `include/kornia_b200.h`.
//! * safe wrappers whose names, argument order and error behaviour equal the reference launchers they
//!   replace (`crates/kornia-imgproc/src/cuda/*.rs`), so the residency adapters
//!   (`resize/cuda.rs:34`, `warp/cuda.rs:29,65`, `filter/cuda.rs:106,185`, `color/cuda_dispatch.rs:49`,
//!   `preprocess.rs:1324`) can call them without any other change.
//!
//! Not compiled in the build container (no Rust toolchain there); kept reviewable and mechanically derived
//! from the header.  The ctypes binding in `kornia-rs_b200/_lib.py` is the binding that IS exercised by the
//! tests and carries the same signatures.
#![allow(clippy::too_many_arguments)]

use std::ffi::{c_char, c_int, c_void, CStr};
use std::sync::Arc;

use cudarc::driver::{CudaContext, CudaSlice, CudaStream, DevicePtr, DevicePtrMut};

pub mod ffi {
    use super::*;

    /// Opaque staging ring of the host-buffer entry points (include/kornia_b200.h, kb200_host_pipeline).
    #[repr(C)]
    pub struct kb200_host_pipeline {
        _private: [u8; 0],
    }

    /// include/kornia_b200.h `kb200_preprocess_desc` — 20 four-byte fields, 80 bytes, C layout.
    #[repr(C)]
    #[derive(Clone, Copy, Debug, Default)]
    pub struct kb200_preprocess_desc {
        pub scale_x: f32,
        pub scale_y: f32,
        pub pad_x: f32,
        pub pad_y: f32,
        pub src_w: i32,
        pub src_h: i32,
        pub src_pitch: i32,
        pub src_bpp: i32,
        pub fmt: i32,
        pub dst_w: i32,
        pub dst_h: i32,
        pub mean: [f32; 3],
        pub inv_std: [f32; 3],
        pub pad_value: f32,
        pub sampling: i32,
    }

    const _: () = assert!(std::mem::size_of::<kb200_preprocess_desc>() == 80);

    /// include/kornia_b200.h `kb200_roi` — region (x, y, w, h) of frame `frame`, 20 bytes, C layout.
    #[repr(C)]
    #[derive(Clone, Copy, Debug, Default)]
    pub struct kb200_roi {
        pub frame: i32,
        pub x: i32,
        pub y: i32,
        pub w: i32,
        pub h: i32,
    }

    const _: () = assert!(std::mem::size_of::<kb200_roi>() == 20);

    /// include/kornia_b200.h `kb200_warp_roi` — frame `frame` through the forward map `m` (row-major 3x3, frame -> output
    /// pixel coordinates), 40 bytes, C layout.
    #[repr(C)]
    #[derive(Clone, Copy, Debug, Default)]
    pub struct kb200_warp_roi {
        pub frame: i32,
        pub m: [f32; 9],
    }

    const _: () = assert!(std::mem::size_of::<kb200_warp_roi>() == 40);

    /// include/kornia_b200.h `kb200_remap_roi` — frame `frame` resampled through map `map` of the call's map arrays,
    /// 8 bytes, C layout.
    #[repr(C)]
    #[derive(Clone, Copy, Debug, Default)]
    pub struct kb200_remap_roi {
        pub frame: i32,
        pub map: i32,
    }

    const _: () = assert!(std::mem::size_of::<kb200_remap_roi>() == 8);

    extern "C" {
        pub fn kb200_version() -> c_int;
        pub fn kb200_last_kernel() -> *const c_char;
        pub fn kb200_debug_set_knob(name: *const c_char, value: c_int) -> c_int;
        pub fn kb200_last_error() -> *const c_char;
        pub fn kb200_status_name(status: c_int) -> *const c_char;
        pub fn kb200_set_device(ordinal: c_int) -> c_int;
        pub fn kb200_device_info(sm_count: *mut c_int, cc_major: *mut c_int, cc_minor: *mut c_int) -> c_int;

        pub fn kb200_resize_bilinear_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize,
                                            src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, mapping: c_int) -> c_int;
        pub fn kb200_resize_nearest_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize,
                                           src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, mapping: c_int) -> c_int;
        pub fn kb200_resize_bilinear_normalize_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32,
                                                      dst_len: usize, src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32,
                                                      mean: *const f32, std: *const f32, mapping: c_int) -> c_int;
        pub fn kb200_resize_f32(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, src_w: u32,
                                src_h: u32, dst_w: u32, dst_h: u32, channels: u32, batch: u32, interp: c_int) -> c_int;
        pub fn kb200_resize_normalize_chw_u8_f32(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut f32, dst_len: usize,
                                                 src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, scale: *const f32,
                                                 bias: *const f32, leaf: c_int) -> c_int;
        pub fn kb200_resize_normalize_chw_u8_f16(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u16, dst_len: usize,
                                                 src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, scale: *const f32,
                                                 bias: *const f32, leaf: c_int) -> c_int;
        pub fn kb200_resize_normalize_chw_u8_bf16(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u16, dst_len: usize,
                                                  src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, scale: *const f32,
                                                  bias: *const f32, leaf: c_int) -> c_int;
        pub fn kb200_resize_row_plan(src_h: u32, dst_h: u32, period: *mut u32, first: *mut u32, keep: *mut u32);
        pub fn kb200_resize_normalize_chw_u8_f32_rows(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut f32, dst_len: usize,
                                                      src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, scale: *const f32,
                                                      bias: *const f32, leaf: c_int, row_period: u32, row_first: u32, row_keep: u32) -> c_int;
        pub fn kb200_host_pipeline_create(device: c_int, src_chunk_bytes: usize, dst_chunk_bytes: usize, depth: c_int,
                                          out: *mut *mut kb200_host_pipeline) -> c_int;
        pub fn kb200_host_pipeline_destroy(pipeline: *mut kb200_host_pipeline);
        pub fn kb200_host_pipeline_last_transfer(pipeline: *const kb200_host_pipeline, h2d_bytes: *mut u64, d2h_bytes: *mut u64) -> c_int;
        pub fn kb200_host_register(ptr: *mut c_void, bytes: usize) -> c_int;
        pub fn kb200_host_unregister(ptr: *mut c_void) -> c_int;
        pub fn kb200_resize_normalize_chw_u8_host(pipeline: *mut kb200_host_pipeline, stream: *mut c_void, host_src: *const u8,
                                                  src_len: usize, host_dst: *mut c_void, dst_len: usize, src_w: u32, src_h: u32,
                                                  dst_w: u32, dst_h: u32, batch: u32, scale: *const f32, bias: *const f32,
                                                  leaf: c_int, out_format: c_int) -> c_int;
        pub fn kb200_resize_normalize_chw_u8_f32_host(pipeline: *mut kb200_host_pipeline, stream: *mut c_void, host_src: *const u8,
                                                      src_len: usize, host_dst: *mut f32, dst_len: usize, src_w: u32, src_h: u32,
                                                      dst_w: u32, dst_h: u32, batch: u32, scale: *const f32, bias: *const f32,
                                                      leaf: c_int) -> c_int;
        pub fn kb200_resize_bilinear_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, src_w: u32,
                                        src_h: u32, dst_w: u32, dst_h: u32, channels: u32, batch: u32) -> c_int;
        pub fn kb200_resize_fast_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, src_w: u32, src_h: u32,
                                    dst_w: u32, dst_h: u32, channels: u32, batch: u32, interp: c_int) -> c_int;
        pub fn kb200_yuyv_from_rgb_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32) -> c_int;
        pub fn kb200_nv12_from_rgb_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32) -> c_int;
        pub fn kb200_warp_affine_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, src_w: u32, src_h: u32,
                                    dst_w: u32, dst_h: u32, channels: u32, batch: u32, m: *const f32) -> c_int;
        pub fn kb200_warp_perspective_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, src_w: u32,
                                         src_h: u32, dst_w: u32, dst_h: u32, channels: u32, batch: u32, h: *const f32) -> c_int;
        pub fn kb200_quantize_kernel_256(kernel: *const f32, n: u32, out: *mut u8);
        pub fn kb200_gaussian_blur_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, cols: u32, rows: u32,
                                      channels: u32, batch: u32, ksize_x: u32, ksize_y: u32, sigma_x: f32, sigma_y: f32) -> c_int;
        pub fn kb200_box_blur_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, cols: u32, rows: u32,
                                 channels: u32, batch: u32, ksize_x: u32, ksize_y: u32) -> c_int;
        pub fn kb200_remap_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, map_x: *const f32,
                                  map_y: *const f32, map_len: usize, src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, interp: c_int) -> c_int;
        pub fn kb200_remap_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, map_x: *const f32,
                              map_y: *const f32, map_len: usize, src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, channels: u32, batch: u32,
                              interp: c_int) -> c_int;
        pub fn kb200_warp_affine_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, src_w: u32,
                                        src_h: u32, dst_w: u32, dst_h: u32, batch: u32, m: *const f32, interp: c_int) -> c_int;
        pub fn kb200_warp_perspective_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize,
                                             src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32, h: *const f32, interp: c_int) -> c_int;
        pub fn kb200_invert_affine_transform(m: *const f32, out: *mut f32);
        pub fn kb200_invert_homography(h: *const f32, out: *mut f32) -> c_int;
        pub fn kb200_get_rotation_matrix2d(cx: f32, cy: f32, angle_deg: f32, scale: f32, out: *mut f32);
        pub fn kb200_separable_filter_f32(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize,
                                          scratch: *mut f32, kx: *const f32, kx_len: u32, ky: *const f32, ky_len: u32, cols: u32,
                                          rows: u32, channels: u32, batch: u32) -> c_int;
        pub fn kb200_gaussian_blur_f32(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, cols: u32,
                                       rows: u32, channels: u32, batch: u32, ksize_x: u32, ksize_y: u32, sigma_x: f32, sigma_y: f32) -> c_int;
        pub fn kb200_sobel_f32(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, cols: u32, rows: u32,
                               channels: u32, batch: u32, ksize: u32) -> c_int;
        pub fn kb200_gradient_magnitude_f32(stream: *mut c_void, gx: *const f32, gy: *const f32, dst: *mut f32, n: usize) -> c_int;
        pub fn kb200_gaussian_kernel_1d(ksize: u32, sigma: f32, out: *mut f32);
        pub fn kb200_gaussian_resolve(kx_in: u32, ky_in: u32, sx_in: f32, sy_in: f32, kx: *mut u32, ky: *mut u32, sx: *mut f32, sy: *mut f32) -> c_int;
        pub fn kb200_gray_from_rgb_f32(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, npixels: usize, leaf: c_int) -> c_int;
        pub fn kb200_gray_from_rgb_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, npixels: usize) -> c_int;
        pub fn kb200_rgb_from_nv12_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32) -> c_int;
        pub fn kb200_rgb_from_yuyv_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32) -> c_int;
        pub fn kb200_rgb_from_yuv420_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32, layout: c_int) -> c_int;
        pub fn kb200_rgb_from_yuv422_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32, layout: c_int) -> c_int;
        pub fn kb200_rgb_from_yuv420_u8_matrix(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32, layout: c_int, matrix: c_int) -> c_int;
        pub fn kb200_rgb_from_yuv422_u8_matrix(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32, layout: c_int, matrix: c_int) -> c_int;
        pub fn kb200_rgb_from_bayer_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32, pattern: c_int) -> c_int;
        pub fn kb200_rgb_from_bayer_u16(stream: *mut c_void, src: *const u16, src_len: usize, dst: *mut u16, dst_len: usize, width: u32, height: u32, batch: u32, pattern: c_int) -> c_int;
        pub fn kb200_rgb_from_bayer_packed(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u16, dst_len: usize, width: u32, height: u32, batch: u32, pattern: c_int, bits: c_int) -> c_int;
        pub fn kb200_rgb_from_yuv420_u16(stream: *mut c_void, src: *const u16, src_len: usize, dst: *mut u16, dst_len: usize, width: u32, height: u32, batch: u32, layout: c_int, bits: c_int, matrix: c_int) -> c_int;
        pub fn kb200_rgb_from_yuv444_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, width: u32, height: u32, batch: u32, matrix: c_int) -> c_int;
        pub fn kb200_rgb_from_yuv444_u16(stream: *mut c_void, src: *const u16, src_len: usize, dst: *mut u16, dst_len: usize, width: u32, height: u32, batch: u32, layout: c_int, bits: c_int, matrix: c_int) -> c_int;
        pub fn kb200_normalize_mean_std_f32(stream: *mut c_void, src: *const f32, dst: *mut f32, npixels: usize, channels: u32, mean: *const f32, std: *const f32) -> c_int;
        pub fn kb200_normalize_rgb_u8_f32(stream: *mut c_void, src: *const u8, dst: *mut f32, npixels: usize, scale: *const f32, offset: *const f32, leaf: c_int) -> c_int;
        pub fn kb200_find_min_max_f32(stream: *mut c_void, src: *const f32, n: usize, minmax_dev: *mut f32) -> c_int;
        pub fn kb200_normalize_min_max_f32(stream: *mut c_void, src: *const f32, dst: *mut f32, n: usize, min: f32, max: f32, minmax_dev: *const f32) -> c_int;
        pub fn kb200_std_mean_u8_c3(stream: *mut c_void, src: *const u8, npixels: usize, sums_dev: *mut u64) -> c_int;
        pub fn kb200_std_mean_finalize(sums: *const u64, npixels: usize, std_out: *mut f64, mean_out: *mut f64);
        pub fn kb200_preprocess_affine(mode: c_int, src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, out_scale_pad: *mut f32);
        pub fn kb200_preprocess_src_bytes(desc: *const kb200_preprocess_desc) -> usize;
        pub fn kb200_preprocess_f32(stream: *mut c_void, desc: *const kb200_preprocess_desc, frames: *const *const u8, frame_len: *const usize, batch: u32, dst: *mut f32, dst_len: usize) -> c_int;
        pub fn kb200_preprocess_f16(stream: *mut c_void, desc: *const kb200_preprocess_desc, frames: *const *const u8, frame_len: *const usize, batch: u32, dst: *mut u16, dst_len: usize) -> c_int;
        pub fn kb200_preprocess_strided_f32(stream: *mut c_void, desc: *const kb200_preprocess_desc, base: *const u8, base_len: usize, frame_stride: usize, batch: u32, dst: *mut f32, dst_len: usize) -> c_int;
        pub fn kb200_preprocess_strided_f16(stream: *mut c_void, desc: *const kb200_preprocess_desc, base: *const u8, base_len: usize, frame_stride: usize, batch: u32, dst: *mut u16, dst_len: usize) -> c_int;
        pub fn kb200_preprocess_bf16(stream: *mut c_void, desc: *const kb200_preprocess_desc, frames: *const *const u8, frame_len: *const usize, batch: u32, dst: *mut u16, dst_len: usize) -> c_int;
        pub fn kb200_preprocess_strided_bf16(stream: *mut c_void, desc: *const kb200_preprocess_desc, base: *const u8, base_len: usize, frame_stride: usize, batch: u32, dst: *mut u16, dst_len: usize) -> c_int;
        pub fn kb200_preprocess_rois(stream: *mut c_void, desc: *const kb200_preprocess_desc, mode: c_int, frames: *const *const u8, frame_len: *const usize, n_frames: u32, rois: *const kb200_roi, n_rois: u32, dst: *mut c_void, dst_len: usize, out_format: c_int) -> c_int;
        pub fn kb200_preprocess_warps(stream: *mut c_void, desc: *const kb200_preprocess_desc, frames: *const *const u8, frame_len: *const usize, n_frames: u32, warps: *const kb200_warp_roi, n_warps: u32, dst: *mut c_void, dst_len: usize, out_format: c_int) -> c_int;
        pub fn kb200_preprocess_remap(stream: *mut c_void, desc: *const kb200_preprocess_desc, frames: *const *const u8, frame_len: *const usize, n_frames: u32, map_x: *const f32, map_y: *const f32, map_len: usize, n_maps: u32, regions: *const kb200_remap_roi, n_regions: u32, dst: *mut c_void, dst_len: usize, out_format: c_int) -> c_int;
        pub fn kb200_selftest_div255(stream: *mut c_void, mismatches_dev: *mut u64) -> c_int;
        pub fn kb200_selftest_div2(stream: *mut c_void, count: u64, seed: u32, mismatches_dev: *mut u64) -> c_int;

        // round 2: bicubic / Lanczos resize, pyramids, undistort maps, fusion pipelines, host-buffer preprocess
        pub fn kb200_resize_bicubic_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, src_w: u32,
                                           src_h: u32, dst_w: u32, dst_h: u32, batch: u32) -> c_int;
        pub fn kb200_resize_lanczos_scratch_len(src_h: u32, dst_w: u32, dst_h: u32, batch: u32) -> usize;
        pub fn kb200_resize_lanczos_f32_c3(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize,
                                           scratch: *mut f32, scratch_len: usize, src_w: u32, src_h: u32, dst_w: u32, dst_h: u32, batch: u32) -> c_int;
        pub fn kb200_pyrdown_f32(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, src_w: u32, src_h: u32,
                                 channels: u32, batch: u32) -> c_int;
        pub fn kb200_pyrup_f32(stream: *mut c_void, src: *const f32, src_len: usize, dst: *mut f32, dst_len: usize, src_w: u32, src_h: u32,
                               channels: u32, batch: u32) -> c_int;
        pub fn kb200_pyrdown_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, src_w: u32, src_h: u32,
                                channels: u32, batch: u32) -> c_int;
        pub fn kb200_pyrup_u8(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut u8, dst_len: usize, src_w: u32, src_h: u32,
                              channels: u32, batch: u32) -> c_int;
        pub fn kb200_generate_correction_map_polynomial(stream: *mut c_void, intrinsic: *const f64, distortion: *const f64, width: u32,
                                                        height: u32, map_x: *mut f32, map_y: *mut f32, map_len: usize) -> c_int;
        pub fn kb200_generate_correction_map_polynomial_to(stream: *mut c_void, intrinsic: *const f64, distortion: *const f64,
                                                           new_intrinsic: *const f64, width: u32, height: u32, map_x: *mut f32,
                                                           map_y: *mut f32, map_len: usize) -> c_int;
        pub fn kb200_fused_pipeline_u8_f32(stream: *mut c_void, src: *const u8, src_len: usize, dst: *mut f32, dst_len: usize, src_w: u32,
                                           src_h: u32, dst_w: u32, dst_h: u32, batch: u32, maps: c_int, scale: *const f32, bias: *const f32,
                                           sink: c_int) -> c_int;
        pub fn kb200_preprocess_host(pipeline: *mut kb200_host_pipeline, stream: *mut c_void, desc: *const kb200_preprocess_desc,
                                     host_base: *const u8, base_len: usize, frame_stride: usize, batch: u32, host_dst: *mut c_void,
                                     dst_len: usize, out_f16: c_int) -> c_int;
        pub fn kb200_preprocess_host_format(pipeline: *mut kb200_host_pipeline, stream: *mut c_void, desc: *const kb200_preprocess_desc,
                                            host_base: *const u8, base_len: usize, frame_stride: usize, batch: u32, host_dst: *mut c_void,
                                            dst_len: usize, out_format: c_int) -> c_int;
    }
}

/// Error type shared by the wrappers; the variants mirror the per-module `Cuda*Error` enums of the reference
/// (`define_cuda_error!`, cuda/mod.rs:96-148) so adapters keep their `map_err(|e| ImageError::Cuda(e.to_string()))`.
#[derive(Debug, thiserror::Error)]
pub enum Kb200Error {
    #[error("{0}")]
    Cuda(String),
    #[error("{0}")]
    SliceTooSmall(String),
    #[error("homography matrix is singular (|det| < 1e-10)")]
    SingularHomography,
}

fn check(status: c_int) -> Result<(), Kb200Error> {
    if status == 0 {
        return Ok(());
    }
    // SAFETY: kb200_last_error returns a thread-local NUL-terminated string valid until the next failing call.
    let msg = unsafe { CStr::from_ptr(ffi::kb200_last_error()) }.to_string_lossy().into_owned();
    Err(match status {
        -2 => Kb200Error::SliceTooSmall(msg),
        -3 => Kb200Error::SingularHomography,
        _ => Kb200Error::Cuda(msg),
    })
}

fn bind(ctx: &Arc<CudaContext>) -> Result<(), Kb200Error> {
    // the reference launchers take `ctx` to compile/launch on the right device; here it selects the device
    check(unsafe { ffi::kb200_set_device(ctx.ordinal() as c_int) })
}

/// `leaf` argument of the fused resize / normalize entry points: which CPU leaf's rounding is reproduced.
pub const LEAF_SCALAR: c_int = 0;
pub const LEAF_X86_AVX2_FMA: c_int = 1;
pub const LEAF_NEON: c_int = 2;

/// `out_format` of `kb200_resize_normalize_chw_u8_host` and `kb200_preprocess_host_format` (kb200_out_format): the CHW element type.  16-bit values are the
/// f32 result rounded once to nearest-even, stored as their raw bits.
pub const OUT_F32: c_int = 0;
pub const OUT_F16: c_int = 1;
pub const OUT_BF16: c_int = 2;

/// `fmt` of `kb200_preprocess_desc` (kb200_src_fmt).  Codes 5-9, 16-19 and 32-47 go beyond the reference's `SourceFormat`.
pub const FMT_RGB: i32 = 0;
pub const FMT_BGR: i32 = 1;
pub const FMT_GRAY: i32 = 2;
pub const FMT_NV12: i32 = 3;
pub const FMT_YUYV: i32 = 4;
pub const FMT_NV21: i32 = 5;
pub const FMT_I420: i32 = 6;
pub const FMT_YV12: i32 = 7;
pub const FMT_UYVY: i32 = 8;
pub const FMT_YVYU: i32 = 9;
pub const FMT_BAYER_RGGB: i32 = 16;
pub const FMT_BAYER_BGGR: i32 = 17;
pub const FMT_BAYER_GRBG: i32 = 18;
pub const FMT_BAYER_GBRG: i32 = 19;
/// 10- to 16-bit Bayer mosaics (one LSB-aligned u16 per sample): `FMT_BAYER16_BASE + 4 * k + pattern`, k = 0..3 for
/// 10, 12, 14 and 16 bits.
pub const FMT_BAYER16_BASE: i32 = 32;
pub const FMT_BAYER_RGGB10: i32 = 32;
pub const FMT_BAYER_RGGB12: i32 = 36;
pub const FMT_BAYER_RGGB14: i32 = 40;
pub const FMT_BAYER_RGGB16: i32 = 44;
/// The 10-, 12- and 14-bit mosaics MIPI CSI-2 packed (V4L2's SRGGB10P ... SGBRG14P, w * bits / 8 bytes per row):
/// `FMT_BAYER_PACKED_BASE + 4 * k + pattern`, k = 0..2 for 10, 12 and 14 bits.
pub const FMT_BAYER_PACKED_BASE: i32 = 64;
pub const FMT_BAYER_RGGB10P: i32 = 64;
pub const FMT_BAYER_RGGB12P: i32 = 68;
pub const FMT_BAYER_RGGB14P: i32 = 72;
/// 10- and 12-bit 4:2:0 video, tight frames of w * h * 3 / 2 little-endian u16 words: P010 / P012 (NV12's layout, the
/// code in the high bits) and I010 / I012 (I420's layout, the code in the low bits).  They take `fmt_yuv_matrix`.
pub const FMT_P010: i32 = 80;
pub const FMT_P012: i32 = 81;
pub const FMT_I010: i32 = 82;
pub const FMT_I012: i32 = 83;
/// 4:4:4 video, three full-resolution planes Y, U, V per tight frame: I444 (bytes, 3 * w * h), and I410 / I412 (16-bit
/// little-endian words, 6 * w * h bytes, the code in the low bits) and I410 / I412 MSB (the code in the high bits:
/// NVDEC's YUV444_16Bit surface).  Any w, h >= 1.  They take `fmt_yuv_matrix`.
pub const FMT_I444: i32 = 11;
pub const FMT_I410: i32 = 85;
pub const FMT_I412: i32 = 86;
pub const FMT_I410_MSB: i32 = 87;
pub const FMT_I412_MSB: i32 = 88;

/// `pattern` of `kb200_rgb_from_bayer_u8` (kb200_bayer_pattern): the mosaic's 2x2 quad read row-major.
pub const BAYER_RGGB: c_int = 0;
pub const BAYER_BGGR: c_int = 1;
pub const BAYER_GRBG: c_int = 2;
pub const BAYER_GBRG: c_int = 3;

/// `layout` of `kb200_rgb_from_yuv420_u8` (kb200_yuv420_layout): the chroma after the Y plane.
pub const YUV420_NV12: c_int = 0;
pub const YUV420_NV21: c_int = 1;
pub const YUV420_I420: c_int = 2;
pub const YUV420_YV12: c_int = 3;

/// `layout` of `kb200_rgb_from_yuv422_u8` (kb200_yuv422_layout): the byte order of each 2-pixel word.
pub const YUV422_YUYV: c_int = 0;
pub const YUV422_UYVY: c_int = 1;
pub const YUV422_YVYU: c_int = 2;

/// `layout` of `kb200_rgb_from_yuv420_u16` (kb200_yuv420_u16_layout): P010 / P012 (interleaved chroma, codes in the
/// high bits of each word) or I010 / I012 (U and V planes, codes in the low bits).
pub const YUV420_P01X: c_int = 0;
pub const YUV420_I01X: c_int = 1;

/// `layout` of `kb200_rgb_from_yuv444_u16` (kb200_yuv444_u16_layout): I410 / I412 (codes in the low bits of each word)
/// or their MSB-aligned form (codes in the high bits).
pub const YUV444_I41X: c_int = 0;
pub const YUV444_I41X_MSB: c_int = 1;

/// `matrix` of `kb200_rgb_from_yuv420_u8_matrix` / `_yuv422_u8_matrix` (kb200_yuv_matrix): the colour matrix and range a
/// YUV frame decodes with.  BT.601 limited is the reference's decode.
pub const YUV_BT601_LIMITED: c_int = 0;
pub const YUV_BT601_FULL: c_int = 1;
pub const YUV_BT709_LIMITED: c_int = 2;
pub const YUV_BT709_FULL: c_int = 3;

/// `KB200_FMT_YUV_MATRIX(m)`: OR it into a YUV format's `fmt` code of `kb200_preprocess_desc` to decode its frames with
/// matrix `m`.  Any other format with a matrix is rejected.
pub const fn fmt_yuv_matrix(matrix: c_int) -> i32 {
    matrix << 8
}

/// `PixelMapping` of cuda/resize.rs:441.
#[derive(Debug, Clone, Copy, PartialEq, Eq)]
pub enum PixelMapping {
    HalfPixel = 0,
    AlignCorners = 1,
}

/// Replaces `launch_resize_bilinear_downscale_cuda` (cuda/resize.rs:503).  `block_dim` is accepted and ignored
/// (grid shape is the kernel's business here).
pub fn launch_resize_bilinear_downscale_cuda(
    ctx: &Arc<CudaContext>, stream: &Arc<CudaStream>, src: &CudaSlice<f32>, dst: &mut CudaSlice<f32>,
    src_width: u32, src_height: u32, dst_width: u32, dst_height: u32, mapping: PixelMapping, _block_dim: Option<(u32, u32)>,
) -> Result<(), Kb200Error> {
    bind(ctx)?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_resize_bilinear_f32_c3(stream.cu_stream() as *mut c_void, sp as *const f32, src_len, dp as *mut f32, dst_len,
                                          src_width, src_height, dst_width, dst_height, 1, mapping as c_int)
    })
}

/// Replaces `launch_warp_perspective_bilinear_cuda` (cuda/warp_perspective.rs:480): forward homography in.
pub fn launch_warp_perspective_bilinear_cuda(
    ctx: &Arc<CudaContext>, stream: &Arc<CudaStream>, src: &CudaSlice<f32>, dst: &mut CudaSlice<f32>,
    src_width: u32, src_height: u32, dst_width: u32, dst_height: u32, h: &[f32; 9], _block_dim: Option<(u32, u32)>,
) -> Result<(), Kb200Error> {
    bind(ctx)?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_warp_perspective_f32_c3(stream.cu_stream() as *mut c_void, sp as *const f32, src_len, dp as *mut f32, dst_len,
                                           src_width, src_height, dst_width, dst_height, 1, h.as_ptr(), 1)
    })
}

/// Replaces `launch_warp_affine_bilinear_cuda` (cuda/warp_affine.rs:541): forward 2x3 in.
pub fn launch_warp_affine_bilinear_cuda(
    ctx: &Arc<CudaContext>, stream: &Arc<CudaStream>, src: &CudaSlice<f32>, dst: &mut CudaSlice<f32>,
    src_width: u32, src_height: u32, dst_width: u32, dst_height: u32, m: &[f32; 6], _block_dim: Option<(u32, u32)>,
) -> Result<(), Kb200Error> {
    bind(ctx)?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_warp_affine_f32_c3(stream.cu_stream() as *mut c_void, sp as *const f32, src_len, dp as *mut f32, dst_len,
                                      src_width, src_height, dst_width, dst_height, 1, m.as_ptr(), 1)
    })
}

/// Replaces `launch_separable_filter_f32` (cuda/filter.rs:361) at the adapter level (`filter/cuda.rs:106`): host taps in,
/// `scratch` no longer needed (the H+V passes are one kernel).
pub fn launch_separable_filter_f32(
    ctx: &Arc<CudaContext>, stream: &Arc<CudaStream>, src: &CudaSlice<f32>, dst: &mut CudaSlice<f32>,
    kx: &[f32], ky: &[f32], cols: u32, rows: u32, channels: u32,
) -> Result<(), Kb200Error> {
    bind(ctx)?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_separable_filter_f32(stream.cu_stream() as *mut c_void, sp as *const f32, src_len, dp as *mut f32, dst_len,
                                        std::ptr::null_mut(), kx.as_ptr(), kx.len() as u32, ky.as_ptr(), ky.len() as u32, cols, rows, channels, 1)
    })
}

/// Replaces `launch_rgb_from_planar420` (cuda/color/video.rs:328) with a choice of colour matrix: `batch` tight 4:2:0
/// frames of `layout` (`YUV420_*`) -> RGB8 HWC, decoded with `matrix` (`YUV_*`).
#[allow(clippy::too_many_arguments)]
pub fn launch_rgb_from_yuv420_matrix(
    stream: &Arc<CudaStream>, src: &CudaSlice<u8>, dst: &mut CudaSlice<u8>, width: u32, height: u32, batch: u32, layout: c_int, matrix: c_int,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_rgb_from_yuv420_u8_matrix(stream.cu_stream() as *mut c_void, sp as *const u8, src_len, dp as *mut u8, dst_len, width, height,
                                             batch, layout, matrix)
    })
}

/// Replaces `launch_rgb_from_packed422` (cuda/color/video.rs:297) with a choice of colour matrix: `batch` tight 4:2:2
/// frames of `layout` (`YUV422_*`) -> RGB8 HWC, decoded with `matrix` (`YUV_*`).
#[allow(clippy::too_many_arguments)]
pub fn launch_rgb_from_yuv422_matrix(
    stream: &Arc<CudaStream>, src: &CudaSlice<u8>, dst: &mut CudaSlice<u8>, width: u32, height: u32, batch: u32, layout: c_int, matrix: c_int,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_rgb_from_yuv422_u8_matrix(stream.cu_stream() as *mut c_void, sp as *const u8, src_len, dp as *mut u8, dst_len, width, height,
                                             batch, layout, matrix)
    })
}

/// An extension with no reference launcher: `batch` tight 8-bit 4:4:4 frames (I444: three w * h byte planes Y, U, V)
/// -> RGB8 HWC, decoded with `matrix` (`YUV_*`).
pub fn launch_rgb_from_yuv444_u8(
    stream: &Arc<CudaStream>, src: &CudaSlice<u8>, dst: &mut CudaSlice<u8>, width: u32, height: u32, batch: u32, matrix: c_int,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_rgb_from_yuv444_u8(stream.cu_stream() as *mut c_void, sp as *const u8, src_len, dp as *mut u8, dst_len, width, height, batch, matrix)
    })
}

/// An extension with no reference launcher: `batch` tight 10- or 12-bit (`bits`) 4:4:4 frames of 16-bit words in
/// `layout` (`YUV444_*`) -> RGB16 HWC holding the n-bit codes, decoded with `matrix` (`YUV_*`).  Lengths in elements.
#[allow(clippy::too_many_arguments)]
pub fn launch_rgb_from_yuv444_u16(
    stream: &Arc<CudaStream>, src: &CudaSlice<u16>, dst: &mut CudaSlice<u16>, width: u32, height: u32, batch: u32, layout: c_int, bits: c_int,
    matrix: c_int,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_rgb_from_yuv444_u16(stream.cu_stream() as *mut c_void, sp as *const u16, src_len, dp as *mut u16, dst_len, width, height,
                                       batch, layout, bits, matrix)
    })
}

/// Replaces `launch_gray_from_rgb_f32` (cuda/color/gray.rs:149).
pub fn launch_gray_from_rgb_f32(stream: &Arc<CudaStream>, src: &CudaSlice<f32>, dst: &mut CudaSlice<f32>, npixels: usize) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe { ffi::kb200_gray_from_rgb_f32(stream.cu_stream() as *mut c_void, sp as *const f32, src_len, dp as *mut f32, dst_len, npixels, 0) })
}

/// Replaces the per-frame loop of `Preprocessor::run_raw_batch_impl` + `launch_view` (preprocess.rs:1258-1282, :1324-1372):
/// one launch for the whole batch.
pub fn launch_preprocess_batch_f32(
    stream: &Arc<CudaStream>, desc: &ffi::kb200_preprocess_desc, frames: &[&CudaSlice<u8>], dst: &mut CudaSlice<f32>,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let mut guards = Vec::with_capacity(frames.len());
    let mut ptrs: Vec<*const u8> = Vec::with_capacity(frames.len());
    let lens: Vec<usize> = frames.iter().map(|f| f.len()).collect();
    for f in frames {
        let (p, g) = f.device_ptr(stream);
        ptrs.push(p as *const u8);
        guards.push(g);
    }
    let dst_len = dst.len();
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_preprocess_f32(stream.cu_stream() as *mut c_void, desc, ptrs.as_ptr(), lens.as_ptr(), frames.len() as u32, dp as *mut f32, dst_len)
    })
}

/// Crop-and-resize `rois` of `frames` into `dst` ([rois.len(), 3, dst_h, dst_w] f32) with `mode` (0 Letterbox, 1 Stretch):
/// one launch per 80 regions.  Replaces a caller's loop of one `launch_view` per crop (an extension beyond the reference).
pub fn launch_preprocess_rois(
    stream: &Arc<CudaStream>, desc: &ffi::kb200_preprocess_desc, mode: i32, frames: &[&CudaSlice<u8>], rois: &[ffi::kb200_roi],
    dst: &mut CudaSlice<f32>,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let mut guards = Vec::with_capacity(frames.len());
    let mut ptrs: Vec<*const u8> = Vec::with_capacity(frames.len());
    let lens: Vec<usize> = frames.iter().map(|f| f.len()).collect();
    for f in frames {
        let (p, g) = f.device_ptr(stream);
        ptrs.push(p as *const u8);
        guards.push(g);
    }
    let dst_len = dst.len();
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_preprocess_rois(stream.cu_stream() as *mut c_void, desc, mode, ptrs.as_ptr(), lens.as_ptr(), frames.len() as u32, rois.as_ptr(),
                                   rois.len() as u32, dp as *mut c_void, dst_len, 0)
    })
}

/// Rotated and perspective crops: `warps[i]` is frame `warps[i].frame` through its forward map (frame -> output pixel
/// coordinates), sampled into `dst` ([warps.len(), 3, dst_h, dst_w] f32) with the descriptor's sampling (Nearest or
/// Bilinear) and normalisation: one launch per 72 regions (an extension beyond the reference).
pub fn launch_preprocess_warps(
    stream: &Arc<CudaStream>, desc: &ffi::kb200_preprocess_desc, frames: &[&CudaSlice<u8>], warps: &[ffi::kb200_warp_roi],
    dst: &mut CudaSlice<f32>,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let mut guards = Vec::with_capacity(frames.len());
    let mut ptrs: Vec<*const u8> = Vec::with_capacity(frames.len());
    let lens: Vec<usize> = frames.iter().map(|f| f.len()).collect();
    for f in frames {
        let (p, g) = f.device_ptr(stream);
        ptrs.push(p as *const u8);
        guards.push(g);
    }
    let dst_len = dst.len();
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_preprocess_warps(stream.cu_stream() as *mut c_void, desc, ptrs.as_ptr(), lens.as_ptr(), frames.len() as u32, warps.as_ptr(),
                                    warps.len() as u32, dp as *mut c_void, dst_len, 0)
    })
}

/// Frames resampled through dense coordinate maps (lens undistortion, rig rectification): `regions[i]` is frame
/// `regions[i].frame` sampled at the coordinates of map `regions[i].map` of `map_x` / `map_y` ([n_maps, dst_h, dst_w] f32)
/// into `dst` ([regions.len(), 3, dst_h, dst_w] f32) with the descriptor's sampling (Nearest or Bilinear) and
/// normalisation; coordinates outside the frame take the pad value.  One launch per 192 regions (an extension beyond the
/// reference).
pub fn launch_preprocess_remap(
    stream: &Arc<CudaStream>, desc: &ffi::kb200_preprocess_desc, frames: &[&CudaSlice<u8>], map_x: &CudaSlice<f32>, map_y: &CudaSlice<f32>,
    n_maps: u32, regions: &[ffi::kb200_remap_roi], dst: &mut CudaSlice<f32>,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let mut guards = Vec::with_capacity(frames.len());
    let mut ptrs: Vec<*const u8> = Vec::with_capacity(frames.len());
    let lens: Vec<usize> = frames.iter().map(|f| f.len()).collect();
    for f in frames {
        let (p, g) = f.device_ptr(stream);
        ptrs.push(p as *const u8);
        guards.push(g);
    }
    let map_len = map_x.len().min(map_y.len());
    let (mx, _gx) = map_x.device_ptr(stream);
    let (my, _gy) = map_y.device_ptr(stream);
    let dst_len = dst.len();
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_preprocess_remap(stream.cu_stream() as *mut c_void, desc, ptrs.as_ptr(), lens.as_ptr(), frames.len() as u32, mx as *const f32,
                                    my as *const f32, map_len, n_maps, regions.as_ptr(), regions.len() as u32, dp as *mut c_void, dst_len, 0)
    })
}

/// Same as `launch_preprocess_batch_f32`, `dst` holding bfloat16 bits: each value the f32 result rounded to nearest even
/// (an extension beyond the reference, which writes f32 and f16 only).
pub fn launch_preprocess_batch_bf16(
    stream: &Arc<CudaStream>, desc: &ffi::kb200_preprocess_desc, frames: &[&CudaSlice<u8>], dst: &mut CudaSlice<u16>,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let mut guards = Vec::with_capacity(frames.len());
    let mut ptrs: Vec<*const u8> = Vec::with_capacity(frames.len());
    let lens: Vec<usize> = frames.iter().map(|f| f.len()).collect();
    for f in frames {
        let (p, g) = f.device_ptr(stream);
        ptrs.push(p as *const u8);
        guards.push(g);
    }
    let dst_len = dst.len();
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_preprocess_bf16(stream.cu_stream() as *mut c_void, desc, ptrs.as_ptr(), lens.as_ptr(), frames.len() as u32, dp as *mut u16, dst_len)
    })
}

/// `batch` frames at `frame_stride`-byte steps in `frames` (a capture ring buffer) -> [batch, 3, dst_h, dst_w] bfloat16 bits.
pub fn launch_preprocess_strided_bf16(
    stream: &Arc<CudaStream>, desc: &ffi::kb200_preprocess_desc, frames: &CudaSlice<u8>, frame_stride: usize, batch: u32,
    dst: &mut CudaSlice<u16>,
) -> Result<(), Kb200Error> {
    bind(stream.context())?;
    let (sp, _g0) = frames.device_ptr(stream);
    let (src_len, dst_len) = (frames.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_preprocess_strided_bf16(stream.cu_stream() as *mut c_void, desc, sp as *const u8, src_len, frame_stride, batch, dp as *mut u16,
                                           dst_len)
    })
}


/// Staging ring for the HOST-buffer form of `resize_normalize_to_tensor_u8_to_f32_bilinear` (resize/fused.rs:147):
/// host `&Image<u8,3>` in, host CHW tensor out, executed on the GPU.  One per device; calls only enqueue.
pub struct HostPipeline {
    raw: *mut ffi::kb200_host_pipeline,
}

// SAFETY: the pipeline owns CUDA streams/buffers that may be used from any thread; calls are serialised by &mut self.
unsafe impl Send for HostPipeline {}

impl HostPipeline {
    pub fn new(device: usize, src_chunk_bytes: usize, dst_chunk_bytes: usize, depth: usize) -> Result<Self, Kb200Error> {
        let mut raw = std::ptr::null_mut();
        check(unsafe { ffi::kb200_host_pipeline_create(device as c_int, src_chunk_bytes, dst_chunk_bytes, depth as c_int, &mut raw) })?;
        Ok(Self { raw })
    }

    /// `src`: `batch` tightly packed HWC u8 images; `dst`: [batch, 3, dst_h, dst_w] f32.  Both should be page-locked.
    /// Enqueue-only: synchronise `stream` before reading `dst`.
    #[allow(clippy::too_many_arguments)]
    pub fn resize_normalize_u8_to_f32(
        &mut self, stream: &Arc<CudaStream>, src: &[u8], src_size: (u32, u32), dst: &mut [f32], dst_size: (u32, u32), batch: u32,
        scale: &[f32; 3], bias: &[f32; 3],
    ) -> Result<(), Kb200Error> {
        check(unsafe {
            ffi::kb200_resize_normalize_chw_u8_f32_host(self.raw, stream.cu_stream() as *mut c_void, src.as_ptr(), src.len(),
                                                        dst.as_mut_ptr(), dst.len(), src_size.0, src_size.1, dst_size.0, dst_size.1,
                                                        batch, scale.as_ptr(), bias.as_ptr(), LEAF_X86_AVX2_FMA)
        })
    }

    /// Same as `resize_normalize_u8_to_f32`, `dst` holding IEEE binary16 bits: RNE of the f32 result (an extension beyond
    /// the reference, which writes f32 only).  The download moves half the bytes.
    #[allow(clippy::too_many_arguments)]
    pub fn resize_normalize_u8_to_f16(
        &mut self, stream: &Arc<CudaStream>, src: &[u8], src_size: (u32, u32), dst: &mut [u16], dst_size: (u32, u32), batch: u32,
        scale: &[f32; 3], bias: &[f32; 3],
    ) -> Result<(), Kb200Error> {
        self.resize_normalize_u8_to_16bit(stream, src, src_size, dst, dst_size, batch, scale, bias, OUT_F16)
    }

    /// Same as `resize_normalize_u8_to_f16`, `dst` holding bfloat16 bits.
    #[allow(clippy::too_many_arguments)]
    pub fn resize_normalize_u8_to_bf16(
        &mut self, stream: &Arc<CudaStream>, src: &[u8], src_size: (u32, u32), dst: &mut [u16], dst_size: (u32, u32), batch: u32,
        scale: &[f32; 3], bias: &[f32; 3],
    ) -> Result<(), Kb200Error> {
        self.resize_normalize_u8_to_16bit(stream, src, src_size, dst, dst_size, batch, scale, bias, OUT_BF16)
    }

    #[allow(clippy::too_many_arguments)]
    fn resize_normalize_u8_to_16bit(
        &mut self, stream: &Arc<CudaStream>, src: &[u8], src_size: (u32, u32), dst: &mut [u16], dst_size: (u32, u32), batch: u32,
        scale: &[f32; 3], bias: &[f32; 3], out_format: c_int,
    ) -> Result<(), Kb200Error> {
        check(unsafe {
            ffi::kb200_resize_normalize_chw_u8_host(self.raw, stream.cu_stream() as *mut c_void, src.as_ptr(), src.len(),
                                                    dst.as_mut_ptr() as *mut c_void, dst.len(), src_size.0, src_size.1, dst_size.0,
                                                    dst_size.1, batch, scale.as_ptr(), bias.as_ptr(), LEAF_X86_AVX2_FMA, out_format)
        })
    }

    /// Camera preprocess from host frames: `batch` raw frames at `frame_stride`-byte steps in `frames` -> `dst`, the raw bits
    /// of [batch, 3, dst_h, dst_w] values of `out_format` (OUT_F32: 4 bytes each; OUT_F16, OUT_BF16: 2).  Both should be
    /// page-locked.  Enqueue-only: synchronise `stream` before reading `dst`.
    pub fn preprocess(
        &mut self, stream: &Arc<CudaStream>, desc: &ffi::kb200_preprocess_desc, frames: &[u8], frame_stride: usize, batch: u32, dst: &mut [u8],
        out_format: c_int,
    ) -> Result<(), Kb200Error> {
        let elem = if out_format == OUT_F32 { 4 } else { 2 };
        check(unsafe {
            ffi::kb200_preprocess_host_format(self.raw, stream.cu_stream() as *mut c_void, desc, frames.as_ptr(), frames.len(), frame_stride,
                                              batch, dst.as_mut_ptr() as *mut c_void, dst.len() / elem, out_format)
        })
    }

    /// (uploaded, downloaded) bytes of the last call — uploads count only the source rows the geometry taps.
    pub fn last_transfer(&self) -> Result<(u64, u64), Kb200Error> {
        let (mut up, mut down) = (0u64, 0u64);
        check(unsafe { ffi::kb200_host_pipeline_last_transfer(self.raw, &mut up, &mut down) })?;
        Ok((up, down))
    }
}

impl Drop for HostPipeline {
    fn drop(&mut self) {
        unsafe { ffi::kb200_host_pipeline_destroy(self.raw) }
    }
}


/// Replaces `launch_warp_perspective_u8_bilinear_cuda` (cuda/warp_perspective_u8.rs:181).  NOTE: takes the FORWARD
/// homography like the public operator (the reference launcher takes the inverse; the adapter inverts) — call it from
/// `warp_perspective_u8_cuda` with `m`, not `m_inv`.
#[allow(clippy::too_many_arguments)]
pub fn launch_warp_perspective_u8_bilinear_cuda(
    ctx: &Arc<CudaContext>, stream: &Arc<CudaStream>, src: &CudaSlice<u8>, dst: &mut CudaSlice<u8>, m: &[f32; 9],
    src_width: u32, src_height: u32, dst_width: u32, dst_height: u32, channels: u32, _block_dim: Option<(u32, u32)>,
) -> Result<(), Kb200Error> {
    bind(ctx)?;
    let (sp, _g0) = src.device_ptr(stream);
    let (src_len, dst_len) = (src.len(), dst.len());
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_warp_perspective_u8(stream.cu_stream() as *mut c_void, sp as *const u8, src_len, dp as *mut u8, dst_len,
                                       src_width, src_height, dst_width, dst_height, channels, 1, m.as_ptr())
    })
}

/// Replaces `launch_remap_bilinear_cuda` (cuda/remap.rs): f32, 3 channels, maps of dst_w*dst_h f32 each.
#[allow(clippy::too_many_arguments)]
pub fn launch_remap_bilinear_cuda(
    ctx: &Arc<CudaContext>, stream: &Arc<CudaStream>, src: &CudaSlice<f32>, dst: &mut CudaSlice<f32>, map_x: &CudaSlice<f32>,
    map_y: &CudaSlice<f32>, src_width: u32, src_height: u32, dst_width: u32, dst_height: u32, _block_dim: Option<(u32, u32)>,
) -> Result<(), Kb200Error> {
    bind(ctx)?;
    let (sp, _g0) = src.device_ptr(stream);
    let (mx, _g2) = map_x.device_ptr(stream);
    let (my, _g3) = map_y.device_ptr(stream);
    let (src_len, dst_len, map_len) = (src.len(), dst.len(), map_x.len().min(map_y.len()));
    let (dp, _g1) = dst.device_ptr_mut(stream);
    check(unsafe {
        ffi::kb200_remap_f32_c3(stream.cu_stream() as *mut c_void, sp as *const f32, src_len, dp as *mut f32, dst_len, mx as *const f32,
                                my as *const f32, map_len, src_width, src_height, dst_width, dst_height, 1, 1)
    })
}
