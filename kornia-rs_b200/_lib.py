"""ctypes binding of libkornia_b200.so (include/kornia_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, an exception is
raised — nothing here ever routes to a CPU implementation (cuda/dispatch.rs:203-211: "never a
silent CPU fallback").
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libkornia_b200.so")

OK = 0
ERR_INVALID_ARGUMENT, ERR_SLICE_TOO_SMALL, ERR_SINGULAR_MATRIX, ERR_UNSUPPORTED = -1, -2, -3, -4
ERR_CUDA, ERR_INVALID_KERNEL, ERR_DIMS_TOO_LARGE, ERR_INVALID_SOURCE = -5, -6, -7, -8
OUT_F32, OUT_F16, OUT_BF16 = 0, 1, 2   # kb200_out_format


class PreprocessDesc(C.Structure):
    """kb200_preprocess_desc"""
    _fields_ = [
        ("scale_x", C.c_float), ("scale_y", C.c_float), ("pad_x", C.c_float), ("pad_y", C.c_float),
        ("src_w", C.c_int32), ("src_h", C.c_int32), ("src_pitch", C.c_int32), ("src_bpp", C.c_int32),
        ("fmt", C.c_int32), ("dst_w", C.c_int32), ("dst_h", C.c_int32),
        ("mean", C.c_float * 3), ("inv_std", C.c_float * 3), ("pad_value", C.c_float), ("sampling", C.c_int32),
    ]


class Roi(C.Structure):
    """kb200_roi: region (x, y, w, h) of frame `frame`"""
    _fields_ = [("frame", C.c_int32), ("x", C.c_int32), ("y", C.c_int32), ("w", C.c_int32), ("h", C.c_int32)]


class WarpRoi(C.Structure):
    """kb200_warp_roi: frame `frame` through the forward map `m` (row-major 3x3, frame -> output pixel coordinates)"""
    _fields_ = [("frame", C.c_int32), ("m", C.c_float * 9)]


class RemapRoi(C.Structure):
    """kb200_remap_roi: frame `frame` resampled through map `map` of the call's map arrays"""
    _fields_ = [("frame", C.c_int32), ("map", C.c_int32)]


_lib = None
_tls = threading.local()


def _declare(l: C.CDLL) -> None:
    vp, sz, u32, i, f = C.c_void_p, C.c_size_t, C.c_uint32, C.c_int, C.c_float
    fp = C.POINTER(C.c_float)
    sig = {
        "kb200_version": ([], i),
        "kb200_last_error": ([], C.c_char_p),
        "kb200_status_name": ([i], C.c_char_p),
        "kb200_last_kernel": ([], C.c_char_p),
        "kb200_debug_set_knob": ([C.c_char_p, i], i),
        "kb200_set_device": ([i], i),
        "kb200_device_info": ([C.POINTER(i)] * 3, i),
        "kb200_resize_bilinear_f32_c3": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, i], i),
        "kb200_resize_nearest_f32_c3": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, i], i),
        "kb200_resize_bilinear_normalize_f32_c3": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, fp, i], i),
        "kb200_resize_f32": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32, i], i),
        "kb200_resize_bicubic_f32_c3": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32], i),
        "kb200_resize_lanczos_scratch_len": ([u32, u32, u32, u32], sz),
        "kb200_resize_lanczos_f32_c3": ([vp, vp, sz, vp, sz, vp, sz, u32, u32, u32, u32, u32], i),
        "kb200_generate_correction_map_polynomial": ([vp, C.POINTER(C.c_double), C.POINTER(C.c_double), u32, u32, vp, vp, sz], i),
        "kb200_generate_correction_map_polynomial_to": ([vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), u32, u32, vp, vp, sz], i),
        "kb200_fused_pipeline_u8_f32": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, i, fp, fp, i], i),
        "kb200_pyrdown_f32": ([vp, vp, sz, vp, sz, u32, u32, u32, u32], i),
        "kb200_pyrup_f32": ([vp, vp, sz, vp, sz, u32, u32, u32, u32], i),
        "kb200_pyrdown_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32], i),
        "kb200_pyrup_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32], i),
        "kb200_resize_normalize_chw_u8_f32": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, fp, i], i),
        "kb200_resize_normalize_chw_u8_f16": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, fp, i], i),
        "kb200_resize_normalize_chw_u8_bf16": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, fp, i], i),
        "kb200_resize_row_plan": ([u32, u32, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)], None),
        "kb200_resize_normalize_chw_u8_f32_rows": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, fp, i, u32, u32, u32], i),
        "kb200_host_pipeline_create": ([i, sz, sz, i, C.POINTER(vp)], i),
        "kb200_host_pipeline_destroy": ([vp], None),
        "kb200_host_pipeline_last_transfer": ([vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)], i),
        "kb200_host_register": ([vp, sz], i),
        "kb200_host_unregister": ([vp], i),
        "kb200_resize_normalize_chw_u8_host": ([vp, vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, fp, i, i], i),
        "kb200_resize_normalize_chw_u8_f32_host": ([vp, vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, fp, i], i),
        "kb200_resize_bilinear_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32], i),
        "kb200_resize_fast_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32, i], i),
        "kb200_warp_affine_f32_c3": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, i], i),
        "kb200_warp_perspective_f32_c3": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, fp, i], i),
        "kb200_quantize_kernel_256": ([fp, u32, vp], None),
        "kb200_gaussian_blur_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32, f, f], i),
        "kb200_box_blur_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32], i),
        "kb200_remap_f32_c3": ([vp, vp, sz, vp, sz, vp, vp, sz, u32, u32, u32, u32, u32, i], i),
        "kb200_remap_u8": ([vp, vp, sz, vp, sz, vp, vp, sz, u32, u32, u32, u32, u32, u32, i], i),
        "kb200_yuyv_from_rgb_u8": ([vp, vp, sz, vp, sz, u32, u32, u32], i),
        "kb200_nv12_from_rgb_u8": ([vp, vp, sz, vp, sz, u32, u32, u32], i),
        "kb200_warp_affine_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32, fp], i),
        "kb200_warp_perspective_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32, fp], i),
        "kb200_invert_affine_transform": ([fp, fp], None),
        "kb200_invert_homography": ([fp, fp], i),
        "kb200_get_rotation_matrix2d": ([f, f, f, f, fp], None),
        "kb200_separable_filter_f32": ([vp, vp, sz, vp, sz, vp, fp, u32, fp, u32, u32, u32, u32, u32], i),
        "kb200_gaussian_blur_f32": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32, u32, f, f], i),
        "kb200_sobel_f32": ([vp, vp, sz, vp, sz, u32, u32, u32, u32, u32], i),
        "kb200_gradient_magnitude_f32": ([vp, vp, vp, vp, sz], i),
        "kb200_gaussian_kernel_1d": ([u32, f, fp], None),
        "kb200_gaussian_resolve": ([u32, u32, f, f, C.POINTER(u32), C.POINTER(u32), fp, fp], i),
        "kb200_gray_from_rgb_f32": ([vp, vp, sz, vp, sz, sz, i], i),
        "kb200_gray_from_rgb_u8": ([vp, vp, sz, vp, sz, sz], i),
        "kb200_rgb_from_nv12_u8": ([vp, vp, sz, vp, sz, u32, u32, u32], i),
        "kb200_rgb_from_yuyv_u8": ([vp, vp, sz, vp, sz, u32, u32, u32], i),
        "kb200_rgb_from_yuv420_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, i], i),
        "kb200_rgb_from_yuv422_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, i], i),
        "kb200_rgb_from_yuv420_u8_matrix": ([vp, vp, sz, vp, sz, u32, u32, u32, i, i], i),
        "kb200_rgb_from_yuv422_u8_matrix": ([vp, vp, sz, vp, sz, u32, u32, u32, i, i], i),
        "kb200_rgb_from_bayer_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, i], i),
        "kb200_rgb_from_bayer_u16": ([vp, vp, sz, vp, sz, u32, u32, u32, i], i),
        "kb200_rgb_from_bayer_packed": ([vp, vp, sz, vp, sz, u32, u32, u32, i, i], i),
        "kb200_rgb_from_yuv420_u16": ([vp, vp, sz, vp, sz, u32, u32, u32, i, i, i], i),
        "kb200_rgb_from_yuv444_u8": ([vp, vp, sz, vp, sz, u32, u32, u32, i], i),
        "kb200_rgb_from_yuv444_u16": ([vp, vp, sz, vp, sz, u32, u32, u32, i, i, i], i),
        "kb200_normalize_mean_std_f32": ([vp, vp, vp, sz, u32, fp, fp], i),
        "kb200_normalize_rgb_u8_f32": ([vp, vp, vp, sz, fp, fp, i], i),
        "kb200_find_min_max_f32": ([vp, vp, sz, vp], i),
        "kb200_normalize_min_max_f32": ([vp, vp, vp, sz, f, f, vp], i),
        "kb200_std_mean_u8_c3": ([vp, vp, sz, vp], i),
        "kb200_std_mean_finalize": ([C.POINTER(C.c_uint64), sz, C.POINTER(C.c_double), C.POINTER(C.c_double)], None),
        "kb200_preprocess_affine": ([i, u32, u32, u32, u32, fp], None),
        "kb200_selftest_div255": ([vp, vp], i),
        "kb200_selftest_div2": ([vp, C.c_uint64, C.c_uint32, vp], i),
        "kb200_preprocess_src_bytes": ([C.POINTER(PreprocessDesc)], sz),
        "kb200_preprocess_f32": ([vp, C.POINTER(PreprocessDesc), C.POINTER(vp), C.POINTER(sz), u32, vp, sz], i),
        "kb200_preprocess_f16": ([vp, C.POINTER(PreprocessDesc), C.POINTER(vp), C.POINTER(sz), u32, vp, sz], i),
        "kb200_preprocess_strided_f32": ([vp, C.POINTER(PreprocessDesc), vp, sz, sz, u32, vp, sz], i),
        "kb200_preprocess_host": ([vp, vp, C.POINTER(PreprocessDesc), vp, sz, sz, u32, vp, sz, i], i),
        "kb200_preprocess_strided_f16": ([vp, C.POINTER(PreprocessDesc), vp, sz, sz, u32, vp, sz], i),
        "kb200_preprocess_bf16": ([vp, C.POINTER(PreprocessDesc), C.POINTER(vp), C.POINTER(sz), u32, vp, sz], i),
        "kb200_preprocess_strided_bf16": ([vp, C.POINTER(PreprocessDesc), vp, sz, sz, u32, vp, sz], i),
        "kb200_preprocess_host_format": ([vp, vp, C.POINTER(PreprocessDesc), vp, sz, sz, u32, vp, sz, i], i),
        "kb200_preprocess_rois": ([vp, C.POINTER(PreprocessDesc), i, C.POINTER(vp), C.POINTER(sz), u32, C.POINTER(Roi), u32, vp, sz, i], i),
        "kb200_preprocess_warps": ([vp, C.POINTER(PreprocessDesc), C.POINTER(vp), C.POINTER(sz), u32, C.POINTER(WarpRoi), u32, vp, sz, i], i),
        "kb200_preprocess_remap": ([vp, C.POINTER(PreprocessDesc), C.POINTER(vp), C.POINTER(sz), u32, vp, vp, sz, u32, C.POINTER(RemapRoi), u32, vp, sz, i],
                                   i),
    }
    for name, (args, res) in sig.items():
        fn = getattr(l, name)  # AttributeError if the symbol is missing: fail loudly
        fn.argtypes = args
        fn.restype = res


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing — run `python __graft_entry__.py` (build()) first. "
                "kornia_rs_b200 has no CPU fallback."
            )
        l = C.CDLL(LIB_PATH)
        _declare(l)
        _lib = l
    return _lib


def last_error() -> str:
    return lib().kb200_last_error().decode("utf-8", "replace")


def last_kernel() -> str:
    """Name of the kernel the calling thread's last launcher call enqueued."""
    return lib().kb200_last_kernel().decode("utf-8", "replace")


def set_knob(name: str, value: int) -> None:
    st = lib().kb200_debug_set_knob(name.encode(), int(value))
    if st != OK:
        raise ValueError(last_error())


def set_device(ordinal: int) -> None:
    """Bind this thread to `ordinal` inside the library's CUDA runtime (cached per thread)."""
    if getattr(_tls, "device", None) != ordinal:
        st = lib().kb200_set_device(int(ordinal))
        if st != OK:
            raise RuntimeError(f"kb200_set_device({ordinal}) failed: {last_error()}")
        _tls.device = ordinal


def f3(values, n: int = 3):
    return (C.c_float * n)(*[float(v) for v in values])
