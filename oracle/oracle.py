"""ctypes front-end of the CPU oracle (oracle/kornia_oracle.cpp).

TEST INFRASTRUCTURE — only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / `--impl reference` leg import this module.  The product package
(kornia-rs_b200/) must never import it.

All arrays are numpy, C-contiguous; images are HWC like the reference's
`Image<T,C>` (kornia-image/src/image.rs:138).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libkornia_oracle.so")

NEAREST, BILINEAR, BICUBIC, LANCZOS = 0, 1, 2, 3
LEAF_SCALAR, LEAF_X86, LEAF_NEON = 0, 1, 2
LETTERBOX, STRETCH = 0, 1
FMT_RGB, FMT_BGR, FMT_GRAY, FMT_NV12, FMT_YUYV = 0, 1, 2, 3, 4


def build(force: bool = False) -> str:
    """Compile the oracle shared library with the committed Makefile."""
    src = os.path.join(_HERE, "kornia_oracle.cpp")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _declare(_lib)
    return _lib


class PreprocessDesc(C.Structure):
    _fields_ = [
        ("scale_x", C.c_float), ("scale_y", C.c_float), ("pad_x", C.c_float), ("pad_y", C.c_float),
        ("src_w", C.c_int32), ("src_h", C.c_int32), ("src_pitch", C.c_int32), ("src_bpp", C.c_int32),
        ("fmt", C.c_int32), ("dst_w", C.c_int32), ("dst_h", C.c_int32),
        ("mean", C.c_float * 3), ("inv_std", C.c_float * 3), ("pad_value", C.c_float), ("sampling", C.c_int32),
    ]


def _declare(l: C.CDLL) -> None:
    sz, vp, f, i = C.c_size_t, C.c_void_p, C.c_float, C.c_int
    l.ko_pattern_u8.argtypes = [vp, sz, C.c_uint32]
    l.ko_pattern_f32.argtypes = [vp, sz, C.c_uint32]
    l.ko_gray_from_rgb_f32.argtypes = [vp, vp, sz, i]
    l.ko_gray_from_rgb_u8.argtypes = [vp, vp, sz]
    l.ko_rgb_from_nv12_u8.argtypes = [vp, vp, sz, sz]
    l.ko_rgb_from_yuyv_u8.argtypes = [vp, vp, sz, sz]
    l.ko_resize_f32.argtypes = [vp, sz, sz, vp, sz, sz, sz, i]
    l.ko_normalize_params_from_mean_std.argtypes = [vp, vp, vp, vp]
    l.ko_resize_normalize_u8_to_f32_chw_bilinear.argtypes = [vp, sz, sz, vp, sz, sz, vp, vp, i]
    l.ko_resize_bilinear_u8.argtypes = [vp, sz, sz, vp, sz, sz, sz]
    l.ko_resize_fast_u8.argtypes = [vp, sz, sz, vp, sz, sz, sz, C.c_int]
    l.ko_quantize_kernel_256.argtypes = [vp, sz, vp]
    l.ko_gaussian_blur_u8.argtypes = [vp, vp, sz, sz, sz, sz, sz, f, f]
    l.ko_gaussian_blur_u8.restype = C.c_int
    l.ko_box_blur_u8.argtypes = [vp, vp, sz, sz, sz, sz, sz]
    l.ko_box_blur_u8.restype = C.c_int
    l.ko_remap_f32.argtypes = [vp, sz, sz, vp, sz, sz, sz, vp, vp, C.c_int]
    l.ko_remap_f32.restype = C.c_int
    l.ko_remap_u8.argtypes = [vp, sz, sz, vp, sz, sz, sz, vp, vp, C.c_int]
    l.ko_remap_u8.restype = C.c_int
    l.ko_yuyv_from_rgb_u8.argtypes = [vp, sz, sz, vp]
    l.ko_yuyv_from_rgb_u8.restype = C.c_int
    l.ko_nv12_from_rgb_u8.argtypes = [vp, sz, sz, vp]
    l.ko_nv12_from_rgb_u8.restype = C.c_int
    l.ko_warp_affine_u8.argtypes = [vp, sz, sz, vp, sz, sz, sz, vp]
    l.ko_warp_affine_u8.restype = C.c_int
    l.ko_warp_perspective_u8.argtypes = [vp, sz, sz, vp, sz, sz, sz, vp]
    l.ko_warp_perspective_u8.restype = C.c_int
    l.ko_resize_fast_u8.restype = C.c_int
    l.ko_invert_affine_transform.argtypes = [vp, vp]
    l.ko_get_rotation_matrix2d.argtypes = [f, f, f, f, vp]
    l.ko_constrain_span.argtypes = [f, f, i, f, C.c_longlong, C.c_longlong, vp, vp]
    l.ko_affine_valid_span.argtypes = [vp, sz, f, vp, vp]
    l.ko_warp_affine_f32.argtypes = [vp, sz, sz, vp, sz, sz, sz, vp, i]
    l.ko_invert_homography.argtypes = [vp, vp]
    l.ko_warp_perspective_f32.argtypes = [vp, sz, sz, vp, sz, sz, sz, vp, i]
    l.ko_gaussian_kernel_1d.argtypes = [sz, f, vp]
    l.ko_sobel_kernel_1d.argtypes = [sz, vp, vp]
    l.ko_separable_filter_f32.argtypes = [vp, vp, sz, sz, sz, vp, sz, vp, sz, i]
    l.ko_gaussian_resolve.argtypes = [sz, sz, f, f, vp, vp, vp, vp]
    l.ko_gaussian_blur_f32.argtypes = [vp, vp, sz, sz, sz, sz, sz, f, f, i]
    l.ko_sobel_f32.argtypes = [vp, vp, sz, sz, sz, sz, i]
    l.ko_normalize_mean_std_f32.argtypes = [vp, vp, sz, sz, vp, vp]
    l.ko_find_min_max_f32.argtypes = [vp, sz, vp, vp]
    l.ko_normalize_min_max_f32.argtypes = [vp, vp, sz, f, f]
    l.ko_normalize_rgb_u8.argtypes = [vp, vp, sz, vp, vp, i]
    l.ko_std_mean_u8_c3.argtypes = [vp, sz, vp, vp, vp]
    l.ko_preprocess_affine.argtypes = [i, sz, sz, sz, sz, vp]
    l.ko_f2h.argtypes = [f]
    l.ko_f2h.restype = C.c_uint16
    l.ko_preprocess_frame.argtypes = [vp, vp, C.POINTER(PreprocessDesc), i, vp]
    l.ko_preprocess_cpu_rgb_bilinear.argtypes = [vp, sz, sz, vp, sz, sz, i, vp, vp, f, i]
    l.ko_count_touched_resize.argtypes = [sz, sz, sz, sz, i]
    l.ko_count_touched_resize.restype = sz
    l.ko_sin_pi.argtypes = [C.c_float]; l.ko_sin_pi.restype = C.c_float
    l.ko_lanczos3.argtypes = [C.c_float]; l.ko_lanczos3.restype = C.c_float
    l.ko_lanczos_axis.argtypes = [sz, sz, vp, vp]; l.ko_lanczos_axis.restype = None
    l.ko_lanczos3_weights.argtypes = [C.c_float, vp]; l.ko_lanczos3_weights.restype = None
    l.ko_set_threads.argtypes = [i]
    l.ko_max_threads.restype = i


def _p(a: np.ndarray) -> int:
    assert a.flags["C_CONTIGUOUS"], "oracle arrays must be C-contiguous"
    return a.ctypes.data


def _f3(v) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(v, dtype=np.float32).reshape(-1))


def set_threads(n: int) -> None:
    lib().ko_set_threads(int(n))


def max_threads() -> int:
    return int(lib().ko_max_threads())


# ── generators ───────────────────────────────────────────────────────────────
def pattern_u8(n: int, seed: int = 0x12345678) -> np.ndarray:
    out = np.empty(n, np.uint8)
    lib().ko_pattern_u8(_p(out), n, seed & 0xFFFFFFFF)
    return out


def pattern_f32(n: int, seed: int = 0x12345678) -> np.ndarray:
    out = np.empty(n, np.float32)
    lib().ko_pattern_f32(_p(out), n, seed & 0xFFFFFFFF)
    return out


# ── colour ───────────────────────────────────────────────────────────────────
def gray_from_rgb_f32(src: np.ndarray, leaf: int = LEAF_SCALAR) -> np.ndarray:
    src = np.ascontiguousarray(src, np.float32)
    h, w, _ = src.shape
    dst = np.empty((h, w, 1), np.float32)
    lib().ko_gray_from_rgb_f32(_p(src), _p(dst), h * w, leaf)
    return dst


def gray_from_rgb_u8(src: np.ndarray) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8)
    h, w, _ = src.shape
    dst = np.empty((h, w, 1), np.uint8)
    lib().ko_gray_from_rgb_u8(_p(src), _p(dst), h * w)
    return dst


def rgb_from_nv12(src: np.ndarray, w: int, h: int) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8).reshape(-1)
    assert src.size >= w * h * 3 // 2
    dst = np.empty((h, w, 3), np.uint8)
    if lib().ko_rgb_from_nv12_u8(_p(src), _p(dst), w, h) != 0:
        raise ValueError("NV12 needs even dimensions")
    return dst


def rgb_from_yuyv(src: np.ndarray, w: int, h: int) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8).reshape(-1)
    assert src.size >= w * h * 2
    dst = np.empty((h, w, 3), np.uint8)
    if lib().ko_rgb_from_yuyv_u8(_p(src), _p(dst), w, h) != 0:
        raise ValueError("YUYV needs an even width")
    return dst


# ── resize ───────────────────────────────────────────────────────────────────
def resize_f32(src: np.ndarray, dw: int, dh: int, mode: int = BILINEAR) -> np.ndarray:
    src = np.ascontiguousarray(src, np.float32)
    sh, sw, c = src.shape
    dst = np.zeros((dh, dw, c), np.float32)
    rc = lib().ko_resize_f32(_p(src), sw, sh, _p(dst), dw, dh, c, mode)
    assert rc == 0
    return dst


def normalize_params_from_mean_std(mean, std):
    m, s = _f3(mean), _f3(std)
    scale, bias = np.empty(3, np.float32), np.empty(3, np.float32)
    lib().ko_normalize_params_from_mean_std(_p(m), _p(s), _p(scale), _p(bias))
    return scale, bias


def resize_normalize_u8_to_f32_chw(src: np.ndarray, dw: int, dh: int, scale, bias, leaf: int = LEAF_X86) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8)
    sh, sw, c = src.shape
    assert c == 3
    scale, bias = _f3(scale), _f3(bias)
    dst = np.zeros((3, dh, dw), np.float32)
    rc = lib().ko_resize_normalize_u8_to_f32_chw_bilinear(_p(src), sw, sh, _p(dst), dw, dh, _p(scale), _p(bias), leaf)
    assert rc == 0
    return dst


def resize_bilinear_u8(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8)
    sh, sw, c = src.shape
    dst = np.zeros((dh, dw, c), np.uint8)
    rc = lib().ko_resize_bilinear_u8(_p(src), sw, sh, _p(dst), dw, dh, c)
    if rc != 0:
        raise ValueError(f"resize_bilinear_u8 rc={rc}")
    return dst


def resize_fast_u8(src: np.ndarray, dw: int, dh: int, interp: int = 1) -> np.ndarray:
    """resize_fast_u8_aa path selection (resize/mod.rs:283-410): interp 0 = Nearest, 1 = Bilinear (exact-2x pyramid arms,
    Q14 generic arm).  Raises ValueError with the reference's error class name."""
    src = np.ascontiguousarray(src, np.uint8)
    sh, sw, c = src.shape
    dst = np.zeros((dh, dw, c), np.uint8)
    rc = lib().ko_resize_fast_u8(_p(src), sw, sh, _p(dst), dw, dh, c, interp)
    if rc != 0:
        raise ValueError({-1: "UnsupportedChannelCount", -2: "InvalidImageSize", -3: "UnsupportedInterpolation"}.get(rc, str(rc)))
    return dst


def warp_affine_u8(src: np.ndarray, dw: int, dh: int, m) -> np.ndarray:
    """warp/affine.rs:373 — Q16 span walk + Q10 sampler, zero fill outside the valid span."""
    src = np.ascontiguousarray(src, np.uint8)
    sh, sw, c = src.shape
    dst = np.full((dh, dw, c), 0xCD, np.uint8)
    lib().ko_warp_affine_u8(_p(src), sw, sh, _p(dst), dw, dh, c, _p(_f3(m)))
    return dst


def warp_perspective_u8(src: np.ndarray, dw: int, dh: int, m) -> np.ndarray:
    """warp/perspective.rs:179 — row classification, direct per-column coordinates, Q10 sampler."""
    src = np.ascontiguousarray(src, np.uint8)
    sh, sw, c = src.shape
    dst = np.full((dh, dw, c), 0xCD, np.uint8)
    rc = lib().ko_warp_perspective_u8(_p(src), sw, sh, _p(dst), dw, dh, c, _p(_f3(m)))
    if rc != 0:
        raise ValueError("CannotComputeDeterminant")
    return dst


# ── warps ────────────────────────────────────────────────────────────────────
def invert_affine_transform(m) -> np.ndarray:
    m = _f3(m)
    out = np.empty(6, np.float32)
    lib().ko_invert_affine_transform(_p(m), _p(out))
    return out


def get_rotation_matrix2d(center, angle: float, scale: float) -> np.ndarray:
    out = np.empty(6, np.float32)
    lib().ko_get_rotation_matrix2d(center[0], center[1], angle, scale, _p(out))
    return out


def constrain_span(a, b, ge, eps, lo, hi):
    lo_o, hi_o = C.c_longlong(), C.c_longlong()
    lib().ko_constrain_span(a, b, int(ge), eps, lo, hi, C.addressof(lo_o), C.addressof(hi_o))
    return lo_o.value, hi_o.value


def affine_valid_span(axes, dst_w, eps):
    ax = _f3(axes)
    lo, hi = C.c_size_t(), C.c_size_t()
    lib().ko_affine_valid_span(_p(ax), dst_w, eps, C.addressof(lo), C.addressof(hi))
    return lo.value, hi.value


def warp_affine_f32(src: np.ndarray, m, dw: int, dh: int, mode: int = BILINEAR, dst_init: np.ndarray | None = None):
    src = np.ascontiguousarray(src, np.float32)
    sh, sw, c = src.shape
    m = _f3(m)
    dst = np.zeros((dh, dw, c), np.float32) if dst_init is None else np.ascontiguousarray(dst_init, np.float32).copy()
    rc = lib().ko_warp_affine_f32(_p(src), sw, sh, _p(dst), dw, dh, c, _p(m), mode)
    assert rc == 0
    return dst


def invert_homography(m):
    m = _f3(m)
    out = np.empty(9, np.float32)
    rc = lib().ko_invert_homography(_p(m), _p(out))
    return None if rc != 0 else out


def warp_perspective_f32(src: np.ndarray, m, dw: int, dh: int, mode: int = BILINEAR, dst_init: np.ndarray | None = None):
    src = np.ascontiguousarray(src, np.float32)
    sh, sw, c = src.shape
    m = _f3(m)
    dst = np.zeros((dh, dw, c), np.float32) if dst_init is None else np.ascontiguousarray(dst_init, np.float32).copy()
    rc = lib().ko_warp_perspective_f32(_p(src), sw, sh, _p(dst), dw, dh, c, _p(m), mode)
    if rc == -2:
        raise ValueError("CannotComputeDeterminant")
    assert rc == 0
    return dst


# ── filters ──────────────────────────────────────────────────────────────────
def gaussian_kernel_1d(ksize: int, sigma: float) -> np.ndarray:
    out = np.empty(ksize, np.float32)
    lib().ko_gaussian_kernel_1d(ksize, sigma, _p(out))
    return out


def sobel_kernel_1d(ksize: int):
    kx, ky = np.zeros(5, np.float32), np.zeros(5, np.float32)
    if lib().ko_sobel_kernel_1d(ksize, _p(kx), _p(ky)) != 0:
        raise ValueError("InvalidKernelLength")
    return kx[:ksize].copy(), ky[:ksize].copy()


def separable_filter(src: np.ndarray, kx, ky, mt: bool = False) -> np.ndarray:
    src = np.ascontiguousarray(src, np.float32)
    h, w, c = src.shape
    kx, ky = _f3(kx), _f3(ky)
    dst = np.zeros_like(src)
    rc = lib().ko_separable_filter_f32(_p(src), _p(dst), h, w, c, _p(kx), kx.size, _p(ky), ky.size, int(mt))
    if rc != 0:
        raise ValueError("InvalidKernelLength")
    return dst


def gaussian_resolve(kx: int, ky: int, sx: float, sy: float):
    okx, oky, osx, osy = C.c_size_t(), C.c_size_t(), C.c_float(), C.c_float()
    rc = lib().ko_gaussian_resolve(kx, ky, sx, sy, C.addressof(okx), C.addressof(oky), C.addressof(osx), C.addressof(osy))
    if rc != 0:
        raise ValueError("InvalidSigmaValue")
    return okx.value, oky.value, osx.value, osy.value


def gaussian_blur(src: np.ndarray, ksize, sigma, mt: bool = False) -> np.ndarray:
    src = np.ascontiguousarray(src, np.float32)
    h, w, c = src.shape
    dst = np.zeros_like(src)
    rc = lib().ko_gaussian_blur_f32(_p(src), _p(dst), h, w, c, ksize[0], ksize[1], sigma[0], sigma[1], int(mt))
    if rc != 0:
        raise ValueError("InvalidSigmaValue")
    return dst


def sobel(src: np.ndarray, ksize: int, mt: bool = False) -> np.ndarray:
    src = np.ascontiguousarray(src, np.float32)
    h, w, c = src.shape
    dst = np.zeros_like(src)
    if lib().ko_sobel_f32(_p(src), _p(dst), h, w, c, ksize, int(mt)) != 0:
        raise ValueError("InvalidKernelLength")
    return dst


# ── normalize / stats ────────────────────────────────────────────────────────
def normalize_mean_std(src: np.ndarray, mean, std) -> np.ndarray:
    src = np.ascontiguousarray(src, np.float32)
    h, w, c = src.shape
    mean, std = _f3(mean), _f3(std)
    dst = np.empty_like(src)
    lib().ko_normalize_mean_std_f32(_p(src), _p(dst), h * w, c, _p(mean), _p(std))
    return dst


def find_min_max(src: np.ndarray):
    src = np.ascontiguousarray(src, np.float32)
    mn, mx = C.c_float(), C.c_float()
    if lib().ko_find_min_max_f32(_p(src), src.size, C.addressof(mn), C.addressof(mx)) != 0:
        raise ValueError("ImageDataNotInitialized")
    return mn.value, mx.value


def normalize_min_max(src: np.ndarray, mn: float, mx: float) -> np.ndarray:
    src = np.ascontiguousarray(src, np.float32)
    dst = np.empty_like(src)
    if lib().ko_normalize_min_max_f32(_p(src), _p(dst), src.size, mn, mx) != 0:
        raise ValueError("ImageDataNotInitialized")
    return dst


def normalize_rgb_u8(src: np.ndarray, scale, offset, leaf: int = LEAF_X86) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8)
    scale, offset = _f3(scale), _f3(offset)
    dst = np.empty(src.shape, np.float32)
    lib().ko_normalize_rgb_u8(_p(src), _p(dst), src.size // 3, _p(scale), _p(offset), leaf)
    return dst


def std_mean(src: np.ndarray):
    """Returns (std[3], mean[3], sums[6] = Σp per channel then Σp² per channel)."""
    src = np.ascontiguousarray(src, np.uint8)
    std, mean = np.empty(3, np.float64), np.empty(3, np.float64)
    sums = np.empty(6, np.uint64)
    lib().ko_std_mean_u8_c3(_p(src), src.size // 3, _p(std), _p(mean), _p(sums))
    return std, mean, sums


# ── camera preprocess ────────────────────────────────────────────────────────
def preprocess_affine(mode: int, sw: int, sh: int, dw: int, dh: int):
    out = np.empty(4, np.float32)
    lib().ko_preprocess_affine(mode, sw, sh, dw, dh, _p(out))
    return tuple(float(v) for v in out)


def f2h(x: float) -> int:
    return int(lib().ko_f2h(C.c_float(x)))


_FMT_GEOM = {FMT_RGB: 3, FMT_BGR: 3, FMT_GRAY: 1, FMT_NV12: 1, FMT_YUYV: 2}


@dataclass
class PreprocessCfg:
    mode: int = LETTERBOX
    fmt: int = FMT_RGB
    bpp: int | None = None          # 3 or 4 for RGB/BGR-order formats
    pitch: int | None = None
    mean: tuple = (0.0, 0.0, 0.0)
    inv_std: tuple = (1.0, 1.0, 1.0)
    pad_value: float = 114.0
    sampling: int = BILINEAR


def make_desc(cfg: PreprocessCfg, sw: int, sh: int, dw: int, dh: int) -> PreprocessDesc:
    a = preprocess_affine(cfg.mode, sw, sh, dw, dh)
    bpp = cfg.bpp if cfg.bpp is not None else _FMT_GEOM[cfg.fmt]
    pitch = cfg.pitch if cfg.pitch is not None else sw * bpp
    d = PreprocessDesc()
    d.scale_x, d.scale_y, d.pad_x, d.pad_y = a
    d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt = sw, sh, pitch, bpp, cfg.fmt
    d.dst_w, d.dst_h = dw, dh
    d.mean = (C.c_float * 3)(*cfg.mean)
    d.inv_std = (C.c_float * 3)(*cfg.inv_std)
    d.pad_value = cfg.pad_value
    d.sampling = cfg.sampling
    return d


def preprocess_frame(src: np.ndarray, cfg: PreprocessCfg, sw: int, sh: int, dw: int, dh: int, f16: bool = False,
                     count_touched: bool = False):
    src = np.ascontiguousarray(src, np.uint8).reshape(-1)
    d = make_desc(cfg, sw, sh, dw, dh)
    dst = np.zeros((3, dh, dw), np.uint16 if f16 else np.float32)
    touched = np.zeros(src.size, np.uint8) if count_touched else None
    rc = lib().ko_preprocess_frame(_p(src), _p(dst), C.byref(d), int(f16), _p(touched) if count_touched else None)
    assert rc == 0
    if f16:
        dst = dst.view(np.float16)
    if count_touched:
        return dst, int(touched.sum())
    return dst


def preprocess_frame_desc(src: np.ndarray, d: PreprocessDesc, f16: bool = False) -> np.ndarray:
    """ko_preprocess_frame on a caller-built descriptor: any scale, pad and sampling, src = (dst - pad) / scale.
    d.fmt is one of the FMT_* codes above (no YUV matrix bits); returns (3, dst_h, dst_w) f32 or f16."""
    src = np.ascontiguousarray(src, np.uint8).reshape(-1)
    dst = np.zeros((3, d.dst_h, d.dst_w), np.uint16 if f16 else np.float32)
    assert lib().ko_preprocess_frame(_p(src), _p(dst), C.byref(d), int(f16), None) == 0
    return dst.view(np.float16) if f16 else dst


def preprocess_cpu_rgb_bilinear(src: np.ndarray, dw: int, dh: int, mode: int, mean, inv_std, pad_value: float,
                                leaf: int = LEAF_X86) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8)
    sh, sw, c = src.shape
    assert c == 3
    mean, inv_std = _f3(mean), _f3(inv_std)
    dst = np.zeros((3, dh, dw), np.float32)
    rc = lib().ko_preprocess_cpu_rgb_bilinear(_p(src), sw, sh, _p(dst), dw, dh, mode, _p(mean), _p(inv_std), pad_value, leaf)
    assert rc == 0
    return dst


def count_touched_resize(sw: int, sh: int, dw: int, dh: int, kind: int) -> int:
    return int(lib().ko_count_touched_resize(sw, sh, dw, dh, kind))


# ── u8 blurs (SURVEY §8(f) #1) ───────────────────────────────────────────────
def quantize_kernel_256(k) -> np.ndarray:
    k = _f3(k)
    out = np.zeros(len(k), np.uint8)
    lib().ko_quantize_kernel_256(_p(k), len(k), _p(out))
    return out


def gaussian_blur_u8(src: np.ndarray, ksize=(0, 0), sigma=(0.0, 0.0)) -> np.ndarray:
    """filter/ops.rs:639 — Q8 two-pass (or the [1,2,1]/4 binomial path for k=3, sigma in [0.6, 1.2]), replicate border."""
    src = np.ascontiguousarray(src, np.uint8)
    rows, cols, c = src.shape
    dst = np.zeros_like(src)
    if lib().ko_gaussian_blur_u8(_p(src), _p(dst), rows, cols, c, ksize[0], ksize[1], sigma[0], sigma[1]) != 0:
        raise ValueError("InvalidSigmaValue")
    return dst


def box_blur_u8(src: np.ndarray, ksize) -> np.ndarray:
    """filter/ops.rs:59 — uniform Q8 kernel through the same two-pass path."""
    src = np.ascontiguousarray(src, np.uint8)
    rows, cols, c = src.shape
    dst = np.zeros_like(src)
    if lib().ko_box_blur_u8(_p(src), _p(dst), rows, cols, c, ksize[0], ksize[1]) != 0:
        raise ValueError("InvalidSigmaValue")
    return dst


# ── remap (SURVEY §8(f) #2) ──────────────────────────────────────────────────
def remap(src: np.ndarray, map_x: np.ndarray, map_y: np.ndarray, mode: int = 1) -> np.ndarray:
    """interpolation/remap.rs:43 (f32) / :157 (u8, Q10 sampler); mode 0 = Nearest, 1 = Bilinear; 0 outside the source."""
    mx = np.ascontiguousarray(map_x, np.float32); my = np.ascontiguousarray(map_y, np.float32)
    dh, dw = mx.shape[:2]
    sh, sw, c = src.shape
    if src.dtype == np.uint8:
        src = np.ascontiguousarray(src)
        dst = np.full((dh, dw, c), 0xCD, np.uint8)
        rc = lib().ko_remap_u8(_p(src), sw, sh, _p(dst), dw, dh, c, _p(mx), _p(my), mode)
    else:
        src = np.ascontiguousarray(src, np.float32)
        dst = np.full((dh, dw, c), np.nan, np.float32)
        rc = lib().ko_remap_f32(_p(src), sw, sh, _p(dst), dw, dh, c, _p(mx), _p(my), mode)
    if rc != 0:
        raise ValueError("UnsupportedInterpolation")
    return dst


# ── video encode (SURVEY §8(f) #4) ───────────────────────────────────────────
def yuyv_from_rgb(src: np.ndarray) -> np.ndarray:
    """color/yuv/mod.rs:280 — RGB8 -> packed YUYV (BT.601 limited, Q8); flat w*h*2 bytes."""
    src = np.ascontiguousarray(src, np.uint8)
    h, w, _ = src.shape
    dst = np.zeros(w * h * 2, np.uint8)
    if lib().ko_yuyv_from_rgb_u8(_p(src), w, h, _p(dst)) != 0:
        raise ValueError("InvalidImageSize")
    return dst


def nv12_from_rgb(src: np.ndarray) -> np.ndarray:
    """color/yuv/mod.rs:296 — RGB8 -> NV12 (Y plane + interleaved UV); flat w*h*3/2 bytes."""
    src = np.ascontiguousarray(src, np.uint8)
    h, w, _ = src.shape
    dst = np.zeros(w * h * 3 // 2, np.uint8)
    if lib().ko_nv12_from_rgb_u8(_p(src), w, h, _p(dst)) != 0:
        raise ValueError("InvalidImageSize")
    return dst


# ── bicubic / Lanczos (SURVEY §8(f) #3) ──────────────────────────────────────
def sin_pi(x: float) -> float:
    return float(lib().ko_sin_pi(float(x)))


def lanczos3(x: float) -> float:
    return float(lib().ko_lanczos3(float(x)))


def lanczos3_weights(frac: float) -> np.ndarray:
    w = np.empty(6, np.float32)
    lib().ko_lanczos3_weights(float(frac), _p(w))
    return w


def lanczos_axis(src_len: int, dst_len: int):
    x0s, w = np.empty(dst_len, np.int32), np.empty(dst_len * 6, np.float32)
    lib().ko_lanczos_axis(src_len, dst_len, _p(x0s), _p(w))
    return x0s, w.reshape(dst_len, 6)


# ── pyramids (SURVEY §8(f) #4) ───────────────────────────────────────────────
def _pyr(fn: str, src: np.ndarray, up: bool, dtype):
    src = np.ascontiguousarray(src, dtype)
    sh, sw, c = src.shape
    dst = np.empty((sh * 2, sw * 2, c) if up else ((sh + 1) // 2, (sw + 1) // 2, c), dtype)
    f = getattr(lib(), fn)
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p]
    f.restype = C.c_int
    assert f(_p(src), sw, sh, c, _p(dst)) == 0
    return dst


def pyrdown_f32(src): return _pyr("ko_pyrdown_f32", src, False, np.float32)
def pyrup_f32(src): return _pyr("ko_pyrup_f32", src, True, np.float32)
def pyrdown_u8(src): return _pyr("ko_pyrdown_u8", src, False, np.uint8)
def pyrup_u8(src): return _pyr("ko_pyrup_u8", src, True, np.uint8)


# ── undistort maps (SURVEY §8(f) #2) ─────────────────────────────────────────
def distort_point_polynomial(x: float, y: float, intrinsic, distortion):
    intr, dist, out = np.array(intrinsic, np.float64), np.array(distortion, np.float64), np.empty(2, np.float64)
    f = lib().ko_distort_point_polynomial
    f.argtypes = [C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]; f.restype = None
    f(float(x), float(y), _p(intr), _p(dist), _p(out))
    return float(out[0]), float(out[1])


def generate_correction_map_polynomial(intrinsic, distortion, w: int, h: int):
    intr, dist = np.array(intrinsic, np.float64), np.array(distortion, np.float64)
    mx, my = np.empty((h, w, 1), np.float32), np.empty((h, w, 1), np.float32)
    f = lib().ko_generate_correction_map_polynomial
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p]; f.restype = None
    f(_p(intr), _p(dist), w, h, _p(mx), _p(my))
    return mx, my


# ── cuda/fusion.rs stage vocabulary ──────────────────────────────────────────
def fused_pipeline_u8(src: np.ndarray, dw: int, dh: int, maps: int, scale=(1.0, 1.0, 1.0), bias=(0.0, 0.0, 0.0), sink: int = 0) -> np.ndarray:
    """maps: 0 none, 1 Normalize, 2 RgbToGray, 3 Normalize->RgbToGray, 4 RgbToGray->Normalize; sink 0 = CHW, 1 = single plane."""
    src = np.ascontiguousarray(src, np.uint8)
    sh, sw, _ = src.shape
    dst = np.empty((3, dh, dw) if sink == 0 else (1, dh, dw), np.float32)
    f = lib().ko_fused_pipeline_u8
    f.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]; f.restype = C.c_int
    sc, bi = _f3(scale), _f3(bias)      # keep the arrays alive across the call
    assert f(_p(src), sw, sh, dw, dh, maps, _p(sc), _p(bi), sink, _p(dst)) == 0
    return dst
