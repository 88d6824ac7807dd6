"""The `kornia-imgproc` operator surface of the hot path, over the C-ABI (include/kornia_b200.h).

Same names, argument meaning and error behaviour as the reference's public functions (cited per
function; paths relative to crates/kornia-imgproc/src).  Every op takes `Image`s (HWC, or NHWC for a
batch), checks residency like `pair_residency` (cuda/dispatch.rs:105) and enqueues ONE kernel on the
current CUDA stream of the images' device — asynchronous, no sync, no allocation of outputs.

The reference's host (rayon/SIMD) path is not part of this build and there is no CPU fallback:
host operands raise `ImageError(UnsupportedDevice)`.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import torch

from . import _lib
from .image import Image, ImageError, ImageSize, InterpolationMode, pair_residency

# kb200_cpu_leaf: which CPU leaf of the reference the f32 bits must equal where its scalar and SIMD
# leaves differ (FMA vs mul+add).  The reference's x86_64 hosts with AVX2+FMA run the FMA leaves.
LEAF_SCALAR, LEAF_X86_AVX2_FMA, LEAF_AARCH64_NEON = 0, 1, 2
DEFAULT_LEAF = LEAF_X86_AVX2_FMA

_INTERP = {InterpolationMode.Nearest: 0, InterpolationMode.Bilinear: 1, InterpolationMode.Bicubic: 2, InterpolationMode.Lanczos: 3}


def _stream(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def _check(status: int) -> None:
    if status != _lib.OK:
        raise ImageError.Cuda(_lib.last_error())


def _prep(op: str, *images: Image) -> torch.device:
    dev = pair_residency(op, *images)
    _lib.set_device(dev.index if dev.index is not None else torch.cuda.current_device())
    return dev


def _interp_code(op: str, mode: InterpolationMode) -> int:
    if mode not in _INTERP:
        raise ImageError.UnsupportedInterpolation(mode)
    return _INTERP[mode]


def _same_batch(src: Image, dst: Image) -> int:
    if src.batch != dst.batch:
        raise ImageError.InvalidImageSize(src.batch, 0, dst.batch, 0)
    return src.batch


def _expect_dtype(im: Image, dtype, what: str) -> None:
    if im.dtype != dtype:
        raise ImageError.DtypeMismatch(dtype, im.dtype)


# ── resize ───────────────────────────────────────────────────────────────────
def resize(src: Image, dst: Image, interpolation: InterpolationMode) -> None:
    """resize/mod.rs:114 `resize<C>(src, dst, mode)` — f32, half-pixel grid, bit-identical to the CPU path."""
    code = _interp_code("resize", interpolation)
    dev = _prep("resize", src, dst)
    _expect_dtype(src, torch.float32, "src"); _expect_dtype(dst, torch.float32, "dst")
    c = src.num_channels()
    if dst.num_channels() != c:
        raise ImageError.InvalidChannelShape(dst.num_channels(), c)
    n = _same_batch(src, dst)
    l = _lib.lib()
    args = (_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(),
            src.cols(), src.rows(), dst.cols(), dst.rows())
    if code >= 2:
        # Bicubic / Lanczos (interpolation/{bicubic,lanczos}.rs): 3-channel device kernels like the reference's
        # (resize/cuda.rs:40-42); same-size is the reference's copy short-circuit (resize/mod.rs:134-137)
        if c != 3:
            raise ImageError.Cuda("CUDA resize supports 3-channel f32 images only; move the images to the host (Image::to_host) to use the CPU path")
        if src.size() == dst.size():
            dst.data.copy_(src.data)
        elif code == 2:
            _check(l.kb200_resize_bicubic_f32_c3(*args, n))
        else:
            need = l.kb200_resize_lanczos_scratch_len(src.rows(), dst.cols(), dst.rows(), n)
            scratch = torch.empty(need, dtype=torch.float32, device=dev)   # stream-ordered, like the reference's stream.alloc
            _check(l.kb200_resize_lanczos_f32_c3(args[0], args[1], args[2], args[3], args[4], scratch.data_ptr(), scratch.numel(), *args[5:], n))
    elif c == 3 and not (src.size() == dst.size()):
        fn = l.kb200_resize_bilinear_f32_c3 if code == 1 else l.kb200_resize_nearest_f32_c3
        _check(fn(*args, n, 0))
    else:
        _check(l.kb200_resize_f32(*args, c, n, code))


def resize_bilinear_normalize(src: Image, dst: Image, mean: Sequence[float], std: Sequence[float],
                              align_corners: bool = False) -> None:
    """cuda/resize.rs:580 `launch_resize_bilinear_normalize_cuda` — bilinear + (v-mean)/std, HWC out."""
    dev = _prep("resize_bilinear_normalize", src, dst)
    _expect_dtype(src, torch.float32, "src"); _expect_dtype(dst, torch.float32, "dst")
    if src.num_channels() != 3 or dst.num_channels() != 3:
        raise ImageError.Cuda("CUDA resize supports 3-channel f32 images only; move the images to the host (Image::to_host) to use the CPU path")
    n = _same_batch(src, dst)
    _check(_lib.lib().kb200_resize_bilinear_normalize_f32_c3(
        _stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), src.cols(), src.rows(),
        dst.cols(), dst.rows(), n, _lib.f3(mean), _lib.f3(std), 1 if align_corners else 0))


def resize_fast_u8(src: Image, dst: Image, interpolation: InterpolationMode = InterpolationMode.Bilinear) -> None:
    """resize/mod.rs:348 `resize_fast_u8_aa` with the reference's path selection (`resize_u8_path`, :283-337): exact 2x
    down / up on RGB → pyramid arms, Nearest → any channel count, Bilinear → Q14 (C ∈ {1,3,4}, source ≥ 2x2).
    Bicubic / Lanczos (the antialiased separable arm) are not built."""
    if interpolation not in (InterpolationMode.Bilinear, InterpolationMode.Nearest):
        raise ImageError.UnsupportedInterpolation(interpolation)
    dev = _prep("resize_fast_u8", src, dst)
    _expect_dtype(src, torch.uint8, "src"); _expect_dtype(dst, torch.uint8, "dst")
    c = src.num_channels()
    sw, sh, dw, dh = src.cols(), src.rows(), dst.cols(), dst.rows()
    pyr = c == 3 and sw >= 2 and sh >= 2 and ((sw == 2 * dw and sh == 2 * dh) or (dw == 2 * sw and dh == 2 * sh))
    if interpolation == InterpolationMode.Bilinear and not pyr:
        if c not in (1, 3, 4):
            raise ImageError.UnsupportedChannelCount(c)
        if sw < 2 or sh < 2:
            raise ImageError.InvalidImageSize(sw, sh, 2, 2)
    n = _same_batch(src, dst)
    code = 1 if interpolation == InterpolationMode.Bilinear else 0
    _check(_lib.lib().kb200_resize_fast_u8(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(),
                                           sw, sh, dw, dh, c, n, code))


class NormalizeParams:
    """resize/fused.rs:17-38 — scale = 1/(std*255), bias = -mean/std (f32 arithmetic)."""

    def __init__(self, scale, bias):
        self.scale = [float(v) for v in scale]
        self.bias = [float(v) for v in bias]

    @staticmethod
    def from_mean_std(mean, std) -> "NormalizeParams":
        m = torch.tensor(list(mean), dtype=torch.float32)
        s = torch.tensor(list(std), dtype=torch.float32)
        scale = torch.tensor(1.0, dtype=torch.float32) / (s * torch.tensor(255.0, dtype=torch.float32))
        bias = -m / s
        return NormalizeParams(scale.tolist(), bias.tolist())


def resize_row_plan(src_h: int, dst_h: int) -> tuple[int, int, int]:
    """(period, first, keep): the source rows a vertical geometry taps are those with
    first <= y % period < first + keep.  (1, 0, 1) = all rows.  kb200_resize_row_plan."""
    a, b, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
    _lib.lib().kb200_resize_row_plan(src_h, dst_h, C.byref(a), C.byref(b), C.byref(c))
    return a.value, b.value, c.value


class HostPipeline:
    """Staging ring for the host-buffer form of the hot path (kb200_host_pipeline): `depth` streams, each with a device
    source and destination chunk buffer.  Created once per device; calls only enqueue."""

    def __init__(self, device=None, src_chunk_bytes: int = 96 << 20, dst_chunk_bytes: int = 96 << 20, depth: int = 3):
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise ImageError.Cuda("HostPipeline needs a CUDA device")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        h = C.c_void_p()
        _check(_lib.lib().kb200_host_pipeline_create(self.device.index, src_chunk_bytes, dst_chunk_bytes, depth, C.byref(h)))
        self._h = h
        self.depth = depth

    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h:
            _lib.lib().kb200_host_pipeline_destroy(h)

    def __del__(self):
        try:
            self.close()
        except Exception:   # interpreter shutdown: the library handle may already be gone
            pass

    def last_transfer(self) -> tuple[int, int]:
        """(h2d_bytes, d2h_bytes) the last call moved over the link."""
        a, b = C.c_uint64(), C.c_uint64()
        _check(_lib.lib().kb200_host_pipeline_last_transfer(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value


_default_pipelines: dict[int, HostPipeline] = {}


def _pipeline_for(pipeline: HostPipeline | None) -> HostPipeline:
    if pipeline is not None:
        return pipeline
    idx = torch.cuda.current_device()
    if idx not in _default_pipelines:
        _default_pipelines[idx] = HostPipeline(torch.device("cuda", idx))
    return _default_pipelines[idx]


# output dtype -> (device entry point, kb200_out_format of the host-buffer form; f32 keeps its own host entry point)
_CHW_OUT = {torch.float32: ("kb200_resize_normalize_chw_u8_f32", None),
            torch.float16: ("kb200_resize_normalize_chw_u8_f16", _lib.OUT_F16),
            torch.bfloat16: ("kb200_resize_normalize_chw_u8_bf16", _lib.OUT_BF16)}


def resize_normalize_to_tensor_u8_to_f32_bilinear(src, dst_w: int, dst_h: int, scale, bias, out: torch.Tensor | None = None,
                                                  leaf: int = DEFAULT_LEAF, pipeline: HostPipeline | None = None) -> torch.Tensor:
    """resize/fused.rs:147 — u8 HWC (or NHWC) → f32 CHW ([N,3,dst_h,dst_w]) bilinear (half-pixel, non-AA)
    resize + `sample*scale[c] + bias[c]`; exact 2x dispatches to the box average (fused.rs:181-183).

    Device images run the kernel in place.  HOST images (the reference operator's own signature) go through a
    `HostPipeline`: chunked upload → kernel → download on the GPU, enqueued on the current stream of the pipeline's
    device — synchronise that stream before reading `out`.  There is no CPU implementation."""
    return _resize_normalize_chw("resize_normalize_to_tensor_u8_to_f32_bilinear", src, dst_w, dst_h, scale, bias, torch.float32, out,
                                 leaf, pipeline)


def resize_normalize_to_tensor_u8_bilinear(src, dst_w: int, dst_h: int, scale, bias, dtype: torch.dtype, out: torch.Tensor | None = None,
                                           leaf: int = DEFAULT_LEAF, pipeline: HostPipeline | None = None) -> torch.Tensor:
    """`resize_normalize_to_tensor_u8_to_f32_bilinear` with the CHW output in `dtype`: torch.float32, torch.float16 or
    torch.bfloat16.  A 16-bit value is the f32 result rounded once to nearest-even — bit-identical to calling the f32
    operator and then `.to(dtype)`, without writing and re-reading the f32 tensor.  (An extension: the reference writes
    f32 only.)  Device and host sources as for the f32 operator; an `out` it allocates for a host source is pinned."""
    if dtype not in _CHW_OUT:
        raise ImageError.DtypeMismatch("torch.float32, torch.float16 or torch.bfloat16", dtype)
    if out is not None and out.dtype != dtype:
        raise ImageError.DtypeMismatch(dtype, out.dtype)
    return _resize_normalize_chw("resize_normalize_to_tensor_u8_bilinear", src, dst_w, dst_h, scale, bias, dtype, out, leaf, pipeline)


def _resize_normalize_chw(op: str, src, dst_w: int, dst_h: int, scale, bias, dtype: torch.dtype, out: torch.Tensor | None, leaf: int,
                          pipeline: HostPipeline | None) -> torch.Tensor:
    fn, out_format = _CHW_OUT[dtype]
    t = src.data if isinstance(src, Image) else src
    if t.dtype != torch.uint8:
        raise ImageError.DtypeMismatch(torch.uint8, t.dtype)
    if not t.is_contiguous():
        raise ImageError.ImageDataNotContiguous()
    if t.dim() == 3:
        t = t.unsqueeze(0)
    n, sh, sw, c = t.shape
    if c != 3:
        raise ImageError.InvalidChannelShape(t.numel(), n * sh * sw * 3)
    if not t.is_cuda:
        if not torch.cuda.is_available():
            raise ImageError.HostPathNotBuilt(op)
        if out is None:
            out = torch.empty((n, 3, dst_h, dst_w), dtype=dtype, pin_memory=True)
        elif out.is_cuda:
            raise ImageError.MixedResidency()
        if out.dtype != dtype or not out.is_contiguous() or out.numel() != n * 3 * dst_h * dst_w:
            raise ImageError.InvalidChannelShape(out.numel(), n * 3 * dst_h * dst_w)
        pipe = _pipeline_for(pipeline)
        _lib.set_device(pipe.device.index)
        args = (pipe._h, _stream(pipe.device), t.data_ptr(), t.numel(), out.data_ptr(), out.numel(), sw, sh, dst_w, dst_h, n,
                _lib.f3(scale), _lib.f3(bias), leaf)
        if out_format is None:
            _check(_lib.lib().kb200_resize_normalize_chw_u8_f32_host(*args))
        else:
            _check(_lib.lib().kb200_resize_normalize_chw_u8_host(*args, out_format))
        return out
    if out is None:
        out = torch.empty((n, 3, dst_h, dst_w), dtype=dtype, device=t.device)
    else:
        if out.device != t.device:
            raise ImageError.DeviceMismatch() if out.is_cuda else ImageError.MixedResidency()
        if out.dtype != dtype or not out.is_contiguous() or out.numel() != n * 3 * dst_h * dst_w:
            raise ImageError.InvalidChannelShape(out.numel(), n * 3 * dst_h * dst_w)
    dev = t.device
    _lib.set_device(dev.index)
    _check(getattr(_lib.lib(), fn)(_stream(dev), t.data_ptr(), t.numel(), out.data_ptr(), out.numel(),
                                   sw, sh, dst_w, dst_h, n, _lib.f3(scale), _lib.f3(bias), leaf))
    return out


def resize_normalize_rows(src_rows: torch.Tensor, src_w: int, src_h: int, dst_w: int, dst_h: int, scale, bias, row_map: tuple[int, int, int],
                          out: torch.Tensor | None = None, leaf: int = DEFAULT_LEAF) -> torch.Tensor:
    """kb200_resize_normalize_chw_u8_f32_rows — same operator over a row-compacted device source
    ([N, src_h/period*keep, src_w, 3] u8), bit-identical to the full-image call."""
    t = src_rows
    if not t.is_cuda:
        raise ImageError.HostPathNotBuilt("resize_normalize_rows")
    if t.dtype != torch.uint8:
        raise ImageError.DtypeMismatch(torch.uint8, t.dtype)
    if not t.is_contiguous():
        raise ImageError.ImageDataNotContiguous()
    n = t.shape[0]
    if out is None:
        out = torch.empty((n, 3, dst_h, dst_w), dtype=torch.float32, device=t.device)
    _lib.set_device(t.device.index)
    _check(_lib.lib().kb200_resize_normalize_chw_u8_f32_rows(_stream(t.device), t.data_ptr(), t.numel(), out.data_ptr(), out.numel(), src_w, src_h,
                                                            dst_w, dst_h, n, _lib.f3(scale), _lib.f3(bias), leaf, *row_map))
    return out


# ── warps ────────────────────────────────────────────────────────────────────
def invert_affine_transform(m: Sequence[float]) -> list[float]:
    """warp/affine.rs:18."""
    out = (C.c_float * 6)()
    _lib.lib().kb200_invert_affine_transform(_lib.f3(m, 6), out)
    return list(out)


def get_rotation_matrix2d(center: tuple[float, float], angle: float, scale: float) -> list[float]:
    """warp/affine.rs:70 — f32 arithmetic with libm cosf/sinf (the reference's f32::cos/sin)."""
    out = (C.c_float * 6)()
    _lib.lib().kb200_get_rotation_matrix2d(center[0], center[1], angle, scale, out)
    return list(out)


def invert_homography(h: Sequence[float]):
    """warp/perspective.rs:41 — None for a singular matrix."""
    out = (C.c_float * 9)()
    st = _lib.lib().kb200_invert_homography(_lib.f3(h, 9), out)
    return None if st != _lib.OK else list(out)


def _warp(op: str, fn_name: str, src: Image, dst: Image, m: Sequence[float], nm: int, interpolation: InterpolationMode) -> None:
    code = _interp_code(op, interpolation)
    dev = _prep(op, src, dst)
    _expect_dtype(src, torch.float32, "src"); _expect_dtype(dst, torch.float32, "dst")
    if src.num_channels() != 3 or dst.num_channels() != 3:  # warp/cuda.rs:36-38: no_gpu_kernel_err
        raise ImageError.Cuda(f"CUDA {op} supports 3-channel f32 images only; move the images to the host (Image::to_host) to use the CPU path")
    if len(m) != nm:
        raise ValueError(f"{op}: expected {nm} matrix entries, got {len(m)}")
    n = _same_batch(src, dst)
    fn = getattr(_lib.lib(), fn_name)
    _check(fn(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), src.cols(), src.rows(),
              dst.cols(), dst.rows(), n, _lib.f3(m, nm), code))


def warp_affine(src: Image, dst: Image, m: Sequence[float], interpolation: InterpolationMode) -> None:
    """warp/affine.rs:123 — forward 2x3 `m` (inverted internally); pixels mapping outside the source are 0."""
    _warp("warp_affine", "kb200_warp_affine_f32_c3", src, dst, m, 6, interpolation)


def warp_perspective(src: Image, dst: Image, m: Sequence[float], interpolation: InterpolationMode) -> None:
    """warp/perspective.rs:115 — forward 3x3 `m`; a singular matrix is an error; out-of-source pixels are
    written 0 (the device twin's rule, cuda/warp_perspective.rs:81-84)."""
    _warp("warp_perspective", "kb200_warp_perspective_f32_c3", src, dst, m, 9, interpolation)


def _warp_u8(op: str, fn_name: str, src: Image, dst: Image, m: Sequence[float], nm: int) -> None:
    dev = _prep(op, src, dst)
    _expect_dtype(src, torch.uint8, "src"); _expect_dtype(dst, torch.uint8, "dst")
    c = src.num_channels()
    if c != dst.num_channels() or c not in (1, 3, 4):
        raise ImageError.UnsupportedChannelCount(c)
    if len(m) != nm:
        raise ValueError(f"{op}: expected {nm} matrix entries, got {len(m)}")
    n = _same_batch(src, dst)
    st = getattr(_lib.lib(), fn_name)(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(),
                                      src.cols(), src.rows(), dst.cols(), dst.rows(), c, n, _lib.f3(m, nm))
    if st == _lib.ERR_SINGULAR_MATRIX:
        raise ImageError.CannotComputeDeterminant()
    _check(st)


def warp_affine_u8(src: Image, dst: Image, m: Sequence[float]) -> None:
    """warp/affine.rs:373 — bilinear u8 affine warp (Q16 coordinates, Q10 weights), forward 2x3 `m`; bit-exact."""
    _warp_u8("warp_affine_u8", "kb200_warp_affine_u8", src, dst, m, 6)


def warp_perspective_u8(src: Image, dst: Image, m: Sequence[float]) -> None:
    """warp/perspective.rs:179 — bilinear u8 perspective warp (direct coordinates, Q10 weights), forward 3x3 `m`;
    a singular matrix raises CannotComputeDeterminant; bit-exact."""
    _warp_u8("warp_perspective_u8", "kb200_warp_perspective_u8", src, dst, m, 9)


def _remap_prep(op: str, src: Image, dst: Image, map_x: Image, map_y: Image, interpolation: InterpolationMode):
    if map_x.size() != map_y.size():   # interpolation/remap.rs:50-57
        raise ImageError.InvalidImageSize(map_x.rows(), map_x.cols(), map_y.rows(), map_y.cols())
    if dst.size() != map_x.size():
        raise ImageError.InvalidImageSize(dst.rows(), dst.cols(), map_x.rows(), map_x.cols())
    if interpolation not in (InterpolationMode.Bilinear, InterpolationMode.Nearest):
        raise ImageError.UnsupportedInterpolation(interpolation)
    dev = _prep(op, src, dst)
    for m in (map_x, map_y):
        if not m.is_device:
            raise ImageError.Cuda(f"{op}: map_x and map_y must be device-resident when src/dst are on GPU")
        if m.data.device != dev:
            raise ImageError.DeviceMismatch()
        _expect_dtype(m, torch.float32, "map")
        if m.num_channels() != 1 or m.batch != 1:
            raise ImageError.InvalidChannelShape(m.numel(), m.cols() * m.rows())
    return dev, _same_batch(src, dst)


def remap(src: Image, dst: Image, map_x: Image, map_y: Image, interpolation: InterpolationMode) -> None:
    """interpolation/remap.rs:43 — dst[y,x] = sample(src, map_x[y,x], map_y[y,x]) (f32, 3 channels on the device);
    coordinates outside the source give 0.  The maps are shared by every image of a batch."""
    dev, n = _remap_prep("remap", src, dst, map_x, map_y, interpolation)
    _expect_dtype(src, torch.float32, "src"); _expect_dtype(dst, torch.float32, "dst")
    if src.num_channels() != 3 or dst.num_channels() != 3:
        raise ImageError.Cuda("CUDA remap supports 3-channel f32 images only; move the images to the host (Image::to_host) to use the CPU path")
    _check(_lib.lib().kb200_remap_f32_c3(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(),
                                         map_x.data.data_ptr(), map_y.data.data_ptr(), map_x.numel(), src.cols(), src.rows(),
                                         dst.cols(), dst.rows(), n, 1 if interpolation == InterpolationMode.Bilinear else 0))


def remap_u8(src: Image, dst: Image, map_x: Image, map_y: Image, interpolation: InterpolationMode) -> None:
    """interpolation/remap.rs:157 — u8 remap: Q10 bilinear sampler (as the u8 warps) or nearest, constant-0 border; bit-exact."""
    dev, n = _remap_prep("remap_u8", src, dst, map_x, map_y, interpolation)
    _expect_dtype(src, torch.uint8, "src"); _expect_dtype(dst, torch.uint8, "dst")
    c = src.num_channels()
    if c != dst.num_channels() or c not in (1, 3, 4):
        raise ImageError.UnsupportedChannelCount(c)
    _check(_lib.lib().kb200_remap_u8(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(),
                                     map_x.data.data_ptr(), map_y.data.data_ptr(), map_x.numel(), src.cols(), src.rows(),
                                     dst.cols(), dst.rows(), c, n, 1 if interpolation == InterpolationMode.Bilinear else 0))


# ── filters ──────────────────────────────────────────────────────────────────
def _filter_prep(op: str, src: Image, dst: Image):
    dev = _prep(op, src, dst)
    _expect_dtype(src, torch.float32, "src"); _expect_dtype(dst, torch.float32, "dst")
    if src.size() != dst.size() or src.num_channels() != dst.num_channels():
        raise ImageError.InvalidImageSize(src.cols(), src.rows(), dst.cols(), dst.rows())
    return dev, _same_batch(src, dst)


def _blur_u8_prep(op: str, src: Image, dst: Image):
    dev = _prep(op, src, dst)
    _expect_dtype(src, torch.uint8, "src"); _expect_dtype(dst, torch.uint8, "dst")
    if src.size() != dst.size() or src.num_channels() != dst.num_channels():
        raise ImageError.InvalidImageSize(src.cols(), src.rows(), dst.cols(), dst.rows())   # filter/ops.rs:645-652
    if src.num_channels() not in (1, 3, 4):
        raise ImageError.UnsupportedChannelCount(src.num_channels())
    return dev, _same_batch(src, dst)


def gaussian_blur_u8(src: Image, dst: Image, kernel_size: tuple[int, int], sigma: tuple[float, float]) -> None:
    """filter/ops.rs:639 — u8 gaussian blur, replicate border: Q8 two-pass with a u8 intermediate, or the [1,2,1]/4
    rounding-half-add path for k = 3 with sigma in [0.6, 1.2] (`blur_u8_path`).  Bit-exact."""
    dev, n = _blur_u8_prep("gaussian_blur_u8", src, dst)
    st = _lib.lib().kb200_gaussian_blur_u8(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), src.cols(),
                                           src.rows(), src.num_channels(), n, int(kernel_size[0]), int(kernel_size[1]),
                                           float(sigma[0]), float(sigma[1]))
    if st == _lib.ERR_INVALID_KERNEL:
        raise ImageError.InvalidSigmaValue(float(sigma[0]), float(sigma[1]))
    _check(st)


def box_blur_u8(src: Image, dst: Image, kernel_size: tuple[int, int]) -> None:
    """filter/ops.rs:59 — u8 box blur through the same Q8 two-pass; kernel sizes must be odd and positive."""
    dev, n = _blur_u8_prep("box_blur_u8", src, dst)
    kx, ky = int(kernel_size[0]), int(kernel_size[1])
    if kx <= 0 or ky <= 0 or kx % 2 == 0 or ky % 2 == 0:
        raise ImageError.InvalidSigmaValue(float(kx), float(ky))
    _check(_lib.lib().kb200_box_blur_u8(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), src.cols(),
                                        src.rows(), src.num_channels(), n, kx, ky))


def separable_filter(src: Image, dst: Image, kernel_x: Sequence[float], kernel_y: Sequence[float]) -> None:
    """filter/separable_filter.rs:166 — correlation, zero border, H then V; one fused kernel here."""
    if len(kernel_x) == 0 or len(kernel_y) == 0:
        raise ImageError.InvalidKernelLength(len(kernel_x), len(kernel_y))
    dev, n = _filter_prep("separable_filter", src, dst)
    _check(_lib.lib().kb200_separable_filter_f32(
        _stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), None,
        _lib.f3(kernel_x, len(kernel_x)), len(kernel_x), _lib.f3(kernel_y, len(kernel_y)), len(kernel_y),
        src.cols(), src.rows(), src.num_channels(), n))


def gaussian_blur(src: Image, dst: Image, kernel_size: tuple[int, int], sigma: tuple[float, float]) -> None:
    """filter/ops.rs:116 — (0,0) kernel sizes / zero sigmas are auto-resolved exactly like the reference."""
    dev, n = _filter_prep("gaussian_blur", src, dst)
    l = _lib.lib()
    kx, ky, sx, sy = C.c_uint32(), C.c_uint32(), C.c_float(), C.c_float()
    if l.kb200_gaussian_resolve(kernel_size[0], kernel_size[1], sigma[0], sigma[1], C.byref(kx), C.byref(ky),
                                C.byref(sx), C.byref(sy)) != _lib.OK:
        sy_in = sigma[1] if sigma[1] > 0 else sigma[0]
        raise ImageError.InvalidSigmaValue(sigma[0], sy_in)
    _check(l.kb200_gaussian_blur_f32(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(),
                                     src.cols(), src.rows(), src.num_channels(), n, kernel_size[0], kernel_size[1],
                                     sigma[0], sigma[1]))


def gaussian_kernel_1d(kernel_size: int, sigma: float) -> list[float]:
    """filter/kernels.rs:25."""
    out = (C.c_float * kernel_size)()
    _lib.lib().kb200_gaussian_kernel_1d(kernel_size, sigma, out)
    return list(out)


def sobel_kernel_1d(kernel_size: int):
    """filter/kernels.rs:55."""
    if kernel_size == 3:
        return [-1.0, 0.0, 1.0], [1.0, 2.0, 1.0]
    if kernel_size == 5:
        return [-1.0, -2.0, 0.0, 2.0, 1.0], [1.0, 4.0, 6.0, 4.0, 1.0]
    raise ImageError.InvalidKernelLength(kernel_size, kernel_size)


def sobel(src: Image, dst: Image, kernel_size: int) -> None:
    """filter/ops.rs:174 — sqrt(gx² + gy²) of the two separable gradients, fused in one kernel."""
    sobel_kernel_1d(kernel_size)
    dev, n = _filter_prep("sobel", src, dst)
    _check(_lib.lib().kb200_sobel_f32(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(),
                                      src.cols(), src.rows(), src.num_channels(), n, kernel_size))


# ── colour ───────────────────────────────────────────────────────────────────
def gray_from_rgb(src: Image, dst: Image, leaf: int = LEAF_SCALAR) -> None:
    """color/gray/mod.rs:104 `gray_from_rgb` (f32; `Rgbf32::convert`, color/convert.rs:42).
    leaf=LEAF_SCALAR reproduces the reference's CUDA kernel and scalar CPU leaf
    (`0.299r + 0.587g + 0.114b`, unfused); LEAF_X86_AVX2_FMA its AVX2 leaf."""
    dev = _prep("gray_from_rgb", src, dst)
    if src.num_channels() != 3 or dst.num_channels() != 1:
        raise ImageError.InvalidChannelShape(dst.num_channels(), 1)
    if src.size() != dst.size() or src.batch != dst.batch:
        raise ImageError.InvalidImageSize(src.cols(), src.rows(), dst.cols(), dst.rows())
    npx = src.rows() * src.cols() * src.batch
    l = _lib.lib()
    if src.dtype == torch.float32 and dst.dtype == torch.float32:
        _check(l.kb200_gray_from_rgb_f32(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), npx, leaf))
    elif src.dtype == torch.uint8 and dst.dtype == torch.uint8:
        _check(l.kb200_gray_from_rgb_u8(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), npx))
    else:
        raise ImageError.DtypeMismatch(src.dtype, dst.dtype)


def _raw_frames(src, what: str) -> torch.Tensor:
    t = src.data if isinstance(src, Image) else src
    if not t.is_cuda:
        raise ImageError.HostPathNotBuilt(what)
    if t.dtype != torch.uint8:
        raise ImageError.DtypeMismatch(torch.uint8, t.dtype)
    if not t.is_contiguous():
        raise ImageError.ImageDataNotContiguous()
    return t


def rgb_from_nv12(src, dst: Image) -> None:
    """color/yuv/mod.rs:235 — `src`: u8 tensor holding, per frame, w*h Y bytes then w*h/2 interleaved UV
    bytes ([len] or [N,len]); BT.601 limited, Q20, bit-exact."""
    t = _raw_frames(src, "rgb_from_nv12")
    if not dst.is_device:
        raise ImageError.MixedResidency()
    if t.device != dst.device:
        raise ImageError.DeviceMismatch()
    _expect_dtype(dst, torch.uint8, "dst")
    w, h, n = dst.cols(), dst.rows(), dst.batch
    need = w * h * 3 // 2 * n
    if dst.num_channels() != 3 or t.numel() != need:
        raise ImageError.InvalidImageSize(t.numel(), 1, need, 1)  # check_dst_size, color/yuv/mod.rs:186-207
    _lib.set_device(t.device.index)
    _check(_lib.lib().kb200_rgb_from_nv12_u8(_stream(t.device), t.data_ptr(), t.numel(), dst.data.data_ptr(), dst.numel(), w, h, n))


def rgb_from_yuyv(src, dst: Image) -> None:
    """color/yuv/mod.rs:209 (impl_packed422!, Yuyv)."""
    t = _raw_frames(src, "rgb_from_yuyv")
    if not dst.is_device:
        raise ImageError.MixedResidency()
    if t.device != dst.device:
        raise ImageError.DeviceMismatch()
    _expect_dtype(dst, torch.uint8, "dst")
    w, h, n = dst.cols(), dst.rows(), dst.batch
    need = w * h * 2 * n
    if dst.num_channels() != 3 or t.numel() != need:
        raise ImageError.InvalidImageSize(t.numel(), 1, need, 1)
    _lib.set_device(t.device.index)
    _check(_lib.lib().kb200_rgb_from_yuyv_u8(_stream(t.device), t.data_ptr(), t.numel(), dst.data.data_ptr(), dst.numel(), w, h, n))


def _encode(op: str, fn_name: str, src: Image, dst: torch.Tensor, bytes_per_px_num: int, bytes_per_px_den: int, need_even_h: bool) -> None:
    if not src.is_device:
        raise ImageError.HostPathNotBuilt(op)
    _expect_dtype(src, torch.uint8, "src")
    if src.num_channels() != 3:
        raise ImageError.UnsupportedChannelCount(src.num_channels())
    if not isinstance(dst, torch.Tensor) or not dst.is_cuda:
        raise ImageError.MixedResidency()
    if dst.device != src.data.device:
        raise ImageError.DeviceMismatch()
    if dst.dtype != torch.uint8 or not dst.is_contiguous():
        raise ImageError.DtypeMismatch(torch.uint8, dst.dtype)
    w, h, n = src.cols(), src.rows(), src.batch
    need = w * h * bytes_per_px_num // bytes_per_px_den * n
    if w % 2 != 0 or (need_even_h and h % 2 != 0) or dst.numel() != need:   # color/yuv/mod.rs:282-284, :298-300
        raise ImageError.InvalidImageSize(dst.numel(), w, h, need)
    _lib.set_device(dst.device.index)
    _check(getattr(_lib.lib(), fn_name)(_stream(dst.device), src.data.data_ptr(), src.numel(), dst.data_ptr(), dst.numel(), w, h, n))


def yuyv_from_rgb(src: Image, dst: torch.Tensor) -> None:
    """color/yuv/mod.rs:280 — RGB8 → packed YUYV (`Y0 U Y1 V`, BT.601 limited); `dst`: u8, width*height*2 bytes per image."""
    _encode("yuyv_from_rgb", "kb200_yuyv_from_rgb_u8", src, dst, 2, 1, False)


def nv12_from_rgb(src: Image, dst: torch.Tensor) -> None:
    """color/yuv/mod.rs:296 — RGB8 → NV12 (Y plane + interleaved UV); `dst`: u8, width*height*3/2 bytes per image."""
    _encode("nv12_from_rgb", "kb200_nv12_from_rgb_u8", src, dst, 3, 2, True)


# ── normalize / statistics ───────────────────────────────────────────────────
def normalize_mean_std(src: Image, dst: Image, mean: Sequence[float], std: Sequence[float]) -> None:
    """normalize.rs:56 — (x - mean[c]) / std[c], true division."""
    dev = _prep("normalize_mean_std", src, dst)
    _expect_dtype(src, torch.float32, "src"); _expect_dtype(dst, torch.float32, "dst")
    if src.size() != dst.size() or src.batch != dst.batch or src.num_channels() != dst.num_channels():
        raise ImageError.InvalidImageSize(src.cols(), src.rows(), dst.cols(), dst.rows())
    c = src.num_channels()
    if len(mean) != c or len(std) != c:
        raise ValueError("mean/std must have one entry per channel")
    _check(_lib.lib().kb200_normalize_mean_std_f32(_stream(dev), src.data.data_ptr(), dst.data.data_ptr(),
                                                  src.rows() * src.cols() * src.batch, c, _lib.f3(mean, c), _lib.f3(std, c)))


def find_min_max(image: Image) -> tuple[float, float]:
    """normalize.rs:123 — synchronises (returns host scalars)."""
    if not image.is_device:
        raise ImageError.HostPathNotBuilt("find_min_max")
    if image.numel() == 0:
        raise ImageError.ImageDataNotInitialized()
    _expect_dtype(image, torch.float32, "image")
    dev = image.device
    _lib.set_device(dev.index)
    mm = torch.empty(2, dtype=torch.float32, device=dev)
    _check(_lib.lib().kb200_find_min_max_f32(_stream(dev), image.data.data_ptr(), image.numel(), mm.data_ptr()))
    lo, hi = mm.tolist()
    return lo, hi


def normalize_min_max(src: Image, dst: Image, min: float, max: float) -> None:
    """normalize.rs:191 — (x - min_v) * (max - min) / (max_v - min_v) + min; min_v/max_v found on the device, no sync."""
    dev = _prep("normalize_min_max", src, dst)
    _expect_dtype(src, torch.float32, "src"); _expect_dtype(dst, torch.float32, "dst")
    if src.size() != dst.size() or src.batch != dst.batch or src.num_channels() != dst.num_channels():
        raise ImageError.InvalidImageSize(src.cols(), src.rows(), dst.cols(), dst.rows())
    if src.numel() == 0:
        raise ImageError.ImageDataNotInitialized()
    mm = torch.empty(2, dtype=torch.float32, device=dev)
    l = _lib.lib()
    _check(l.kb200_find_min_max_f32(_stream(dev), src.data.data_ptr(), src.numel(), mm.data_ptr()))
    _check(l.kb200_normalize_min_max_f32(_stream(dev), src.data.data_ptr(), dst.data.data_ptr(), src.numel(), min, max, mm.data_ptr()))


def normalize_rgb_u8(src, dst, npixels: int, scale: Sequence[float], offset: Sequence[float], leaf: int = DEFAULT_LEAF) -> None:
    """normalize.rs:235 — u8 RGB → f32: src[i]*scale[ch] + offset[ch] (`src`, `dst`: tensors or Images)."""
    s = src.data if isinstance(src, Image) else src
    d = dst.data if isinstance(dst, Image) else dst
    if not (s.is_cuda and d.is_cuda):
        raise ImageError.HostPathNotBuilt("normalize_rgb_u8") if not (s.is_cuda or d.is_cuda) else ImageError.MixedResidency()
    if s.device != d.device:
        raise ImageError.DeviceMismatch()
    if s.dtype != torch.uint8 or d.dtype != torch.float32:
        raise ImageError.DtypeMismatch("u8->f32", (s.dtype, d.dtype))
    if s.numel() < npixels * 3 or d.numel() < npixels * 3:
        raise ImageError.InvalidChannelShape(min(s.numel(), d.numel()), npixels * 3)
    _lib.set_device(s.device.index)
    _check(_lib.lib().kb200_normalize_rgb_u8_f32(_stream(s.device), s.data_ptr(), d.data_ptr(), npixels, _lib.f3(scale), _lib.f3(offset), leaf))


def std_mean_sums(image: Image) -> torch.Tensor:
    """The six exact integer sums (Σp per channel, Σp² per channel) as a device uint64[6] tensor — no sync.
    Shard-wise sums add (one all-reduce over 6 integers gives the global statistic, SURVEY §8(e))."""
    if not image.is_device:
        raise ImageError.HostPathNotBuilt("std_mean")
    _expect_dtype(image, torch.uint8, "image")
    if image.num_channels() != 3:
        raise ImageError.InvalidChannelShape(image.num_channels(), 3)
    dev = image.device
    _lib.set_device(dev.index)
    sums = torch.empty(6, dtype=torch.int64, device=dev)
    _check(_lib.lib().kb200_std_mean_u8_c3(_stream(dev), image.data.data_ptr(), image.rows() * image.cols() * image.batch, sums.data_ptr()))
    return sums


def std_mean_finalize(sums, npixels: int) -> tuple[list[float], list[float]]:
    """core.rs:58-66 in f64, same operation order.  Returns (std, mean) like the reference."""
    arr = (C.c_uint64 * 6)(*[int(v) for v in sums])
    std, mean = (C.c_double * 3)(), (C.c_double * 3)()
    _lib.lib().kb200_std_mean_finalize(arr, npixels, std, mean)
    return list(std), list(mean)


def std_mean(image: Image) -> tuple[list[float], list[float]]:
    """core.rs:42 `std_mean(&Image<u8,3>) -> (std, mean)` (synchronises to return host f64s)."""
    sums = std_mean_sums(image).tolist()
    return std_mean_finalize(sums, image.rows() * image.cols() * image.batch)


# ── Gaussian pyramids (pyramid.rs) ───────────────────────────────────────────
def _pyr(op: str, src: Image, dst: Image, up: bool) -> None:
    dev = _prep(op, src, dst)
    if src.dtype not in (torch.float32, torch.uint8) or dst.dtype != src.dtype:
        raise ImageError.DtypeMismatch("f32 or u8, equal on both sides", (src.dtype, dst.dtype))
    c = src.num_channels()
    if dst.num_channels() != c:
        raise ImageError.InvalidChannelShape(dst.num_channels(), c)
    ew, eh = (src.cols() * 2, src.rows() * 2) if up else ((src.cols() + 1) // 2, (src.rows() + 1) // 2)
    if dst.cols() != ew or dst.rows() != eh:   # pyramid.rs:217-225 / :319-327
        raise ImageError.InvalidImageSize(ew, eh, dst.cols(), dst.rows())
    n = _same_batch(src, dst)
    name = f"kb200_pyr{'up' if up else 'down'}_{'f32' if src.dtype == torch.float32 else 'u8'}"
    _check(getattr(_lib.lib(), name)(_stream(dev), src.data.data_ptr(), src.numel(), dst.data.data_ptr(), dst.numel(), src.cols(), src.rows(), c, n))


def pyrdown(src: Image, dst: Image) -> None:
    """pyramid.rs:312 `pyrdown_f32` / :469 `pyrdown_u8` — 5x5 Gaussian + 2x decimation, BORDER_REFLECT_101; dst = ceil(src / 2)."""
    _pyr("pyrdown", src, dst, False)


def pyrup(src: Image, dst: Image) -> None:
    """pyramid.rs:210 `pyrup_f32` / :804 `pyrup_u8` — 2x polyphase upsampling; dst = 2 * src."""
    _pyr("pyrup", src, dst, True)


def build_pyramid(src: Image, max_level: int) -> list[Image]:
    """pyramid.rs:431 `build_pyramid` — [src, pyrdown(src), ...] with max_level + 1 entries (level sizes by div_ceil)."""
    levels = [src]
    for _ in range(max_level):
        cur = levels[-1]
        nxt = Image.zeros_cuda(ImageSize((cur.cols() + 1) // 2, (cur.rows() + 1) // 2), cur.num_channels(), cur.dtype, cur.device, batch=cur.batch)
        pyrdown(cur, nxt)
        levels.append(nxt)
    return levels


# ── calibration: undistort maps (calibration/distortion.rs) ──────────────────
def generate_correction_map_polynomial(intrinsic: Sequence[float], distortion: Sequence[float], size: ImageSize, device) -> tuple[Image, Image]:
    """calibration/distortion.rs:135 — (map_x, map_y), each an H x W x 1 f32 device Image, for `remap`: the distorted source
    coordinate of every destination pixel under the polynomial (Brown-Conrady rational) model.  `intrinsic` = (fx, fy, cx,
    cy) of CameraIntrinsic, `distortion` = (k1, k2, k3, k4, k5, k6, p1, p2) of PolynomialDistortion.  Generated on the
    device — the reference builds the maps on the host and uploads them."""
    if len(intrinsic) != 4 or len(distortion) != 8:
        raise ValueError("intrinsic = (fx, fy, cx, cy), distortion = (k1..k6, p1, p2)")
    dev = torch.device(device)
    _lib.set_device(dev.index if dev.index is not None else torch.cuda.current_device())
    mx = Image.zeros_cuda(size, 1, torch.float32, dev)
    my = Image.zeros_cuda(size, 1, torch.float32, dev)
    _check(_lib.lib().kb200_generate_correction_map_polynomial(_stream(dev), (C.c_double * 4)(*[float(v) for v in intrinsic]),
                                                              (C.c_double * 8)(*[float(v) for v in distortion]), size.width, size.height,
                                                              mx.data.data_ptr(), my.data.data_ptr(), mx.numel()))
    return mx, my
