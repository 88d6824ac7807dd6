"""kornia-rs_b200 — the H100 (sm_90a) implementation of kornia-rs's kornia-imgproc pixel-kernel hot
path, behind the reference's own operator surface.

    import kornia_rs_b200 as kb
    src = kb.Image(torch_u8_hwc_cuda_tensor)
    kb.imgproc.resize(src_f32, dst_f32, kb.InterpolationMode.Bilinear)
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).normalize(kb.Normalize.imagenet()).build_cuda()
    pre.run_raw_batch(frames, 1920, 1080, dst)        # one launch for the whole batch

Layers: `_lib` (ctypes over include/kornia_b200.h → lib/libkornia_b200.so, hand-written CUDA in csrc/),
`image` (Image<T,C> / errors / DLPack / __cuda_array_interface__), `imgproc` (the operators),
`preprocess` (Preprocessor), `dist` (one-process-per-GPU sharding).  No CPU fallback anywhere: if the
native library is missing, importing this package raises.
"""
from . import _lib

_lib.lib()  # fail loudly at import when libkornia_b200.so is absent

from . import dist, fusion, imgproc  # noqa: E402
from .image import Image, ImageError, ImageSize, InterpolationMode  # noqa: E402
from .imgproc import YuvMatrix  # noqa: E402
from .preprocess import (  # noqa: E402
    IMAGENET_MEAN,
    IMAGENET_STD,
    Normalize,
    PitchedSurface,
    PreprocessError,
    Preprocessor,
    PreprocessorBuilder,
    ResizeMode,
    SourceFormat,
)

__version__ = "0.1.0"


def native_version() -> int:
    return _lib.lib().kb200_version()


def device_info() -> dict:
    import ctypes as C

    sm, major, minor = C.c_int(), C.c_int(), C.c_int()
    st = _lib.lib().kb200_device_info(C.byref(sm), C.byref(major), C.byref(minor))
    if st != 0:
        raise RuntimeError(_lib.last_error())
    return {"sm_count": sm.value, "cc": (major.value, minor.value)}


__all__ = [
    "Image", "ImageError", "ImageSize", "InterpolationMode", "imgproc", "dist", "fusion", "Preprocessor", "PreprocessorBuilder",
    "PreprocessError", "ResizeMode", "Normalize", "SourceFormat", "YuvMatrix", "PitchedSurface", "IMAGENET_MEAN", "IMAGENET_STD",
    "native_version", "device_info",
]
