"""`Image<T,C>` and friends — the containers the hot path's signatures mention (SURVEY §8(a) a13).

Mirrors kornia-image (`crates/kornia-image/src/image.rs:25,60,138`, `error.rs:3-121`, `cuda.rs:53-219`,
`dlpack.rs:35,81`): an image is a tight, contiguous HWC tensor; `Image.to_cuda / zeros_cuda /
to_host_owned` move it between residencies; a device image exports `__dlpack__` and
`__cuda_array_interface__` (CAI v3: `shape, typestr, data(ptr, False), strides None, version 3,
stream` — kornia-py/src/cuda_ext/mod.rs:438-480) so torch / CuPy / TensorRT consume it zero-copy.

Storage is a `torch.Tensor` (device memory + streams are torch's; that is plumbing, not the product).
A batch of same-sized images is an Image whose tensor has a leading N dimension ([N,H,W,C]) — the
reference loops over frames; here batch is a kernel grid dimension.
"""
from __future__ import annotations

import enum
from dataclasses import dataclass

import torch


class ImageError(Exception):
    """kornia_image::ImageError (error.rs).  `kind` names the variant."""

    def __init__(self, kind: str, message: str):
        super().__init__(message)
        self.kind = kind

    # constructors named after the reference variants
    @staticmethod
    def InvalidImageSize(a, b, c, d):
        return ImageError("InvalidImageSize", f"Invalid image size ({a}, {b}) mismatch ({c}, {d})")

    @staticmethod
    def InvalidChannelShape(a, b):
        return ImageError("InvalidChannelShape", f"Data length ({a}) does not match the image size ({b})")

    @staticmethod
    def MixedResidency():
        return ImageError("MixedResidency", "source and destination have different residency (host vs device)")

    @staticmethod
    def DeviceMismatch():
        return ImageError("DeviceMismatch", "source and destination device images are on different CUDA devices; move both to one device")

    @staticmethod
    def Cuda(msg):
        return ImageError("Cuda", f"CUDA error: {msg}")

    @staticmethod
    def CannotComputeDeterminant():
        return ImageError("CannotComputeDeterminant", "Cannot compute the determinant: matrix is singular")

    @staticmethod
    def InvalidKernelLength(a, b):
        return ImageError("InvalidKernelLength", f"Invalid kernel length {a} and {b}")

    @staticmethod
    def InvalidSigmaValue(a, b):
        return ImageError("InvalidSigmaValue", f"Invalid sigma values {a} and {b}")

    @staticmethod
    def UnsupportedChannelCount(c):
        return ImageError("UnsupportedChannelCount", f"Unsupported channel count {c}")

    @staticmethod
    def UnsupportedInterpolation(m):
        return ImageError("UnsupportedInterpolation", f"Unsupported interpolation mode: {m!r}")

    @staticmethod
    def ImageDataNotInitialized():
        return ImageError("ImageDataNotInitialized", "Image data is not initialized")

    @staticmethod
    def ImageDataNotContiguous():
        return ImageError("ImageDataNotContiguous", "Image data is not contiguous")

    @staticmethod
    def DtypeMismatch(expected, got):
        return ImageError("DtypeMismatch", f"pixel format mismatch: expected {expected}, got {got}")

    @staticmethod
    def HostPathNotBuilt(op):
        # The reference runs its rayon/SIMD CPU path for host pairs.  This build is the device path only
        # and NEVER falls back to a CPU implementation: host operands are a typed error.
        return ImageError("UnsupportedDevice", f"{op}: host-resident operands — this build implements the device path only; "
                          "move the images to the device (Image.to_cuda)")


class InterpolationMode(enum.Enum):
    """kornia_image::InterpolationMode (image.rs:25)."""
    Nearest = 0
    Bilinear = 1
    Bicubic = 2
    Lanczos = 3


@dataclass(frozen=True)
class ImageSize:
    """kornia_image::ImageSize (image.rs:60)."""
    width: int
    height: int


_TYPESTR = {torch.float32: "<f4", torch.float16: "<f2", torch.uint8: "|u1", torch.float64: "<f8", torch.uint16: "<u2"}


class Image:
    """A tight HWC (or batched NHWC) image over a contiguous torch tensor."""

    __slots__ = ("data",)

    def __init__(self, size_or_tensor, data=None, channels: int | None = None, dtype=None):
        if isinstance(size_or_tensor, torch.Tensor) and data is None:
            t = size_or_tensor
        else:  # Image::new(size, data) — image.rs:180: data length must match
            size = size_or_tensor
            t = torch.as_tensor(data, dtype=dtype)
            if channels is None:
                if t.numel() % (size.width * size.height) != 0:
                    raise ImageError.InvalidChannelShape(t.numel(), size.width * size.height)
                channels = t.numel() // (size.width * size.height)
            if t.numel() != size.width * size.height * channels:
                raise ImageError.InvalidChannelShape(t.numel(), size.width * size.height * channels)
            t = t.reshape(size.height, size.width, channels)
        if t.dim() not in (3, 4):
            raise ImageError("InvalidImageShape", f"expected [H,W,C] or [N,H,W,C], got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ImageError.ImageDataNotContiguous()
        self.data = t

    # ── constructors ────────────────────────────────────────────────────────
    @staticmethod
    def from_size_val(size: ImageSize, val, channels: int, dtype=torch.float32, device="cpu", batch: int | None = None) -> "Image":
        shape = (size.height, size.width, channels) if batch is None else (batch, size.height, size.width, channels)
        return Image(torch.full(shape, val, dtype=dtype, device=device))

    @staticmethod
    def zeros_cuda(size: ImageSize, channels: int, dtype=torch.float32, device="cuda", batch: int | None = None) -> "Image":
        """kornia-image/src/cuda.rs `zeros_cuda`."""
        return Image.from_size_val(size, 0, channels, dtype, device, batch)

    @staticmethod
    def from_dlpack(obj) -> "Image":
        """Zero-copy import of any `__dlpack__` producer (kornia-image/src/dlpack.rs:81)."""
        return Image(torch.from_dlpack(obj))

    @staticmethod
    def from_cuda_array_interface(obj) -> "Image":
        """Zero-copy import of a `__cuda_array_interface__` producer (CuPy, numba, cuda-python …)."""
        return Image(torch.as_tensor(obj, device="cuda"))

    # ── residency ───────────────────────────────────────────────────────────
    def to_cuda(self, device="cuda", non_blocking: bool = False) -> "Image":
        return Image(self.data.to(device, non_blocking=non_blocking).contiguous())

    def to_host_owned(self) -> "Image":
        return Image(self.data.cpu())

    @property
    def is_device(self) -> bool:
        return self.data.is_cuda

    @property
    def device(self) -> torch.device:
        return self.data.device

    # ── geometry ────────────────────────────────────────────────────────────
    @property
    def batch(self) -> int:
        return self.data.shape[0] if self.data.dim() == 4 else 1

    @property
    def is_batched(self) -> bool:
        return self.data.dim() == 4

    def rows(self) -> int:
        return self.data.shape[-3]

    def cols(self) -> int:
        return self.data.shape[-2]

    def height(self) -> int:
        return self.rows()

    def width(self) -> int:
        return self.cols()

    def num_channels(self) -> int:
        return self.data.shape[-1]

    def size(self) -> ImageSize:
        return ImageSize(self.cols(), self.rows())

    @property
    def dtype(self):
        return self.data.dtype

    def numel(self) -> int:
        return self.data.numel()

    def as_tensor(self) -> torch.Tensor:
        return self.data

    def as_slice(self) -> torch.Tensor:
        return self.data.reshape(-1)

    def numpy(self):
        return self.data.detach().cpu().numpy()

    # ── interop ─────────────────────────────────────────────────────────────
    def __dlpack__(self, stream=None, **kw):
        return self.data.__dlpack__(stream=stream, **kw) if stream is not None or kw else self.data.__dlpack__()

    def __dlpack_device__(self):
        return self.data.__dlpack_device__()

    @property
    def __cuda_array_interface__(self):
        if not self.is_device:
            raise AttributeError("__cuda_array_interface__ is only present on a device Image")
        t = self.data
        raw = torch.cuda.current_stream(t.device).cuda_stream
        return {
            "shape": tuple(t.shape),
            "typestr": _TYPESTR[t.dtype],
            "data": (t.data_ptr(), False),
            "strides": None,
            "version": 3,
            "stream": 1 if raw == 0 else int(raw),  # cai_stream_value: legacy default stream is 1
        }

    def __repr__(self):
        return f"Image(shape={tuple(self.data.shape)}, dtype={self.data.dtype}, device={self.data.device})"


def pair_residency(op: str, *images: Image) -> torch.device:
    """cuda/dispatch.rs:105-130: both host → (CPU path, not built here); both device → launch; mixed → error;
    different devices → DeviceMismatch.  Returns the device to launch on."""
    dev_flags = [im.is_device for im in images]
    if all(dev_flags):
        d0 = images[0].device
        if any(im.device != d0 for im in images[1:]):
            raise ImageError.DeviceMismatch()
        return d0
    if not any(dev_flags):
        raise ImageError.HostPathNotBuilt(op)
    raise ImageError.MixedResidency()
