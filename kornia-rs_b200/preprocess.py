"""`Preprocessor` — the fused camera preprocess (a12), mirroring preprocess.rs:67-149, :654-1282.

Built once via `Preprocessor.builder()…build_cuda()`, then applied to any number of frames of any
resolution: the target H/W is read from the destination tensor each call.  Camera formats
(NV12 / YUYV / Gray, the other YUV layouts, the 10- and 12-bit 4:2:0 video P010 / P012 / I010 / I012, the 4:4:4 video
I444 / I410 / I412 / I410Msb / I412Msb and the 8- to
16-bit Bayer mosaics, unpacked or MIPI-packed) go through `run_raw*`; colour decode is fused into the resample taps.  Unlike the
reference (one launch per frame, preprocess.rs:1277-1280) a batch is ONE launch.

Only the CUDA preprocessor exists here (`build()` = the reference's CPU preprocessor is out of scope:
it raises).  Errors mirror `PreprocessError` (preprocess.rs:252-332).
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass
from typing import NamedTuple, Sequence

import torch

from . import _lib
from .image import Image, InterpolationMode
from .imgproc import YuvMatrix

IMAGENET_MEAN = (0.485, 0.456, 0.406)  # preprocess.rs:93
IMAGENET_STD = (0.229, 0.224, 0.225)   # preprocess.rs:95

# The output dtype of each kb200_out_format, indexed by it.  The Preprocessor's internal `out` arguments are these codes,
# so False and True still mean f32 and f16.
_OUT_DTYPES = (torch.float32, torch.float16, torch.bfloat16)
_TABLE_ENTRIES = ("kb200_preprocess_f32", "kb200_preprocess_f16", "kb200_preprocess_bf16")
_STRIDED_ENTRIES = ("kb200_preprocess_strided_f32", "kb200_preprocess_strided_f16", "kb200_preprocess_strided_bf16")


class PreprocessError(Exception):
    """preprocess.rs:252-332; `kind` names the variant."""

    def __init__(self, kind: str, message: str, **fields):
        super().__init__(message)
        self.kind = kind
        self.fields = fields


class ResizeMode(enum.Enum):  # preprocess.rs:67
    Letterbox = 0
    Stretch = 1


class SourceFormat(enum.Enum):  # preprocess.rs:130
    Rgb8 = "rgb8"
    Bgr8 = "bgr8"
    Rgba8 = "rgba8"
    Bgra8 = "bgra8"
    Gray8 = "gray8"
    Nv12 = "nv12"
    Yuyv = "yuyv"
    # Beyond the reference's SourceFormat: the other 4:2:0 layouts (tight w*h*3/2 frames, like Nv12) and 4:2:2 layouts
    # (w*h*2, like Yuyv).  Each decodes to exactly what its byte-repacked Nv12 / Yuyv twin decodes to.
    Nv21 = "nv21"
    I420 = "i420"
    Yv12 = "yv12"
    Uyvy = "uyvy"
    Yvyu = "yvyu"
    # Beyond the reference too: 8-bit Bayer mosaics (one byte per pixel, w*h like Gray8, at least 3x3), named by their
    # 2x2 quad read row-major.  A tap is the bilinear demosaic of OpenCV's cvtColor(COLOR_Bayer??2RGB) at that pixel.
    BayerRggb = "bayer_rggb"
    BayerBggr = "bayer_bggr"
    BayerGrbg = "bayer_grbg"
    BayerGbrg = "bayer_gbrg"
    # 10- to 16-bit Bayer mosaics: one little-endian 16-bit word per sample, the value in its low bits (V4L2's unpacked
    # SRGGB10 ... SGBRG16), rows of 2*w bytes.  The demosaic is the 8-bit one on the 16-bit values; the bit depth sets
    # only the white level W = 2^bits - 1 a tap is normalised by, (px / W - mean) * inv_std.  pad_value stays 0..255.
    BayerRggb10 = "bayer_rggb10"
    BayerBggr10 = "bayer_bggr10"
    BayerGrbg10 = "bayer_grbg10"
    BayerGbrg10 = "bayer_gbrg10"
    BayerRggb12 = "bayer_rggb12"
    BayerBggr12 = "bayer_bggr12"
    BayerGrbg12 = "bayer_grbg12"
    BayerGbrg12 = "bayer_gbrg12"
    BayerRggb14 = "bayer_rggb14"
    BayerBggr14 = "bayer_bggr14"
    BayerGrbg14 = "bayer_grbg14"
    BayerGbrg14 = "bayer_gbrg14"
    BayerRggb16 = "bayer_rggb16"
    BayerBggr16 = "bayer_bggr16"
    BayerGrbg16 = "bayer_grbg16"
    BayerGbrg16 = "bayer_gbrg16"
    # The 10-, 12- and 14-bit mosaics MIPI CSI-2 packed (V4L2's SRGGB10P ... SGBRG14P): each row packed on its own in
    # w*bits/8 bytes, groups of 4 samples in 5 bytes (RAW10), 2 in 3 (RAW12) or 4 in 7 (RAW14), the first bytes of a
    # group holding the high 8 bits of each sample.  A tap is exactly the tap of the unpacked format of the same depth.
    BayerRggb10p = "bayer_rggb10p"
    BayerBggr10p = "bayer_bggr10p"
    BayerGrbg10p = "bayer_grbg10p"
    BayerGbrg10p = "bayer_gbrg10p"
    BayerRggb12p = "bayer_rggb12p"
    BayerBggr12p = "bayer_bggr12p"
    BayerGrbg12p = "bayer_grbg12p"
    BayerGbrg12p = "bayer_gbrg12p"
    BayerRggb14p = "bayer_rggb14p"
    BayerBggr14p = "bayer_bggr14p"
    BayerGrbg14p = "bayer_grbg14p"
    BayerGbrg14p = "bayer_gbrg14p"
    # 10- and 12-bit 4:2:0 video: tight frames of w*h*3/2 little-endian 16-bit words (3*w*h bytes), w and h even.  P010 /
    # P012 (NVDEC, VA-API and V4L2 output of HEVC Main10, AV1 10-bit) are Nv12's layout with each code in the high bits of
    # its word; I010 / I012 (libavcodec's yuv420p10le / yuv420p12le) are I420's with each code in the low bits.  A tap is
    # the decoded n-bit RGB code normalised by W = 2^n - 1, (px / W - mean) * inv_std; pad_value stays 0..255.
    P010 = "p010"
    P012 = "p012"
    I010 = "i010"
    I012 = "i012"
    # 4:4:4 video: three full-resolution planes Y, U, V, every pixel with its own chroma; any w and h.  I444: w*h bytes each
    # (libavcodec's yuv444p, nvJPEG's planar 4:4:4, NVDEC's YUV444 surface), decoded like I420.  I410 / I412: w*h
    # little-endian 16-bit words each (6*w*h bytes), the code in the low bits (yuv444p10le / yuv444p12le); I410Msb /
    # I412Msb: the code in the high bits (NVDEC's YUV444_16Bit surface of 10- and 12-bit content).  A 16-bit tap is
    # normalised like a P010 tap by W = 2^n - 1; pad_value stays 0..255.
    I444 = "i444"
    I410 = "i410"
    I412 = "i412"
    I410Msb = "i410msb"
    I412Msb = "i412msb"

    def _rec(self) -> "_Rec":
        return _RECORDS[self.name]

    def fmt_code(self) -> int:  # :153-161
        return self._rec().code

    def bpp(self) -> int:  # :164-171
        """Bytes per sample; 1 for the packed Bayer formats, whose rows pitch() counts."""
        return self._rec().bpp or 1

    def pitch(self, w: int) -> int:
        """Bytes of a tight row of w pixels."""
        r = self._rec()
        return w * r.bits // 8 if r.bpp == 0 else w * r.bpp

    def is_yuv420(self) -> bool:
        """An 8-bit 4:2:0 format (one byte per sample); is_yuv16() names the 16-bit-word ones."""
        return self._rec().family == "yuv420" and self._rec().bpp == 1

    def is_yuv16(self) -> bool:
        """A 10- or 12-bit 4:2:0 format of 16-bit words: P010, P012, I010, I012."""
        return self._rec().family == "yuv420" and self._rec().bpp == 2

    def is_yuv422(self) -> bool:
        return self._rec().family == "yuv422"

    def is_yuv444(self) -> bool:
        """A 4:4:4 format: I444 (bytes) or I410, I412, I410Msb, I412Msb (16-bit words)."""
        return self._rec().family == "yuv444"

    def is_yuv(self) -> bool:
        """A YUV format: one a YuvMatrix applies to."""
        return self._rec().family in ("yuv420", "yuv422", "yuv444")

    def is_bayer(self) -> bool:
        return self._rec().family == "bayer"

    def is_bayer16(self) -> bool:
        """A Bayer format of 16-bit samples (10 to 16 bits per pixel)."""
        return self.is_bayer() and self._rec().bpp == 2

    def is_bayer_packed(self) -> bool:
        """A MIPI-packed Bayer format (10, 12 or 14 bits per pixel)."""
        return self.is_bayer() and self._rec().bpp == 0

    def bit_depth(self) -> int | None:
        """Bits per sample of a Bayer format (8 for the byte mosaics), of a 16-bit-word 4:2:0 format (10, 12) or of a 4:4:4
        format (8, 10, 12), None for the other formats."""
        return self._rec().bits

    def buffer_len(self, w: int, h: int) -> int:  # :177-186
        # 4:2:0 chroma after the luma rows: w*h/2 samples, of 1 byte (is_yuv420) or 2 bytes (is_yuv16)
        chroma = w * h // 2 if self.is_yuv420() else w * h if self.is_yuv16() else 0
        if self.is_yuv444():   # two more full planes
            return self.pitch(w) * h * 3
        return self.pitch(w) * h + chroma

    def dims_ok(self, w: int, h: int) -> bool:  # :188-195
        if self.is_yuv420() or self.is_yuv16():
            return w % 2 == 0 and h % 2 == 0
        if self.is_yuv422():
            return w % 2 == 0
        if self.is_bayer_packed():   # whole packed groups: 2 samples at 12 bits, 4 at 10 and 14
            return w >= 3 and h >= 3 and w % (2 if self.bit_depth() == 12 else 4) == 0
        if self.is_bayer():
            return w >= 3 and h >= 3
        return True

    def interleaved(self) -> bool:  # :211-216
        return self._rec().family == "rgb"

    @staticmethod
    def from_name(name: str):  # :221-233
        name = name.lower()
        return next((m for m in SourceFormat if name == m.value or name in m._rec().aliases), None)


class _Rec(NamedTuple):   # one SourceFormat's facts
    code: int                 # kb200_src_fmt
    family: str               # "rgb" (interleaved RGB / BGR, with or without alpha), "gray", "yuv420", "yuv422", "yuv444" or "bayer"
    bits: int | None = None   # bits per sample of a Bayer, 16-bit-word 4:2:0 or 4:4:4 format
    bpp: int = 1              # bytes per sample (per pixel for "rgb" and "yuv422"); 0: MIPI-packed, bits / 8 per sample
    aliases: tuple = ()       # from_name spellings besides the value


_RECORDS = {
    "Rgb8": _Rec(0, "rgb", bpp=3, aliases=("rgb",)), "Bgr8": _Rec(1, "rgb", bpp=3, aliases=("bgr",)),
    "Rgba8": _Rec(0, "rgb", bpp=4, aliases=("rgba",)), "Bgra8": _Rec(1, "rgb", bpp=4, aliases=("bgra",)),
    "Gray8": _Rec(2, "gray", aliases=("gray",)), "Nv12": _Rec(3, "yuv420"), "Yuyv": _Rec(4, "yuv422", bpp=2),
    "Nv21": _Rec(5, "yuv420"), "I420": _Rec(6, "yuv420"), "Yv12": _Rec(7, "yuv420"),
    "Uyvy": _Rec(8, "yuv422", bpp=2), "Yvyu": _Rec(9, "yuv422", bpp=2),
    "P010": _Rec(80, "yuv420", 10, 2, ("p010le",)), "P012": _Rec(81, "yuv420", 12, 2, ("p012le",)),
    "I010": _Rec(82, "yuv420", 10, 2, ("yuv420p10le",)), "I012": _Rec(83, "yuv420", 12, 2, ("yuv420p12le",)),
    "I444": _Rec(11, "yuv444", 8, 1, ("yuv444p",)),
    "I410": _Rec(85, "yuv444", 10, 2, ("yuv444p10le",)), "I412": _Rec(86, "yuv444", 12, 2, ("yuv444p12le",)),
    "I410Msb": _Rec(87, "yuv444", 10, 2), "I412Msb": _Rec(88, "yuv444", 12, 2),
}
for _k, _p in enumerate(("rggb", "bggr", "grbg", "gbrg")):   # kb200_bayer_pattern order; codes 16 + pattern; 32 + 4*d + pattern, d = 0..3; 64 + 4*d + pattern, d = 0..2
    _RECORDS[f"Bayer{_p.capitalize()}"] = _Rec(16 + _k, "bayer", 8)
    for _d, _b in enumerate((10, 12, 14, 16)):
        _RECORDS[f"Bayer{_p.capitalize()}{_b}"] = _Rec(32 + 4 * _d + _k, "bayer", _b, 2)
    for _d, _b in enumerate((10, 12, 14)):
        _RECORDS[f"Bayer{_p.capitalize()}{_b}p"] = _Rec(64 + 4 * _d + _k, "bayer", _b, 0)


@dataclass(frozen=True)
class Normalize:  # preprocess.rs:77
    mean: tuple | None = None
    std: tuple | None = None

    @staticmethod
    def UnitScale() -> "Normalize":
        return Normalize()

    @staticmethod
    def MeanStd(mean, std) -> "Normalize":
        return Normalize(tuple(mean), tuple(std))

    @staticmethod
    def imagenet() -> "Normalize":
        return Normalize(IMAGENET_MEAN, IMAGENET_STD)

    def mean_inv_std(self):  # :113-125, f32 arithmetic for 1/std
        if self.mean is None:
            return (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)
        import math

        std32 = torch.tensor(self.std, dtype=torch.float32)
        mean32 = torch.tensor(self.mean, dtype=torch.float32)
        if any((not math.isfinite(s)) or s <= 0.0 for s in std32.tolist()) or any(not math.isfinite(m) for m in mean32.tolist()):
            raise PreprocessError("InvalidNormalize", f"invalid normalize: mean {self.mean} must be finite, std {self.std} must be finite and > 0",
                                  mean=self.mean, std=self.std)
        inv = (torch.tensor(1.0, dtype=torch.float32) / std32).tolist()
        return tuple(mean32.tolist()), tuple(inv)


@dataclass
class PitchedSurface:  # preprocess.rs:380-392
    data: torch.Tensor
    width: int
    height: int
    row_pitch: int
    channels: int

    def validate(self) -> None:  # :829-842
        if self.channels not in (3, 4):
            raise PreprocessError("UnsupportedChannels", f"unsupported source channel count {self.channels} (expected 3 or 4)")
        if (self.row_pitch < self.width * self.channels or self.data.numel() < self.row_pitch * self.height
                or self.width == 0 or self.height == 0):
            raise PreprocessError("InvalidSurface", "invalid pitched surface (need pitch >= width*channels and len >= pitch*height)")


class PreprocessorBuilder:  # preprocess.rs:654-779
    def __init__(self):
        self._mode = ResizeMode.Letterbox
        self._normalize = Normalize.UnitScale()
        self._pad_value = 114
        self._sampling = InterpolationMode.Bilinear
        self._source_format = SourceFormat.Rgb8
        self._yuv_matrix = YuvMatrix.Bt601Limited

    def source_format(self, fmt: SourceFormat):
        self._source_format = fmt
        return self

    def mode(self, mode: ResizeMode):
        self._mode = mode
        return self

    def normalize(self, normalize: Normalize):
        self._normalize = normalize
        return self

    def pad_value(self, pad_value: int):
        self._pad_value = int(pad_value) & 0xFF
        return self

    def sampling(self, sampling: InterpolationMode):
        self._sampling = sampling
        return self

    def yuv_matrix(self, matrix: YuvMatrix):
        """The colour matrix and range YUV frames decode with (default Bt601Limited, the reference's decode).  Only the YUV
        source formats take one: build_cuda() rejects any other matrix on an RGB, Gray or Bayer format."""
        self._yuv_matrix = YuvMatrix(matrix)
        return self

    def _validated(self):
        if self._sampling not in (InterpolationMode.Nearest, InterpolationMode.Bilinear, InterpolationMode.Lanczos):
            raise PreprocessError("UnsupportedSampling", f"unsupported sampling mode {self._sampling!r} (expected Nearest, Bilinear, or Lanczos)")
        if self._yuv_matrix != YuvMatrix.Bt601Limited and not self._source_format.is_yuv():
            raise PreprocessError("YuvMatrixNeedsYuvSource", f"YUV matrix {self._yuv_matrix!r} given for source format {self._source_format!r}, "
                                  "which is not a YUV format", matrix=self._yuv_matrix, format=self._source_format)
        return self._normalize.mean_inv_std()

    def build(self):
        """The reference's CPU preprocessor (host image → host tensor) is out of this tier's scope."""
        self._validated()
        raise PreprocessError("NotDeviceImage", "CPU preprocessor not built in this tier: use build_cuda() (device operands)")

    def build_cuda(self, device: str | torch.device | None = None) -> "Preprocessor":
        mean, inv_std = self._validated()
        _lib.lib()  # fail loudly if the native library is missing
        return Preprocessor(self._mode, self._sampling, self._source_format, mean, inv_std, float(self._pad_value),
                            torch.device(device) if device is not None else None, self._yuv_matrix)


class Preprocessor:
    def __init__(self, mode, sampling, source_format, mean, inv_std, pad_value, device, yuv_matrix=YuvMatrix.Bt601Limited):
        self._mode, self._sampling, self._fmt = mode, sampling, source_format
        self._mean, self._inv_std, self._pad = mean, inv_std, pad_value
        self._device = device
        self._yuv_matrix = YuvMatrix(yuv_matrix)

    @staticmethod
    def builder() -> PreprocessorBuilder:
        return PreprocessorBuilder()

    @staticmethod
    def letterbox(device=None) -> "Preprocessor":
        return PreprocessorBuilder().mode(ResizeMode.Letterbox).build_cuda(device)

    @staticmethod
    def stretch(device=None) -> "Preprocessor":
        return PreprocessorBuilder().mode(ResizeMode.Stretch).build_cuda(device)

    @staticmethod
    def with_mode(mode: ResizeMode, device=None) -> "Preprocessor":
        return PreprocessorBuilder().mode(mode).build_cuda(device)

    def mode(self) -> ResizeMode:
        return self._mode

    def yuv_matrix(self) -> YuvMatrix:
        return self._yuv_matrix

    # ── helpers ─────────────────────────────────────────────────────────────
    def _desc(self, sw, sh, pitch, bpp, fmt_code, dw, dh) -> _lib.PreprocessDesc:
        lim = 2 ** 31 - 1
        if sw > lim or sh > lim or pitch > lim or dw * dh > lim:  # :1336-1339
            raise PreprocessError("DimensionsTooLarge", "dimensions exceed the 32-bit CUDA kernel index limit")
        a = (C.c_float * 4)()
        _lib.lib().kb200_preprocess_affine(self._mode.value, sw, sh, dw, dh, a)
        d = _lib.PreprocessDesc()
        d.scale_x, d.scale_y, d.pad_x, d.pad_y = a[0], a[1], a[2], a[3]
        d.src_w, d.src_h, d.src_pitch, d.src_bpp = sw, sh, pitch, bpp
        d.fmt = fmt_code | (int(self._yuv_matrix) << 8)   # KB200_FMT_YUV_MATRIX: 0 unless the format is a YUV one (build_cuda)
        d.dst_w, d.dst_h = dw, dh
        d.mean = (C.c_float * 3)(*self._mean)
        d.inv_std = (C.c_float * 3)(*self._inv_std)
        d.pad_value = self._pad
        d.sampling = {InterpolationMode.Nearest: 0, InterpolationMode.Bilinear: 1, InterpolationMode.Lanczos: 3}[self._sampling]
        return d

    @staticmethod
    def _validate_dst(dst: torch.Tensor, expected_n: int, out: int) -> None:
        shape = tuple(dst.shape)
        if dst.dim() != 4 or shape[1] != 3 or (expected_n == 1 and shape[0] != 1):  # :805-808
            raise PreprocessError("BadOutputShape", f"destination tensor must be [1, 3, H, W], got {list(shape)}")
        if shape[0] != expected_n:
            raise PreprocessError("BatchMismatch", f"destination batch dim {shape[0]} != frame count {expected_n}",
                                  dst_n=shape[0], frames=expected_n)
        if not dst.is_cuda:
            raise PreprocessError("NotDeviceTensor", "CUDA preprocessor requires a device-resident destination tensor")
        want = _OUT_DTYPES[out]
        if dst.dtype != want or not dst.is_contiguous():
            raise PreprocessError("BadOutputShape", f"destination tensor must be contiguous {want}, got {dst.dtype}")

    def _launch(self, desc, frames: Sequence[torch.Tensor], dst: torch.Tensor, out: int) -> None:
        self._call(frames, dst, lambda s, ptrs, lens, n: getattr(_lib.lib(), _TABLE_ENTRIES[out])(
            s, C.byref(desc), ptrs, lens, n, dst.data_ptr(), dst.numel()))

    def _call(self, frames: Sequence[torch.Tensor], dst: torch.Tensor, entry, src_wh: tuple[int, int] | None = None) -> None:
        """One call of a frame-table entry: each frame is checked (its raw size against src_wh = (src_w, src_h) when given,
        then that it is on dst's device), entry(stream, frame pointers, frame lengths, frame count) runs on the current
        stream of dst's device, and a status other than OK is raised.  The region entries build their descriptor inside
        `entry`, so that its DimensionsTooLarge comes after the frame checks."""
        dev = dst.device
        for f in frames:
            if src_wh:
                self._validate_raw(f.numel() * f.element_size(), *src_wh)
            if not f.is_cuda:
                raise PreprocessError("NotDeviceImage", "CUDA preprocessor requires a device-resident source image")
            if f.device != dev:
                raise PreprocessError("Cuda", "CUDA error: source and destination are on different CUDA devices")
        _lib.set_device(dev.index)
        n = len(frames)
        ptrs = (C.c_void_p * max(n, 1))(*[f.data_ptr() for f in frames])
        lens = (C.c_size_t * max(n, 1))(*[f.numel() * f.element_size() for f in frames])
        st = entry(torch.cuda.current_stream(dev).cuda_stream, ptrs, lens, n)
        if st != _lib.OK:
            kind = {_lib.ERR_INVALID_SOURCE: "InvalidRawSource", _lib.ERR_DIMS_TOO_LARGE: "DimensionsTooLarge"}.get(st, "Cuda")
            raise PreprocessError(kind, ("CUDA error: " if kind == "Cuda" else "") + _lib.last_error())

    def _validate_typed_format(self, c: int) -> None:  # :913-923
        f = self._fmt
        ok = (c == 4) if f in (SourceFormat.Rgba8, SourceFormat.Bgra8) else f.interleaved()
        if not ok:
            raise PreprocessError("FormatNeedsRawBuffer", f"source format {f!r} needs run_raw (raw device buffer), not the typed run()")

    def _validate_raw(self, got: int, w: int, h: int) -> None:  # :1287-1300
        f = self._fmt
        need = f.buffer_len(w, h)
        if not f.dims_ok(w, h) or got < need:
            raise PreprocessError("InvalidRawSource", f"invalid raw source for {f!r} at {w}x{h} (got {got} bytes, need {need})",
                                  format=f, width=w, height=h, got=got, need=need)

    # ── typed entries (interleaved RGB/BGR[A] images) ───────────────────────
    def _run_typed(self, src: Image, dst: torch.Tensor, out: int) -> None:
        c = src.num_channels()
        if c not in (3, 4):
            raise PreprocessError("UnsupportedChannels", f"unsupported source channel count {c} (expected 3 or 4)")
        self._validate_dst_shape_only(dst)
        self._validate_typed_format(c)
        if not src.is_device:
            raise PreprocessError("NotDeviceImage", "CUDA preprocessor requires a device-resident source image")
        self._validate_dst(dst, 1, out)
        if src.dtype != torch.uint8 or src.is_batched:
            raise PreprocessError("UnsupportedChannels", "typed run() takes one u8 HWC image")
        w, h = src.width(), src.height()
        desc = self._desc(w, h, w * c, c, self._fmt.fmt_code(), dst.shape[3], dst.shape[2])
        self._launch(desc, [src.data], dst, out)

    @staticmethod
    def _validate_dst_shape_only(dst: torch.Tensor) -> None:
        shape = tuple(dst.shape)
        if dst.dim() != 4 or shape[1] != 3 or shape[0] != 1:
            raise PreprocessError("BadOutputShape", f"destination tensor must be [1, 3, H, W], got {list(shape)}")

    def run(self, src: Image, dst: torch.Tensor) -> None:
        """preprocess.rs:887 — `src` u8 HWC C∈{3,4} → `dst` [1,3,H,W] f32."""
        self._run_typed(src, dst, _lib.OUT_F32)

    def run_f16(self, src: Image, dst: torch.Tensor) -> None:
        """preprocess.rs:1086."""
        self._run_typed(src, dst, _lib.OUT_F16)

    def run_bf16(self, src: Image, dst: torch.Tensor) -> None:
        """`run` into a torch.bfloat16 `dst`: each value is the f32 result rounded to nearest even (beyond the reference,
        which writes f32 and f16 only)."""
        self._run_typed(src, dst, _lib.OUT_BF16)

    # ── pitched surfaces ────────────────────────────────────────────────────
    def _run_surface(self, src: PitchedSurface, dst: torch.Tensor, out: int) -> None:
        src.validate()
        self._validate_dst(dst, 1, out)
        if not self._fmt.interleaved():  # :1150-1156
            raise PreprocessError("FormatNeedsRawBuffer", f"source format {self._fmt!r} needs run_raw (raw device buffer), not the typed run()")
        desc = self._desc(src.width, src.height, src.row_pitch, src.channels, self._fmt.fmt_code(), dst.shape[3], dst.shape[2])
        self._launch(desc, [src.data], dst, out)

    def run_surface(self, src: PitchedSurface, dst: torch.Tensor) -> None:
        """preprocess.rs:1112."""
        self._run_surface(src, dst, _lib.OUT_F32)

    def run_surface_f16(self, src: PitchedSurface, dst: torch.Tensor) -> None:
        self._run_surface(src, dst, _lib.OUT_F16)

    def run_surface_bf16(self, src: PitchedSurface, dst: torch.Tensor) -> None:
        self._run_surface(src, dst, _lib.OUT_BF16)

    # ── raw camera buffers ──────────────────────────────────────────────────
    def _run_raw_batch(self, frames: Sequence[torch.Tensor], src_w: int, src_h: int, dst: torch.Tensor, out: int,
                       single: bool) -> None:
        self._validate_dst(dst, 1 if single else len(frames), out)
        for f in frames:
            self._validate_raw(f.numel() * f.element_size(), src_w, src_h)
        fmt = self._fmt
        desc = self._desc(src_w, src_h, fmt.pitch(src_w), fmt.bpp(), fmt.fmt_code(), dst.shape[3], dst.shape[2])
        self._launch(desc, list(frames), dst, out)

    def run_raw(self, src: torch.Tensor, src_w: int, src_h: int, dst: torch.Tensor) -> None:
        """preprocess.rs:1184 — one raw device frame in the builder's SourceFormat → [1,3,H,W]."""
        self._run_raw_batch([src], src_w, src_h, dst, _lib.OUT_F32, True)

    def run_raw_f16(self, src: torch.Tensor, src_w: int, src_h: int, dst: torch.Tensor) -> None:
        self._run_raw_batch([src], src_w, src_h, dst, _lib.OUT_F16, True)

    def run_raw_bf16(self, src: torch.Tensor, src_w: int, src_h: int, dst: torch.Tensor) -> None:
        self._run_raw_batch([src], src_w, src_h, dst, _lib.OUT_BF16, True)

    def run_raw_batch(self, frames: Sequence[torch.Tensor], src_w: int, src_h: int, dst: torch.Tensor) -> None:
        """preprocess.rs:1234 — N same-sized raw frames → [N,3,H,W], ONE launch (≤256 frames per launch)."""
        self._run_raw_batch(frames, src_w, src_h, dst, _lib.OUT_F32, False)

    def run_raw_batch_f16(self, frames: Sequence[torch.Tensor], src_w: int, src_h: int, dst: torch.Tensor) -> None:
        self._run_raw_batch(frames, src_w, src_h, dst, _lib.OUT_F16, False)

    def run_raw_batch_bf16(self, frames: Sequence[torch.Tensor], src_w: int, src_h: int, dst: torch.Tensor) -> None:
        self._run_raw_batch(frames, src_w, src_h, dst, _lib.OUT_BF16, False)

    @staticmethod
    def _out_format(f16: bool, dtype) -> int:
        """The kb200_out_format of run_raw_host / run_raw_strided: `dtype` when given, else `f16` decides."""
        if dtype is None:
            return _lib.OUT_F16 if f16 else _lib.OUT_F32
        if dtype not in _OUT_DTYPES:
            raise PreprocessError("BadOutputShape", f"unsupported output dtype {dtype} (expected torch.float32, torch.float16 or torch.bfloat16)")
        if f16 and dtype != torch.float16:
            raise PreprocessError("BadOutputShape", f"f16=True conflicts with dtype={dtype}")
        return _OUT_DTYPES.index(dtype)

    def run_raw_host(self, host_frames: torch.Tensor, src_w: int, src_h: int, dst_size: tuple[int, int], out: torch.Tensor | None = None,
                     f16: bool = False, pipeline=None, *, dtype: torch.dtype | None = None) -> torch.Tensor:
        """HOST camera frames in, HOST tensor out — what the reference's Python `Preprocessor` does around its kernel (pinned
        staging, upload, launch: kornia-py/src/cuda_ext/mod.rs:700-760), as one call: `host_frames` is a [N, frame_bytes] uint8
        host tensor, or [N, w*h] uint16 for the 16-bit Bayer formats, [N, w*h*3/2] uint16 for P010 / P012 / I010 / I012 and
        [N, 3*w*h] uint16 for I410 / I412 / I410Msb / I412Msb (page-locked
        for overlap), the result a [N,3,H,W] host tensor (pinned when allocated here) of `dtype`: torch.float32, torch.float16 or
        torch.bfloat16; without `dtype`, f16 when `f16`, else f32.
        Chunks ride a `HostPipeline` ring: upload -> ONE fused launch per chunk -> download.  Enqueue-only: synchronise the
        current stream of the pipeline's device before reading the result."""
        from . import imgproc

        t = host_frames
        if t.is_cuda:
            raise PreprocessError("NotDeviceImage", "run_raw_host takes host frames; use run_raw_batch / run_raw_strided for device frames")
        if t.dtype not in (torch.uint8, torch.uint16) or t.dim() != 2 or not t.is_contiguous():
            raise PreprocessError("InvalidRawSource", "host frames must be a contiguous [N, frame_bytes] uint8 or [N, samples] uint16 tensor")
        n, stride = t.shape[0], t.shape[1] * t.element_size()   # bytes
        self._validate_raw(stride, src_w, src_h)
        dw, dh = dst_size
        fmt_out = self._out_format(f16, dtype)
        want = _OUT_DTYPES[fmt_out]
        if out is None:
            out = torch.empty((n, 3, dh, dw), dtype=want, pin_memory=True)
        if out.is_cuda or out.dtype != want or not out.is_contiguous() or tuple(out.shape) != (n, 3, dh, dw):
            raise PreprocessError("BadOutputShape", f"destination must be a contiguous host {want} tensor of shape {[n, 3, dh, dw]}")
        fmt = self._fmt
        desc = self._desc(src_w, src_h, fmt.pitch(src_w), fmt.bpp(), fmt.fmt_code(), dw, dh)
        pipe = imgproc._pipeline_for(pipeline)
        _lib.set_device(pipe.device.index)
        st = _lib.lib().kb200_preprocess_host_format(pipe._h, torch.cuda.current_stream(pipe.device).cuda_stream, C.byref(desc), t.data_ptr(),
                                                    n * stride, stride, n, out.data_ptr(), out.numel(), fmt_out)
        if st != _lib.OK:
            kind = {_lib.ERR_INVALID_SOURCE: "InvalidRawSource"}.get(st, "Cuda")
            raise PreprocessError(kind, _lib.last_error())
        return out

    def run_raw_strided(self, base: torch.Tensor, frame_stride: int, batch: int, src_w: int, src_h: int,
                        dst: torch.Tensor, f16: bool = False, *, dtype: torch.dtype | None = None) -> None:
        """Frames at `base + i*frame_stride` bytes (a capture ring buffer): no pointer table.  `base` may be uint8 or, for
        the formats of 16-bit samples (16-bit Bayer, P010 / P012 / I010 / I012, I410 / I412 / I410Msb / I412Msb), uint16: its
        length is counted in bytes.  `dst` is of `dtype` (torch.float32, torch.float16 or torch.bfloat16); without `dtype`,
        float16 when `f16`, else float32."""
        out = self._out_format(f16, dtype)
        self._validate_dst(dst, batch, out)
        fmt = self._fmt
        nbytes = base.numel() * base.element_size()
        self._validate_raw(min(frame_stride, nbytes) if batch > 1 else nbytes, src_w, src_h)
        desc = self._desc(src_w, src_h, fmt.pitch(src_w), fmt.bpp(), fmt.fmt_code(), dst.shape[3], dst.shape[2])
        if not base.is_cuda:
            raise PreprocessError("NotDeviceImage", "CUDA preprocessor requires a device-resident source image")
        dev = dst.device
        _lib.set_device(dev.index)
        l = _lib.lib()
        fn = getattr(l, _STRIDED_ENTRIES[out])
        st = fn(torch.cuda.current_stream(dev).cuda_stream, C.byref(desc), base.data_ptr(), nbytes, frame_stride, batch,
                dst.data_ptr(), dst.numel())
        if st != _lib.OK:
            kind = {_lib.ERR_INVALID_SOURCE: "InvalidRawSource"}.get(st, "Cuda")
            raise PreprocessError(kind, _lib.last_error())

    # ── regions of interest ─────────────────────────────────────────────────
    def run_rois(self, frames: Sequence[torch.Tensor], src_w: int, src_h: int, rois, dst: torch.Tensor) -> None:
        """Crop-and-resize regions of raw device frames in the builder's SourceFormat: region i = (frame, x, y, w, h), the
        rectangle (x, y, w, h) of frames[frame], is resampled into dst[i] with the builder's mode (its affine is the one a
        w x h frame gets), sampling, normalisation, pad value and YUV matrix; taps are clamped to the region and decode at
        frame coordinates.  `rois`: a sequence of (frame, x, y, w, h), or an integer CPU tensor [M, 5].  `dst`: a contiguous
        device [M, 3, H, W] tensor of torch.float32, torch.float16 or torch.bfloat16, which selects the output.  One launch per
        80 regions.  A region outside its frame (or naming a frame that is not there) raises PreprocessError("InvalidRoi")."""
        if isinstance(rois, torch.Tensor):
            if rois.is_cuda or rois.dim() != 2 or rois.shape[1] != 5 or rois.dtype.is_floating_point or rois.dtype.is_complex or rois.dtype == torch.bool:
                raise PreprocessError("InvalidRoi", f"rois must be an integer CPU tensor [M, 5], got {rois.dtype} {list(rois.shape)} on {rois.device}")
            table = [tuple(int(v) for v in r) for r in rois.tolist()]
        else:
            table = [tuple(r) for r in rois]
            if any(len(r) != 5 or not all(isinstance(v, int) or (isinstance(v, torch.Tensor) and v.dim() == 0) for v in r) for r in table):
                raise PreprocessError("InvalidRoi", "each region must be (frame, x, y, w, h) of integers")
            table = [tuple(int(v) for v in r) for r in table]
        lim = 2 ** 31
        if not table:
            raise PreprocessError("InvalidRoi", "no regions given")
        if any(not -lim <= v < lim for r in table for v in r):
            raise PreprocessError("InvalidRoi", "region values must fit in 32-bit signed integers")
        for i, (k, x, y, w, h) in enumerate(table):   # the C entry's region rules, checked here so that the kind is InvalidRoi
            if not 0 <= k < len(frames):
                raise PreprocessError("InvalidRoi", f"region {i}: frame index {k} is outside [0, {len(frames)})", region=i)
            if x < 0 or y < 0:
                raise PreprocessError("InvalidRoi", f"region {i}: origin ({x}, {y}) is negative", region=i)
            if w < 1 or h < 1:
                raise PreprocessError("InvalidRoi", f"region {i}: size {w}x{h} is empty", region=i)
            if x + w > src_w or y + h > src_h:
                raise PreprocessError("InvalidRoi", f"region {i}: ({x}, {y}) + {w}x{h} reaches outside the {src_w}x{src_h} frame", region=i)
        out = self._out_format(False, dst.dtype)
        self._validate_dst(dst, len(table), out)
        regions = (_lib.Roi * len(table))(*[_lib.Roi(*r) for r in table])

        def call(s, ptrs, lens, n):
            desc = self._desc(src_w, src_h, self._fmt.pitch(src_w), self._fmt.bpp(), self._fmt.fmt_code(), dst.shape[3], dst.shape[2])
            return _lib.lib().kb200_preprocess_rois(s, C.byref(desc), self._mode.value, ptrs, lens, n, regions, len(table), dst.data_ptr(), dst.numel(), out)
        self._call(frames, dst, call, (src_w, src_h))

    # ── rotated and perspective regions ─────────────────────────────────────
    def run_warps(self, frames: Sequence[torch.Tensor], src_w: int, src_h: int, frame_index, matrices, dst: torch.Tensor) -> None:
        """Rotated and perspective crops of raw device frames in the builder's SourceFormat: region i is frames[frame_index[i]]
        through the FORWARD map matrices[i] (frame pixel coordinates -> output pixel coordinates, as cv2.warpAffine /
        warpPerspective without WARP_INVERSE_MAP; a 2x3 map gets the row (0, 0, 1)), sampled into dst[i] with the builder's
        sampling (Nearest or Bilinear), normalisation, pad value and YUV matrix.  The builder's mode does not apply: the map
        is the geometry.  `frame_index`: a sequence of ints or an integer CPU tensor [M]; `matrices`: a CPU tensor or nested
        sequence [M, 2, 3] or [M, 3, 3], converted to float32; `dst`: a contiguous device [M, 3, H, W] tensor of
        torch.float32, torch.float16 or torch.bfloat16, which selects the output.  A bad frame index, a map of another shape,
        with a non-finite entry or singular raises PreprocessError("InvalidWarp", region=i); Lanczos sampling raises
        "UnsupportedSampling"."""
        import math

        if self._sampling not in (InterpolationMode.Nearest, InterpolationMode.Bilinear):
            raise PreprocessError("UnsupportedSampling", f"unsupported sampling mode {self._sampling!r} for warped regions (expected Nearest or Bilinear)")
        if isinstance(frame_index, torch.Tensor):
            if (frame_index.is_cuda or frame_index.dim() != 1 or frame_index.dtype.is_floating_point or frame_index.dtype.is_complex
                    or frame_index.dtype == torch.bool):
                raise PreprocessError("InvalidWarp", f"frame_index must be an integer CPU tensor [M], got {frame_index.dtype} "
                                      f"{list(frame_index.shape)} on {frame_index.device}")
            index = [int(v) for v in frame_index.tolist()]
        else:
            index = list(frame_index)
            if not all(isinstance(v, int) or (isinstance(v, torch.Tensor) and v.dim() == 0 and not v.dtype.is_floating_point) for v in index):
                raise PreprocessError("InvalidWarp", "frame_index must hold integers")
            index = [int(v) for v in index]
        if not index:
            raise PreprocessError("InvalidWarp", "no regions given")
        if isinstance(matrices, torch.Tensor):
            if matrices.is_cuda or matrices.dim() != 3 or tuple(matrices.shape[1:]) not in ((2, 3), (3, 3)):
                raise PreprocessError("InvalidWarp", f"matrices must be a CPU tensor [M, 2, 3] or [M, 3, 3], got {list(matrices.shape)} on {matrices.device}")
            maps = list(matrices.to(torch.float32).unbind(0))
        else:
            maps = []
            for i, mi in enumerate(matrices):
                try:
                    t = torch.as_tensor(mi, dtype=torch.float32)
                except (TypeError, ValueError, RuntimeError) as e:
                    raise PreprocessError("InvalidWarp", f"region {i}: the map is not a 2x3 or 3x3 array of numbers ({e})", region=i) from None
                if tuple(t.shape) not in ((2, 3), (3, 3)):
                    raise PreprocessError("InvalidWarp", f"region {i}: the map has shape {list(t.shape)} (expected 2x3 or 3x3)", region=i)
                maps.append(t)
        if len(maps) != len(index):
            raise PreprocessError("InvalidWarp", f"{len(maps)} maps for {len(index)} frame indices")
        table = []
        for i, (k, mi) in enumerate(zip(index, maps)):   # the C entry's region rules, checked here so that the kind is InvalidWarp
            if not 0 <= k < len(frames):
                raise PreprocessError("InvalidWarp", f"region {i}: frame index {k} is outside [0, {len(frames)})", region=i)
            flat = mi.reshape(-1).tolist() + ([0.0, 0.0, 1.0] if mi.shape[0] == 2 else [])
            if not all(math.isfinite(v) for v in flat):
                raise PreprocessError("InvalidWarp", f"region {i}: the map has a non-finite entry", region=i)
            table.append((k, flat))
        out = self._out_format(False, dst.dtype)
        self._validate_dst(dst, len(table), out)
        warps = (_lib.WarpRoi * len(table))(*[_lib.WarpRoi(k, (C.c_float * 9)(*flat)) for k, flat in table])

        def call(s, ptrs, lens, n):
            desc = self._desc(src_w, src_h, self._fmt.pitch(src_w), self._fmt.bpp(), self._fmt.fmt_code(), dst.shape[3], dst.shape[2])
            st = _lib.lib().kb200_preprocess_warps(s, C.byref(desc), ptrs, lens, n, warps, len(table), dst.data_ptr(), dst.numel(), out)
            if st == _lib.ERR_SINGULAR_MATRIX:   # "region <i>: ..." (preprocess_warp.cu invert_warp)
                msg = _lib.last_error()
                raise PreprocessError("InvalidWarp", msg, region=int(msg.split(":")[0].split()[1]))
            return st
        self._call(frames, dst, call, (src_w, src_h))

    # ── dense coordinate maps ───────────────────────────────────────────────
    @staticmethod
    def _remap_map(name: str, m) -> torch.Tensor:
        """A map argument of run_remap as a [K, H, W] tensor: a tensor [H, W] or [K, H, W], or an H x W x 1 Image."""
        if isinstance(m, Image):
            m = m.data
            if m.dim() != 3 or m.shape[2] != 1:
                raise PreprocessError("InvalidMap", f"{name} must be a one-channel H x W x 1 Image, got {list(m.shape)}")
            m = m[..., 0]
        if not isinstance(m, torch.Tensor):
            raise PreprocessError("InvalidMap", f"{name} must be a device tensor or an Image, got {type(m).__name__}")
        if m.dim() not in (2, 3) or m.numel() == 0:
            raise PreprocessError("InvalidMap", f"{name} must be [H, W] or [K, H, W], got {list(m.shape)}")
        if m.dtype != torch.float32 or not m.is_cuda or not m.is_contiguous():
            raise PreprocessError("InvalidMap", f"{name} must be a contiguous float32 device tensor, got {m.dtype} on {m.device}")
        if m.data_ptr() % 4:
            raise PreprocessError("InvalidMap", f"{name} must be 4-byte aligned")
        return m if m.dim() == 3 else m.unsqueeze(0)

    def run_remap(self, frames: Sequence[torch.Tensor], src_w: int, src_h: int, map_x, map_y, dst: torch.Tensor, regions=None) -> None:
        """Raw device frames in the builder's SourceFormat resampled through dense coordinate maps (lens undistortion, rig
        rectification, fisheye views): region i = (frame k, map j) writes dst[i], output pixel (x, y) sampled at frame
        coordinate (map_x[j, y, x], map_y[j, y, x]) with the builder's sampling (Nearest or Bilinear), normalisation, pad
        value and YUV matrix.  A coordinate outside [0, src_w) x [0, src_h) (NaN included) takes the pad value.  The
        builder's mode does not apply: the map is the geometry.  `map_x` / `map_y`: contiguous float32 device tensors
        [H, W] or [K, H, W] of the same shape, or the Images generate_correction_map_polynomial returns; H x W is dst's.
        `regions`: a sequence of (frame, map) pairs or an integer CPU tensor [M, 2]; None is (i, 0) for every frame.
        `dst`: a contiguous device [M, 3, H, W] tensor of torch.float32, torch.float16 or torch.bfloat16, which selects the
        output.  A bad region raises PreprocessError("InvalidMap", region=i); a map of the wrong shape, dtype, device or
        alignment raises "InvalidMap"; Lanczos sampling raises "UnsupportedSampling"."""
        if self._sampling not in (InterpolationMode.Nearest, InterpolationMode.Bilinear):
            raise PreprocessError("UnsupportedSampling", f"unsupported sampling mode {self._sampling!r} for remapped regions (expected Nearest or Bilinear)")
        mx, my = self._remap_map("map_x", map_x), self._remap_map("map_y", map_y)
        if mx.shape != my.shape or mx.device != my.device:
            raise PreprocessError("InvalidMap", f"map_x {list(mx.shape)} on {mx.device} and map_y {list(my.shape)} on {my.device} differ")
        k, mh, mw = mx.shape
        if regions is None:
            table = [(i, 0) for i in range(len(frames))]
        elif isinstance(regions, torch.Tensor):
            if (regions.is_cuda or regions.dim() != 2 or regions.shape[1] != 2 or regions.dtype.is_floating_point or regions.dtype.is_complex
                    or regions.dtype == torch.bool):
                raise PreprocessError("InvalidMap", f"regions must be an integer CPU tensor [M, 2], got {regions.dtype} {list(regions.shape)} on {regions.device}")
            table = [(int(a), int(b)) for a, b in regions.tolist()]
        else:
            table = []
            for i, q in enumerate(regions):
                q = tuple(q) if isinstance(q, (tuple, list)) else None
                if q is None or len(q) != 2 or not all(isinstance(v, int) and not isinstance(v, bool) for v in q):
                    raise PreprocessError("InvalidMap", f"region {i}: expected a (frame, map) pair of integers", region=i)
                table.append(q)
        if not table:
            raise PreprocessError("InvalidMap", "no regions given")
        for i, (f, j) in enumerate(table):   # the C entry's region rules, checked here so that the kind is InvalidMap
            if not 0 <= f < len(frames):
                raise PreprocessError("InvalidMap", f"region {i}: frame index {f} is outside [0, {len(frames)})", region=i)
            if not 0 <= j < k:
                raise PreprocessError("InvalidMap", f"region {i}: map index {j} is outside [0, {k})", region=i)
        out = self._out_format(False, dst.dtype)
        self._validate_dst(dst, len(table), out)
        if (dst.shape[2], dst.shape[3]) != (mh, mw):
            raise PreprocessError("InvalidMap", f"the maps are {mh} x {mw} (H x W) but dst is {dst.shape[2]} x {dst.shape[3]}")
        if mx.device != dst.device:
            raise PreprocessError("InvalidMap", f"the maps are on {mx.device} but dst is on {dst.device}")
        rois = (_lib.RemapRoi * len(table))(*[_lib.RemapRoi(f, j) for f, j in table])

        def call(s, ptrs, lens, n):
            desc = self._desc(src_w, src_h, self._fmt.pitch(src_w), self._fmt.bpp(), self._fmt.fmt_code(), mw, mh)
            return _lib.lib().kb200_preprocess_remap(s, C.byref(desc), ptrs, lens, n, mx.data_ptr(), my.data_ptr(), mx.numel(), k, rois, len(table),
                                                     dst.data_ptr(), dst.numel(), out)
        self._call(frames, dst, call, (src_w, src_h))
