"""cuda/fusion.rs — the fusion engine's stage vocabulary and `FusedPipeline`, over pre-instantiated sm_90a kernels.

    from kornia_rs_b200.fusion import FusedPipeline, ReadU8RgbBilinear, Normalize, RgbToGray, WriteChwF32, WriteC1F32
    pipe = FusedPipeline.build([ReadU8RgbBilinear(sw, sh, dw, dh), Normalize(scale, bias), RgbToGray(), WriteC1F32()], dw, dh)
    pipe.launch(src_u8_hwc, dst_f32)            # one image, or [N,H,W,3] -> [N,planes,dh,dw] in one launch

The reference composes CUDA snippets at run time (NVRTC); this library ships AOT code only, so `build` maps the stage
list onto one of the compiled shapes — source, then any chain of distinct map stages, then a sink — and raises
FusionError("invalid pipeline: ...") for anything else (the reference's FusionError::Pipeline, cuda/fusion.rs:43-58).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Sequence

import torch

from . import _lib
from .image import Image


class FusionError(Exception):
    pass


@dataclass(frozen=True)
class ReadU8RgbBilinear:
    """cuda/fusion.rs:520 — source stage: u8 HWC RGB sampled bilinearly on the half-pixel grid."""
    src_w: int
    src_h: int
    dst_w: int
    dst_h: int

    def name(self) -> str:
        return "read_u8rgb_bilinear"


@dataclass(frozen=True)
class Normalize:
    """cuda/fusion.rs:592 — map stage: v * scale[c] + bias[c]."""
    scale: Sequence[float]
    bias: Sequence[float]

    def name(self) -> str:
        return "normalize"


@dataclass(frozen=True)
class RgbToGray:
    """cuda/fusion.rs:624 — map stage: BT.601 luma replicated to the three lanes."""

    def name(self) -> str:
        return "rgb_to_gray"


@dataclass(frozen=True)
class WriteChwF32:
    """cuda/fusion.rs:645 — sink: three f32 planes."""

    def name(self) -> str:
        return "write_chw_f32"


@dataclass(frozen=True)
class WriteC1F32:
    """cuda/fusion.rs:669 — sink: one f32 plane (the .x lane)."""

    def name(self) -> str:
        return "write_c1_f32"


class FusedPipeline:
    def __init__(self, read: ReadU8RgbBilinear, maps: int, norm: Normalize | None, sink: int, names: list[str]):
        self._read, self._maps, self._norm, self._sink, self._names = read, maps, norm, sink, names

    @staticmethod
    def build(stages: Sequence[object], dst_w: int, dst_h: int) -> "FusedPipeline":
        """FusedPipeline::build (cuda/fusion.rs:233): `stages` = source, maps..., sink over a dst_w x dst_h grid."""
        if len(stages) < 2:
            raise FusionError("invalid pipeline: need at least a source and a sink stage")
        read, sink_stage, mids = stages[0], stages[-1], list(stages[1:-1])
        if not isinstance(read, ReadU8RgbBilinear):
            raise FusionError("invalid pipeline: the first stage must be a source (ReadU8RgbBilinear)")
        if not isinstance(sink_stage, (WriteChwF32, WriteC1F32)):
            raise FusionError("invalid pipeline: the last stage must be a sink (WriteChwF32 / WriteC1F32)")
        if (read.dst_w, read.dst_h) != (dst_w, dst_h):
            raise FusionError(f"invalid pipeline: source maps to {read.dst_w}x{read.dst_h}, grid is {dst_w}x{dst_h}")
        kinds = []
        norm = None
        for st in mids:
            if isinstance(st, Normalize):
                if len(st.scale) != 3 or len(st.bias) != 3:
                    raise FusionError("invalid pipeline: Normalize needs three scale and three bias values")
                kinds.append("N"); norm = st
            elif isinstance(st, RgbToGray):
                kinds.append("G")
            else:
                raise FusionError(f"invalid pipeline: {type(st).__name__} is not a map stage")
        code = {"": 0, "N": 1, "G": 2, "NG": 3, "GN": 4}.get("".join(kinds))
        if code is None:
            raise FusionError(f"invalid pipeline: map chain {'+'.join(k for k in kinds)} is not a pre-instantiated shape (each map stage at most once)")
        return FusedPipeline(read, code, norm, 0 if isinstance(sink_stage, WriteChwF32) else 1, [s.name() for s in stages])

    def name(self) -> str:
        return "+".join(self._names)

    def out_planes(self) -> int:
        return 3 if self._sink == 0 else 1

    def launch(self, src, dst: torch.Tensor) -> None:
        """FusedPipeline::launch / launch_batched (cuda/fusion.rs:420-520): `src` u8 [H,W,3] or [N,H,W,3] on the device,
        `dst` f32 [N,planes,dh,dw] (or [planes,dh,dw] for one image) on the same device.  One launch."""
        t = src.data if isinstance(src, Image) else src
        r = self._read
        if t.dim() == 3:
            t = t.unsqueeze(0)
        if not (t.is_cuda and dst.is_cuda) or t.device != dst.device:
            raise FusionError("fusion kernel compile/launch error: source and destination must be on the same CUDA device")
        if t.dtype != torch.uint8 or dst.dtype != torch.float32 or not t.is_contiguous() or not dst.is_contiguous():
            raise FusionError("invalid pipeline: source must be contiguous u8 HWC, destination contiguous f32")
        n = t.shape[0]
        if tuple(t.shape[1:]) != (r.src_h, r.src_w, 3):
            raise FusionError(f"source slice too small: expected [{r.src_h},{r.src_w},3] images, got {list(t.shape[1:])}")
        if dst.numel() != n * self.out_planes() * r.dst_w * r.dst_h:
            raise FusionError(f"destination holds {dst.numel()} elements, the sink writes {n * self.out_planes() * r.dst_w * r.dst_h}")
        _lib.set_device(t.device.index)
        sc = _lib.f3(self._norm.scale) if self._norm else None
        bi = _lib.f3(self._norm.bias) if self._norm else None
        st = _lib.lib().kb200_fused_pipeline_u8_f32(torch.cuda.current_stream(t.device).cuda_stream, t.data_ptr(), t.numel(), dst.data_ptr(), dst.numel(),
                                                   r.src_w, r.src_h, r.dst_w, r.dst_h, n, self._maps, sc, bi, self._sink)
        if st != _lib.OK:
            raise FusionError(_lib.last_error())
