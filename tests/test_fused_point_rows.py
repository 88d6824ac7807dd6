"""The fused resize's full-row point kernel (csrc/resize_fused.cu, `fused_point_rows_kernel`, launched as
"fused_rows_kernel"): one CTA per (image, destination row) copies the whole tapped source row into shared memory and
writes the three whole plane rows, a thread owning 4 adjacent columns per vector.

A host mirror of the dispatcher lets every case assert which kernel it runs: the full-row kernel by default and under
fr.rows = 2, the tiled one under fr.rows = 1 or any tiled-schedule knob.  The GPU tests compare every frame, bit for bit,
with the oracle (f32, and its f16 / bf16 roundings) and with the tiled kernel, for the scalar and x86 leaves.
"""
import numpy as np
import pytest
import torch

from harness import dev, knobs
from restate import fused_schedule


FRR_CT, FRR_V, FRR_MAX_NPX = 256, 4, 2


def full_rows_npx(sw, sh, dw, dh, batch, sm, rows=0, tiled_knobs=False):
    """launch_fused_full_rows and its dispatch (csrc/resize_fused.cu) on the host, for a destination aligned to a vector:
    the vectors per thread, or None when the tiled kernel runs."""
    if fused_schedule(sw, sh, dw, dh, batch, sm).mode != "POINT" or rows == 1 or (rows != 2 and tiled_knobs):
        return None
    npx = -(-dw // (FRR_CT * FRR_V))
    if sw * 3 > 48 * 1024 - 16 or npx > FRR_MAX_NPX or dw % FRR_V or batch * dh > 0x7FFFFFFF:
        return None
    return npx


# (sw, sh, dw, dh, batch, vectors per thread): 3:1 and 5:1 with dw % 256 != 0, x 1:1 with y 3:1
GEOMETRIES = [
    (1008, 576, 336, 192, 7, 1),     # 3:1: 84 of the 256 threads own a vector
    (1680, 960, 336, 192, 5, 1),     # 5:1
    (400, 216, 400, 72, 9, 1),       # x 1:1, y 3:1
    (1600, 216, 1600, 72, 5, 2),     # x 1:1, y 3:1: two vectors per thread, the second one on 144 of 256 threads
]
KNOBS = [{"fr.rows": 1}, {"fr.rows": 2}, {}]


# ── host: the dispatcher ────────────────────────────────────────────────────────────────────────────────────────
def test_full_rows_headline_dispatch():
    """bench.py's headline takes the full-row kernel, two 4-column vectors per thread (the second on 64 of 256 threads);
    any tiled-schedule knob, fr.rows = 1, another mode, a row beyond 48 KB or dw > 2048 keeps the tiled kernel."""
    sm = 132
    assert full_rows_npx(3840, 2160, 1280, 720, 64, sm) == 2
    assert full_rows_npx(3840, 2160, 1280, 720, 64, sm, rows=2, tiled_knobs=True) == 2
    assert full_rows_npx(3840, 2160, 1280, 720, 64, sm, tiled_knobs=True) is None
    assert full_rows_npx(3840, 2160, 1280, 720, 64, sm, rows=1) is None
    assert full_rows_npx(3840, 2160, 1920, 1080, 64, sm) is None
    assert full_rows_npx(16400, 2160, 16400, 720, 1, sm) is None
    assert full_rows_npx(2064, 216, 2064, 72, 1, sm) is None
    assert full_rows_npx(2048, 216, 2048, 72, 1, sm) == 2


@pytest.mark.parametrize("sw,sh,dw,dh,batch,npx", GEOMETRIES)
def test_full_rows_geometries(sw, sh, dw, dh, batch, npx):
    """Each geometry runs the kernel it is listed for: point mode, dw % 256 != 0, the listed vectors per thread."""
    assert dw % FRR_CT != 0
    for k in KNOBS:
        got = full_rows_npx(sw, sh, dw, dh, batch, 132, k.get("fr.rows", 0))
        assert got == (None if k.get("fr.rows") == 1 else npx), (k, got)


# ── device: every frame against the oracle and the tiled kernel ─────────────────────────────────────────────────
def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _want(w32, dtype):
    """The oracle's f32 result, or its round-to-nearest-even f16 / bf16 value, on the host."""
    if dtype == torch.float32:
        return torch.from_numpy(w32)
    if dtype == torch.float16:
        return torch.from_numpy(w32.astype(np.float16))
    return torch.from_numpy(w32).to(torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize("sw,sh,dw,dh,batch,npx", GEOMETRIES)
@pytest.mark.parametrize("leaf", [0, 1])
def test_full_rows_match_oracle(kb, oracle, dev, sw, sh, dw, dh, batch, npx, leaf):
    src_h = np.stack([oracle.pattern_u8(sw * sh * 3, 0xF00D + i).reshape(sh, sw, 3) for i in range(batch)])
    src = torch.from_numpy(src_h).to(dev)
    scale, bias = oracle.normalize_params_from_mean_std(kb.IMAGENET_MEAN, kb.IMAGENET_STD)
    want32 = np.stack([oracle.resize_normalize_u8_to_f32_chw(src_h[i], dw, dh, scale, bias, leaf) for i in range(batch)])
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        want = _bits(_want(want32, dtype))
        tiled = None
        for k in KNOBS:
            what = f"{sw}x{sh}->{dw}x{dh} x{batch} leaf {leaf} {dtype} {k}"
            with knobs(kb, k):
                out = kb.imgproc.resize_normalize_to_tensor_u8_bilinear(src, dw, dh, scale, bias, dtype, leaf=leaf)
                assert kb._lib.last_kernel() == "fused_rows_kernel", what
            got = _bits(out).cpu()
            # the oracle and the device may disagree on the sign of an exact zero (assert_f32_bits_or_signed_zero's rule)
            mag = 0x7FFFFFFF if dtype == torch.float32 else 0x7FFF
            differ = (got != want) & ~(((got & mag) == 0) & ((want & mag) == 0))
            for i in range(batch):
                n = int(differ[i].sum())
                assert n == 0, f"{what}: frame {i}: {n} values differ from the oracle"
            if tiled is None:
                tiled = got
            else:
                assert torch.equal(got, tiled), f"{what}: not bit-identical to the tiled kernel"
