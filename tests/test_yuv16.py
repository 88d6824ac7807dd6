"""10- and 12-bit 4:2:0 video: P010, P012 (NV12's layout in 16-bit words, each code in the high bits) and I010, I012
(I420's layout, each code in the low bits), in the standalone decoders and the camera preprocess.

The decode is the Q16 form of the 8-bit Q20 decode (include/kornia_b200.h): a torch restatement that reads each layout
directly pins the decoders bit for bit, and is itself held within one level of the float64 formula.  In the preprocess a
tap is the decoded n-bit RGB code, normalised by W = 2^n - 1, so a frame is checked through its decode against
test_bayer16's restatement of the oracle's preprocess for 16-bit RGB (`preprocess_rgb16`).
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from harness import check_against_restatement, dev, make_pre, offset_buf, random_words, restated, yuv16_identity
from restate import BITS, KR_KB, MATRICES, TABLE16, decode_yuv16, q16, white


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FORMATS = ("P010", "P012", "I010", "I012")
CODE = {"P010": 80, "P012": 81, "I010": 82, "I012": 83}
LAYOUT = {"P010": 0, "P012": 0, "I010": 1, "I012": 1}   # kb200_yuv420_u16_layout: P01X, I01X


def float_coeffs16(m, bits):
    """(y_off, cy, cvr, cub, cug, cvg) as exact float64 coefficients for n-bit codes."""
    kr, kb_ = KR_KB[m[:5]]
    kg = 1.0 - kr - kb_
    s, w = 1 << (bits - 8), white(bits)
    full = m.endswith("Full")
    sy, sc = (1.0, 1.0) if full else (w / (219.0 * s), w / (224.0 * s))
    return (0 if full else 16 * s, sy, 2 * (1 - kr) * sc, 2 * (1 - kb_) * sc, -2 * kb_ * (1 - kb_) / kg * sc, -2 * kr * (1 - kr) / kg * sc)


def pack(yc, uc, vc, fmt, junk=None):
    """Code planes (int64 [h, w], [h/2, w/2], [h/2, w/2]) -> one `fmt` frame of uint16 words, with `junk` (int64 words of
    the frame's length, or None for zeros) in the bits the format ignores."""
    bits = BITS[fmt]
    if fmt[0] == "P":
        words = torch.cat([yc.reshape(-1), torch.stack([uc, vc], -1).reshape(-1)]) << (16 - bits)
        if junk is not None:
            words = words | (junk & ((1 << (16 - bits)) - 1))
    else:
        words = torch.cat([yc.reshape(-1), uc.reshape(-1), vc.reshape(-1)])
        if junk is not None:
            words = words | ((junk << bits) & 0xFFFF)
    return words.to(torch.int32).to(torch.uint16)


# ═══ CPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def test_table_is_the_derived_coefficients():
    """Every set is round(c * 2^16) of the float64 derivation, and the i32 sums keep their headroom at 12 bits."""
    for bits in (10, 12):
        for m in MATRICES:
            yo, *cs = float_coeffs16(m, bits)
            assert TABLE16[bits][m] == (yo, *(int(round(c * 2 ** 16)) for c in cs)), (bits, m)
            yo, cy, cvr, cub, cug, cvg = TABLE16[bits][m]
            w, half = white(bits), 1 << (bits - 1)
            terms = (w * cy, half * abs(cvr), half * abs(cub), half * (abs(cug) + abs(cvg)) + (1 << 15))
            assert max(terms) < 5.8e8 and terms[0] + max(terms[1:]) + (1 << 15) < 2 ** 31, (bits, m)
    assert TABLE16[10]["Bt709Limited"] == (64, 76533, 117835, 138846, -14017, -35027)


def test_native_sources_carry_the_table():
    """The kernels' table (kb200_common.cuh) and the header's documentation list exactly TABLE16, in kb200 order."""
    src = open(os.path.join(ROOT, "kornia-rs_b200", "csrc", "kb200_common.cuh")).read()
    block = src.split("YUV16_COEFFS[2][4] = {", 1)[1].split("};", 1)[0]
    rows = [tuple(int(x) for x in r.split(",")) for r in re.findall(r"\{([-\d, ]+)\}", block)]
    assert rows == [TABLE16[b][m] for b in (10, 12) for m in MATRICES]
    hdr = open(os.path.join(ROOT, "include", "kornia_b200.h")).read()
    doc = hdr.split("kb200_rgb_from_yuv420_u16: 4:2:0 frames", 1)[1].split("*/", 1)[0]
    for bits in (10, 12):
        part = doc.split(f"{bits} bits", 1)[1]
        for m, name in zip(MATRICES, ("BT601_LIMITED", "BT601_FULL", "BT709_LIMITED", "BT709_FULL")):
            assert re.search(rf"{name} +" + r" +".join(str(c) for c in TABLE16[bits][m][1:]), part), (bits, name)
    assert "KB200_YUV420_P01X = 0, KB200_YUV420_I01X = 1" in hdr
    for fmt, code in CODE.items():
        assert f"KB200_FMT_{fmt} = {code}" in hdr


@pytest.mark.parametrize("bits", [10, 12])
@pytest.mark.parametrize("m", MATRICES)
def test_within_one_level_of_float64(m, bits):
    """10 bits: every (U, V) pair at every 8th Y; 12 bits: a 64-step (U, V) grid at every 16th Y.  Within one level of
    the float64 formula rounded half up, and equal to it for almost every triple."""
    yo, cy, cvr, cub, cug, cvg = float_coeffs16(m, bits)
    w, half = white(bits), 1 << (bits - 1)
    step_uv, step_y = (1, 8) if bits == 10 else (64, 16)
    uv = torch.arange(0, w + 1, step_uv, dtype=torch.int64)
    u, v = torch.meshgrid(uv, uv, indexing="ij")
    u, v = u.reshape(-1), v.reshape(-1)
    uf, vf = (u - half).double(), (v - half).double()
    worst, differ, total = 0, 0, 0
    for yv in range(0, w + 1, step_y):
        y = torch.full_like(u, yv)
        yy = max(yv - yo, 0) * cy
        ref = torch.stack([yy + cvr * vf, yy + cug * uf + cvg * vf, yy + cub * uf], -1)
        ref = torch.floor(ref + 0.5).clamp(0, w).to(torch.int64)
        d = (q16(y, u, v, m, bits) - ref).abs()
        worst = max(worst, int(d.max()))
        differ += int((d.amax(-1) > 0).sum())
        total += u.numel()
    assert worst <= 1, (m, bits, worst)
    assert differ / total < 0.03, (m, bits, differ / total)


def test_source_format_members(kb):
    SF = kb.SourceFormat
    for fmt in FORMATS:
        f = SF[fmt]
        assert f.value == fmt.lower() and f.fmt_code() == CODE[fmt] and f.bit_depth() == BITS[fmt]
        assert f.bpp() == 2 and f.pitch(10) == 20 and f.buffer_len(8, 6) == 3 * 8 * 6 and f.buffer_len(1920, 1080) == 3 * 1920 * 1080
        assert f.dims_ok(8, 6) and f.dims_ok(2, 2) and not f.dims_ok(7, 6) and not f.dims_ok(8, 5)
        assert f.is_yuv() and f.is_yuv16() and not f.is_yuv420() and not f.is_yuv422() and not f.is_bayer() and not f.interleaved()
        assert SF.from_name(fmt.lower()) is f and SF.from_name(fmt) is f
    for alias, fmt in (("p010le", "P010"), ("p012le", "P012"), ("yuv420p10le", "I010"), ("yuv420p12le", "I012"), ("P010LE", "P010")):
        assert SF.from_name(alias) is SF[fmt]
    assert SF.from_name("p016") is None and SF.from_name("i014") is None
    assert sorted(f.fmt_code() for f in SF if f.is_yuv16()) == [80, 81, 82, 83]
    assert not any(f.is_yuv16() for f in SF if f not in [SF[x] for x in FORMATS])
    assert SF.Nv12.buffer_len(8, 6) == 72 and SF.Nv12.bit_depth() is None   # the 8-bit layouts are unchanged
    for fmt in FORMATS:   # every matrix is accepted, and travels in bits 8-9
        pre = kb.Preprocessor.builder().source_format(SF[fmt]).yuv_matrix(kb.YuvMatrix.Bt709Full).build_cuda()
        assert pre._desc(8, 6, 16, 2, SF[fmt].fmt_code(), 4, 4).fmt == CODE[fmt] | (3 << 8)


def test_abi_validation_without_a_gpu(kb):
    """Every argument check of the decoder and of the preprocess entries fails on the host, before any CUDA call, with
    its message."""
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = (C.addressof(buf) + 15) & ~15
    n = 2048   # elements of 16-bit room
    dec = l.kb200_rgb_from_yuv420_u16
    assert dec(None, p + 1, n, p, n, 8, 6, 1, 0, 10, 0) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "'src' is not 2-byte aligned (16-bit samples)"
    assert dec(None, p, n, p + 3, n, 8, 6, 1, 0, 10, 0) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "'dst' is not 2-byte aligned (16-bit samples)"
    for bad in (-1, 2, 4):
        assert dec(None, p, n, p, n, 8, 6, 1, bad, 10, 0) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown 16-bit 4:2:0 layout {bad}"
    for bad in (8, 11, 14, 16):
        assert dec(None, p, n, p, n, 8, 6, 1, 0, bad, 0) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"16-bit 4:2:0 samples are 10 or 12 bits, got {bad}"
    for bad in (-1, 4):
        assert dec(None, p, n, p, n, 8, 6, 1, 1, 12, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown YUV matrix {bad}"
    for fmt in FORMATS:
        lay, bits = LAYOUT[fmt], BITS[fmt]
        for w, h in ((7, 6), (8, 5)):
            assert dec(None, p, n, p, n, w, h, 1, lay, bits, 2) == _lib.ERR_INVALID_ARGUMENT
            assert _lib.last_error() == f"{fmt} needs even dimensions, got {w}x{h}"
        # lengths are in elements: a frame is w*h*3/2 words, its output w*h*3
        assert dec(None, p, 8 * 6 * 3 // 2 * 2 - 1, p, n, 8, 6, 2, lay, bits, 0) == _lib.ERR_SLICE_TOO_SMALL
        assert dec(None, p, n, p, 8 * 6 * 3 * 2 - 1, 8, 6, 2, lay, bits, 0) == _lib.ERR_SLICE_TOO_SMALL
    # the 8-bit decoder keeps rejecting a fifth layout
    assert l.kb200_rgb_from_yuv420_u8_matrix(None, p, 4096, p, 4096, 4, 4, 1, 4, 0) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "unknown 4:2:0 layout 4"

    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(100)
    M = lambda m: m << 8   # KB200_FMT_YUV_MATRIX

    def status(fmt, w=8, h=6, pitch=16):
        d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = w, h, pitch, 2, fmt, 4, 4, 1
        return l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64)

    for fmt in FORMATS:
        code = CODE[fmt]
        for w, h in ((7, 6), (8, 5), (5, 5)):
            assert status(code, w, h, 2 * w) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source for {fmt} at {w}x{h} (even dimensions required)"
        for pitch in (15, 14, 18, 32):
            assert status(code, pitch=pitch) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == (f"invalid pitched surface for {fmt} (pitch {pitch} bytes at width 8: frames must be tightly packed, "
                                         "pitch == 2*width)")
        # a frame is 3*w*h bytes; every matrix is accepted, and the check reaches the frame size
        d.src_w, d.src_h, d.src_pitch, d.fmt = 8, 6, 16, code
        assert l.kb200_preprocess_src_bytes(C.byref(d)) == 144
        for m in range(4):
            assert status(code | M(m)) == _lib.ERR_INVALID_SOURCE, (fmt, m)
            assert _lib.last_error() == "invalid raw source at 8x6 (got 100 bytes, need 144)"
        for stray in (M(4), M(7), 1 << 10):
            assert status(code | stray) == _lib.ERR_INVALID_ARGUMENT
            assert _lib.last_error() == f"source format code {code | stray} has bits set above bit 9 (bits 8-9 are the YUV matrix, 0-3)"
        # frames that do not start 2-byte aligned: the pointer table, the strided base and the strided stride
        status(code)
        odd = (C.c_void_p * 1)(p + 1)
        assert l.kb200_preprocess_f32(None, C.byref(d), odd, (C.c_size_t * 1)(4096), 1, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == f"{fmt} frame 0 is not 2-byte aligned"
        assert l.kb200_preprocess_strided_f32(None, C.byref(d), p + 1, 4096, 144, 1, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error().startswith(f"{fmt} frames must start 2-byte aligned")
        assert l.kb200_preprocess_strided_f16(None, C.byref(d), p, 4096, 145, 2, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error().startswith(f"{fmt} frames must start 2-byte aligned")
        assert l.kb200_preprocess_strided_f32(None, C.byref(d), p, 4096, 142, 2, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == "frame stride 142 smaller than a frame (144 bytes)"
    for bad in (79, 84, 84 | M(1), 79 | M(2), 255):
        assert status(bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown source format code {bad}"


def test_python_decoders_check_their_operands(kb):
    from kornia_rs_b200.image import ImageError

    src = torch.zeros(8 * 6 * 3 // 2, dtype=torch.uint16)
    for name in ("rgb_from_p010", "rgb_from_p012", "rgb_from_i010", "rgb_from_i012"):
        with pytest.raises(ImageError):
            getattr(kb.imgproc, name)(src, kb.Image(torch.zeros(6, 8, 3, dtype=torch.uint16)))   # host frames


# ═══ GPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def run_decode(kb, dev, fmt, src, w, h, n, m, dst_off=0):
    out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint16)
    out.fill_(0xCDCD)
    getattr(kb.imgproc, f"rgb_from_{fmt.lower()}")(src, kb.Image(out.view(n, h, w, 3)), matrix=kb.YuvMatrix[m])
    return out.view(n, h, w, 3), kb._lib.last_kernel()


def decode_kernel(fmt, w, soff, doff):
    vec = w % 8 == 0 and (2 * soff) % 16 == 0 and (2 * doff) % 16 == 0
    return f"rgb_from_{fmt[0].lower()}01x_{'vec' if vec else 'generic'}"


DECODE_CASES = [   # w, h, batch, src offset, dst offset (in samples): the vec kernel, then the generic one by width and by alignment
    (64, 48, 3, 0, 0), (2064, 6, 2, 0, 0), (8, 2, 2, 0, 0), (264, 4, 1, 0, 0),
    (18, 6, 2, 0, 0), (70, 4, 3, 0, 0), (2, 2, 1, 0, 0),
    (64, 48, 2, 1, 0), (64, 16, 2, 0, 3), (64, 16, 1, 8, 8), (64, 16, 1, 4, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("m", MATRICES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_decode(kb, dev, fmt, m):
    """Every format x matrix, batched, on both kernels and unaligned bases: equal to the restatement.  The frames are
    random 16-bit words, so the ignored bits hold garbage throughout."""
    for w, h, n, soff, doff in DECODE_CASES:
        nw = w * h * 3 // 2
        raws = random_words((n, nw), w * 131 + h + 7 * n + 1000 * MATRICES.index(m) + 17 * CODE[fmt])
        src = offset_buf(dev, n * nw, soff, torch.uint16)
        src.copy_(raws.reshape(-1).to(dev))
        got, kern = run_decode(kb, dev, fmt, src.view(n, nw), w, h, n, m, doff)
        what = f"{fmt} {m} {(w, h, n, soff, doff)}"
        assert kern == decode_kernel(fmt, w, soff, doff), what
        want = decode_yuv16(raws, w, h, fmt, m)
        assert torch.equal(got.cpu().to(torch.int32).to(torch.int64), want), what


@pytest.mark.gpu
@pytest.mark.parametrize("m", ["Bt601Limited", "Bt709Full"])
@pytest.mark.parametrize("w,h", [(64, 6), (38, 4)])
def test_decode_ignored_bits_extremes_and_repack(kb, dev, w, h, m):
    """The bits outside the code are ignored (garbage there gives the clean frame's output); all-zero and all-max codes
    decode as the restatement says; a P01x frame and its I01x repack give identical output."""
    for bits in (10, 12):
        pf, i_f = f"P01{bits - 10}", f"I01{bits - 10}"
        gen = torch.Generator().manual_seed(w + bits)
        yc = torch.randint(0, 1 << bits, (h, w), generator=gen, dtype=torch.int64)
        uc, vc = (torch.randint(0, 1 << bits, (h // 2, w // 2), generator=gen, dtype=torch.int64) for _ in range(2))
        junk = torch.randint(0, 1 << 16, (w * h * 3 // 2,), generator=gen, dtype=torch.int64)
        zeros, maxed = torch.zeros_like(yc), torch.full_like(yc, white(bits))
        zc, mc = torch.zeros_like(uc), torch.full_like(uc, white(bits))
        outs = {}
        for fmt in (pf, i_f):
            frames = torch.stack([pack(yc, uc, vc, fmt), pack(yc, uc, vc, fmt, junk), pack(zeros, zc, zc, fmt, junk),
                                  pack(maxed, mc, mc, fmt), pack(maxed, mc, mc, fmt, junk)])
            got, _ = run_decode(kb, dev, fmt, frames.to(dev), w, h, len(frames), m)
            g = got.cpu().to(torch.int32).to(torch.int64)
            assert torch.equal(g, decode_yuv16(frames, w, h, fmt, m)), fmt
            assert torch.equal(g[0], g[1]), f"{fmt}: garbage in the ignored bits changed the output"
            assert torch.equal(g[3], g[4]), fmt
            outs[fmt] = g
        assert torch.equal(outs[pf], outs[i_f])


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,m", [("P010", "Bt709Limited"), ("I012", "Bt601Full")])
def test_decode_1080p_batch(kb, dev, fmt, m):
    w, h, n = 1920, 1080, 64
    nw = w * h * 3 // 2
    g = torch.Generator(device=dev).manual_seed(0x1010 + CODE[fmt])
    raw = torch.randint(0, 1 << 16, (n, nw), dtype=torch.int32, device=dev, generator=g).to(torch.uint16)
    got, kern = run_decode(kb, dev, fmt, raw, w, h, n, m)
    assert kern == decode_kernel(fmt, w, 0, 0)
    for k0 in range(0, n, 16):
        assert torch.equal(got[k0:k0 + 16].to(torch.int32).to(torch.int64), decode_yuv16(raw[k0:k0 + 16], w, h, fmt, m)), f"frames {k0}.."
    del got, raw
    torch.cuda.empty_cache()


# ── camera preprocess ──
GEOMS = [(64, 48, 64, 48), (192, 108, 64, 64), (30, 20, 61, 47), (64, 48, 42, 40), (8, 6, 8, 6), (20, 2, 20, 2)]


def expected_preprocess_kernel(fmt, sampling, w, h, dw, dh, mode):
    if sampling == "Lanczos":
        return "preprocess_generic_kernel"
    k = fmt[0].lower() + "01x"
    if (dw, dh) == (w, h) and w % 4 == 0:
        return f"preprocess_{k}_identity_kernel"
    return f"preprocess_{k}_kernel" if dw % 4 == 0 else "preprocess_generic_kernel"


@pytest.mark.gpu
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("mode", ["Letterbox", "Stretch"])
@pytest.mark.parametrize("m", ["Bt601Limited", "Bt709Limited", "Bt709Full"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_preprocess(kb, dev, fmt, m, mode, sampling, f16):
    """Every geometry, two frames through the pointer table and the strided entry: bit-equal to the restated oracle on
    the decoded RGB16 twin (Lanczos: within test_bayer16's tolerance), with the kernel the dispatch promises."""
    dt, it = (torch.float16, torch.int16) if f16 else (torch.float32, torch.int32)
    pre = make_pre(kb, fmt, mode, sampling, m)
    n = 2
    for w, h, dw, dh in GEOMS:
        what = f"{fmt} {m} {mode} {sampling} {(w, h, dw, dh)} {'f16' if f16 else 'f32'}"
        nw = w * h * 3 // 2
        raws = random_words((n, nw), w * 7 + h * 3 + dw + CODE[fmt])
        got = torch.full((n, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([raws[k].to(dev) for k in range(n)], w, h, got)
        assert kb._lib.last_kernel() == expected_preprocess_kernel(fmt, sampling, w, h, dw, dh, mode), what
        ring = torch.cat([raws, torch.full((n, 12), 0xA5A5, dtype=torch.int32).to(torch.uint16)], 1).to(dev)
        strided = torch.full_like(got, float("nan"))
        pre.run_raw_strided(ring.view(-1), 2 * (nw + 12), n, w, h, strided, f16=f16)
        assert torch.equal(strided.view(it), got.view(it)), what
        rgb = decode_yuv16(raws, w, h, fmt, m).numpy().astype(np.uint16)
        for k in range(n):
            o = restated(kb, rgb[k], BITS[fmt], mode, sampling, dw, dh, f16 and sampling != "Lanczos")
            check_against_restatement(got[k], o, sampling, f16, f"{what} frame {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_preprocess_unaligned_frames(kb, dev, fmt):
    """A frame 2 bytes off an 8-byte boundary leaves the identity kernel for the 3b kernel (which reads 16-bit words
    only) with the same bits; the 3b geometry is unaffected."""
    w, h = 64, 48
    nw = w * h * 3 // 2
    raw = random_words((nw,), 99 + CODE[fmt]).to(dev)
    pre = make_pre(kb, fmt, "Stretch", "Bilinear", "Bt709Limited")
    for dw, dh in ((64, 48), (32, 24)):
        want = torch.full((1, 3, dh, dw), float("nan"), device=dev)
        pre.run_raw(raw, w, h, want)
        k_aligned = kb._lib.last_kernel()
        shifted = offset_buf(dev, nw, 1, torch.uint16)
        shifted.copy_(raw)
        got = torch.full_like(want, float("nan"))
        pre.run_raw(shifted, w, h, got)
        k = fmt[0].lower() + "01x"
        assert k_aligned == (f"preprocess_{k}_identity_kernel" if dw == w else f"preprocess_{k}_kernel")
        assert kb._lib.last_kernel() == f"preprocess_{k}_kernel"
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,m", [("P010", "Bt709Limited"), ("I012", "Bt601Full")])
@pytest.mark.parametrize("n", [256, 300])
def test_preprocess_identity_1080p(kb, dev, fmt, m, n):
    """Config 3a from 1080p frames at 256 and 300 frames (a second launch with frame0 > 0), through the pointer table and
    the strided entry, against the restatement for every frame."""
    w, h = 1920, 1080
    nw = w * h * 3 // 2
    g = torch.Generator(device=dev).manual_seed(0x3A10 + CODE[fmt])
    ring = torch.randint(0, 1 << 16, (n, nw + 32), dtype=torch.int32, device=dev, generator=g).to(torch.uint16)   # padded strided slots
    frames = ring[:, :nw]
    pre = make_pre(kb, fmt, "Stretch", "Bilinear", m)
    kernel = f"preprocess_{fmt[0].lower()}01x_identity_kernel"
    got = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)

    def check(entry):
        assert kb._lib.last_kernel() == kernel, entry
        for k0 in range(0, n, 16):
            want = yuv16_identity(frames[k0:k0 + 16], w, h, fmt, m, kb)
            assert torch.equal(got[k0:k0 + 16].view(torch.int32), want.contiguous().view(torch.int32)), f"{entry} frames {k0}.."

    pre.run_raw_batch([frames[k] for k in range(n)], w, h, got)
    check("pointer table")
    got.fill_(float("nan"))
    pre.run_raw_strided(ring.view(-1), 2 * (nw + 32), n, w, h, got)
    check("strided")
    for k in sorted({0, 255, n - 1}):   # the f32 restatement of the oracle on frames on both sides of the launch split
        rgb = decode_yuv16(frames[k].cpu(), w, h, fmt, m).numpy().astype(np.uint16)
        o = restated(kb, rgb, BITS[fmt], "Stretch", "Bilinear", w, h)
        np.testing.assert_array_equal(got[k].cpu().numpy().view(np.uint32), o.view(np.uint32), f"frame {k}")
    del got, ring, frames
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["P012", "I010"])
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 192, 108), ("Letterbox", 64, 64)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_pipeline(kb, dev, fmt, mode, dw, dh, f16):
    """run_raw_host carries [N, w*h*3/2] uint16 frames (and the same bytes as [N, 3*w*h] uint8): host frames in / host
    tensor out equal the device path, and the transfers are exactly the frames' 3*w*h bytes and the outputs' bytes."""
    w, h, n = 192, 108, 7
    host = random_words((n, w * h * 3 // 2), 5 + CODE[fmt]).pin_memory()
    pre = make_pre(kb, fmt, mode, "Bilinear", "Bt709Limited")
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
    it = torch.int16 if f16 else torch.int32
    for frames in (host, host.view(torch.uint8)):
        pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * 3 * w * h, dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
        got = pre.run_raw_host(frames, w, h, (dw, dh), f16=f16, pipeline=pipe)
        torch.cuda.synchronize()
        h2d, d2h = pipe.last_transfer()
        pipe.close()
        assert h2d == n * 3 * w * h and d2h == n * 3 * dw * dh * (2 if f16 else 4)
        assert torch.equal(got.view(it), want.cpu().view(it))
