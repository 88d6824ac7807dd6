"""4:4:4 video: I444 (three byte planes Y, U, V) and I410, I412, I410Msb, I412Msb (three planes of 16-bit words, each code in
the low or the high bits), in the standalone decoders and the camera preprocess.

Every pixel decodes from its own U and V with the existing arithmetic: Q20 for bytes (test_yuv_matrix's `q20`), Q16 for
words (test_yuv16's `q16`).  A torch / numpy restatement that reads the planes directly pins the decoders bit for bit.
The twin identities tie the family to the formats already served: an I444 frame whose chroma is an I420 frame's chroma
replicated 2x2 decodes and preprocesses to the I420 frame's bits (likewise I41x against I01x), and an Msb frame decodes
like its low-bit twin.  In the preprocess an 8-bit frame is checked against the oracle on its RGB8 twin, a 16-bit one
against test_bayer16's restatement on its RGB16 twin.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from harness import FootprintCase, Guarded, check_against_restatement, dev, make_pre, neighbour_frames, offset_buf, oracle_cfg, poison, random_bytes, random_words, restated, run_guarded
from restate import BITS, MATRICES, TABLE, decode_yuv444, decode_yuv444_16, white


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FORMATS = ("I444", "I410", "I412", "I410Msb", "I412Msb")
WORDS = FORMATS[1:]
CODE = {"I444": 11, "I410": 85, "I412": 86, "I410Msb": 87, "I412Msb": 88}
LAYOUT = {"I410": 0, "I412": 0, "I410Msb": 1, "I412Msb": 1}   # kb200_yuv444_u16_layout: I41X, I41X_MSB
TWIN420 = {"I410": "I010", "I412": "I012"}


def pack16(yc, uc, vc, fmt, junk=None):
    """Code planes (int64 [h, w] each) -> one `fmt` frame of uint16 words, with `junk` in the bits the format ignores."""
    bits = BITS[fmt]
    words = torch.cat([yc.reshape(-1), uc.reshape(-1), vc.reshape(-1)])
    if fmt.endswith("Msb"):
        words = words << (16 - bits)
        if junk is not None:
            words = words | (junk & ((1 << (16 - bits)) - 1))
    elif junk is not None:
        words = words | ((junk << bits) & 0xFFFF)
    return words.to(torch.int32).to(torch.uint16)


def i420_to_i444(raw, w, h):
    """An I420 frame (bytes) -> the I444 frame with its chroma replicated 2x2."""
    q = (w // 2) * (h // 2)
    up = lambda a: np.repeat(np.repeat(a.reshape(h // 2, w // 2), 2, 0), 2, 1).reshape(-1)
    return np.concatenate([raw[:w * h], up(raw[w * h:w * h + q]), up(raw[w * h + q:])])


def i01x_to_i41x(raw, w, h):
    """An I010 / I012 frame (uint16 tensor, any word values) -> the I41x frame with its chroma replicated 2x2."""
    q = (w // 2) * (h // 2)
    up = lambda a: a.reshape(h // 2, w // 2).repeat_interleave(2, 0).repeat_interleave(2, 1).reshape(-1)
    return torch.cat([raw[:w * h], up(raw[w * h:w * h + q]), up(raw[w * h + q:])])


# ═══ CPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def test_source_format_members(kb):
    SF = kb.SourceFormat
    for fmt in FORMATS:
        f = SF[fmt]
        b = 1 if fmt == "I444" else 2
        assert f.value == fmt.lower() and f.fmt_code() == CODE[fmt] and f.bit_depth() == BITS[fmt]
        assert f.bpp() == b and f.pitch(10) == 10 * b and f.buffer_len(8, 6) == 3 * 8 * 6 * b and f.buffer_len(7, 5) == 3 * 7 * 5 * b
        assert f.dims_ok(8, 6) and f.dims_ok(7, 5) and f.dims_ok(1, 1)
        assert f.is_yuv() and f.is_yuv444() and not f.is_yuv420() and not f.is_yuv16() and not f.is_yuv422()
        assert not f.is_bayer() and not f.is_bayer16() and not f.is_bayer_packed() and not f.interleaved()
        assert SF.from_name(fmt.lower()) is f and SF.from_name(fmt) is f
    for alias, fmt in (("yuv444p", "I444"), ("yuv444p10le", "I410"), ("yuv444p12le", "I412"), ("YUV444P10LE", "I410")):
        assert SF.from_name(alias) is SF[fmt]
    assert SF.from_name("i414") is None and SF.from_name("yuv444p16le") is None
    assert sorted(f.fmt_code() for f in SF if f.is_yuv444()) == [11, 85, 86, 87, 88]
    for fmt in FORMATS:   # every matrix is accepted, and travels in bits 8-9
        for m in range(4):
            pre = kb.Preprocessor.builder().source_format(SF[fmt]).yuv_matrix(kb.YuvMatrix(m)).build_cuda()
            assert pre._desc(8, 6, SF[fmt].pitch(8), SF[fmt].bpp(), SF[fmt].fmt_code(), 4, 4).fmt == CODE[fmt] | (m << 8)


def test_header_documents_the_family():
    hdr = open(os.path.join(ROOT, "include", "kornia_b200.h")).read()
    for fmt, code in CODE.items():
        assert f"KB200_FMT_{fmt.upper().replace('MSB', '_MSB')} = {code}" in hdr
    assert "KB200_YUV444_I41X = 0, KB200_YUV444_I41X_MSB = 1" in hdr
    assert "Codes 10, 12-15, 20-31, 48-63, 76-79, 84 and 89 to 255 are not formats." in hdr
    assert "kb200_rgb_from_yuv444_u8(" in hdr and "kb200_rgb_from_yuv444_u16(" in hdr


def test_decoder_validation_without_a_gpu(kb):
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = (C.addressof(buf) + 15) & ~15
    n = 2048
    d8, d16 = l.kb200_rgb_from_yuv444_u8, l.kb200_rgb_from_yuv444_u16
    for bad in (-1, 4, 99):
        assert d8(None, p, n, p, n, 8, 6, 1, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown YUV matrix {bad}"
        assert d16(None, p, n, p, n, 8, 6, 1, 0, 10, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown YUV matrix {bad}"
    assert d16(None, p + 1, n, p, n, 8, 6, 1, 0, 10, 0) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "'src' is not 2-byte aligned (16-bit samples)"
    assert d16(None, p, n, p + 3, n, 8, 6, 1, 0, 10, 0) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "'dst' is not 2-byte aligned (16-bit samples)"
    for bad in (-1, 2, 4):
        assert d16(None, p, n, p, n, 8, 6, 1, bad, 10, 0) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown 16-bit 4:4:4 layout {bad}"
    for bad in (8, 11, 14, 16):
        assert d16(None, p, n, p, n, 8, 6, 1, 1, bad, 0) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"16-bit 4:4:4 samples are 10 or 12 bits, got {bad}"
    for w, h in ((0, 6), (8, 0)):
        assert d8(None, p, n, p, n, w, h, 1, 0) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "image dimensions must be non-zero"
    # a frame is 3*w*h elements in and out; odd sizes are frames too
    for w, h in ((8, 6), (7, 5)):
        e = 3 * w * h * 2
        assert d8(None, p, e - 1, p, e, w, h, 2, 0) == _lib.ERR_SLICE_TOO_SMALL and "'src'" in _lib.last_error()
        assert d8(None, p, e, p, e - 1, w, h, 2, 0) == _lib.ERR_SLICE_TOO_SMALL and "'dst'" in _lib.last_error()
        for fmt in WORDS:
            assert d16(None, p, e - 1, p, e, w, h, 2, LAYOUT[fmt], BITS[fmt], 0) == _lib.ERR_SLICE_TOO_SMALL and "'src'" in _lib.last_error()
            assert d16(None, p, e, p, e - 1, w, h, 2, LAYOUT[fmt], BITS[fmt], 0) == _lib.ERR_SLICE_TOO_SMALL and "'dst'" in _lib.last_error()


def test_preprocess_validation_without_a_gpu(kb):
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = (C.addressof(buf) + 15) & ~15
    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(100)
    M = lambda m: m << 8   # KB200_FMT_YUV_MATRIX

    def status(fmt, w=8, h=6, pitch=8, bpp=1):
        d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = w, h, pitch, bpp, fmt, 4, 4, 1
        return l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64)

    # I444: tight byte planes, pitch == w
    assert status(11, pitch=7) == _lib.ERR_INVALID_SOURCE
    assert _lib.last_error() == "invalid pitched surface (need pitch >= width*channels and len >= pitch*height)"
    for pitch in (9, 16):
        assert status(11, pitch=pitch) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == "I444 frames must be tightly packed (pitch == width)"
    for fmt in WORDS:
        code = CODE[fmt]
        for pitch in (15, 14, 18, 32):
            assert status(code, pitch=pitch, bpp=2) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == (f"invalid pitched surface for {fmt} (pitch {pitch} bytes at width 8: frames must be tightly packed, "
                                         "pitch == 2*width)")
    for fmt in FORMATS:
        code, b = CODE[fmt], 1 if fmt == "I444" else 2
        for w, h in ((8, 6), (7, 5), (1, 1)):   # any size is a frame of 3*w*h samples
            d.src_w, d.src_h, d.src_pitch, d.fmt = w, h, w * b, code
            assert l.kb200_preprocess_src_bytes(C.byref(d)) == 3 * w * h * b
        need = 3 * 8 * 6 * b
        for m in range(4):
            assert status(code | M(m), pitch=8 * b, bpp=b) == _lib.ERR_INVALID_SOURCE, (fmt, m)
            assert _lib.last_error() == f"invalid raw source at 8x6 (got 100 bytes, need {need})"
        for stray in (M(4), M(7), 1 << 10):
            assert status(code | stray, pitch=8 * b, bpp=b) == _lib.ERR_INVALID_ARGUMENT
            assert _lib.last_error() == f"source format code {code | stray} has bits set above bit 9 (bits 8-9 are the YUV matrix, 0-3)"
    for fmt in WORDS:   # frames that do not start 2-byte aligned: the pointer table, the strided base and the strided stride
        status(CODE[fmt], pitch=16, bpp=2)
        odd = (C.c_void_p * 1)(p + 1)
        assert l.kb200_preprocess_f32(None, C.byref(d), odd, (C.c_size_t * 1)(4096), 1, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == f"{fmt} frame 0 is not 2-byte aligned"
        assert l.kb200_preprocess_strided_f32(None, C.byref(d), p + 1, 4096, 288, 1, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error().startswith(f"{fmt} frames must start 2-byte aligned")
        assert l.kb200_preprocess_strided_f16(None, C.byref(d), p, 4096, 289, 2, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error().startswith(f"{fmt} frames must start 2-byte aligned")
        assert l.kb200_preprocess_strided_f32(None, C.byref(d), p, 4096, 286, 2, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == "frame stride 286 smaller than a frame (288 bytes)"
    for bad in (10, 84, 89, 84 | M(1), 89 | M(2), 12):   # the neighbouring codes name no format
        assert status(bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown source format code {bad}"


def test_python_decoders_check_their_operands(kb):
    from kornia_rs_b200.image import ImageError

    with pytest.raises(ImageError):
        kb.imgproc.rgb_from_i444(torch.zeros(3 * 8 * 6, dtype=torch.uint8), kb.Image(torch.zeros(6, 8, 3, dtype=torch.uint8)))
    for name in ("rgb_from_i410", "rgb_from_i412", "rgb_from_i410msb", "rgb_from_i412msb"):
        with pytest.raises(ImageError):
            getattr(kb.imgproc, name)(torch.zeros(3 * 8 * 6, dtype=torch.uint16), kb.Image(torch.zeros(6, 8, 3, dtype=torch.uint16)))


def test_bt601_full_i444_within_one_level_of_cv2():
    """JPEG's 4:4:4: an I444 frame decoded with Bt601Full is within one level of cv2 on the interleaved (Y, Cr, Cb) image."""
    cv2 = pytest.importorskip("cv2")
    w, h = 256, 192
    raw = random_bytes(3 * w * h, 444)
    y, u, v = (raw[k * w * h:(k + 1) * w * h].reshape(h, w) for k in range(3))
    ref = cv2.cvtColor(np.ascontiguousarray(np.stack([y, v, u], -1)), cv2.COLOR_YCrCb2RGB).astype(np.int64)
    assert np.abs(decode_yuv444(raw, w, h, "Bt601Full").astype(np.int64) - ref).max() <= 1


# ═══ GPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def run_decode(kb, dev, fmt, src, w, h, n, m, dst_off=0):
    if fmt == "I444":
        out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint8)
        out.fill_(0xCD)
    else:
        out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint16)
        out.fill_(0xCDCD)
    getattr(kb.imgproc, f"rgb_from_{fmt.lower()}")(src, kb.Image(out.view(n, h, w, 3)), matrix=kb.YuvMatrix[m])
    return out.view(n, h, w, 3), kb._lib.last_kernel()


def decode_kernel(fmt, w, soff, doff):
    if fmt == "I444":
        vec = w % 16 == 0 and soff % 16 == 0 and doff % 16 == 0
        return f"rgb_from_i444_{'vec16' if vec else 'generic'}"
    vec = w % 8 == 0 and (2 * soff) % 16 == 0 and (2 * doff) % 16 == 0
    return f"rgb_from_i41x_{'vec' if vec else 'generic'}"


DECODE_CASES = [   # w, h, batch, src offset, dst offset (in samples): the vec kernels, then the generic one by width and by alignment
    (64, 48, 3, 0, 0), (2064, 3, 2, 0, 0), (16, 1, 2, 0, 0), (4112, 2, 1, 0, 0),
    (24, 5, 2, 0, 0), (70, 3, 3, 0, 0), (1, 1, 2, 0, 0), (33, 7, 1, 0, 0),
    (64, 48, 2, 1, 0), (64, 16, 2, 0, 3), (64, 16, 1, 8, 8), (64, 16, 1, 4, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("m", MATRICES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_decode(kb, dev, fmt, m):
    """Every format x matrix, batched, on both kernels and offset bases: equal to the restatement.  16-bit frames are
    random words, so the ignored bits hold garbage throughout."""
    for w, h, n, soff, doff in DECODE_CASES:
        ne = 3 * w * h
        seed = w * 131 + h + 7 * n + 1000 * MATRICES.index(m) + 17 * CODE[fmt] + soff + 5 * doff
        what = f"{fmt} {m} {(w, h, n, soff, doff)}"
        if fmt == "I444":
            raws = random_bytes(n * ne, seed).reshape(n, ne)
            src = offset_buf(dev, n * ne, soff, torch.uint8)
            src.copy_(torch.from_numpy(raws.reshape(-1)))
            got, kern = run_decode(kb, dev, fmt, src.view(n, ne), w, h, n, m, doff)
            g = got.cpu().numpy()
            for k in range(n):
                np.testing.assert_array_equal(g[k], decode_yuv444(raws[k], w, h, m), f"{what} frame {k}")
        else:
            raws = random_words((n, ne), seed)
            src = offset_buf(dev, n * ne, soff, torch.uint16)
            src.copy_(raws.reshape(-1).to(dev))
            got, kern = run_decode(kb, dev, fmt, src.view(n, ne), w, h, n, m, doff)
            assert torch.equal(got.cpu().to(torch.int32).to(torch.int64), decode_yuv444_16(raws, w, h, fmt, m)), what
        assert kern == decode_kernel(fmt, w, soff, doff), what


@pytest.mark.gpu
@pytest.mark.parametrize("m", MATRICES)
@pytest.mark.parametrize("w,h", [(64, 6), (38, 4)])
def test_decode_twins(kb, dev, w, h, m):
    """An I444 frame holding an I420 frame's chroma replicated 2x2 decodes to the I420 frame's bits; the same for I41x
    against I01x (random words, garbage in the ignored bits); an Msb frame holding code << (16 - n) with junk in the low
    bits decodes like its low-bit twin."""
    n = 3
    i420 = random_bytes(n * w * h * 3 // 2, w + h).reshape(n, -1)
    want = torch.empty(n, h, w, 3, dtype=torch.uint8, device=dev)
    kb.imgproc.rgb_from_i420(torch.from_numpy(i420).to(dev), kb.Image(want), matrix=kb.YuvMatrix[m])
    i444 = np.stack([i420_to_i444(f, w, h) for f in i420])
    got, _ = run_decode(kb, dev, "I444", torch.from_numpy(i444).to(dev), w, h, n, m)
    assert torch.equal(got, want)
    for fmt, twin in TWIN420.items():
        bits = BITS[fmt]
        i01x = random_words((n, w * h * 3 // 2), w * bits + h)
        want = torch.empty(n, h, w, 3, dtype=torch.uint16, device=dev)
        getattr(kb.imgproc, f"rgb_from_{twin.lower()}")(i01x.to(dev), kb.Image(want), matrix=kb.YuvMatrix[m])
        i41x = torch.stack([i01x_to_i41x(f, w, h) for f in i01x])
        got, _ = run_decode(kb, dev, fmt, i41x.to(dev), w, h, n, m)
        assert torch.equal(got, want), fmt
        gen = torch.Generator().manual_seed(bits * w)
        planes = [torch.randint(0, 1 << bits, (h, w), generator=gen, dtype=torch.int64) for _ in range(3)]
        junk = torch.randint(0, 1 << 16, (3 * w * h,), generator=gen, dtype=torch.int64)
        low, _ = run_decode(kb, dev, fmt, pack16(*planes, fmt, junk).to(dev)[None], w, h, 1, m)
        low = low.clone()
        msb, _ = run_decode(kb, dev, f"{fmt}Msb", pack16(*planes, f"{fmt}Msb", junk).to(dev)[None], w, h, 1, m)
        assert torch.equal(low, msb), fmt


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,m", [("I444", "Bt601Full"), ("I410Msb", "Bt709Limited")])
def test_decode_1080p_batch(kb, dev, fmt, m):
    w, h, n = 1920, 1080, 32
    ne = 3 * w * h
    g = torch.Generator(device=dev).manual_seed(0x444 + CODE[fmt])
    if fmt == "I444":
        raw = torch.randint(0, 256, (n, ne), dtype=torch.int32, device=dev, generator=g).to(torch.uint8)
    else:
        raw = torch.randint(0, 1 << 16, (n, ne), dtype=torch.int32, device=dev, generator=g).to(torch.uint16)
    got, kern = run_decode(kb, dev, fmt, raw, w, h, n, m)
    assert kern == decode_kernel(fmt, w, 0, 0)
    for k in (0, 13, n - 1):
        if fmt == "I444":
            np.testing.assert_array_equal(got[k].cpu().numpy(), decode_yuv444(raw[k].cpu().numpy(), w, h, m), f"frame {k}")
        else:
            assert torch.equal(got[k].cpu().to(torch.int32).to(torch.int64), decode_yuv444_16(raw[k].cpu(), w, h, fmt, m)), f"frame {k}"
    del got, raw
    torch.cuda.empty_cache()


# ── camera preprocess ──
# identity (3a), a 3:1 letterbox (3b), a non-integer stretch, a geometry the fast kernel cannot store (dst_w % 4 != 0),
# an odd-sized source, and a one-row frame
GEOMS = [("Stretch", 64, 48, 64, 48), ("Letterbox", 192, 108, 64, 64), ("Stretch", 30, 20, 61, 47), ("Letterbox", 64, 48, 42, 40),
         ("Letterbox", 33, 17, 40, 40), ("Stretch", 20, 1, 20, 1)]


def expected_preprocess_kernel(fmt, sampling, w, h, dw, dh):
    if sampling == "Lanczos":
        return "preprocess_generic_kernel"
    k = "i444" if fmt == "I444" else "i41x"
    if (dw, dh) == (w, h) and w % 4 == 0:
        return f"preprocess_{k}_identity_kernel"
    return f"preprocess_{k}_kernel" if dw % 4 == 0 else "preprocess_generic_kernel"


def frames_of(fmt, w, h, n, seed):
    if fmt == "I444":
        return [torch.from_numpy(random_bytes(3 * w * h, seed + k)) for k in range(n)]
    return list(random_words((n, 3 * w * h), seed))


@pytest.mark.gpu
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("m", ["Bt601Limited", "Bt709Limited", "Bt601Full"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_preprocess(kb, oracle, dev, fmt, m, sampling, f16):
    """Every geometry and both modes' shapes, two frames through the pointer table and the strided entry: I444 bit-equal to
    the device run and the oracle on the RGB8 twins, 16-bit formats to test_bayer16's restatement on the RGB16 twins
    (Lanczos: the existing tolerances), with the kernel the dispatch promises."""
    dt, it = (torch.float16, torch.int16) if f16 else (torch.float32, torch.int32)
    n = 2
    for mode, w, h, dw, dh in GEOMS:
        what = f"{fmt} {m} {mode} {sampling} {(w, h, dw, dh)} {'f16' if f16 else 'f32'}"
        pre = make_pre(kb, fmt, mode, sampling, m)
        raws = frames_of(fmt, w, h, n, w * 7 + h * 3 + dw + CODE[fmt])
        got = torch.full((n, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([r.to(dev) for r in raws], w, h, got)
        assert kb._lib.last_kernel() == expected_preprocess_kernel(fmt, sampling, w, h, dw, dh), what
        pad = torch.full((12,), 0xA5, dtype=torch.uint8).view(raws[0].dtype) if fmt == "I444" else torch.full((12,), 0xA5A5, dtype=torch.int32).to(torch.uint16)
        ring = torch.cat([torch.cat([r, pad]) for r in raws]).to(dev)
        strided = torch.full_like(got, float("nan"))
        pre.run_raw_strided(ring, (raws[0].numel() + 12) * raws[0].element_size(), n, w, h, strided, f16=f16)
        assert torch.equal(strided.view(it), got.view(it)), what
        if fmt == "I444":
            twins = [decode_yuv444(r.numpy(), w, h, m) for r in raws]
            twin_pre = make_pre(kb, "Rgb8", mode, sampling)
            want = torch.full_like(got, float("nan"))
            (twin_pre.run_raw_batch_f16 if f16 else twin_pre.run_raw_batch)([torch.from_numpy(t.reshape(-1)).to(dev) for t in twins], w, h, want)
            assert torch.equal(got.view(it), want.view(it)), what
            cfg = oracle_cfg(kb, oracle, mode, sampling)
            for k in range(n):
                o = oracle.preprocess_frame(twins[k].reshape(-1), cfg, w, h, dw, dh, f16=f16 and sampling != "Lanczos")
                g = got[k].cpu().numpy()
                if sampling == "Lanczos":
                    assert np.max(np.abs(g.astype(np.float32) - o)) <= (2e-3 if f16 else 1e-4), what
                else:
                    np.testing.assert_array_equal(g.view(np.uint16 if f16 else np.uint32), o.view(np.uint16 if f16 else np.uint32), what)
        else:
            rgb = decode_yuv444_16(torch.stack(raws), w, h, fmt, m).numpy().astype(np.uint16)
            for k in range(n):
                o = restated(kb, rgb[k], BITS[fmt], mode, sampling, dw, dh, f16 and sampling != "Lanczos")
                check_against_restatement(got[k], o, sampling, f16, f"{what} frame {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
def test_preprocess_twins(kb, dev, sampling, f16):
    """An I444 frame holding an I420 frame's chroma replicated 2x2 preprocesses to the I420 frame's bits, and an I41x frame
    to its I01x frame's, on every kernel."""
    it = torch.int16 if f16 else torch.int32
    for mode, w, h, dw, dh in GEOMS[:4]:
        for fmt, twin in (("I444", "I420"), ("I410", "I010"), ("I412Msb", None)):
            if fmt == "I444":
                small = torch.from_numpy(random_bytes(w * h * 3 // 2, w + dw))
                big = torch.from_numpy(i420_to_i444(small.numpy(), w, h))
            elif twin:
                small = random_words((w * h * 3 // 2,), w + dw)
                big = i01x_to_i41x(small, w, h)
            else:   # I412Msb against I412: the same codes, shifted up with junk below
                gen = torch.Generator().manual_seed(w + dh)
                planes = [torch.randint(0, 1 << 12, (h, w), generator=gen, dtype=torch.int64) for _ in range(3)]
                junk = torch.randint(0, 1 << 16, (3 * w * h,), generator=gen, dtype=torch.int64)
                twin, small, big = "I412", pack16(*planes, "I412", junk), pack16(*planes, "I412Msb", junk)
            outs = []
            for f, raw in ((twin, small), (fmt, big)):
                out = torch.full((1, 3, dh, dw), float("nan"), dtype=torch.float16 if f16 else torch.float32, device=dev)
                (make_pre(kb, f, mode, sampling, "Bt709Limited").run_raw_f16 if f16 else make_pre(kb, f, mode, sampling, "Bt709Limited").run_raw)(
                    raw.to(dev), w, h, out)
                outs.append(out)
            assert torch.equal(outs[0].view(it), outs[1].view(it)), f"{fmt} vs {twin} {mode} {(w, h, dw, dh)}"


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["I444", "I412"])
def test_preprocess_unaligned_frames(kb, dev, fmt):
    """A frame off the identity kernel's load alignment leaves it for the 3b kernel with the same bits; a width that is
    not a multiple of 4 takes the generic kernel."""
    w, h = 64, 48
    b = 1 if fmt == "I444" else 2
    raw = frames_of(fmt, w, h, 1, 77)[0].to(dev)
    k = "i444" if fmt == "I444" else "i41x"
    for mode, dw, dh in (("Stretch", 64, 48), ("Stretch", 32, 24)):
        pre = make_pre(kb, fmt, mode, "Bilinear", "Bt709Limited")
        want = torch.full((1, 3, dh, dw), float("nan"), device=dev)
        pre.run_raw(raw, w, h, want)
        assert kb._lib.last_kernel() == (f"preprocess_{k}_identity_kernel" if dw == w else f"preprocess_{k}_kernel")
        shifted = offset_buf(dev, raw.numel(), 2, torch.uint8) if b == 1 else offset_buf(dev, raw.numel(), 1, torch.uint16)
        shifted.copy_(raw)
        got = torch.full_like(want, float("nan"))
        pre.run_raw(shifted, w, h, got)
        assert kb._lib.last_kernel() == f"preprocess_{k}_kernel"
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    # an odd width at the identity shape: the generic kernel, equal to the oracle path checked in test_preprocess
    raw = frames_of(fmt, 62, 48, 1, 78)[0].to(dev)
    out = torch.full((1, 3, 48, 62), float("nan"), device=dev)
    make_pre(kb, fmt, "Stretch", "Bilinear").run_raw(raw, 62, 48, out)
    assert kb._lib.last_kernel() == "preprocess_generic_kernel"


def torch_identity(raw, w, h, fmt, m, kb):
    """Config 3a of frames [n, 3*w*h] on the device: the restatement's decode, then (px / W - mean) * inv_std as separate
    IEEE f32 operations (W = 255 for bytes)."""
    wl = torch.full((1,), float(white(BITS[fmt])), dtype=torch.float32, device=raw.device)
    if fmt == "I444":
        y, u, v = (raw[:, k * w * h:(k + 1) * w * h].to(torch.int64).reshape(-1, h, w) for k in range(3))
        yo, cy, cvr, cub, cug, cvg = TABLE[m]
        yy = (y - yo).clamp(min=0) * cy
        u, v = u - 128, v - 128
        rgb = torch.stack([(yy + cvr * v + (1 << 19)) >> 20, (yy + cug * u + cvg * v + (1 << 19)) >> 20, (yy + cub * u + (1 << 19)) >> 20], -1).clamp(0, 255)
    else:
        rgb = decode_yuv444_16(raw, w, h, fmt, m)
    rgb = rgb.to(torch.float32) / wl
    mean = torch.tensor(kb.IMAGENET_MEAN, dtype=torch.float32, device=raw.device)
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(kb.IMAGENET_STD, dtype=torch.float32)
    return ((rgb - mean) * inv.to(raw.device)).permute(0, 3, 1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,m", [("I444", "Bt601Full"), ("I410Msb", "Bt709Limited"), ("I412", "Bt601Limited")])
@pytest.mark.parametrize("n", [256, 300])
def test_preprocess_identity_1080p(kb, dev, fmt, m, n):
    """Config 3a from 1080p frames at 256 and 300 frames (a second launch with frame0 > 0), through the pointer table and
    the strided entry, against the restatement for every frame."""
    w, h = 1920, 1080
    ne = 3 * w * h
    g = torch.Generator(device=dev).manual_seed(0x3A44 + CODE[fmt])
    if fmt == "I444":
        ring = torch.randint(0, 256, (n, ne + 64), dtype=torch.int32, device=dev, generator=g).to(torch.uint8)
    else:
        ring = torch.randint(0, 1 << 16, (n, ne + 32), dtype=torch.int32, device=dev, generator=g).to(torch.uint16)
    frames = ring[:, :ne]
    pre = make_pre(kb, fmt, "Stretch", "Bilinear", m)
    kernel = f"preprocess_{'i444' if fmt == 'I444' else 'i41x'}_identity_kernel"
    got = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)

    def check(entry):
        assert kb._lib.last_kernel() == kernel, entry
        for k0 in range(0, n, 16):
            want = torch_identity(frames[k0:k0 + 16], w, h, fmt, m, kb)
            assert torch.equal(got[k0:k0 + 16].view(torch.int32), want.contiguous().view(torch.int32)), f"{entry} frames {k0}.."

    pre.run_raw_batch([frames[k] for k in range(n)], w, h, got)
    check("pointer table")
    got.fill_(float("nan"))
    pre.run_raw_strided(ring.view(-1), ring.shape[1] * ring.element_size(), n, w, h, got)
    check("strided")
    del got, ring, frames
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["I444", "I410Msb"])
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 192, 108), ("Letterbox", 64, 64)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_pipeline(kb, dev, fmt, mode, dw, dh, f16):
    """run_raw_host carries [N, 3*w*h] frames (uint8 for I444, uint16 words for the 16-bit formats, and the same bytes as
    uint8): host frames in / host tensor out equal the device path, and the transfers are exactly the frames' bytes and
    the outputs' bytes."""
    w, h, n = 192, 108, 7
    b = 1 if fmt == "I444" else 2
    host = torch.stack(frames_of(fmt, w, h, n, 5 + CODE[fmt])).pin_memory()
    pre = make_pre(kb, fmt, mode, "Bilinear", "Bt709Limited")
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
    it = torch.int16 if f16 else torch.int32
    for frames in ((host,) if b == 1 else (host, host.view(torch.uint8))):
        pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * 3 * w * h * b, dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
        got = pre.run_raw_host(frames, w, h, (dw, dh), f16=f16, pipeline=pipe)
        torch.cuda.synchronize()
        h2d, d2h = pipe.last_transfer()
        pipe.close()
        assert h2d == n * 3 * w * h * b and d2h == n * 3 * dw * dh * (2 if f16 else 4)
        assert torch.equal(got.view(it), want.cpu().view(it))


# ── memory footprint (test_footprint's guards and poison) ──
def _footprint_cases():
    cases = []
    for (w, h), off, v in (((64, 48), False, "vec16"), ((70, 3), False, "generic"), ((64, 16), True, "generic")):
        cases.append(FootprintCase(f"i444-{w}x{h}{'-unaligned' if off else ''}", f"rgb_from_i444_{v}",
                          lambda k, w=w, h=h: random_bytes(3 * w * h, 90 + k),
                          lambda f, w=w, h=h: decode_yuv444(f, w, h, "Bt601Limited"),
                          lambda lib, s, sl, d, dl, n, aux, a=(w, h): lib.kb200_rgb_from_yuv444_u8(None, s, sl, d, dl, a[0], a[1], n, 0),
                          3 * w * h, 3 * w * h, batch=3, offset=off, row=w * 3))
    for fmt, (w, h), off, v in (("I410", (64, 48), False, "vec"), ("I412Msb", (70, 3), False, "generic"), ("I410Msb", (64, 16), True, "generic")):
        cases.append(FootprintCase(f"i41x-{fmt}-{w}x{h}{'-unaligned' if off else ''}", f"rgb_from_i41x_{v}",
                          lambda k, w=w, h=h: random_bytes(6 * w * h, 91 + k).view(np.uint16).copy(),
                          lambda f, w=w, h=h, fmt=fmt: decode_yuv444_16(torch.from_numpy(f.astype(np.int32)), w, h, fmt, "Bt601Limited").numpy().astype(np.uint16),
                          lambda lib, s, sl, d, dl, n, aux, a=(w, h, LAYOUT[fmt], BITS[fmt]): lib.kb200_rgb_from_yuv444_u16(None, s, sl, d, dl, a[0], a[1], n,
                                                                                                                          a[2], a[3], 0),
                          3 * w * h, 3 * w * h, batch=3, offset=off, row=w * 6))
    return {c.id: c for c in cases}


FOOTPRINT = _footprint_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(FOOTPRINT))
def test_decoder_footprint(kb, dev, cid):
    """Guards untouched, 0x00 and 0xFF prefills give the same bits, one element less of src or dst is refused; then three
    frames with the middle one poisoned (all max between all 0) leave the outer results alone."""
    lib, case = kb._lib.lib(), FOOTPRINT[cid]
    run_guarded(kb, lib, dev, case, [case.frame(k) for k in range(case.batch)], range(case.batch), True)
    run_guarded(kb, lib, dev, case, neighbour_frames(case), (0, 2), False)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["I444", "I412Msb"])
@pytest.mark.parametrize("geom", ["identity", "letterbox", "lanczos"])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_footprint(kb, dev, fmt, geom, f16):
    """Both device entries: the strided one with a poisoned gap between frames, the pointer-table one with each frame in
    its own guarded allocation; guards, 0x00 / 0xFF prefills, exact lengths, and results equal to the device run on the
    same frames packed tight."""
    lib = kb._lib.lib()
    mode, (dw, dh), sampling = {"identity": ("Stretch", (64, 48), "Bilinear"), "letterbox": ("Letterbox", (40, 40), "Bilinear"),
                                "lanczos": ("Letterbox", (40, 40), "Lanczos")}[geom]
    w, h, n = 64, 48, 3
    pre = make_pre(kb, fmt, mode, sampling, "Bt709Limited")
    frames = [f.numpy().reshape(-1).view(np.uint8) for f in frames_of(fmt, w, h, n, 0x444)]
    need = frames[0].size
    want = torch.full((n, 3, dh, dw), float("nan"), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([torch.from_numpy(f).to(dev).view(torch.uint8 if fmt == "I444" else torch.uint16)
                                                           for f in frames], w, h, want)
    want = want.cpu().numpy().reshape(-1).view(np.uint8)
    kernel = expected_preprocess_kernel(fmt, sampling, w, h, dw, dh)
    d = pre._desc(w, h, kb.SourceFormat[fmt].pitch(w), kb.SourceFormat[fmt].bpp(), kb.SourceFormat[fmt].fmt_code(), dw, dh)
    esz = 2 if f16 else 4
    out_elems = 3 * dw * dh
    gap = 48
    stride = need + gap
    ring = Guarded(dev, stride * (n - 1) + need, dw * esz)
    ring.load("u8", np.concatenate([np.concatenate([f, poison("u8", gap)]) for f in frames])[:stride * (n - 1) + need])
    ring_before = ring.snapshot()
    singles = [Guarded(dev, need, dw * esz).load("u8", frames[k]) for k in range(n)]
    singles_before = [g.snapshot() for g in singles]
    strided_fn = lib.kb200_preprocess_strided_f16 if f16 else lib.kb200_preprocess_strided_f32
    table_fn = lib.kb200_preprocess_f16 if f16 else lib.kb200_preprocess_f32
    ptrs = (C.c_void_p * n)(*[g.ptr for g in singles])
    lens = (C.c_size_t * n)(*[need] * n)
    calls = {
        "strided": lambda dst, dl, bl=ring.n: strided_fn(None, C.byref(d), ring.ptr, bl, stride, n, dst, dl),
        "table": lambda dst, dl, ln=lens: table_fn(None, C.byref(d), ptrs, ln, n, dst, dl),
    }
    for entry, call in calls.items():
        what = f"{fmt} {geom} {entry}"
        outs = []
        for fill in (0x00, 0xFF):
            dst = Guarded(dev, out_elems * esz * n, dw * esz).fill(fill)
            assert call(dst.ptr, out_elems * n) == 0, f"{what}: {kb._lib.last_error()}"
            assert kb._lib.last_kernel() == kernel, what
            torch.cuda.synchronize()
            lead, tail = dst.guards()
            assert np.all(lead == fill) and np.all(tail == fill), f"{what}: write outside dst"
            outs.append(dst.out())
        assert np.array_equal(outs[0], outs[1]), f"{what}: output left unwritten"
        assert np.array_equal(outs[0], want), f"{what}: differs from the tight device run"
        dst.fill(0x5A)
        before = dst.snapshot()
        assert call(dst.ptr, out_elems * n - 1) == -2 and "'dst'" in kb._lib.last_error()
        if entry == "strided":
            assert call(dst.ptr, out_elems * n, ring.n - 1) == -8 and f"need {ring.n}" in kb._lib.last_error()
        else:
            short = (C.c_size_t * n)(need, need - 1, need)
            assert call(dst.ptr, out_elems * n, short) == -8 and f"need {need}" in kb._lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(dst.snapshot(), before)
    assert np.array_equal(ring.snapshot(), ring_before)
    assert all(np.array_equal(g.snapshot(), b) for g, b in zip(singles, singles_before))
