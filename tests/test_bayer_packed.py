"""MIPI CSI-2 packed Bayer mosaics (RAW10, RAW12, RAW14): the packed demosaic and packed frames in the camera preprocess.

The packing only changes how samples are read from memory, so every check is against the frame's unpacked 16-bit twin:
a packed frame must give the same bits as the same samples unpacked into one LSB-aligned word each, on every path —
the decoder against `rgb_from_bayer16` and the numpy restatement of tests/restate.py, the preprocess against the
`BayerXxxNN` format of the same depth and the restated oracle.  A numpy / torch unpacker defines the packing and is
pinned by a known-answer table.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from harness import bayer16_identity, check_against_restatement, dev, make_pre, offset_buf, restated, to_dev16, to_np16
from restate import GROUP, GROUP_BYTES, PATTERNS, PATTERN_CODE, demosaic, fmt_name, pack, unpack, white


PDEPTHS = (10, 12, 14)


def pfmt_name(pattern, bits):
    return f"Bayer{pattern.capitalize()}{bits}p"


def pfmt_code(pattern, bits):
    return 64 + 4 * PDEPTHS.index(bits) + PATTERN_CODE[pattern]


def row_bytes(w, bits):
    return w * bits // 8


KNOWN = [(10, [0xFF, 0x00, 0x80, 0x01, 0xE4], [1020, 1, 514, 7]),
         (12, [0xAB, 0xCD, 0x21], [2737, 3282]),
         (14, [0x80, 0x01, 0xFF, 0x00, 0xBF, 0x5A, 0x05], [8255, 106, 16341, 1])]


# ═══ CPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
@pytest.mark.parametrize("bits,packed,samples", KNOWN)
def test_known_answers(bits, packed, samples):
    np.testing.assert_array_equal(unpack(np.array([packed], np.uint8), bits), [samples])
    np.testing.assert_array_equal(pack(np.array([samples]), bits), [packed])
    np.testing.assert_array_equal(unpack(torch.tensor([packed], dtype=torch.uint8), bits).numpy(), [samples])


@pytest.mark.parametrize("bits", PDEPTHS)
def test_pack_round_trip(bits):
    rng = np.random.default_rng(bits)
    v = rng.integers(0, 1 << bits, (3, 5, 8 * GROUP[bits]))
    v[0, 0, :4] = (1 << bits) - 1
    p = pack(v, bits)
    assert p.shape == (3, 5, 8 * GROUP_BYTES[bits]) and p.dtype == np.uint8
    np.testing.assert_array_equal(unpack(p, bits), v)
    np.testing.assert_array_equal(unpack(torch.from_numpy(p), bits).numpy(), v)
    # every byte string is a frame: unpack then pack gives it back
    raw = rng.integers(0, 256, (4, 6 * GROUP_BYTES[bits]), dtype=np.uint8)
    np.testing.assert_array_equal(pack(unpack(raw, bits), bits), raw)


def test_source_format_members(kb):
    SF = kb.SourceFormat
    for bits in PDEPTHS:
        for p in PATTERNS:
            f = SF[pfmt_name(p, bits)]
            assert f.value == f"bayer_{p.lower()}{bits}p" and f.fmt_code() == pfmt_code(p, bits)
            assert f.is_bayer() and f.is_bayer_packed() and not f.is_bayer16() and f.bit_depth() == bits
            assert SF.from_name(f"bayer_{p.lower()}{bits}p") is f and SF.from_name(f"BAYER_{p}{bits}P") is f
            assert not f.interleaved() and not f.is_yuv420() and not f.is_yuv422()
            assert f.pitch(8) == 8 * bits // 8 and f.pitch(1920) == 1920 * bits // 8
            assert f.buffer_len(8, 5) == 5 * 8 * bits // 8
            g = GROUP[bits]
            assert f.dims_ok(4, 3) and f.dims_ok(4 * g, 5) and not f.dims_ok(2, 9) and not f.dims_ok(8, 2)
            assert f.dims_ok(6, 3) == (g == 2)
    codes = sorted(f.fmt_code() for f in SF if f.is_bayer_packed())
    assert codes == list(range(64, 76))
    assert sorted(f.fmt_code() for f in SF if f.is_bayer16()) == list(range(32, 48))
    assert SF.from_name("bayer_rggb16p") is None and SF.from_name("bayer_rggb8p") is None


def test_validation_without_a_gpu(kb):
    """Every rejection of both entry points, with its message, before any CUDA call."""
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = (C.addressof(buf) + 15) & ~15
    n = 2048
    for bad in (-1, 4):
        assert l.kb200_rgb_from_bayer_packed(None, p, n, p, n, 4, 4, 1, bad, 12) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown Bayer pattern {bad}"
    for bits in (8, 11, 16, 0):
        assert l.kb200_rgb_from_bayer_packed(None, p, n, p, n, 4, 4, 1, 0, bits) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"packed Bayer samples are 10, 12 or 14 bits, got {bits}"
    assert l.kb200_rgb_from_bayer_packed(None, p, n, p + 1, n, 8, 4, 1, 0, 12) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "'dst' is not 2-byte aligned (16-bit samples)"
    for p_name, code in PATTERN_CODE.items():
        for bits in PDEPTHS:
            g, gb = GROUP[bits], GROUP_BYTES[bits]
            for w, h in ((4, 2), (2, 7), (2, 2)):
                assert l.kb200_rgb_from_bayer_packed(None, p, n, p, n, w, h, 1, code, bits) == _lib.ERR_INVALID_ARGUMENT
                assert _lib.last_error() == f"Bayer {p_name}{bits}P needs at least 3x3 pixels, got {w}x{h}"
            for w in (g + 1, 2 * g + 1, 6 if g == 4 else 7):
                assert l.kb200_rgb_from_bayer_packed(None, p, n, p, n, w, 4, 1, code, bits) == _lib.ERR_INVALID_ARGUMENT
                assert _lib.last_error() == f"Bayer {p_name}{bits}P needs a width that is a multiple of {g} (whole {gb}-byte groups), got {w}"
            # src in bytes (any alignment), dst in elements
            w, h, b = 8, 4, 2
            assert l.kb200_rgb_from_bayer_packed(None, p + 1, row_bytes(w, bits) * h * b - 1, p, n, w, h, b, code, bits) == _lib.ERR_SLICE_TOO_SMALL
            assert _lib.last_error() == f"device slice 'src' length {row_bytes(w, bits) * h * b - 1} < required {row_bytes(w, bits) * h * b}"
            assert l.kb200_rgb_from_bayer_packed(None, p + 1, n, p, w * h * 3 * b - 1, w, h, b, code, bits) == _lib.ERR_SLICE_TOO_SMALL
            assert _lib.last_error() == f"device slice 'dst' length {w * h * 3 * b - 1} < required {w * h * 3 * b}"
    with pytest.raises(ValueError):
        kb.imgproc.rgb_from_bayer_packed(None, None, 4, 12)
    with pytest.raises(ValueError, match="packed Bayer samples are 10, 12 or 14 bits, got 16"):
        kb.imgproc.rgb_from_bayer_packed(None, None, 0, 16)

    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(80)
    for bits in PDEPTHS:
        for p_name in PATTERNS:
            name = pfmt_name(p_name, bits)
            g, gb = GROUP[bits], GROUP_BYTES[bits]
            d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = 8, 2, 16, 1, pfmt_code(p_name, bits), 4, 4, 1
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source for {name} at 8x2 (at least 3x3 required)"
            d.src_w, d.src_h = 2, 6
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source for {name} at 2x6 (at least 3x3 required)"
            d.src_w = g + 1
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source for {name} at {g + 1}x6 (the width must be a multiple of {g}: whole {gb}-byte groups)"
            d.src_w, d.src_pitch = 8, row_bytes(8, bits) - 1
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid pitched surface for {name} (pitch {row_bytes(8, bits) - 1} < {row_bytes(8, bits)} bytes of a packed row)"
            d.src_pitch = row_bytes(8, bits) + 3   # any pitch >= the row: no alignment requirement
            assert l.kb200_preprocess_src_bytes(C.byref(d)) == d.src_pitch * 6
            small = (C.c_size_t * 1)(d.src_pitch * 6 - 1)
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, small, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert f"got {d.src_pitch * 6 - 1} bytes, need {d.src_pitch * 6}" in _lib.last_error()
            assert l.kb200_preprocess_strided_f16(None, C.byref(d), p + 1, d.src_pitch * 6 - 1, d.src_pitch, 1, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
            assert f"need {d.src_pitch * 6}" in _lib.last_error()
    for code in (60, 61, 62, 63, 76, 79):
        d.fmt = code
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown source format code {code}"

    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.BayerRggb12p).build_cuda()
    with pytest.raises(kb.PreprocessError, match="need 54"):
        pre._validate_raw(53, 12, 3)
    with pytest.raises(kb.PreprocessError):
        pre._validate_raw(1000, 13, 3)   # not a whole number of groups


# ═══ GPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def decode(kb, dev, pattern, bits, src, w, h, n, dst_off=0):
    out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint16)
    out.fill_(0xCDCD)
    kb.imgproc.rgb_from_bayer_packed(src, kb.Image(out.view(n, h, w, 3)), kb.imgproc.BayerPattern[pattern], bits)
    return out.view(n, h, w, 3), kb._lib.last_kernel()


def decode16(kb, dev, pattern, samples, w, h, n):
    out = torch.empty((n, h, w, 3), dtype=torch.uint16, device=dev)
    kb.imgproc.rgb_from_bayer16(samples.to(torch.uint16).reshape(n, h * w), kb.Image(out), kb.imgproc.BayerPattern[pattern])
    return out


def decode_kernel(pattern, bits, w, soff, doff):
    vec = (w * bits) % 128 == 0 and soff % 16 == 0 and (2 * doff) % 16 == 0
    return f"rgb_from_bayer{bits}p_{pattern.lower()}_{'vec' if vec else 'generic'}"


def contents(bits, w, h, seed):
    """Full-range random, all-white, only the low bit fields set, and a 0 / W checkerboard and stripes."""
    W = white(bits)
    yy, xx = np.mgrid[0:h, 0:w]
    rng = np.random.default_rng(seed)
    return np.stack([rng.integers(0, 1 << bits, (h, w)), np.full((h, w), W), rng.integers(0, 1 << (bits - 8), (h, w)),
                     ((xx + yy) & 1) * W, (xx & 1) * W]).astype(np.int64)


SIZES = [(1920, 1080), (256, 6), (320, 7), (64, 5), (36, 5), (4, 3), (132, 9)]   # (w * bits) % 128 == 0: the first four
OFFSETS = [(0, 0), (1, 0), (16, 0), (0, 3), (0, 8)]   # src offset in bytes, dst offset in elements
DECODE_CASES = [(b, p, s, o) for b in PDEPTHS for p in PATTERNS for s in SIZES for o in (OFFSETS if s == (256, 6) else OFFSETS[:1])]
DECODE_CASES += [(12, p, (38, 5), (0, 0)) for p in PATTERNS]   # a RAW12 width that is not a multiple of 4


@pytest.mark.gpu
@pytest.mark.parametrize("bits,pattern,size,offs", DECODE_CASES,
                         ids=[f"{b}p-{p}-{s[0]}x{s[1]}-off{o[0]}.{o[1]}" for b, p, s, o in DECODE_CASES])
def test_decode_packed(kb, dev, bits, pattern, size, offs):
    """Every depth x pattern on fast and generic geometries and offsets: bit-equal to rgb_from_bayer16 on the unpacked
    mosaic and to the restatement, with the kernel the dispatch promises."""
    w, h = size
    soff, doff = offs
    v = contents(bits, w, h, w * 31 + h + 7 * bits + PATTERN_CODE[pattern])
    n = len(v)
    packed = pack(v, bits)
    src = offset_buf(dev, packed.size, soff, torch.uint8)
    src.copy_(torch.from_numpy(packed.reshape(-1)).to(dev))
    got, kern = decode(kb, dev, pattern, bits, src, w, h, n, doff)
    assert kern == decode_kernel(pattern, bits, w, soff, doff)
    samples = to_dev16(v.reshape(-1), dev)
    twin = decode16(kb, dev, pattern, samples, w, h, n)
    assert torch.equal(got.view(torch.int16), twin.view(torch.int16))
    if w * h <= 320 * 7:
        g = to_np16(got)
        for k in range(n):
            np.testing.assert_array_equal(g[k], demosaic(v[k].astype(np.uint16), pattern), f"frame {k}")
    else:
        for k in range(n):
            assert torch.equal(got[k].view(torch.int16), demosaic(samples.view(n, h, w)[k], pattern).view(torch.int16)), f"frame {k}"
    if w >= 36:
        assert (to_np16(got[1]) == white(bits)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("bits", PDEPTHS)
def test_decode_packed_1080p_batch(kb, dev, bits):
    """1080p x 256 of random bytes (every byte string is a packed frame): the fast kernel, bit-equal to rgb_from_bayer16
    on the device-unpacked samples."""
    w, h, n = 1920, 1080, 256
    g = torch.Generator(device=dev).manual_seed(0x10AD + bits)
    raw = torch.randint(0, 256, (n, h * row_bytes(w, bits)), dtype=torch.uint8, device=dev, generator=g)
    got, kern = decode(kb, dev, "GRBG", bits, raw.view(-1), w, h, n)
    assert kern == f"rgb_from_bayer{bits}p_grbg_vec"
    for k0 in range(0, n, 32):
        samples = unpack(raw[k0:k0 + 32].view(-1, h, row_bytes(w, bits)), bits)
        assert torch.equal(got[k0:k0 + 32].view(torch.int16), decode16(kb, dev, "GRBG", samples, w, h, 32).view(torch.int16)), f"frames {k0}.."
    del got, raw
    torch.cuda.empty_cache()


# ── camera preprocess ──
PGEOMS = [(8, 6, 7, 5), (64, 48, 40, 40), (64, 48, 64, 48), (28, 20, 61, 47), (128, 72, 40, 24),
          (96, 54, 32, 32), (32, 24, 64, 48), (192, 108, 64, 36), (36, 21, 36, 21), (20, 3, 20, 3)]
PFORMATS = [("RGGB", b) for b in PDEPTHS] + [(p, 12) for p in PATTERNS[1:]]


def expected_kernel(pattern, bits, sampling, w, h, dw, dh, pitch):
    if sampling != "Lanczos" and (dw, dh) == (w, h) and w % 4 == 0 and pitch % 16 == 0:
        return f"preprocess_bayer{bits}p_{pattern.lower()}_identity_kernel"
    return "preprocess_generic_kernel"


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,bits", PFORMATS)
@pytest.mark.parametrize("mode", ["Letterbox", "Stretch"])
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_packed(kb, dev, pattern, bits, mode, sampling, f16):
    """Every geometry: bit-equal to the same frame unpacked and run as the 16-bit format of its depth, and to the
    restated oracle on the RGB16 twin (Lanczos: within test_bayer16's tolerance)."""
    pre = make_pre(kb, pfmt_name(pattern, bits), mode, sampling)
    twin_pre = make_pre(kb, fmt_name(pattern, bits), mode, sampling)
    dt = torch.float16 if f16 else torch.float32
    it = torch.int16 if f16 else torch.int32
    for w, h, dw, dh in PGEOMS:
        what = f"{pattern}{bits}p {mode} {sampling} {'f16' if f16 else 'f32'} {(w, h, dw, dh)}"
        v = contents(bits, w, h, w + h + bits)[(w + h) % 5]
        got = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_f16 if f16 else pre.run_raw)(torch.from_numpy(pack(v, bits).reshape(-1)).to(dev), w, h, got)
        assert kb._lib.last_kernel() == expected_kernel(pattern, bits, sampling, w, h, dw, dh, row_bytes(w, bits)), what
        want = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (twin_pre.run_raw_f16 if f16 else twin_pre.run_raw)(to_dev16(v.reshape(-1), dev), w, h, want)
        assert torch.equal(got.view(it), want.view(it)), what
        o = restated(kb, demosaic(v.astype(np.uint16), pattern), bits, mode, sampling, dw, dh, f16 and sampling != "Lanczos")
        check_against_restatement(got[0], o, sampling, f16, what)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,bits", [("RGGB", 12), ("GBRG", 10), ("BGGR", 14)])
@pytest.mark.parametrize("n", [256, 300])
def test_preprocess_packed_identity_1080p(kb, dev, pattern, bits, n):
    """Config 3a from 1080p packed frames at 256 and 300 frames (a second launch with frame0 > 0), through the pointer
    table and the strided entry: every frame bit-equal to the device-unpacked samples normalised in torch."""
    w, h = 1920, 1080
    fb = row_bytes(w, bits) * h
    g = torch.Generator(device=dev).manual_seed(0x3A0 + bits + PATTERN_CODE[pattern])
    ring = torch.randint(0, 256, (n, fb + 32), dtype=torch.uint8, device=dev, generator=g)   # padded strided slots
    frames = ring[:, :fb]
    pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat[pfmt_name(pattern, bits)]).mode(kb.ResizeMode.Stretch)
           .normalize(kb.Normalize.imagenet()).build_cuda())
    kernel = f"preprocess_bayer{bits}p_{pattern.lower()}_identity_kernel"
    got = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)

    def check(entry):
        assert kb._lib.last_kernel() == kernel, entry
        for k0 in range(0, n, 32):
            want = bayer16_identity(unpack(frames[k0:k0 + 32].reshape(-1, h, row_bytes(w, bits)), bits), pattern, bits, kb)
            assert torch.equal(got[k0:k0 + 32].view(torch.int32), want.contiguous().view(torch.int32)), f"{entry} frames {k0}.."

    pre.run_raw_batch([frames[k] for k in range(n)], w, h, got)
    check("pointer table")
    got.fill_(float("nan"))
    pre.run_raw_strided(ring.view(-1), fb + 32, n, w, h, got)
    check("strided")
    del got, ring, frames
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("pitch_pad", [16, 5])
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 128, 54), ("Letterbox", 40, 40)])
def test_preprocess_packed_pitched(kb, dev, pitch_pad, mode, dw, dh):
    """A pitched packed frame (pitch > w*bits/8 bytes) gives the bits of its tight copy, on the identity kernel (a
    16-aligned pitch) and on the generic one (a pitch that is not)."""
    from kornia_rs_b200 import _lib

    w, h, bits = 128, 54, 14   # tight rows of 224 bytes: 16-B aligned
    rb = row_bytes(w, bits)
    pitch = rb + pitch_pad
    tight = torch.from_numpy(pack(contents(bits, w, h, 3)[0], bits)).to(dev)
    pitched = torch.full((h, pitch), 0xEE, dtype=torch.uint8, device=dev)
    pitched[:, :rb] = tight
    pre = make_pre(kb, "BayerGrbg14p", mode, "Bilinear")
    want = torch.full((1, 3, dh, dw), float("nan"), device=dev)
    pre.run_raw(tight.view(-1), w, h, want)
    tight_kernel = kb._lib.last_kernel()
    got = torch.full((1, 3, dh, dw), float("nan"), device=dev)
    desc = pre._desc(w, h, pitch, 1, kb.SourceFormat.BayerGrbg14p.fmt_code(), dw, dh)
    assert _lib.lib().kb200_preprocess_src_bytes(C.byref(desc)) == pitch * h
    pre._launch(desc, [pitched.view(-1)], got, False)
    identity = mode == "Stretch" and pitch % 16 == 0
    assert kb._lib.last_kernel() == ("preprocess_bayer14p_grbg_identity_kernel" if identity else "preprocess_generic_kernel")
    assert tight_kernel == ("preprocess_bayer14p_grbg_identity_kernel" if mode == "Stretch" else "preprocess_generic_kernel")
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 192, 108), ("Letterbox", 64, 64)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_pipeline_packed(kb, dev, mode, dw, dh, f16):
    """run_raw_host carries [N, pitch*h] uint8 packed frames: host frames in / host tensor out equal the device path, and
    the upload is exactly N * pitch * h bytes."""
    w, h, n, bits = 192, 108, 7, 12
    fb = row_bytes(w, bits) * h
    host = torch.from_numpy(np.stack([pack(contents(bits, w, h, k)[0], bits).reshape(-1) for k in range(n)])).pin_memory()
    pre = make_pre(kb, "BayerRggb12p", mode, "Bilinear")
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * fb, dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
    got = pre.run_raw_host(host, w, h, (dw, dh), f16=f16, pipeline=pipe)
    torch.cuda.synchronize()
    h2d, d2h = pipe.last_transfer()
    pipe.close()
    assert h2d == n * fb and d2h == n * 3 * dw * dh * (2 if f16 else 4)
    it = torch.int16 if f16 else torch.int32
    assert torch.equal(got.view(it), want.cpu().view(it))
