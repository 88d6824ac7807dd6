"""10- to 16-bit Bayer mosaics: the standalone 16-bit demosaic and 16-bit-sample Bayer frames in the camera preprocess.

Samples are LSB-aligned little-endian 16-bit words (V4L2's unpacked SRGGB10 ... SGBRG16).  The demosaic is the 8-bit
one on the 16-bit values, pinned to OpenCV through tests/golden/bayer16_cv2.npz (cv2.cvtColor on uint16 mosaics) and a
numpy / torch restatement.  In the preprocess a tap is the demosaiced pixel at the tap's coordinate, normalised by the
format's white level W = 2^bits - 1, so a frame is checked through its RGB16 twin (the restatement's demosaic) against
a numpy restatement of the oracle's preprocess for interleaved 16-bit RGB with `px / W` in place of `px / 255`.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from harness import bayer16_identity, check_against_restatement, dev, make_pre, offset_buf, restated, to_dev16, to_np16
from restate import DEPTHS, PATTERNS, PATTERN_CODE, demosaic, fmt_name

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def fmt_code(pattern, bits):
    return 32 + 4 * DEPTHS.index(bits) + PATTERN_CODE[pattern]


# ═══ CPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def test_cv2_fixture_matches_the_restatement():
    """cv2's COLOR_Bayer??2RGB on uint16 mosaics = the restatement, numpy and torch: every pattern, 10-, 12- and
    full-range 16-bit content, odd and even sizes, and an all-65535 frame."""
    fx = np.load(os.path.join(GOLDEN, "bayer16_cv2.npz"))
    names = sorted({k.rsplit("_", 1)[0] for k in fx.files})
    assert len(names) == 4 * (3 * 5 + 1)
    for name in names:
        pattern = name.split("_")[0].upper()
        raw, want, (w, h) = fx[f"{name}_raw"], fx[f"{name}_rgb"], (int(v) for v in fx[f"{name}_wh"])
        assert raw.shape == (h, w) and raw.dtype == np.uint16 and want.dtype == np.uint16, name
        np.testing.assert_array_equal(demosaic(raw, pattern), want, name)
        np.testing.assert_array_equal(demosaic(torch.from_numpy(raw.astype(np.int32)).to(torch.uint16), pattern).to(torch.int32).numpy(),
                                      want.astype(np.int32), name)
        if name.split("_")[1] == "max":
            assert (want == 65535).all(), name


def test_source_format_members(kb):
    SF = kb.SourceFormat
    for bits in DEPTHS:
        for p in PATTERNS:
            f = SF[fmt_name(p, bits)]
            assert f.value == f"bayer_{p.lower()}{bits}" and f.fmt_code() == fmt_code(p, bits)
            assert f.bpp() == 2 and f.pitch(10) == 20 and f.bit_depth() == bits and f.is_bayer() and f.is_bayer16()
            assert SF.from_name(f"bayer_{p.lower()}{bits}") is f and SF.from_name(f"BAYER_{p}{bits}") is f
            assert not f.interleaved() and not f.is_yuv420() and not f.is_yuv422()
            assert f.buffer_len(8, 5) == 80 and f.dims_ok(3, 3) and f.dims_ok(7, 5) and not f.dims_ok(2, 9) and not f.dims_ok(9, 2)
    for p in PATTERNS:
        assert SF["Bayer" + p.capitalize()].bit_depth() == 8 and not SF["Bayer" + p.capitalize()].is_bayer16()
    assert SF.Nv12.bit_depth() is None and SF.Rgb8.bit_depth() is None
    codes = sorted(f.fmt_code() for f in SF if f.is_bayer16())
    assert codes == list(range(32, 48))
    assert SF.from_name("bayer_rggb8") is None and SF.from_name("bayer_rggb11") is None


def test_validation_without_a_gpu(kb):
    """Misaligned pointers, unknown patterns, sides below 3, short buffers, odd or short pitches and unknown format codes
    fail on the host, before any CUDA call."""
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = (C.addressof(buf) + 15) & ~15
    n = 2048   # elements of 16-bit room
    for bad in (-1, 4):
        assert l.kb200_rgb_from_bayer_u16(None, p, n, p, n, 4, 4, 1, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown Bayer pattern {bad}"
    assert l.kb200_rgb_from_bayer_u16(None, p + 1, n, p, n, 16, 4, 1, 0) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "'src' is not 2-byte aligned (16-bit samples)"
    assert l.kb200_rgb_from_bayer_u16(None, p, n, p + 3, n, 16, 4, 1, 0) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "'dst' is not 2-byte aligned (16-bit samples)"
    for p_name, code in PATTERN_CODE.items():
        for w, h in ((2, 7), (7, 2), (2, 2)):
            assert l.kb200_rgb_from_bayer_u16(None, p, n, p, n, w, h, 1, code) == _lib.ERR_INVALID_ARGUMENT
            assert _lib.last_error() == f"Bayer {p_name} needs at least 3x3 pixels, got {w}x{h}"
        # lengths are in elements
        assert l.kb200_rgb_from_bayer_u16(None, p, 5 * 4 * 2 - 1, p, n, 5, 4, 2, code) == _lib.ERR_SLICE_TOO_SMALL
        assert l.kb200_rgb_from_bayer_u16(None, p, n, p, 5 * 4 * 3 * 2 - 1, 5, 4, 2, code) == _lib.ERR_SLICE_TOO_SMALL
    with pytest.raises(ValueError):
        kb.imgproc.rgb_from_bayer16(None, None, 4)

    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(80)
    for bits in DEPTHS:
        for p_name in PATTERNS:
            name = fmt_name(p_name, bits)
            d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = 8, 2, 16, 2, fmt_code(p_name, bits), 4, 4, 1
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source for {name} at 8x2 (at least 3x3 required)"
            d.src_w, d.src_h, d.src_pitch = 2, 6, 4
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source for {name} at 2x6 (at least 3x3 required)"
            d.src_w, d.src_h, d.src_pitch = 8, 6, 17   # odd pitch
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid pitched surface for {name} (pitch 17 is odd: rows of 16-bit samples must start 2-byte aligned)"
            d.src_pitch = 14   # even, but < 2 * width
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error().startswith("invalid pitched surface")
            d.src_pitch = 18
            assert l.kb200_preprocess_src_bytes(C.byref(d)) == 108
            assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
            assert "got 80 bytes, need 108" in _lib.last_error()
            # frames that do not start 2-byte aligned: the pointer table, the strided base and the strided stride
            d.src_pitch = 16
            odd = (C.c_void_p * 1)(p + 1)
            assert l.kb200_preprocess_f32(None, C.byref(d), odd, (C.c_size_t * 1)(4096), 1, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"{name} frame 0 is not 2-byte aligned"
            assert l.kb200_preprocess_strided_f32(None, C.byref(d), p + 1, 4096, 96, 1, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error().startswith(f"{name} frames must start 2-byte aligned")
            assert l.kb200_preprocess_strided_f16(None, C.byref(d), p, 4096, 97, 2, p, 1 << 20) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error().startswith(f"{name} frames must start 2-byte aligned")
    for code in (10, 15, 20, 31, 48, 63, -1):
        d.fmt = code
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown source format code {code}"


def test_u16_image_exports_a_typestr(kb):
    from kornia_rs_b200 import image

    assert image._TYPESTR[torch.uint16] == "<u2"


# ═══ GPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def run_decode(kb, dev, pattern, raw_dev, w, h, n, dst_off=0):
    out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint16)
    out.fill_(0xCDCD)
    kb.imgproc.rgb_from_bayer16(raw_dev, kb.Image(out.view(n, h, w, 3)), kb.imgproc.BayerPattern[pattern])
    return out.view(n, h, w, 3), kb._lib.last_kernel()


def decode_kernel(pattern, w, soff, doff):
    vec = w % 8 == 0 and (2 * soff) % 16 == 0 and (2 * doff) % 16 == 0
    return f"rgb_from_bayer16_{pattern.lower()}_{'vec' if vec else 'generic'}"


CASES = [   # w, h, batch, src offset, dst offset (in samples)
    (64, 48, 1, 0, 0), (128, 31, 3, 0, 0), (512, 16, 4, 0, 0), (2056, 5, 2, 0, 0), (8, 3, 2, 0, 0), (16, 4, 1, 0, 0),  # vec
    (70, 6, 2, 0, 0), (131, 9, 3, 0, 0), (3, 3, 1, 0, 0), (7, 5, 4, 0, 0), (36, 17, 2, 0, 0),                         # 8 ∤ w
    (64, 48, 2, 1, 0), (64, 48, 2, 0, 3), (64, 48, 1, 8, 8), (130, 14, 1, 5, 0), (64, 48, 1, 4, 4),                   # unaligned
]
DECODE_CASES = [(p, c) for p in PATTERNS for c in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,case", DECODE_CASES, ids=[f"{p}-{'x'.join(map(str, c))}" for p, c in DECODE_CASES])
def test_decode_bayer16(kb, dev, pattern, case):
    w, h, n, soff, doff = case
    bits = DEPTHS[(w + h) % 4]
    raws = np.random.default_rng(w * 7919 + h * 31 + n + 1000 * PATTERN_CODE[pattern]).integers(0, 1 << bits, (n, h, w), dtype=np.uint16)
    src = offset_buf(dev, n * w * h, soff, torch.uint16)
    src.copy_(to_dev16(raws.reshape(-1), dev))
    got, kern = run_decode(kb, dev, pattern, src.view(n, w * h), w, h, n, doff)
    assert kern == decode_kernel(pattern, w, soff, doff)
    g = to_np16(got)
    for k in range(n):
        np.testing.assert_array_equal(g[k], demosaic(raws[k], pattern), f"{pattern} {case} frame {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("w,h", [(64, 6), (37, 5)])
def test_decode_bayer16_extremes(kb, dev, pattern, w, h):
    """All-65535, all-zero and 0 / 65535 checkerboard and stripe frames: the largest sums and the sharpest edges."""
    yy, xx = np.mgrid[0:h, 0:w]
    frames = np.stack([np.full((h, w), 65535), np.zeros((h, w)), ((xx + yy) & 1) * 65535, (xx & 1) * 65535,
                       (yy & 1) * 65535, 65535 - ((xx + yy) & 1)]).astype(np.uint16)
    n = len(frames)
    got, kern = run_decode(kb, dev, pattern, to_dev16(frames.reshape(n, -1), dev), w, h, n)
    assert kern == decode_kernel(pattern, w, 0, 0)
    g = to_np16(got)
    for k in range(n):
        np.testing.assert_array_equal(g[k], demosaic(frames[k], pattern), f"frame {k}")
    assert (g[0] == 65535).all()


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
def test_decode_bayer16_1080p_batch(kb, dev, pattern):
    w, h, n = 1920, 1080, 256
    g = torch.Generator(device=dev).manual_seed(0x1016 + PATTERN_CODE[pattern])
    raw = torch.randint(0, 1 << 16, (n, h * w), dtype=torch.int32, device=dev, generator=g).to(torch.uint16)
    got, kern = run_decode(kb, dev, pattern, raw, w, h, n)
    assert kern == f"rgb_from_bayer16_{pattern.lower()}_vec"
    for k0 in range(0, n, 32):
        assert torch.equal(got[k0:k0 + 32].view(torch.int16), demosaic(raw[k0:k0 + 32].view(-1, h, w), pattern).view(torch.int16)), f"frames {k0}.."
    del got, raw
    torch.cuda.empty_cache()


# ── camera preprocess ──
GEOMS = [(8, 6, 7, 5), (64, 48, 40, 40), (64, 48, 64, 48), (30, 20, 61, 47), (128, 72, 40, 24),
         (96, 54, 32, 32), (32, 24, 64, 48), (192, 108, 64, 36), (37, 21, 37, 21), (20, 3, 20, 3)]   # test_bayer's
FORMATS = [("RGGB", b) for b in DEPTHS] + [(p, 12) for p in PATTERNS[1:]]


def raw_samples(n, bits, k=0):
    return ((np.arange(n, dtype=np.int64) * 7919 + 13 + 4099 * k) % (1 << bits)).astype(np.uint16)


def expected_preprocess_kernel(pattern, sampling, w, h, dw, dh):
    if sampling != "Lanczos" and (dw, dh) == (w, h) and w % 4 == 0:
        return f"preprocess_bayer16_{pattern.lower()}_identity_kernel"
    return "preprocess_generic_kernel"


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,bits", FORMATS)
@pytest.mark.parametrize("mode", ["Letterbox", "Stretch"])
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_bayer16(kb, dev, pattern, bits, mode, sampling, f16):
    """Every geometry: bit-equal to the restated oracle on the RGB16 twin (Lanczos: within the tolerance of
    test_preprocess_lanczos_vs_oracle), with the kernel the dispatch promises."""
    pre = make_pre(kb, fmt_name(pattern, bits), mode, sampling)
    dt = torch.float16 if f16 else torch.float32
    for w, h, dw, dh in GEOMS:
        what = f"{pattern}{bits} {mode} {sampling} {'f16' if f16 else 'f32'} {(w, h, dw, dh)}"
        raw = raw_samples(w * h, bits, PATTERN_CODE[pattern])
        got = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_f16 if f16 else pre.run_raw)(to_dev16(raw, dev), w, h, got)
        assert kb._lib.last_kernel() == expected_preprocess_kernel(pattern, sampling, w, h, dw, dh), what
        o = restated(kb, demosaic(raw.reshape(h, w), pattern), bits, mode, sampling, dw, dh, f16 and sampling != "Lanczos")
        check_against_restatement(got[0], o, sampling, f16, what)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,bits", [("RGGB", 12), ("GBRG", 10)])
@pytest.mark.parametrize("n", [256, 300])
def test_preprocess_bayer16_identity_1080p(kb, dev, pattern, bits, n):
    """Config 3a from 1080p 16-bit Bayer frames at 256 and 300 frames (a second launch with frame0 > 0), through the
    pointer table and the strided entry, against the restatement for every frame."""
    w, h = 1920, 1080
    ns = w * h
    g = torch.Generator(device=dev).manual_seed(0x3A16 + PATTERN_CODE[pattern])
    ring = torch.randint(0, 1 << bits, (n, ns + 32), dtype=torch.int32, device=dev, generator=g).to(torch.uint16)   # padded strided slots
    frames = ring[:, :ns]
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt_name(pattern, bits)]).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda()
    kernel = f"preprocess_bayer16_{pattern.lower()}_identity_kernel"
    got = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)

    def check(entry):
        assert kb._lib.last_kernel() == kernel, entry
        for k0 in range(0, n, 32):
            want = bayer16_identity(frames[k0:k0 + 32].reshape(-1, h, w), pattern, bits, kb)
            assert torch.equal(got[k0:k0 + 32].view(torch.int32), want.contiguous().view(torch.int32)), f"{entry} frames {k0}.."

    pre.run_raw_batch([frames[k] for k in range(n)], w, h, got)
    check("pointer table")
    got.fill_(float("nan"))
    pre.run_raw_strided(ring.view(-1), 2 * (ns + 32), n, w, h, got)
    check("strided")
    for k in sorted({0, 255, n - 1}):   # the f32 restatement of the oracle on frames on both sides of the launch split
        o = restated(kb, demosaic(to_np16(frames[k]).reshape(h, w), pattern), bits, "Stretch", "Bilinear", w, h)
        np.testing.assert_array_equal(got[k].cpu().numpy().view(np.uint32), o.view(np.uint32), f"frame {k}")
    del got, ring, frames
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("pitch_pad", [16, 4])
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 96, 54), ("Letterbox", 40, 40)])
def test_preprocess_bayer16_pitched(kb, dev, pitch_pad, mode, dw, dh):
    """A pitched 16-bit Bayer frame (row pitch > 2*width bytes) gives the bits of its tight copy, on the identity kernel
    (pitch % 8 == 0) and on the generic one (an even pitch that is not a multiple of 8)."""
    from kornia_rs_b200 import _lib

    w, h = 96, 54
    pitch = 2 * w + pitch_pad   # bytes
    tight = to_dev16(raw_samples(w * h, 14, 3), dev)
    pitched = torch.full((h, pitch // 2), 0xEEEE, dtype=torch.int32, device=dev).to(torch.uint16)
    pitched[:, :w] = tight.view(h, w)
    pre = make_pre(kb, "BayerGrbg14", mode, "Bilinear")
    want = torch.full((1, 3, dh, dw), float("nan"), device=dev)
    pre.run_raw(tight, w, h, want)
    tight_kernel = kb._lib.last_kernel()
    got = torch.full((1, 3, dh, dw), float("nan"), device=dev)
    desc = pre._desc(w, h, pitch, 2, kb.SourceFormat.BayerGrbg14.fmt_code(), dw, dh)
    assert _lib.lib().kb200_preprocess_src_bytes(C.byref(desc)) == pitch * h
    pre._launch(desc, [pitched.view(-1)], got, False)
    identity = mode == "Stretch" and pitch % 8 == 0
    assert kb._lib.last_kernel() == ("preprocess_bayer16_grbg_identity_kernel" if identity else "preprocess_generic_kernel")
    assert tight_kernel == ("preprocess_bayer16_grbg_identity_kernel" if mode == "Stretch" else "preprocess_generic_kernel")
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,dw,dh,sampling", [("Stretch", 64, 48, "Bilinear"), ("Letterbox", 40, 40, "Bilinear"),
                                                  ("Stretch", 40, 30, "Lanczos")])
def test_preprocess_bayer16_above_white(kb, dev, mode, dw, dh, sampling):
    """A 10-bit format fed samples up to 65535: nothing is clamped, the taps run through (px / 1023 - mean) * inv_std."""
    w, h = 64, 48
    raw = np.random.default_rng(7).integers(0, 65536, w * h, dtype=np.uint16)
    raw[:64] = 65535
    pre = make_pre(kb, "BayerBggr10", mode, sampling)
    got = torch.full((1, 3, dh, dw), float("nan"), device=dev)
    pre.run_raw(to_dev16(raw, dev), w, h, got)
    assert kb._lib.last_kernel() == expected_preprocess_kernel("BGGR", sampling, w, h, dw, dh)
    o = restated(kb, demosaic(raw.reshape(h, w), "BGGR"), 10, mode, sampling, dw, dh)
    check_against_restatement(got[0], o, sampling, False, mode)
    assert got.max().item() > 100.0   # far above what a 10-bit sample reaches


@pytest.mark.gpu
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 192, 108), ("Letterbox", 64, 64)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_pipeline_bayer16(kb, dev, mode, dw, dh, f16):
    """run_raw_host carries [N, w*h] uint16 frames: host frames in / host tensor out equal the device path, and the
    transfers are exactly the frames' 2*w*h bytes and the outputs' bytes."""
    w, h, n = 192, 108, 7
    host = torch.from_numpy(np.stack([raw_samples(w * h, 12, k) for k in range(n)]).astype(np.int32)).to(torch.uint16).pin_memory()
    pre = make_pre(kb, "BayerRggb12", mode, "Bilinear")
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * 2 * w * h, dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
    got = pre.run_raw_host(host, w, h, (dw, dh), f16=f16, pipeline=pipe)
    torch.cuda.synchronize()
    h2d, d2h = pipe.last_transfer()
    pipe.close()
    assert h2d == n * 2 * w * h and d2h == n * 3 * dw * dh * (2 if f16 else 4)
    it = torch.int16 if f16 else torch.int32
    assert torch.equal(got.view(it), want.cpu().view(it))
