"""8-bit Bayer mosaics (RGGB, BGGR, GRBG, GBRG): the standalone demosaic and Bayer frames in the camera preprocess.

The demosaic is an extension pinned to OpenCV: bit-identical to cv2.cvtColor(raw, COLOR_Bayer??2RGB), through
tests/golden/bayer_cv2.npz and a numpy restatement of the arithmetic (bayer.cuh).  In the preprocess every tap is the
demosaiced pixel at the tap's coordinate, so a Bayer frame must give exactly the bits of its RGB twin (the device
demosaic's output run as SourceFormat.Rgb8), in every geometry, sampler and output dtype; the oracle's preprocess of
that twin is checked as well.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from harness import dev, make_pre, offset_buf, oracle_cfg, raw_bytes
from restate import PATTERNS, PATTERN_CODE, demosaic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def fmt_name(pattern):
    return "Bayer" + pattern.capitalize()


# ═══ CPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def test_cv2_fixture_matches_the_restatement():
    """cv2's COLOR_Bayer??2RGB = the restatement, numpy and torch, for every pattern and size (odd ones included)."""
    fx = np.load(os.path.join(GOLDEN, "bayer_cv2.npz"))
    names = sorted({k.rsplit("_", 1)[0] for k in fx.files})
    assert len(names) == 4 * 6
    for name in names:
        pattern = name.split("_")[0].upper()
        raw, want, (w, h) = fx[f"{name}_raw"], fx[f"{name}_rgb"], (int(v) for v in fx[f"{name}_wh"])
        assert raw.shape == (h, w), name
        np.testing.assert_array_equal(demosaic(raw, pattern), want, name)
        np.testing.assert_array_equal(demosaic(torch.from_numpy(raw), pattern).numpy(), want, name)


def test_source_format_members(kb):
    SF = kb.SourceFormat
    for k, p in enumerate(PATTERNS):
        f = SF[fmt_name(p)]
        assert f.value == f"bayer_{p.lower()}" and f.fmt_code() == 16 + k and f.bpp() == 1 and f.pitch(10) == 10
        assert SF.from_name(f"bayer_{p.lower()}") is f and SF.from_name(f"BAYER_{p}") is f
        assert not f.interleaved() and not f.is_yuv420() and not f.is_yuv422() and f.is_bayer()
        assert f.buffer_len(8, 5) == 40 and f.dims_ok(3, 3) and f.dims_ok(7, 5) and not f.dims_ok(2, 9) and not f.dims_ok(9, 2)
    assert not any(f.is_bayer() for f in SF if not f.value.startswith("bayer_"))
    assert [int(kb.imgproc.BayerPattern[p]) for p in PATTERNS] == [0, 1, 2, 3]


def test_validation_without_a_gpu(kb):
    """Unknown patterns, sides below 3, short buffers, unknown format codes and short pitches fail before any CUDA call."""
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf)
    for bad in (-1, 4):
        assert l.kb200_rgb_from_bayer_u8(None, p, 4096, p, 4096, 4, 4, 1, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown Bayer pattern {bad}"
    for p_name, code in PATTERN_CODE.items():
        for w, h in ((2, 7), (7, 2), (2, 2)):
            assert l.kb200_rgb_from_bayer_u8(None, p, 4096, p, 4096, w, h, 1, code) == _lib.ERR_INVALID_ARGUMENT
            assert _lib.last_error() == f"Bayer {p_name} needs at least 3x3 pixels, got {w}x{h}"
        assert l.kb200_rgb_from_bayer_u8(None, p, 5 * 4 * 2 - 1, p, 4096, 5, 4, 2, code) == _lib.ERR_SLICE_TOO_SMALL
        assert l.kb200_rgb_from_bayer_u8(None, p, 4096, p, 5 * 4 * 3 * 2 - 1, 5, 4, 2, code) == _lib.ERR_SLICE_TOO_SMALL
    with pytest.raises(ValueError):
        kb.imgproc.rgb_from_bayer(None, None, 4)

    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(40)
    for k, p_name in enumerate(PATTERNS):
        d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = 8, 2, 8, 1, 16 + k, 4, 4, 1
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == f"invalid raw source for {fmt_name(p_name)} at 8x2 (at least 3x3 required)"
        d.src_w, d.src_h, d.src_pitch = 2, 6, 2
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == f"invalid raw source for {fmt_name(p_name)} at 2x6 (at least 3x3 required)"
        d.src_w, d.src_h, d.src_pitch = 8, 6, 7   # pitch < width
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error().startswith("invalid pitched surface")
        d.src_pitch = 9
        assert l.kb200_preprocess_src_bytes(C.byref(d)) == 54
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert "got 40 bytes, need 54" in _lib.last_error()
    for code in (10, 15, 20):
        d.fmt = code
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown source format code {code}"


# ═══ GPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def run_decode(kb, dev, pattern, raw_dev, w, h, n, dst_off=0):
    out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint8)
    out.fill_(0xCD)
    kb.imgproc.rgb_from_bayer(raw_dev, kb.Image(out.view(n, h, w, 3)), kb.imgproc.BayerPattern[pattern])
    return out.view(n, h, w, 3), kb._lib.last_kernel()


CASES = [   # w, h, batch, src offset, dst offset
    (64, 48, 1, 0, 0), (128, 31, 3, 0, 0), (512, 16, 4, 0, 0), (2064, 5, 2, 0, 0), (16, 3, 2, 0, 0), (16, 4, 1, 0, 0),  # vec16
    (70, 6, 2, 0, 0), (131, 9, 3, 0, 0), (3, 3, 1, 0, 0), (7, 5, 4, 0, 0), (33, 17, 2, 0, 0),                          # 16 ∤ w
    (64, 48, 2, 1, 0), (64, 48, 2, 0, 3), (64, 48, 1, 8, 8), (130, 14, 1, 5, 0),                                       # unaligned
]
DECODE_CASES = [(p, c) for p in PATTERNS for c in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("pattern,case", DECODE_CASES, ids=[f"{p}-{'x'.join(map(str, c))}" for p, c in DECODE_CASES])
def test_decode_bayer(kb, dev, pattern, case):
    w, h, n, soff, doff = case
    raws = np.random.default_rng(w * 7919 + h * 31 + n + 1000 * PATTERN_CODE[pattern]).integers(0, 256, (n, h, w), dtype=np.uint8)
    src = offset_buf(dev, n * w * h, soff, torch.uint8)
    src.copy_(torch.from_numpy(raws.reshape(-1)))
    got, kern = run_decode(kb, dev, pattern, src.view(n, w * h), w, h, n, doff)
    vec = w % 16 == 0 and soff % 16 == 0 and doff % 16 == 0
    assert kern == f"rgb_from_bayer_{pattern.lower()}_{'vec16' if vec else 'generic'}"
    g = got.cpu().numpy()
    for k in range(n):
        np.testing.assert_array_equal(g[k], demosaic(raws[k], pattern), f"{pattern} {case} frame {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
def test_decode_bayer_1080p_batch(kb, dev, pattern):
    w, h, n = 1920, 1080, 256
    g = torch.Generator(device=dev).manual_seed(0x1080 + PATTERN_CODE[pattern])
    raw = torch.randint(0, 256, (n, h * w), dtype=torch.uint8, device=dev, generator=g)
    got, kern = run_decode(kb, dev, pattern, raw, w, h, n)
    assert kern == f"rgb_from_bayer_{pattern.lower()}_vec16"
    for k0 in range(0, n, 32):
        assert torch.equal(got[k0:k0 + 32], demosaic(raw[k0:k0 + 32].view(-1, h, w), pattern)), f"frames {k0}.."
    del got, raw
    torch.cuda.empty_cache()


# ── camera preprocess ──
GEOMS = [(8, 6, 7, 5), (64, 48, 40, 40), (64, 48, 64, 48), (30, 20, 61, 47), (128, 72, 40, 24),
         (96, 54, 32, 32), (32, 24, 64, 48), (192, 108, 64, 36), (37, 21, 37, 21), (20, 3, 20, 3)]   # test_yuv_layouts' + odd sizes


def expected_preprocess_kernel(pattern, sampling, w, h, dw, dh):
    if sampling != "Lanczos" and (dw, dh) == (w, h) and w % 4 == 0:
        return f"preprocess_bayer_{pattern.lower()}_identity_kernel"
    return "preprocess_generic_kernel"


def device_twin(kb, dev, pattern, raw_dev, w, h):
    """The RGB twin of device frames [n, w*h]: the device demosaic's output, [n, h*w*3]."""
    n = raw_dev.shape[0]
    rgb, _ = run_decode(kb, dev, pattern, raw_dev, w, h, n)
    return rgb.reshape(n, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("mode", ["Letterbox", "Stretch"])
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_bayer(kb, oracle, dev, pattern, mode, sampling, f16):
    """Every geometry: bit-equal to the device run on the RGB twin, with the kernel the dispatch promises; bit-equal to
    the oracle on the twin (Lanczos: within the tolerance of test_preprocess_lanczos_vs_oracle)."""
    pre, twin_pre = make_pre(kb, fmt_name(pattern), mode, sampling), make_pre(kb, "Rgb8", mode, sampling)
    cfg = oracle_cfg(kb, oracle, mode, sampling)
    dt, it = (torch.float16, torch.int16) if f16 else (torch.float32, torch.int32)
    for w, h, dw, dh in GEOMS:
        what = f"{pattern} {mode} {sampling} {'f16' if f16 else 'f32'} {(w, h, dw, dh)}"
        raw = torch.from_numpy(raw_bytes(w * h, PATTERN_CODE[pattern])).to(dev)
        twin = device_twin(kb, dev, pattern, raw.view(1, -1), w, h)[0]
        np.testing.assert_array_equal(twin.cpu().numpy().reshape(h, w, 3), demosaic(raw.cpu().numpy().reshape(h, w), pattern))
        got = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_f16 if f16 else pre.run_raw)(raw, w, h, got)
        assert kb._lib.last_kernel() == expected_preprocess_kernel(pattern, sampling, w, h, dw, dh), what
        want = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (twin_pre.run_raw_f16 if f16 else twin_pre.run_raw)(twin, w, h, want)
        assert torch.equal(got.view(it), want.view(it)), what
        o = oracle.preprocess_frame(twin.cpu().numpy(), cfg, w, h, dw, dh, f16=f16 and sampling != "Lanczos")
        g = got[0].cpu().numpy()
        if sampling == "Lanczos":
            assert np.max(np.abs(g.astype(np.float32) - o)) <= (2e-3 if f16 else 1e-4), what
        elif f16:
            np.testing.assert_array_equal(g.view(np.uint16), o.view(np.uint16), what)
        else:
            np.testing.assert_array_equal(g.view(np.uint32), o.view(np.uint32), what)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["RGGB", "GBRG"])
@pytest.mark.parametrize("n", [256, 300])
def test_preprocess_bayer_identity_1080p(kb, oracle, dev, pattern, n):
    """Config 3a from 1080p Bayer frames at 256 and 300 frames (a second launch with frame0 > 0), through the pointer
    table and the strided entry, against the RGB twin on the device for every frame and the oracle for frames on both
    sides of the 256-frame launch split."""
    w, h = 1920, 1080
    nb = w * h
    g = torch.Generator(device=dev).manual_seed(0x3A + PATTERN_CODE[pattern])
    ring = torch.randint(0, 256, (n, nb + 64), dtype=torch.uint8, device=dev, generator=g)   # padded strided slots
    frames = ring[:, :nb]
    twin = torch.cat([device_twin(kb, dev, pattern, frames[k0:k0 + 64].contiguous(), w, h) for k0 in range(0, n, 64)])
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt_name(pattern)]).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda()
    twin_pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Rgb8).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda()
    kernel = f"preprocess_bayer_{pattern.lower()}_identity_kernel"
    want = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)
    twin_pre.run_raw_batch([twin[k] for k in range(n)], w, h, want)
    del twin
    got = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)
    pre.run_raw_batch([frames[k] for k in range(n)], w, h, got)
    assert kb._lib.last_kernel() == kernel
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    got.fill_(float("nan"))
    pre.run_raw_strided(ring.view(-1), nb + 64, n, w, h, got)
    assert kb._lib.last_kernel() == kernel
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    cfg = oracle_cfg(kb, oracle, "Stretch", "Bilinear")
    for k in sorted({0, 255, n - 1}):
        rgb = demosaic(frames[k].cpu().numpy().reshape(h, w), pattern)
        o = oracle.preprocess_frame(rgb, cfg, w, h, w, h)
        np.testing.assert_array_equal(got[k].cpu().numpy().view(np.uint32), o.view(np.uint32), f"frame {k}")
    del got, want, ring
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("pitch_pad", [12, 5])
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 96, 54), ("Letterbox", 40, 40)])
def test_preprocess_bayer_pitched(kb, dev, pitch_pad, mode, dw, dh):
    """A pitched Bayer frame (row pitch > width) gives the bits of its tight copy, on the identity kernel (pitch % 4 == 0)
    and on the generic one."""
    from kornia_rs_b200 import _lib

    w, h = 96, 54
    pitch = w + pitch_pad
    tight = torch.from_numpy(raw_bytes(w * h, 3)).to(dev)
    pitched = torch.full((h, pitch), 0xEE, dtype=torch.uint8, device=dev)
    pitched[:, :w] = tight.view(h, w)
    pre = make_pre(kb, "BayerGrbg", mode, "Bilinear")
    want = torch.full((1, 3, dh, dw), float("nan"), device=dev)
    pre.run_raw(tight, w, h, want)
    tight_kernel = kb._lib.last_kernel()
    got = torch.full((1, 3, dh, dw), float("nan"), device=dev)
    desc = pre._desc(w, h, pitch, 1, kb.SourceFormat.BayerGrbg.fmt_code(), dw, dh)
    assert _lib.lib().kb200_preprocess_src_bytes(C.byref(desc)) == pitch * h
    pre._launch(desc, [pitched.view(-1)], got, False)
    identity = mode == "Stretch" and pitch % 4 == 0
    assert kb._lib.last_kernel() == ("preprocess_bayer_grbg_identity_kernel" if identity else "preprocess_generic_kernel")
    assert tight_kernel == ("preprocess_bayer_grbg_identity_kernel" if mode == "Stretch" else "preprocess_generic_kernel")
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 192, 108), ("Letterbox", 64, 64)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_pipeline_bayer(kb, dev, mode, dw, dh, f16):
    """run_raw_host carries Bayer frames (w*h bytes each) unchanged: host frames in / host tensor out equal the device
    path, and the transfers are exactly the frames' and the outputs' bytes."""
    w, h, n = 192, 108, 7
    nbytes = w * h
    host = torch.from_numpy(np.stack([raw_bytes(nbytes, k) for k in range(n)])).pin_memory()
    pre = make_pre(kb, "BayerBggr", mode, "Bilinear")
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * nbytes, dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
    got = pre.run_raw_host(host, w, h, (dw, dh), f16=f16, pipeline=pipe)
    torch.cuda.synchronize()
    h2d, d2h = pipe.last_transfer()
    pipe.close()
    assert h2d == n * nbytes and d2h == n * 3 * dw * dh * (2 if f16 else 4)
    it = torch.int16 if f16 else torch.int32
    assert torch.equal(got.view(it), want.cpu().view(it))
