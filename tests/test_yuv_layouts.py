"""The YUV layouts beyond NV12 and YUYV: NV21, I420, YV12 (4:2:0) and UYVY, YVYU (4:2:2).

Every layout decodes with the Q20 BT.601-limited arithmetic of NV12 / YUYV; only the chroma addressing differs.  So a
frame in a new layout must give exactly the bits its byte-repacked NV12 (4:2:0) or YUYV (4:2:2) twin gives, in the
standalone decode and in every preprocess geometry, sampler and output dtype.  The tests check that property on the
device, check both sides against the oracle (through the twin), and anchor the layouts themselves to cv2 through
tests/golden/yuv_layouts_cv2.npz and a numpy restatement of the decode that reads each layout directly.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from harness import dev, make_pre, offset_buf
from restate import L420, L422, decode_direct, expected_decode_kernel, layout_bytes, nv12_to_yuv420, to_twin, yuv420_to_nv12, yuv422_swap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

LAYOUT_CODE = {"Nv12": 0, "Nv21": 1, "I420": 2, "Yv12": 3, "Yuyv": 0, "Uyvy": 1, "Yvyu": 2}   # kb200_yuv420/422_layout


def oracle_decode(oracle, raw, w, h, layout):
    twin = to_twin(raw, w, h, layout)
    return oracle.rgb_from_nv12(twin, w, h) if layout in L420 else oracle.rgb_from_yuyv(twin, w, h)


# ═══ CPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def test_cv2_fixture_matches_the_direct_decode_and_the_oracle_twin(oracle):
    """cv2's COLOR_YUV2RGB_<layout> = the Q20 decode read in that layout = the oracle's NV12 / YUYV decode of the
    repacked twin, bit for bit."""
    fx = np.load(os.path.join(GOLDEN, "yuv_layouts_cv2.npz"))
    names = sorted({k.rsplit("_", 1)[0] for k in fx.files})
    assert len(names) == 3 * 5 + 2 * 4
    for name in names:
        layout = {"nv21": "Nv21", "i420": "I420", "yv12": "Yv12", "uyvy": "Uyvy", "yvyu": "Yvyu"}[name.split("_")[0]]
        raw, want, (w, h) = fx[f"{name}_raw"], fx[f"{name}_rgb"], (int(v) for v in fx[f"{name}_wh"])
        assert raw.size == layout_bytes(layout, w, h), name
        np.testing.assert_array_equal(decode_direct(raw, w, h, layout), want, name)
        np.testing.assert_array_equal(oracle_decode(oracle, raw, w, h, layout).reshape(h, w, 3), want, name)


def test_existing_cv2_fixtures_match_the_direct_decode():
    """The restatement above also reproduces the NV12 / YUYV fixtures the oracle is pinned to."""
    for path, layout in (("nv12_cv2.npz", "Nv12"), ("yuyv_cv2.npz", "Yuyv")):
        fx = np.load(os.path.join(GOLDEN, path))
        for name in sorted({k.rsplit("_", 1)[0] for k in fx.files}):
            w, h = (int(v) for v in fx[f"{name}_wh"])
            np.testing.assert_array_equal(decode_direct(fx[f"{name}_raw"], w, h, layout), fx[f"{name}_rgb"], f"{path} {name}")


@pytest.mark.parametrize("layout", L420)
def test_yuv420_repack_round_trip(layout):
    for w, h in ((4, 2), (70, 4), (130, 2), (64, 48)):
        nv12 = np.random.default_rng(w * h).integers(0, 256, (2, w * h * 3 // 2), dtype=np.uint8)
        there = nv12_to_yuv420(nv12, w, h, layout)
        assert not np.array_equal(there, nv12)
        np.testing.assert_array_equal(yuv420_to_nv12(there, w, h, layout), nv12)


def test_source_format_members(kb):
    SF = kb.SourceFormat
    new = {"Nv21": (5, 1), "I420": (6, 1), "Yv12": (7, 1), "Uyvy": (8, 2), "Yvyu": (9, 2)}
    for name, (code, bpp) in new.items():
        f = SF[name]
        assert f.fmt_code() == code and f.bpp() == bpp and f.pitch(10) == 10 * bpp
        assert SF.from_name(name.upper()) is f and SF.from_name(name.lower()) is f
        assert not f.interleaved()
        if bpp == 1:   # 4:2:0
            assert f.buffer_len(8, 6) == 72 and f.dims_ok(8, 6) and not f.dims_ok(8, 5) and not f.dims_ok(7, 6)
        else:
            assert f.buffer_len(8, 6) == 96 and f.dims_ok(8, 5) and not f.dims_ok(7, 5)
    assert [f.fmt_code() for f in (SF.Rgb8, SF.Rgba8, SF.Bgr8, SF.Bgra8, SF.Gray8, SF.Nv12, SF.Yuyv)] == [0, 0, 1, 1, 2, 3, 4]


def test_validation_without_a_gpu(kb):
    """Unknown layouts, odd dimensions, short buffers and untight planar frames fail before any CUDA call."""
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf)
    for bad in (-1, 4, 99):
        assert l.kb200_rgb_from_yuv420_u8(None, p, 4096, p, 4096, 4, 4, 1, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown 4:2:0 layout {bad}"
    for bad in (-1, 3):
        assert l.kb200_rgb_from_yuv422_u8(None, p, 4096, p, 4096, 4, 4, 1, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown 4:2:2 layout {bad}"
    for name, code in (("NV12", 0), ("NV21", 1), ("I420", 2), ("YV12", 3)):
        assert l.kb200_rgb_from_yuv420_u8(None, p, 4096, p, 4096, 6, 5, 1, code) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"{name} needs even dimensions, got 6x5"
        assert l.kb200_rgb_from_yuv420_u8(None, p, 35, p, 4096, 6, 4, 1, code) == _lib.ERR_SLICE_TOO_SMALL
    for name, code in (("YUYV", 0), ("UYVY", 1), ("YVYU", 2)):
        assert l.kb200_rgb_from_yuv422_u8(None, p, 4096, p, 4096, 5, 2, 1, code) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"{name} needs an even width, got 5"
        assert l.kb200_rgb_from_yuv422_u8(None, p, 4096, p, 17, 6, 1, 1, code) == _lib.ERR_SLICE_TOO_SMALL
    # the NV12 / YUYV entry points are the layout-0 cases, with the same messages
    assert l.kb200_rgb_from_nv12_u8(None, p, 4096, p, 4096, 5, 4, 1) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "NV12 needs even dimensions, got 5x4"
    assert l.kb200_rgb_from_yuyv_u8(None, p, 4096, p, 4096, 5, 4, 1) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "YUYV needs an even width, got 5"

    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(60)
    for name, code in (("Nv21", 5), ("I420", 6), ("Yv12", 7)):
        d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = 8, 5, 8, 1, code, 4, 4, 1
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == f"invalid raw source for {name} at 8x5 (even dimensions required)"
        d.src_h = 6
        assert l.kb200_preprocess_src_bytes(C.byref(d)) == 72
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert "got 60 bytes, need 72" in _lib.last_error()
        d.src_pitch = 12
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == f"{name.upper()} frames must be tightly packed (pitch == width)"
    for name, code in (("Uyvy", 8), ("Yvyu", 9)):
        d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt = 7, 5, 14, 2, code
        assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_SOURCE
        assert _lib.last_error() == f"invalid raw source for {name} at 7x5 (even width required)"
        d.src_w, d.src_pitch = 8, 16
        assert l.kb200_preprocess_src_bytes(C.byref(d)) == 80
    d.fmt = 10
    assert l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "unknown source format code 10"


# ═══ GPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def run_decode(kb, dev, layout, raw_dev, w, h, n, dst_off=0):
    out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint8)
    out.fill_(0xCD)
    img = kb.Image(out.view(n, h, w, 3))
    getattr(kb.imgproc, f"rgb_from_{layout.lower()}")(raw_dev, img)
    return out.view(n, h, w, 3), kb._lib.last_kernel()


CASES_420 = [   # w, h, batch, src offset, dst offset
    (64, 48, 1, 0, 0), (128, 32, 3, 0, 0), (512, 16, 4, 0, 0), (2064, 6, 2, 0, 0),    # 16 | w: vec16
    (70, 6, 2, 0, 0), (130, 2, 3, 0, 0), (2, 2, 1, 0, 0), (6, 4, 4, 0, 0),            # 16 ∤ w: generic
    (64, 48, 2, 1, 0), (64, 48, 2, 0, 3), (64, 48, 1, 8, 8), (130, 14, 1, 5, 0),      # unaligned src / dst: generic
]
CASES_422 = [
    (64, 48, 1, 0, 0), (128, 31, 3, 0, 0), (512, 1, 4, 0, 0), (2064, 5, 2, 0, 0),     # px % 16 == 0: vec16
    (70, 5, 2, 0, 0), (130, 1, 3, 0, 0), (2, 1, 1, 0, 0), (6, 3, 4, 0, 0),            # ragged tail: generic last
    (64, 48, 2, 1, 0), (64, 48, 2, 0, 3), (64, 48, 1, 8, 8), (130, 7, 1, 5, 0),       # unaligned src / dst: generic
]
DECODE_CASES = [(l, c) for l in L420 for c in CASES_420] + [(l, c) for l in L422 for c in CASES_422]


@pytest.mark.gpu
@pytest.mark.parametrize("layout,case", DECODE_CASES, ids=[f"{l}-{'x'.join(map(str, c))}" for l, c in DECODE_CASES])
def test_decode_layout(kb, oracle, dev, layout, case):
    """Every layout on both paths: equal to the numpy restatement, to the oracle's decode of the twin and to the device
    decode of the twin."""
    w, h, n, soff, doff = case
    nb = layout_bytes(layout, w, h)
    raws = np.random.default_rng(w * 7919 + h * 31 + n + 1000 * LAYOUT_CODE[layout]).integers(0, 256, (n, nb), dtype=np.uint8)
    src = offset_buf(dev, n * nb, soff, torch.uint8)
    src.copy_(torch.from_numpy(raws.reshape(-1)))
    got, kern = run_decode(kb, dev, layout, src.view(n, nb), w, h, n, doff)
    assert kern == expected_decode_kernel(layout, w, h, n, soff, doff)
    twin = offset_buf(dev, n * nb, soff, torch.uint8)
    twin.copy_(torch.from_numpy(to_twin(raws, w, h, layout).reshape(-1)))
    twin_out, twin_kern = run_decode(kb, dev, "Nv12" if layout in L420 else "Yuyv", twin.view(n, nb), w, h, n, doff)
    assert twin_kern.endswith(kern.rsplit("_", 1)[1])   # the twin took the same path
    assert torch.equal(got, twin_out)
    g = got.cpu().numpy()
    for k in range(n):
        np.testing.assert_array_equal(g[k], decode_direct(raws[k], w, h, layout), f"{layout} {case} frame {k}")
        np.testing.assert_array_equal(g[k], oracle_decode(oracle, raws[k], w, h, layout).reshape(h, w, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("layout", L420 + L422)
def test_decode_layout_1080p_batch(kb, oracle, dev, layout):
    w, h, n = 1920, 1080, 8
    nb = layout_bytes(layout, w, h)
    g = torch.Generator(device=dev).manual_seed(0x1080)
    raw = torch.randint(0, 256, (n, nb), dtype=torch.uint8, device=dev, generator=g)
    got, kern = run_decode(kb, dev, layout, raw, w, h, n)
    assert kern == f"rgb_from_{layout.lower()}_vec16"
    twin_out, _ = run_decode(kb, dev, "Nv12" if layout in L420 else "Yuyv", to_twin(raw, w, h, layout).contiguous(), w, h, n)
    assert torch.equal(got, twin_out)
    for k in (0, n - 1):
        np.testing.assert_array_equal(got[k].cpu().numpy(), decode_direct(raw[k].cpu().numpy(), w, h, layout))


# ── camera preprocess ──
GEOMS = [(8, 6, 7, 5), (64, 48, 40, 40), (64, 48, 64, 48), (30, 20, 61, 47), (128, 72, 40, 24),
         (96, 54, 32, 32), (32, 24, 64, 48), (192, 108, 64, 36)]   # the geometries of test_preprocess_formats


def raw_bytes(n, k=0):
    return ((np.arange(n, dtype=np.int64) * 7 + 13) % 251 + 31 * k).astype(np.uint8)


def expected_preprocess_kernel(layout, sampling, w, h, dw, dh):
    if layout in L422 or sampling == "Lanczos":
        return "preprocess_generic_kernel"
    if (dw, dh) == (w, h) and w % 4 == 0:
        return f"preprocess_{layout.lower()}_identity_kernel"
    return f"preprocess_{layout.lower()}_kernel" if dw % 4 == 0 else "preprocess_generic_kernel"


def oracle_cfg(kb, oracle, twin_fmt, mode, sampling):
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    return oracle.PreprocessCfg(mode=oracle.LETTERBOX if mode == "Letterbox" else oracle.STRETCH,
                                fmt=oracle.FMT_NV12 if twin_fmt == "Nv12" else oracle.FMT_YUYV, mean=kb.IMAGENET_MEAN,
                                inv_std=inv, pad_value=114.0,
                                sampling={"Bilinear": oracle.BILINEAR, "Nearest": oracle.NEAREST, "Lanczos": oracle.LANCZOS}[sampling])


@pytest.mark.gpu
@pytest.mark.parametrize("layout", L420 + L422)
@pytest.mark.parametrize("mode", ["Letterbox", "Stretch"])
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_layout(kb, oracle, dev, layout, mode, sampling, f16):
    """Every geometry of test_preprocess_formats: bit-equal to the run on the NV12 / YUYV twin, with the kernel the
    dispatch promises; bit-equal to the oracle (Lanczos: within the tolerance of test_preprocess_lanczos_vs_oracle)."""
    twin_fmt = "Nv12" if layout in L420 else "Yuyv"
    pre, twin_pre = make_pre(kb, layout, mode, sampling), make_pre(kb, twin_fmt, mode, sampling)
    cfg = oracle_cfg(kb, oracle, twin_fmt, mode, sampling)
    dt = torch.float16 if f16 else torch.float32
    for w, h, dw, dh in GEOMS:
        what = f"{layout} {mode} {sampling} {'f16' if f16 else 'f32'} {(w, h, dw, dh)}"
        raw = nv12_to_yuv420(raw_bytes(w * h * 3 // 2), w, h, layout) if layout in L420 else yuv422_swap(raw_bytes(w * h * 2), layout)
        twin = to_twin(raw, w, h, layout)
        got = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_f16 if f16 else pre.run_raw)(torch.from_numpy(raw).to(dev), w, h, got)
        assert kb._lib.last_kernel() == expected_preprocess_kernel(layout, sampling, w, h, dw, dh), what
        want = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (twin_pre.run_raw_f16 if f16 else twin_pre.run_raw)(torch.from_numpy(np.ascontiguousarray(twin)).to(dev), w, h, want)
        assert torch.equal(got.view(torch.int16 if f16 else torch.int32), want.view(torch.int16 if f16 else torch.int32)), what
        o = oracle.preprocess_frame(twin, cfg, w, h, dw, dh, f16=f16 and sampling != "Lanczos")
        g = got[0].cpu().numpy()
        if sampling == "Lanczos":
            assert np.max(np.abs(g.astype(np.float32) - o)) <= (2e-3 if f16 else 1e-4), what
        elif f16:
            np.testing.assert_array_equal(g.view(np.uint16), o.view(np.uint16), what)
        else:
            np.testing.assert_array_equal(g.view(np.uint32), o.view(np.uint32), what)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["I420", "Nv21"])
@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 1920, 1080), ("Letterbox", 640, 640)], ids=["3a", "3b"])
@pytest.mark.parametrize("n", [256, 300])
def test_preprocess_config3_layout(kb, oracle, dev, layout, mode, dw, dh, n):
    """Configs 3a / 3b on 1080p frames, through the pointer table and the strided entry, against the NV12 twin on the
    device for every frame and against the oracle for frames on both sides of the 256-frame launch split."""
    w, h = 1920, 1080
    nb = w * h * 3 // 2
    g = torch.Generator(device=dev).manual_seed(0x3A3B)
    ring = torch.randint(0, 256, (n, nb + 64), dtype=torch.uint8, device=dev, generator=g)   # padded strided slots
    frames = ring[:, :nb]
    twin = yuv420_to_nv12(frames, w, h, layout).contiguous()
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat[layout]).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda()
    twin_pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda()
    kernel = f"preprocess_{layout.lower()}_identity_kernel" if mode == "Stretch" else f"preprocess_{layout.lower()}_kernel"
    want = torch.full((n, 3, dh, dw), float("nan"), dtype=torch.float32, device=dev)
    twin_pre.run_raw_batch([twin[k] for k in range(n)], w, h, want)
    got = torch.full((n, 3, dh, dw), float("nan"), dtype=torch.float32, device=dev)
    pre.run_raw_batch([frames[k] for k in range(n)], w, h, got)
    assert kb._lib.last_kernel() == kernel
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    got.fill_(float("nan"))
    pre.run_raw_strided(ring.view(-1), nb + 64, n, w, h, got)
    assert kb._lib.last_kernel() == kernel
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    cfg = oracle_cfg(kb, oracle, "Nv12", mode, "Bilinear")
    for k in sorted({0, 255, n - 1}):
        o = oracle.preprocess_frame(twin[k].cpu().numpy(), cfg, w, h, dw, dh)
        np.testing.assert_array_equal(got[k].cpu().numpy().view(np.uint32), o.view(np.uint32), f"frame {k}")
    del got, want, ring, twin
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("layout,mode,dw,dh", [("I420", "Letterbox", 64, 64), ("Uyvy", "Stretch", 100, 60)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_pipeline_layout(kb, dev, layout, mode, dw, dh, f16):
    """run_raw_host sizes frames from the format alone: host frames in / host tensor out equal the device path, and the
    transfers are exactly the frames' and the outputs' bytes."""
    w, h, n = 192, 108, 7
    nbytes = layout_bytes(layout, w, h)
    host = torch.from_numpy(np.stack([raw_bytes(nbytes, k) for k in range(n)])).pin_memory()
    pre = make_pre(kb, layout, mode, "Bilinear")
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * ((nbytes + 15) // 16 * 16), dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
    got = pre.run_raw_host(host, w, h, (dw, dh), f16=f16, pipeline=pipe)
    torch.cuda.synchronize()
    h2d, d2h = pipe.last_transfer()
    pipe.close()
    assert h2d == n * nbytes and d2h == n * 3 * dw * dh * (2 if f16 else 4)
    assert torch.equal(got.view(torch.int16 if f16 else torch.int32), want.cpu().view(torch.int16 if f16 else torch.int32))
