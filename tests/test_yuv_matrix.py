"""YUV colour matrices: BT.601 / BT.709, limited / full range, for every YUV layout, in the decoders and the preprocess.

Every matrix is the Q20 arithmetic of the BT.601-limited decode with another coefficient set.  The CPU tests pin that
set: the table below is round(c * 2^20) of the exact coefficients (matrix 0 keeps the reference's literal constants),
the native sources carry the same table, every matrix is within one level of the float64 formula over all 2^24 (Y, U, V)
triples, and BT.601 full range is within one level of cv2's COLOR_YCrCb2RGB.  The GPU tests check the device against
the numpy restatement (decoders) and against the preprocess of each frame's RGB8 twin, the restatement's decode of it:
a YUV tap and an RGB8 tap hand the resampler the same integers, so the two must agree bit for bit.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from harness import dev, make_pre, offset_buf, oracle_cfg, raw_bytes
from restate import KR_KB, L420, L422, MATRICES, TABLE, YUV420, decode_yuv8, expected_decode_kernel, layout_bytes, nv12_to_yuv420, q20, yuv422_swap


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

FORMATS = ("Nv12",) + L420 + ("Yuyv",) + L422
LAYOUT_CODE = {"Nv12": 0, "Nv21": 1, "I420": 2, "Yv12": 3, "Yuyv": 0, "Uyvy": 1, "Yvyu": 2}
FMT_CODE = {"Nv12": 3, "Yuyv": 4, "Nv21": 5, "I420": 6, "Yv12": 7, "Uyvy": 8, "Yvyu": 9}


def float_coeffs(m):
    """(y_off, cy, cvr, cub, cug, cvg) as exact float64 coefficients, from (Kr, Kb) and the range."""
    kr, kb_ = KR_KB[m[:5]]
    kg = 1.0 - kr - kb_
    full = m.endswith("Full")
    sy, sc = (1.0, 1.0) if full else (255.0 / 219.0, 255.0 / 224.0)
    return (0 if full else 16, sy, 2 * (1 - kr) * sc, 2 * (1 - kb_) * sc, -2 * kb_ * (1 - kb_) / kg * sc, -2 * kr * (1 - kr) / kg * sc)


# ═══ CPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def test_table_is_the_derived_coefficients():
    """Matrices 1-3: round(c * 2^20) of the exact coefficients.  Matrix 0: the reference's literal constants, which the
    same derivation reproduces only to within a few units."""
    for m in MATRICES[1:]:
        yo, *cs = float_coeffs(m)
        assert TABLE[m] == (yo, *(int(round(c * 2 ** 20)) for c in cs)), m
    assert TABLE["Bt601Limited"] == (16, 1220542, 1673527, 2116026, -409993, -852492)
    for m in MATRICES:   # i32 headroom: every term below 5.8e8, so yy plus the largest chroma sum stays below 2^31
        yo, cy, cvr, cub, cug, cvg = TABLE[m]
        terms = (255 * cy, 128 * abs(cvr), 128 * abs(cub), 128 * (abs(cug) + abs(cvg)) + (1 << 19))
        assert max(terms) < 5.8e8 and terms[0] + max(terms[1:]) + (1 << 19) < 2 ** 31


def test_native_sources_carry_the_table():
    """The kernels' table (kb200_common.cuh) and the header's documentation list exactly TABLE, in kb200_yuv_matrix order."""
    src = open(os.path.join(ROOT, "kornia-rs_b200", "csrc", "kb200_common.cuh")).read()
    block = src.split("YUV_COEFFS[4] = {", 1)[1].split("};", 1)[0]
    rows = [tuple(int(x) for x in r.split(",")) for r in re.findall(r"\{([-\d, ]+)\}", block)]
    assert rows == [TABLE[m] for m in MATRICES]
    hdr = open(os.path.join(ROOT, "include", "kornia_b200.h")).read()
    for m, name in zip(MATRICES, ("BT601_LIMITED", "BT601_FULL", "BT709_LIMITED", "BT709_FULL")):
        assert re.search(rf"\* +{name} +" + r" +".join(str(c) for c in TABLE[m][1:]), hdr), name
        assert f"KB200_YUV_{name} = {MATRICES.index(m)}" in hdr


def test_matrix0_reproduces_the_cv2_fixtures():
    for path, layout in (("nv12_cv2.npz", "Nv12"), ("yuyv_cv2.npz", "Yuyv")):
        fx = np.load(os.path.join(GOLDEN, path))
        for name in sorted({k.rsplit("_", 1)[0] for k in fx.files}):
            w, h = (int(v) for v in fx[f"{name}_wh"])
            np.testing.assert_array_equal(decode_yuv8(fx[f"{name}_raw"], w, h, layout, "Bt601Limited"), fx[f"{name}_rgb"], f"{path} {name}")


def all_triples(y_lo, y_hi):
    y, u, v = np.meshgrid(np.arange(y_lo, y_hi), np.arange(256), np.arange(256), indexing="ij")
    return y.astype(np.uint8).ravel(), u.astype(np.uint8).ravel(), v.astype(np.uint8).ravel()


@pytest.mark.parametrize("m", MATRICES)
def test_every_triple_within_one_level_of_float64(m):
    yo, cy, cvr, cub, cug, cvg = float_coeffs(m)
    worst = 0
    for y0 in range(0, 256, 32):
        y, u, v = all_triples(y0, y0 + 32)
        yy = np.maximum(y.astype(np.float64) - yo, 0) * cy
        uf, vf = u.astype(np.float64) - 128, v.astype(np.float64) - 128
        ref = np.stack([yy + cvr * vf, yy + cug * uf + cvg * vf, yy + cub * uf], -1)
        ref = np.clip(np.floor(ref + 0.5), 0, 255)
        worst = max(worst, int(np.abs(q20(y, u, v, m).astype(np.float64) - ref).max()))
    assert worst <= 1, (m, worst)


def test_bt601_full_within_one_level_of_cv2():
    cv2 = pytest.importorskip("cv2")
    differ = 0
    for y0 in range(0, 256, 64):
        y, u, v = all_triples(y0, y0 + 64)
        ycrcb = np.stack([y, v, u], -1).reshape(-1, 256, 3)
        ref = cv2.cvtColor(ycrcb, cv2.COLOR_YCrCb2RGB).reshape(-1, 3).astype(np.int64)
        d = np.abs(q20(y, u, v, "Bt601Full").astype(np.int64) - ref)
        assert d.max() <= 1
        differ += int(np.count_nonzero(d.max(-1)))
    assert differ < 2 ** 24 // 8   # most triples agree exactly


def test_abi_validation_without_a_gpu(kb):
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf)
    for bad in (-1, 4, 99):
        assert l.kb200_rgb_from_yuv420_u8_matrix(None, p, 4096, p, 4096, 4, 4, 1, 0, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown YUV matrix {bad}"
        assert l.kb200_rgb_from_yuv422_u8_matrix(None, p, 4096, p, 4096, 4, 4, 1, 0, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown YUV matrix {bad}"
    # the layout and geometry checks are those of the matrix-0 entry points, with their messages
    assert l.kb200_rgb_from_yuv420_u8_matrix(None, p, 4096, p, 4096, 4, 4, 1, 4, 2) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "unknown 4:2:0 layout 4"
    assert l.kb200_rgb_from_yuv420_u8_matrix(None, p, 4096, p, 4096, 6, 5, 1, 2, 3) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "I420 needs even dimensions, got 6x5"
    assert l.kb200_rgb_from_yuv422_u8_matrix(None, p, 4096, p, 17, 6, 1, 1, 1, 1) == _lib.ERR_SLICE_TOO_SMALL

    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(60)

    def status(fmt, w=8, h=6, pitch=8, bpp=1):
        d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = w, h, pitch, bpp, fmt, 4, 4, 1
        return l.kb200_preprocess_f32(None, C.byref(d), ptrs, lens, 1, p, 64)

    M = lambda m: m << 8   # KB200_FMT_YUV_MATRIX
    for code, name in ((0, "RGB"), (2, "GRAY"), (16, "BAYER_RGGB"), (38, "BAYER_GRBG12"), (69, "BAYER_BGGR12P")):
        for m in (1, 2, 3):
            assert status(code | M(m), pitch=24, bpp=3) == _lib.ERR_INVALID_ARGUMENT, (name, m)
            assert _lib.last_error() == (f"source format code {code | M(m)}: a YUV matrix ({m}) applies only to the YUV formats, "
                                         f"not format code {code}")
    for stray in (1 << 10, 1 << 16, 1 << 30, M(4), M(7)):
        for code in (3, 6, 9, 0):
            assert status(code | stray) == _lib.ERR_INVALID_ARGUMENT
            assert _lib.last_error() == f"source format code {code | stray} has bits set above bit 9 (bits 8-9 are the YUV matrix, 0-3)"
    # codes that name no format keep their message, with the full value
    for bad in (-1, 10, 79, 10 | M(1), 255 | M(3), -(1 << 31) | 3):
        assert status(bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown source format code {bad}"
    # a valid YUV code with a matrix validates like the plain code: the frame size check sees the 4:2:0 chroma
    for fmt in FORMATS:
        for m in range(4):
            pitch = 16 if fmt in ("Yuyv",) + L422 else 8
            d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt = 8, 6, pitch, pitch // 8, FMT_CODE[fmt] | M(m)
            want = 72 if fmt in YUV420 else 96
            assert l.kb200_preprocess_src_bytes(C.byref(d)) == want, (fmt, m)
            assert status(FMT_CODE[fmt] | M(m), pitch=pitch, bpp=pitch // 8) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source at 8x6 (got 60 bytes, need {want})"
        d.fmt = FMT_CODE[fmt] | M(2)
        d.src_h = 5
        if fmt in YUV420:
            assert status(d.fmt, h=5) == _lib.ERR_INVALID_SOURCE
            assert _lib.last_error() == f"invalid raw source for {fmt} at 8x5 (even dimensions required)"


def test_builder_rejects_a_matrix_on_other_formats(kb):
    for fmt in ("Rgb8", "BayerRggb", "Gray8", "BayerGbrg12p"):
        b = kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).yuv_matrix(kb.YuvMatrix.Bt709Limited)
        with pytest.raises(kb.PreprocessError) as e:
            b.build_cuda()
        assert e.value.kind == "YuvMatrixNeedsYuvSource" and f"SourceFormat.{fmt}" in str(e.value), str(e.value)
        b.yuv_matrix(kb.YuvMatrix.Bt601Limited).build_cuda()   # the default matrix is every format's
    for fmt in FORMATS:
        pre = kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).yuv_matrix(kb.YuvMatrix.Bt709Full).build_cuda()
        assert pre.yuv_matrix() is kb.YuvMatrix.Bt709Full
        assert pre._desc(8, 6, 8, 1, kb.SourceFormat[fmt].fmt_code(), 4, 4).fmt == FMT_CODE[fmt] | (3 << 8)
    assert [int(m) for m in kb.YuvMatrix] == [0, 1, 2, 3] and [m.name for m in kb.YuvMatrix] == list(MATRICES)
    with pytest.raises(ValueError):
        kb.Preprocessor.builder().yuv_matrix(4)


# ═══ GPU ═══════════════════════════════════════════════════════════════════════════════════════════════════════
def run_decode(kb, dev, layout, src, w, h, n, m, dst_off=0):
    out = offset_buf(dev, n * h * w * 3, dst_off, torch.uint8)
    out.fill_(0xCD)
    getattr(kb.imgproc, f"rgb_from_{layout.lower()}")(src, kb.Image(out.view(n, h, w, 3)), matrix=kb.YuvMatrix[m])
    return out.view(n, h, w, 3), kb._lib.last_kernel()


DECODE_CASES = {   # w, h, batch, src offset, dst offset: the vec16 kernel, then the generic one by width and by alignment
    "420": [(64, 48, 3, 0, 0), (2064, 6, 2, 0, 0), (18, 6, 2, 0, 0), (70, 4, 3, 0, 0), (64, 48, 2, 1, 0), (64, 16, 2, 0, 3)],
    "422": [(64, 48, 3, 0, 0), (2064, 5, 2, 0, 0), (18, 5, 2, 0, 0), (70, 5, 3, 0, 0), (64, 48, 2, 1, 0), (64, 16, 2, 0, 3)],
}


@pytest.mark.gpu
@pytest.mark.parametrize("m", MATRICES)
@pytest.mark.parametrize("layout", FORMATS)
def test_decode_matrix(kb, dev, layout, m):
    """Every layout x matrix, batched, on both kernels: equal to the restatement.  Matrix 0 through the new entry points
    equals the old ones; every other matrix gives another picture."""
    from kornia_rs_b200 import _lib

    for w, h, n, soff, doff in DECODE_CASES["420" if layout in YUV420 else "422"]:
        nb = layout_bytes(layout, w, h)
        raws = np.random.default_rng(w * 131 + h + 7 * n + 1000 * MATRICES.index(m)).integers(0, 256, (n, nb), dtype=np.uint8)
        src = offset_buf(dev, n * nb, soff, torch.uint8)
        src.copy_(torch.from_numpy(raws.reshape(-1)))
        got, kern = run_decode(kb, dev, layout, src.view(n, nb), w, h, n, m, doff)
        what = f"{layout} {m} {(w, h, n, soff, doff)}"
        assert kern == expected_decode_kernel(layout, w, h, n, soff, doff), what
        g = got.cpu().numpy()
        for k in range(n):
            np.testing.assert_array_equal(g[k], decode_yuv8(raws[k], w, h, layout, m), f"{what} frame {k}")
        if m == "Bt601Limited":
            old = offset_buf(dev, n * h * w * 3, doff, torch.uint8)
            fn = "kb200_rgb_from_yuv420_u8" if layout in YUV420 else "kb200_rgb_from_yuv422_u8"
            st = getattr(_lib.lib(), fn)(torch.cuda.current_stream(dev).cuda_stream, src.data_ptr(), src.numel(), old.data_ptr(), old.numel(),
                                         w, h, n, LAYOUT_CODE[layout])
            assert st == _lib.OK and _lib.last_kernel() == kern
            assert torch.equal(old.view(n, h, w, 3), got), what
        else:
            assert not np.array_equal(g[0], decode_yuv8(raws[0], w, h, layout, "Bt601Limited")), what


def expected_preprocess_kernel(fmt, sampling, w, h, dw, dh):
    if fmt not in YUV420 or sampling == "Lanczos":
        return "preprocess_generic_kernel"
    if (dw, dh) == (w, h) and w % 4 == 0:
        return f"preprocess_{fmt.lower()}_identity_kernel"
    return f"preprocess_{fmt.lower()}_kernel" if dw % 4 == 0 else "preprocess_generic_kernel"


# identity (the 3a shape), a 3:1 letterbox (the 3b shape), a non-integer stretch, and a 4:2:0 geometry the fast kernel
# cannot store (dst_w % 4 != 0: the generic kernel)
PRE_GEOMS = [("Stretch", 64, 48, 64, 48), ("Letterbox", 192, 108, 64, 64), ("Stretch", 30, 20, 61, 47), ("Letterbox", 64, 48, 42, 40)]


def raw_frame(fmt, w, h, k):
    if fmt in YUV420:
        return nv12_to_yuv420(raw_bytes(w * h * 3 // 2, k), w, h, fmt)
    return yuv422_swap(raw_bytes(w * h * 2, k), fmt) if fmt != "Yuyv" else raw_bytes(w * h * 2, k)


@pytest.mark.gpu
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
@pytest.mark.parametrize("sampling", ["Nearest", "Bilinear", "Lanczos"])
@pytest.mark.parametrize("m", MATRICES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_preprocess_matrix(kb, oracle, dev, fmt, m, sampling, f16):
    """Each geometry, two frames through the pointer table and the strided entry: bit-equal to the device run on the RGB8
    twins, and to the oracle on the twins (Lanczos: within the tolerance of test_preprocess_lanczos_vs_oracle)."""
    dt, it = (torch.float16, torch.int16) if f16 else (torch.float32, torch.int32)
    n = 2
    for mode, w, h, dw, dh in PRE_GEOMS:
        what = f"{fmt} {m} {sampling} {mode} {(w, h, dw, dh)} {'f16' if f16 else 'f32'}"
        pre, twin_pre = make_pre(kb, fmt, mode, sampling, m), make_pre(kb, "Rgb8", mode, sampling)
        raws = [raw_frame(fmt, w, h, k) for k in range(n)]
        twins = [decode_yuv8(r, w, h, fmt, m) for r in raws]
        got = torch.full((n, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([torch.from_numpy(r).to(dev) for r in raws], w, h, got)
        assert kb._lib.last_kernel() == expected_preprocess_kernel(fmt, sampling, w, h, dw, dh), what
        want = torch.full((n, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (twin_pre.run_raw_batch_f16 if f16 else twin_pre.run_raw_batch)([torch.from_numpy(t.reshape(-1)).to(dev) for t in twins], w, h, want)
        assert torch.equal(got.view(it), want.view(it)), what
        nb = raws[0].size
        ring = torch.from_numpy(np.concatenate([np.concatenate([r, np.full(24, 0xA5, np.uint8)]) for r in raws])).to(dev)
        strided = torch.full_like(got, float("nan"))
        pre.run_raw_strided(ring, nb + 24, n, w, h, strided, f16=f16)
        assert torch.equal(strided.view(it), want.view(it)), what
        cfg = oracle_cfg(kb, oracle, mode, sampling)
        for k in range(n):
            o = oracle.preprocess_frame(twins[k].reshape(-1), cfg, w, h, dw, dh, f16=f16 and sampling != "Lanczos")
            g = got[k].cpu().numpy()
            if sampling == "Lanczos":
                assert np.max(np.abs(g.astype(np.float32) - o)) <= (2e-3 if f16 else 1e-4), what
            else:
                np.testing.assert_array_equal(g.view(np.uint16 if f16 else np.uint32), o.view(np.uint16 if f16 else np.uint32), what)


@pytest.mark.gpu
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
def test_preprocess_host_pipeline_matrix(kb, dev, f16):
    """run_raw_host with BT.709 limited equals run_raw_batch on the same frames."""
    for fmt, mode, dw, dh in (("Nv12", "Letterbox", 64, 64), ("Yuyv", "Stretch", 100, 60), ("I420", "Stretch", 192, 108)):
        w, h, n = 192, 108, 5
        nbytes = layout_bytes(fmt, w, h)
        host = torch.from_numpy(np.stack([raw_frame(fmt, w, h, k) for k in range(n)])).pin_memory()
        pre = make_pre(kb, fmt, mode, "Bilinear", "Bt709Limited")
        want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
        (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
        pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=2 * ((nbytes + 15) // 16 * 16), dst_chunk_bytes=2 * 3 * dw * dh * 4, depth=2)
        got = pre.run_raw_host(host, w, h, (dw, dh), f16=f16, pipeline=pipe)
        torch.cuda.synchronize()
        h2d, _ = pipe.last_transfer()
        pipe.close()
        assert h2d == n * nbytes
        it = torch.int16 if f16 else torch.int32
        assert torch.equal(got.view(it), want.cpu().view(it)), fmt
        base = make_pre(kb, fmt, mode, "Bilinear")
        other = torch.zeros_like(want)
        (base.run_raw_batch_f16 if f16 else base.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, other)
        assert not torch.equal(other, want)


@pytest.mark.gpu
def test_config3a_shape_bt709(kb, oracle, dev):
    """Config 3a's shape: 1080p x 256 NV12 frames, BT.709 limited, identity geometry.  Sampled frames equal the device run
    on their RGB8 twins and the oracle on them."""
    w, h, n = 1920, 1080, 256
    nb = w * h * 3 // 2
    g = torch.Generator(device=dev).manual_seed(0x709)
    frames = torch.randint(0, 256, (n, nb), dtype=torch.uint8, device=dev, generator=g)
    pre = make_pre(kb, "Nv12", "Stretch", "Bilinear", "Bt709Limited")
    got = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)
    pre.run_raw_batch([frames[k] for k in range(n)], w, h, got)
    assert kb._lib.last_kernel() == "preprocess_nv12_identity_kernel"
    twin_pre = make_pre(kb, "Rgb8", "Stretch", "Bilinear")
    cfg = oracle_cfg(kb, oracle, "Stretch", "Bilinear")
    for k in (0, 101, n - 1):
        twin = decode_yuv8(frames[k].cpu().numpy(), w, h, "Nv12", "Bt709Limited")
        want = torch.full((1, 3, h, w), float("nan"), dtype=torch.float32, device=dev)
        twin_pre.run_raw(torch.from_numpy(twin.reshape(-1)).to(dev), w, h, want)
        assert torch.equal(got[k:k + 1].view(torch.int32), want.view(torch.int32)), k
        if k == 0:
            o = oracle.preprocess_frame(twin.reshape(-1), cfg, w, h, w, h)
            np.testing.assert_array_equal(got[k].cpu().numpy().view(np.uint32), o.view(np.uint32))
    del got, frames
    torch.cuda.empty_cache()
