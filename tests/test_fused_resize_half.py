"""The fused u8 HWC -> CHW resize+normalize with 16-bit outputs (f16 / bf16).

The rule under test: for the same arguments and leaf, a 16-bit output is round_to_nearest_even(the f32 output) — so it
must equal, bit for bit, the f32 operator followed by torch's `.to(dtype)`, in every kernel variant the dispatcher can
pick, through the device and the host-buffer entry points.  The CPU tests at the bottom check argument validation of the
new C entry points and the Python dtype errors, which need no device.
"""
import ctypes as C

import numpy as np
import pytest
import torch

HALF = [torch.float16, torch.bfloat16]
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def cu(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int16).numpy()


def assert_same_bits(got, want, what=""):
    """16-bit tensors with identical bit patterns (NaNs included)."""
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    g, w = bits(got), bits(want)
    nbad = int((g != w).sum())
    assert nbad == 0, f"{what}: {nbad} of {g.size} values differ"


def assert_matches_oracle(got, want_f32, dtype, what=""):
    """`got` (16-bit) against the oracle's f32 result rounded on the host; like assert_f32_equal, +0 and -0 are the same
    value (the oracle and the device may disagree on the sign of an exact zero)."""
    if dtype == torch.float16:
        w = np.asarray(want_f32, np.float32).astype(np.float16).view(np.int16)
    else:
        w = torch.from_numpy(np.ascontiguousarray(want_f32, np.float32)).to(torch.bfloat16).view(torch.int16).numpy()
    g = bits(got)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    zero = ((g & 0x7FFF) == 0) & ((w & 0x7FFF) == 0)
    nbad = int(((g != w) & ~zero).sum())
    assert nbad == 0, f"{what}: {nbad} values differ from the rounded oracle"


def scale_bias(oracle, kb):
    return oracle.normalize_params_from_mean_std(kb.IMAGENET_MEAN, kb.IMAGENET_STD)


def run(kb, src, dw, dh, scale, bias, dtype, **kw):
    return kb.imgproc.resize_normalize_to_tensor_u8_bilinear(src, dw, dh, scale, bias, dtype, **kw)


def f32_then_cast(kb, src, dw, dh, scale, bias, dtype, **kw):
    return kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(src, dw, dh, scale, bias, **kw).to(dtype)


# ── (1) every kernel variant, named ──────────────────────────────────────────────────────────
@gpu
@pytest.mark.parametrize("sw,sh,dw,dh,kernel", [
    (384, 216, 128, 72, "fused_rows_kernel"),      # 3:1 -> FR_POINT
    (384, 216, 192, 108, "fused_rows_kernel"),     # 2:1 -> FR_BOX
    (384, 216, 160, 90, "fused_rows_kernel"),      # 2.4:1 -> FR_GENERAL
    (384, 216, 384, 72, "fused_rows_kernel"),      # y 3:1, x 1:1 -> FR_YZERO (x general)
    (383, 216, 128, 72, "fused_resize_gather_kernel"),   # row_bytes % 16 != 0 -> gather fallback
    (3840, 40, 512, 20, "fused_resize_gather_kernel"),   # scale_x > 6 -> gather fallback
])
@pytest.mark.parametrize("leaf", [0, 1])
@pytest.mark.parametrize("dtype", HALF)
def test_half_modes_named(kb, oracle, dev, sw, sh, dw, dh, kernel, leaf, dtype):
    n = 2
    src = np.stack([oracle.pattern_u8(sw * sh * 3, 77 + i).reshape(sh, sw, 3) for i in range(n)])
    scale, bias = scale_bias(oracle, kb)
    s = cu(src, dev)
    out = run(kb, s, dw, dh, scale, bias, dtype, leaf=leaf)
    assert kb._lib.last_kernel() == kernel, kb._lib.last_kernel()
    assert out.dtype == dtype and out.shape == (n, 3, dh, dw) and out.device == s.device
    assert_same_bits(out, f32_then_cast(kb, s, dw, dh, scale, bias, dtype, leaf=leaf), f"{sw}x{sh}->{dw}x{dh} leaf {leaf}")
    want = np.stack([oracle.resize_normalize_u8_to_f32_chw(src[i], dw, dh, scale, bias, leaf) for i in range(n)])
    assert_matches_oracle(out, want, dtype, f"oracle {sw}x{sh}->{dw}x{dh} leaf {leaf}")


# ── (2) config 2 at full size, plus the 4K box and general modes ─────────────────────────────
@gpu
@pytest.mark.parametrize("dw,dh,n", [(1280, 720, 3), (1920, 1080, 1), (1600, 900, 1)])
@pytest.mark.parametrize("dtype", HALF)
def test_half_full_size_4k(kb, oracle, dev, dw, dh, n, dtype):
    sw, sh = 3840, 2160
    src = np.stack([oracle.pattern_u8(sw * sh * 3, 0x4B + i).reshape(sh, sw, 3) for i in range(n)])
    scale, bias = scale_bias(oracle, kb)
    s = cu(src, dev)
    out = run(kb, s, dw, dh, scale, bias, dtype)
    assert kb._lib.last_kernel() == "fused_rows_kernel"
    assert_same_bits(out, f32_then_cast(kb, s, dw, dh, scale, bias, dtype), f"4K -> {dw}x{dh}")
    want = np.stack([oracle.resize_normalize_u8_to_f32_chw(src[i], dw, dh, scale, bias, oracle.LEAF_X86) for i in range(n)])
    assert_matches_oracle(out, want, dtype, f"oracle 4K -> {dw}x{dh}")


# ── (3) rounding edges ───────────────────────────────────────────────────────────────────────
EDGE_GEOMS = [(384, 216, 128, 72), (384, 216, 160, 90), (384, 216, 192, 108), (383, 216, 128, 72)]


@gpu
@pytest.mark.parametrize("geom", EDGE_GEOMS)
@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("case", ["overflow", "f16_subnormal", "bf16_subnormal", "ties"])
def test_half_rounding_edges(kb, oracle, dev, geom, dtype, case):
    sw, sh, dw, dh = geom
    src = cu(oracle.pattern_u8(sw * sh * 3, 0xED).reshape(1, sh, sw, 3), dev)
    scale, bias = {
        "overflow": ([300.0, -300.0, 257.0], [0.0, 0.0, 65504.0]),         # f16: up to +-76500 -> +-inf
        "f16_subnormal": ([1e-8, -3e-8, 2.4e-7], [0.0, 0.0, 0.0]),        # f16 subnormals (< 6.1e-5), both signs
        "bf16_subnormal": ([1e-41, -3e-41, 4e-42], [0.0, 0.0, 0.0]),      # f32 and bf16 subnormals (< 1.2e-38)
        "ties": ([4.5, 0.5, 1.0 / 8.0], [1024.0, 128.0, 1.0]),             # f16 / bf16 ties at .5 steps
    }[case]
    out = run(kb, src, dw, dh, scale, bias, dtype)
    ref32 = kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(src, dw, dh, scale, bias)
    assert_same_bits(out, ref32.to(dtype), f"{case} {geom}")
    assert_same_bits(out, ref32.cpu().to(dtype), f"{case} {geom} (host conversion)")
    f = ref32.cpu().numpy()
    u = f.view(np.uint32)
    if case == "overflow" and dtype == torch.float16:
        assert np.isposinf(out.float().cpu().numpy()).sum() > 0 and np.isneginf(out.float().cpu().numpy()).sum() > 0
    if case == "f16_subnormal" and dtype == torch.float16:
        o = out.float().cpu().numpy()
        assert ((o != 0) & (np.abs(o) < 6.1e-5)).sum() > 1000
    if case == "bf16_subnormal":
        assert ((f != 0) & (np.abs(f) < 1.17e-38)).sum() > 1000           # the f32 values themselves are subnormal
        if dtype == torch.bfloat16:
            o = out.float().cpu().numpy()
            assert ((o != 0) & (np.abs(o) < 1.17e-38)).sum() > 1000
    if case == "ties" and geom in ((384, 216, 128, 72), (384, 216, 192, 108)):   # exact taps (point, box): the .5 steps survive
        tie = (u & 0x1FFF) == 0x1000 if dtype == torch.float16 else (u & 0xFFFF) == 0x8000
        assert tie.sum() > 1000, int(tie.sum())


@gpu
@pytest.mark.parametrize("geom", EDGE_GEOMS)
@pytest.mark.parametrize("dtype", HALF)
def test_half_signed_zero_and_nan(kb, oracle, dev, geom, dtype):
    sw, sh, dw, dh = geom
    zeros = torch.zeros((1, sh, sw, 3), dtype=torch.uint8, device=dev)
    # 0 * -s = -0; -0 + -0 = -0, while -0 + +0 = +0 (round to nearest)
    out = run(kb, zeros, dw, dh, [-1.0, -1.0, 1.0], [-0.0, 0.0, -0.0], dtype)
    sign = (bits(out) & np.int16(-0x8000)) != 0
    assert np.all((bits(out) & 0x7FFF) == 0)
    assert sign[:, 0].all() and not sign[:, 1].any() and not sign[:, 2].any()
    assert_same_bits(out, f32_then_cast(kb, zeros, dw, dh, [-1.0, -1.0, 1.0], [-0.0, 0.0, -0.0], dtype), f"zeros {geom}")
    # scale = inf: 0 * inf = NaN on zero bytes, +inf elsewhere — only NaN-ness is defined for a NaN
    src = cu(oracle.pattern_u8(sw * sh * 3, 0xAA).reshape(1, sh, sw, 3), dev)
    src[0, : sh // 2] = 0
    inf = float("inf")
    out = run(kb, src, dw, dh, [inf] * 3, [0.0] * 3, dtype).float().cpu()
    ref = kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(src, dw, dh, [inf] * 3, [0.0] * 3).cpu()
    assert torch.isnan(ref).any()
    assert torch.equal(torch.isnan(out), torch.isnan(ref))
    m = ~torch.isnan(ref)
    assert torch.equal(out[m], ref.to(dtype).float()[m])


# ── (4) odd layouts ──────────────────────────────────────────────────────────────────────────
@gpu
@pytest.mark.parametrize("sw,sh,dw,dh", [(384, 216, 127, 72), (384, 216, 129, 71), (384, 216, 191, 108), (383, 216, 127, 73)])
@pytest.mark.parametrize("dtype", HALF)
def test_half_odd_width_and_odd_offset_out(kb, oracle, dev, sw, sh, dw, dh, dtype):
    n = 2
    src = np.stack([oracle.pattern_u8(sw * sh * 3, 0x0DD + i).reshape(sh, sw, 3) for i in range(n)])
    scale, bias = scale_bias(oracle, kb)
    s = cu(src, dev)
    ref = f32_then_cast(kb, s, dw, dh, scale, bias, dtype)
    assert_same_bits(run(kb, s, dw, dh, scale, bias, dtype), ref, f"odd width {dw}")
    total = n * 3 * dh * dw
    buf = torch.full((total + 2,), 7.0, dtype=dtype, device=dev)
    view = buf[1:1 + total].view(n, 3, dh, dw)          # starts at an odd element: 2-byte, not 4-byte, aligned
    assert view.data_ptr() % 4 == 2
    got = run(kb, s, dw, dh, scale, bias, dtype, out=view)
    assert got is view
    assert_same_bits(view, ref, f"odd offset {dw}x{dh}")
    assert buf[0].item() == 7.0 and buf[-1].item() == 7.0   # nothing written outside the view
    want = np.stack([oracle.resize_normalize_u8_to_f32_chw(src[i], dw, dh, scale, bias, oracle.LEAF_X86) for i in range(n)])
    assert_matches_oracle(view, want, dtype, f"oracle odd {dw}x{dh}")


# ── (5) host pipeline ────────────────────────────────────────────────────────────────────────
@gpu
@pytest.mark.parametrize("sw,sh,dw,dh", [(384, 216, 128, 72), (256, 64, 64, 16), (100, 75, 33, 41), (384, 216, 192, 108)])
@pytest.mark.parametrize("dtype", HALF)
def test_half_host_pipeline(kb, oracle, dev, sw, sh, dw, dh, dtype):
    n = 11
    src = np.stack([oracle.pattern_u8(sw * sh * 3, 0xC0DE + i).reshape(sh, sw, 3) for i in range(n)])
    scale, bias = scale_bias(oracle, kb)
    want = run(kb, cu(src, dev), dw, dh, scale, bias, dtype)
    hs = torch.from_numpy(src).pin_memory()
    # staging for 2 source frames and 3 f16 frames per chunk: several chunks per stream, a ragged last one, ring wrap
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=2 * sw * sh * 3 + 7, dst_chunk_bytes=3 * dw * dh * 6, depth=2)
    with torch.cuda.device(dev):
        hd32 = torch.zeros((n, 3, dh, dw), dtype=torch.float32).pin_memory()
        kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(hs, dw, dh, scale, bias, out=hd32, pipeline=pipe)
        torch.cuda.current_stream().synchronize()
        up32, down32 = pipe.last_transfer()
        hd = torch.zeros((n, 3, dh, dw), dtype=dtype).pin_memory()
        for _ in range(2):  # second call reuses the ring
            hd.zero_()
            out = run(kb, hs, dw, dh, scale, bias, dtype, out=hd, pipeline=pipe)
            torch.cuda.current_stream().synchronize()
            assert out is hd
            assert_same_bits(hd, want, f"host {sw}x{sh}->{dw}x{dh}")
        up, down = pipe.last_transfer()
        assert up == up32 and down32 == n * 3 * dw * dh * 4 and down == n * 3 * dw * dh * 2
        alloc = run(kb, hs, dw, dh, scale, bias, dtype, pipeline=pipe)   # an output it allocates is pinned host memory
        torch.cuda.current_stream().synchronize()
        assert alloc.is_pinned() and not alloc.is_cuda and alloc.dtype == dtype
        assert_same_bits(alloc, want, "allocated host output")
        assert_same_bits(hd32.to(dtype), want, "host f32 then cast")
    pipe.close()


# ── CPU: argument validation of the C entry points, Python dtype errors ──────────────────────
def test_half_entry_points_validate_without_a_gpu(kb):
    from kornia_rs_b200 import _lib

    l = _lib.lib()
    src = (C.c_uint8 * 64)()
    dst = (C.c_uint16 * 64)()
    s, d = C.addressof(src), C.addressof(dst)
    sc, bi = _lib.f3([1.0, 1.0, 1.0]), _lib.f3([0.0, 0.0, 0.0])
    for fn in (l.kb200_resize_normalize_chw_u8_f16, l.kb200_resize_normalize_chw_u8_bf16):
        assert fn(None, None, 48, d, 12, 4, 4, 2, 2, 1, sc, bi, 1) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "null pointer for 'src'"
        assert fn(None, s, 48, None, 12, 4, 4, 2, 2, 1, sc, bi, 1) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "null pointer for 'dst'"
        assert fn(None, s, 48, d, 12, 4, 4, 2, 2, 1, None, bi, 1) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "null pointer for 'scale'"
        assert fn(None, s, 48, d, 12, 4, 4, 2, 2, 1, sc, None, 1) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "null pointer for 'bias'"
        assert fn(None, s, 48, d, 11, 4, 4, 2, 2, 1, sc, bi, 1) == _lib.ERR_SLICE_TOO_SMALL
        assert _lib.last_error() == "device slice 'dst' length 11 < required 12"
        assert fn(None, s, 47, d, 12, 4, 4, 2, 2, 1, sc, bi, 1) == _lib.ERR_SLICE_TOO_SMALL
        assert _lib.last_error() == "device slice 'src' length 47 < required 48"
        assert fn(None, s, 48, d, 12, 4, 4, 2, 2, 1, sc, bi, 3) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "unknown cpu leaf 3"
        assert fn(None, s, 48, d, 12, 4, 4, 2, 2, 0, sc, bi, 1) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "batch must be non-zero"
        assert fn(None, s, 48, d, 12, 4, 4, 2, 2, 65536, sc, bi, 1) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == "batch 65536 exceeds 65535 per call"
        assert fn(None, s, 48, d, 0, 4, 4, 0, 2, 1, sc, bi, 1) == _lib.OK   # empty destination: a no-op, no device call

    # host-buffer form: validation returns before the pipeline is used, so an opaque non-null handle suffices here
    fake = (C.c_uint8 * 1024)()
    hp = C.addressof(fake)
    host = l.kb200_resize_normalize_chw_u8_host
    assert host(None, None, s, 48, d, 12, 4, 4, 2, 2, 1, sc, bi, 1, _lib.OUT_F16) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "null pointer for 'pipeline'"
    assert host(hp, None, None, 48, d, 12, 4, 4, 2, 2, 1, sc, bi, 1, _lib.OUT_F16) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "null pointer for 'src'"
    assert host(hp, None, s, 48, None, 12, 4, 4, 2, 2, 1, sc, bi, 1, _lib.OUT_BF16) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "null pointer for 'dst'"
    for bad in (3, -1, 16):
        assert host(hp, None, s, 48, d, 12, 4, 4, 2, 2, 1, sc, bi, 1, bad) == _lib.ERR_INVALID_ARGUMENT
        assert _lib.last_error() == f"unknown output format {bad}"
    assert host(hp, None, s, 48, d, 12, 4, 4, 2, 2, 1, sc, bi, 5, _lib.OUT_F16) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "unknown cpu leaf 5"
    assert host(hp, None, s, 48, d, 12, 4, 4, 2, 2, 0, sc, bi, 1, _lib.OUT_BF16) == _lib.ERR_INVALID_ARGUMENT
    assert _lib.last_error() == "batch must be non-zero"
    for fmt in (_lib.OUT_F32, _lib.OUT_F16, _lib.OUT_BF16):
        assert host(hp, None, s, 48, d, 11, 4, 4, 2, 2, 1, sc, bi, 1, fmt) == _lib.ERR_SLICE_TOO_SMALL
        assert _lib.last_error() == "device slice 'dst' length 11 < required 12"
    # the f32 host form is the same function with KB200_OUT_F32
    assert l.kb200_resize_normalize_chw_u8_f32_host(hp, None, s, 48, d, 11, 4, 4, 2, 2, 1, sc, bi, 1) == _lib.ERR_SLICE_TOO_SMALL
    assert _lib.last_error() == "device slice 'dst' length 11 < required 12"


def test_half_python_dtype_errors(kb):
    ip = kb.imgproc
    src = torch.zeros((1, 8, 8, 3), dtype=torch.uint8)
    for bad in (torch.float64, torch.int16, torch.uint8):
        with pytest.raises(kb.ImageError) as e:
            ip.resize_normalize_to_tensor_u8_bilinear(src, 4, 4, [1.0] * 3, [0.0] * 3, bad)
        assert e.value.kind == "DtypeMismatch"
    for want, have in ((torch.float16, torch.bfloat16), (torch.bfloat16, torch.float16), (torch.float16, torch.float32),
                       (torch.float32, torch.float16)):
        out = torch.zeros((1, 3, 4, 4), dtype=have)
        with pytest.raises(kb.ImageError) as e:
            ip.resize_normalize_to_tensor_u8_bilinear(src, 4, 4, [1.0] * 3, [0.0] * 3, want, out=out)
        assert e.value.kind == "DtypeMismatch" and str(want) in str(e.value) and str(have) in str(e.value)
    with pytest.raises(kb.ImageError) as e:   # the source checks are the f32 operator's
        ip.resize_normalize_to_tensor_u8_bilinear(src.float(), 4, 4, [1.0] * 3, [0.0] * 3, torch.float16)
    assert e.value.kind == "DtypeMismatch"
