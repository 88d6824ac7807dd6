"""GPU parity, part 2: every kernel VARIANT the dispatchers can pick — and every kernel bench.py times — compared with
the oracle at geometries that actually reach it, with `kb200_last_kernel()` proving which variant produced the result.

Round-1 review found two bench-timed code paths no parity test had executed (the interior-strip loop of
`sep_filter_stream2_kernel`, which needs a row of >= 1032 floats, and `warp_tiled_kernel`, which needs a rotation on an
image with sw % 4 == 0 and >= 64 px).  The cases below are sized from the dispatch conditions in csrc/filter.cu
(`try_sep_stream`, strips of 512 floats) and csrc/warp.cu (`launch_warp`), and BASELINE configs 3b / 4 / 5 are checked
at FULL size against the oracle (whole image, not a sample — the oracle needs < 1 s per 4K image).
"""
import numpy as np
import pytest
import torch

from harness import assert_f32_bits_or_signed_zero, cu, dev, knobs, raw_bytes, rot
from restate import NAMED_FUSED_MODES, _remap_maps, fused_schedule

pytestmark = pytest.mark.gpu


def last_kernel(kb):
    return kb._lib.last_kernel()


# ── sep_filter_stream2: interior strips ───────────────────────────────────────
# strip = 512 floats; an interior strip needs e0 - HL >= 0 and e0 + 512 + HR <= cols*C, i.e. rows of >= 1032 floats.
STREAM_SHAPES = [(1100, 40, 1, 1), (700, 37, 3, 1), (3840, 24, 3, 1), (520, 33, 4, 2), (1376, 19, 3, 2), (2064, 70, 1, 1)]


@pytest.mark.parametrize("w,h,c,n", STREAM_SHAPES)
@pytest.mark.parametrize("k,sigma", [((3, 3), (0.8, 0.8)), ((5, 5), (1.5, 1.5)), ((7, 7), (2.0, 2.0))])
def test_gaussian_blur_interior_strips(kb, oracle, dev, w, h, c, n, k, sigma):
    if c == 4 and k[0] == 7:
        pytest.skip("no streaming instance for C=4, K=7 (tile kernel; covered by test_gaussian_blur)")
    assert w * c >= 1032 and (w * c) % 4 == 0
    src = oracle.pattern_f32(n * w * h * c).reshape(n, h, w, c)
    dst = kb.Image.zeros_cuda(kb.ImageSize(w, h), c, torch.float32, dev, batch=n)
    kb.imgproc.gaussian_blur(kb.Image(cu(src, dev)), dst, k, sigma)
    assert last_kernel(kb) == "sep_filter_stream2_kernel"
    want = np.stack([oracle.gaussian_blur(src[i], k, sigma) for i in range(n)])
    assert_f32_bits_or_signed_zero(dst.numpy(), want, f"gaussian interior {w}x{h}x{c} k={k}")


@pytest.mark.parametrize("w,h,c,n", [(1100, 40, 1, 1), (700, 37, 3, 2), (3840, 24, 3, 1), (2064, 70, 1, 1)])
@pytest.mark.parametrize("ksize", [3, 5])
def test_sobel_interior_strips(kb, oracle, dev, w, h, c, n, ksize):
    src = oracle.pattern_f32(n * w * h * c).reshape(n, h, w, c)
    dst = kb.Image.zeros_cuda(kb.ImageSize(w, h), c, torch.float32, dev, batch=n)
    kb.imgproc.sobel(kb.Image(cu(src, dev)), dst, ksize)
    assert last_kernel(kb) == "sep_filter_stream2_kernel"
    want = np.stack([oracle.sobel(src[i], ksize) for i in range(n)])
    assert_f32_bits_or_signed_zero(dst.numpy(), want, f"sobel interior {w}x{h}x{c} k={ksize}")


def test_filter_stream_nonfinite_and_chunk_seams(kb, oracle, dev):
    """Chunk seams (rows_per_chunk boundaries re-stage KY-1 halo rows) and non-finite inputs: inf/NaN must propagate
    exactly like the reference's skip-OOB-tap loop (zero-filled halos add +0, never 0*inf)."""
    w, h, c = 1376, 300, 3
    src = oracle.pattern_f32(w * h * c).reshape(h, w, c).copy()
    src[0, 0, 0] = np.inf; src[h - 1, w - 1, 2] = -np.inf; src[150, 700, 1] = np.nan; src[0, w - 1, 1] = np.inf
    dst = kb.Image.zeros_cuda(kb.ImageSize(w, h), c, torch.float32, dev)
    kb.imgproc.gaussian_blur(kb.Image(cu(src, dev)), dst, (5, 5), (1.5, 1.5))
    want = oracle.gaussian_blur(src, (5, 5), (1.5, 1.5))
    got = dst.numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    m = ~np.isnan(want)
    assert np.array_equal(got[m], want[m])


@pytest.mark.parametrize("sw,sh", [(128, 96), (256, 192), (640, 360)])
@pytest.mark.parametrize("angle", [30.0, 45.0, -17.5, 75.0])
@pytest.mark.parametrize("mode", ["Bilinear", "Nearest"])
def test_warp_affine_tiled(kb, oracle, dev, sw, sh, angle, mode):
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    m = rot(kb, sw, sh, angle)
    dst = kb.Image.from_size_val(kb.ImageSize(sw, sh), -3.0, 3, torch.float32, dev)
    kb.imgproc.warp_affine(kb.Image(cu(src, dev)), dst, m, kb.InterpolationMode[mode])
    assert last_kernel(kb) == "warp_tiled_kernel", last_kernel(kb)
    want = oracle.warp_affine_f32(src, m, sw, sh, oracle.BILINEAR if mode == "Bilinear" else oracle.NEAREST)
    assert_f32_bits_or_signed_zero(dst.numpy(), want, f"tiled affine {angle} {mode} {sw}x{sh}")


@pytest.mark.parametrize("mode", ["Bilinear", "Nearest"])
def test_warp_perspective_tiled_strong_shear(kb, oracle, dev, mode):
    sw, sh, n = 256, 192, 2
    h = [0.8, 0.45, -20.0, -0.5, 0.85, 60.0, 1.0e-4, -6.0e-5, 1.0]
    src = oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3)
    dst = kb.Image.from_size_val(kb.ImageSize(sw, sh), 9.0, 3, torch.float32, dev, batch=n)
    kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst, h, kb.InterpolationMode[mode])
    assert last_kernel(kb) == "warp_tiled_kernel", last_kernel(kb)
    om = oracle.BILINEAR if mode == "Bilinear" else oracle.NEAREST
    want = np.stack([oracle.warp_perspective_f32(src[i], h, sw, sh, om) for i in range(n)])
    assert_f32_bits_or_signed_zero(dst.numpy(), want, f"tiled perspective {mode}")


def test_warp_two_devices_one_process(kb, oracle):
    """The library is used from one process on several devices (kb200_set_device): per-device function attributes
    (dynamic shared memory opt-in) must be set on every device, not once per process."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs in one process")
    sw, sh = 256, 192
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    m = rot(kb, sw, sh, 30.0)
    want = oracle.warp_affine_f32(src, m, sw, sh, oracle.BILINEAR)
    for d in (0, 1, 0):
        dev = torch.device(f"cuda:{d}")
        dst = kb.Image.zeros_cuda(kb.ImageSize(sw, sh), 3, torch.float32, dev)
        kb.imgproc.warp_affine(kb.Image(cu(src, dev)), dst, m, kb.InterpolationMode.Bilinear)
        assert last_kernel(kb) == "warp_tiled_kernel"
        assert_f32_bits_or_signed_zero(dst.numpy(), want, f"device {d}")
        blur = kb.Image.zeros_cuda(kb.ImageSize(sw, sh), 3, torch.float32, dev)
        kb.imgproc.gaussian_blur(kb.Image(cu(src, dev)), blur, (5, 5), (1.5, 1.5))
        assert_f32_bits_or_signed_zero(blur.numpy(), oracle.gaussian_blur(src, (5, 5), (1.5, 1.5)), f"blur device {d}")


# ── BASELINE configs at FULL size, whole image against the oracle ───────────────
H_CFG5 = [1.02, 0.03, -40.0, -0.03, 1.01, 25.0, 2.0e-6, 1.2e-6, 1.0]


def test_full_size_config4_blur_sobel_4k(kb, oracle, dev):
    """Config 4 (4K f32, gaussian 5x5 sigma 1.5 -> sobel 3): every pixel of one 4K image, borders included."""
    w, h = 3840, 2160
    src = oracle.pattern_f32(w * h * 3).reshape(h, w, 3)
    a = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.float32, dev)
    b = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.float32, dev)
    kb.imgproc.gaussian_blur(kb.Image(cu(src, dev)), a, (5, 5), (1.5, 1.5))
    assert last_kernel(kb) == "sep_filter_stream2_kernel"
    blur = oracle.gaussian_blur(src, (5, 5), (1.5, 1.5), mt=True)
    assert_f32_bits_or_signed_zero(a.numpy(), blur, "cfg4 blur 4K")
    kb.imgproc.sobel(a, b, 3)
    assert last_kernel(kb) == "sep_filter_stream2_kernel"
    assert_f32_bits_or_signed_zero(b.numpy(), oracle.sobel(blur, 3, mt=True), "cfg4 sobel 4K")


@pytest.mark.parametrize("mode", ["Bilinear", "Nearest"])
def test_full_size_config5_warp_perspective_4k(kb, oracle, dev, mode):
    """Config 5 (4K f32, BASELINE homography): every pixel of two 4K images (batch > 1 exercises the image walk)."""
    w, h, n = 3840, 2160, 2
    src = oracle.pattern_f32(n * w * h * 3).reshape(n, h, w, 3)
    dst = kb.Image.from_size_val(kb.ImageSize(w, h), 5.0, 3, torch.float32, dev, batch=n)
    kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst, H_CFG5, kb.InterpolationMode[mode])
    om = oracle.BILINEAR if mode == "Bilinear" else oracle.NEAREST
    got = dst.numpy()
    for i in range(n):
        assert_f32_bits_or_signed_zero(got[i], oracle.warp_perspective_f32(src[i], H_CFG5, w, h, om), f"cfg5 image {i} {mode} ({last_kernel(kb)})")


def test_full_size_warp_affine_rot30_4k(kb, oracle, dev):
    """The bench's `warp_affine_rot30_4k_f32` row at full size."""
    w, h = 3840, 2160
    src = oracle.pattern_f32(w * h * 3).reshape(h, w, 3)
    m = rot(kb, w, h, 30.0)
    dst = kb.Image.from_size_val(kb.ImageSize(w, h), 5.0, 3, torch.float32, dev)
    kb.imgproc.warp_affine(kb.Image(cu(src, dev)), dst, m, kb.InterpolationMode.Bilinear)
    assert_f32_bits_or_signed_zero(dst.numpy(), oracle.warp_affine_f32(src, m, w, h, oracle.BILINEAR), f"rot30 4K ({last_kernel(kb)})")


@pytest.mark.parametrize("f16", [False, True])
def test_full_size_config3b_nv12_letterbox640(kb, oracle, dev, f16):
    """Config 3b at full size: 1080p NV12 -> letterbox 640x640 (pad 114), ImageNet normalisation; whole frames,
    pad rows included, f32 and f16 (RNE)."""
    w, h, n, d = 1920, 1080, 3, 640
    frame = w * h * 3 // 2
    raws = [raw_bytes(frame, k) for k in range(n)]
    pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).mode(kb.ResizeMode.Letterbox)
           .normalize(kb.Normalize.imagenet()).build_cuda())
    dst = torch.zeros((n, 3, d, d), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([cu(r, dev) for r in raws], w, h, dst)
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    cfg = oracle.PreprocessCfg(mode=oracle.LETTERBOX, fmt=oracle.FMT_NV12, mean=kb.IMAGENET_MEAN, inv_std=inv)
    want = np.stack([oracle.preprocess_frame(r, cfg, w, h, d, d, f16=f16) for r in raws])
    got = dst.cpu().numpy()
    if f16:
        np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    else:
        assert_f32_bits_or_signed_zero(got, want, "cfg3b")
    # rows 0..139 and 500..639 are padding: the normalised pad value, exactly
    pad = ((np.float32(114.0) / np.float32(255.0) - np.array(kb.IMAGENET_MEAN, np.float32)) * np.array(inv, np.float32))
    top = got[:, :, :140, :].astype(np.float32)
    for c in range(3):
        ref = np.float16(pad[c]) if f16 else pad[c]
        assert np.all(top[:, c] == np.float32(ref))


# ── fused resize: every mode of fused_rows + the gather fallback, with the kernel named ─────
# the mode each geometry below must reach, checked with the host mirror of the dispatcher (restate.fused_schedule)


@pytest.mark.parametrize("sw,sh,dw,dh,kernel", [
    (384, 216, 128, 72, "fused_rows_kernel"),      # 3:1 -> FR_POINT
    (384, 216, 192, 108, "fused_rows_kernel"),     # 2:1 -> FR_BOX
    (384, 216, 160, 90, "fused_rows_kernel"),      # 2.4:1 -> FR_GENERAL
    (384, 216, 384, 72, "fused_rows_kernel"),      # y 3:1, x 1:1 -> FR_POINT (a 1:1 axis has all-zero weights too)
    (384, 216, 160, 72, "fused_rows_kernel"),      # y 3:1, x 2.4:1 -> FR_YZERO (x general)
    (383, 216, 128, 72, "fused_resize_gather_kernel"),   # row_bytes % 16 != 0 -> gather fallback
    (3840, 40, 512, 20, "fused_resize_gather_kernel"),   # scale_x > 6 -> gather fallback
])
@pytest.mark.parametrize("leaf", [0, 1])
def test_fused_resize_modes_named(kb, oracle, dev, sw, sh, dw, dh, kernel, leaf):

    n = 2
    assert fused_schedule(sw, sh, dw, dh, n, torch.cuda.get_device_properties(dev).multi_processor_count).mode == NAMED_FUSED_MODES[(sw, sh, dw, dh)]
    src = np.stack([oracle.pattern_u8(sw * sh * 3, 77 + i).reshape(sh, sw, 3) for i in range(n)])
    scale, bias = oracle.normalize_params_from_mean_std(kb.IMAGENET_MEAN, kb.IMAGENET_STD)
    out = kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(cu(src, dev), dw, dh, scale, bias, leaf=leaf)
    assert last_kernel(kb) == kernel, last_kernel(kb)
    want = np.stack([oracle.resize_normalize_u8_to_f32_chw(src[i], dw, dh, scale, bias, leaf) for i in range(n)])
    assert_f32_bits_or_signed_zero(out.cpu().numpy(), want, f"fused {sw}x{sh}->{dw}x{dh} leaf {leaf}")


def test_std_mean_unaligned_base(kb, oracle, dev):
    """A tensor slice at an odd byte offset: the head-peel path must give the same exact sums (ADVICE r1)."""
    npx = 4096 * 3 + 7
    raw = oracle.pattern_u8(npx * 3 + 5, 4242)
    t = cu(raw, dev)
    for off in (1, 2, 3, 5):
        view = t[off:off + npx * 3].reshape(1, npx, 3)
        got = kb.imgproc.std_mean_sums(kb.Image(view)).tolist()
        _, _, osums = oracle.std_mean(raw[off:off + npx * 3].reshape(1, npx, 3))
        assert got == [int(v) for v in osums], (off, got, osums)


def test_find_min_max_nan_first(kb, dev):
    """normalize.rs:123-146 seeds with the first element: NaN first -> (NaN, NaN); NaN elsewhere never wins."""
    a = torch.tensor([float("nan"), 1.0, -2.0, 5.0], device=dev).reshape(1, 4, 1)
    mn, mx = kb.imgproc.find_min_max(kb.Image(a))
    assert np.isnan(mn) and np.isnan(mx)
    b = torch.tensor([1.0, float("nan"), -2.0, 5.0], device=dev).reshape(1, 4, 1)
    assert kb.imgproc.find_min_max(kb.Image(b)) == (-2.0, 5.0)


# ── a1: f32 HWC resize — the row-streaming kernel and its fallback, named ───────
@pytest.mark.parametrize("sw,sh,dw,dh,kernel", [
    (384, 216, 128, 72, "resize_rows_f32_kernel"),     # 3:1 exact (weights 0, all four taps still fetched)
    (640, 360, 320, 180, "resize_rows_f32_kernel"),    # 2:1
    (640, 360, 212, 120, "resize_rows_f32_kernel"),    # non-integer ratio
    (64, 48, 128, 96, "resize_rows_f32_kernel"),       # 2x upscale (y1 == y0 rows, x1 == x0 at the right edge)
    (1280, 16, 1000, 37, "resize_rows_f32_kernel"),    # several column tiles, ragged last tile, vertical upscale
    (129, 97, 64, 48, "resize_f32_c3_kernel"),         # sw % 4 != 0 -> gather fallback
    (128, 96, 66, 50, "resize_f32_c3_kernel"),         # dw % 4 != 0 -> gather fallback
])
def test_resize_f32_rows_named(kb, oracle, dev, sw, sh, dw, dh, kernel):
    n = 3
    src = oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3)
    dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), -1.0, 3, torch.float32, dev, batch=n)
    kb.imgproc.resize(kb.Image(cu(src, dev)), dst, kb.InterpolationMode.Bilinear)
    assert last_kernel(kb) == kernel, last_kernel(kb)
    want = np.stack([oracle.resize_f32(src[i], dw, dh) for i in range(n)])
    assert_f32_bits_or_signed_zero(dst.numpy(), want, f"resize rows {sw}x{sh}->{dw}x{dh}")


def test_resize_f32_rows_nonfinite_taps(kb, oracle, dev):
    """A zero-weight tap on inf must give NaN exactly where the reference does (0 * inf): the f32 path may not skip taps."""
    sw, sh, dw, dh = 384, 216, 128, 72
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3).copy()
    src[5, 8, 0] = np.inf      # tapped with weight 0 by (dx, dy) = (2, 1): x0 = 7, x1 = 8; y0 = 4, y1 = 5
    src[100, 200, 1] = np.nan
    src[215, 383, 2] = -np.inf
    dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev)
    kb.imgproc.resize(kb.Image(cu(src, dev)), dst, kb.InterpolationMode.Bilinear)
    assert last_kernel(kb) == "resize_rows_f32_kernel"
    got, want = dst.numpy(), oracle.resize_f32(src, dw, dh)
    assert np.isnan(want).any()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    m = ~np.isnan(want)
    assert np.array_equal(got[m], want[m])


@pytest.mark.parametrize("align", [False, True])
def test_resize_bilinear_normalize_rows(kb, oracle, dev, align):
    sw, sh, dw, dh, n = 640, 360, 320, 180, 2
    src = oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev, batch=n)
    kb.imgproc.resize_bilinear_normalize(kb.Image(cu(src, dev)), dst, mean, std, align_corners=align)
    assert last_kernel(kb) == "resize_rows_f32_kernel"
    if not align:   # (v - mean) * (1/std) on the bilinear sample, cuda/resize.rs:183-235
        base = np.stack([oracle.resize_f32(src[i], dw, dh) for i in range(n)])
        inv = (np.float32(1.0) / np.array(std, np.float32))
        want = (base - np.array(mean, np.float32)) * inv
        assert_f32_bits_or_signed_zero(dst.numpy(), want.astype(np.float32), "resize+normalize rows")
    # both mappings: a different column tiling (3 columns per thread) must give the same bits
    with knobs(kb, {"rs.npx": 3}):
        again = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev, batch=n)
        kb.imgproc.resize_bilinear_normalize(kb.Image(cu(src, dev)), again, mean, std, align_corners=align)
    assert torch.equal(again.data, dst.data)


def test_full_size_resize_f32_4k(kb, oracle, dev):
    """The bench's resize_f32 rows at full size: 4K -> 720p / 1080p / 1600x900, whole image against the oracle."""
    w, h = 3840, 2160
    src = oracle.pattern_f32(w * h * 3).reshape(h, w, 3)
    t = kb.Image(cu(src, dev))
    for dw, dh in ((1280, 720), (1920, 1080), (1600, 900)):
        dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev)
        kb.imgproc.resize(t, dst, kb.InterpolationMode.Bilinear)
        assert last_kernel(kb) == "resize_rows_f32_kernel"
        assert_f32_bits_or_signed_zero(dst.numpy(), oracle.resize_f32(src, dw, dh), f"4K -> {dw}x{dh}")


# ── warp_stream_kernel (row-streaming, TMA row ring): gentle maps ───────────────
STREAM_H = [
    ("cfg5-like", [1.02, 0.03, -7.0, -0.03, 1.01, 4.0, 1.2e-5, 7.0e-6, 1.0]),
    ("identity", [1, 0, 0, 0, 1, 0, 0, 0, 1]),
    ("shift", [1, 0, 5.5, 0, 1, -3.25, 0, 0, 1]),
    ("zoom-out", [0.6, 0.02, 30.0, -0.01, 0.7, 20.0, 0, 0, 1]),        # destination smaller than the source footprint: zero fill around
    ("zoom-in", [1.8, 0.05, -200.0, 0.04, 1.7, -120.0, 1e-5, 0, 1]),   # rows re-used by several destination rows
    ("keystone", [1.0, 0.08, -10.0, 0.0, 1.05, -5.0, 0.0, 2.5e-4, 1.0]),
]


@pytest.mark.parametrize("name,h", STREAM_H)
@pytest.mark.parametrize("mode", ["Bilinear", "Nearest"])
@pytest.mark.parametrize("size", [(640, 360), (388, 211)])
def test_warp_perspective_stream(kb, oracle, dev, name, h, mode, size):
    sw, sh = size
    n = 2
    src = oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3)
    dst = kb.Image.from_size_val(kb.ImageSize(sw, sh), 9.0, 3, torch.float32, dev, batch=n)
    with knobs(kb, {"warp.path": 3}):
        kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst, h, kb.InterpolationMode[mode])
        k = last_kernel(kb)
    assert k == ("warp_stream2_kernel" if mode == "Bilinear" else "warp_stream_kernel"), k
    om = oracle.BILINEAR if mode == "Bilinear" else oracle.NEAREST
    want = np.stack([oracle.warp_perspective_f32(src[i], h, sw, sh, om) for i in range(n)])
    assert_f32_bits_or_signed_zero(dst.numpy(), want, f"stream perspective {name} {mode} {size}")


# ── warp_bilinear_lean_kernel (round 2, second pass): interior fast path + per-pixel general path ──────────
def _scaled(h, k):
    return [v * k for v in h]


LEAN_H = STREAM_H + [
    ("cfg5", H_CFG5),
    ("negative-denominator", _scaled(STREAM_H[0][1], -1.0)),       # the same map; every w of the inverse is negative
    ("denominator-1e3", _scaled(STREAM_H[0][1], 1.0e-3)),          # inverse scaled by 1e3: w ~ 1e3, numerators ~ 1e6
    ("denominator-3e-4", _scaled(STREAM_H[0][1], 3.0e3)),          # w ~ 3e-4: just inside the host-proved window
    ("denominator-outside-window", _scaled(STREAM_H[0][1], 3.0e4)),    # w ~ 3e-5: the host refuses the fast path
    ("w-crosses-zero", [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 3.0e-3, 0.0, 1.0]),   # inverse denominator changes sign inside the image
    ("origin-on-a-pixel", [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 1.0e-4, 2.0e-4, 1.0]),   # numerators exactly 0 along the first row / column
]


@pytest.mark.parametrize("name,h", LEAN_H)
@pytest.mark.parametrize("size", [(640, 360), (389, 211), (97, 61)])
def test_warp_perspective_lean(kb, oracle, dev, name, h, size):
    """Every dispatch of the bilinear gather: the lean kernel with the fast path allowed (knob a = 0), with the general path
    forced (a = 4) and the round-2 x4 kernel (a = 3) must all give the oracle's bits.  Sizes: multiples of 32 and not (partial
    warps vote with the live-lane mask; a last block row with one or two rows of a pair missing)."""
    sw, sh = size
    n = 2
    src = oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3)
    want = np.stack([oracle.warp_perspective_f32(src[i], h, sw, sh, oracle.BILINEAR) for i in range(n)])
    t = kb.Image(cu(src, dev))
    stg = "" if sw % 4 == 0 else "/stg"       # TMA tile stores need 16-byte aligned destination rows
    lean, gen = "warp_bilinear_lean_kernel", "warp_bilinear_lean_kernel/general"
    # knob a: 0 default (one 4-D tensor-map store per warp when dh % 8 == 0, else four 1-D row copies), 7 the 1-D row copies, 4 general
    # path only, 5 STG stores, 3 the round-2 x4 kernel
    for a, d, kernels in ((0, 0, (lean + stg, gen + stg)), (7, 0, (lean + stg, gen + stg)), (4, 0, (gen + stg,)), (5, 0, (lean + "/stg", gen + "/stg")),
                          (3, 0, ("warp_bilinear_x4_kernel",))):
        dst = kb.Image.from_size_val(kb.ImageSize(sw, sh), 9.0, 3, torch.float32, dev, batch=n)
        with knobs(kb, {"a": a, "d": d, "warp.path": 1}):
            kb.imgproc.warp_perspective(t, dst, h, kb.InterpolationMode.Bilinear)
            k = last_kernel(kb)
        assert k in kernels, k
        if a == 0 and (name == "denominator-outside-window" or (name == "w-crosses-zero" and sw > 340)):   # w = 1 - 0.003 x
            assert k == gen + stg, k
        if a == 0 and name in ("cfg5", "cfg5-like", "negative-denominator", "denominator-1e3", "denominator-3e-4", "identity"):
            assert k == lean + stg, k
        assert_f32_bits_or_signed_zero(dst.numpy(), want, f"lean perspective {name} {size} a={a} d={d} ({k})")


@pytest.mark.parametrize("angle,scale", [(0.0, 1.0), (2.0, 1.0), (-3.5, 0.9), (8.0, 1.2), (90.0, 1.0), (180.0, 0.7)])
@pytest.mark.parametrize("dsize", [(480, 260), (333, 201)])
def test_warp_affine_lean(kb, oracle, dev, angle, scale, dsize):
    """Affine maps through the lean gather kernel (path knob 1 keeps rotations off the tiled kernel); 90 degrees is the
    degenerate-axis case (|m0| < 1e-6: validity judged on the row constant) which must take the general path."""
    sw, sh = 512, 300
    dw, dh = dsize
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    m = rot(kb, sw, sh, angle, scale)
    want = oracle.warp_affine_f32(src, m, dw, dh, oracle.BILINEAR)
    t = kb.Image(cu(src, dev))
    for a, d in ((0, 0), (4, 0), (5, 0), (3, 0)):
        dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), 9.0, 3, torch.float32, dev)
        with knobs(kb, {"a": a, "d": d, "warp.path": 1}):
            kb.imgproc.warp_affine(t, dst, m, kb.InterpolationMode.Bilinear)
            k = last_kernel(kb)
        if a == 0:
            stg = "" if dw % 4 == 0 else "/stg"
            # cos 90 / sin 180 are ~1e-8 in f32, not 0: degenerate axes (|m| < 1e-6, judged on the row constant) -> general path;
            # sin 0 is exactly 0: coordinate == row constant, the fast path stays
            assert k == ("warp_bilinear_lean_kernel/general" if angle in (90.0, 180.0) else "warp_bilinear_lean_kernel") + stg, k
        assert_f32_bits_or_signed_zero(dst.numpy(), want, f"lean affine {angle} x{scale} {dsize} a={a} d={d} ({k})")


def test_warp_lean_nonfinite_and_degenerate_matrices(kb, oracle, dev):
    """A source holding inf / NaN (0 * inf must stay NaN: all four taps are always read) and a homography whose inverse has a
    NaN-producing row: the result must match the oracle element for element (NaN == NaN here)."""
    sw, sh = 160, 96
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3).copy()
    src[10, 20, 0] = np.inf; src[11, 21, 1] = -np.inf; src[40, 50, 2] = np.nan
    h = [1.01, 0.02, -3.0, -0.02, 1.02, 2.0, 1.0e-5, 5.0e-6, 1.0]
    dst = kb.Image.from_size_val(kb.ImageSize(sw, sh), 9.0, 3, torch.float32, dev)
    with knobs(kb, {"warp.path": 1}):
        kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst, h, kb.InterpolationMode.Bilinear)
        assert last_kernel(kb) == "warp_bilinear_lean_kernel"
    got, want = dst.numpy(), oracle.warp_perspective_f32(src, h, sw, sh, oracle.BILINEAR)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = ~np.isnan(want)
    assert np.array_equal(got[fin].view(np.uint32), want[fin].view(np.uint32))


@pytest.mark.parametrize("angle,scale", [(0.0, 1.0), (2.0, 1.0), (-3.5, 0.9), (8.0, 1.2), (30.0, 1.0)])
@pytest.mark.parametrize("mode", ["Bilinear", "Nearest"])
def test_warp_affine_stream(kb, oracle, dev, angle, scale, mode):
    """Small rotations stream; 30 degrees has a tall band (forced here: most taps take the resident path through a deep
    ring or the global fallback — either way the bits must not change)."""
    sw, sh, dw, dh = 512, 300, 480, 260
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    m = rot(kb, sw, sh, angle, scale)
    dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), 9.0, 3, torch.float32, dev)
    with knobs(kb, {"warp.path": 3}):
        kb.imgproc.warp_affine(kb.Image(cu(src, dev)), dst, m, kb.InterpolationMode[mode])
        k = last_kernel(kb)
    if angle < 20:
        assert k == ("warp_stream2_kernel" if mode == "Bilinear" else "warp_stream_kernel"), k
    om = oracle.BILINEAR if mode == "Bilinear" else oracle.NEAREST
    assert_f32_bits_or_signed_zero(dst.numpy(), oracle.warp_affine_f32(src, m, dw, dh, om), f"stream affine {angle} x{scale} {mode} ({k})")


def test_warp_stream_small_ring_and_chunks(kb, oracle, dev):
    """A ring smaller than the band (taps beyond it fall back to global loads), short row chunks (many unit seams) and
    one column per thread: every knob combination must give the oracle's bits."""
    sw, sh = 640, 360
    h = [1.02, 0.06, -7.0, -0.05, 1.01, 9.0, 1.2e-5, 7.0e-6, 1.0]
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    want = oracle.warp_perspective_f32(src, h, sw, sh, oracle.BILINEAR)
    t = kb.Image(cu(src, dev))
    # ws.npx: 1 = pair-row fast consumer (bilinear default), 2 / 3 = generic consumer with two / one columns per thread
    for stages, rc, npx in ((4, 0, 2), (8, 7, 1), (16, 33, 3), (64, 360, 1), (4, 10, 1), (8, 0, 2)):
        with knobs(kb, {"warp.path": 3, "ws.stages": stages, "ws.rc": rc, "ws.npx": npx}):
            dst = kb.Image.from_size_val(kb.ImageSize(sw, sh), 9.0, 3, torch.float32, dev)
            kb.imgproc.warp_perspective(t, dst, h, kb.InterpolationMode.Bilinear)
            assert last_kernel(kb) == ("warp_stream2_kernel" if npx == 1 else "warp_stream_kernel")
        assert_f32_bits_or_signed_zero(dst.numpy(), want, f"stream knobs stages={stages} rc={rc} npx={npx}")


def test_warp_stream_unaligned_destination(kb, oracle, dev):
    """dw % 4 != 0: the scalar-store path of the streaming kernel."""
    sw, sh, dw, dh = 640, 360, 333, 201
    h = [1.9, 0.03, -3.0, -0.02, 1.8, 2.0, 0.0, 0.0, 1.0]
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), 9.0, 3, torch.float32, dev)
    with knobs(kb, {"warp.path": 3}):
        kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst, h, kb.InterpolationMode.Bilinear)
        assert last_kernel(kb) == "warp_stream2_kernel"
        with knobs(kb, {"ws.npx": 2}):
            dst2 = kb.Image.from_size_val(kb.ImageSize(dw, dh), 9.0, 3, torch.float32, dev)
            kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst2, h, kb.InterpolationMode.Bilinear)
            assert last_kernel(kb) == "warp_stream_kernel"
    want = oracle.warp_perspective_f32(src, h, dw, dh, oracle.BILINEAR)
    assert_f32_bits_or_signed_zero(dst.numpy(), want, "stream2 unaligned dst")
    assert_f32_bits_or_signed_zero(dst2.numpy(), want, "stream unaligned dst")


# ── bicubic / Lanczos samplers (SURVEY §8(f) #3) against the oracle ──────────────
HQ = [("Bicubic", 2), ("Lanczos", 3)]


@pytest.mark.parametrize("name,code", HQ)
@pytest.mark.parametrize("sw,sh,dw,dh", [(129, 97, 64, 48), (64, 48, 129, 97), (258, 195, 128, 128), (31, 17, 7, 5), (5, 7, 31, 17), (640, 360, 213, 120)])
def test_resize_hq(kb, oracle, dev, name, code, sw, sh, dw, dh):
    n = 2
    src = oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3)
    dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev, batch=n)
    kb.imgproc.resize(kb.Image(cu(src, dev)), dst, kb.InterpolationMode[name])
    want = np.stack([oracle.resize_f32(src[i], dw, dh, code) for i in range(n)])
    assert_f32_bits_or_signed_zero(dst.numpy(), want, f"resize {name} {sw}x{sh}->{dw}x{dh}")


@pytest.mark.parametrize("name,code", HQ)
def test_warps_hq(kb, oracle, dev, name, code):
    sw, sh, dw, dh = 97, 61, 80, 70
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    for angle in (0.0, 30.0, 90.0, -17.5):
        m = rot(kb, sw, sh, angle, 0.9)
        dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), 4.0, 3, torch.float32, dev)
        kb.imgproc.warp_affine(kb.Image(cu(src, dev)), dst, m, kb.InterpolationMode[name])
        assert_f32_bits_or_signed_zero(dst.numpy(), oracle.warp_affine_f32(src, m, dw, dh, code), f"warp_affine {name} {angle}")
    for h in ([1.03, 0.05, -3.0, -0.02, 0.97, 4.0, 2.0 / (97 * 129), 1.5 / (129 * 97), 1.0], [0.9, 0.15, 10.0, -0.1, 1.1, -6.0, 0.0, 0.0, 1.0]):
        dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev)   # CPU leaves OOB untouched, GPU writes 0
        kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst, h, kb.InterpolationMode[name])
        assert_f32_bits_or_signed_zero(dst.numpy(), oracle.warp_perspective_f32(src, h, dw, dh, code), f"warp_perspective {name}")
    gray = kb.Image.zeros_cuda(kb.ImageSize(8, 8), 1, torch.float32, dev)
    with pytest.raises(kb.ImageError, match="3-channel f32 images only"):
        kb.imgproc.resize(gray, kb.Image.zeros_cuda(kb.ImageSize(4, 4), 1, torch.float32, dev), kb.InterpolationMode[name])


@pytest.mark.parametrize("fmt,bpp", [("Rgb8", 3), ("Nv12", 1), ("Yuyv", 2), ("Gray8", 1)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_lanczos_vs_oracle(kb, oracle, dev, fmt, bpp, f16):
    """Lanczos sampling of the camera preprocess: the reference kernel calls sinf (CUDA math library); the oracle calls
    host sinf — checked within the north-star tolerance (1e-4 on [0,1]-scaled values); bit-equality with the reference's
    own kernel is asserted in test_ref_gpu_kernels.py."""
    w, h, dw, dh, n = 96, 64, 50, 40, 2
    nbytes = {"Rgb8": w * h * 3, "Nv12": w * h * 3 // 2, "Yuyv": w * h * 2, "Gray8": w * h}[fmt]
    raws = [oracle.pattern_u8(nbytes, 900 + k) for k in range(n)]
    pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode.Letterbox).sampling(kb.InterpolationMode.Lanczos)
           .normalize(kb.Normalize.UnitScale()).build_cuda())
    dst = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([cu(r, dev) for r in raws], w, h, dst)
    code = {"Rgb8": oracle.FMT_RGB, "Nv12": oracle.FMT_NV12, "Yuyv": oracle.FMT_YUYV, "Gray8": oracle.FMT_GRAY}[fmt]
    cfg = oracle.PreprocessCfg(mode=oracle.LETTERBOX, fmt=code, sampling=oracle.LANCZOS)
    want = np.stack([oracle.preprocess_frame(r, cfg, w, h, dw, dh) for r in raws])
    got = dst.float().cpu().numpy()
    tol = 2e-3 if f16 else 1e-4
    assert np.max(np.abs(got - want)) <= tol, np.max(np.abs(got - want))


# ── pyramids (SURVEY §8(f) #4) ───────────────────────────────────────────────────
@pytest.mark.parametrize("w,h,c,n", [(53, 37, 3, 2), (16, 16, 1, 1), (7, 5, 4, 3), (2, 2, 3, 1), (1, 1, 1, 1), (1, 6, 3, 1), (9, 1, 1, 2), (640, 360, 3, 2)])
def test_pyramids(kb, oracle, dev, w, h, c, n):
    f = oracle.pattern_f32(n * w * h * c, 8).reshape(n, h, w, c)
    u = oracle.pattern_u8(n * w * h * c, 9).reshape(n, h, w, c)
    for data, dt, down, up in ((f, torch.float32, oracle.pyrdown_f32, oracle.pyrup_f32), (u, torch.uint8, oracle.pyrdown_u8, oracle.pyrup_u8)):
        src = kb.Image(cu(data, dev))
        dn = kb.Image.zeros_cuda(kb.ImageSize((w + 1) // 2, (h + 1) // 2), c, dt, dev, batch=n)
        kb.imgproc.pyrdown(src, dn)
        want = np.stack([down(data[i]) for i in range(n)])
        (assert_f32_bits_or_signed_zero if dt == torch.float32 else np.testing.assert_array_equal)(dn.numpy().reshape(want.shape), want)
        upi = kb.Image.zeros_cuda(kb.ImageSize(2 * w, 2 * h), c, dt, dev, batch=n)
        kb.imgproc.pyrup(src, upi)
        want = np.stack([up(data[i]) for i in range(n)])
        (assert_f32_bits_or_signed_zero if dt == torch.float32 else np.testing.assert_array_equal)(upi.numpy().reshape(want.shape), want)
    with pytest.raises(kb.ImageError, match="Invalid image size"):
        kb.imgproc.pyrdown(kb.Image(cu(f, dev)), kb.Image.zeros_cuda(kb.ImageSize(w + 3, h), c, torch.float32, dev, batch=n))


def test_build_pyramid_levels(kb, oracle, dev):
    """pyramid.rs:851-883 `test_build_pyramid_levels_and_sizes_odd_dimensions`: 5x7 -> 3x4 -> 2x2 -> 1x1."""
    src = kb.Image(cu(np.ones((7, 5, 1), np.float32), dev))
    pyr = kb.imgproc.build_pyramid(src, 3)
    assert [(p.cols(), p.rows()) for p in pyr] == [(5, 7), (3, 4), (2, 2), (1, 1)]
    for p in pyr:
        assert np.all(p.numpy() == np.float32(1.0))


# ── undistort maps on the device (SURVEY §8(f) #2) ───────────────────────────────
DIST_INTR = (577.48583984375, 652.8748779296875, 577.48583984375, 386.1428833007813)
DIST_COEF = (1.7547749280929563, 0.0097926277667284, -0.027250492945313457, 2.1092164516448975, 0.462927520275116, -0.08215277642011642,
             -0.00005457743463921361, 0.00003006766564794816)


@pytest.mark.parametrize("w,h", [(8, 4), (641, 479), (1920, 1080)])
def test_generate_correction_map_polynomial(kb, oracle, dev, w, h):
    mx, my = kb.imgproc.generate_correction_map_polynomial(DIST_INTR, DIST_COEF, kb.ImageSize(w, h), dev)
    ox, oy = oracle.generate_correction_map_polynomial(DIST_INTR, DIST_COEF, w, h)
    assert_f32_bits_or_signed_zero(mx.numpy(), ox, "map_x"); assert_f32_bits_or_signed_zero(my.numpy(), oy, "map_y")


def test_undistort_pipeline_map_then_remap(kb, oracle, dev):
    """The undistort caller of config 5: maps generated on the device feed remap on the same stream, f32 and u8."""
    w, h = 640, 480
    intr, coef = (612.3, 610.8, 320.1, 241.7), (-0.12, 0.03, 0.0, 0.0, 0.0, 0.0, 1e-4, -2e-4)
    mx, my = kb.imgproc.generate_correction_map_polynomial(intr, coef, kb.ImageSize(w, h), dev)
    ox, oy = oracle.generate_correction_map_polynomial(intr, coef, w, h)
    src = oracle.pattern_f32(w * h * 3).reshape(h, w, 3)
    dst = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.float32, dev)
    kb.imgproc.remap(kb.Image(cu(src, dev)), dst, mx, my, kb.InterpolationMode.Bilinear)
    assert_f32_bits_or_signed_zero(dst.numpy(), oracle.remap(src, ox, oy, oracle.BILINEAR), "undistort f32")


# ── host-buffer form of the camera preprocess (kb200_preprocess_host) ────────────
@pytest.mark.parametrize("fmt,mode,dw,dh", [("Nv12", "Stretch", 192, 108), ("Nv12", "Letterbox", 64, 64), ("Yuyv", "Letterbox", 100, 60), ("Rgb8", "Stretch", 77, 41)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_pipeline(kb, oracle, dev, fmt, mode, dw, dh, f16):
    """Host frames in / host tensor out must equal the device-buffer path bit for bit, across chunk boundaries of a small
    staging ring (several chunks per call, ring depth 2)."""
    w, h, n = 192, 108, 7
    nbytes = {"Nv12": w * h * 3 // 2, "Yuyv": w * h * 2, "Rgb8": w * h * 3}[fmt]
    host = torch.from_numpy(np.stack([raw_bytes(nbytes, k) for k in range(n)])).pin_memory()
    pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda())
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([host[i].to(dev) for i in range(n)], w, h, want)
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * ((nbytes + 15) // 16 * 16), dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
    got = pre.run_raw_host(host, w, h, (dw, dh), f16=f16, pipeline=pipe)
    torch.cuda.synchronize()
    h2d, d2h = pipe.last_transfer()
    assert h2d == n * nbytes and d2h == n * 3 * dw * dh * (2 if f16 else 4)
    assert torch.equal(got.view(torch.int16 if f16 else torch.int32), want.cpu().view(torch.int16 if f16 else torch.int32))
    pipe.close()


# ── cuda/fusion.rs stage vocabulary as pre-instantiated pipelines ────────────────
@pytest.mark.parametrize("chain,code", [("", 0), ("N", 1), ("G", 2), ("NG", 3), ("GN", 4)])
@pytest.mark.parametrize("sink", [0, 1])
def test_fused_pipelines(kb, oracle, dev, chain, code, sink):
    """cuda/fusion.rs:762-840 (`fused_resize_normalize_chw_matches_cpu`, `fused_novel_gray_chain`): every composable shape,
    batched, against the restated generated kernel; the reference's own tolerance is 1e-4 relative — here bit equality."""
    from kornia_rs_b200.fusion import FusedPipeline, Normalize, ReadU8RgbBilinear, RgbToGray, WriteC1F32, WriteChwF32
    sw, sh, dw, dh, n = 100, 80, 47, 33, 3
    src = np.stack([oracle.pattern_u8(sw * sh * 3, 11 + i).reshape(sh, sw, 3) for i in range(n)])
    scale, bias = [1.0 / 255.0, 0.5 / 255.0, 2.0 / 255.0], [0.1, -0.2, 0.05]
    stages = [ReadU8RgbBilinear(sw, sh, dw, dh)] + [Normalize(scale, bias) if k == "N" else RgbToGray() for k in chain] + [WriteChwF32() if sink == 0 else WriteC1F32()]
    pipe = FusedPipeline.build(stages, dw, dh)
    dst = torch.zeros((n, pipe.out_planes(), dh, dw), dtype=torch.float32, device=dev)
    pipe.launch(cu(src, dev), dst)
    assert last_kernel(kb) == "fused_pipeline_kernel"
    want = np.stack([oracle.fused_pipeline_u8(src[i], dw, dh, code, scale, bias, sink) for i in range(n)])
    assert_f32_bits_or_signed_zero(dst.cpu().numpy(), want, f"fusion chain '{chain}' sink {sink}")


def test_fused_pipeline_shape_errors(kb, dev):
    from kornia_rs_b200.fusion import FusedPipeline, FusionError, Normalize, ReadU8RgbBilinear, RgbToGray, WriteChwF32
    read = ReadU8RgbBilinear(64, 64, 32, 32)
    with pytest.raises(FusionError, match="at least a source and a sink"):
        FusedPipeline.build([read], 32, 32)
    with pytest.raises(FusionError, match="first stage must be a source"):
        FusedPipeline.build([RgbToGray(), WriteChwF32()], 32, 32)
    with pytest.raises(FusionError, match="not a pre-instantiated shape"):
        FusedPipeline.build([read, RgbToGray(), RgbToGray(), WriteChwF32()], 32, 32)
    pipe = FusedPipeline.build([read, Normalize([1, 1, 1], [0, 0, 0]), WriteChwF32()], 32, 32)
    with pytest.raises(FusionError, match="destination holds"):
        pipe.launch(torch.zeros((64, 64, 3), dtype=torch.uint8, device=dev), torch.zeros((3, 16, 16), dtype=torch.float32, device=dev))


def test_shared_reciprocal_division_is_exact(kb, dev):
    """warp_div2 (one reciprocal for the two perspective quotients) must equal two IEEE divisions bit for bit: 2^31 random
    operand triples over a wide exponent range + zero / denormal / window-edge cases, compared on the device."""
    mism = torch.zeros(1, dtype=torch.int64, device=dev)
    for seed in (1, 77):
        st = kb._lib.lib().kb200_selftest_div2(torch.cuda.current_stream(dev).cuda_stream, 1 << 30, seed, mism.data_ptr())
        assert st == 0, kb._lib.last_error()
        assert int(mism.item()) == 0, f"{int(mism.item())} operand triples differ from __fdiv_rn (seed {seed})"


# ── u8 blurs: the row-streaming kernel (round 2) and the tile kernels, named ──────
@pytest.mark.parametrize("cols,rows,c,n,k,sigma", [
    (1376, 19, 3, 2, 5, 1.5),     # several strips (4128-byte rows), Q8 5x5
    (3840, 40, 3, 1, 5, 1.5),     # the bench geometry's row length
    (256, 40, 1, 2, 3, 0.8),      # binomial [1,2,1]/4 path, one partial strip
    (256, 33, 1, 1, 7, 2.0),      # 7 taps
    (640, 33, 4, 2, 7, 2.5),      # C = 4, 12-byte halo
    (1024, 70, 4, 1, 3, 2.0),     # k = 3 outside the binomial sigma window -> Q8
    (96, 300, 3, 1, 5, 1.2),      # one short strip (288-byte rows), many row chunks
])
def test_gaussian_blur_u8_stream(kb, oracle, dev, cols, rows, c, n, k, sigma):
    assert (cols * c) % 16 == 0
    src = np.stack([oracle.pattern_u8(rows * cols * c, 0x51 + i).reshape(rows, cols, c) for i in range(n)])
    d = kb.Image(torch.full((n, rows, cols, c), 0xCD, dtype=torch.uint8, device=dev))
    kb.imgproc.gaussian_blur_u8(kb.Image(cu(src, dev)), d, (k, k), (sigma, sigma))
    assert last_kernel(kb) == "blur_u8_stream_kernel", last_kernel(kb)
    want = np.stack([oracle.gaussian_blur_u8(src[i], (k, k), (sigma, sigma)) for i in range(n)])
    np.testing.assert_array_equal(d.numpy(), want)
    # the tile kernel on the same input (knob b = 3 disables streaming) must agree too
    with knobs(kb, {"b": 3}):
        d2 = kb.Image.zeros_cuda(kb.ImageSize(cols, rows), c, torch.uint8, dev, batch=n)
        kb.imgproc.gaussian_blur_u8(kb.Image(cu(src, dev)), d2, (k, k), (sigma, sigma))
        assert last_kernel(kb) in ("blur_u8_tile_w_kernel", "blur_u8_tile_kernel")
    np.testing.assert_array_equal(d2.numpy(), want)


def test_box_blur_u8_stream_and_full_4k(kb, oracle, dev):
    src = oracle.pattern_u8(64 * 512 * 3, 0x91).reshape(64, 512, 3)
    d = kb.Image.zeros_cuda(kb.ImageSize(512, 64), 3, torch.uint8, dev)
    kb.imgproc.box_blur_u8(kb.Image(cu(src, dev)), d, (5, 5))
    assert last_kernel(kb) == "blur_u8_stream_kernel"
    np.testing.assert_array_equal(d.numpy(), oracle.box_blur_u8(src, (5, 5)))
    # the bench row at full size: 4K RGB u8, gaussian 5x5 sigma 1.5 — every byte
    w, h = 3840, 2160
    big = oracle.pattern_u8(w * h * 3, 0x92).reshape(h, w, 3)
    d4 = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev)
    kb.imgproc.gaussian_blur_u8(kb.Image(cu(big, dev)), d4, (5, 5), (1.5, 1.5))
    assert last_kernel(kb) == "blur_u8_stream_kernel"
    np.testing.assert_array_equal(d4.numpy(), oracle.gaussian_blur_u8(big, (5, 5), (1.5, 1.5)))


@pytest.mark.parametrize("mode", ["Bilinear", "Nearest"])
def test_warp_gather64_fallback(kb, oracle, dev, mode):
    """The >= 2^31-element fallback (64-bit indexing) forced on a small image: same shared arithmetic, same bits."""
    sw, sh = 129, 97
    src = oracle.pattern_f32(sw * sh * 3).reshape(sh, sw, 3)
    h = [1.03, 0.05, -3.0, -0.02, 0.97, 4.0, 2.0 / (97 * 129), 1.5 / (129 * 97), 1.0]
    m = rot(kb, sw, sh, 30.0)
    om = oracle.BILINEAR if mode == "Bilinear" else oracle.NEAREST
    with knobs(kb, {"warp.path": 4}):
        dst = kb.Image.zeros_cuda(kb.ImageSize(sw, sh), 3, torch.float32, dev)
        kb.imgproc.warp_perspective(kb.Image(cu(src, dev)), dst, h, kb.InterpolationMode[mode])
        assert last_kernel(kb) == "warp_gather64_kernel"
        assert_f32_bits_or_signed_zero(dst.numpy(), oracle.warp_perspective_f32(src, h, sw, sh, om), "gather64 perspective")
        kb.imgproc.warp_affine(kb.Image(cu(src, dev)), dst, m, kb.InterpolationMode[mode])
        assert last_kernel(kb) == "warp_gather64_kernel"
        assert_f32_bits_or_signed_zero(dst.numpy(), oracle.warp_affine_f32(src, m, sw, sh, om), "gather64 affine")


# ── remap f32 bilinear through the lean gather kernel (round 2, second pass) ──
@pytest.mark.parametrize("kind", ["identity", "swirl", "random"])
@pytest.mark.parametrize("dw,dh", [(64, 40), (57, 39), (132, 70)])
def test_remap_f32_lean(kb, oracle, dev, kind, dw, dh):
    """remap (bilinear) = the warps' lean gather with coordinates from the maps: fast path / general path / STG stores / the
    thread-per-pixel kernel (knob a = 0 / 4 / 5 / 6) against the oracle; maps with NaN, inf, out-of-range and last-row/column taps."""
    n, sw, sh = 2, 64, 48
    rng = np.random.default_rng(31)
    mx, my = _remap_maps(dw, dh, sw, sh, kind, rng)
    mxi, myi = kb.Image(cu(mx[..., None], dev)), kb.Image(cu(my[..., None], dev))
    src = np.stack([oracle.pattern_f32(sw * sh * 3, 0x291 + i).reshape(sh, sw, 3) for i in range(n)])
    want = np.stack([oracle.remap(src[i], mx, my, 1) for i in range(n)])
    stg = "" if dw % 4 == 0 else "/stg"
    for a, kernel in ((0, "remap_lean_kernel" + stg), (4, "remap_lean_kernel/general" + stg), (5, "remap_lean_kernel/stg"), (6, "remap_f32_c3_kernel")):
        with knobs(kb, {"a": a}):
            d = kb.Image(torch.full((n, dh, dw, 3), float("nan"), dtype=torch.float32, device=dev))
            kb.imgproc.remap(kb.Image(cu(src, dev)), d, mxi, myi, kb.InterpolationMode.Bilinear)
            assert last_kernel(kb) == kernel, last_kernel(kb)
        assert_f32_bits_or_signed_zero(d.numpy(), want, f"remap lean {kind} {dw}x{dh} a={a}")


# ── u8 warps / remap: interior fast path (round 2, second pass) ───────────────
@pytest.mark.parametrize("sw,sh", [(640, 360), (389, 211), (132, 35)])
def test_u8_interior_fast_path(kb, oracle, dev, sw, sh):
    """q10_blend_c3_interior (u8_sampler.cuh) is taken by warps whose 32 pixels are all interior (taps inside, two rows of
    slack below); everything else goes through the clamped sampler.  Half-pixel shifts, a mild homography and a rotation put
    the fast/general seam on the last rows and columns; knob b = 1 (no word taps: general sampler everywhere) must agree."""
    n = 2
    src = np.stack([oracle.pattern_u8(sw * sh * 3, 0x331 + i).reshape(sh, sw, 3) for i in range(n)])
    s_img = kb.Image(cu(src, dev))
    affines = [[1, 0, 0.5, 0, 1, 0.5], [1, 0, -0.5, 0, 1, -1.5], [1.01, 0.02, -3.0, -0.015, 0.99, 2.5], [0.5, 0, 0, 0, 0.5, 0]]
    persps = [[1, 0, 0.5, 0, 1, 0.5, 0, 0, 1], [1.02, 0.03, -5.0, -0.03, 1.01, 2.0, 0.00005, 0.00003, 1.0], [-1.0, 0, sw - 1.5, 0, -1.0, sh - 1.5, 0, 0, -1.0]]
    y, x = np.meshgrid(np.arange(sh, dtype=np.float32), np.arange(sw, dtype=np.float32), indexing="ij")
    maps = [(x + np.float32(0.5), y + np.float32(0.5)), (x * np.float32(0.999) + np.float32(0.25), y * np.float32(1.001) - np.float32(0.125))]
    for b in (0, 1):
        with knobs(kb, {"b": b}):
            for m in affines:
                d = kb.Image(torch.full((n, sh, sw, 3), 0xCD, dtype=torch.uint8, device=dev))
                kb.imgproc.warp_affine_u8(s_img, d, m)
                np.testing.assert_array_equal(d.numpy(), np.stack([oracle.warp_affine_u8(src[i], sw, sh, m) for i in range(n)]), err_msg=f"affine {m} b={b}")
            for hm in persps:
                d = kb.Image(torch.full((n, sh, sw, 3), 0xCD, dtype=torch.uint8, device=dev))
                kb.imgproc.warp_perspective_u8(s_img, d, hm)
                np.testing.assert_array_equal(d.numpy(), np.stack([oracle.warp_perspective_u8(src[i], sw, sh, hm) for i in range(n)]), err_msg=f"perspective {hm} b={b}")
            for mx, my in maps:
                d = kb.Image(torch.full((n, sh, sw, 3), 0xCD, dtype=torch.uint8, device=dev))
                kb.imgproc.remap_u8(s_img, d, kb.Image(cu(mx[..., None], dev)), kb.Image(cu(my[..., None], dev)), kb.InterpolationMode.Bilinear)
                np.testing.assert_array_equal(d.numpy(), np.stack([oracle.remap(src[i], mx, my, 1) for i in range(n)]), err_msg=f"remap b={b}")


# ── randomized geometry sweep: every f32 / u8 sampler dispatch against the oracle ─────────────
def _rand_homography(rng, sw, sh, strength):
    """Identity + random affine and projective perturbations scaled by `strength` (0 .. 1)."""
    a = np.eye(3)
    a[:2, :2] += rng.uniform(-0.35, 0.35, (2, 2)) * strength
    a[:2, 2] = rng.uniform(-0.2, 0.2, 2) * np.array([sw, sh]) * strength
    a[2, :2] = rng.uniform(-1.0, 1.0, 2) * strength * 0.6 / max(sw, sh)
    return [float(v) for v in a.reshape(-1)]


@pytest.mark.parametrize("seed", range(12))
def test_random_geometry_sweep(kb, oracle, dev, seed):
    """Random source / destination sizes (multiples of 32, of 8, of 4, odd) and random maps from near-identity to strongly
    projective: warp_perspective / warp_affine f32 (bilinear, nearest), their u8 twins and remap (f32, u8) must all equal the
    oracle bit for bit, whichever kernel the dispatcher picks (lean fast / general path, TMA tile or STG stores, tiled, u8
    interior sampler)."""
    rng = np.random.default_rng(1000 + seed)
    sw, sh = int(rng.choice([64, 96, 131, 200, 256, 333])), int(rng.choice([48, 61, 96, 120, 161]))
    dw, dh = int(rng.choice([32, 64, 100, 132, 257, 320])), int(rng.choice([24, 40, 56, 75, 128]))
    n = int(rng.integers(1, 4))
    strength = float(rng.choice([0.02, 0.1, 0.4, 1.0]))
    h = _rand_homography(rng, sw, sh, strength)
    m = h[:6]
    src = oracle.pattern_f32(n * sw * sh * 3, 0x5000 + seed).reshape(n, sh, sw, 3)
    t = kb.Image(cu(src, dev))
    for mode, om in (("Bilinear", oracle.BILINEAR), ("Nearest", oracle.NEAREST)):
        d = kb.Image.from_size_val(kb.ImageSize(dw, dh), 7.0, 3, torch.float32, dev, batch=n)
        kb.imgproc.warp_perspective(t, d, h, kb.InterpolationMode[mode])
        k = last_kernel(kb)
        assert_f32_bits_or_signed_zero(d.numpy(), np.stack([oracle.warp_perspective_f32(src[i], h, dw, dh, om) for i in range(n)]), f"seed {seed} perspective {mode} {sw}x{sh}->{dw}x{dh} ({k})")
        d = kb.Image.from_size_val(kb.ImageSize(dw, dh), 7.0, 3, torch.float32, dev, batch=n)
        kb.imgproc.warp_affine(t, d, m, kb.InterpolationMode[mode])
        k = last_kernel(kb)
        assert_f32_bits_or_signed_zero(d.numpy(), np.stack([oracle.warp_affine_f32(src[i], m, dw, dh, om) for i in range(n)]), f"seed {seed} affine {mode} {sw}x{sh}->{dw}x{dh} ({k})")
    src8 = np.stack([oracle.pattern_u8(sw * sh * 3, 0x6000 + seed + i).reshape(sh, sw, 3) for i in range(n)])
    t8 = kb.Image(cu(src8, dev))
    d8 = kb.Image(torch.full((n, dh, dw, 3), 0xCD, dtype=torch.uint8, device=dev))
    kb.imgproc.warp_perspective_u8(t8, d8, h)
    np.testing.assert_array_equal(d8.numpy(), np.stack([oracle.warp_perspective_u8(src8[i], dw, dh, h) for i in range(n)]), err_msg=f"seed {seed} perspective u8")
    d8 = kb.Image(torch.full((n, dh, dw, 3), 0xCD, dtype=torch.uint8, device=dev))
    kb.imgproc.warp_affine_u8(t8, d8, m)
    np.testing.assert_array_equal(d8.numpy(), np.stack([oracle.warp_affine_u8(src8[i], dw, dh, m) for i in range(n)]), err_msg=f"seed {seed} affine u8")
    # remap through the same homography's coordinate field, with a few holes
    hi = np.linalg.inv(np.array(h, dtype=np.float64).reshape(3, 3))
    yy, xx = np.meshgrid(np.arange(dh, dtype=np.float64), np.arange(dw, dtype=np.float64), indexing="ij")
    wq = hi[2, 0] * xx + hi[2, 1] * yy + hi[2, 2]
    mx = ((hi[0, 0] * xx + hi[0, 1] * yy + hi[0, 2]) / wq).astype(np.float32)
    my = ((hi[1, 0] * xx + hi[1, 1] * yy + hi[1, 2]) / wq).astype(np.float32)
    mx[0, 0] = np.nan; my[dh // 2, dw // 2] = np.inf; mx[dh - 1, dw - 1] = sw - 1.0; my[dh - 1, 0] = sh - 1.0
    mxi, myi = kb.Image(cu(mx[..., None], dev)), kb.Image(cu(my[..., None], dev))
    d = kb.Image(torch.full((n, dh, dw, 3), float("nan"), dtype=torch.float32, device=dev))
    kb.imgproc.remap(t, d, mxi, myi, kb.InterpolationMode.Bilinear)
    assert_f32_bits_or_signed_zero(d.numpy(), np.stack([oracle.remap(src[i], mx, my, 1) for i in range(n)]), f"seed {seed} remap f32 ({last_kernel(kb)})")
    d8 = kb.Image(torch.full((n, dh, dw, 3), 0xCD, dtype=torch.uint8, device=dev))
    kb.imgproc.remap_u8(t8, d8, mxi, myi, kb.InterpolationMode.Bilinear)
    np.testing.assert_array_equal(d8.numpy(), np.stack([oracle.remap(src8[i], mx, my, 1) for i in range(n)]), err_msg=f"seed {seed} remap u8")
