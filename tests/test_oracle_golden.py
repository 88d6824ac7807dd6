"""Pins the CPU oracle against the reference's OWN known-answer tests.

Every test cites the reference test it transcribes (paths relative to
kornia-rs's crates/kornia-imgproc/src).  The Rust reference cannot run here (no cargo), so
these vectors — plus the cv2 fixtures the reference declares byte-parity with — are what makes the
oracle "pinned" (SURVEY §8(c)).  CPU only: no GPU, no access to the reference's sources at run time.
"""
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def f32(*v):
    return np.array(v, dtype=np.float32)


# ── generators ───────────────────────────────────────────────────────────────
def test_pattern_u8_prefix_and_lcg(oracle):
    # cuda/color/mod.rs:303-316
    p = oracle.pattern_u8(20)
    assert list(p[:15]) == [0, 255, 255, 0, 0, 0, 255, 255, 255, 1, 254, 128, 128, 128, 64]
    state = 0x12345678
    for i in range(15, 20):
        state = (state * 1664525 + 1013904223) & 0xFFFFFFFF
        assert p[i] == state >> 24
    assert oracle.pattern_u8(7).tolist() == [0, 255, 255, 0, 0, 0, 255]
    pf = oracle.pattern_f32(20)
    assert pf[1] == 1.0 and pf[0] == 0.0
    np.testing.assert_array_equal(pf, p.astype(np.float32) / np.float32(255.0))


# ── a1 resize ────────────────────────────────────────────────────────────────
def test_resize_smoke_ch3(oracle):
    # resize/mod.rs:447-489
    img = np.arange(3 * 4 * 3, dtype=np.float32).reshape(4, 3, 3)
    out = oracle.resize_f32(img, 2, 3, oracle.BILINEAR)
    expected = f32(2.25, 3.25, 4.25, 6.75, 7.75, 8.75, 14.25, 15.25, 16.25, 18.75, 19.75, 20.75, 26.25, 27.25,
                   28.25, 30.75, 31.75, 32.75)
    assert np.abs(out.reshape(-1) - expected).max() < 1e-4


def test_resize_same_size_is_copy(oracle):
    # resize/mod.rs:134-137 and resize_smoke_ch1 :491-519
    img = f32(0, 1, 2, 3, 4, 5).reshape(3, 2, 1)
    np.testing.assert_array_equal(oracle.resize_f32(img, 2, 3, oracle.NEAREST), img)


def test_pixel_mapping_coeffs_table(oracle):
    # cuda/resize.rs:930-940 — HalfPixel (a, b) = (src/dst, 0.5a-0.5): checked through the sampler:
    # 4 -> 2 samples at 0.5, 2.5 ; 2 -> 4 samples at clamp(-0.25)=0, 0.25, 0.75, 1 (clamped 1.25)
    ramp = f32(0, 10, 20, 30).reshape(1, 4, 1)
    np.testing.assert_array_equal(oracle.resize_f32(ramp, 2, 1).reshape(-1), f32(5.0, 25.0))
    ramp2 = f32(0, 8).reshape(1, 2, 1)
    np.testing.assert_array_equal(oracle.resize_f32(ramp2, 4, 1).reshape(-1), f32(0.0, 2.0, 6.0, 8.0))


# ── a2 fused resize ──────────────────────────────────────────────────────────
@pytest.mark.parametrize("leaf", [0, 1, 2])
def test_fused_2x_normalize_matches_f64_reference(oracle, leaf):
    # resize/fused.rs:1047-1087
    dw, dh = 37, 5
    sw, sh = 2 * dw, 2 * dh
    src = np.array([(i * 7 + 3) % 256 for i in range(sh * sw * 3)], np.uint8).reshape(sh, sw, 3)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    scale, bias = oracle.normalize_params_from_mean_std(mean, std)
    out = oracle.resize_normalize_u8_to_f32_chw(src, dw, dh, scale, bias, leaf)
    s = src.astype(np.float64)
    avg = (s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2]) / 4.0
    m64 = np.array(mean, np.float32).astype(np.float64)
    s64 = np.array(std, np.float32).astype(np.float64)
    expect = ((avg / 255.0 - m64) / s64).transpose(2, 0, 1)
    assert np.abs(out - expect).max() < 1e-4


def test_fused_2x_zero_input(oracle):
    # resize/fused.rs:1091-1121
    dw, dh = 16, 2
    src = np.zeros((2 * dh, 2 * dw, 3), np.uint8)
    mean, std = [0.5, 0.25, 0.75], [0.5, 0.25, 0.75]
    scale, bias = oracle.normalize_params_from_mean_std(mean, std)
    out = oracle.resize_normalize_u8_to_f32_chw(src, dw, dh, scale, bias)
    for ch in range(3):
        assert np.abs(out[ch] - (-mean[ch] / std[ch])).max() < 1e-6


@pytest.mark.parametrize("leaf", [0, 1, 2])
def test_fused_bilinear_general_matches_f64_reference(oracle, leaf):
    # resize/fused.rs:1125-1170
    sw, sh, dw, dh = 60, 40, 37, 23
    src = np.array([(i * 13 + 7) % 256 for i in range(sh * sw * 3)], np.uint8).reshape(sh, sw, 3)
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    scale, bias = oracle.normalize_params_from_mean_std(mean, std)
    out = oracle.resize_normalize_u8_to_f32_chw(src, dw, dh, scale, bias, leaf)
    sx, sy = sw / dw, sh / dh
    s = src.astype(np.float64)
    for dy in range(dh):
        fy = max((dy + 0.5) * sy - 0.5, 0.0)
        y0 = min(int(fy), sh - 1)
        y1 = min(y0 + 1, sh - 1)
        wy = fy - y0
        for dx in range(dw):
            fx = max((dx + 0.5) * sx - 0.5, 0.0)
            x0 = min(int(fx), sw - 1)
            x1 = min(x0 + 1, sw - 1)
            wx = fx - x0
            for c in range(3):
                top = s[y0, x0, c] + wx * (s[y0, x1, c] - s[y0, x0, c])
                bot = s[y1, x0, c] + wx * (s[y1, x1, c] - s[y1, x0, c])
                val = top + wy * (bot - top)
                expect = (val / 255.0 - float(np.float32(mean[c]))) / float(np.float32(std[c]))
                assert abs(out[c, dy, dx] - expect) < 1e-3


def test_fused_bilinear_dispatches_2x(oracle):
    # resize/fused.rs:1173-1187 — exact 2x goes down the box path: out = sum*0.25*scale + bias
    dw, dh = 20, 12
    sw, sh = 2 * dw, 2 * dh
    src = np.array([i % 251 for i in range(sh * sw * 3)], np.uint8).reshape(sh, sw, 3)
    scale, bias = oracle.normalize_params_from_mean_std([0.5, 0.4, 0.3], [0.25, 0.2, 0.3])
    out = oracle.resize_normalize_u8_to_f32_chw(src, dw, dh, scale, bias, oracle.LEAF_SCALAR)
    s = src.astype(np.uint32)
    ssum = (s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2]).astype(np.float32)
    expect = (ssum * (scale * np.float32(0.25)) + bias).transpose(2, 0, 1)
    np.testing.assert_array_equal(out, expect)


# ── a3 u8 bilinear Q14 ───────────────────────────────────────────────────────
def test_bilinear_u8_q14_independent_python(oracle):
    # resize/bilinear.rs:25-38 + resize/kernels.rs:1141-1166, restated independently in Python ints
    import math

    sw, sh, dw, dh, C = 13, 9, 7, 5, 3
    src = oracle.pattern_u8(sw * sh * C).reshape(sh, sw, C)
    out = oracle.resize_bilinear_u8(src, dw, dh)

    def tap(i, scale, n):
        s = (i + 0.5) * scale - 0.5
        i0 = math.floor(s)
        f = s - i0
        if i0 < 0:
            i0, f = 0, 0.0
        elif i0 >= n - 1:
            i0, f = n - 2, 1.0
        fq = min(int(math.floor(f * 16384 + 0.5)), 16384)
        return i0, fq

    for y in range(dh):
        yi, fy = tap(y, sh / dh, sh)
        for x in range(dw):
            xi, fx = tap(x, sw / dw, sw)
            for c in range(C):
                p00, p01 = int(src[yi, xi, c]), int(src[yi, xi + 1, c])
                p10, p11 = int(src[yi + 1, xi, c]), int(src[yi + 1, xi + 1, c])
                top = p00 * (16384 - fx) + p01 * fx
                bot = p10 * (16384 - fx) + p11 * fx
                want = (top * (16384 - fy) + bot * fy + (1 << 27)) >> 28
                assert out[y, x, c] == want
    with pytest.raises(ValueError):
        oracle.resize_bilinear_u8(np.zeros((1, 5, 3), np.uint8), 3, 3)  # resize/mod.rs:318-320


# ── a4 warp_affine ───────────────────────────────────────────────────────────
def test_span_units(oracle):
    # warp/span.rs:95-138
    sp = lambda a, b, ge: oracle.constrain_span(a, b, ge, 1e-6, 0, 10)
    assert sp(1.0, -3.0, True) == (3, 10)
    assert sp(-1.0, 3.0, True) == (0, 4)
    assert sp(1.0, -3.0, False) == (0, 3)
    assert sp(-1.0, 3.0, False) == (4, 10)
    assert sp(1.0, -2.5, True) == (3, 10)
    assert sp(-1.0, 2.5, True) == (0, 3)
    assert sp(1.0, -2.5, False) == (0, 3)
    assert sp(-1.0, 2.5, False) == (3, 10)
    assert sp(0.0, 1.0, True) == (0, 10)
    assert sp(0.0, -1.0, True) == (0, 0)
    assert sp(0.0, -1.0, False) == (0, 10)
    assert sp(0.0, 1.0, False) == (0, 0)
    assert oracle.affine_valid_span([-1.0, 3.0, 4.0, 0.0, 0.5, 2.0], 4, 1e-6) == (0, 4)


def test_warp_affine_edge_flip_nearest(oracle):
    # warp/affine.rs:470-495
    src = f32(1, 2, 3, 4, 5, 6, 7, 8).reshape(2, 4, 1)
    init = np.full((2, 4, 1), -1.0, np.float32)
    out = oracle.warp_affine_f32(src, [-1.0, 0.0, 3.0, 0.0, 1.0, 0.0], 4, 2, oracle.NEAREST, dst_init=init)
    np.testing.assert_array_equal(out.reshape(-1), f32(4, 3, 2, 1, 8, 7, 6, 5))


def test_warp_affine_identity_and_rot90(oracle):
    # warp/affine.rs:584-612, :615-645
    img = np.arange(20, dtype=np.float32).reshape(5, 4, 1)
    out = oracle.warp_affine_f32(img, [1.0, 0.0, 0.0, 0.0, 1.0, 0.0], 4, 5, oracle.NEAREST)
    np.testing.assert_array_equal(out, img)
    img2 = f32(0, 1, 2, 3).reshape(2, 2, 1)
    m = oracle.get_rotation_matrix2d((0.5, 0.5), 90.0, 1.0)
    out = oracle.warp_affine_f32(img2, m, 2, 2, oracle.NEAREST)
    np.testing.assert_array_equal(out.reshape(-1), f32(1, 3, 0, 2))


def test_invert_affine(oracle):
    # warp/affine.rs:18-38 — identity and a translation
    np.testing.assert_array_equal(oracle.invert_affine_transform([1, 0, 0, 0, 1, 0]), f32(1, 0, -0.0, 0, 1, -0.0))
    inv = oracle.invert_affine_transform([1, 0, 2, 0, 1, 3])
    np.testing.assert_array_equal(inv, f32(1, -0.0, -2, -0.0, 1, -3))


# ── a5 warp_perspective ──────────────────────────────────────────────────────
def test_invert_homography_cases(oracle):
    # warp/perspective.rs:377-430
    inv = oracle.invert_homography([1, 0, 2, 0, 1, 3, 0, 0, 1])
    assert np.abs(inv - f32(1, 0, -2, 0, 1, -3, 0, 0, 1)).max() < 1e-6
    h = f32(1.02, 0.03, -5.0, -0.01, 0.99, 2.0, 0.00005, 0.00003, 1.0)
    inv = oracle.invert_homography(h)
    prod = h.reshape(3, 3).astype(np.float64) @ inv.reshape(3, 3).astype(np.float64)
    assert np.abs(prod - np.eye(3)).max() < 1e-5
    assert oracle.invert_homography(np.zeros(9)) is None
    assert oracle.invert_homography([1, 2, 3, 2, 4, 6, 3, 6, 9]) is None
    small = f32(1, 0, 2, 0, 1, 3, 0, 0, 1) * np.float32(0.001)
    assert oracle.invert_homography(small) is not None
    # inverse_perspective_matrix :432-439 — exact
    inv = oracle.invert_homography([1, 0, -1, 0, 1, 1, 0, 0, 1])
    np.testing.assert_array_equal(inv, f32(1, 0, 1, 0, 1, -1, 0, 0, 1))


def test_warp_perspective_hflip_resize_shift(oracle):
    # warp/perspective.rs:499-535 (hflip)
    img = f32(0, 1, 2, 3, 4, 5).reshape(3, 2, 1)
    out = oracle.warp_perspective_f32(img, [-1, 0, 1, 0, 1, 0, 0, 0, 1], 2, 3)
    np.testing.assert_array_equal(out.reshape(-1), f32(1, 0, 3, 2, 5, 4))
    # :537-589 (resize equivalence, bit exact) ; :591-633 (shift)
    img = np.arange(16, dtype=np.float32).reshape(4, 4, 1)
    out = oracle.warp_perspective_f32(img, [0.5, 0, -0.25, 0, 0.5, -0.25, 0, 0, 1], 2, 2)
    np.testing.assert_array_equal(out.reshape(-1), f32(2.5, 4.5, 10.5, 12.5))
    np.testing.assert_array_equal(out, oracle.resize_f32(img, 2, 2))
    out = oracle.warp_perspective_f32(img, [1, 0, -1, 0, 1, 0, 0, 0, 1], 4, 4)
    np.testing.assert_array_equal(out.reshape(-1), f32(1, 2, 3, 0, 5, 6, 7, 0, 9, 10, 11, 0, 13, 14, 15, 0))
    with pytest.raises(ValueError):
        oracle.warp_perspective_f32(img, np.zeros(9), 4, 4)


# ── a6/a7 filters ────────────────────────────────────────────────────────────
def test_gaussian_kernel_1d_exact(oracle):
    # filter/kernels.rs:201-216 — exact f32 equality (pins libm expf + the sum/divide order)
    k = oracle.gaussian_kernel_1d(5, 0.5)
    np.testing.assert_array_equal(k, f32(0.00026386508, 0.10645077, 0.78657067, 0.10645077, 0.00026386508))


def test_sobel_kernels(oracle):
    # filter/kernels.rs:176-189
    kx, ky = oracle.sobel_kernel_1d(3)
    assert kx.tolist() == [-1, 0, 1] and ky.tolist() == [1, 2, 1]
    kx, ky = oracle.sobel_kernel_1d(5)
    assert kx.tolist() == [-1, -2, 0, 2, 1] and ky.tolist() == [1, 4, 6, 4, 1]
    with pytest.raises(ValueError):
        oracle.sobel_kernel_1d(7)


def test_separable_impulse(oracle):
    # filter/separable_filter.rs:264-303
    img = np.zeros((5, 5, 1), np.float32)
    img[2, 2, 0] = 1.0
    out = oracle.separable_filter(img, [1, 1, 1], [1, 1, 1])
    want = np.zeros((5, 5), np.float32)
    want[1:4, 1:4] = 1.0
    np.testing.assert_array_equal(out[:, :, 0], want)
    assert out.sum() == 9.0


def test_gaussian_blur_exact_outputs(oracle):
    # filter/ops.rs:2184-2262 — three exact (assert_eq!) 5x5 outputs
    img = np.arange(25, dtype=np.float32).reshape(5, 5, 1)
    out = oracle.gaussian_blur(img, (3, 3), (0.5, 0.5)).reshape(-1)
    np.testing.assert_array_equal(out, f32(
        0.57097936, 1.4260278, 2.3195207, 3.213014, 3.5739717, 4.5739717, 5.999999, 7.0, 7.999999, 7.9349294,
        9.041435, 10.999999, 12.0, 12.999998, 12.402394, 13.5089, 15.999998, 17.0, 17.999996, 16.86986,
        15.58594, 18.230816, 19.124311, 20.017801, 18.588936))
    out = oracle.gaussian_blur(img, (0, 0), (0.5, 0.5)).reshape(-1)
    np.testing.assert_array_equal(out, f32(
        0.573374, 1.4282724, 2.3214629, 3.2134287, 3.5740836, 4.5745554, 5.999999, 7.000791, 7.997888, 7.9328527,
        9.039831, 10.997623, 11.999999, 12.996041, 12.399015, 13.500337, 15.989445, 16.992872, 17.987333,
        16.858635, 15.576923, 18.21976, 19.117384, 20.004917, 18.577633))
    out = oracle.gaussian_blur(img, (3, 3), (0.0, 0.0)).reshape(-1)
    np.testing.assert_array_equal(out, f32(
        0.002010752, 1.001341, 2.001006, 3.0006707, 3.9986594, 4.998659, 6.0, 7.0000005, 8.0, 8.996648,
        9.996984, 11.0, 12.000002, 13.0, 13.994974, 14.995307, 16.0, 17.0, 18.000002, 18.9933,
        19.985254, 20.991283, 21.990952, 22.990616, 23.981903))
    with pytest.raises(ValueError):
        oracle.gaussian_blur(img, (2, 3), (1.0, 1.0))  # even kernel -> InvalidSigmaValue ops.rs:138-140
    assert oracle.gaussian_resolve(0, 0, 1.5, 0.0) == (13, 13, 1.5, 1.5)  # auto-k = 2*round(4σ)+1 | 1


def test_sobel_composition(oracle):
    # filter/ops.rs:187-200: gx = sep(kx,ky), gy = sep(ky,kx), sqrt(gx²+gy²)
    img = oracle.pattern_f32(11 * 7 * 3).reshape(7, 11, 3)
    kx, ky = oracle.sobel_kernel_1d(3)
    gx = oracle.separable_filter(img, kx, ky)
    gy = oracle.separable_filter(img, ky, kx)
    np.testing.assert_array_equal(oracle.sobel(img, 3), np.sqrt(gx * gx + gy * gy, dtype=np.float32))
    # the multi-threaded variant is arithmetic-identical
    np.testing.assert_array_equal(oracle.sobel(img, 3, mt=True), oracle.sobel(img, 3))


# ── a8 gray ──────────────────────────────────────────────────────────────────
def test_gray_regression(oracle):
    # color/gray/mod.rs:270-301
    img = f32(1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0).reshape(3, 2, 3)
    for leaf in (0, 1):
        out = oracle.gray_from_rgb_f32(img, leaf).reshape(-1)
        assert np.abs(out - f32(0.299, 0.587, 0.114, 0, 0, 0)).max() < 1e-6


def test_gray_u8_q14(oracle):
    # color/gray/kernels.rs:229-238
    src = oracle.pattern_u8(3 * 1000).reshape(1, 1000, 3)
    out = oracle.gray_from_rgb_u8(src).reshape(-1)
    s = src.reshape(-1, 3).astype(np.uint32)
    want = ((4899 * s[:, 0] + 9617 * s[:, 1] + 1868 * s[:, 2] + 8192) >> 14).astype(np.uint8)
    np.testing.assert_array_equal(out, want)
    assert out[0] == ((4899 * 0 + 9617 * 255 + 1868 * 255 + 8192) >> 14)


# ── a9 NV12 / YUYV ───────────────────────────────────────────────────────────
def _decode_px_py(y, u, v):
    yy = max(y - 16, 0) * 1220542
    u -= 128
    v -= 128
    b = (yy + 2116026 * u + (1 << 19)) >> 20
    g = (yy - 409993 * u - 852492 * v + (1 << 19)) >> 20
    r = (yy + 1673527 * v + (1 << 19)) >> 20
    c = lambda t: min(max(t, 0), 255)
    return c(r), c(g), c(b)


def test_nv12_reference_generators(oracle):
    # color/yuv/kernels.rs:2078-2105 and :2108-2150 (NV12 leg), independent per-pixel reference
    for (w, h, yg, ug) in [(4, 4, lambda v: (v * 9 + 16) & 0xFF, lambda v: (v * 5 + 100) & 0xFF),
                           (64, 6, lambda i: (i * 7 + 16) % 240, lambda i: (i * 5 + 90) % 250),
                           (70, 4, lambda i: (i * 7 + 16) % 240, lambda i: (i * 5 + 90) % 250)]:
        y = [yg(i) for i in range(w * h)]
        uv = [ug(i) for i in range(w * h // 2)]
        out = oracle.rgb_from_nv12(np.array(y + uv, np.uint8), w, h)
        cw = w // 2
        for row in range(h):
            for col in range(w):
                idx = (row // 2) * cw * 2 + (col // 2) * 2
                assert tuple(out[row, col]) == _decode_px_py(y[row * w + col], uv[idx], uv[idx + 1])


def test_nv12_and_yuyv_match_cv2_fixtures(oracle):
    # SURVEY §8(c): cv2.COLOR_YUV2RGB_NV12 equals the Q20 formula bit-for-bit; fixtures made by
    # tests/golden/make_fixtures.py
    z = np.load(os.path.join(GOLD, "nv12_cv2.npz"))
    for k in "abcd":
        w, h = z[f"{k}_wh"]
        np.testing.assert_array_equal(oracle.rgb_from_nv12(z[f"{k}_raw"], int(w), int(h)), z[f"{k}_rgb"])
    z = np.load(os.path.join(GOLD, "yuyv_cv2.npz"))
    for k in "abc":
        w, h = z[f"{k}_wh"]
        np.testing.assert_array_equal(oracle.rgb_from_yuyv(z[f"{k}_raw"], int(w), int(h)), z[f"{k}_rgb"])
    # packed422_known_gray yuv/kernels.rs:2068-2075
    assert oracle.rgb_from_yuyv(np.array([16, 128, 16, 128], np.uint8), 2, 1).reshape(-1).tolist() == [0] * 6
    with pytest.raises(ValueError):
        oracle.rgb_from_nv12(np.zeros(100, np.uint8), 5, 4)


# ── a10 normalize / a11 std_mean ─────────────────────────────────────────────
def test_normalize_family(oracle):
    # normalize.rs:426-462, :481-515, :518-539, :583-620
    img = f32(0, 1, 0, 1, 2, 3, 0, 1, 0, 1, 2, 3).reshape(2, 2, 3)
    out = oracle.normalize_mean_std(img, [0.5, 1.0, 0.5], [1.0, 1.0, 1.0]).reshape(-1)
    assert np.abs(out - f32(-0.5, 0, -0.5, 0.5, 1, 2.5, -0.5, 0, -0.5, 0.5, 1, 2.5)).max() < 1e-6
    assert oracle.find_min_max(img) == (0.0, 3.0)
    out = oracle.normalize_min_max(img, 0.0, 1.0).reshape(-1)
    want = f32(0, 0.33333334, 0, 0.33333334, 0.6666667, 1, 0, 0.33333334, 0, 0.33333334, 0.6666667, 1)
    assert np.abs(out - want).max() < 1e-6
    src = np.array([0, 128, 255, 100, 200, 50], np.uint8).reshape(1, 2, 3)
    out = oracle.normalize_rgb_u8(src, [1 / 255.0] * 3, [0.0] * 3).reshape(-1)
    assert np.abs(out - f32(0, 128 / 255, 1, 100 / 255, 200 / 255, 50 / 255)).max() < 1e-5
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    scale = [1 / (s * 255) for s in std]
    off = [-m / s for m, s in zip(mean, std)]
    out = oracle.normalize_rgb_u8(np.array([255, 0, 128], np.uint8).reshape(1, 1, 3), scale, off).reshape(-1)
    want = [(1 - mean[0]) / std[0], (0 - mean[1]) / std[1], (128 / 255 - mean[2]) / std[2]]
    assert np.abs(out - f32(*want)).max() < 1e-3
    # avx2-vs-scalar agreement :542-580
    src = oracle.pattern_u8(3000, 0xDEADBEEF).reshape(1, 1000, 3)
    a = oracle.normalize_rgb_u8(src, scale, off, oracle.LEAF_X86)
    b = oracle.normalize_rgb_u8(src, scale, off, oracle.LEAF_SCALAR)
    assert np.abs(a - b).max() < 1e-5


def test_std_mean_doctest(oracle):
    # core.rs:27-40 — exact f64 equality
    img = np.array([0, 1, 2, 253, 254, 255, 128, 129, 130, 64, 65, 66], np.uint8).reshape(2, 2, 3)
    std, mean, sums = oracle.std_mean(img)
    assert std.tolist() == [93.5183805462862] * 3
    assert mean.tolist() == [111.25, 112.25, 113.25]
    assert sums.tolist() == [445, 449, 453, 0 + 253 ** 2 + 128 ** 2 + 64 ** 2, 1 + 254 ** 2 + 129 ** 2 + 65 ** 2,
                             4 + 255 ** 2 + 130 ** 2 + 66 ** 2]


# ── a12 preprocess ───────────────────────────────────────────────────────────
def test_preprocess_affine(oracle):
    # preprocess.rs:349-370 ; 4x4 into 8x4 letterbox -> scale 1, pad_x 2 (cpu_letterbox_pad_geometry :1454)
    assert oracle.preprocess_affine(oracle.LETTERBOX, 4, 4, 8, 4) == (1.0, 1.0, 2.0, 0.0)
    sx, sy, px, py = oracle.preprocess_affine(oracle.LETTERBOX, 1920, 1080, 640, 640)
    assert sx == sy == float(np.float32(640) / np.float32(1920)) and px == 0.0
    assert py == float((np.float32(640) - np.float32(1080) * np.float32(sx)) * np.float32(0.5))
    assert oracle.preprocess_affine(oracle.STRETCH, 5, 3, 4, 4) == (float(np.float32(4) / np.float32(5)),
                                                                     float(np.float32(4) / np.float32(3)), 0.0, 0.0)


def test_preprocess_solid_all_sampling(oracle):
    # preprocess.rs:1428-1451 (CPU) and :1562-1588 (CUDA twin): solid stays solid, out == v/255
    src = np.tile(np.array([10, 20, 30], np.uint8), (3, 5, 1))
    for sampling in (oracle.NEAREST, oracle.BILINEAR):
        cfg = oracle.PreprocessCfg(mode=oracle.STRETCH, sampling=sampling)
        out = oracle.preprocess_frame(src, cfg, 5, 3, 4, 4)
        for c, v in enumerate([10.0, 20.0, 30.0]):
            assert np.abs(out[c] - v / 255.0).max() < 1e-4
    out = oracle.preprocess_cpu_rgb_bilinear(src, 4, 4, oracle.STRETCH, [0, 0, 0], [1, 1, 1], 114.0)
    for c, v in enumerate([10.0, 20.0, 30.0]):
        assert np.abs(out[c] - v / 255.0).max() < 1e-4


def test_preprocess_letterbox_pad_geometry(oracle):
    # preprocess.rs:1454-1472
    src = np.full((4, 4, 3), 100, np.uint8)
    cfg = oracle.PreprocessCfg(mode=oracle.LETTERBOX, pad_value=32.0)
    for out in (oracle.preprocess_frame(src, cfg, 4, 4, 8, 4),
                oracle.preprocess_cpu_rgb_bilinear(src, 8, 4, oracle.LETTERBOX, [0, 0, 0], [1, 1, 1], 32.0)):
        for x in range(8):
            want = (100.0 if 2 <= x < 6 else 32.0) / 255.0
            assert np.abs(out[:, :, x] - want).max() < 1e-4


def test_preprocess_imagenet_and_rgba(oracle):
    # preprocess.rs:1493-1508 (imagenet), :1475-1490 (rgba == rgb)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in std)
    src = np.full((4, 4, 3), 128, np.uint8)
    cfg = oracle.PreprocessCfg(mode=oracle.STRETCH, mean=mean, inv_std=inv)
    out = oracle.preprocess_frame(src, cfg, 4, 4, 4, 4)
    for c in range(3):
        assert abs(out[c, 0, 0] - (128.0 / 255.0 - mean[c]) / std[c]) < 1e-4
    rgb = np.tile(np.array([40, 80, 120], np.uint8), (4, 6, 1))
    rgba = np.tile(np.array([40, 80, 120, 200], np.uint8), (4, 6, 1))
    a = oracle.preprocess_frame(rgb, oracle.PreprocessCfg(mode=oracle.STRETCH), 6, 4, 8, 8)
    b = oracle.preprocess_frame(rgba, oracle.PreprocessCfg(mode=oracle.STRETCH, bpp=4), 6, 4, 8, 8)
    np.testing.assert_array_equal(a, b)


def _raw_bytes(n, k=0):
    return np.array([(((i * 7 + 13) % 251) + 31 * k) & 0xFF for i in range(n)], np.uint8)


def test_preprocess_fused_formats_match_chained(oracle):
    # preprocess.rs:1771-1848: decode-in-the-taps == decode to RGB (a9) then RGB preprocess, <= 1e-6
    # (bit-exact here: same arithmetic on identical integer taps)
    w, h = 8, 6
    for sampling in (oracle.NEAREST, oracle.BILINEAR):
        raw = _raw_bytes(w * h * 3 // 2)
        fused = oracle.preprocess_frame(raw, oracle.PreprocessCfg(fmt=oracle.FMT_NV12, sampling=sampling), w, h, 7, 5)
        chained = oracle.preprocess_frame(oracle.rgb_from_nv12(raw, w, h), oracle.PreprocessCfg(sampling=sampling),
                                          w, h, 7, 5)
        np.testing.assert_array_equal(fused, chained)
        raw = _raw_bytes(w * h * 2)
        fused = oracle.preprocess_frame(raw, oracle.PreprocessCfg(fmt=oracle.FMT_YUYV, sampling=sampling), w, h, 7, 5)
        chained = oracle.preprocess_frame(oracle.rgb_from_yuyv(raw, w, h), oracle.PreprocessCfg(sampling=sampling),
                                          w, h, 7, 5)
        np.testing.assert_array_equal(fused, chained)
        raw = _raw_bytes(w * h)
        fused = oracle.preprocess_frame(raw, oracle.PreprocessCfg(fmt=oracle.FMT_GRAY, sampling=sampling), w, h, 7, 5)
        chained = oracle.preprocess_frame(np.repeat(raw.reshape(h, w, 1), 3, 2),
                                          oracle.PreprocessCfg(sampling=sampling), w, h, 7, 5)
        np.testing.assert_array_equal(fused, chained)
        raw = _raw_bytes(w * h * 3)
        fused = oracle.preprocess_frame(raw, oracle.PreprocessCfg(fmt=oracle.FMT_BGR, sampling=sampling), w, h, 7, 5)
        chained = oracle.preprocess_frame(raw.reshape(h, w, 3)[:, :, ::-1].copy(),
                                          oracle.PreprocessCfg(sampling=sampling), w, h, 7, 5)
        np.testing.assert_array_equal(fused, chained)


def test_preprocess_f16_is_rne_of_f32(oracle):
    # preprocess.rs:1646-1675: f16 output == half::f16::from_f32(f32 output), bit for bit
    w, h = 23, 17
    src = np.zeros((h, w, 3), np.uint8)
    for y in range(h):
        for x in range(w):
            for c in range(3):
                src[y, x, c] = min((x * 127 // (w - 1) + y * 127 // (h - 1)) + c * 20, 255)  # host_gradient :1397
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in std)
    for sampling in (oracle.NEAREST, oracle.BILINEAR):
        cfg = oracle.PreprocessCfg(mode=oracle.LETTERBOX, sampling=sampling, mean=mean, inv_std=inv)
        o32 = oracle.preprocess_frame(src, cfg, w, h, 8, 6)
        o16 = oracle.preprocess_frame(src, cfg, w, h, 8, 6, f16=True)
        np.testing.assert_array_equal(o32.astype(np.float16).view(np.uint16), o16.view(np.uint16))
    # spot values of the hand-rolled converter (normals, subnormals, ties, inf, nan)
    for v in [0.0, -0.0, 1.0, -2.5, 65504.0, 6.1e-5, 5.96e-8, 2.98e-8, 1.0009765625, 1.00048828125, float("inf")]:
        assert oracle.f2h(v) == int(np.float32(v).astype(np.float16).view(np.uint16)), v
    assert oracle.f2h(float("nan")) & 0x7C00 == 0x7C00 and oracle.f2h(float("nan")) & 0x3FF != 0


def test_cfg1_dog_fixture(oracle):
    # BASELINE.json configs[0]: dog-rgb8 258x195 → f32/255 → gray → resize 128x128 (README.md:154-178)
    z = np.load(os.path.join(GOLD, "dog_cfg1.npz"))
    rgb = z["rgb"]
    assert rgb.shape == (195, 258, 3)
    f = rgb.astype(np.float32) * np.float32(1.0 / 255.0)
    gray = oracle.gray_from_rgb_f32(f, oracle.LEAF_SCALAR)
    np.testing.assert_array_equal(gray, z["gray"])
    small = oracle.resize_f32(gray, 128, 128, oracle.BILINEAR)
    np.testing.assert_array_equal(small, z["resized"])
    # independent cross-check of the resized plane with a float64 half-pixel bilinear (≤1e-4)
    g64 = gray[:, :, 0].astype(np.float64)
    ax, ay = 258 / 128, 195 / 128
    xs = np.clip(ax * np.arange(128) + 0.5 * ax - 0.5, 0, 257)
    ys = np.clip(ay * np.arange(128) + 0.5 * ay - 0.5, 0, 194)
    x0 = np.floor(xs).astype(int); y0 = np.floor(ys).astype(int)
    x1 = np.minimum(x0 + 1, 257); y1 = np.minimum(y0 + 1, 194)
    fx = xs - x0; fy = ys - y0
    want = ((1 - fy)[:, None] * (1 - fx)[None] * g64[y0][:, x0] + (1 - fy)[:, None] * fx[None] * g64[y0][:, x1]
            + fy[:, None] * (1 - fx)[None] * g64[y1][:, x0] + fy[:, None] * fx[None] * g64[y1][:, x1])
    assert np.abs(small[:, :, 0] - want).max() < 1e-4


# ── §8(f)#1: the other arms of resize_fast_u8_aa ──────────────────────────────
def test_pyrdown_2x_matches_the_rounded_box_mean(oracle):
    """resize/kernels.rs:64-75: (a+b+c+d+2)>>2 — restated independently with numpy integer arithmetic."""
    rng = np.random.default_rng(5)
    for (w, h) in [(2, 2), (6, 4), (34, 10), (130, 6)]:
        src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        s = src.astype(np.uint16)
        want = ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)
        np.testing.assert_array_equal(oracle.resize_fast_u8(src, w // 2, h // 2, 1), want)


def test_pyrup_2x_reference_properties(oracle):
    """resize/mod.rs:597-645 `resize_fast_2x_upscale`: same sizes and generator; corner pixels are preserved exactly.
    Plus: a constant image stays constant, the horizontal stage of a hand-worked row, and every output is within 2 LSB
    of the real-valued half-pixel bilinear value (four rounding half-adds, resize/kernels.rs:168-181, :274-281)."""
    for (w, h) in [(2, 2), (3, 4), (17, 9), (32, 5), (33, 6)]:
        src = (np.arange(w * h * 3) % 251).astype(np.uint8).reshape(h, w, 3)
        dst = oracle.resize_fast_u8(src, 2 * w, 2 * h, 1)
        for (dy, dx, sy, sx) in [(0, 0, 0, 0), (0, 2 * w - 1, 0, w - 1), (2 * h - 1, 0, h - 1, 0), (2 * h - 1, 2 * w - 1, h - 1, w - 1)]:
            np.testing.assert_array_equal(dst[dy, dx], src[sy, sx])
        # real-valued reference: half-pixel bilinear with edge clamp
        ys = np.clip((np.arange(2 * h) + 0.5) * 0.5 - 0.5, 0, h - 1); xs = np.clip((np.arange(2 * w) + 0.5) * 0.5 - 0.5, 0, w - 1)
        y0 = np.floor(ys).astype(int); x0 = np.floor(xs).astype(int)
        y1 = np.minimum(y0 + 1, h - 1); x1 = np.minimum(x0 + 1, w - 1)
        fy = (ys - y0)[:, None, None]; fx = (xs - x0)[None, :, None]
        f = src.astype(np.float64)
        ref = (f[y0][:, x0] * (1 - fx) + f[y0][:, x1] * fx) * (1 - fy) + (f[y1][:, x0] * (1 - fx) + f[y1][:, x1] * fx) * fy
        assert np.abs(dst.astype(np.float64) - ref).max() < 2.0   # four round-half-up half-adds, each off by < 0.5
    const = np.full((5, 7, 3), 173, np.uint8)
    assert (oracle.resize_fast_u8(const, 14, 10, 1) == 173).all()
    row = np.array([[[0, 0, 0], [100, 100, 100]], [[0, 0, 0], [100, 100, 100]]], np.uint8)   # identical rows: vertical stage is the identity
    np.testing.assert_array_equal(oracle.resize_fast_u8(row, 4, 4, 1)[0, :, 0], [0, 25, 75, 100])   # avg=50: (0+50+1)>>1, (100+50+1)>>1


def test_nearest_u8_index_rule(oracle):
    """resize/nearest.rs:18-21: clamp(floor((i+0.5)*scale)) in f64 (pixel centre then floor, no -0.5)."""
    rng = np.random.default_rng(6)
    for (sw, sh, dw, dh, c) in [(7, 5, 3, 2, 3), (5, 5, 9, 7, 1), (64, 48, 1, 1, 4), (1, 1, 8, 8, 2), (23, 37, 11, 17, 5), (4, 5, 2, 3, 3)]:
        src = rng.integers(0, 256, (sh, sw, c), dtype=np.uint8)
        xi = np.clip(np.floor((np.arange(dw) + 0.5) * (sw / dw)).astype(np.int64), 0, sw - 1)
        yi = np.clip(np.floor((np.arange(dh) + 0.5) * (sh / dh)).astype(np.int64), 0, sh - 1)
        np.testing.assert_array_equal(oracle.resize_fast_u8(src, dw, dh, 0), src[yi][:, xi])


def test_resize_fast_u8_path_selection_errors(oracle):
    """resize/mod.rs:283-337: Bilinear needs C in {1,3,4} and a source of at least 2x2 (unless an exact-2x RGB arm applies)."""
    with pytest.raises(ValueError, match="UnsupportedChannelCount"):
        oracle.resize_fast_u8(np.zeros((4, 4, 2), np.uint8), 3, 3, 1)
    with pytest.raises(ValueError, match="InvalidImageSize"):
        oracle.resize_fast_u8(np.zeros((4, 1, 3), np.uint8), 3, 3, 1)
    assert oracle.resize_fast_u8(np.zeros((4, 4, 2), np.uint8), 3, 3, 0).shape == (3, 3, 2)   # Nearest takes any channel count
    # generic (non-2x) bilinear still goes to the Q14 arm
    src = oracle.pattern_u8(13 * 9 * 3).reshape(9, 13, 3)
    np.testing.assert_array_equal(oracle.resize_fast_u8(src, 7, 5, 1), oracle.resize_bilinear_u8(src, 7, 5))


# ── §8(f)#1: u8 warps ─────────────────────────────────────────────────────────
def test_warp_u8_reference_known_answers(oracle):
    """warp/perspective.rs:338-358 (edge column of a horizontal flip is sampled, not zero-filled), its affine analogue
    (warp/affine.rs:471), identity = exact copy, and the set-up of warp/perspective.rs:636-668."""
    src = np.array([10, 20, 30, 40, 50, 60, 70, 80], np.uint8).reshape(2, 4, 1)
    want = np.array([40, 30, 20, 10, 80, 70, 60, 50], np.uint8).reshape(2, 4, 1)
    np.testing.assert_array_equal(oracle.warp_perspective_u8(src, 4, 2, [-1, 0, 3, 0, 1, 0, 0, 0, 1]), want)
    np.testing.assert_array_equal(oracle.warp_affine_u8(src, 4, 2, [-1, 0, 3, 0, 1, 0]), want)
    img = oracle.pattern_u8(37 * 23 * 3).reshape(23, 37, 3)
    np.testing.assert_array_equal(oracle.warp_perspective_u8(img, 37, 23, [1, 0, 0, 0, 1, 0, 0, 0, 1]), img)
    np.testing.assert_array_equal(oracle.warp_affine_u8(img, 37, 23, [1, 0, 0, 0, 1, 0]), img)
    h, w = 120, 160
    data = ((np.arange(w * h * 3, dtype=np.uint64) * 37) & 0xFF).astype(np.uint8).reshape(h, w, 3)
    out = oracle.warp_perspective_u8(data, w, h, [1.02, 0.03, -5.0, -0.03, 1.01, 2.0, 0.00005, 0.00003, 1.0])
    assert int(out[h // 2, w // 2].astype(np.uint32).sum()) > 0
    with pytest.raises(ValueError, match="CannotComputeDeterminant"):
        oracle.warp_perspective_u8(img, 37, 23, [1, 2, 3, 2, 4, 6, 0, 0, 1])


def _persp_u8_numpy(src, dw, dh, m, oracle):
    """Independent per-pixel restatement in numpy float32 (IEEE, unfused): direct coordinate (warp/kernels.rs:107-122) and
    the bounds-checked Q10 sampler (warp/common.rs:14-63).  No span logic — every pixel is decided by its own coordinate."""
    f = np.float32
    inv = oracle.invert_homography(m).astype(f)
    sh, sw, c = src.shape
    y = np.arange(dh, dtype=f)[:, None]; x = np.arange(dw, dtype=f)[None, :]
    nx = (inv[1] * y + inv[2]) + inv[0] * x
    ny = (inv[4] * y + inv[5]) + inv[3] * x
    nd = (inv[7] * y + inv[8]) + inv[6] * x
    with np.errstate(all="ignore"):
        inv_nd = f(1.0) / nd
        xf = nx * inv_nd; yf = ny * inv_nd
    ok = np.isfinite(xf) & np.isfinite(yf)
    xi = np.floor(np.where(ok, xf, 0)).astype(np.int64); yi = np.floor(np.where(ok, yf, 0)).astype(np.int64)
    ok &= (xi >= 0) & (xi < sw) & (yi >= 0) & (yi < sh)
    xi = np.clip(xi, 0, sw - 1); yi = np.clip(yi, 0, sh - 1)
    fx = ((xf - xi.astype(f)) * f(1024.0)).astype(f); fy = ((yf - yi.astype(f)) * f(1024.0)).astype(f)
    fx = np.where(ok, fx, 0).astype(np.int64).astype(np.uint32); fy = np.where(ok, fy, 0).astype(np.int64).astype(np.uint32)
    xi1 = np.minimum(xi + 1, sw - 1); yi1 = np.minimum(yi + 1, sh - 1)
    s32 = src.astype(np.uint32)
    top = s32[yi, xi] * (1024 - fx)[..., None] + s32[yi, xi1] * fx[..., None]
    bot = s32[yi1, xi] * (1024 - fx)[..., None] + s32[yi1, xi1] * fx[..., None]
    v = (top * (1024 - fy)[..., None] + bot * fy[..., None] + (1 << 19)) >> 20
    return np.where(ok[..., None], v, 0).astype(np.uint8)


PERSP_U8 = [
    [1.02, 0.03, -5.0, -0.03, 1.01, 2.0, 0.00005, 0.00003, 1.0],
    [0.9, 0.15, 10.0, -0.1, 1.1, -6.0, 0.0, 0.0, 1.0],
    [1.03, 0.05, -3.0, -0.02, 0.97, 4.0, 2.0 / (97 * 129), 1.5 / (129 * 97), 1.0],
    [-1.0, 0.0, 63.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0],
    [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.02, 0.0, -0.5],       # denominator changes sign inside the row: per-pixel fallback
    [0.7, 0.0, 3.0, 0.0, 1.3, -2.0, 0.0, 0.001, 1.0],
]


@pytest.mark.parametrize("m", PERSP_U8)
def test_warp_perspective_u8_span_logic_equals_per_pixel_decision(oracle, m):
    """The row classification + analytic span of warp/perspective.rs:214-300 must zero exactly the pixels whose own
    coordinate is outside — checked against the independent per-pixel numpy restatement."""
    src = oracle.pattern_u8(64 * 48 * 3, 0x77).reshape(48, 64, 3)
    np.testing.assert_array_equal(oracle.warp_perspective_u8(src, 64, 48, m), _persp_u8_numpy(src, 64, 48, m, oracle))


# ── §8(f)#1: u8 blurs ─────────────────────────────────────────────────────────
def _knuth_u8(n):
    """the reference tests' generator: ((i * 2654435761) >> 24) as u8 with usize wrapping (filter/ops.rs:1992-1994)"""
    i = np.arange(n, dtype=np.uint64)
    return (((i * np.uint64(2654435761)) & np.uint64(0xFFFFFFFFFFFFFFFF)) >> np.uint64(24)).astype(np.uint8)


def _q8_two_pass_numpy(src, ikx, iky):
    """Independent numpy restatement of the general path: replicate border, (acc+128)>>8 after EACH pass."""
    rows, cols, c = src.shape
    hx, hy = len(ikx) // 2, len(iky) // 2
    p = np.pad(src.astype(np.uint32), ((0, 0), (hx, hx), (0, 0)), mode="edge")
    h = sum(p[:, k:k + cols] * np.uint32(ikx[k]) for k in range(len(ikx)))
    h = ((h + 128) >> 8).astype(np.uint32)
    p = np.pad(h, ((hy, hy), (0, 0), (0, 0)), mode="edge")
    v = sum(p[k:k + rows] * np.uint32(iky[k]) for k in range(len(iky)))
    return ((v + 128) >> 8).astype(np.uint8)


def test_quantize_kernel_256(oracle):
    """filter/ops.rs:759-770: (k*256 + 0.5) as u8, centre tap absorbs the rounding so the sum is exactly 256."""
    np.testing.assert_array_equal(oracle.quantize_kernel_256([0.0625, 0.25, 0.375, 0.25, 0.0625]), [16, 64, 96, 64, 16])
    for k in (3, 5, 7, 9, 15, 31):
        assert int(oracle.quantize_kernel_256(np.full(k, 1.0 / k, np.float32)).astype(np.uint32).sum()) == 256
    for (k, sg) in [(3, 0.85), (5, 1.0), (5, 1.5), (7, 2.0), (9, 1.0), (31, 4.0)]:
        q = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(k, sg))
        assert int(q.astype(np.uint32).sum()) == 256 and (q == q[::-1]).all()


def test_gaussian_blur_u8_general_path(oracle):
    """filter/ops.rs:2020-2061 (5x5 goes to the general Q8 path) on the reference's 37x83 generator image, plus other
    kernel sizes / channel counts, against the independent numpy two-pass."""
    src = _knuth_u8(37 * 83).reshape(37, 83, 1)
    ik = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(5, 1.0))
    np.testing.assert_array_equal(oracle.gaussian_blur_u8(src, (5, 5), (1.0, 1.0)), _q8_two_pass_numpy(src, ik, ik))
    for (kx, ky, sx, sy, c) in [(7, 7, 2.0, 2.0, 1), (5, 3, 1.5, 2.0, 3), (9, 9, 0.0, 0.0, 4), (3, 3, 2.0, 2.0, 3), (0, 0, 0.8, 0.0, 3)]:
        img = _knuth_u8(23 * 31 * c).reshape(23, 31, c)
        kxn, kyn, rsx, rsy = oracle.gaussian_resolve(kx, ky, sx, sy)
        ikx = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(kxn, rsx)); iky = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(kyn, rsy))
        np.testing.assert_array_equal(oracle.gaussian_blur_u8(img, (kx, ky), (sx, sy)), _q8_two_pass_numpy(img, ikx, iky))


def test_gaussian_blur_u8_binomial_path(oracle):
    """k = 3, sigma in [0.6, 1.2] takes the [1,2,1]/4 half-add path (filter/ops.rs:22-29); it stays within 2 LSB of the
    general Q8 path at sigma 0.85 (filter/ops.rs:2063-2104), and 1-column / 1-row images work (:2107-2156)."""
    for (rows, cols, c) in [(37, 83, 1), (17, 45, 3)]:
        src = _knuth_u8(rows * cols * c).reshape(rows, cols, c)
        binom = oracle.gaussian_blur_u8(src, (3, 3), (1.0, 1.0))
        ik = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(3, 0.85))
        gen = _q8_two_pass_numpy(src, ik, ik)
        assert int(np.abs(binom.astype(np.int16) - gen.astype(np.int16)).max()) <= 2
        # independent restatement of the half-add form
        s = src.astype(np.uint32)
        rh = lambda a, b: (a + b + 1) >> 1
        p = np.pad(s, ((0, 0), (1, 1), (0, 0)), mode="edge")
        h = rh(rh(p[:, :-2], p[:, 1:-1]), rh(p[:, 1:-1], p[:, 2:]))
        p = np.pad(h, ((1, 1), (0, 0), (0, 0)), mode="edge")
        np.testing.assert_array_equal(binom, rh(rh(p[:-2], p[1:-1]), rh(p[1:-1], p[2:])).astype(np.uint8))
    col = (np.arange(5) * 50).astype(np.uint8).reshape(5, 1, 1)
    assert oracle.gaussian_blur_u8(col, (3, 3), (1.0, 1.0)).shape == (5, 1, 1)
    assert oracle.gaussian_blur_u8(col.reshape(1, 5, 1), (3, 3), (1.0, 1.0)).shape == (1, 5, 1)
    # sigma outside [0.6, 1.2] -> general path even for k = 3
    src = _knuth_u8(9 * 11 * 3).reshape(9, 11, 3)
    ik = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(3, 2.0))
    np.testing.assert_array_equal(oracle.gaussian_blur_u8(src, (3, 3), (2.0, 2.0)), _q8_two_pass_numpy(src, ik, ik))


def test_box_blur_u8(oracle):
    src = _knuth_u8(19 * 27 * 3).reshape(19, 27, 3)
    for (kx, ky) in [(3, 3), (5, 5), (7, 3), (1, 9)]:
        ikx = oracle.quantize_kernel_256(np.full(kx, 1.0 / kx, np.float32)); iky = oracle.quantize_kernel_256(np.full(ky, 1.0 / ky, np.float32))
        np.testing.assert_array_equal(oracle.box_blur_u8(src, (kx, ky)), _q8_two_pass_numpy(src, ikx, iky))
    for bad in [(0, 3), (4, 3), (3, 2)]:
        with pytest.raises(ValueError, match="InvalidSigmaValue"):
            oracle.box_blur_u8(src, bad)
    with pytest.raises(ValueError, match="InvalidSigmaValue"):
        oracle.gaussian_blur_u8(src, (4, 4), (1.0, 1.0))


# ── §8(f)#2: remap ────────────────────────────────────────────────────────────
def test_remap_reference_known_answers(oracle):
    """interpolation/remap.rs:499-549 (f32 smoke), :551-612 (u8 identity, 1 and 3 channels), :613-643 (Q10 weight
    quantisation: 0.1 -> 102/1024 -> 25), :644-672 (nearest zeroes out-of-range maps)."""
    img = np.arange(9, dtype=np.float32).reshape(3, 3, 1)
    out = oracle.remap(img, np.array([[0, 2], [0, 2]], np.float32), np.array([[0, 0], [2, 2]], np.float32), 1)
    np.testing.assert_allclose(out[..., 0], [[0, 2], [6, 8]], atol=1e-6)
    ident_x = np.array([[0, 1], [0, 1]], np.float32); ident_y = np.array([[0, 0], [1, 1]], np.float32)
    g = np.array([1, 2, 3, 4], np.uint8).reshape(2, 2, 1)
    np.testing.assert_array_equal(oracle.remap(g, ident_x, ident_y, 1), g)
    rgb = np.arange(1, 13, dtype=np.uint8).reshape(2, 2, 3)
    np.testing.assert_array_equal(oracle.remap(rgb, ident_x, ident_y, 1), rgb)
    two = np.array([0, 255], np.uint8).reshape(1, 2, 1)
    assert oracle.remap(two, np.array([[0.1]], np.float32), np.array([[0.0]], np.float32), 1)[0, 0, 0] == 25
    q = np.array([10, 20, 30, 40], np.uint8).reshape(2, 2, 1)
    out = oracle.remap(q, np.array([[0.49, 1.49], [-1.0, 0.5]], np.float32), np.array([[0.49, 0.49], [0.5, 2.0]], np.float32), 0)
    np.testing.assert_array_equal(out[..., 0], [[10, 20], [0, 0]])
    # NaN / inf coordinates are outside
    bad = np.array([[np.nan, np.inf], [-np.inf, 0.5]], np.float32)
    assert (oracle.remap(q, bad, np.zeros((2, 2), np.float32), 1)[..., 0] == [[0, 0], [0, 15]]).all()
    assert (oracle.remap(q.astype(np.float32), bad, np.zeros((2, 2), np.float32), 1)[..., 0] == [[0, 0], [0, 15.0]]).all()


def test_remap_equals_warp_for_an_affine_map(oracle):
    """A map generated from an affine transform must reproduce the u8 perspective warp's sampler output wherever both
    evaluate the same coordinate (identity homography bottom row => xf = nx * (1/1))."""
    src = oracle.pattern_u8(40 * 30 * 3, 5).reshape(30, 40, 3)
    H = [0.9, 0.15, 3.0, -0.1, 1.1, -2.0, 0.0, 0.0, 1.0]
    inv = oracle.invert_homography(H).astype(np.float32)
    y = np.arange(30, dtype=np.float32)[:, None]; x = np.arange(40, dtype=np.float32)[None, :]
    nd = (inv[7] * y + inv[8]) + inv[6] * x
    inv_nd = np.float32(1.0) / nd
    mx = ((inv[1] * y + inv[2]) + inv[0] * x) * inv_nd
    my = ((inv[4] * y + inv[5]) + inv[3] * x) * inv_nd
    np.testing.assert_array_equal(oracle.remap(src, mx, my, 1), oracle.warp_perspective_u8(src, 40, 30, H))


# ── §8(f)#4: video encode ─────────────────────────────────────────────────────
def test_video_encode_reference_known_answers(oracle):
    """color/yuv/kernels.rs:1890-1925 (constant colour survives encode -> decode within 2 LSB, YUYV and NV12),
    :1927-1950 (YUYV layout `Y0 U Y1 V`, chroma from the rounded pair average) and an independent numpy restatement
    of the Q8 formulas (:1223-1252)."""
    w, h = 8, 6
    for (r, g, b) in [(200, 50, 25), (0, 0, 0), (255, 255, 255), (17, 200, 99)]:
        rgb = np.tile(np.array([r, g, b], np.uint8), (h, w, 1))
        back = oracle.rgb_from_yuyv(oracle.yuyv_from_rgb(rgb), w, h)
        assert int(np.abs(back.astype(int) - rgb.astype(int)).max()) <= 2
        back = oracle.rgb_from_nv12(oracle.nv12_from_rgb(rgb), w, h)
        assert int(np.abs(back.astype(int) - rgb.astype(int)).max()) <= 2
    ey = lambda R, G, B: np.clip(((66 * R + 129 * G + 25 * B + 128) >> 8) + 16, 0, 255)
    eu = lambda R, G, B: np.clip(((-38 * R - 74 * G + 112 * B + 128) >> 8) + 128, 0, 255)
    ev = lambda R, G, B: np.clip(((112 * R - 94 * G - 18 * B + 128) >> 8) + 128, 0, 255)
    out = oracle.yuyv_from_rgb(np.array([[[255, 0, 0], [0, 0, 255]]], np.uint8))
    assert list(out) == [ey(255, 0, 0), eu(128, 0, 128), ey(0, 0, 255), ev(128, 0, 128)]
    img = oracle.pattern_u8(34 * 18 * 3, 21).reshape(18, 34, 3).astype(np.int64)
    R, G, B = img[..., 0], img[..., 1], img[..., 2]
    yuyv = oracle.yuyv_from_rgb(img.astype(np.uint8)).reshape(18, 17, 4)
    np.testing.assert_array_equal(yuyv[..., 0], ey(R[:, 0::2], G[:, 0::2], B[:, 0::2]))
    np.testing.assert_array_equal(yuyv[..., 2], ey(R[:, 1::2], G[:, 1::2], B[:, 1::2]))
    pa = lambda c: (c[:, 0::2] + c[:, 1::2] + 1) >> 1
    np.testing.assert_array_equal(yuyv[..., 1], eu(pa(R), pa(G), pa(B)))
    np.testing.assert_array_equal(yuyv[..., 3], ev(pa(R), pa(G), pa(B)))
    nv = oracle.nv12_from_rgb(img.astype(np.uint8))
    np.testing.assert_array_equal(nv[:34 * 18].reshape(18, 34), ey(R, G, B))
    qa = lambda c: (c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + 2) >> 2
    uv = nv[34 * 18:].reshape(9, 17, 2)
    np.testing.assert_array_equal(uv[..., 0], eu(qa(R), qa(G), qa(B)))
    np.testing.assert_array_equal(uv[..., 1], ev(qa(R), qa(G), qa(B)))
    with pytest.raises(ValueError):
        oracle.nv12_from_rgb(np.zeros((5, 4, 3), np.uint8))


# ── bicubic / Lanczos samplers (SURVEY §8(f) #3) ──────────────────────────────
def test_lanczos_four_eval_weights_match_per_tap_form(oracle):
    """interpolation/lanczos.rs:242-265 `four_eval_weights_match_per_tap_form`: the 4-sin_pi weight path agrees with the
    per-tap lanczos3 to 1e-6 over the whole frac range; exact edge values w0[2] == 1, w0[5] == 0."""
    for i in range(0, 10001, 7):
        frac = np.float32(i) / np.float32(10001.0)
        w = oracle.lanczos3_weights(frac)
        per_tap = [oracle.lanczos3(np.float32(frac) + np.float32(o)) for o in (2.0, 1.0, 0.0, -1.0, -2.0, -3.0)]
        assert np.max(np.abs(w - np.array(per_tap, np.float32))) < 1e-6, frac
    w0 = oracle.lanczos3_weights(0.0)
    assert w0[2] == 1.0 and w0[5] == 0.0


def test_sin_pi_and_lanczos_axis_properties(oracle):
    """sin_pi (lanczos.rs:19-35) against libm in f64; lanczos_axis rows are normalised and centred on the tap base."""
    for x in np.linspace(-3.0, 3.0, 601):
        assert abs(oracle.sin_pi(np.float32(x)) - np.sin(np.pi * float(np.float32(x)))) < 5e-7
    x0s, w = oracle.lanczos_axis(97, 40)
    assert x0s.shape == (40,) and w.shape == (40, 6)
    assert np.all(np.abs(w.sum(axis=1) - 1.0) < 1e-6)
    a = np.float32(97) / np.float32(40)
    s = np.clip(a * np.arange(40, dtype=np.float32) + (np.float32(0.5) * a - np.float32(0.5)), 0, 96)
    assert np.array_equal(x0s, np.floor(s).astype(np.int32))


def _keys_f64(t):
    t = abs(t)
    if t <= 1:
        return 1.5 * t ** 3 - 2.5 * t ** 2 + 1
    if t < 2:
        return -0.5 * t ** 3 + 2.5 * t ** 2 - 4 * t + 2
    return 0.0


def test_bicubic_resize_against_f64_restatement(oracle):
    """resize Bicubic (resize/mod.rs:197 -> interpolation/bicubic.rs:33-61) against an independent f64 Keys a=-0.5
    implementation on the same half-pixel grid with replicate-clamped taps; and exactness on constant / linear ramps."""
    sw, sh, dw, dh, c = 23, 17, 31, 11, 3
    src = oracle.pattern_f32(sw * sh * c).reshape(sh, sw, c)
    got = oracle.resize_f32(src, dw, dh, oracle.BICUBIC)
    want = np.zeros((dh, dw, c))
    ax, ay = np.float32(sw) / np.float32(dw), np.float32(sh) / np.float32(dh)
    for y in range(dh):
        sy = float(np.clip(ay * np.float32(y) + (np.float32(0.5) * ay - np.float32(0.5)), 0, sh - 1))
        y0 = int(np.floor(sy))
        for x in range(dw):
            sx = float(np.clip(ax * np.float32(x) + (np.float32(0.5) * ax - np.float32(0.5)), 0, sw - 1))
            x0 = int(np.floor(sx))
            acc = np.zeros(c)
            for j in range(-1, 3):
                for i in range(-1, 3):
                    acc += _keys_f64(sx - (x0 + i)) * _keys_f64(sy - (y0 + j)) * src[min(max(y0 + j, 0), sh - 1), min(max(x0 + i, 0), sw - 1)]
            want[y, x] = acc
    assert np.max(np.abs(got - want)) < 2e-6
    const = np.full((9, 12, 1), 0.375, np.float32)
    assert np.max(np.abs(oracle.resize_f32(const, 20, 15, oracle.BICUBIC) - 0.375)) < 1e-6     # weights sum to 1
    assert np.max(np.abs(oracle.resize_f32(const, 5, 4, oracle.LANCZOS) - 0.375)) < 1e-6


def test_warps_support_all_modes_identity(oracle):
    """warp/affine.rs:528-550 `warp_affine_supports_all_modes`, warp/perspective.rs:475-496: identity warps succeed in
    every mode; on integer coordinates bicubic reproduces the source exactly (Keys weights are 0,1,0,0 at frac 0)."""
    src = oracle.pattern_f32(8 * 6 * 3).reshape(6, 8, 3)
    for mode in (oracle.NEAREST, oracle.BILINEAR, oracle.BICUBIC):
        assert np.array_equal(oracle.warp_affine_f32(src, [1, 0, 0, 0, 1, 0], 8, 6, mode), src)
        assert np.array_equal(oracle.warp_perspective_f32(src, [1, 0, 0, 0, 1, 0, 0, 0, 1], 8, 6, mode), src)
    lz = oracle.warp_affine_f32(src, [1, 0, 0, 0, 1, 0], 8, 6, oracle.LANCZOS)
    assert np.max(np.abs(lz - src)) < 1e-6      # w[2] = 1 exactly, the other taps are sin_pi(0) * ... = 0, renormalised by 1


def test_preprocess_lanczos_solid_and_bounds(oracle):
    """preprocess.rs sample_lanczos (kernel source :565-590): a solid frame stays solid (weights renormalised by their
    sum); letterbox pad pixels keep the pad value."""
    w, h = 32, 24
    src = np.full((h, w, 3), 200, np.uint8)
    cfg = oracle.PreprocessCfg(mode=oracle.LETTERBOX, fmt=oracle.FMT_RGB, mean=(0.0, 0.0, 0.0), inv_std=(1.0, 1.0, 1.0), sampling=oracle.LANCZOS)
    out = oracle.preprocess_frame(src.reshape(-1), cfg, w, h, 20, 20)
    inside = out[:, 3:17, :]
    assert np.max(np.abs(inside - np.float32(200.0) / np.float32(255.0))) < 1e-5
    assert np.all(out[:, 0, :] == np.float32(114.0) / np.float32(255.0))


# ── pyramids (SURVEY §8(f) #4) ────────────────────────────────────────────────
def test_pyrdown_reference_vectors(oracle):
    """pyramid.rs:915-994 `test_pyrdown`, `test_pyrdown_3c` expected arrays; :1372-1418 `test_pyrdown_u8_3c` (cv2.pyrDown)."""
    got = oracle.pyrdown_f32(np.arange(16, dtype=np.float32).reshape(4, 4, 1)).reshape(-1)
    assert np.max(np.abs(got - np.array([3.75, 4.875, 8.25, 9.375], np.float32))) < 1e-4
    got = oracle.pyrdown_f32(np.arange(48, dtype=np.float32).reshape(4, 4, 3)).reshape(-1)
    want = [11.25, 12.25, 13.25, 14.625, 15.625, 16.625, 24.75, 25.75, 26.75, 28.125, 29.125, 30.125]
    assert np.max(np.abs(got - np.array(want, np.float32))) < 1e-4
    got8 = oracle.pyrdown_u8(np.arange(48, dtype=np.uint8).reshape(4, 4, 3)).reshape(-1)
    assert np.array_equal(got8, [11, 12, 13, 15, 16, 17, 25, 26, 27, 28, 29, 30])


def test_pyramids_against_cv2(oracle):
    """The reference documents cv2 as the cross-check of its pyramid levels (pyramid.rs:1373-1376).  pyrdown: byte-exact
    (u8) / 1e-6 (f32) everywhere; pyrup: the interior (the reference's border rule is its own)."""
    cv2 = pytest.importorskip("cv2")
    for (h, w, c) in ((37, 53, 3), (16, 16, 1), (5, 7, 4), (2, 2, 3)):
        a = oracle.pattern_u8(h * w * c, 5).reshape(h, w, c)
        f = oracle.pattern_f32(h * w * c, 6).reshape(h, w, c)
        assert np.array_equal(oracle.pyrdown_u8(a), cv2.pyrDown(a).reshape((h + 1) // 2, (w + 1) // 2, c))
        assert np.max(np.abs(oracle.pyrdown_f32(f) - cv2.pyrDown(f).reshape((h + 1) // 2, (w + 1) // 2, c))) < 1e-6
        if h > 4 and w > 4:
            up8 = oracle.pyrup_u8(a).astype(int)[2:-2, 2:-2]
            assert np.max(np.abs(up8 - cv2.pyrUp(a).reshape(2 * h, 2 * w, c).astype(int)[2:-2, 2:-2])) <= 1
            upf = oracle.pyrup_f32(f)[2:-2, 2:-2]
            assert np.max(np.abs(upf - cv2.pyrUp(f).reshape(2 * h, 2 * w, c)[2:-2, 2:-2])) < 1e-6


def test_pyramid_min_sizes_and_flat(oracle):
    """pyramid.rs:1050-1111 / :1218-1244 / :1246-1278: 1x1, 1xN, Nx1 inputs work; a flat image stays flat."""
    for (h, w) in ((1, 1), (1, 5), (5, 1), (2, 3)):
        f = np.full((h, w, 1), 0.625, np.float32)
        assert np.all(oracle.pyrdown_f32(f) == np.float32(0.625)) and np.all(oracle.pyrup_f32(f) == np.float32(0.625))
        u = np.full((h, w, 3), 77, np.uint8)
        assert np.all(oracle.pyrdown_u8(u) == 77) and np.all(oracle.pyrup_u8(u) == 77)


# ── undistort maps (SURVEY §8(f) #2) ──────────────────────────────────────────
DIST_INTR = (577.48583984375, 652.8748779296875, 577.48583984375, 386.1428833007813)
DIST_COEF = (1.7547749280929563, 0.0097926277667284, -0.027250492945313457, 2.1092164516448975, 0.462927520275116, -0.08215277642011642,
             -0.00005457743463921361, 0.00003006766564794816)


def test_distort_point_polynomial_reference_value(oracle):
    """calibration/distortion.rs:603-628 `test_distort_point_polynomial`: y is asserted EXACTLY in f64."""
    x, y = oracle.distort_point_polynomial(100.0, 20.0, DIST_INTR, DIST_COEF)
    assert y == 98.83006704526377
    assert x != 194.24656721843076 and abs(x - 202.86576969976807) < 1e-9   # the reference asserts `ne` on that literal


def test_correction_map_shape_and_identity(oracle):
    """:630-672 map shapes; zero distortion is the identity map (:723-743 `test_identity_no_distortion` spirit)."""
    mx, my = oracle.generate_correction_map_polynomial(DIST_INTR, DIST_COEF, 8, 4)
    assert mx.shape == (4, 8, 1) and my.shape == (4, 8, 1)
    mx, my = oracle.generate_correction_map_polynomial((612.3, 610.8, 320.1, 241.7), (0,) * 8, 16, 9)
    xs, ys = np.meshgrid(np.arange(16, dtype=np.float32), np.arange(9, dtype=np.float32))
    assert np.max(np.abs(mx[..., 0] - xs)) < 1e-4 and np.max(np.abs(my[..., 0] - ys)) < 1e-4
