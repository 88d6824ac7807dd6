"""The values a kernel can be given, not only the bytes / 255 of `oracle.pattern_f32`: full-range f32 data, extreme
normalisation parameters and saturated u8 frames, every result bit for bit against the oracle.

The rest of the suite covers shapes and dispatch variants with data in [0, 1]; here the same kernels, reached with the
geometries and knobs of test_gpu_variants.py and named through `kb200_last_kernel()`, see

* f32 data of six kinds (`gen_f32`): negative values, every finite binade, sums and differences that overflow, tap
  products that underflow into the subnormal range (an FTZ path on data would flush them), signed zeros, inf and NaN;
* camera-preprocess normalisation parameters that push f16 outputs to inf, to subnormals and to exact (signed) zeros,
  and, through the C ABI, parameters the Python builder refuses (negative or infinite inv_std, pad values outside 0..255);
* saturated, striped and impulse u8 frames (the integer bounds: Q14 / Q10 / Q8 / Q20 terms at their largest), every
  (Y, U, V) triple through the YUV decoders, and `std_mean` past the flush point of its 32-bit accumulators.

Comparison (`assert_same`): finite values and zeros bit for bit (+0 and -0 differ); an f32 NaN only as "is NaN", because
the GPU produces the canonical NaN 0x7FFFFFFF while x86 SSE propagates payloads and produces the negative default NaN
0xFFC00000; in f16 outputs of the preprocess, an element whose f32 value was NaN exactly 0x7E00 (f2h_ref turns the
canonical NaN into that value; the oracle's own f16 NaN may carry the x86 sign), every other element bit for bit.
"""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest
import torch

from harness import compare_frames, cu, dev, free_device_memory, knobs, rot
from restate import NAMED_FUSED_MODES, _remap_maps, demosaic, filter_kernel, preprocess_rgb16


F32 = np.float32
FLT_MIN = float(np.finfo(np.float32).tiny)
KINDS = ("signed", "wide", "huge", "tiny", "zeros", "nonfinite")
F16_NAN = 0x7E00


# ── data generators ──────────────────────────────────────────────────────────────────────────────────────────────
def gen_f32(kind, n, seed=0):
    """n f32 values of one kind, seeded."""
    rng = np.random.default_rng([seed, KINDS.index(kind)])
    sign = rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)
    if kind == "signed":                     # spread over +-1e3
        v = rng.uniform(-1e3, 1e3, n).astype(F32)
    elif kind in ("wide", "nonfinite"):      # random sign, exponent (0..254: zeros and subnormals too) and mantissa
        exp = rng.integers(0, 255, n, dtype=np.uint32) << np.uint32(23)
        v = (sign | exp | rng.integers(0, 1 << 23, n, dtype=np.uint32)).view(F32)
        if kind == "nonfinite":
            idx = rng.choice(n, max(3, n // 64), replace=False)
            v[idx] = np.array([np.inf, -np.inf, np.nan], F32)[np.arange(idx.size) % 3]
    elif kind == "huge":                     # +-1e37 .. +-3.4e38: b - a and filter sums overflow
        mag = (10.0 ** rng.uniform(37.0, np.log10(3.4e38), n)).astype(F32)
        v = (mag.view(np.uint32) | sign).view(F32)
    elif kind == "tiny":                     # subnormals and values near FLT_MIN: tap products underflow
        sub = rng.integers(1, 1 << 23, n, dtype=np.uint32)
        near = (rng.uniform(0.5, 8.0, n) * FLT_MIN).astype(F32).view(np.uint32)
        v = (np.where(rng.random(n) < 0.5, sub, near).astype(np.uint32) | sign).view(F32)
    elif kind == "zeros":                    # +-0 and small values
        small = rng.uniform(-1e-3, 1e-3, n).astype(F32)
        v = np.where(rng.random(n) < 0.6, sign.view(F32), small).astype(F32)   # sign.view(F32) is +0.0 or -0.0
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(v, F32)


def img_f32(kind, shape, seed=0):
    return gen_f32(kind, int(np.prod(shape)), seed).reshape(shape)


def all_bytes(n, seed):
    """n bytes in which every value 0..255 occurs (n >= 256), shuffled."""
    rng = np.random.default_rng(seed)
    return rng.permutation(np.resize(np.arange(256, dtype=np.uint8), n)).astype(np.uint8)


def u8_patterns(h, w, c):
    """Saturated u8 frames: the largest integer terms and the sharpest edges."""
    yy, xx = np.mgrid[0:h, 0:w]
    full = lambda m: np.ascontiguousarray(np.repeat((m.astype(np.uint8) * 255)[..., None], c, axis=2))
    imp0, imp1 = np.zeros((h, w), bool), np.ones((h, w), bool)
    imp0[h // 2, w // 3] = True
    imp1[h // 3, w // 2] = False
    return {"zeros": full(np.zeros((h, w), bool)), "ones": full(np.ones((h, w), bool)), "checker": full((xx + yy) % 2 == 0),
            "cols2": full(xx % 2 == 0), "rows2": full(yy % 2 == 0), "cols3": full(xx % 3 == 0), "rows3": full(yy % 3 == 1),
            "impulse": full(imp0), "hole": full(imp1),
            "chan": np.ascontiguousarray(np.broadcast_to((np.arange(c) % 2 * 255).astype(np.uint8), (h, w, c)))}


# ── comparison ───────────────────────────────────────────────────────────────────────────────────────────────────
def _f16_nan(bits):
    return ((bits & 0x7C00) == 0x7C00) & ((bits & 0x03FF) != 0)


def mismatches(got, want, f16=False, zero_sign_ok=None, f32_nan=None):
    """Boolean mask of the elements that differ.  f32: NaN matches NaN (any payload), everything else bit for bit.
    f16 (uint16 bits): bit for bit, except where the f32 value before the conversion was a NaN (`f32_nan`, from the
    reference's f32 run): there the device must write exactly 0x7E00, whatever the oracle's x86 NaN turned into.  (A
    finite f32 beyond the f16 range with a nonzero mantissa also converts to a NaN pattern, by the reference's
    f2h rule; those bits are compared exactly.)  `zero_sign_ok`: an optional mask of elements where +0 and -0 are
    accepted as equal (each caller names its reason)."""
    if f16:
        g, w = np.asarray(got).view(np.uint16), np.asarray(want).view(np.uint16)
        nan = np.zeros(g.shape, bool) if f32_nan is None else np.asarray(f32_nan)
        bad = np.where(nan, (g != F16_NAN) | ~_f16_nan(w), g != w)
    else:
        g, w = np.asarray(got, F32), np.asarray(want, F32)
        gn, wn = np.isnan(g), np.isnan(w)
        bad = np.where(gn | wn, gn != wn, g.view(np.uint32) != w.view(np.uint32))
        if zero_sign_ok is not None:
            bad &= ~(zero_sign_ok & (g == 0) & (w == 0))
    return bad


def assert_same(got, want, what, f16=False, zero_sign_ok=None, f32_nan=None):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = mismatches(got, want, f16, zero_sign_ok, f32_nan)
    n = int(bad.sum())
    if n:
        i = np.flatnonzero(bad.reshape(-1))[:4]
        gb, wb = got.reshape(-1)[i], want.reshape(-1)[i]
        gb, wb = (gb.view(np.uint16), wb.view(np.uint16)) if f16 else (gb.view(np.uint32), wb.view(np.uint32))
        raise AssertionError(f"{what}: {n} of {got.size} elements differ; first at {i.tolist()}: got "
                             f"{[hex(int(v)) for v in gb]} want {[hex(int(v)) for v in wb]}")


def last_kernel(kb):
    return kb._lib.last_kernel()


# ═══ CPU: the file's own generators, comparator and host assumptions ═══════════════════════════════════════════
def test_generators_cover_their_domains():
    n = 1 << 14
    s, wd, hg, tn, z, nf = (gen_f32(k, n, 1) for k in KINDS)
    assert s.min() < -900 and s.max() > 900 and (s < 0).mean() > 0.4
    e = (wd.view(np.uint32) >> 23) & 0xFF
    assert np.isfinite(wd).all() and len(np.unique(e)) == 255 and (wd < 0).mean() > 0.4
    with np.errstate(over="ignore"):
        assert (np.abs(hg) >= 1e37).all() and np.isfinite(hg).all() and np.isinf(hg[:-1] + hg[1:]).any() and np.isinf(hg[:-1] - hg[1:]).any()
    assert ((tn != 0) & (np.abs(tn) < FLT_MIN)).mean() > 0.4 and (np.abs(tn) < 8 * FLT_MIN).all()
    assert (tn[:-1] * tn[1:] == 0).all() and ((tn * F32(0.25) != 0) & (np.abs(tn * F32(0.25)) < FLT_MIN)).any()   # products underflow
    zb = z.view(np.uint32)
    assert (zb == 0).sum() > n // 5 and (zb == 0x80000000).sum() > n // 5 and ((z != 0) & (np.abs(z) < 1e-3)).any()
    assert np.isposinf(nf).any() and np.isneginf(nf).any() and np.isnan(nf).any() and np.isfinite(nf).mean() > 0.95
    assert np.array_equal(gen_f32("wide", 100, 7).view(np.uint32), gen_f32("wide", 100, 7).view(np.uint32))   # seeded
    b = all_bytes(3000, 3)
    assert len(np.unique(b)) == 256
    for name, p in u8_patterns(12, 18, 3).items():
        assert set(np.unique(p).tolist()) <= {0, 255}, name


def test_comparator_is_strict():
    a = np.array([1.0, -0.0, np.nan, 3.0], F32)
    assert not mismatches(a, a.copy()).any()
    assert mismatches(np.array([0.0], F32), np.array([-0.0], F32)).all()                        # zeros differ by sign
    assert not mismatches(np.array([-0.0], F32), np.array([0.0], F32), zero_sign_ok=np.array([True])).any()
    assert mismatches(np.array([np.nan], F32), np.array([1.0], F32)).all()
    assert mismatches(np.array([np.inf], F32), np.array([np.nan], F32)).all()
    assert mismatches(np.array([1.0], F32), np.nextafter(F32(1.0), F32(2.0)).reshape(1)).all()  # one ulp
    x86 = np.array([0xFFC00000], np.uint32).view(F32)
    gpu = np.array([0x7FFFFFFF], np.uint32).view(F32)
    assert not mismatches(gpu, x86).any()                                                       # NaN: "is NaN" only
    h = lambda *v: np.array(v, np.uint16)
    nan = np.array([True, False])
    assert not mismatches(h(0x7E00, 0x3C00), h(0xFE00, 0x3C00), f16=True, f32_nan=nan).any()   # device 0x7E00, oracle x86 NaN
    assert mismatches(h(0x7FFF, 0x3C00), h(0x7E00, 0x3C00), f16=True, f32_nan=nan)[0]          # any other device NaN is wrong
    assert mismatches(h(0x7E00), h(0xFE00), f16=True).all()                  # an f2h NaN pattern of a finite value: exact bits
    assert mismatches(h(0x8000), h(0x0000), f16=True).all() and mismatches(h(0x7C00), h(0x7E00), f16=True).all()


def test_oracle_keeps_subnormals(oracle):
    """The oracle stands as the reference for subnormal data only if its process does not flush them (FTZ / DAZ in
    MXCSR, in the calling thread and in its OpenMP workers)."""
    d = np.full((4, 64, 3), 1e-40, F32)
    assert oracle.normalize_mean_std(d, [0.0] * 3, [1.0] * 3).view(np.uint32).tolist() == d.view(np.uint32).tolist()   # no DAZ
    half = oracle.normalize_mean_std(d, [0.0] * 3, [2.0] * 3)
    assert (half == F32(1e-40) / F32(2.0)).all() and (half != 0).all()                                                  # no FTZ
    t = img_f32("tiny", (64, 96, 3), 5)
    blur = oracle.gaussian_blur(t, (5, 5), (1.5, 1.5), mt=True)
    assert ((blur != 0) & (np.abs(blur) < FLT_MIN)).sum() > 1000


def _rn32(x):
    """Fraction -> the nearest f32 (ties to even), as a Python float; no double rounding."""
    if x == 0:
        return 0.0
    s, x = (-1 if x < 0 else 1), abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    m = x / ulp
    fl = m.numerator // m.denominator
    r = m - fl
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and fl % 2):
        fl += 1
    return s * float(fl * ulp)


C255 = Fraction(float(np.float32(1.0 / 255.0)))   # RN(1/255) = 0x3b808081, the constant of div255_exact


def markstein_div255(p):
    """preprocess.cu div255_exact, restated: q = p*c; e = fma(-q, 255, p); fma(e, c, q), each step rounded once."""
    if not np.isfinite(p):
        q = F32(p) * F32(C255)
        with np.errstate(invalid="ignore"):
            return float(np.float32(np.float32(-q * F32(255) + F32(p)) * F32(C255) + q))   # inf: -inf + inf = NaN
    q = Fraction(_rn32(Fraction(p) * C255))
    e = Fraction(_rn32(-q * 255 + Fraction(p)))
    return _rn32(e * C255 + q)


def ieee_div255(p):
    return float(np.float32(p) / np.float32(255)) if not np.isfinite(p) else _rn32(Fraction(p) / 255)


def test_pad_division_forms():
    """The generic preprocess divides a caller-supplied pad value by 255 with the IEEE division, not with the Markstein
    form it uses for decoded taps.  The Markstein form is exact on [0, 256) (kb200_selftest_div255); its three steps
    scale exactly by powers of two, so it is exact for every finite value.  The only pad values where the two differ
    are the infinities: inf * c = inf, then -inf * 255 + inf = NaN, while inf / 255 = inf."""
    assert _rn32(Fraction(1, 255)) == float(C255)
    rng = np.random.default_rng(0)
    finite = [255.5, -1e3, 256.0, 257.25, 1e4, 3.0e38, -3.0e38, 1e-30, 2.0 ** 100] + [float(F32(v)) for v in rng.uniform(256, 1e6, 200)]
    for p in finite:
        assert markstein_div255(p) == ieee_div255(p), p
    for p in (np.inf, -np.inf):
        assert np.isnan(markstein_div255(p)) and ieee_div255(p) == p


def test_blur_taps_reach_the_u8_bound(oracle):
    """The u8 blur's 16-bit lanes rely on sum(k) <= 256: the 5x5 sigma 1.5 blur of the saturated tests sits on it."""
    q = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(5, 1.5))
    assert int(q.astype(np.int64).sum()) == 256


# ═══ GPU ════════════════════════════════════════════════════════════════════════════════════════════════════════
def stack(fn, src):
    return np.stack([fn(s) for s in src])


# ── f32 resize ──
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_resize_f32_values(kb, oracle, dev, kind):
    n = 2
    cases = [((640, 360, 212, 120), 3, "Bilinear", "resize_rows_f32_kernel"), ((64, 48, 128, 96), 3, "Bilinear", "resize_rows_f32_kernel"),
             ((129, 97, 64, 48), 3, "Bilinear", "resize_f32_c3_kernel"), ((129, 97, 64, 48), 3, "Nearest", "resize_f32_c3_kernel"),
             ((97, 61, 40, 30), 1, "Bilinear", "resize_f32_generic_kernel"), ((97, 61, 40, 30), 4, "Nearest", "resize_f32_generic_kernel"),
             ((129, 97, 64, 48), 3, "Bicubic", "resize_bicubic_c3_kernel"), ((64, 48, 129, 97), 3, "Lanczos", "resize_lanczos_kernels")]
    for (sw, sh, dw, dh), c, mode, kernel in cases:
        src = img_f32(kind, (n, sh, sw, c), sw + c)
        dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), -1.0, c, torch.float32, dev, batch=n)
        kb.imgproc.resize(kb.Image(cu(src, dev)), dst, kb.InterpolationMode[mode])
        assert last_kernel(kb) == kernel, (mode, last_kernel(kb))
        code = {"Nearest": oracle.NEAREST, "Bilinear": oracle.BILINEAR, "Bicubic": oracle.BICUBIC, "Lanczos": oracle.LANCZOS}[mode]
        assert_same(dst.numpy(), stack(lambda s: oracle.resize_f32(s, dw, dh, code), src), f"{kind} resize {mode} c={c} {sw}x{sh}->{dw}x{dh}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_resize_bilinear_normalize_values(kb, oracle, dev, kind):
    sw, sh, dw, dh, n = 640, 360, 320, 180, 2
    src = img_f32(kind, (n, sh, sw, 3), 11)
    for mean, std in (([0.485, 0.456, 0.406], [0.229, 0.224, 0.225]), ([-2.5e38, 1e-3, 0.0], [1e-38, 3e38, -0.5])):
        dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev, batch=n)
        kb.imgproc.resize_bilinear_normalize(kb.Image(cu(src, dev)), dst, mean, std)
        assert last_kernel(kb) == "resize_rows_f32_kernel"
        with np.errstate(all="ignore"):
            inv = F32(1.0) / np.array(std, F32)
            want = ((stack(lambda s: oracle.resize_f32(s, dw, dh), src) - np.array(mean, F32)) * inv).astype(F32)
        assert_same(dst.numpy(), want, f"{kind} resize+normalize mean={mean}")


# ── f32 warps: every dispatch of test_gpu_variants ──
H_GENTLE = [1.02, 0.03, -7.0, -0.03, 1.01, 4.0, 1.2e-5, 7.0e-6, 1.0]
WARP_RUNS = [  # (label, knobs, interpolation, expected kernels)
    ("lean", {"warp.path": 1}, "Bilinear", ("warp_bilinear_lean_kernel",)),
    ("lean-1d", {"warp.path": 1, "a": 7}, "Bilinear", ("warp_bilinear_lean_kernel",)),
    ("general", {"warp.path": 1, "a": 4}, "Bilinear", ("warp_bilinear_lean_kernel/general",)),
    ("stg", {"warp.path": 1, "a": 5}, "Bilinear", ("warp_bilinear_lean_kernel/stg",)),
    ("x4", {"warp.path": 1, "a": 3}, "Bilinear", ("warp_bilinear_x4_kernel",)),
    ("stream2", {"warp.path": 3}, "Bilinear", ("warp_stream2_kernel",)),
    ("stream", {"warp.path": 3}, "Nearest", ("warp_stream_kernel",)),
    ("stream-npx2", {"warp.path": 3, "ws.npx": 2}, "Bilinear", ("warp_stream_kernel",)),
    ("gather64", {"warp.path": 4}, "Bilinear", ("warp_gather64_kernel",)),
    ("gather64-nearest", {"warp.path": 4}, "Nearest", ("warp_gather64_kernel",)),
    ("bicubic", {}, "Bicubic", ("warp_bicubic_kernel",)), ("lanczos", {}, "Lanczos", ("warp_lanczos_kernel",)),
]
ORACLE_MODE = {"Nearest": 0, "Bilinear": 1, "Bicubic": 2, "Lanczos": 3}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_warps_f32_values(kb, oracle, dev, kind):
    sw, sh, n = 640, 360, 2
    src = img_f32(kind, (n, sh, sw, 3), 21)
    t = kb.Image(cu(src, dev))
    m = rot(kb, sw, sh, 2.0, 1.0)
    for label, kn, mode, kernels in WARP_RUNS:
        for op in ("perspective", "affine"):
            fill = 0.0 if mode in ("Bicubic", "Lanczos") else 9.0      # the HQ perspective writes 0 where the oracle leaves dst
            dst = kb.Image.from_size_val(kb.ImageSize(sw, sh), fill, 3, torch.float32, dev, batch=n)
            with knobs(kb, kn):
                if op == "perspective":
                    kb.imgproc.warp_perspective(t, dst, H_GENTLE, kb.InterpolationMode[mode])
                else:
                    kb.imgproc.warp_affine(t, dst, m, kb.InterpolationMode[mode])
                k = last_kernel(kb)
            assert k in kernels, (label, op, k)
            om = ORACLE_MODE[mode]
            fn = (lambda s: oracle.warp_perspective_f32(s, H_GENTLE, sw, sh, om)) if op == "perspective" else (lambda s: oracle.warp_affine_f32(s, m, sw, sh, om))
            assert_same(dst.numpy(), stack(fn, src), f"{kind} warp_{op} {label} ({k})")
    # the TMA-tile kernel: rotations on 16-byte aligned rows
    tw, th = 256, 192
    small = img_f32(kind, (tw * th * 3,), 22).reshape(th, tw, 3)
    for mode in ("Bilinear", "Nearest"):
        mr = rot(kb, tw, th, 30.0)
        dst = kb.Image.from_size_val(kb.ImageSize(tw, th), -3.0, 3, torch.float32, dev)
        kb.imgproc.warp_affine(kb.Image(cu(small, dev)), dst, mr, kb.InterpolationMode[mode])
        assert last_kernel(kb) == "warp_tiled_kernel"
        assert_same(dst.numpy(), oracle.warp_affine_f32(small, mr, tw, th, ORACLE_MODE[mode]), f"{kind} tiled {mode}")


# ── remap ──
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_remap_f32_values(kb, oracle, dev, kind):
    n, sw, sh, dw, dh = 2, 64, 48, 64, 40
    mx, my = _remap_maps(dw, dh, sw, sh, "swirl", np.random.default_rng(3))
    mxi, myi = kb.Image(cu(mx[..., None], dev)), kb.Image(cu(my[..., None], dev))
    src = img_f32(kind, (n, sh, sw, 3), 31)
    want = stack(lambda s: oracle.remap(s, mx, my, 1), src)
    for a, kernel in ((0, "remap_lean_kernel"), (4, "remap_lean_kernel/general"), (6, "remap_f32_c3_kernel")):
        d = kb.Image(torch.full((n, dh, dw, 3), float("nan"), dtype=torch.float32, device=dev))
        with knobs(kb, {"a": a}):
            kb.imgproc.remap(kb.Image(cu(src, dev)), d, mxi, myi, kb.InterpolationMode.Bilinear)
            assert last_kernel(kb) == kernel
        assert_same(d.numpy(), want, f"{kind} remap a={a}")


# ── filters ──
FILTER_SHAPES = [(1100, 40, 1, 1), (700, 37, 3, 1), (97, 61, 3, 2), (33, 50, 4, 1), (5, 5, 1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_filters_f32_values(kb, oracle, dev, kind):
    seen = set()
    for w, h, c, n in FILTER_SHAPES:
        src = img_f32(kind, (n, h, w, c), w + c)
        t = kb.Image(cu(src, dev))
        for op in ("gauss5", "gauss3", "sobel3", "sobel5", "sep"):
            if op == "sobel5" and c == 4:
                continue
            dst = kb.Image.from_size_val(kb.ImageSize(w, h), 9.0, c, torch.float32, dev, batch=n)
            if op.startswith("gauss"):
                k = int(op[-1])
                kb.imgproc.gaussian_blur(t, dst, (k, k), (1.5, 1.5))
                fn = lambda s: oracle.gaussian_blur(s, (k, k), (1.5, 1.5))
            elif op.startswith("sobel"):
                k = int(op[-1])
                kb.imgproc.sobel(t, dst, k)
                fn = lambda s: oracle.sobel(s, k)
            else:   # separable_filter with the gaussian's own taps reaches the same kernels; other taps, negative ones
                kx, ky = [0.25, -0.5, 1.0, 0.5, 0.125], [-1.0, 3.0, -1.0]
                kb.imgproc.separable_filter(t, dst, kx, ky)
                fn = lambda s: oracle.separable_filter(s, kx, ky)
            got_k = last_kernel(kb)
            assert got_k == filter_kernel(w, c, op), (w, c, op, got_k)
            seen.add((got_k, op[:3]))
            assert_same(dst.numpy(), stack(fn, src), f"{kind} {op} {w}x{h}x{c} ({got_k})")
    assert seen >= {(k, o) for k in ("sep_filter_stream2_kernel", "sep_filter_fused_kernel") for o in ("gau", "sob")}, seen


@pytest.mark.gpu
@pytest.mark.parametrize("sw,sh,dw,dh,c,kernel", [(64, 48, 128, 96, 3, "resize_rows_f32_kernel"), (65, 49, 130, 98, 3, "resize_f32_c3_kernel"),
                                                  (65, 49, 130, 98, 1, "resize_f32_generic_kernel")])
def test_resize_f32_bilinear_edge_taps_nonfinite(kb, oracle, dev, sw, sh, dw, dh, c, kernel):
    """At the last source column / row the reference's sampler (interpolation/bilinear.rs) replicates the top-left tap
    for every missing neighbour, the diagonal one included: an inf below or right of it, at weight 0, must not turn the
    result into NaN.  Upscales put many destination pixels on the clamped column and row."""
    n = 2
    src = img_f32("nonfinite", (n, sh, sw, c), sw + c).copy()
    src[:, :, -1, :] = np.where(np.arange(sh)[None, :, None] % 2 == 0, np.inf, -np.inf)   # the last column: +-inf rows
    src[:, -1, :, :] = np.float32(np.nan)                                                  # the last row: NaN
    src[:, -2, -2, :] = np.float32(1.5)
    dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), c, torch.float32, dev, batch=n)
    kb.imgproc.resize(kb.Image(cu(src, dev)), dst, kb.InterpolationMode.Bilinear)
    assert last_kernel(kb) == kernel
    want = stack(lambda s: oracle.resize_f32(s, dw, dh), src)
    assert np.isinf(want).any()
    assert_same(dst.numpy(), want, f"nonfinite edges resize bilinear {sw}x{sh}->{dw}x{dh} c={c}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gradient_magnitude_values(kb, dev, kind):
    """cuda/filter.rs:515-530 sqrtf(a*a + b*b): numpy's f32 operations are each correctly rounded, like the kernel's."""
    n = 1 << 16
    gx, gy = gen_f32(kind, n, 41), gen_f32(kind, n, 42)[::-1].copy()
    dx, dy = cu(gx, dev), cu(gy, dev)
    out = torch.full((n,), 7.0, dtype=torch.float32, device=dev)
    st = kb._lib.lib().kb200_gradient_magnitude_f32(torch.cuda.current_stream(dev).cuda_stream, dx.data_ptr(), dy.data_ptr(), out.data_ptr(), n)
    assert st == 0, kb._lib.last_error()
    assert last_kernel(kb) == "gradient_magnitude_kernel"
    with np.errstate(all="ignore"):
        want = np.sqrt(gx * gx + gy * gy).astype(F32)
    assert_same(out.cpu().numpy(), want, f"{kind} gradient magnitude")


# ── pyramids, gray, normalisation ──
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_pyramids_f32_values(kb, oracle, dev, kind):
    for w, h, c, n in ((53, 37, 3, 2), (640, 360, 3, 1), (7, 5, 4, 1)):
        src = img_f32(kind, (n, h, w, c), 51 + w)
        dn = kb.Image.zeros_cuda(kb.ImageSize((w + 1) // 2, (h + 1) // 2), c, torch.float32, dev, batch=n)
        kb.imgproc.pyrdown(kb.Image(cu(src, dev)), dn)
        assert last_kernel(kb) == "pyrdown_f32_kernel"
        assert_same(dn.numpy().reshape(n, (h + 1) // 2, (w + 1) // 2, c), stack(oracle.pyrdown_f32, src), f"{kind} pyrdown {w}x{h}x{c}")
        up = kb.Image.zeros_cuda(kb.ImageSize(2 * w, 2 * h), c, torch.float32, dev, batch=n)
        kb.imgproc.pyrup(kb.Image(cu(src, dev)), up)
        assert last_kernel(kb) == "pyrup_f32_kernel"
        assert_same(up.numpy().reshape(n, 2 * h, 2 * w, c), stack(oracle.pyrup_f32, src), f"{kind} pyrup {w}x{h}x{c}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gray_f32_values(kb, oracle, dev, kind):
    npx = 4096 * 3
    src = img_f32(kind, (1, npx, 3), 61)
    shifted = cu(np.concatenate([np.zeros(1, F32), src.reshape(-1)]), dev)[1:].reshape(1, npx, 3)   # 4-byte aligned only
    for leaf in (0, 1):
        for t, kernel in ((cu(src, dev), "gray_from_rgb_f32_vec4"), (shifted, "gray_from_rgb_f32_scalar")):
            dst = kb.Image.zeros_cuda(kb.ImageSize(npx, 1), 1, torch.float32, dev)
            kb.imgproc.gray_from_rgb(kb.Image(t), dst, leaf=leaf)
            assert last_kernel(kb) == kernel
            assert_same(dst.numpy(), oracle.gray_from_rgb_f32(src, leaf), f"{kind} gray leaf {leaf} {kernel}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_normalize_mean_std_values(kb, oracle, dev, kind):
    """Both kernels (16-byte aligned C = 3, and the generic one for C = 4 and for the tail), with std = 0 (x / 0 = +-inf,
    0 / 0 = NaN) and extreme statistics."""
    params = [([0.485, 0.456, 0.406, 0.5], [0.229, 0.224, 0.225, 0.25]), ([0.0, -1e3, 3e38, -0.0], [0.0, 1e-30, 1e-38, 0.0]),
              ([-0.0, 0.0, 1e-40, 0.0], [-3e38, 1e38, 1e-45, -1.0])]
    for c, npx, kernel in ((3, 4099, "normalize_mean_std_generic"), (4, 1001, "normalize_mean_std_generic")):
        src = img_f32(kind, (1, npx, c), 71 + c)
        for mean, std in params:
            dst = kb.Image.zeros_cuda(kb.ImageSize(npx, 1), c, torch.float32, dev)
            kb.imgproc.normalize_mean_std(kb.Image(cu(src, dev)), dst, mean[:c], std[:c])
            assert last_kernel(kb) == kernel   # C = 3: 4099 * 3 = 12297 elements, the vector kernel and then the generic one for the tail
            assert_same(dst.numpy(), oracle.normalize_mean_std(src, mean[:c], std[:c]), f"{kind} normalize C={c} {mean} {std}")
    # the vector kernel alone: a whole number of float4
    src = img_f32(kind, (1, 4096, 3), 79)
    for mean, std in params:
        dst = kb.Image.zeros_cuda(kb.ImageSize(4096, 1), 3, torch.float32, dev)
        kb.imgproc.normalize_mean_std(kb.Image(cu(src, dev)), dst, mean[:3], std[:3])
        assert last_kernel(kb) == "normalize_mean_std_c3_vec"
        assert_same(dst.numpy(), oracle.normalize_mean_std(src, mean[:3], std[:3]), f"{kind} normalize vec {mean} {std}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_min_max_values(kb, oracle, dev, kind):
    """find_min_max and normalize_min_max.  The min / max reduction resolves a tie between -0.0 and +0.0 by bit order
    (-0 for the minimum, +0 for the maximum) instead of by first occurrence (normalize.cu:136): where the oracle's
    extreme is a zero of the other sign, the two are numerically equal and the normalised outputs may differ only in
    the sign of an exact zero: (x - min) * range / (max - min) + lo is a zero of either sign exactly where x is a zero
    and lo is 0.  That is the one +-0 difference accepted here, only when such a tie exists and only at those elements
    (DESIGN.md §4, "Exactness shortcuts")."""
    src = img_f32(kind, (61, 97, 3), 81)
    im = kb.Image(cu(src, dev))
    got, want = kb.imgproc.find_min_max(im), oracle.find_min_max(src)
    assert last_kernel(kb) == "minmax_kernel"
    g32, w32 = np.array(got, F32), np.array(want, F32)
    tie = (g32 == 0) & (w32 == 0) & (g32.view(np.uint32) != w32.view(np.uint32))
    assert not mismatches(g32, w32, zero_sign_ok=tie).any(), (got, want)
    if kind != "zeros":
        assert not tie.any(), (got, want)    # a signed-zero extreme needs both zeros in the data
    for lo, hi in ((-1.0, 2.0), (0.0, 1.0), (-3e38, 3e38)):
        dst = kb.Image.zeros_cuda(kb.ImageSize(97, 61), 3, torch.float32, dev)
        kb.imgproc.normalize_min_max(im, dst, lo, hi)
        assert last_kernel(kb) == "normalize_min_max_kernel"
        o = oracle.normalize_min_max(src, lo, hi)
        assert_same(dst.numpy(), o, f"{kind} normalize_min_max [{lo}, {hi}] (extremes {got} / {want})",
                    zero_sign_ok=bool(tie.any()) & (src == 0))


# ── fused resize: f32 scale / bias that overflow, and a -0 bias ──
@pytest.mark.gpu
@pytest.mark.parametrize("leaf", [0, 1])
def test_fused_resize_extreme_scale_bias(kb, oracle, dev, leaf):
    n = 2
    params = [([3e38, 1e37, -2e36], [1e38, -3e38, 0.0]), ([1.0 / 255.0, -1.0, 0.0], [-0.0, -0.0, -0.0]),
              ([0.0, -0.0, 1e-40], [-0.0, 0.0, -1e-41])]
    for (sw, sh, dw, dh), mode in NAMED_FUSED_MODES.items():
        src = np.stack([all_bytes(sw * sh * 3, 90 + i).reshape(sh, sw, 3) for i in range(n)])
        src[:, 0] = 255
        for scale, bias in params:
            out = kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(cu(src, dev), dw, dh, scale, bias, leaf=leaf)
            assert last_kernel(kb) == ("fused_resize_gather_kernel" if mode == "gather" else "fused_rows_kernel")
            want = stack(lambda s: oracle.resize_normalize_u8_to_f32_chw(s, dw, dh, scale, bias, leaf), src)
            assert_same(out.cpu().numpy(), want, f"fused {mode} {sw}x{sh}->{dw}x{dh} leaf {leaf} scale {scale} bias {bias}")


# ── camera preprocess: normalisation parameters and pad values ──
def _q(byte):
    """q = byte / 255 as the device forms it (the IEEE quotient)."""
    return float(F32(byte) / F32(255))


# (name, mean, std or None, inv_std or None, pad_value): std -> Normalize.MeanStd through the builder (inv = 1/std in
# f32); inv_std -> the C ABI only (the builder refuses it)
PARAMS = [
    ("0-255-stats", (123.675, 116.28, 103.53), (58.395, 57.12, 57.375), None, 114.0),
    ("std-1e-5", (0.485, 0.456, 0.406), (1e-5, 1e-5, 1e-5), None, 114.0),
    ("std-1e30", (0.485, 0.456, 0.406), (1e30, 1e30, 1e30), None, 114.0),
    ("std-3e38", (0.0, 0.5, 1.0), (3e38, 3e38, 3e38), None, 0.0),
    ("mean-is-q", (_q(128), _q(0), _q(255)), (0.25, 1e-5, 3.0), None, 128.0),
    ("neg-inv-std", (_q(128), _q(17), _q(255)), None, (-4.0, -1e30, -1.0), 114.0),
    ("inf-inv-std", (_q(128), _q(0), _q(200)), None, (np.inf, -np.inf, np.inf), 114.0),
    ("pad-neg-1e3", (0.485, 0.456, 0.406), None, (4.0, 4.0, 4.0), -1e3),
    ("pad-255.5", (0.485, 0.456, 0.406), None, (1e-5, 1.0, 7.0), 255.5),
    ("pad-inf", (0.0, 0.5, 1.0), None, (1.0, -2.0, 0.5), float("inf")),   # test_pad_division_forms: IEEE inf, Markstein NaN
]
PARAM_IDS = [p[0] for p in PARAMS]


def make_pre(kb, fmt, mode, sampling, param):
    name, mean, std, inv, pad = param
    if std is not None:
        pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode[mode]).sampling(kb.InterpolationMode[sampling])
               .normalize(kb.Normalize.MeanStd(mean, std)).pad_value(int(pad)).build_cuda())
        return pre, pre._mean, pre._inv_std, float(int(pad))
    mean32 = tuple(float(F32(m)) for m in mean)
    inv32 = tuple(float(F32(v)) for v in inv)
    pre = kb.Preprocessor(kb.ResizeMode[mode], kb.InterpolationMode[sampling], kb.SourceFormat[fmt], mean32, inv32, float(F32(pad)), None)
    return pre, mean32, inv32, float(F32(pad))


PRE_KERNELS = [  # (label, fmt, mode, sampling, (w, h, dw, dh), expected kernel)
    ("nv12-identity", "Nv12", "Stretch", "Bilinear", (64, 48, 64, 48), "preprocess_nv12_identity_kernel"),
    ("nv21-identity", "Nv21", "Stretch", "Bilinear", (64, 48, 64, 48), "preprocess_nv21_identity_kernel"),
    ("i420-identity", "I420", "Stretch", "Nearest", (64, 48, 64, 48), "preprocess_i420_identity_kernel"),
    ("yv12-identity", "Yv12", "Stretch", "Bilinear", (64, 48, 64, 48), "preprocess_yv12_identity_kernel"),
    ("nv12-letterbox", "Nv12", "Letterbox", "Bilinear", (64, 48, 40, 40), "preprocess_nv12_kernel"),
    ("nv12-letterbox-nearest", "Nv12", "Letterbox", "Nearest", (96, 54, 32, 32), "preprocess_nv12_kernel"),
    ("rgb8-bilinear", "Rgb8", "Letterbox", "Bilinear", (64, 48, 40, 40), "preprocess_generic_kernel"),
    ("rgb8-nearest", "Rgb8", "Letterbox", "Nearest", (30, 20, 61, 47), "preprocess_generic_kernel"),
    ("yuyv-bilinear", "Yuyv", "Letterbox", "Bilinear", (64, 48, 40, 40), "preprocess_generic_kernel"),
    ("nv12-generic", "Nv12", "Letterbox", "Bilinear", (64, 48, 41, 40), "preprocess_generic_kernel"),
    ("gray-lanczos", "Gray8", "Letterbox", "Lanczos", (64, 48, 40, 40), "preprocess_generic_kernel"),
    ("bayer-identity", "BayerGrbg", "Stretch", "Bilinear", (64, 48, 64, 48), "preprocess_bayer_grbg_identity_kernel"),
    ("bayer-generic", "BayerRggb", "Letterbox", "Bilinear", (64, 48, 40, 40), "preprocess_generic_kernel"),
]
ORACLE_FMT = {"Nv12": 3, "Nv21": 3, "I420": 3, "Yv12": 3, "Rgb8": 0, "Yuyv": 4, "Gray8": 2}


def nv12_to(layout, nv12, w, h):
    """An NV12 frame re-laid as NV21 / I420 / YV12 (the same pixels)."""
    y, uv = nv12[:w * h], nv12[w * h:].reshape(-1, 2)
    if layout == "Nv21":
        return np.concatenate([y, uv[:, ::-1].reshape(-1)])
    if layout == "I420":
        return np.concatenate([y, uv[:, 0], uv[:, 1]])
    if layout == "Yv12":
        return np.concatenate([y, uv[:, 1], uv[:, 0]])
    return nv12


def f2h_bits(oracle, o):
    return np.array([oracle.f2h(float(v)) for v in o.reshape(-1)], np.uint16).reshape(o.shape)


@pytest.mark.gpu
@pytest.mark.parametrize("param", PARAMS, ids=PARAM_IDS)
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_normalisation_values(kb, oracle, dev, param, f16):
    """Every preprocess kernel, f32 and f16, on frames whose bytes cover 0..255, against oracle.preprocess_frame (on the
    NV12 twin for the other 4:2:0 layouts, on the demosaiced RGB twin for Bayer).  Lanczos: the device's own unit-scale
    run gives q = px / 255 exactly (q - 0 = q, q * 1 = q), and the normalisation of q is restated in f32; the sinf of two
    math libraries keeps Lanczos taps from being compared with the oracle bit for bit (test_gpu_variants)."""
    dt = torch.float16 if f16 else torch.float32
    for label, fmt, mode, sampling, (w, h, dw, dh), kernel in PRE_KERNELS:
        bayer = fmt.startswith("Bayer")
        nbytes = {"Rgb8": w * h * 3, "Yuyv": w * h * 2, "Gray8": w * h}.get(fmt, w * h if bayer else w * h * 3 // 2)
        raw = all_bytes(nbytes, 0x5A + len(label))
        frame = nv12_to(fmt, raw, w, h) if fmt in ("Nv21", "I420", "Yv12") else raw
        pre, mean, inv, pad = make_pre(kb, fmt, mode, sampling, param)
        got = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
        (pre.run_raw_f16 if f16 else pre.run_raw)(cu(frame, dev), w, h, got)
        assert last_kernel(kb) == kernel, (label, last_kernel(kb))
        what = f"{param[0]} {label} {'f16' if f16 else 'f32'}"
        om = oracle.LETTERBOX if mode == "Letterbox" else oracle.STRETCH
        if bayer:
            src, code = demosaic(raw.reshape(h, w), fmt[5:].upper()).reshape(-1), oracle.FMT_RGB
        else:
            src, code = raw, ORACLE_FMT[fmt]
        if sampling == "Lanczos":
            unit = kb.Preprocessor(kb.ResizeMode[mode], kb.InterpolationMode.Lanczos, kb.SourceFormat[fmt], (0.0,) * 3, (1.0,) * 3, pad, None)
            q = torch.full((1, 3, dh, dw), float("nan"), dtype=torch.float32, device=dev)
            unit.run_raw(cu(frame, dev), w, h, q)
            with np.errstate(all="ignore"):
                o = ((q[0].cpu().numpy() - np.array(mean, F32)[:, None, None]) * np.array(inv, F32)[:, None, None]).astype(F32)
            want = f2h_bits(oracle, o) if f16 else o
        else:
            cfg = oracle.PreprocessCfg(mode=om, fmt=code, mean=mean, inv_std=inv, pad_value=pad,
                                       sampling=oracle.BILINEAR if sampling == "Bilinear" else oracle.NEAREST)
            want = oracle.preprocess_frame(src, cfg, w, h, dw, dh, f16=f16)
            o = oracle.preprocess_frame(src, cfg, w, h, dw, dh) if f16 else want
        g = got[0].cpu().numpy()
        assert_same(g.view(np.uint16) if f16 else g, want.view(np.uint16) if f16 else want, what, f16=f16, f32_nan=np.isnan(o))


@pytest.mark.gpu
@pytest.mark.parametrize("param", PARAMS, ids=PARAM_IDS)
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_bayer16_normalisation_values(kb, oracle, dev, param, f16):
    """The 16-bit Bayer identity kernel and the generic Bayer16 kernel against the f32 restatement in restate.py
    (samples over the whole 12-bit range), converted to f16 by the oracle's f2h (the reference's conversion rules)."""
    w, h, bits = 64, 48, 12
    raw = np.random.default_rng(0xB16).permutation(np.resize(np.arange(1 << bits, dtype=np.uint16), w * h))
    raw[:8] = (1 << bits) - 1
    raw[8:16] = 0
    for mode, sampling, (dw, dh), kernel in (("Stretch", "Bilinear", (64, 48), "preprocess_bayer16_rggb_identity_kernel"),
                                             ("Letterbox", "Bilinear", (40, 40), "preprocess_generic_kernel"),
                                             ("Letterbox", "Nearest", (61, 47), "preprocess_generic_kernel")):
        pre, mean, inv, pad = make_pre(kb, "BayerRggb12", mode, sampling, param)
        got = torch.full((1, 3, dh, dw), float("nan"), dtype=torch.float16 if f16 else torch.float32, device=dev)
        (pre.run_raw_f16 if f16 else pre.run_raw)(torch.from_numpy(raw.astype(np.int32)).to(dev).to(torch.uint16), w, h, got)
        assert last_kernel(kb) == kernel
        a = (C.c_float * 4)()
        kb._lib.lib().kb200_preprocess_affine(kb.ResizeMode[mode].value, w, h, dw, dh, a)
        with np.errstate(all="ignore"):
            o = preprocess_rgb16(demosaic(raw.reshape(h, w), "RGGB"), bits, tuple(a), dw, dh, sampling, mean, inv, pad)
        g = got[0].cpu().numpy()
        assert_same(g.view(np.uint16) if f16 else g, f2h_bits(oracle, o) if f16 else o, f"{param[0]} bayer16 {mode} {sampling}", f16=f16,
                    f32_nan=np.isnan(o))


@pytest.mark.gpu
def test_preprocess_f16_nan_is_canonical_0x7e00(kb, dev):
    """0 * inf in the normalisation gives the device's canonical NaN; its f16 store writes 0x7E00 on every kernel: the
    identity kernels and the 4:2:0 letterbox kernel through nv12_store4, the generic kernel through f2h_ref."""
    w, h = 64, 48
    nv12 = np.full(w * h * 3 // 2, 128, np.uint8)
    nv12[:w * h] = 16                                     # Y = 16, U = V = 128: black, every channel decodes to 0
    rgb = np.zeros(w * h * 3, np.uint8)
    for fmt, frame, mode, dwh in (("Nv12", nv12, "Stretch", (64, 48)), ("Nv12", nv12, "Letterbox", (40, 40)), ("Rgb8", rgb, "Letterbox", (40, 40))):
        pre, *_ = make_pre(kb, fmt, mode, "Bilinear", ("nan", (0.0,) * 3, None, (np.inf,) * 3, 114.0))
        got = torch.zeros((1, 3, dwh[1], dwh[0]), dtype=torch.float16, device=dev)
        pre.run_raw_f16(cu(frame, dev), w, h, got)
        assert last_kernel(kb) == {"Stretch": "preprocess_nv12_identity_kernel", "Letterbox": "preprocess_nv12_kernel"}[mode] if fmt == "Nv12" \
            else last_kernel(kb) == "preprocess_generic_kernel"
        bits = got.cpu().numpy().view(np.uint16)
        content = bits[:, 10:30] if mode == "Letterbox" else bits     # 64x48 letterboxed into 40x40: rows 5..34 are content
        assert _f16_nan(content).all(), (fmt, mode, "(0 / 255 - 0) * inf")
        assert (content == F16_NAN).all(), (fmt, mode, np.unique(content))


# ── saturated u8 frames ──
@pytest.mark.gpu
def test_u8_kernels_on_saturated_frames(kb, oracle, dev):
    """All-0, all-255, 0/255 checkerboards, stripes of period 2 and 3 and single impulses through the Q14 resizes, the
    u8 warps (interior and clamped samplers), remap_u8, the u8 blurs (streaming and tile), the u8 pyramids and gray."""
    h, w, c = 72, 96, 3
    pats = u8_patterns(h, w, c)
    names = list(pats)
    src = np.stack([pats[k] for k in names])
    n = len(names)
    t = kb.Image(cu(src, dev))

    def check(d, fn, what):
        want = stack(fn, src)
        got = d.numpy().reshape(want.shape)
        for i in range(n):
            np.testing.assert_array_equal(got[i], want[i], err_msg=f"{what}: {names[i]}")

    for (dw, dh), kernel in (((40, 30), "resize_bilinear_u8_kernel"), ((32, 24), "resize_bilinear_u8_c3_3to1_kernel"),
                             ((48, 36), "pyrdown_2x_rgb_u8_w4_kernel"), ((192, 144), "pyrup_2x_rgb_u8_kernel"), ((31, 23), "resize_bilinear_u8_kernel")):
        d = kb.Image(torch.full((n, dh, dw, c), 0xCD, dtype=torch.uint8, device=dev))
        kb.imgproc.resize_fast_u8(t, d, kb.InterpolationMode.Bilinear)
        assert last_kernel(kb) == kernel
        check(d, lambda s: oracle.resize_fast_u8(s, dw, dh, 1), f"resize_fast_u8 -> {dw}x{dh}")
    for b in (0, 1):   # knob b = 1: the clamped sampler everywhere
        with knobs(kb, {"b": b}):
            for m in ([1, 0, 0.5, 0, 1, 0.5], [1.01, 0.02, -3.0, -0.015, 0.99, 2.5], [0.5, 0, 0, 0, 0.5, 0]):
                d = kb.Image(torch.full((n, h, w, c), 0xCD, dtype=torch.uint8, device=dev))
                kb.imgproc.warp_affine_u8(t, d, m)
                assert last_kernel(kb) == "warp_affine_u8_kernel"
                check(d, lambda s: oracle.warp_affine_u8(s, w, h, m), f"warp_affine_u8 {m} b={b}")
            for hm in ([1, 0, 0.5, 0, 1, 0.5, 0, 0, 1], [1.02, 0.03, -5.0, -0.03, 1.01, 2.0, 0.00005, 0.00003, 1.0]):
                d = kb.Image(torch.full((n, h, w, c), 0xCD, dtype=torch.uint8, device=dev))
                kb.imgproc.warp_perspective_u8(t, d, hm)
                assert last_kernel(kb) == "warp_perspective_u8_kernel"
                check(d, lambda s: oracle.warp_perspective_u8(s, w, h, hm), f"warp_perspective_u8 {hm} b={b}")
            y, x = np.meshgrid(np.arange(h, dtype=F32), np.arange(w, dtype=F32), indexing="ij")
            for mx, my in ((x + F32(0.5), y + F32(0.5)), (x * F32(0.999) + F32(0.25), y * F32(1.001) - F32(0.375))):
                d = kb.Image(torch.full((n, h, w, c), 0xCD, dtype=torch.uint8, device=dev))
                kb.imgproc.remap_u8(t, d, kb.Image(cu(mx[..., None], dev)), kb.Image(cu(my[..., None], dev)), kb.InterpolationMode.Bilinear)
                assert last_kernel(kb) == "remap_u8_kernel"
                check(d, lambda s: oracle.remap(s, mx, my, 1), f"remap_u8 b={b}")
    assert int(oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(5, 1.5)).astype(np.int64).sum()) == 256
    for k, sig in ((5, 1.5), (3, 0.8), (7, 2.0)):
        for b, kernels in ((0, ("blur_u8_stream_kernel",)), (3, ("blur_u8_tile_w_kernel", "blur_u8_tile_kernel"))):
            d = kb.Image(torch.full((n, h, w, c), 0xCD, dtype=torch.uint8, device=dev))
            with knobs(kb, {"b": b}):
                kb.imgproc.gaussian_blur_u8(t, d, (k, k), (sig, sig))
                assert last_kernel(kb) in kernels
            check(d, lambda s: oracle.gaussian_blur_u8(s, (k, k), (sig, sig)), f"gaussian_blur_u8 k={k} b={b}")
    dn = kb.Image.zeros_cuda(kb.ImageSize(w // 2, h // 2), c, torch.uint8, dev, batch=n)
    kb.imgproc.pyrdown(t, dn)
    assert last_kernel(kb) == "pyrdown_u8_kernel"
    check(dn, oracle.pyrdown_u8, "pyrdown_u8")
    up = kb.Image.zeros_cuda(kb.ImageSize(2 * w, 2 * h), c, torch.uint8, dev, batch=n)
    kb.imgproc.pyrup(t, up)
    assert last_kernel(kb) == "pyrup_u8_kernel"
    check(up, oracle.pyrup_u8, "pyrup_u8")
    g = kb.Image.zeros_cuda(kb.ImageSize(w, h), 1, torch.uint8, dev, batch=n)
    kb.imgproc.gray_from_rgb(t, g)
    assert last_kernel(kb) == "gray_from_rgb_u8_vec16"
    check(g, oracle.gray_from_rgb_u8, "gray_from_rgb_u8")


# ── every (Y, U, V) triple ──
YUV_W = YUV_H = 512
YUV_FRAMES = 64


def nv12_all_triples(f):
    """Frame f of 64: chroma sample (cx, cy) = (U, V), so each frame holds all 2^16 pairs; its 2x2 luma block is
    4f + {0, 1, 2, 3}, so the 64 frames give every pair with every luma value."""
    yy, xx = np.mgrid[0:YUV_H, 0:YUV_W]
    y = (4 * f + (xx & 1) + 2 * (yy & 1)).astype(np.uint8)
    cy, cx = np.mgrid[0:YUV_H // 2, 0:YUV_W // 2]
    uv = np.stack([cx, cy], -1).astype(np.uint8)
    return np.concatenate([y.reshape(-1), uv.reshape(-1)])


def yuyv_all_triples(f):
    """Frame f of 64: group g of row r carries U = g, V = r % 256 and the luma 4f + 2 (r // 256) + {0, 1}."""
    r, g = np.mgrid[0:YUV_H, 0:YUV_W // 2]
    y0 = (4 * f + 2 * (r // 256)).astype(np.uint8)
    return np.stack([y0, g.astype(np.uint8), y0 + 1, (r % 256).astype(np.uint8)], -1).reshape(-1)


def test_all_triples_layouts_cover_every_triple():
    seen = np.zeros((256, 256, 256), bool)
    for f in range(YUV_FRAMES):
        fr = nv12_all_triples(f)
        y = fr[:YUV_W * YUV_H].reshape(YUV_H, YUV_W)
        uv = fr[YUV_W * YUV_H:].reshape(YUV_H // 2, YUV_W // 2, 2)
        for dy in (0, 1):
            for dx in (0, 1):
                seen[y[dy::2, dx::2], uv[..., 0], uv[..., 1]] = True
    assert seen.all()
    seen[:] = False
    for f in range(YUV_FRAMES):
        g = yuyv_all_triples(f).reshape(YUV_H, YUV_W // 2, 4)
        seen[g[..., 0], g[..., 1], g[..., 3]] = True
        seen[g[..., 2], g[..., 1], g[..., 3]] = True
    assert seen.all()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["Nv12", "Yuyv"])
def test_yuv_every_triple(kb, oracle, dev, fmt):
    """The decoder and the identity preprocess (f32, unit scale) on 64 frames holding every (Y, U, V) triple."""
    make, decode, ofmt = ((nv12_all_triples, kb.imgproc.rgb_from_nv12, oracle.FMT_NV12) if fmt == "Nv12" else
                          (yuyv_all_triples, kb.imgproc.rgb_from_yuyv, oracle.FMT_YUYV))
    n, w, h = YUV_FRAMES, YUV_W, YUV_H
    raw = torch.from_numpy(np.stack([make(f) for f in range(n)])).to(dev)
    rgb = kb.Image(torch.full((n, h, w, 3), 0xCD, dtype=torch.uint8, device=dev))
    decode(raw, rgb)
    assert last_kernel(kb) == f"rgb_from_{fmt.lower()}_vec16"
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode.Stretch).build_cuda()
    out = torch.full((n, 3, h, w), float("nan"), dtype=torch.float32, device=dev)
    pre.run_raw_batch([raw[i] for i in range(n)], w, h, out)
    assert last_kernel(kb) == ("preprocess_nv12_identity_kernel" if fmt == "Nv12" else "preprocess_generic_kernel")
    del raw
    dec = oracle.rgb_from_nv12 if fmt == "Nv12" else oracle.rgb_from_yuyv
    cfg = oracle.PreprocessCfg(mode=oracle.STRETCH, fmt=ofmt)
    compare_frames(oracle, n, lambda f: (dec(make(f), w, h), oracle.preprocess_frame(make(f), cfg, w, h, w, h).view(np.uint32)),
                   lambda f: (rgb.data[f].cpu().numpy(), out[f].cpu().numpy().view(np.uint32)), "exact", f"{fmt} every triple")
    del rgb, out
    free_device_memory()


@pytest.mark.gpu
@pytest.mark.parametrize("leaf", [0, 1])
def test_normalize_rgb_u8_every_byte(kb, oracle, dev, leaf):
    """Every byte value in every channel, with the bulk / tail split of the leaf (npixels not a multiple of 8)."""
    npx = 256 * 3 + 4         # whole words: the vector kernel runs last; npx % 8 = 4 leaves a non-FMA tail in the x86 leaf
    i = np.arange(npx)
    src = np.stack([i % 256, (i + 85) % 256, (255 - i) % 256], -1).astype(np.uint8).reshape(-1)
    for scale, off in (([1 / (0.229 * 255), 1 / (0.224 * 255), 1 / (0.225 * 255)], [-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225]),
                       ([3e36, -1e38, 1e-40], [-3e38, 0.0, -0.0]), ([0.0, -0.0, 1.0], [-0.0, -0.0, -255.0])):
        for base, kernel in ((cu(src, dev), "normalize_rgb_u8_vec"), (cu(np.concatenate([[0], src]).astype(np.uint8), dev)[1:], "normalize_rgb_u8_generic")):
            dst = torch.full((npx * 3,), float("nan"), dtype=torch.float32, device=dev)
            kb.imgproc.normalize_rgb_u8(base, dst, npx, scale, off, leaf=leaf)
            assert last_kernel(kb) == kernel
            assert_same(dst.cpu().numpy(), oracle.normalize_rgb_u8(src, scale, off, leaf).reshape(-1), f"normalize_rgb_u8 leaf {leaf} {scale} {kernel}")


# ── std_mean at and past its integer bounds ──
STD_MEAN_BLOCK, STD_MEAN_CTAS_PER_SM, STD_MEAN_FLUSH = 256, 6, 8192
SQ_PER_VECTOR = 255 * 255 * 6      # a 16-byte vector holds at most 6 bytes of one channel


def std_mean_threads(nvec, sm):
    """stream_grid3(nvec, 256, 6) (normalize.cu) x 256."""
    g = max(1, min(-(-nvec // STD_MEAN_BLOCK), sm * STD_MEAN_CTAS_PER_SM))
    return (g + 2) // 3 * 3 * STD_MEAN_BLOCK


def std_mean_sums_of(kb, dev, t, npx):
    sums = torch.empty(6, dtype=torch.int64, device=dev)
    st = kb._lib.lib().kb200_std_mean_u8_c3(torch.cuda.current_stream(dev).cuda_stream, t.data_ptr(), npx, sums.data_ptr())
    assert st == 0, kb._lib.last_error()
    assert last_kernel(kb) == "std_mean_kernel"
    return [int(v) for v in sums.tolist()]


@pytest.mark.gpu
def test_std_mean_saturated_4k_x16_unaligned(kb, dev):
    """All-255 4K x16 from a base 1 byte past an aligned allocation: the 15-byte head peel and the body, every channel at
    255: sums n*255 and n*255^2 in closed form."""
    npx = 16 * 3840 * 2160
    buf = torch.full((npx * 3 + 1,), 255, dtype=torch.uint8, device=dev)
    assert std_mean_sums_of(kb, dev, buf[1:], npx) == [npx * 255] * 3 + [npx * 255 * 255] * 3
    del buf
    free_device_memory()


@pytest.mark.gpu
def test_std_mean_past_the_accumulator_flush(kb, dev):
    """12,288 vectors per thread of all-255 data (about 40 GB): a thread's 32-bit square sum would wrap after
    2^32 / (255^2 * 6) = 11,008 vectors, so the sums are right only if the accumulators are flushed at 8192 vectors
    (a flush point of 16384 would wrap them).  The regime is computed from the launcher's grid and the SM count.  No
    other test reaches the flush, so the test fails, rather than skips, when the device lacks the memory."""
    sm = torch.cuda.get_device_properties(dev).multi_processor_count
    per_thread = 12288
    threads = std_mean_threads(1 << 40, sm)
    nvec = per_thread * threads
    assert std_mean_threads(nvec, sm) == threads
    assert STD_MEAN_FLUSH <= per_thread and per_thread * SQ_PER_VECTOR >= 1 << 32 and (per_thread // 2) * SQ_PER_VECTOR < 1 << 32
    assert STD_MEAN_FLUSH * SQ_PER_VECTOR < 1 << 32 < 16384 * SQ_PER_VECTOR and per_thread < 16384
    nbytes = 16 * nvec
    assert nbytes % 3 == 0
    free_device_memory()
    free, _ = torch.cuda.mem_get_info(dev)
    assert free >= nbytes + (1 << 30), f"needs {nbytes / 1e9:.1f} GB of free device memory, {free / 1e9:.1f} GB free"
    buf = torch.full((nbytes,), 255, dtype=torch.uint8, device=dev)
    try:
        npx = nbytes // 3
        assert buf.data_ptr() % 16 == 0
        assert std_mean_sums_of(kb, dev, buf, npx) == [npx * 255] * 3 + [npx * 255 * 255] * 3
    finally:
        del buf
        free_device_memory()
