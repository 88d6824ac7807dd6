"""Cross-check against the REFERENCE'S OWN CUDA kernels.

Every case compares this library's output with a SHA-256 digest stored in tests/golden/ref_gpu_kernels.json (float32
outputs with -0.0 folded to +0.0, as the bit comparison below treats them; other dtypes byte for byte).  Each stored
digest is the digest of the reference kernel's output for that case: the cases matched the reference's kernels bit for
bit, and the digests were recorded from this library on the same inputs.

When `baseline/_ref/` has been built (baseline/extract_ref_kernels.py, from the kornia-rs checkout $KORNIA_RS_SRC names),
the reference's kernels are also run here with the reference's launch geometry (baseline/ref_gpu.py): our output must
then have the SAME BITS as theirs, and their output must match the stored digest.

KB_RECORD_REF_DIGESTS=<file> records the digest of every case that has none stored (the reference kernel's output when
it is available, else this library's) as JSON lines in <file> instead of failing.
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "baseline"))
DIGESTS = os.path.join(ROOT, "tests", "golden", "ref_gpu_kernels.json")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ref(dev):
    """The reference's kernels, or None when baseline/_ref/ was not built (the stored digests still apply)."""
    import ref_gpu

    return ref_gpu.RefGpu(0) if ref_gpu.available() else None


@pytest.fixture(scope="module")
def digests():
    with open(DIGESTS) as f:
        return json.load(f)


@pytest.fixture
def check(request, digests):
    """check(got, want_or_None, what): the output's stored digest (and the reference kernel's bits, when run) must match."""
    seen = []

    def run(got: torch.Tensor, want, what=""):
        if want is not None:
            same_bits(got, want, what)
        seen.append(None)
        case = f"{request.node.name}#{len(seen)}"      # a test may check several outputs, in a fixed order
        d = digest(want if want is not None else got)
        stored = digests.get(case)
        rec = os.environ.get("KB_RECORD_REF_DIGESTS")
        if stored is None and rec:
            with open(rec, "a") as f:
                f.write(json.dumps({case: d}) + "\n")
            return
        assert stored is not None, f"{case}: no digest stored in {os.path.relpath(DIGESTS, ROOT)}"
        assert d == stored, f"{what}: output digest {d[:16]}... differs from the reference kernel's ({stored[:16]}...) ({case})"

    return run


def digest(t: torch.Tensor) -> str:
    a = np.ascontiguousarray(t.detach().cpu().numpy())
    if a.dtype == np.float32:
        a = np.where(a == 0, np.float32(0), a)      # -0.0 -> +0.0
    return hashlib.sha256(a.tobytes()).hexdigest()


def cu(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def same_bits(a: torch.Tensor, b: torch.Tensor, what=""):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    if a.dtype == np.float32:
        neq = (a.view(np.uint32) != b.view(np.uint32)) & ~((a == 0) & (b == 0))
    else:
        neq = a != b
    assert not neq.any(), f"{what}: {int(neq.sum())} of {a.size} elements differ from the reference kernel (max abs {np.abs(a.astype(np.float64) - b.astype(np.float64)).max()})"


@pytest.mark.parametrize("sw,sh,dw,dh", [(384, 216, 128, 72), (640, 360, 320, 180), (640, 360, 213, 120), (129, 97, 64, 48), (64, 48, 129, 97)])
def test_resize_bilinear_matches_reference_kernel(kb, oracle, ref, dev, check, sw, sh, dw, dh):
    n = 2
    src = cu(oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3), dev)
    want = torch.zeros((n, dh, dw, 3), dtype=torch.float32, device=dev)
    if ref is not None:
        ref.resize_bilinear(src, want)
    got = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev, batch=n)
    kb.imgproc.resize(kb.Image(src), got, kb.InterpolationMode.Bilinear)
    check(got.data, want if ref is not None else None, f"resize {sw}x{sh}->{dw}x{dh}")


H_CASES = [((129, 97), [1.03, 0.05, -3.0, -0.02, 0.97, 4.0, 2.0 / (97 * 129), 1.5 / (129 * 97), 1.0]),
           ((320, 240), [0.9, 0.15, 10.0, -0.1, 1.1, -6.0, 0.0, 0.0, 1.0]),
           ((640, 360), [1.02, 0.03, -7.0, -0.03, 1.01, 4.0, 1.2e-5, 7.0e-6, 1.0]),
           ((256, 192), [0.8, 0.45, -20.0, -0.5, 0.85, 60.0, 1.0e-4, -6.0e-5, 1.0])]


@pytest.mark.parametrize("size,h", H_CASES)
@pytest.mark.parametrize("interp", ["bilinear", "nearest"])
def test_warp_perspective_matches_reference_kernel(kb, oracle, ref, dev, check, size, h, interp):
    sw, sh = size
    src = cu(oracle.pattern_f32(sw * sh * 3).reshape(1, sh, sw, 3), dev)
    want = torch.full((1, sh, sw, 3), 3.0, dtype=torch.float32, device=dev)
    if ref is not None:
        ref.warp("perspective", interp, src, want, oracle.invert_homography(h))
    got = kb.Image.from_size_val(kb.ImageSize(sw, sh), 3.0, 3, torch.float32, dev)
    kb.imgproc.warp_perspective(kb.Image(src[0]), got, h, kb.InterpolationMode.Bilinear if interp == "bilinear" else kb.InterpolationMode.Nearest)
    check(got.data.reshape(want.shape), want if ref is not None else None, f"warp_perspective {interp} {size} ({kb._lib.last_kernel()})")


@pytest.mark.parametrize("size,angle", [((128, 96), 30.0), ((256, 192), -17.5), ((97, 61), 45.0), ((640, 360), 3.0)])
@pytest.mark.parametrize("interp", ["bilinear", "nearest"])
def test_warp_affine_matches_reference_kernel(kb, oracle, ref, dev, check, size, angle, interp):
    sw, sh = size
    src = cu(oracle.pattern_f32(sw * sh * 3).reshape(1, sh, sw, 3), dev)
    m = kb.imgproc.get_rotation_matrix2d((sw / 2.0, sh / 2.0), angle, 1.0)
    want = torch.full((1, sh, sw, 3), 3.0, dtype=torch.float32, device=dev)
    if ref is not None:
        ref.warp("affine", interp, src, want, oracle.invert_affine_transform(m))
    got = kb.Image.from_size_val(kb.ImageSize(sw, sh), 3.0, 3, torch.float32, dev)
    kb.imgproc.warp_affine(kb.Image(src[0]), got, m, kb.InterpolationMode.Bilinear if interp == "bilinear" else kb.InterpolationMode.Nearest)
    check(got.data.reshape(want.shape), want if ref is not None else None, f"warp_affine {interp} {size} {angle} ({kb._lib.last_kernel()})")


@pytest.mark.parametrize("w,h,c", [(97, 61, 3), (700, 37, 3), (1100, 40, 1), (520, 33, 4)])
@pytest.mark.parametrize("k", [3, 5, 7])
def test_gaussian_blur_matches_reference_kernels(kb, oracle, ref, dev, check, w, h, c, k):
    src = cu(oracle.pattern_f32(w * h * c).reshape(1, h, w, c), dev)
    taps = oracle.gaussian_kernel_1d(k, 1.5).tolist()
    want, scratch = torch.zeros_like(src), torch.zeros_like(src[0])
    if ref is not None:
        ref.separable_filter(src, want, scratch, taps, taps)
    got = kb.Image.zeros_cuda(kb.ImageSize(w, h), c, torch.float32, dev)
    kb.imgproc.gaussian_blur(kb.Image(src[0]), got, (k, k), (1.5, 1.5))
    check(got.data.reshape(want.shape), want if ref is not None else None, f"gaussian k={k} {w}x{h}x{c} ({kb._lib.last_kernel()})")


@pytest.mark.parametrize("w,h,c", [(97, 61, 3), (700, 37, 3), (1100, 40, 1)])
@pytest.mark.parametrize("ksize", [3, 5])
def test_sobel_matches_reference_kernels(kb, oracle, ref, dev, check, w, h, c, ksize):
    src = cu(oracle.pattern_f32(w * h * c).reshape(1, h, w, c), dev)
    want, scratch = torch.zeros_like(src), torch.zeros_like(src[0])
    gx, gy = torch.zeros_like(src), torch.zeros_like(src)
    if ref is not None:
        ref.sobel(src, want, scratch, gx, gy, ksize)
    got = kb.Image.zeros_cuda(kb.ImageSize(w, h), c, torch.float32, dev)
    kb.imgproc.sobel(kb.Image(src[0]), got, ksize)
    check(got.data.reshape(want.shape), want if ref is not None else None, f"sobel k={ksize} {w}x{h}x{c}")


def test_gray_and_nv12_match_reference_kernels(kb, oracle, ref, dev, check):
    w, h = 320, 180
    f = cu(oracle.pattern_f32(w * h * 3).reshape(1, h, w, 3), dev)
    want = torch.zeros((1, h, w, 1), dtype=torch.float32, device=dev)
    if ref is not None:
        ref.gray_f32(f, want)
    got = kb.Image.zeros_cuda(kb.ImageSize(w, h), 1, torch.float32, dev)
    kb.imgproc.gray_from_rgb(kb.Image(f[0]), got)   # LEAF_SCALAR = the CUDA kernel's expression
    check(got.data.reshape(want.shape), want if ref is not None else None, "gray f32")
    u = cu(oracle.pattern_u8(w * h * 3).reshape(1, h, w, 3), dev)
    want8 = torch.zeros((1, h, w, 1), dtype=torch.uint8, device=dev)
    if ref is not None:
        ref.gray_u8(u, want8)
    got8 = kb.Image.zeros_cuda(kb.ImageSize(w, h), 1, torch.uint8, dev)
    kb.imgproc.gray_from_rgb(kb.Image(u[0]), got8)
    check(got8.data.reshape(want8.shape), want8 if ref is not None else None, "gray u8")
    n = 2
    raw = cu(oracle.pattern_u8(n * w * h * 3 // 2, 0xC0FFEE).reshape(n, w * h * 3 // 2), dev)
    wantrgb = torch.zeros((n, h, w, 3), dtype=torch.uint8, device=dev)
    if ref is not None:
        ref.rgb_from_nv12(raw, wantrgb, w, h)
    gotrgb = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n)
    kb.imgproc.rgb_from_nv12(raw, gotrgb)
    check(gotrgb.data, wantrgb if ref is not None else None, "nv12")


def raw_bytes(n, k):
    i = np.arange(n, dtype=np.int64)
    return (((i * 7 + 13) % 251) + 31 * k).astype(np.uint8)


@pytest.mark.parametrize("mode,dw,dh", [("Stretch", 192, 108), ("Letterbox", 64, 64), ("Letterbox", 100, 60), ("Stretch", 77, 41)])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_nv12_matches_reference_kernel(kb, oracle, ref, dev, check, mode, dw, dh, f16):
    """The camera preprocess has no CPU implementation: the reference's CUDA source IS the spec — run it."""
    w, h, n = 192, 108, 3
    frames = [cu(raw_bytes(w * h * 3 // 2, k), dev) for k in range(n)]
    inv = [float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD]
    aff = oracle.preprocess_affine(oracle.LETTERBOX if mode == "Letterbox" else oracle.STRETCH, w, h, dw, dh)
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float16 if f16 else torch.float32, device=dev)
    if ref is not None:
        ref.preprocess(frames, w, h, want, aff, kb.IMAGENET_MEAN, inv, 114.0, fmt=3, bpp=1, sampler="bilinear", f16=f16)
    pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda())
    got = torch.zeros_like(want)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)(frames, w, h, got)
    if f16:
        check(got.view(torch.int16), want.view(torch.int16) if ref is not None else None, f"preprocess f16 {mode} {dw}x{dh}")
    else:
        check(got, want if ref is not None else None, f"preprocess {mode} {dw}x{dh}")


# ── bicubic / Lanczos: the reference's own kernels are the byte-exact spec (interpolation/bicubic.rs:1-8) ──────
@pytest.mark.parametrize("sw,sh,dw,dh", [(129, 97, 64, 48), (64, 48, 129, 97), (320, 180, 213, 120), (40, 30, 40, 77)])
def test_resize_bicubic_and_lanczos_match_reference_kernels(kb, oracle, ref, dev, check, sw, sh, dw, dh):
    n = 2
    src = cu(oracle.pattern_f32(n * sw * sh * 3).reshape(n, sh, sw, 3), dev)
    want = torch.zeros((n, dh, dw, 3), dtype=torch.float32, device=dev)
    if ref is not None:
        ref.resize_bilinear(src, want, kernel="resize_bicubic_3c")
    got = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev, batch=n)
    kb.imgproc.resize(kb.Image(src), got, kb.InterpolationMode.Bicubic)
    check(got.data, want if ref is not None else None, f"bicubic {sw}x{sh}->{dw}x{dh}")
    x0s, wx = oracle.lanczos_axis(sw, dw)
    y0s, wy = oracle.lanczos_axis(sh, dh)
    inter = torch.zeros((sh, dw, 3), dtype=torch.float32, device=dev)
    if ref is not None:
        ref.resize_lanczos(src, want, inter, cu(x0s, dev), cu(wx, dev), cu(y0s, dev), cu(wy, dev))
    kb.imgproc.resize(kb.Image(src), got, kb.InterpolationMode.Lanczos)
    check(got.data, want if ref is not None else None, f"lanczos {sw}x{sh}->{dw}x{dh}")


@pytest.mark.parametrize("interp", ["bicubic", "lanczos"])
@pytest.mark.parametrize("size,h", H_CASES)
def test_warp_perspective_hq_matches_reference_kernel(kb, oracle, ref, dev, check, size, h, interp):
    sw, sh = size
    src = cu(oracle.pattern_f32(sw * sh * 3).reshape(1, sh, sw, 3), dev)
    want = torch.full((1, sh, sw, 3), 3.0, dtype=torch.float32, device=dev)
    if ref is not None:
        ref.warp("perspective", interp, src, want, oracle.invert_homography(h))
    got = kb.Image.from_size_val(kb.ImageSize(sw, sh), 3.0, 3, torch.float32, dev)
    kb.imgproc.warp_perspective(kb.Image(src[0]), got, h, kb.InterpolationMode.Bicubic if interp == "bicubic" else kb.InterpolationMode.Lanczos)
    check(got.data.reshape(want.shape), want if ref is not None else None, f"warp_perspective {interp} {size}")


@pytest.mark.parametrize("interp", ["bicubic", "lanczos"])
@pytest.mark.parametrize("size,angle", [((128, 96), 30.0), ((97, 61), 90.0), ((256, 192), -17.5)])
def test_warp_affine_hq_matches_reference_kernel(kb, oracle, ref, dev, check, size, angle, interp):
    sw, sh = size
    src = cu(oracle.pattern_f32(sw * sh * 3).reshape(1, sh, sw, 3), dev)
    m = kb.imgproc.get_rotation_matrix2d((sw / 2.0, sh / 2.0), angle, 1.0)
    want = torch.full((1, sh, sw, 3), 3.0, dtype=torch.float32, device=dev)
    if ref is not None:
        ref.warp("affine", interp, src, want, oracle.invert_affine_transform(m))
    got = kb.Image.from_size_val(kb.ImageSize(sw, sh), 3.0, 3, torch.float32, dev)
    kb.imgproc.warp_affine(kb.Image(src[0]), got, m, kb.InterpolationMode.Bicubic if interp == "bicubic" else kb.InterpolationMode.Lanczos)
    check(got.data.reshape(want.shape), want if ref is not None else None, f"warp_affine {interp} {size} {angle}")


@pytest.mark.parametrize("mode,dw,dh", [("Letterbox", 64, 64), ("Stretch", 77, 41), ("Stretch", 300, 200)])
@pytest.mark.parametrize("fmt", ["Nv12", "Rgb8"])
def test_preprocess_lanczos_matches_reference_kernel(kb, oracle, ref, dev, check, mode, dw, dh, fmt):
    """sample_lanczos (preprocess.rs:565-590) uses the CUDA math library's sinf: the reference's kernel, run here, is the
    bit spec; the C++ oracle (host sinf) is checked within the 1e-4 tolerance in test_gpu_variants.py."""
    w, h, n = 192, 108, 2
    nbytes = w * h * 3 // 2 if fmt == "Nv12" else w * h * 3
    frames = [cu(raw_bytes(nbytes, k), dev) for k in range(n)]
    inv = [float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD]
    aff = oracle.preprocess_affine(oracle.LETTERBOX if mode == "Letterbox" else oracle.STRETCH, w, h, dw, dh)
    want = torch.zeros((n, 3, dh, dw), dtype=torch.float32, device=dev)
    if ref is not None:
        ref.preprocess(frames, w, h, want, aff, kb.IMAGENET_MEAN, inv, 114.0, fmt=3 if fmt == "Nv12" else 0, bpp=1 if fmt == "Nv12" else 3, sampler="lanczos")
    pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode[mode]).sampling(kb.InterpolationMode.Lanczos)
           .normalize(kb.Normalize.imagenet()).build_cuda())
    got = torch.zeros_like(want)
    pre.run_raw_batch(frames, w, h, got)
    check(got, want if ref is not None else None, f"preprocess lanczos {fmt} {mode} {dw}x{dh}")
