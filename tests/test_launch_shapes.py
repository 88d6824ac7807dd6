"""The launches that actually run, against the oracle: every row bench.py times, at its benchmarked batch and seeds; the
persistent kernels across their schedule knobs; and batches that cross the preprocess launch split.

The persistent kernels (fused_rows, resize_rows_f32, sep_filter_stream2, blur_u8_stream) size their schedule from
batch x SM count — rows per chunk, units per CTA, and the CTA stride's carry through tiles, chunks and images — so a
small-batch test does not run the schedule a large batch runs.  The host mirrors below restate the two tiled schedules
(`launch_fused_resize_rows`, `launch_resize_rows_f32`) so that each case asserts the regime it claims (mode, more units
than CTAs, an image carry in the stride, a ragged last chunk).  If a dispatcher change moves a case out of its regime,
the mirror assert fails and the case has to be re-chosen: a case must not pass vacuously.

Every frame of every batch is compared, never a sample.  The oracle runs one frame per worker in a thread pool (a ctypes
CDLL releases the GIL) and one device frame at a time is copied to the host, so host memory stays bounded.
"""
import contextlib
import math
import os
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import bench

from harness import POOL, _one_omp_thread, compare_frames, dev, free_device_memory, knobs
from restate import Schedule, _lround, _pick_npx, _walk, fused_schedule

pytestmark = pytest.mark.gpu

f32 = np.float32


@pytest.fixture(scope="module")
def sm_count(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def resize_rows_schedule(sw, sh, dw, dh, batch, sm, resident, npx_knob=0, stages_knob=0, ctas_knob=0):
    """launch_resize_rows_f32 (csrc/resize_rows.cu) on the host, half-pixel mapping.  `resident` is the occupancy
    calculator's answer, which the host cannot know; with rs.ctas = 1 it cannot matter (per_sm = min(1, resident))."""
    ax = f32(sw) / f32(dw)
    if sw % 4 or dw % 4 or sw < 8 or dw < 4 or not (0 <= ax <= 16):
        return Schedule("gather")
    npx = _pick_npx(dw, (2, 1, 3), 0.02)
    if 1 <= npx_knob <= 3:
        npx = npx_knob
    tw = 128 * npx
    slot = int(((tw - 1) * float(ax) + 4.0) * 3.0) + 8
    slot = min((slot + 31) & ~31, (sw * 3 + 31) & ~31)
    stage_bytes, out_bytes = slot * 8, tw * 3 * 4 * 2
    stages = stages_knob if 2 <= stages_knob <= 8 else 3
    while out_bytes + stage_bytes * stages > 200 * 1024 and stages > 2:
        stages -= 1
    if out_bytes + stage_bytes * stages > 200 * 1024:
        return Schedule("gather")
    per_sm = max(2, min(_lround(64 * 1024 / (stage_bytes * stages)), 8))
    if ctas_knob > 0:
        per_sm = ctas_knob
    per_sm = min(per_sm, resident)
    s = Schedule("rows", npx=npx, stages=stages, per_sm=per_sm, tiles_x=-(-dw // tw))
    return _walk(s, dh, batch, sm * per_sm, 8)


def first_bad_frame(bad):
    """bad: a device bool tensor [n, ...] -> (first frame with a difference, its count) or None."""
    per = bad.reshape(bad.shape[0], -1).sum(1)
    idx = torch.nonzero(per).flatten()
    if idx.numel() == 0:
        return None
    i = int(idx[0])
    return i, int(per[i])


def assert_same_bits_on_device(got, want, what, zero_ok=False):
    """got / want: device tensors of one dtype; bits equal everywhere (and with zero_ok, +0 == -0)."""
    it = {4: torch.int32, 2: torch.int16, 1: torch.uint8}[got.element_size()]
    bad = got.view(it) != want.view(it)
    if zero_ok:
        bad &= ~((got == 0) & (want == 0))
    r = first_bad_frame(bad)
    assert r is None, f"{what}: frame {r[0]} of {got.shape[0]}: {r[1]} of {got[0].numel()} elements differ"


# ── bench inputs, built as bench.py builds them ─────────────────────────────────────────────────────────────────
W4K, H4K = 3840, 2160
SEED_F32, SEED_U8 = 0x12345678, 0x0BADF00D     # bench.py: 4K f32 sources / u8 sources, + image index


def lcg_u8_batch(n, w, h, seed0, dev):
    src = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
    gen = bench.LcgPattern(w * h * 3, dev)
    for i in range(n):
        gen.frame(seed0 + i, src[i].view(-1))
    return src


def lcg_f32_batch(n, seed0, dev):
    """bench.py's src5: pattern_u8 / 255 as f32, on the device."""
    src = torch.empty((n, H4K, W4K, 3), dtype=torch.float32, device=dev)
    gen = bench.LcgPattern(W4K * H4K * 3, dev)
    tmp = torch.empty(W4K * H4K * 3, dtype=torch.uint8, device=dev)
    for i in range(n):
        gen.frame(seed0 + i, tmp)
        src[i] = (tmp.to(torch.float32) / 255.0).view(H4K, W4K, 3)
    return src


def host_u8(oracle, seed, w=W4K, h=H4K):
    return oracle.pattern_u8(w * h * 3, seed).reshape(h, w, 3)


def host_frame(t):
    """The oracle's input for a device-generated f32 source: the device's own bits (bench.py forms u8 / 255.0 with torch)."""
    return t.cpu().numpy()


def nv12_bench_frames(n, dev, w=1920, h=1080):
    """bench.py config 3: bytes ((i*7+13) % 251) + 31k."""
    frame = w * h * 3 // 2
    base = (torch.arange(frame, device=dev, dtype=torch.int64) * 7 + 13) % 251
    raw = torch.empty((n, frame), dtype=torch.uint8, device=dev)
    for k in range(n):
        raw[k] = ((base + 31 * k) & 0xFF).to(torch.uint8)
    return raw


def nv12_bench_host(k, w=1920, h=1080):
    i = np.arange(w * h * 3 // 2, dtype=np.int64)
    return ((((i * 7 + 13) % 251) + 31 * k) & 0xFF).astype(np.uint8)


def assert_regime(s, what, **want):
    got = s.regime()
    bad = {k: (got[k], v) for k, v in want.items() if got[k] != v}
    assert not bad, f"{what}: schedule {s} is not the regime the case claims: {bad}"


def imagenet(kb, oracle):
    p = kb.imgproc.NormalizeParams.from_mean_std(bench.IMAGENET_MEAN, bench.IMAGENET_STD)
    scale, bias = oracle.normalize_params_from_mean_std(bench.IMAGENET_MEAN, bench.IMAGENET_STD)
    assert p.scale == scale.tolist() and p.bias == bias.tolist()
    return p.scale, p.bias, scale, bias


# ═══ 1. bench shapes, whole batch ═══════════════════════════════════════════════════════════════════════════════
def test_bench_headline_config2_all_outputs(kb, oracle, dev, sm_count):
    """The headline: 64 x 4K u8 -> 1280x720 CHW, ImageNet normalisation, seeds 0x12345678 + i, f32 / f16 / bf16 outputs.
    Regime: FR_POINT, more than one unit per CTA, an image carry in the CTA stride (dimg >= 1), a ragged last chunk."""
    n, dw, dh = bench.BATCH, bench.DW, bench.DH
    s = fused_schedule(W4K, H4K, dw, dh, n, sm_count)
    print("headline schedule:", s)
    assert_regime(s, "headline", mode="POINT", multi=True, dimg=True, ragged=True)
    sc, bi, osc, obi = imagenet(kb, oracle)
    src = lcg_u8_batch(n, W4K, H4K, SEED_F32, dev)
    outs = {}
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        outs[dt] = kb.imgproc.resize_normalize_to_tensor_u8_bilinear(src, dw, dh, sc, bi, dt)
        assert kb._lib.last_kernel() == "fused_rows_kernel"
    del src

    def want(i):   # the f32 oracle, and its round-to-nearest-even f16 / bf16 values, compared as bits
        w = oracle.resize_normalize_u8_to_f32_chw(host_u8(oracle, SEED_F32 + i), dw, dh, osc, obi, oracle.LEAF_X86)
        return w.view(np.int32), w.astype(np.float16).view(np.int16), torch.from_numpy(w).to(torch.bfloat16).view(torch.int16).numpy()

    compare_frames(oracle, n, want, lambda i: tuple(outs[dt][i].view(torch.int32 if dt == torch.float32 else torch.int16).cpu().numpy()
                                                    for dt in (torch.float32, torch.float16, torch.bfloat16)),
                   "exact", "headline (f32, f16, bf16)")
    del outs
    free_device_memory()


@pytest.mark.parametrize("sw,dw,dh,kernel,mode", [
    (W4K, 1920, 1080, "fused_rows_kernel", "BOX"),
    (W4K, 1600, 900, "fused_rows_kernel", "GENERAL"),
    (3838, 1280, 720, "fused_resize_gather_kernel", "gather"),
])
def test_bench_fused_modes_x16(kb, oracle, dev, sm_count, sw, dw, dh, kernel, mode):
    """bench.py's other fused rows: 16 frames (seeds 0x0BADF00D + i; the 3838-wide source is the first 2160 x 3838 x 3
    bytes of each 4K frame), every frame bit for bit."""
    n = 16
    s = fused_schedule(sw, H4K, dw, dh, n, sm_count)
    print(f"{sw}x{H4K}->{dw}x{dh} x{n}:", s)
    assert s.mode == mode
    if s.staged:
        assert_regime(s, "fused x16", multi=True)
    sc, bi, osc, obi = imagenet(kb, oracle)
    full = lcg_u8_batch(n, W4K, H4K, SEED_U8, dev)
    src = full if sw == W4K else full.view(n, -1)[:, :H4K * sw * 3].contiguous().view(n, H4K, sw, 3)
    out = kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(src, dw, dh, sc, bi)
    assert kb._lib.last_kernel() == kernel
    del full, src
    compare_frames(oracle, n,
                   lambda i: oracle.resize_normalize_u8_to_f32_chw(
                       np.ascontiguousarray(host_u8(oracle, SEED_U8 + i).reshape(-1)[:H4K * sw * 3].reshape(H4K, sw, 3)), dw, dh, osc, obi).view(np.int32),
                   lambda i: out[i].view(torch.int32).cpu().numpy(), "exact", f"fused {sw}->{dw}x{dh}")
    del out
    free_device_memory()


def test_bench_config5_warp_perspective_x64(kb, oracle, dev):
    """Config 5: 64 x 4K f32 warp_perspective with H_CFG5 (the bench holds 2 x 6.4 GB on the device, so does this)."""
    n = 64
    src = lcg_f32_batch(n, SEED_F32, dev)
    dst = kb.Image.from_size_val(kb.ImageSize(W4K, H4K), 5.0, 3, torch.float32, dev, batch=n)
    kb.imgproc.warp_perspective(kb.Image(src), dst, bench.H_CFG5, kb.InterpolationMode.Bilinear)
    assert kb._lib.last_kernel() == "warp_bilinear_lean_kernel"
    compare_frames(oracle, n, lambda i: oracle.warp_perspective_f32(host_frame(src[i]), bench.H_CFG5, W4K, H4K, oracle.BILINEAR),
                   lambda i: dst.data[i].cpu().numpy(), "f32", "cfg5 warp_perspective")
    del src, dst
    free_device_memory()


@pytest.fixture(scope="module")
def f32_4k_x16(dev):
    """bench.py's S4: the first 16 of the config-5 sources."""
    src = lcg_f32_batch(16, SEED_F32, dev)
    yield src
    del src
    free_device_memory()


def rot30(kb):
    return kb.imgproc.get_rotation_matrix2d((W4K / 2, H4K / 2), 30.0, 1.0)


def test_bench_warp_affine_rot30_x16(kb, oracle, dev, f32_4k_x16):
    m = rot30(kb)
    dst = kb.Image.from_size_val(kb.ImageSize(W4K, H4K), 5.0, 3, torch.float32, dev, batch=16)
    kb.imgproc.warp_affine(kb.Image(f32_4k_x16), dst, m, kb.InterpolationMode.Bilinear)
    assert kb._lib.last_kernel() == "warp_tiled_kernel"
    compare_frames(oracle, 16, lambda i: oracle.warp_affine_f32(host_frame(f32_4k_x16[i]), m, W4K, H4K, oracle.BILINEAR),
                   lambda i: dst.data[i].cpu().numpy(), "f32", "warp_affine rot30")


def test_bench_config4_blur_then_sobel_x16(kb, oracle, dev, f32_4k_x16):
    """Config 4: gaussian 5x5 sigma 1.5, then sobel 3 on its output, 16 x 4K f32."""
    a = kb.Image.zeros_cuda(kb.ImageSize(W4K, H4K), 3, torch.float32, dev, batch=16)
    b = kb.Image.zeros_cuda(kb.ImageSize(W4K, H4K), 3, torch.float32, dev, batch=16)
    kb.imgproc.gaussian_blur(kb.Image(f32_4k_x16), a, (5, 5), (1.5, 1.5))
    assert kb._lib.last_kernel() == "sep_filter_stream2_kernel"
    kb.imgproc.sobel(a, b, 3)
    assert kb._lib.last_kernel() == "sep_filter_stream2_kernel"

    def want(i):
        blur = oracle.gaussian_blur(host_frame(f32_4k_x16[i]), (5, 5), (1.5, 1.5))
        return blur, oracle.sobel(blur, 3)

    compare_frames(oracle, 16, want, lambda i: (a.data[i].cpu().numpy(), b.data[i].cpu().numpy()), "f32", "cfg4 (blur, sobel)")


@pytest.mark.parametrize("dw,dh", [(1280, 720), (1920, 1080), (1600, 900)])
def test_bench_resize_f32_x16(kb, oracle, dev, sm_count, f32_4k_x16, dw, dh):
    s = resize_rows_schedule(W4K, H4K, dw, dh, 16, sm_count, resident=8)
    print(f"resize 4K->{dw}x{dh} x16 (if 8 CTAs fit per SM):", s)
    assert s.staged
    dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), -1.0, 3, torch.float32, dev, batch=16)
    kb.imgproc.resize(kb.Image(f32_4k_x16), dst, kb.InterpolationMode.Bilinear)
    assert kb._lib.last_kernel() == "resize_rows_f32_kernel"
    compare_frames(oracle, 16, lambda i: oracle.resize_f32(host_frame(f32_4k_x16[i]), dw, dh),
                   lambda i: dst.data[i].cpu().numpy(), "f32", f"resize 4K->{dw}x{dh}")


def test_bench_colour_and_normalize_x16(kb, oracle, dev, f32_4k_x16):
    gray = kb.Image.zeros_cuda(kb.ImageSize(W4K, H4K), 1, torch.float32, dev, batch=16)
    kb.imgproc.gray_from_rgb(kb.Image(f32_4k_x16), gray)
    assert kb._lib.last_kernel() == "gray_from_rgb_f32_vec4"
    norm = kb.Image.zeros_cuda(kb.ImageSize(W4K, H4K), 3, torch.float32, dev, batch=16)
    kb.imgproc.normalize_mean_std(kb.Image(f32_4k_x16), norm, bench.IMAGENET_MEAN, bench.IMAGENET_STD)
    assert kb._lib.last_kernel() == "normalize_mean_std_c3_vec"

    def want(i):
        src = host_frame(f32_4k_x16[i])
        return oracle.gray_from_rgb_f32(src), oracle.normalize_mean_std(src, bench.IMAGENET_MEAN, bench.IMAGENET_STD)

    compare_frames(oracle, 16, want, lambda i: (gray.data[i].cpu().numpy(), norm.data[i].cpu().numpy()), "f32", "gray / normalize")


# ── u8 rows (16 x 4K, seeds 0x0BADF00D + i) ──
@pytest.fixture(scope="module")
def u8_4k_x16(dev):
    src = lcg_u8_batch(16, W4K, H4K, SEED_U8, dev)
    yield src
    del src
    free_device_memory()


def test_bench_std_mean_u8_x16(kb, oracle, dev, u8_4k_x16):
    """Integer sums: exact, for the batch (the bench row) and for every frame on its own."""
    total = kb.imgproc.std_mean_sums(kb.Image(u8_4k_x16)).tolist()
    assert kb._lib.last_kernel() == "std_mean_kernel"
    per = [kb.imgproc.std_mean_sums(kb.Image(u8_4k_x16[i])).tolist() for i in range(16)]
    with ThreadPoolExecutor(POOL, initializer=_one_omp_thread, initargs=(oracle,)) as ex:
        want = list(ex.map(lambda i: [int(v) for v in oracle.std_mean(host_u8(oracle, SEED_U8 + i))[2]], range(16)))
    for i in range(16):
        assert per[i] == want[i], f"frame {i}: {per[i]} != {want[i]}"
    assert total == [sum(w[k] for w in want) for k in range(6)]


@pytest.mark.parametrize("dw,dh,kernel", [(1920, 1080, "pyrdown_2x_rgb_u8_w4_kernel"), (1280, 720, "resize_bilinear_u8_c3_3to1_kernel")])
def test_bench_resize_fast_u8_x16(kb, oracle, dev, u8_4k_x16, dw, dh, kernel):
    d = kb.Image(torch.full((16, dh, dw, 3), 0xCD, dtype=torch.uint8, device=dev))
    kb.imgproc.resize_fast_u8(kb.Image(u8_4k_x16), d, kb.InterpolationMode.Bilinear)
    assert kb._lib.last_kernel() == kernel
    compare_frames(oracle, 16, lambda i: oracle.resize_fast_u8(host_u8(oracle, SEED_U8 + i), dw, dh, 1),
                   lambda i: d.data[i].cpu().numpy(), "exact", f"resize_fast_u8 -> {dw}x{dh}")


def radial_maps(kb, dev):
    """bench.py's radial-distortion map, built the same way on the device."""
    w, h = W4K, H4K
    yy, xx = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32), torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
    r2 = ((xx - w / 2) ** 2 + (yy - h / 2) ** 2) / float(w * w)
    mx = (w / 2 + (xx - w / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous()
    my = (h / 2 + (yy - h / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous()
    return mx, my


@pytest.mark.parametrize("op", ["warp_perspective_u8", "warp_affine_u8", "gaussian_blur_u8", "remap_u8"])
def test_bench_u8_ops_x16(kb, oracle, dev, u8_4k_x16, op):
    d = kb.Image(torch.full((16, H4K, W4K, 3), 0xCD, dtype=torch.uint8, device=dev))
    s = kb.Image(u8_4k_x16)
    if op == "warp_perspective_u8":
        kb.imgproc.warp_perspective_u8(s, d, bench.H_CFG5)
        fn = lambda src: oracle.warp_perspective_u8(src, W4K, H4K, bench.H_CFG5)
    elif op == "warp_affine_u8":
        m = rot30(kb)
        kb.imgproc.warp_affine_u8(s, d, m)
        fn = lambda src: oracle.warp_affine_u8(src, W4K, H4K, m)
    elif op == "gaussian_blur_u8":
        kb.imgproc.gaussian_blur_u8(s, d, (5, 5), (1.5, 1.5))
        fn = lambda src: oracle.gaussian_blur_u8(src, (5, 5), (1.5, 1.5))
    else:
        mx, my = radial_maps(kb, dev)
        kb.imgproc.remap_u8(s, d, kb.Image(mx), kb.Image(my), kb.InterpolationMode.Bilinear)
        hx, hy = mx[..., 0].cpu().numpy(), my[..., 0].cpu().numpy()
        fn = lambda src: oracle.remap(src, hx, hy, oracle.BILINEAR)
    assert kb._lib.last_kernel() == {"warp_perspective_u8": "warp_perspective_u8_kernel", "warp_affine_u8": "warp_affine_u8_kernel",
                                     "gaussian_blur_u8": "blur_u8_stream_kernel", "remap_u8": "remap_u8_kernel"}[op]
    compare_frames(oracle, 16, lambda i: fn(host_u8(oracle, SEED_U8 + i)), lambda i: d.data[i].cpu().numpy(), "exact", op)


def test_bench_remap_f32_x16(kb, oracle, dev, f32_4k_x16):
    mx, my = radial_maps(kb, dev)
    d = kb.Image.from_size_val(kb.ImageSize(W4K, H4K), 5.0, 3, torch.float32, dev, batch=16)
    kb.imgproc.remap(kb.Image(f32_4k_x16), d, kb.Image(mx), kb.Image(my), kb.InterpolationMode.Bilinear)
    assert kb._lib.last_kernel() == "remap_lean_kernel"
    hx, hy = mx[..., 0].cpu().numpy(), my[..., 0].cpu().numpy()
    compare_frames(oracle, 16, lambda i: oracle.remap(host_frame(f32_4k_x16[i]), hx, hy, oracle.BILINEAR),
                   lambda i: d.data[i].cpu().numpy(), "f32", "remap f32")


# ── preprocess rows (256 x NV12 1080p) ──
@pytest.mark.parametrize("mode,dw,dh,kernel", [("Stretch", 1920, 1080, "preprocess_nv12_identity_kernel"),
                                               ("Letterbox", 640, 640, "preprocess_nv12_kernel")])
def test_bench_config3_preprocess_x256(kb, oracle, dev, mode, dw, dh, kernel):
    """Config 3a / 3b: 256 NV12 1080p frames, one launch, every frame against the oracle."""
    n, w, h = 256, 1920, 1080
    raw = nv12_bench_frames(n, dev)
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda()
    dst = torch.full((n, 3, dh, dw), float("nan"), dtype=torch.float32, device=dev)
    pre.run_raw_batch([raw[i] for i in range(n)], w, h, dst)
    assert kb._lib.last_kernel() == kernel
    del raw
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    cfg = oracle.PreprocessCfg(mode=oracle.LETTERBOX if mode == "Letterbox" else oracle.STRETCH, fmt=oracle.FMT_NV12,
                               mean=kb.IMAGENET_MEAN, inv_std=inv)
    compare_frames(oracle, n, lambda k: oracle.preprocess_frame(nv12_bench_host(k), cfg, w, h, dw, dh),
                   lambda k: dst[k].cpu().numpy(), "f32", f"config 3 {mode}")
    del dst
    free_device_memory()


def test_bench_rgb_from_nv12_x256(kb, oracle, dev):
    n, w, h = 256, 1920, 1080
    raw = nv12_bench_frames(n, dev)
    rgb = kb.Image(torch.full((n, h, w, 3), 0xCD, dtype=torch.uint8, device=dev))
    kb.imgproc.rgb_from_nv12(raw, rgb)
    assert kb._lib.last_kernel() == "rgb_from_nv12_vec16"
    del raw
    compare_frames(oracle, n, lambda k: oracle.rgb_from_nv12(nv12_bench_host(k), w, h), lambda k: rgb.data[k].cpu().numpy(), "exact", "rgb_from_nv12")
    del rgb
    free_device_memory()


# ═══ 2. schedule sweeps ═════════════════════════════════════════════════════════════════════════════════════════
@pytest.fixture(scope="module")
def oracle_cache():
    """One oracle result per geometry (on the device), shared by every knob setting; released with the module."""
    cache = {}
    yield cache
    cache.clear()
    free_device_memory()


def cached(cache, key, make):
    if key not in cache:
        cache[key] = make()
    return cache[key]


def oracle_batch(oracle, n, fn):
    with ThreadPoolExecutor(POOL, initializer=_one_omp_thread, initargs=(oracle,)) as ex:
        return np.stack(list(ex.map(fn, range(n))))


FR_BATCH = 64
FR_KNOBS = [(npx, st, ct) for npx in (1, 2, 3, 4, 5) for st in (3, 4, 16) for ct in (2, 8)]


# (mode, sw, sh, dw, dh, leaf, dtype, ragged at fr.ctas = 2): camera-sized frames, 64 per batch, so the persistent walk
# is long — more units than CTAs and an image carry in the CTA stride for every case.  dw % 8 == 0 with the x86 leaf runs
# the ALLFMA instantiation; the scalar leaf and dw % 8 != 0 (BOX: dw % 16 != 0) run the per-column bulk / tail split.
FR_SWEEP = [
    ("POINT", 640, 480, 640, 160, 0, torch.float32, True),
    ("POINT", 640, 480, 640, 160, 1, torch.float32, True),
    ("POINT", 640, 480, 640, 160, 1, torch.float16, True),
    ("GENERAL", 640, 480, 224, 224, 0, torch.float32, False),
    ("GENERAL", 640, 480, 224, 224, 1, torch.float32, False),
    ("GENERAL", 640, 480, 224, 224, 1, torch.float16, False),
    ("GENERAL", 640, 480, 230, 230, 1, torch.float32, True),
    ("BOX", 640, 482, 320, 241, 0, torch.float32, True),
    ("BOX", 640, 482, 320, 241, 1, torch.float32, True),
    ("BOX", 656, 482, 328, 241, 1, torch.float32, True),
    ("YZERO", 640, 483, 224, 161, 0, torch.float32, True),
    ("YZERO", 640, 483, 224, 161, 1, torch.float32, True),
    ("YZERO", 640, 483, 230, 161, 1, torch.float32, True),
]


@pytest.mark.parametrize("mode,sw,sh,dw,dh,leaf,dtype,ragged", FR_SWEEP)
def test_fused_rows_schedule_sweep(kb, oracle, dev, sm_count, oracle_cache, mode, sw, sh, dw, dh, leaf, dtype, ragged):
    """fused_rows_kernel at fr.npx 1-5 x fr.stages {3, 4, 16} x fr.ctas {2, 8}: every setting reproduces the oracle's bits."""
    n = FR_BATCH
    assert_regime(fused_schedule(sw, sh, dw, dh, n, sm_count, stages_knob=3, ctas_knob=2), f"{sw}x{sh}->{dw}x{dh}",
                  mode=mode, multi=True, dimg=True, ragged=ragged)
    sc, bi, osc, obi = imagenet(kb, oracle)
    src_h = cached(oracle_cache, ("fr-src", sw, sh), lambda: oracle_batch(oracle, n, lambda i: oracle.pattern_u8(sw * sh * 3, 0x5EED + i).reshape(sh, sw, 3)))
    src = cached(oracle_cache, ("fr-src-dev", sw, sh), lambda: torch.from_numpy(src_h).to(dev))
    want32 = cached(oracle_cache, ("fr", sw, sh, dw, dh, leaf), lambda: oracle_batch(
        oracle, n, lambda i: oracle.resize_normalize_u8_to_f32_chw(src_h[i], dw, dh, osc, obi, leaf)))
    want = cached(oracle_cache, ("fr-dev", sw, sh, dw, dh, leaf, dtype),
                  lambda: torch.from_numpy(want32 if dtype == torch.float32 else want32.astype(np.float16)).to(dev))
    for npx, st, ct in FR_KNOBS:
        s = fused_schedule(sw, sh, dw, dh, n, sm_count, npx, st, ct)
        what = f"fused {sw}x{sh}->{dw}x{dh} x{n} leaf {leaf} {dtype} fr.npx={npx} fr.stages={st} fr.ctas={ct}: {s}"
        print(what, flush=True)
        assert s.mode == mode and s.npx == npx and s.stages == st, what
        with knobs(kb, {"fr.npx": npx, "fr.stages": st, "fr.ctas": ct}):
            out = kb.imgproc.resize_normalize_to_tensor_u8_bilinear(src, dw, dh, sc, bi, dtype, leaf=leaf)
            assert kb._lib.last_kernel() == "fused_rows_kernel", what
        assert_same_bits_on_device(out, want, what)


@pytest.mark.parametrize("op", ["resize", "resize_bilinear_normalize"])
def test_resize_rows_schedule_sweep(kb, oracle, dev, sm_count, op):
    """resize_rows_f32_kernel at rs.npx 1-3 x rs.stages {2, 3, 8} x rs.ctas {1, 2, 8}, 8 frames 640x360 -> 428x244.
    With rs.ctas = 1 (exact whatever the occupancy): more units than CTAs, an image carry, a ragged last chunk."""
    n, sw, sh, dw, dh = 8, 640, 360, 428, 244
    assert_regime(resize_rows_schedule(sw, sh, dw, dh, n, sm_count, resident=1, ctas_knob=1), "resize rows", multi=True, dimg=True, ragged=True)
    src_h = oracle_batch(oracle, n, lambda i: oracle.pattern_f32(sw * sh * 3, 0xF00 + i).reshape(sh, sw, 3))
    want = oracle_batch(oracle, n, lambda i: oracle.resize_f32(src_h[i], dw, dh))
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    if op == "resize_bilinear_normalize":   # (v - mean) * (1 / std) on the bilinear sample, as test_resize_bilinear_normalize_rows
        want = ((want - np.array(mean, np.float32)) * (np.float32(1.0) / np.array(std, np.float32))).astype(np.float32)
    src, want = kb.Image(torch.from_numpy(src_h).to(dev)), torch.from_numpy(want).to(dev)
    for npx in (1, 2, 3):
        for st in (2, 3, 8):
            for ct in (1, 2, 8):
                s = resize_rows_schedule(sw, sh, dw, dh, n, sm_count, resident=ct, npx_knob=npx, stages_knob=st, ctas_knob=ct)
                what = f"{op} {sw}x{sh}->{dw}x{dh} x{n} rs.npx={npx} rs.stages={st} rs.ctas={ct}: {s} (if {ct} CTAs fit per SM)"
                print(what, flush=True)
                assert s.staged and s.npx == npx and s.stages == st, what
                dst = kb.Image.from_size_val(kb.ImageSize(dw, dh), -1.0, 3, torch.float32, dev, batch=n)
                with knobs(kb, {"rs.npx": npx, "rs.stages": st, "rs.ctas": ct}):
                    if op == "resize":
                        kb.imgproc.resize(src, dst, kb.InterpolationMode.Bilinear)
                    else:
                        kb.imgproc.resize_bilinear_normalize(src, dst, mean, std)
                    assert kb._lib.last_kernel() == "resize_rows_f32_kernel", what
                assert_same_bits_on_device(dst.data, want, what, zero_ok=True)


# try_sep_stream (csrc/filter.cu): every streaming instance (C, K, sobel); rows = 61, which no tested chunk height but 1 and
# 61 divides; rows of >= 1032 floats so that interior strips run too
SEP_STREAM = [(3, 5, False), (3, 3, False), (3, 7, False), (1, 5, False), (1, 3, False), (1, 7, False), (4, 5, False), (4, 3, False),
              (3, 3, True), (3, 5, True), (1, 3, True), (1, 5, True)]
SEP_COLS = {1: 1100, 3: 700, 4: 520}
SIGMA = {3: 0.8, 5: 1.5, 7: 2.0}


@pytest.mark.parametrize("c,k,sobel", SEP_STREAM)
def test_sep_filter_stream2_schedule_sweep(kb, oracle, dev, c, k, sobel):
    """ss.rc {1, 2, KY-1, 7, rows} x ss.stages {2, 4, 12 (the maximum)} x ss.ctas {1, 6}.  ss.rc = 1 makes every output
    row its own chunk: the KY-1 halo rows are re-staged for every row and the ring wraps mid-window."""
    n, w, h = 2, SEP_COLS[c], 61
    src_h = oracle.pattern_f32(n * w * h * c, 0x5E9 + 16 * c + k).reshape(n, h, w, c)
    if sobel:
        want = np.stack([oracle.sobel(src_h[i], k) for i in range(n)])
    else:
        want = np.stack([oracle.gaussian_blur(src_h[i], (k, k), (SIGMA[k], SIGMA[k])) for i in range(n)])
    src, want = kb.Image(torch.from_numpy(src_h).to(dev)), torch.from_numpy(want).to(dev)
    for rc in sorted({1, 2, k - 1, 7, h}):
        for st in (2, 4, 12):
            for ct in (1, 6):
                what = f"{'sobel' if sobel else 'gaussian'} C={c} K={k} {w}x{h} x{n} ss.rc={rc} ss.stages={st} ss.ctas={ct}"
                print(what, flush=True)
                dst = kb.Image.from_size_val(kb.ImageSize(w, h), 9.0, c, torch.float32, dev, batch=n)
                with knobs(kb, {"ss.rc": rc, "ss.stages": st, "ss.ctas": ct}):
                    if sobel:
                        kb.imgproc.sobel(src, dst, k)
                    else:
                        kb.imgproc.gaussian_blur(src, dst, (k, k), (SIGMA[k], SIGMA[k]))
                    assert kb._lib.last_kernel() == "sep_filter_stream2_kernel", what
                assert_same_bits_on_device(dst.data, want, what, zero_ok=True)


@pytest.mark.parametrize("c,kind,k", [(3, "gaussian", 3), (3, "gaussian", 5), (3, "gaussian", 7), (3, "box", 5), (1, "gaussian", 5), (4, "gaussian", 7)])
def test_blur_u8_stream_schedule_sweep(kb, oracle, dev, c, kind, k):
    """blur_u8_stream_kernel at knob c (CTAs per SM) {1, 8} x knob d (rows per chunk) {1, 2, 5, rows}; 800-pixel rows
    make several strips with a ragged last one."""
    n, w, h = 2, 800, 37
    src_h = oracle.pattern_u8(n * w * h * c, 0xB1 + 16 * c + k).reshape(n, h, w, c)
    sig = (SIGMA[k], SIGMA[k])
    want = np.stack([oracle.gaussian_blur_u8(src_h[i], (k, k), sig) if kind == "gaussian" else oracle.box_blur_u8(src_h[i], (k, k))
                     for i in range(n)])
    src, want = kb.Image(torch.from_numpy(src_h).to(dev)), torch.from_numpy(want).to(dev)
    for ctas in (1, 8):
        for rc in (1, 2, 5, h):
            what = f"{kind} u8 C={c} K={k} {w}x{h} x{n} c={ctas} d={rc}"
            print(what, flush=True)
            dst = kb.Image(torch.full((n, h, w, c), 0xCD, dtype=torch.uint8, device=dev))
            with knobs(kb, {"c": ctas, "d": rc}):
                if kind == "gaussian":
                    kb.imgproc.gaussian_blur_u8(src, dst, (k, k), sig)
                else:
                    kb.imgproc.box_blur_u8(src, dst, (k, k))
                assert kb._lib.last_kernel() == "blur_u8_stream_kernel", what
            assert_same_bits_on_device(dst.data, want, what)


# ═══ 3. batch chunk boundaries ══════════════════════════════════════════════════════════════════════════════════
# launch_preprocess splits a batch into launches of <= 256 frames (frame0 = 0, 256, 512, ...): 300 and 513 frames run a
# second and a third launch on each of the three kernels.
PRE_CASES = {   # fmt, mode, sampling, dst size, kernel
    "nv12-identity": ("Nv12", "Stretch", "Bilinear", (64, 48), "preprocess_nv12_identity_kernel"),
    "nv12-letterbox": ("Nv12", "Letterbox", "Bilinear", (40, 40), "preprocess_nv12_kernel"),
    "rgb8-generic": ("Rgb8", "Letterbox", "Bilinear", (40, 40), "preprocess_generic_kernel"),
    "lanczos-generic": ("Nv12", "Letterbox", "Lanczos", (40, 40), "preprocess_generic_kernel"),
}
PRE_W, PRE_H = 64, 48


def preprocess_setup(kb, oracle, case, n):
    fmt, mode, sampling, (dw, dh), kernel = PRE_CASES[case]
    nbytes = PRE_W * PRE_H * 3 if fmt == "Rgb8" else PRE_W * PRE_H * 3 // 2
    norm = kb.Normalize.UnitScale() if sampling == "Lanczos" else kb.Normalize.imagenet()
    pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode[mode]).sampling(kb.InterpolationMode[sampling])
           .normalize(norm).build_cuda())
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    cfg = oracle.PreprocessCfg(mode=oracle.LETTERBOX if mode == "Letterbox" else oracle.STRETCH,
                               fmt=oracle.FMT_RGB if fmt == "Rgb8" else oracle.FMT_NV12,
                               sampling={"Bilinear": oracle.BILINEAR, "Lanczos": oracle.LANCZOS}[sampling],
                               **({} if sampling == "Lanczos" else {"mean": kb.IMAGENET_MEAN, "inv_std": inv}))
    frames = np.stack([oracle.pattern_u8(nbytes, 0x7000 + k) for k in range(n)])
    return pre, cfg, frames, nbytes, (dw, dh), kernel


@pytest.mark.parametrize("case", list(PRE_CASES))
@pytest.mark.parametrize("n", [300, 513])
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_beyond_256_frames(kb, oracle, dev, case, n, f16):
    """Pointer-array (run_raw_batch) and strided (run_raw_strided) addressing, every frame against the oracle."""
    pre, cfg, frames, nbytes, (dw, dh), kernel = preprocess_setup(kb, oracle, case, n)
    stride = (nbytes + 15) // 16 * 16 + 16      # padded ring slots
    ring = torch.zeros((n, stride), dtype=torch.uint8, device=dev)
    ring[:, :nbytes] = torch.from_numpy(frames).to(dev)
    dt = torch.float16 if f16 else torch.float32
    by_ptr = torch.full((n, 3, dh, dw), float("nan"), dtype=dt, device=dev)
    (pre.run_raw_batch_f16 if f16 else pre.run_raw_batch)([ring[k, :nbytes] for k in range(n)], PRE_W, PRE_H, by_ptr)
    assert kb._lib.last_kernel() == kernel
    strided = torch.full((n, 3, dh, dw), float("nan"), dtype=dt, device=dev)
    pre.run_raw_strided(ring.view(-1), stride, n, PRE_W, PRE_H, strided, f16=f16)
    assert kb._lib.last_kernel() == kernel
    lanczos = cfg.sampling == oracle.LANCZOS
    if lanczos:   # the f32 oracle within the tolerance of test_preprocess_lanczos_vs_oracle
        rule = 2e-3 if f16 else 1e-4
        want_fn = lambda k: (oracle.preprocess_frame(frames[k], cfg, PRE_W, PRE_H, dw, dh),) * 2
        got_fn = lambda k: (by_ptr[k].float().cpu().numpy(), strided[k].float().cpu().numpy())
    elif f16:
        rule = "exact"
        want_fn = lambda k: (oracle.preprocess_frame(frames[k], cfg, PRE_W, PRE_H, dw, dh, f16=True).view(np.uint16),) * 2
        got_fn = lambda k: (by_ptr[k].cpu().numpy().view(np.uint16), strided[k].cpu().numpy().view(np.uint16))
    else:
        rule = "f32"
        want_fn = lambda k: (oracle.preprocess_frame(frames[k], cfg, PRE_W, PRE_H, dw, dh),) * 2
        got_fn = lambda k: (by_ptr[k].cpu().numpy(), strided[k].cpu().numpy())
    compare_frames(oracle, n, want_fn, got_fn, rule, f"preprocess {case} x{n} {'f16' if f16 else 'f32'} (pointer array, strided)")


def test_preprocess_host_beyond_256_frames(kb, oracle, dev):
    """run_raw_host with 300 frames and staging for all of them: the host pipeline splits its launches at 256 frames
    (host_pipeline.cu) and must give the device path's bits."""
    n = 300
    pre, cfg, frames, nbytes, (dw, dh), kernel = preprocess_setup(kb, oracle, "nv12-letterbox", n)
    want = torch.full((n, 3, dh, dw), float("nan"), dtype=torch.float32, device=dev)
    pre.run_raw_batch([torch.from_numpy(frames[k]).to(dev) for k in range(n)], PRE_W, PRE_H, want)
    host = torch.from_numpy(frames).pin_memory()
    dev_stride = (nbytes + 15) // 16 * 16
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=n * dev_stride, dst_chunk_bytes=n * 3 * dw * dh * 4, depth=2)
    got = pre.run_raw_host(host, PRE_W, PRE_H, (dw, dh), pipeline=pipe)
    torch.cuda.synchronize()
    h2d, d2h = pipe.last_transfer()
    pipe.close()
    assert h2d == n * nbytes and d2h == n * 3 * dw * dh * 4
    r = first_bad_frame(got.view(torch.int32) != want.cpu().view(torch.int32))
    assert r is None, f"host pipeline: frame {r[0]} of {n}: {r[1]} elements differ from the device path"
    compare_frames(oracle, n, lambda k: oracle.preprocess_frame(frames[k], cfg, PRE_W, PRE_H, dw, dh), lambda k: want[k].cpu().numpy(),
                   "f32", "preprocess nv12-letterbox x300 (device path)")
