"""Camera preprocess with bfloat16 output: kb200_preprocess_bf16, kb200_preprocess_strided_bf16 and
kb200_preprocess_host_format(..., KB200_OUT_BF16), and the Preprocessor methods over them.

The rule under test: a bf16 value is __float2bfloat16_rn(the f32 value the f32 entry writes for the same arguments), so
the bf16 output must equal the f32 output converted with torch's .to(torch.bfloat16), bit for bit (a NaN by NaN-ness
only), and come from the kernel the f32 and f16 calls run.  The f32 output is pinned to the oracle by the other
preprocess tests, so this anchors bf16 everywhere, Lanczos included.

  * parity: every case of test_preprocess_sweep's seeded sweep and its hand-picked edges, run in f32, f16 and bf16
    through the case's entry, and in bf16 once more into a destination 2 bytes past a 16-byte boundary (the generic
    kernel);
  * rounding edges on white frames (every tap exactly 1.0), where mean and inv_std set each output exactly: ties, overflow
    to +-inf, subnormals, +-0, NaN from 0 * inf and from a NaN pad value;
  * 1080p batches of 256 and 300 frames (the second launch starts at frame 256);
  * the host pipeline, and the memory footprint of every new entry on one kernel of each family.
The CPU tests check the header, the binding, argument validation and the Python dtype rules.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from harness import Guarded, dev, lib, poison
from restate import BILINEAR, EDGES, FORMATS, GENERIC, LANCZOS, N_SWEEP, case, edge, expected_kernel, frame_bytes, host_chunk, row_bytes


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_F32, OUT_F16, OUT_BF16 = 0, 1, 2
ESZ = {OUT_F32: 4, OUT_F16: 2, OUT_BF16: 2}
gpu = pytest.mark.gpu


# ── helpers ──────────────────────────────────────────────────────────────────────────────────────────────────────
def bf16_of_f32(raw):
    """Raw f32 output bytes -> the int16 bits of torch's .to(torch.bfloat16)."""
    f = torch.from_numpy(np.ascontiguousarray(raw).view(np.float32).copy())
    return f.to(torch.bfloat16).view(torch.int16).numpy()


def assert_bf16_matches(got_raw, f32_raw, what):
    """bf16 output bytes against the f32 output bytes of the same call rounded by torch; NaNs by NaN-ness."""
    g = np.ascontiguousarray(got_raw).view(np.int16)
    w = bf16_of_f32(f32_raw)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    gn = (g & 0x7FFF) > 0x7F80
    wn = (w & 0x7FFF) > 0x7F80
    assert np.array_equal(gn, wn), f"{what}: NaN-ness differs at {int((gn != wn).sum())} values"
    bad = np.flatnonzero((g != w) & ~wn)
    assert bad.size == 0, f"{what}: {bad.size} of {g.size} values differ, first at element {bad[0]}: {int(g[bad[0]]) & 0xFFFF:#06x} vs {int(w[bad[0]]) & 0xFFFF:#06x}"


def desc_of(c):
    from kornia_rs_b200._lib import PreprocessDesc
    return c.desc(PreprocessDesc)


DEVICE_FN = {("table", OUT_F32): "kb200_preprocess_f32", ("table", OUT_F16): "kb200_preprocess_f16", ("table", OUT_BF16): "kb200_preprocess_bf16",
             ("strided", OUT_F32): "kb200_preprocess_strided_f32", ("strided", OUT_F16): "kb200_preprocess_strided_f16",
             ("strided", OUT_BF16): "kb200_preprocess_strided_bf16"}


# ── (1) parity with the f32 entry over the seeded sweep and its edges ───────────────────────────────────────────────
def run_parity(kb, lib, dev, c):
    d = desc_of(c)
    need = c.need
    frames = [frame_bytes(c, k) for k in range(c.batch)]
    out_elems = 3 * c.dw * c.dh
    starts = list(c.frames) if c.entry == "table" else [c.frames[0] + k * c.stride for k in range(c.batch)]
    span = starts[-1] + need
    image = np.zeros(span, np.uint8)
    for s, fr in zip(starts, frames):
        image[s:s + need] = fr
    dev_src = Guarded(dev, span).load("u8", image)
    host_src = Guarded(dev, span, host=True).load("u8", image) if c.entry == "host" else None

    def call(out, dst, entry):
        n = out_elems * c.batch
        if entry == "host":
            _, src_chunk, dst_chunk = host_chunk(need, out_elems * ESZ[out], c.batch)
            pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=src_chunk, dst_chunk_bytes=dst_chunk, depth=2)
            try:
                st = lib.kb200_preprocess_host_format(pipe._h, None, C.byref(d), host_src.ptr + c.frames[0], host_src.n - c.frames[0], c.stride,
                                                      c.batch, dst.ptr, n, out)
                ran = kb._lib.last_kernel()
                torch.cuda.synchronize()
            finally:
                pipe.close()
            return st, ran, c.planned()
        fn = getattr(lib, DEVICE_FN[entry, out])
        if entry == "table":
            ptrs = (C.c_void_p * c.batch)(*[dev_src.ptr + s for s in starts])
            lens = (C.c_size_t * c.batch)(*[need] * c.batch)
            st = fn(None, C.byref(d), ptrs, lens, c.batch, dst.ptr, n)
            mirror = expected_kernel(d, [dev_src.ptr + s for s in starts], None, dst.ptr, c.sampling)
        else:
            st = fn(None, C.byref(d), dev_src.ptr + c.frames[0], dev_src.n - c.frames[0], c.stride, c.batch, dst.ptr, n)
            mirror = expected_kernel(d, [dev_src.ptr + c.frames[0]], c.stride, dst.ptr, c.sampling)
        ran = kb._lib.last_kernel()
        torch.cuda.synchronize()
        return st, ran, mirror

    outs, kernels = {}, {}
    for out in (OUT_F32, OUT_F16, OUT_BF16):
        nbytes = out_elems * ESZ[out] * c.batch
        dst = Guarded(dev, nbytes, min(nbytes, 1 << 16), host=c.entry == "host").fill(0xFF)
        st, ran, mirror = call(out, dst, c.entry)
        assert st == 0, f"{c}: out {out}: status {st}: {kb._lib.last_error()}"
        assert ran == mirror, f"{c}: out {out} ran {ran}, the dispatch mirror says {mirror}"
        lead, tail = dst.guards()
        assert np.all(lead == 0xFF) and np.all(tail == 0xFF), f"{c}: out {out} wrote outside dst"
        outs[out], kernels[out] = dst.out(), ran
    assert kernels[OUT_BF16] == kernels[OUT_F32] == kernels[OUT_F16], f"{c}: kernels {kernels}"
    assert not (outs[OUT_BF16].view(np.uint16) == 0xFFFF).any(), f"{c}: bf16 output elements left unwritten"
    assert not (outs[OUT_F32].view(np.uint32) == 0xFFFFFFFF).any(), f"{c}: f32 output elements left unwritten"
    assert_bf16_matches(outs[OUT_BF16], outs[OUT_F32], str(c))
    if c.sampling != LANCZOS:   # 2 bytes past a 16-byte boundary: the identity and fast kernels refuse it, the generic kernel runs
        nbytes = out_elems * 2 * c.batch
        dst = Guarded(dev, nbytes, min(nbytes, 1 << 16), 2).fill(0xFF)
        st, ran, mirror = call(OUT_BF16, dst, "table" if c.entry == "table" else "strided")
        assert st == 0 and ran == mirror == GENERIC, f"{c}: dst +2 B: status {st}, ran {ran}, mirror {mirror}"
        lead, tail = dst.guards()
        assert np.all(lead == 0xFF) and np.all(tail == 0xFF), f"{c}: dst +2 B: write outside dst"
        assert np.array_equal(dst.out(), outs[OUT_BF16]), f"{c}: {kernels[OUT_BF16]} and {GENERIC} differ in bf16"


@gpu
@pytest.mark.parametrize("i", range(N_SWEEP))
def test_bf16_sweep(kb, lib, dev, i):
    run_parity(kb, lib, dev, case(i))


@gpu
@pytest.mark.parametrize("name", list(EDGES))
def test_bf16_edge(kb, lib, dev, name):
    run_parity(kb, lib, dev, EDGES[name])


def test_bf16_sweep_covers_every_kernel():
    """The parity cases reach every format, kernel, YUV matrix, sampler and entry the f32 sweep does (test_sweep_coverage
    checks that set), plus the odd-address NV12 / NV21 frames and odd destination widths that fall back to the generic
    kernel."""
    cases = [case(i) for i in range(N_SWEEP)] + list(EDGES.values())
    ran = {(c.code, c.planned()) for c in cases}
    for code, f in FORMATS.items():
        assert {k for k in (f.identity, f.fast, GENERIC) if k} <= {k for cc, k in ran if cc == code}, f.name
    assert {c.entry for c in cases} == {"table", "strided", "host"}
    assert {c.sampling for c in cases} == {0, 1, 3}
    assert {c.matrix for c in cases} == {0, 1, 2, 3}
    assert any(c.name.startswith("odd-frame-") and c.planned() == GENERIC for c in cases)
    assert any(c.dw % 4 and c.fmt.fast and c.planned() == GENERIC for c in cases)


# ── (2) rounding edges on white frames ──────────────────────────────────────────────────────────────────────────────
def f32(v):
    return float(np.float32(v))


# channel values on a white frame (every tap q == 1.0 exactly): o = (1 - mean) * inv_std, with mean = 1 - delta exact and
# 1 - mean == delta exact (Sterbenz), so o = delta * inv_std exactly.  Each: (delta, inv_std, expected bf16 bits) per channel.
EDGE_VALUES = {
    # ties: 1 + 2^-8 -> 1.0 (even), 1 + 3 * 2^-8 -> 1 + 2^-6 (even), -(1 + 2^-8) -> -1.0
    "ties": [(2.0 ** -8 + 2.0 ** -16, 256.0, 0x3F80), (2.0 ** -8 + 3 * 2.0 ** -16, 256.0, 0x3F82), (2.0 ** -8 + 2.0 ** -16, -256.0, 0xBF80)],
    # the tie above the largest finite bf16 (0x7F7F, odd) rounds to +-inf from a finite f32; just below it stays finite
    "overflow": [(2.0 - 2.0 ** -8, 2.0 ** 127, 0x7F80), (2.0 - 2.0 ** -8, -(2.0 ** 127), 0xFF80), (2.0 - 2.0 ** -7, 2.0 ** 127, 0x7F7F)],
    # subnormals: 2^-130 + 2^-134 ties to 2^-130 (0x0008); -(2^-130 + 3 * 2^-134) ties to -(2^-130 + 2^-132) (0x800A);
    # 2^-149, the least f32 subnormal, rounds to +0
    "subnormal": [(1.0 + 2.0 ** -4, 2.0 ** -130, 0x0008), (1.0 + 3 * 2.0 ** -4, -(2.0 ** -130), 0x800A), (1.0, 2.0 ** -149, 0x0000)],
    # +0 * 1 = +0, +0 * -1 = -0, 0 * inf = NaN
    "zero_nan": [(0.0, 1.0, 0x0000), (0.0, -1.0, 0x8000), (0.0, math.inf, None)],
}

# (format code, bpp, w, h, white frame) -> the geometries: identity kernels and a letterbox (fast or generic kernel)
WHITE = {
    "rgb": (0, 3, 64, 48), "nv12": (3, 1, 64, 48), "i444": (11, 1, 64, 48), "bayer8": (16, 1, 64, 48), "bayer12": (36, 2, 64, 48),
    "p010": (80, 2, 64, 48),
}


def white_frame(name):
    code, bpp, w, h = WHITE[name]
    if name == "rgb":
        return np.full(w * h * 3, 255, np.uint8), w * 3
    if name == "nv12":
        return np.concatenate([np.full(w * h, 255, np.uint8), np.full(w * h // 2, 128, np.uint8)]), w
    if name == "i444":
        return np.concatenate([np.full(w * h, 255, np.uint8), np.full(2 * w * h, 128, np.uint8)]), w
    if name == "bayer8":
        return np.full(w * h, 255, np.uint8), w
    if name == "bayer12":
        return np.full(w * h, 4095, "<u2").view(np.uint8), 2 * w
    words = np.concatenate([np.full(w * h, 1023 << 6, "<u2"), np.full(w * h // 2, 512 << 6, "<u2")])   # P010: codes in the high bits
    return words.view(np.uint8), 2 * w


def white_desc(name, geom, values, pad_value=255.0):
    from kornia_rs_b200._lib import PreprocessDesc
    code, bpp, w, h = WHITE[name]
    d = PreprocessDesc()
    if geom == "identity":
        d.scale_x, d.scale_y, d.pad_x, d.pad_y, d.dst_w, d.dst_h = 1.0, 1.0, 0.0, 0.0, w, h
    else:   # letterbox 64x48 -> 40x40: scale 0.625, 5 pad rows above and below
        a = (C.c_float * 4)()
        from kornia_rs_b200 import _lib
        _lib.lib().kb200_preprocess_affine(0, w, h, 40, 40, a)
        d.scale_x, d.scale_y, d.pad_x, d.pad_y, d.dst_w, d.dst_h = a[0], a[1], a[2], a[3], 40, 40
    d.src_w, d.src_h, d.src_bpp, d.fmt = w, h, bpp, code
    d.src_pitch = white_frame(name)[1]
    d.mean = (C.c_float * 3)(*[f32(1.0 - v[0]) for v in values])
    d.inv_std = (C.c_float * 3)(*[v[1] for v in values])
    d.pad_value, d.sampling = pad_value, BILINEAR
    return d


WHITE_RUNS = [(n, g) for n in WHITE for g in ("identity", "letterbox")]
WHITE_KERNELS = {("rgb", "identity"): GENERIC, ("rgb", "letterbox"): GENERIC, ("nv12", "identity"): "preprocess_nv12_identity_kernel",
                 ("nv12", "letterbox"): "preprocess_nv12_kernel", ("i444", "identity"): "preprocess_i444_identity_kernel",
                 ("i444", "letterbox"): "preprocess_i444_kernel", ("bayer8", "identity"): "preprocess_bayer_rggb_identity_kernel",
                 ("bayer8", "letterbox"): GENERIC, ("bayer12", "identity"): "preprocess_bayer16_rggb_identity_kernel",
                 ("bayer12", "letterbox"): GENERIC, ("p010", "identity"): "preprocess_p01x_identity_kernel", ("p010", "letterbox"): "preprocess_p01x_kernel"}


def run_strided(kb, lib, dev, d, frame, out, n=1):
    src = torch.from_numpy(np.tile(frame, n)).to(dev)
    elems = 3 * d.dst_w * d.dst_h * n
    dst = torch.empty(elems * ESZ[out], dtype=torch.uint8, device=dev)
    st = getattr(lib, DEVICE_FN["strided", out])(None, C.byref(d), src.data_ptr(), src.numel(), frame.size, n, dst.data_ptr(), elems)
    assert st == 0, kb._lib.last_error()
    ran = kb._lib.last_kernel()
    return dst.cpu().numpy(), ran


@gpu
@pytest.mark.parametrize("name,geom", WHITE_RUNS)
@pytest.mark.parametrize("edge_case", list(EDGE_VALUES))
def test_bf16_rounding_edges(kb, lib, dev, name, geom, edge_case):
    values = EDGE_VALUES[edge_case]
    d = white_desc(name, geom, values)
    frame = white_frame(name)[0]
    got, ran = run_strided(kb, lib, dev, d, frame, OUT_BF16)
    ref, ran32 = run_strided(kb, lib, dev, d, frame, OUT_F32)
    assert ran == ran32 == WHITE_KERNELS[name, geom], (ran, ran32)
    assert_bf16_matches(got, ref, f"{name} {geom} {edge_case}")
    planes = got.view(np.uint16).reshape(3, -1)
    f = ref.view(np.float32).reshape(3, -1)
    for ch, (_, _, bits) in enumerate(values):
        if bits is None:
            assert np.isnan(f[ch]).all() and np.all((planes[ch] & 0x7FFF) > 0x7F80), f"{name} {geom} {edge_case} channel {ch}: not NaN"
        else:
            assert np.all(planes[ch] == bits), f"{name} {geom} {edge_case} channel {ch}: {sorted(set(planes[ch].tolist()))[:4]} != {bits:#06x}"
    if edge_case == "overflow":
        assert np.isfinite(f[:2]).all()   # the f32 values are finite: the infinities come from the bf16 rounding
    if edge_case == "subnormal":
        assert np.all((f[:2] != 0) & (np.abs(f[:2]) < 1.17e-38))


@gpu
@pytest.mark.parametrize("name", list(WHITE))
def test_bf16_nan_pad_value(kb, lib, dev, name):
    """A NaN pad value: the letterbox rows are NaN, the frame's pixels are not."""
    d = white_desc(name, "letterbox", EDGE_VALUES["ties"], pad_value=float("nan"))
    frame = white_frame(name)[0]
    got, ran = run_strided(kb, lib, dev, d, frame, OUT_BF16)
    ref, _ = run_strided(kb, lib, dev, d, frame, OUT_F32)
    assert ran == WHITE_KERNELS[name, "letterbox"]
    assert_bf16_matches(got, ref, f"{name} NaN pad")
    nan = (got.view(np.uint16).reshape(3, 40, 40) & 0x7FFF) > 0x7F80
    assert nan[:, :5].all() and nan[:, -5:].all() and not nan[:, 5:-5].any()


# ── (3) batches over 256 frames at 1080p ────────────────────────────────────────────────────────────────────────────
@gpu
@pytest.mark.parametrize("n", [256, 300])
def test_bf16_1080p_batch(kb, lib, dev, n):
    w, h = 1920, 1080
    need = w * h * 3 // 2
    g = torch.Generator(device=dev).manual_seed(0xB16 + n)
    src = torch.randint(0, 256, (n * need,), dtype=torch.uint8, device=dev, generator=g)
    c = edge(f"nv12-1080p-{n}", 3, w, h, entry="strided", batch=n)
    d = desc_of(c)
    elems = 3 * w * h * n
    out = {}
    for o, dtype in ((OUT_F32, torch.float32), (OUT_BF16, torch.bfloat16)):
        dst = torch.empty(elems, dtype=dtype, device=dev)
        st = getattr(lib, DEVICE_FN["strided", o])(None, C.byref(d), src.data_ptr(), src.numel(), need, n, dst.data_ptr(), elems)
        assert st == 0, kb._lib.last_error()
        assert kb._lib.last_kernel() == "preprocess_nv12_identity_kernel"
        out[o] = dst
    torch.cuda.synchronize()
    want = out[OUT_F32].to(torch.bfloat16)
    assert torch.equal(out[OUT_BF16].view(torch.int16), want.view(torch.int16))
    del out, want
    # and through the Preprocessor's strided entry with dtype=torch.bfloat16
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda()
    dst = torch.empty((n, 3, h, w), dtype=torch.bfloat16, device=dev)
    pre.run_raw_strided(src, need, n, w, h, dst, dtype=torch.bfloat16)
    ref = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
    pre.run_raw_strided(src, need, n, w, h, ref)
    assert torch.equal(dst.view(torch.int16), ref.to(torch.bfloat16).view(torch.int16))


# ── (4) host pipeline ───────────────────────────────────────────────────────────────────────────────────────────────
@gpu
@pytest.mark.parametrize("code,w,h,dw,dh", [(3, 64, 48, 64, 48), (3, 64, 48, 40, 40), (80, 64, 48, 40, 40), (16, 64, 48, 64, 48), (4, 64, 48, 33, 17)])
def test_bf16_host_pipeline(kb, lib, dev, code, w, h, dw, dh):
    n = 7
    c = edge(f"host-{code}-{dw}x{dh}", code, w, h, dw, dh, mode=None if (w, h) == (dw, dh) else 0, entry="strided", batch=n)
    d = desc_of(c)
    need = c.need
    frames = np.concatenate([frame_bytes(c, k) for k in range(n)])
    elems = 3 * dw * dh * n
    dsrc = torch.from_numpy(frames).to(dev)
    device = {}
    for o in (OUT_F32, OUT_F16, OUT_BF16):
        dst = torch.empty(elems * ESZ[o], dtype=torch.uint8, device=dev)
        assert getattr(lib, DEVICE_FN["strided", o])(None, C.byref(d), dsrc.data_ptr(), dsrc.numel(), need, n, dst.data_ptr(), elems) == 0
        device[o] = (dst.cpu().numpy(), kb._lib.last_kernel())
    hsrc = torch.from_numpy(frames).pin_memory()
    # staging for 3 frames per chunk: several chunks per stream, a ragged last one, ring wrap
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * ((need + 15) // 16 * 16), dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
    try:
        for o in (OUT_F32, OUT_F16, OUT_BF16):
            hd = torch.zeros(elems * ESZ[o], dtype=torch.uint8).pin_memory()
            st = lib.kb200_preprocess_host_format(pipe._h, None, C.byref(d), hsrc.data_ptr(), hsrc.numel(), need, n, hd.data_ptr(), elems, o)
            assert st == 0, kb._lib.last_error()
            assert kb._lib.last_kernel() == device[o][1]
            torch.cuda.synchronize()
            up, down = C.c_uint64(), C.c_uint64()
            assert lib.kb200_host_pipeline_last_transfer(pipe._h, C.byref(up), C.byref(down)) == 0
            assert up.value == need * n and down.value == elems * ESZ[o]
            assert np.array_equal(hd.numpy(), device[o][0]), f"host out {o} differs from the device entry"
            if o != OUT_BF16:   # the old entry is the same call with out_f16 = 0 / 1
                old = torch.zeros_like(hd).pin_memory()
                assert lib.kb200_preprocess_host(pipe._h, None, C.byref(d), hsrc.data_ptr(), hsrc.numel(), need, n, old.data_ptr(), elems, o) == 0
                torch.cuda.synchronize()
                assert np.array_equal(old.numpy(), hd.numpy())
        assert_bf16_matches(device[OUT_BF16][0], device[OUT_F32][0], f"host {code}")
        # the Preprocessor: run_raw_host(dtype=torch.bfloat16), into a given tensor and into one it allocates
        fmt = {3: kb.SourceFormat.Nv12, 80: kb.SourceFormat.P010, 16: kb.SourceFormat.BayerRggb, 4: kb.SourceFormat.Yuyv}[code]
        pre = kb.Preprocessor.builder().source_format(fmt).mode(kb.ResizeMode.Letterbox).normalize(kb.Normalize.imagenet()).build_cuda()
        frames_t = torch.from_numpy(frames.reshape(n, need)).pin_memory()
        with torch.cuda.device(dev):
            got = pre.run_raw_host(frames_t, w, h, (dw, dh), dtype=torch.bfloat16, pipeline=pipe)
            torch.cuda.current_stream().synchronize()
            assert got.dtype == torch.bfloat16 and got.is_pinned() and not got.is_cuda
            assert pipe.last_transfer() == (need * n, elems * 2)
            ref = torch.empty((n, 3, dh, dw), dtype=torch.float32, device=dev)
            pre.run_raw_batch([dsrc[k * need:(k + 1) * need] for k in range(n)], w, h, ref)
            want = ref.to(torch.bfloat16).cpu()
            assert torch.equal(got.view(torch.int16), want.view(torch.int16))
            dev_bf16 = torch.empty((n, 3, dh, dw), dtype=torch.bfloat16, device=dev)
            pre.run_raw_batch_bf16([dsrc[k * need:(k + 1) * need] for k in range(n)], w, h, dev_bf16)
            assert torch.equal(dev_bf16.cpu().view(torch.int16), want.view(torch.int16))
            given = torch.zeros((n, 3, dh, dw), dtype=torch.bfloat16).pin_memory()
            assert pre.run_raw_host(frames_t, w, h, (dw, dh), given, dtype=torch.bfloat16, pipeline=pipe) is given
            torch.cuda.current_stream().synchronize()
            assert torch.equal(given.view(torch.int16), want.view(torch.int16))
    finally:
        pipe.close()


@gpu
def test_bf16_preprocessor_methods(kb, dev):
    """run_bf16, run_surface_bf16, run_raw_bf16 and run_raw_batch_bf16 equal their f32 twins rounded; a dst of any other
    dtype is refused with the f32 / f16 twins' error."""
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Rgb8).normalize(kb.Normalize.imagenet()).build_cuda()
    rng = np.random.default_rng(0xBF16)
    img = torch.from_numpy(rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)).to(dev)
    ref = torch.empty((1, 3, 40, 40), dtype=torch.float32, device=dev)
    image = kb.Image(img)
    pre.run(image, ref)
    want = ref.to(torch.bfloat16).view(torch.int16)
    surface = kb.PitchedSurface(img.view(-1), 64, 48, 64 * 3, 3)
    calls = {
        "run_bf16": lambda dst: pre.run_bf16(image, dst),
        "run_surface_bf16": lambda dst: pre.run_surface_bf16(surface, dst),
        "run_raw_bf16": lambda dst: pre.run_raw_bf16(img.view(-1), 64, 48, dst),
        "run_raw_batch_bf16": lambda dst: pre.run_raw_batch_bf16([img.view(-1)], 64, 48, dst),
    }
    for name, call in calls.items():
        dst = torch.full((1, 3, 40, 40), float("nan"), dtype=torch.bfloat16, device=dev)
        call(dst)
        assert torch.equal(dst.view(torch.int16), want), name
        for bad in (torch.float32, torch.float16, torch.float64):
            with pytest.raises(kb.PreprocessError) as e:
                call(torch.zeros((1, 3, 40, 40), dtype=bad, device=dev))
            assert e.value.kind == "BadOutputShape" and str(e.value) == f"destination tensor must be contiguous torch.bfloat16, got {bad}", name


# ── (5) memory footprint of the new entries ────────────────────────────────────────────────────────────────────────
FOOT = {   # one kernel of each family: (fmt code, w, h, dst size or None for the identity, letterbox mode, pitch padding)
    "generic": (0, 64, 48, (40, 40), 0, 16),
    "yuv420_identity": (3, 64, 48, None, None, 0),
    "yuv_fast": (3, 64, 48, (40, 40), 0, 0),
    "yuv444_identity": (11, 64, 48, None, None, 0),
    "bayer_identity": (16, 64, 48, None, None, 16),
}
FOOT_KERNEL = {"generic": GENERIC, "yuv420_identity": "preprocess_nv12_identity_kernel", "yuv_fast": "preprocess_nv12_kernel",
               "yuv444_identity": "preprocess_i444_identity_kernel", "bayer_identity": "preprocess_bayer_rggb_identity_kernel"}


def padding_mask(c):
    """True at the pitch padding bytes of a frame of case c."""
    m = np.zeros(c.need, bool)
    row = row_bytes(c.fmt, c.w, c.bpp)
    if c.pitch > row:
        m[:c.pitch * c.h].reshape(c.h, c.pitch)[:, row:] = True
    return m


@gpu
@pytest.mark.parametrize("family", list(FOOT))
def test_bf16_footprint(kb, lib, dev, family):
    code, w, h, dsize, mode, pp = FOOT[family]
    n = 3
    dw, dh = dsize or (w, h)
    c = edge(f"foot-{family}", code, w, h, dw, dh, mode=mode, pitch_pad=pp, entry="strided", batch=n)
    d = desc_of(c)
    need = c.need
    pad = padding_mask(c)
    clean = [np.where(pad, 0x00, frame_bytes(c, k)).astype(np.uint8) for k in range(n)]
    dirty = [np.where(pad, 0xFF, f).astype(np.uint8) for f in clean]
    out_elems = 3 * dw * dh
    # the reference: f32 from the clean frames, tight, rounded by torch
    tight = torch.from_numpy(np.concatenate(clean)).to(dev)
    ref = torch.empty(out_elems * n, dtype=torch.float32, device=dev)
    assert lib.kb200_preprocess_strided_f32(None, C.byref(d), tight.data_ptr(), tight.numel(), need, n, ref.data_ptr(), out_elems * n) == 0
    want = ref.cpu().numpy().view(np.uint8)
    gap = 48
    stride = need + gap
    ring_bytes = np.concatenate([np.concatenate([f, poison("u8", gap)]) for f in dirty])[:stride * (n - 1) + need]
    ring = Guarded(dev, ring_bytes.size, dw * 2).load("u8", ring_bytes)
    ring_before = ring.snapshot()
    hring = Guarded(dev, ring_bytes.size, host=True).load("u8", ring_bytes)
    singles = [Guarded(dev, need, dw * 2).load("u8", dirty[k]) for k in range(n)]
    ptrs = (C.c_void_p * n)(*[g.ptr for g in singles])
    lens = (C.c_size_t * n)(*[need] * n)
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=2 * ((need + 15) // 16 * 16), dst_chunk_bytes=2 * out_elems * 2, depth=2)
    calls = {
        "table": lambda dst, dl, ln=lens: lib.kb200_preprocess_bf16(None, C.byref(d), ptrs, ln, n, dst, dl),
        "strided": lambda dst, dl, bl=ring.n: lib.kb200_preprocess_strided_bf16(None, C.byref(d), ring.ptr, bl, stride, n, dst, dl),
        "host": lambda dst, dl, bl=hring.n: lib.kb200_preprocess_host_format(pipe._h, None, C.byref(d), hring.ptr, bl, stride, n, dst, dl, OUT_BF16),
    }
    try:
        for entry, call in calls.items():
            host = entry == "host"
            outs = []
            for fill in (0x00, 0xFF):
                dst = Guarded(dev, out_elems * 2 * n, dw * 2, host=host).fill(fill)
                st = call(dst.ptr, out_elems * n)
                assert st == 0, f"{family} {entry}: {kb._lib.last_error()}"
                assert kb._lib.last_kernel() == FOOT_KERNEL[family], f"{family} {entry}: ran {kb._lib.last_kernel()}"
                torch.cuda.synchronize()
                lead, tail = dst.guards()
                assert np.all(lead == fill) and np.all(tail == fill), f"{family} {entry}: write outside dst"
                outs.append(dst.out())
            assert np.array_equal(outs[0], outs[1]), f"{family} {entry}: output left unwritten"
            assert_bf16_matches(outs[0], want, f"{family} {entry}: poison reached the output")
            dst.fill(0x5A)
            before = dst.snapshot()
            assert call(dst.ptr, out_elems * n - 1) == -2 and "'dst'" in kb._lib.last_error(), f"{family} {entry}"
            if entry == "table":
                short = (C.c_size_t * n)(need, need - 1, need)
                assert call(dst.ptr, out_elems * n, short) == -8 and f"need {need}" in kb._lib.last_error()
            else:
                assert call(dst.ptr, out_elems * n, ring.n - 1) == -8 and f"need {ring.n}" in kb._lib.last_error()
            torch.cuda.synchronize()
            assert np.array_equal(dst.snapshot(), before), f"{family} {entry}: a refused call wrote"
    finally:
        pipe.close()
    assert np.array_equal(ring.snapshot(), ring_before)


# ── CPU: header, binding, validation, Python dtype rules ───────────────────────────────────────────────────────────
def test_header_declares_bf16_entries():
    hdr = open(os.path.join(ROOT, "include", "kornia_b200.h")).read()
    flat = " ".join(hdr.split())
    assert ("KB200_API int kb200_preprocess_bf16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* const* frames, "
            "const size_t* frame_len, uint32_t batch, uint16_t* dst, size_t dst_len);") in flat
    assert ("KB200_API int kb200_preprocess_strided_bf16(kb200_stream_t stream, const kb200_preprocess_desc* desc, const uint8_t* base, "
            "size_t base_len, size_t frame_stride, uint32_t batch, uint16_t* dst, size_t dst_len);") in flat
    assert ("KB200_API int kb200_preprocess_host_format(kb200_host_pipeline* pipeline, kb200_stream_t stream, const kb200_preprocess_desc* desc, "
            "const uint8_t* host_base, size_t base_len, size_t frame_stride, uint32_t batch, void* host_dst, size_t dst_len, int out_format);") in flat
    # the rounding rule, and kb200_preprocess_host's contract kept
    for words in ("__float2bfloat16_rn(the f32 value _f32 writes", "round to nearest even", "overflow to ±inf", "signed zeros and subnormals kept",
                  "a NaN stays a NaN (its payload unspecified)", "binary16 when out_f16 != 0",
                  "typedef enum { KB200_OUT_F32 = 0, KB200_OUT_F16 = 1, KB200_OUT_BF16 = 2 } kb200_out_format;", "kb200_preprocess_host_format)"):
        assert words in flat, words


def test_lib_binds_bf16_entries(kb):
    from kornia_rs_b200 import _lib
    l = _lib.lib()
    for name, n in (("kb200_preprocess_bf16", 7), ("kb200_preprocess_strided_bf16", 8), ("kb200_preprocess_host_format", 10)):
        fn = getattr(l, name)
        assert fn.argtypes is not None and len(fn.argtypes) == n and fn.restype is C.c_int, name
    assert l.kb200_preprocess_bf16.argtypes == l.kb200_preprocess_f16.argtypes
    assert l.kb200_preprocess_strided_bf16.argtypes == l.kb200_preprocess_strided_f16.argtypes
    assert l.kb200_preprocess_host_format.argtypes == l.kb200_preprocess_host.argtypes


def test_bf16_entries_validate_without_a_gpu(kb):
    """Every check runs before any device call, with the f16 entries' messages."""
    from kornia_rs_b200 import _lib
    l = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = (C.addressof(buf) + 15) & ~15
    d = _lib.PreprocessDesc()
    d.scale_x = d.scale_y = 1.0
    d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt, d.dst_w, d.dst_h, d.sampling = 8, 6, 8, 1, 3, 4, 4, 1   # NV12 8x6 -> 4x4
    need = 72
    ptrs, lens = (C.c_void_p * 1)(p), (C.c_size_t * 1)(need)
    table, strided, host = l.kb200_preprocess_bf16, l.kb200_preprocess_strided_bf16, l.kb200_preprocess_host_format
    fake = (C.c_uint8 * 1024)()   # validation returns before the pipeline is used: an opaque non-null handle suffices
    hp = C.addressof(fake)
    ERR_ARG, SLICE, SRC = _lib.ERR_INVALID_ARGUMENT, _lib.ERR_SLICE_TOO_SMALL, _lib.ERR_INVALID_SOURCE

    assert table(None, C.byref(d), None, lens, 1, p, 48) == ERR_ARG
    assert _lib.last_error() == "null pointer for 'frames'"
    assert table(None, C.byref(d), ptrs, lens, 1, None, 48) == ERR_ARG
    assert _lib.last_error() == "null pointer for 'dst'"
    assert strided(None, C.byref(d), p, need, need, 1, None, 48) == ERR_ARG
    assert _lib.last_error() == "null pointer for 'dst'"
    assert strided(None, C.byref(d), None, need, need, 1, p, 48) == ERR_ARG
    assert _lib.last_error() == "null pointer for 'base'"
    assert table(None, C.byref(d), ptrs, lens, 1, p, 47) == SLICE
    assert _lib.last_error() == "device slice 'dst' length 47 < required 48"
    assert strided(None, C.byref(d), p, need, need, 1, p, 47) == SLICE
    assert _lib.last_error() == "device slice 'dst' length 47 < required 48"
    assert table(None, C.byref(d), ptrs, lens, 0, p, 48) == ERR_ARG
    assert _lib.last_error() == "batch must be non-zero"
    assert strided(None, C.byref(d), p, need - 1, need, 1, p, 48) == SRC
    assert _lib.last_error() == f"invalid raw source at 8x6 (got {need - 1} bytes, need {need})"

    # the host form: the same checks, and an unknown output format with the fused resize host entry's message
    assert host(None, None, C.byref(d), p, need, need, 1, p, 48, OUT_BF16) == ERR_ARG
    assert _lib.last_error() == "null pointer for 'pipeline'"
    assert host(hp, None, C.byref(d), None, need, need, 1, p, 48, OUT_BF16) == ERR_ARG
    assert _lib.last_error() == "null pointer for 'base'"
    assert host(hp, None, C.byref(d), p, need, need, 1, None, 48, OUT_BF16) == ERR_ARG
    assert _lib.last_error() == "null pointer for 'dst'"
    for bad in (3, -1):
        assert host(hp, None, C.byref(d), p, need, need, 1, p, 48, bad) == ERR_ARG
        assert _lib.last_error() == f"unknown output format {bad}"
    for fmt in (OUT_F32, OUT_F16, OUT_BF16):
        assert host(hp, None, C.byref(d), p, need, need, 1, p, 47, fmt) == SLICE
        assert _lib.last_error() == "device slice 'dst' length 47 < required 48"
    assert host(hp, None, C.byref(d), p, need - 1, need, 1, p, 48, OUT_BF16) == SRC

    # a YUV matrix on a format that is not YUV
    d.fmt, d.src_pitch, d.src_bpp = 0 | (2 << 8), 24, 3
    for call in (lambda: table(None, C.byref(d), ptrs, lens, 1, p, 48), lambda: strided(None, C.byref(d), p, 4096, 144, 1, p, 48),
                 lambda: host(hp, None, C.byref(d), p, 4096, 144, 1, p, 48, OUT_BF16)):
        assert call() == ERR_ARG
        assert _lib.last_error() == "source format code 512: a YUV matrix (2) applies only to the YUV formats, not format code 0"

    # 16-bit frames that do not start 2-byte aligned: the pointer table, the strided base and the strided stride
    d.fmt, d.src_pitch, d.src_bpp = 80, 16, 2   # P010 8x6
    odd = (C.c_void_p * 1)(p + 1)
    assert table(None, C.byref(d), odd, (C.c_size_t * 1)(4096), 1, p, 1 << 20) == SRC
    assert _lib.last_error() == "P010 frame 0 is not 2-byte aligned"
    assert strided(None, C.byref(d), p + 1, 4096, 144, 1, p, 1 << 20) == SRC
    assert _lib.last_error().startswith("P010 frames must start 2-byte aligned")
    assert strided(None, C.byref(d), p, 4096, 145, 2, p, 1 << 20) == SRC
    assert _lib.last_error().startswith("P010 frames must start 2-byte aligned")


def test_bf16_python_dtype_rules(kb):
    """run_raw_host / run_raw_strided: dtype selects the output, f16=True with any dtype but float16 is an error; the host
    destination of a bf16 call must be bfloat16.  All refused before any device call."""
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).build_cuda()
    frames = torch.zeros((2, 8 * 6 * 3 // 2), dtype=torch.uint8)
    for dt in (torch.bfloat16, torch.float32):
        with pytest.raises(kb.PreprocessError) as e:
            pre.run_raw_host(frames, 8, 6, (4, 4), f16=True, dtype=dt)
        assert e.value.kind == "BadOutputShape" and str(e.value) == f"f16=True conflicts with dtype={dt}"
        with pytest.raises(kb.PreprocessError) as e:
            pre.run_raw_strided(frames.view(-1), 72, 2, 8, 6, torch.zeros((2, 3, 4, 4), dtype=dt), f16=True, dtype=dt)
        assert e.value.kind == "BadOutputShape" and str(e.value) == f"f16=True conflicts with dtype={dt}"
    for bad in (torch.float64, torch.int16, torch.uint8):
        with pytest.raises(kb.PreprocessError) as e:
            pre.run_raw_host(frames, 8, 6, (4, 4), dtype=bad)
        assert e.value.kind == "BadOutputShape" and "unsupported output dtype" in str(e.value)
    for have in (torch.float32, torch.float16):
        with pytest.raises(kb.PreprocessError) as e:
            pre.run_raw_host(frames, 8, 6, (4, 4), torch.zeros((2, 3, 4, 4), dtype=have), dtype=torch.bfloat16)
        assert e.value.kind == "BadOutputShape" and str(e.value) == "destination must be a contiguous host torch.bfloat16 tensor of shape [2, 3, 4, 4]"
    with pytest.raises(kb.PreprocessError) as e:   # without dtype, f16 still decides
        pre.run_raw_host(frames, 8, 6, (4, 4), torch.zeros((2, 3, 4, 4), dtype=torch.bfloat16), f16=True)
    assert str(e.value) == "destination must be a contiguous host torch.float16 tensor of shape [2, 3, 4, 4]"
