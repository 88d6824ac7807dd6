"""The suite's device-side plumbing: fixtures, developer knobs, guarded buffers, comparators and the calls the camera
preprocess tests share.  The restatements these compare against live in restate.py.
"""
import contextlib
import ctypes as C
import os
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from typing import Callable

import numpy as np
import pytest
import torch

from restate import BITS, ESZ, F32, IMAGENET_INV, LANCZOS, NORMS, decode_yuv16, demosaic, frame_bytes, preprocess_rgb16, white

@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


@contextlib.contextmanager
def knobs(kb, values):
    """Developer knobs (names contain dots, hence a dict), always reset to 0 (= the dispatcher's own choice)."""
    try:
        for name, v in values.items():
            kb._lib.set_knob(name, v)
        yield
    finally:
        for name in values:
            kb._lib.set_knob(name, 0)


def free_device_memory():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ── frame-by-frame comparison against the oracle ──
POOL = max(1, min(16, len(os.sched_getaffinity(0))))


def _one_omp_thread(oracle):
    oracle.set_threads(1)   # this worker's OpenMP teams: the pool is the parallelism


def check_frame(got, want, rule, what):
    """rule: "f32" = assert_f32_bits_or_signed_zero (bit-identical, +0 == -0); "exact" = equal elements (integers, 16-bit float bits);
    a float = within that absolute tolerance (Lanczos: sinf of two math libraries)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if rule == "f32":
        bad = (got.view(np.uint32) != want.view(np.uint32)) & ~((got == 0) & (want == 0))
        n = int(bad.sum())
        if n:
            assert_f32_bits_or_signed_zero(got, want, f"{what} ({n} of {got.size} elements differ)")
    elif rule == "exact":
        n = int((got != want).sum())
        assert n == 0, f"{what}: {n} of {got.size} elements differ"
    else:
        n = int((~(np.abs(got.astype(np.float64) - want.astype(np.float64)) <= rule)).sum())
        assert n == 0, f"{what}: {n} of {got.size} elements differ by more than {rule}"


def compare_frames(oracle, n, want_fn, got_fn, rule, what):
    """want_fn(i) -> the oracle's frame i (run in the pool, at most POOL frames ahead); got_fn(i) -> device frame i on the
    host.  Either may return a tuple (several outputs of one frame).  Stops at the first frame that differs and names it."""
    with ThreadPoolExecutor(POOL, initializer=_one_omp_thread, initargs=(oracle,)) as ex:
        pending = deque(ex.submit(want_fn, i) for i in range(min(POOL, n)))
        for i in range(n):
            want = pending.popleft().result()
            if i + POOL < n:
                pending.append(ex.submit(want_fn, i + POOL))
            got = got_fn(i)
            if isinstance(want, tuple):
                for k, (g, w) in enumerate(zip(got, want, strict=True)):
                    check_frame(g, w, rule, f"{what} (output {k}): frame {i} of {n}")
            else:
                check_frame(got, want, rule, f"{what}: frame {i} of {n}")


@pytest.fixture(scope="module")
def lib(kb):
    return kb._lib.lib()


# ── f32 comparators ──
TOL = 1e-4  # north_star: f32 interpolation / filter paths within 1e-4 abs


def cu(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def assert_f32_bits(got, want, what=""):
    """Within TOL, and the same bits everywhere."""
    got = np.asarray(got)
    want = np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert np.nanmax(d) <= TOL, f"{what}: max abs diff {np.nanmax(d)} > {TOL}"
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
        f"{what}: within tolerance (max {np.nanmax(d):.3g}) but not bit-identical ({int((got.view(np.uint32) != want.view(np.uint32)).sum())} elements)"


def assert_f32_bits_or_signed_zero(got, want, what=""):
    """Within TOL, and the same bits everywhere except +0.0 against -0.0."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert np.nanmax(d) <= TOL, f"{what}: max abs diff {np.nanmax(d)} > {TOL}"
    nbad = int((got.view(np.uint32) != want.view(np.uint32)).sum())
    # +0.0 / -0.0 are the same value; everything else must be the same bits
    if nbad:
        both_zero = (got == 0) & (want == 0)
        nbad = int(((got.view(np.uint32) != want.view(np.uint32)) & ~both_zero).sum())
    assert nbad == 0, f"{what}: within tolerance (max {np.nanmax(d):.3g}) but {nbad} elements are not bit-identical"


def rot(kb, w, h, angle, scale=1.0):
    return kb.imgproc.get_rotation_matrix2d((w / 2.0, h / 2.0), angle, scale)


# ── guarded buffers (the memory-footprint checks) ──
GUARD = 4096


NAN_INF = np.array([0x7FC00000, 0x7F800000, 0xFF800000], np.uint32)   # f32 poison: NaN, +inf, -inf


OK, SLICE = 0, -2


def poison(kind, n):
    if kind == "f32":
        return np.resize(NAN_INF, (n + 3) // 4).view(np.uint8)[:n].copy()
    return np.full(n, 0xFF, np.uint8)   # u8 255, u16 0xFFFF


def as_bytes(a):
    return np.ascontiguousarray(a).reshape(-1).view(np.uint8)


class Guarded:
    """One allocation [lead | region | tail]: `region` (nbytes, `offset` bytes past a 16-B boundary) is what a call gets."""

    def __init__(self, dev, nbytes, guard=GUARD, offset=0, host=False):
        g = -(-(guard + GUARD) // 16) * 16
        self.lead, self.n = g + offset, nbytes
        t = torch.empty(self.lead + nbytes + g, dtype=torch.uint8, device=None if host else dev)
        self.buf = t.pin_memory() if host else t
        assert self.buf.data_ptr() % 16 == 0
        self.region = self.buf[self.lead:self.lead + nbytes]

    @property
    def ptr(self):
        return self.region.data_ptr()

    def fill(self, byte):
        self.buf.fill_(byte)
        return self

    def load(self, kind, data):
        """Poison everywhere, then `data` (bytes) in the region."""
        self.buf.copy_(torch.from_numpy(poison(kind, self.buf.numel())))
        self.region.copy_(torch.from_numpy(np.ascontiguousarray(data)))
        return self

    def snapshot(self):
        return self.buf.cpu().numpy().copy()

    def guards(self):
        b = self.buf.cpu().numpy()
        return b[:self.lead], b[self.lead + self.n:]

    def out(self):
        return self.region.cpu().numpy().copy()


def expect_refused(kb, st, what):
    assert st == SLICE, f"short '{what}' was accepted (status {st})"
    assert f"'{what}'" in kb._lib.last_error(), kb._lib.last_error()


@dataclass
class FootprintCase:
    id: str
    kernel: str | tuple          # kb200_last_kernel() of the launch (the last one when a call launches several)
    frame: Callable              # k -> clean source frame k (numpy; its dtype is the source element type)
    oracle: Callable             # frame -> expected output of that frame (numpy; its dtype is the output element type)
    call: Callable               # (lib, src, src_len, dst, dst_len, batch, aux) -> status; lengths in elements
    src_elems: int | None        # per frame (None: the size of the case's frames)
    dst_elems: int               # per frame
    batch: int = 2
    offset: bool = False         # element-aligned but not 16-B aligned src and dst (the fallbacks)
    knobs: dict = field(default_factory=dict)
    aux: dict = field(default_factory=dict)   # name -> (numpy input, poison kind), or name -> (lib, batch) -> scratch bytes
    lengths: bool = True         # the entry point takes src_len / dst_len
    row: int = 0                 # bytes of one output row (guard size); 0: the whole output frame
    pre: Callable = None         # extra assertion run before the call (schedule mirrors)


def kind_of(dtype):
    return {np.dtype(np.float32): "f32", np.dtype(np.uint8): "u8", np.dtype(np.uint16): "u16"}[np.dtype(dtype)]


def compare_to_oracle(got, want, what):
    if want.dtype == np.float32:
        assert_f32_bits_or_signed_zero(got.view(np.float32), want.reshape(-1), what)
    else:
        g, w = got, as_bytes(want)
        bad = np.flatnonzero(g != w)
        assert bad.size == 0, f"{what}: {bad.size} bytes differ from the oracle, first at byte {bad[0]}"


def run_guarded(kb, lib, dev, case, frames, check_frames, check_lengths):
    """Runs `case` on `frames` (a tight batch) with guarded buffers; returns nothing, asserts everything."""
    batch = len(frames)
    s_item = frames[0].dtype.itemsize
    want = [case.oracle(frames[k]) for k in check_frames]
    d_item = want[0].dtype.itemsize
    src_elems = frames[0].size
    assert case.src_elems in (None, src_elems), (case.id, case.src_elems, src_elems)
    src_bytes, dst_bytes = src_elems * s_item * batch, case.dst_elems * d_item * batch
    s_off, d_off = (s_item if s_item < 4 else 4, d_item if d_item < 4 else 4) if case.offset else (0, 0)
    guard = case.row or case.dst_elems * d_item
    # the source guards hold at least one whole source frame, so a tap one row past the last frame stays inside the allocation
    src = Guarded(dev, src_bytes, max(guard, min(src_elems * s_item, 8 << 20)), s_off).load(kind_of(frames[0].dtype), np.concatenate([as_bytes(f) for f in frames]))
    src_before = src.snapshot()
    aux, aux_before = {}, {}
    for name, spec in case.aux.items():
        if callable(spec):
            aux[name] = Guarded(dev, spec(lib, batch)).fill(0xA5)
        else:
            aux[name] = Guarded(dev, spec[0].nbytes).load(spec[1], as_bytes(spec[0]))
        aux_before[name] = aux[name].snapshot()
    ptrs = {k: v.ptr for k, v in aux.items()}
    s_len, d_len = src_elems * batch, case.dst_elems * batch
    outs = []
    with knobs(kb, case.knobs):
        for fill in (0x00, 0xFF):
            dst = Guarded(dev, dst_bytes, guard, d_off).fill(fill)
            st = case.call(lib, src.ptr, s_len, dst.ptr, d_len, batch, ptrs)
            assert st == OK, f"{case.id}: status {st}: {kb._lib.last_error()}"
            k = kb._lib.last_kernel()
            assert k in ((case.kernel,) if isinstance(case.kernel, str) else case.kernel), f"{case.id}: ran {k}"
            torch.cuda.synchronize()
            lead, tail = dst.guards()
            for what, g in (("lead", lead), ("tail", tail)):
                bad = np.flatnonzero(g != fill)
                assert bad.size == 0, f"{case.id}: {bad.size} bytes written in the {what} guard (first at {bad[0] - (g.size if what == 'lead' else 0)} from the region)"
            outs.append(dst.out())
        nw = np.flatnonzero(outs[0] != outs[1])
        assert nw.size == 0, f"{case.id}: {nw.size} output bytes left unwritten (first at byte {nw[0]})"
        fb = case.dst_elems * d_item
        for k, w in zip(check_frames, want):
            compare_to_oracle(outs[0][k * fb:(k + 1) * fb], w, f"{case.id} frame {k}")
        assert np.array_equal(src.snapshot(), src_before), f"{case.id}: the source allocation changed"
        for name, g in aux.items():
            now = g.snapshot()
            if callable(case.aux[name]):   # scratch: contents are the call's, the guards are not
                lead, tail = g.guards()
                assert np.all(lead == 0xA5) and np.all(tail == 0xA5), f"{case.id}: write around '{name}'"
            else:
                assert np.array_equal(now, aux_before[name]), f"{case.id}: input '{name}' or its guards changed"
        if check_lengths and case.lengths:
            dst.fill(0x5A)
            before = dst.snapshot()
            expect_refused(kb, case.call(lib, src.ptr, s_len, dst.ptr, d_len - 1, batch, ptrs), "dst")
            expect_refused(kb, case.call(lib, src.ptr, s_len - 1, dst.ptr, d_len, batch, ptrs), "src")
            torch.cuda.synchronize()
            assert np.array_equal(dst.snapshot(), before), f"{case.id}: a refused call wrote to dst"
            assert np.array_equal(src.snapshot(), src_before)


def neighbour_frames(case):
    """Batch of three tight frames: f32 -> finite, all NaN, finite; integer -> all 0, all max, all 0."""
    f = case.frame(0)
    if f.dtype == np.float32:
        return [case.frame(0), np.full_like(f, np.nan), case.frame(2)]
    return [np.zeros_like(f), np.full_like(f, np.iinfo(f.dtype).max), np.zeros_like(f)]


# ── device buffers and frame generators ──
def offset_buf(dev, n, off, dtype):
    """A device buffer of n elements whose data pointer is `off` elements past the start of a fresh allocation."""
    return torch.empty(n + off, dtype=dtype, device=dev)[off:]


def to_dev16(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a).astype(np.int32)).to(dev).to(torch.uint16)


def to_np16(t):
    return t.to(torch.int32).cpu().numpy().astype(np.uint16)


# ── the camera preprocess, against the restatements ──
def make_pre(kb, fmt, mode, sampling, matrix=None):
    """A CUDA Preprocessor for `fmt` with ImageNet normalisation and pad value 114 (and YUV `matrix` when given)."""
    b = (kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode[mode]).sampling(kb.InterpolationMode[sampling])
         .normalize(kb.Normalize.imagenet()).pad_value(114))
    return (b.yuv_matrix(kb.YuvMatrix[matrix]) if matrix else b).build_cuda()


def restated(kb, rgb, bits, mode, sampling, dw, dh, f16=False):
    from kornia_rs_b200 import _lib

    h, w = rgb.shape[:2]
    a = (C.c_float * 4)()
    _lib.lib().kb200_preprocess_affine(kb.ResizeMode[mode].value, w, h, dw, dh, a)
    inv = tuple(F32(1.0) / F32(s) for s in kb.IMAGENET_STD)
    return preprocess_rgb16(rgb, bits, tuple(a), dw, dh, sampling, kb.IMAGENET_MEAN, inv, 114.0, f16)


def check_against_restatement(got, o, sampling, f16, what):
    g = got.cpu().numpy()
    if sampling == "Lanczos":
        assert np.max(np.abs(g.astype(np.float32) - o.astype(np.float32))) <= (2e-3 if f16 else 1e-4), what
    elif f16:
        np.testing.assert_array_equal(g.view(np.uint16), o.view(np.uint16), what)
    else:
        np.testing.assert_array_equal(g.view(np.uint32), o.view(np.uint32), what)


def bayer16_identity(raw, pattern, bits, kb):
    """Config 3a of 16-bit frames [n, h, w] on the device: the restatement's demosaic, then (px / W - mean) * inv_std
    as separate IEEE f32 operations."""
    # the divisor is a device tensor: torch turns division by a host scalar into a multiplication by its reciprocal
    wl = torch.full((1,), float(white(bits)), dtype=torch.float32, device=raw.device)
    rgb = demosaic(raw, pattern).to(torch.int32).to(torch.float32) / wl
    mean = torch.tensor(kb.IMAGENET_MEAN, dtype=torch.float32, device=raw.device)
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(kb.IMAGENET_STD, dtype=torch.float32)
    return ((rgb - mean) * inv.to(raw.device)).permute(0, 3, 1, 2)


def raw_bytes(n, k=0):
    """The reference's frame generator (preprocess.rs): bytes ((i*7+13) % 251) + 31k, wrapping to u8."""
    return ((np.arange(n, dtype=np.int64) * 7 + 13) % 251 + 31 * k).astype(np.uint8)


def oracle_cfg(kb, oracle, mode, sampling):
    """The oracle's PreprocessCfg for RGB8 frames matching make_pre."""
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    return oracle.PreprocessCfg(mode=oracle.LETTERBOX if mode == "Letterbox" else oracle.STRETCH, fmt=oracle.FMT_RGB,
                                mean=kb.IMAGENET_MEAN, inv_std=inv, pad_value=114.0,
                                sampling={"Bilinear": oracle.BILINEAR, "Nearest": oracle.NEAREST, "Lanczos": oracle.LANCZOS}[sampling])


def random_bytes(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def random_words(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 1 << 16, shape, generator=g, dtype=torch.int32).to(torch.uint16)


def yuv16_identity(raw, w, h, fmt, m, kb):
    """Config 3a of frames [n, w*h*3/2] on the device: the restatement's decode, then (px / W - mean) * inv_std as
    separate IEEE f32 operations."""
    # the divisor is a device tensor: torch turns division by a host scalar into a multiplication by its reciprocal
    wl = torch.full((1,), float(white(BITS[fmt])), dtype=torch.float32, device=raw.device)
    rgb = decode_yuv16(raw, w, h, fmt, m).to(torch.float32) / wl
    mean = torch.tensor(kb.IMAGENET_MEAN, dtype=torch.float32, device=raw.device)
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(kb.IMAGENET_STD, dtype=torch.float32)
    return ((rgb - mean) * inv.to(raw.device)).permute(0, 3, 1, 2)


def compare_region(got, want, rc, what):
    c = rc.base
    if rc.out == "bf16" and c.sampling != LANCZOS:
        want = torch.from_numpy(np.ascontiguousarray(want, np.float32)).to(torch.bfloat16).view(torch.int16).numpy()
    if c.sampling == LANCZOS:
        g = (torch.from_numpy(got.copy()).view(torch.bfloat16).float().numpy() if rc.out == "bf16"
             else got.view(np.float16 if rc.out == "f16" else np.float32).astype(np.float32))
        want = want.reshape(-1).astype(np.float32)
        step = {"f32": 0.0, "f16": np.spacing(np.abs(want).astype(np.float16)).astype(np.float32),
                "bf16": np.abs(want) * 2.0 ** -7 + 1e-38}[rc.out]
        tol = 1e-4 * max(1.0, max(NORMS[c.norm][1]) / max(IMAGENET_INV)) + step
        over = np.abs(g - want) - tol
        assert over.max() <= 0, f"{what}: error {float(np.abs(g - want)[over.argmax()])} at element {int(over.argmax())}"
    else:
        w = np.ascontiguousarray(want).reshape(-1).view(np.uint8)
        bad = np.flatnonzero(got != w)
        assert bad.size == 0, f"{what}: {bad.size} bytes differ, first at byte {bad[0]}"


# ── the region entries ──
def roi_array(rois):
    from kornia_rs_b200._lib import Roi
    return (Roi * max(1, len(rois)))(*[Roi(*r) for r in rois])


def load_frames(dev, rc):
    c = rc.base
    need = c.need
    raws = [frame_bytes(c, k) for k in range(rc.n_frames)]
    span = rc.offsets[-1] + need + 16
    image = np.random.default_rng(c.seed ^ 0xBAD).integers(0, 256, span, dtype=np.int64).astype(np.uint8)   # poisoned gaps
    for s, r in zip(rc.offsets, raws):
        image[s:s + need] = r
    return raws, Guarded(dev, span).load("u8", image)


def inverse(lib, m):
    """(the library's f32 inverse of forward map m as a 3x3 float32 array, perspective?) — the entry's host computation."""
    m = (C.c_float * 9)(*m)
    out = (C.c_float * 9)()
    persp = not (m[6] == 0.0 and m[7] == 0.0 and m[8] == 1.0)
    if persp:
        assert lib.kb200_invert_homography(m, out) == 0
    else:
        lib.kb200_invert_affine_transform(m, out)
        out[6], out[7], out[8] = 0.0, 0.0, 1.0
    return np.array(out[:], F32).reshape(3, 3), persp


def warp_array(warps):
    from kornia_rs_b200._lib import WarpRoi
    return (WarpRoi * max(1, len(warps)))(*[WarpRoi(k, (C.c_float * 9)(*m)) for k, m in warps])


def batch_entry(lib, c, out, ptrs, dst):
    """The batch entry on the frames at ptrs with the descriptor's scale 1, pad 0 (Stretch of a frame to its own size)."""
    from kornia_rs_b200._lib import PreprocessDesc
    d = c.desc(PreprocessDesc)
    fn = getattr(lib, f"kb200_preprocess_{out}")
    return fn(None, C.byref(d), (C.c_void_p * len(ptrs))(*ptrs), None, len(ptrs), dst.data_ptr(), dst.numel() * dst.element_size() // ESZ[out])
