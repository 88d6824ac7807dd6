"""Camera preprocess: kb200_preprocess_warps, rotated and perspective crops of a set of frames, one forward map per region,
for every source format.

The reference (`warp_reference`) is a numpy float32 restatement: each numpy float32 operation rounds once and is never
fused, as the library is compiled (-fmad=false).  It restates warp_coord's affine and perspective expressions and inside
rules, the clamp of a degenerate axis, the bilinear / nearest sampler over the decoded picture (test_preprocess_roi.picture)
and the normalisation of the picture's bit depth; the inverse map is the library's kb200_invert_* of the forward map.

On the GPU:
  * twins, bit for bit: an identity map of a whole frame against the batch entry (every format, sampler and output type);
    integer translations and power-of-two downscales against kb200_preprocess_rois on the same rectangle; 90 / 180 / 270
    degree rotations and both flips of RGB8 / BGR8 / Gray8 / I444 / I41x frames against the batch entry on the frame
    rotated on the host;
  * a seeded sweep (`wcase(i)`, a pure function of i, every format twice) of similarity, general affine and perspective
    maps against the reference, each run into a harness.Guarded destination with a 0xFF prefill, on the kernel a
    host mirror of the dispatch rule names, and again one element past a 16-byte boundary, where the generic kernel must
    give the same bytes;
  * region counts around the launch chunk, a captured graph, Preprocessor.run_warps with both matrix shapes;
  * an independent anchor: cv2.warpAffine / warpPerspective (INTER_LINEAR, BORDER_CONSTANT) on smooth RGB8 frames.
On the CPU: every host refusal, the header and binding symbols, run_warps' argument rules and what the sweep covers.
"""
import ctypes as C
import os
import re
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from harness import Guarded, batch_entry, compare_region, dev, inverse, lib, load_frames, roi_array, warp_array
from restate import BILINEAR, CODES, Case, ESZ, FORMATS, LANCZOS, NEAREST, NORMS, OUTS, RCase, SAMPLING_NAME, draw_map, forward_of, frame_bytes, make_case, pad_step, picture, place, row_bytes, size_rule, smooth_rgb, src_bytes, warp_coords, warp_reference, yuv


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = 0x3A7F0000
CHUNK = 72   # regions per launch (preprocess_warp.cu WARP_CHUNK)
VECTOR, GENERIC = "preprocess_warp_kernel", "preprocess_warp_generic_kernel"
INVALID, SLICE, SINGULAR, UNSUPPORTED, INVALID_SOURCE = -1, -2, -3, -4, -8
F32 = np.float32
KINDS = ("similarity", "affine", "perspective", "edges", "wzero", "wcross", "rot90", "tiny")


# ── the dispatch rule, restated (preprocess_warp.cu warp_vector_ok) ──────────────────────────────────────────────────
def expected_kernel(dw, out, dst):
    return VECTOR if dw % 4 == 0 and dst % (16 if out == "f32" else 8) == 0 else GENERIC


# ── the cases ──────────────────────────────────────────────────────────────────────────────────────────────────────────
@dataclass(frozen=True)
class WCase:
    base: Case                # format, frame geometry, sampler, normalisation, pad value, dst size
    out: str
    n_frames: int
    offsets: tuple            # each frame's byte offset in one allocation (16-B aligned base)
    warps: tuple              # (k, forward map of 9 floats)
    kinds: tuple = ()         # the kind of each map (coverage)

    @property
    def rcase(self):   # the region tests' case, for load_frames and compare
        return RCase(self.base, 1, self.out, self.n_frames, self.offsets, ())

    def kernel(self, dst=0):
        return expected_kernel(self.base.dw, self.out, dst)

    def __str__(self):
        c = self.base
        return (f"{c.name}: {c.fmt.name} matrix {c.matrix} bpp {c.bpp} {c.w}x{c.h} pitch {c.pitch} -> {c.dw}x{c.dh} {SAMPLING_NAME[c.sampling]} "
                f"{self.out} norm {c.norm} pad {c.pad_value} frames {self.offsets} {len(self.warps)} maps, first {self.warps[:2]}")


def wcase(i):
    """Case i of the sweep: a pure function of i.  Format i % 51; the first pass over the formats writes a width the vector
    kernel takes, from even frame addresses."""
    rng = np.random.default_rng(BASE + i)
    f = FORMATS[CODES[i % len(CODES)]]
    bpp = int(rng.choice([3, 4])) if f.family == "rgb" else 1
    mw, mh, sw, sh = size_rule(f)
    w = max(mw, int(rng.integers(mw, 49)) // sw * sw)
    h = max(mh, int(rng.integers(mh, 41)) // sh * sh)
    step = pad_step(f)
    pitch = row_bytes(f, w, bpp) + (step * int(rng.integers(1, 8)) if step and rng.random() < 0.5 else 0)
    dw, dh = int(rng.integers(1, 41)), int(rng.integers(1, 41))
    first = i < len(CODES)
    if first or rng.random() < 0.4:
        dw = max(4, dw // 4 * 4)
    sampling = int(rng.choice([NEAREST, BILINEAR]))
    n_frames = int(rng.integers(1, 4))
    n = int(rng.choice([int(rng.integers(1, 8)), int(rng.integers(1, 101))]))
    base = make_case(f"warp-{i}", BASE + i, f.code, (i % len(CODES) + 2 * (i // len(CODES))) % 4 if yuv(f) else 0, bpp, w, h, pitch, dw, dh,
                     sampling, str(rng.choice(list(NORMS))), float(rng.integers(0, 256)))
    offs = place(rng, f, src_bytes(f, w, h, pitch), n_frames, odd=not first and rng.random() < 0.3)
    kinds = tuple(KINDS[j % len(KINDS)] if j < len(KINDS) and rng.random() < 0.7 else str(rng.choice(KINDS)) for j in range(n))
    warps = tuple((int(rng.integers(0, n_frames)), draw_map(rng, k, w, h, dw, dh)) for k in kinds)
    return WCase(base, str(rng.choice(OUTS)), n_frames, offs, warps, kinds)


N_SWEEP = 2 * len(CODES)


def chunk_cases():
    """n_warps around the launch chunk, mixed frame indices and map kinds: NV12 and 8-bit GRBG Bayer."""
    out = []
    for j, n in enumerate((CHUNK - 1, CHUNK, CHUNK + 1, 300)):
        for code in (3, 18):
            rng = np.random.default_rng(BASE + 0x1000 + 16 * j + code)
            f = FORMATS[code]
            w, h = 24, 16
            base = make_case(f"chunk-{n}-{f.name}", BASE + 0x1000 + n, code, 1 if code == 3 else 0, 1, w, h, row_bytes(f, w, 1), 8, 6, BILINEAR,
                             "imagenet", 114.0)
            kinds = tuple(KINDS[q % len(KINDS)] for q in range(n))
            warps = tuple((int(rng.integers(0, 3)), draw_map(rng, k, w, h, 8, 6)) for k in kinds)
            out.append(WCase(base, OUTS[j % 3], 3, place(rng, f, src_bytes(f, w, h, base.pitch), 3), warps, kinds))
    return out


CHUNKS = chunk_cases()


def call(lib, c, ptrs, lens, warps, dst_ptr, dst_len, out, stream=None, desc=None):
    from kornia_rs_b200._lib import PreprocessDesc
    d = desc if desc is not None else c.desc(PreprocessDesc)
    n = len(ptrs)
    return lib.kb200_preprocess_warps(stream, C.byref(d), (C.c_void_p * max(1, n))(*ptrs), (C.c_size_t * max(1, n))(*lens) if lens is not None else None,
                                      n, warp_array(warps), len(warps), dst_ptr, dst_len, OUTS.index(out))


def run_wcase(kb, lib, dev, wc):
    c = wc.base
    raws, src = load_frames(dev, wc.rcase)
    ptrs = [src.ptr + o for o in wc.offsets]
    m = len(wc.warps)
    elems = 3 * c.dw * c.dh
    nbytes = m * elems * ESZ[wc.out]
    outs = []
    for off in (0, ESZ[wc.out]):
        dst = Guarded(dev, nbytes, min(nbytes, 1 << 16), off).fill(0xFF)
        st = call(lib, c, ptrs, [c.need] * wc.n_frames, wc.warps, dst.ptr, m * elems, wc.out)
        assert st == 0, f"{wc}: status {st}: {kb._lib.last_error()}"
        ran = kb._lib.last_kernel()
        torch.cuda.synchronize()
        want = expected_kernel(c.dw, wc.out, dst.ptr)
        assert ran == want == wc.kernel(off), f"{wc}: dst +{off} B ran {ran}, the dispatch mirror says {want}"
        for what, g in zip(("lead", "tail"), dst.guards()):
            assert (g == 0xFF).all(), f"{wc}: dst +{off} B: bytes written in the {what} guard"
        outs.append(dst.out())
    esz = ESZ[wc.out]
    ones = outs[0].view(np.uint16 if esz == 2 else np.uint32) == (0xFFFF if esz == 2 else 0xFFFFFFFF)
    assert not ones.any(), f"{wc}: {int(ones.sum())} output elements left unwritten"
    pics = {}
    fb = elems * esz
    for i, (k, fwd) in enumerate(wc.warps):
        if k not in pics:
            pics[k] = picture(c, raws[k])
        inv, persp = inverse(lib, fwd)
        want = warp_reference(pics[k], inv, persp, c.dw, c.dh, c.sampling, c.norm, c.pad_value, wc.out)
        compare_region(outs[0][i * fb:(i + 1) * fb], want, wc.rcase, f"{wc}: region {i} frame {k} map {fwd}")
    bad = np.flatnonzero(outs[0] != outs[1])
    assert bad.size == 0, f"{wc}: {wc.kernel()} and {GENERIC} differ in {bad.size} bytes"


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_SWEEP))
def test_sweep(kb, lib, dev, i):
    run_wcase(kb, lib, dev, wcase(i))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.base.name for c in CHUNKS])
def test_chunking(kb, lib, dev, name):
    run_wcase(kb, lib, dev, next(c for c in CHUNKS if c.base.name == name))


@pytest.mark.gpu
@pytest.mark.parametrize("code", CODES)
def test_identity_twin(kb, lib, dev, code):
    """An identity map of each whole frame == the batch entry on that frame at dst = src_w x src_h (Stretch: scale 1, pad 0;
    the identity kernel where the format has one), for Nearest and Bilinear and every output type."""
    f = FORMATS[code]
    mw, mh, sw, sh = size_rule(f)
    w, h = max(mw, 20 // sw * sw), max(mh, 12 // sh * sh)
    ident = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)
    for j, (samp, out) in enumerate([(s, o) for s in (NEAREST, BILINEAR) for o in OUTS]):
        c = make_case(f"identity-{f.name}", BASE + 0x3000 + code, code, j % 4 if yuv(f) else 0, 3, w, h, row_bytes(f, w, 3), w, h, samp,
                      "imagenet", 114.0)
        wc = WCase(c, out, 2, (16, 16 + -(-c.need // 16) * 16), ((1, ident), (0, ident)))
        raws, src = load_frames(dev, wc.rcase)
        ptrs = [src.ptr + o for o in wc.offsets]
        got = torch.full((2 * 3 * w * h * ESZ[out],), 0xFF, dtype=torch.uint8, device=dev)
        assert call(lib, c, ptrs, [c.need] * 2, wc.warps, got.data_ptr(), 2 * 3 * w * h, out) == 0, kb._lib.last_error()
        want = torch.zeros_like(got)
        assert batch_entry(lib, c, out, [ptrs[1], ptrs[0]], want) == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"{f.name} {SAMPLING_NAME[samp]} {out}: identity map differs from the batch entry"


@pytest.mark.gpu
@pytest.mark.parametrize("code", CODES)
def test_translation_and_downscale_twin(kb, lib, dev, code):
    """Integer translations (s = 1) and power-of-two downscales (s = 1/2, 1/4) of a rw x rh rectangle at (x, y) into
    dst = rw*s x rh*s == kb200_preprocess_rois on that rectangle (Stretch).  The region's and the frame's clamps coincide
    because neither is reached: rw and rh are multiples of 1/s, so every sample lands on the integer frame pixel
    x + ox/s (inside the rectangle), bilinear reads only its (x0, y0) tap and nearest rounds nothing.  The test asserts
    that the library's inverse of each map is exactly (1/s, 0, x; 0, 1/s, y)."""
    f = FORMATS[code]
    mw, mh, sw, sh = size_rule(f)
    w, h = max(mw, 40 // sw * sw), max(mh, 24 // sh * sh)
    rng = np.random.default_rng(BASE + 0x4000 + code)
    for s, (samp, out) in zip((1.0, 0.5, 0.25, 1.0, 0.5, 0.25), [(NEAREST, "f32"), (BILINEAR, "f16"), (BILINEAR, "bf16"), (BILINEAR, "f32"),
                                                                  (NEAREST, "bf16"), (NEAREST, "f16")]):
        k = int(round(1 / s))
        rw, rh = (int(rng.integers(1, w // k + 1)) * k, int(rng.integers(1, h // k + 1)) * k)
        dw, dh = rw // k, rh // k
        c = make_case(f"shift-{f.name}", BASE + 0x4000 + code, code, int(rng.integers(0, 4)) if yuv(f) else 0, 3, w, h, row_bytes(f, w, 3), dw, dh,
                      samp, "imagenet", float(rng.integers(0, 256)))
        rois = [(int(rng.integers(0, 2)), int(rng.integers(0, w - rw + 1)), int(rng.integers(0, h - rh + 1)), rw, rh) for _ in range(5)]
        warps = [(q, (s, 0.0, -s * x, 0.0, s, -s * y, 0.0, 0.0, 1.0)) for q, x, y, _, _ in rois]
        for (q, x, y, _, _), (_, fwd) in zip(rois, warps):
            inv, persp = inverse(lib, fwd)
            assert not persp and np.array_equal(inv, np.array([[1 / s, 0, x], [0, 1 / s, y], [0, 0, 1]], F32)), (fwd, inv)
        wc = WCase(c, out, 2, (16, 16 + -(-c.need // 16) * 16), tuple(warps))
        raws, src = load_frames(dev, wc.rcase)
        ptrs = [src.ptr + o for o in wc.offsets]
        n = len(rois) * 3 * dw * dh
        got = torch.full((n * ESZ[out],), 0xFF, dtype=torch.uint8, device=dev)
        want = torch.zeros_like(got)
        assert call(lib, c, ptrs, [c.need] * 2, warps, got.data_ptr(), n, out) == 0, kb._lib.last_error()
        from kornia_rs_b200._lib import PreprocessDesc
        d = c.desc(PreprocessDesc)
        assert lib.kb200_preprocess_rois(None, C.byref(d), 1, (C.c_void_p * 2)(*ptrs), None, 2, roi_array(rois), len(rois), want.data_ptr(), n,
                                         OUTS.index(out)) == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"{f.name} s {s} {SAMPLING_NAME[samp]} {out} {rois}: differs from kb200_preprocess_rois"


def rotations(w, h):
    """(name, numpy transform of an (h, w, ...) array, forward map frame -> transformed array coordinates)."""
    return [("rot90", lambda a: np.rot90(a, 1), (0, 1, 0, -1, 0, w - 1)), ("rot180", lambda a: np.rot90(a, 2), (-1, 0, w - 1, 0, -1, h - 1)),
            ("rot270", lambda a: np.rot90(a, 3), (0, -1, h - 1, 1, 0, 0)), ("flip_x", lambda a: a[:, ::-1], (-1, 0, w - 1, 0, 1, 0)),
            ("flip_y", lambda a: a[::-1], (1, 0, 0, 0, -1, h - 1))]


def transformed_frame(f, raw, w, h, bpp, fn):
    """Frame `raw` (tight rows) with transform fn applied to each plane, and its new (w, h)."""
    if f.family in ("rgb", "gray"):
        a = raw[:w * h * bpp].reshape(h, w, bpp) if f.family == "rgb" else raw[:w * h].reshape(h, w)
        t = np.ascontiguousarray(fn(a))
        return t.reshape(-1), t.shape[1], t.shape[0]
    dt = np.dtype("<u2") if f.words else np.uint8
    planes = raw.view(dt)[:3 * w * h].reshape(3, h, w)
    t = np.ascontiguousarray(np.stack([fn(p) for p in planes]))
    return t.reshape(-1).view(np.uint8), t.shape[2], t.shape[1]


def test_rotation_maps_match_numpy():
    """The forward maps of rotations() move frame pixel (sx, sy) to where the numpy transform puts it."""
    w, h = 7, 5
    a = np.arange(w * h).reshape(h, w)
    for name, fn, m in rotations(w, h):
        t = fn(a)
        for oy in range(t.shape[0]):
            for ox in range(t.shape[1]):
                fwd = np.array([m[:3], m[3:], (0, 0, 1)], np.float64)
                sx, sy, _ = np.linalg.inv(fwd) @ (ox, oy, 1)
                assert t[oy, ox] == a[int(round(sy)), int(round(sx))], name


@pytest.mark.gpu
@pytest.mark.parametrize("code", (0, 1, 2, 11, 85, 86, 87, 88))
def test_rotation_twin(kb, lib, dev, code):
    """90, 180 and 270 degree rotations and both flips of RGB8 / BGR8 / Gray8 / I444 / I41x frames == the batch entry on the
    frame transformed on the host (Stretch to its own size), for Nearest and Bilinear and every output type."""
    f = FORMATS[code]
    w, h, bpp = 20, 12, 3
    c0 = make_case(f"rot-{f.name}", BASE + 0x5000 + code, code, 2 if yuv(f) else 0, bpp, w, h, row_bytes(f, w, bpp), w, h, BILINEAR, "imagenet", 9.0)
    raw = frame_bytes(c0, 0)
    dsrc = torch.from_numpy(raw).to(dev)
    for j, (name, fn, m) in enumerate(rotations(w, h)):
        t, tw, th = transformed_frame(f, raw, w, h, bpp, fn)
        dt = torch.from_numpy(np.ascontiguousarray(t)).to(dev)
        for samp in (NEAREST, BILINEAR):
            out = OUTS[(j + samp) % 3]
            c = make_case(c0.name, c0.seed, code, c0.matrix, bpp, w, h, c0.pitch, tw, th, samp, "imagenet", 9.0)
            got = torch.full((3 * tw * th * ESZ[out],), 0xFF, dtype=torch.uint8, device=dev)
            assert call(lib, c, [dsrc.data_ptr()], [raw.size], [(0, tuple(float(v) for v in m) + (0.0, 0.0, 1.0))], got.data_ptr(), 3 * tw * th,
                        out) == 0, kb._lib.last_error()
            ct = make_case(c0.name, c0.seed, code, c0.matrix, bpp, tw, th, row_bytes(f, tw, bpp), tw, th, samp, "imagenet", 9.0)
            want = torch.zeros_like(got)
            assert batch_entry(lib, ct, out, [dt.data_ptr()], want) == 0, kb._lib.last_error()
            torch.cuda.synchronize()
            assert torch.equal(got, want), f"{f.name} {name} {SAMPLING_NAME[samp]} {out}: differs from the batch entry on the transformed frame"


@pytest.mark.gpu
def test_graph_capture(kb, lib, dev):
    wc = CHUNKS[-2]   # 300 NV12 maps: five launches
    c = wc.base
    raws, src = load_frames(dev, wc.rcase)
    ptrs = [src.ptr + o for o in wc.offsets]
    n = len(wc.warps) * 3 * c.dw * c.dh
    eager = torch.empty(n, dtype=torch.float16, device=dev)
    replay = torch.zeros_like(eager)
    assert call(lib, c, ptrs, [c.need] * 3, wc.warps, eager.data_ptr(), n, "f16") == 0
    s = torch.cuda.Stream(dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            st = call(lib, c, ptrs, [c.need] * 3, wc.warps, replay.data_ptr(), n, "f16", stream=s.cuda_stream)
    assert st == 0, kb._lib.last_error()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.view(torch.int16), replay.view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ("Rgb8", "Bgra8", "Nv12", "Yuyv", "BayerGrbg12p", "P010", "I444"))
def test_python_run_warps(kb, lib, dev, fmt):
    """Preprocessor.run_warps == the C entry, with [M, 2, 3] and [M, 3, 3] tensors and nested sequences, for all three dtypes."""
    sf = kb.SourceFormat[fmt]
    w, h = 24, 18
    rng = np.random.default_rng(len(fmt))
    n = sf.buffer_len(w, h)
    frames = [torch.from_numpy(rng.integers(0, 256, n, dtype=np.int64).astype(np.uint8)).to(dev) for _ in range(2)]
    maps = [draw_map(rng, k, w, h, 12, 8) for k in ("similarity", "perspective", "affine", "rot90")]
    maps[1] = forward_of(np.linalg.inv(np.array(maps[1], np.float64).reshape(3, 3)))   # keep the perspective one at a normal scale
    index = [1, 0, 1, 0]
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        pre = (kb.Preprocessor.builder().source_format(sf).sampling(kb.InterpolationMode.Bilinear).normalize(kb.Normalize.imagenet()).build_cuda())
        desc = pre._desc(w, h, sf.pitch(w), sf.bpp(), sf.fmt_code(), 12, 8)
        want = torch.empty((4, 3, 8, 12), dtype=dtype, device=dev)
        ptrs = (C.c_void_p * 2)(*[f.data_ptr() for f in frames])
        st = lib.kb200_preprocess_warps(None, C.byref(desc), ptrs, (C.c_size_t * 2)(n, n), 2, warp_array(list(zip(index, maps))), 4, want.data_ptr(),
                                        want.numel(), (torch.float32, torch.float16, torch.bfloat16).index(dtype))
        assert st == 0, kb._lib.last_error()
        got = []
        for arg in (torch.tensor(maps, dtype=torch.float32).reshape(4, 3, 3), [np.array(m).reshape(3, 3).tolist() for m in maps]):
            dst = torch.empty_like(want)
            pre.run_warps(frames, w, h, torch.tensor(index), arg, dst)
            got.append(dst)
        affine = [0, 2, 3]   # the 2 x 3 form of the affine maps, with the perspective one run alone in its 3 x 3 form
        dst23 = torch.empty((3, 3, 8, 12), dtype=dtype, device=dev)
        pre.run_warps(frames, w, h, [index[i] for i in affine], torch.tensor([maps[i] for i in affine], dtype=torch.float32).reshape(3, 3, 3)[:, :2], dst23)
        torch.cuda.synchronize()
        for g in got:
            assert torch.equal(g.view(torch.uint8), want.view(torch.uint8)), (fmt, dtype)
        assert torch.equal(dst23.view(torch.uint8), want[affine].view(torch.uint8)), (fmt, dtype)


@pytest.mark.gpu
def test_cv2_anchor(kb, lib, dev):
    """Bilinear f32 output x 255 (unit normalisation) against cv2.warpAffine / warpPerspective (INTER_LINEAR,
    BORDER_CONSTANT) on smooth RGB8 frames, over the pixels whose sample lies at least one pixel inside the frame.
    cv2 rounds each coordinate to 1/32 px (error <= 1/64 per axis), weighs the taps in 15-bit fixed point and rounds to u8,
    so |ours - cv2| <= 0.5 + 2 * G / 64 + 4 * 255 / 2^15, G the frame's largest difference between neighbouring pixels."""
    cv2 = pytest.importorskip("cv2")
    w, h, dw, dh = 96, 64, 80, 56
    rng = np.random.default_rng(BASE + 0x6000)
    for t in range(12):
        img = smooth_rgb(w, h, BASE + t)
        g = max(np.abs(np.diff(img.astype(np.int32), axis=0)).max(), np.abs(np.diff(img.astype(np.int32), axis=1)).max())
        tol = 0.5 + 2 * g / 64 + 4 * 255 / 2 ** 15
        kind = ("similarity", "affine", "perspective")[t % 3]
        while True:   # a map with at least a fifth of its output on interior samples, and not the tiny-scale inverse (the |w| rule cv2 lacks)
            fwd = draw_map(rng, kind, w, h, dw, dh)
            inv, persp = inverse(lib, fwd)
            sx, sy, inside, _ = warp_coords(inv, persp, dw, dh, w, h)
            interior = inside & (sx >= 1) & (sx <= w - 2) & (sy >= 1) & (sy <= h - 2)
            if abs(fwd[8]) < 1e6 and interior.sum() > 0.2 * dw * dh:
                break
        c = make_case("cv2", 0, 0, 0, 3, w, h, 3 * w, dw, dh, BILINEAR, "unit", 0.0)
        src = torch.from_numpy(img.reshape(-1).copy()).to(dev)
        out = torch.empty((3, dh, dw), dtype=torch.float32, device=dev)
        assert call(lib, c, [src.data_ptr()], [src.numel()], [(0, fwd)], out.data_ptr(), out.numel(), "f32") == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        ours = out.cpu().numpy().transpose(1, 2, 0) * 255.0
        m = np.array(fwd, np.float64).reshape(3, 3)
        flags, border = cv2.INTER_LINEAR, cv2.BORDER_CONSTANT
        ref = (cv2.warpPerspective(img, m, (dw, dh), flags=flags, borderMode=border) if m[2, 0] or m[2, 1] or m[2, 2] != 1
               else cv2.warpAffine(img, m[:2], (dw, dh), flags=flags, borderMode=border)).astype(np.float64)
        err = np.abs(ours - ref)[interior]
        assert err.max() <= tol, f"{kind} map {fwd}: max |ours - cv2| {err.max():.3f} > {tol:.3f}"


# ── CPU: validation, symbols, run_warps argument rules, coverage ─────────────────────────────────────────────────────
FAKE = 0x7F0000000000   # never dereferenced: every call below is refused on the host
IDENT = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)


def _valid_case(code=3, sampling=BILINEAR):
    f = FORMATS[code]
    return make_case("valid", 1, code, 0, 3, 64, 48, row_bytes(f, 64, 3), 16, 16, sampling, "imagenet", 114.0)


@pytest.mark.parametrize("warp, status, rule", [
    ((2, IDENT), INVALID, "frame index 2 is outside [0, 2)"), ((-1, IDENT), INVALID, "frame index -1"),
    ((0, (float("nan"),) + IDENT[1:]), INVALID, "matrix entry 0 is not finite"), ((0, IDENT[:8] + (float("inf"),)), INVALID, "entry 8 is not finite"),
    ((0, (1.0, 2.0, 0.0, 2.0, 4.0, 0.0, 0.0, 0.0, 1.0)), SINGULAR, "affine map is singular"),
    ((0, (0.0,) * 6 + (0.0, 0.0, 1.0)), SINGULAR, "affine map is singular"),
    ((0, (1e-20, 0.0, 0.0, 0.0, 1e-20, 0.0, 0.0, 0.0, 1.0)), SINGULAR, "non-finite entry"),
    ((0, (1.0, 2.0, 3.0, 2.0, 4.0, 6.0, 1.0, 2.0, 3.0)), SINGULAR, "perspective map is singular"),
    ((0, (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 2.0)), 0, None)])   # a valid perspective map, refused later for the short dst
def test_invalid_region_is_refused_on_the_host(kb, warp, status, rule):
    lib = kb._lib.lib()
    c = _valid_case()
    st = call(lib, c, [FAKE, FAKE + 8192], [c.need] * 2, [(1, IDENT), warp], FAKE, 2 * 3 * 16 * 16 - 1, "f32")
    msg = kb._lib.last_error()
    if status == 0:
        assert st == SLICE, (st, msg)
    else:
        assert st == status and msg.startswith("region 1:") and rule in msg, (st, msg)


def test_invalid_call_is_refused_on_the_host(kb):
    from kornia_rs_b200._lib import PreprocessDesc
    lib = kb._lib.lib()
    c = _valid_case()
    w = [(0, IDENT)]
    ok = dict(ptrs=[FAKE, FAKE + 8192], lens=[c.need] * 2, warps=w, dst_ptr=FAKE, dst_len=3 * 16 * 16, out="f32")

    def go(case=c, **kw):
        a = dict(ok, **kw)
        return call(lib, case, a["ptrs"], a["lens"], a["warps"], a["dst_ptr"], a["dst_len"], a["out"])

    assert go(warps=[]) == INVALID and "n_warps" in kb._lib.last_error()
    assert go(case=_valid_case(sampling=LANCZOS)) == UNSUPPORTED and "Nearest or Bilinear" in kb._lib.last_error()
    d = c.desc(PreprocessDesc)
    assert lib.kb200_preprocess_warps(None, C.byref(d), (C.c_void_p * 1)(FAKE), None, 1, warp_array(w), 1, FAKE, 768, 3) == INVALID
    assert "output format" in kb._lib.last_error()
    assert lib.kb200_preprocess_warps(None, C.byref(d), None, None, 1, warp_array(w), 1, FAKE, 768, 0) == INVALID
    assert "'frames'" in kb._lib.last_error()
    assert lib.kb200_preprocess_warps(None, C.byref(d), (C.c_void_p * 1)(FAKE), None, 1, None, 1, FAKE, 768, 0) == INVALID
    assert "'warps'" in kb._lib.last_error()
    assert lib.kb200_preprocess_warps(None, C.byref(d), (C.c_void_p * 1)(FAKE), None, 1, warp_array(w), 1, None, 768, 0) == INVALID
    assert "'dst'" in kb._lib.last_error()
    assert lib.kb200_preprocess_warps(None, None, (C.c_void_p * 1)(FAKE), None, 1, warp_array(w), 1, FAKE, 768, 0) == INVALID
    assert go(dst_len=3 * 16 * 16 - 1) == SLICE and "'dst'" in kb._lib.last_error()
    assert go(lens=[c.need, c.need - 1]) == INVALID_SOURCE
    assert go(ptrs=[FAKE, 0]) == INVALID and "null frame pointer at index 1" in kb._lib.last_error()
    p010 = _valid_case(code=80)
    assert go(case=p010, ptrs=[FAKE, FAKE + 1], lens=[p010.need] * 2) == INVALID_SOURCE and "2-byte aligned" in kb._lib.last_error()
    # the descriptor's own rules still hold; its scale and pad are ignored
    from dataclasses import replace
    assert go(case=replace(c, w=63)) == INVALID_SOURCE   # odd NV12 width
    d = c.desc(PreprocessDesc)
    d.scale_x, d.pad_y = -1.0, float("nan")
    assert lib.kb200_preprocess_warps(None, C.byref(d), (C.c_void_p * 2)(FAKE, FAKE), None, 2, warp_array(w), 1, FAKE, 10, 0) == SLICE
    # the status of every refusal comes before anything is enqueued: a singular map after a short frame is still the map
    assert go(warps=[(0, IDENT), (1, (0.0,) * 9)], lens=[1, 1]) == SINGULAR


def test_header_and_binding_symbols(kb):
    import __graft_entry__ as ge
    from kornia_rs_b200._lib import WarpRoi
    assert "kb200_preprocess_warps" in ge.declared_symbols()
    assert C.sizeof(WarpRoi) == 40 and WarpRoi.m.offset == 4
    hdr = open(os.path.join(ROOT, "include", "kornia_b200.h")).read()
    assert re.search(r"typedef struct kb200_warp_roi \{\s*int32_t frame;\s*float m\[9\];\s*\} kb200_warp_roi;", hdr)
    rs = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    assert "pub struct kb200_warp_roi" in rs and "pub fn kb200_preprocess_warps(" in rs and "pub fn launch_preprocess_warps(" in rs
    assert kb._lib.lib().kb200_preprocess_warps.restype is C.c_int


def test_run_warps_argument_rules(kb):
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).build_cuda()
    frame = torch.zeros(64 * 48 * 3 // 2, dtype=torch.uint8)
    dst = torch.zeros((1, 3, 8, 8))
    eye = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]
    nan = [[float("nan"), 0.0, 0.0], [0.0, 1.0, 0.0]]
    for index, maps, region in (([0], torch.zeros((1, 2, 2)), None), ([0], torch.zeros((1, 6)), None), ([0], torch.zeros((1, 4, 3)), None),
                                (torch.zeros((1,), dtype=torch.float32), [eye], None), (torch.zeros((1, 1), dtype=torch.int64), [eye], None),
                                ([0.0], [eye], None), ([], [], None), ([0, 0], [eye], None), ([1], [eye], 0), ([0, -1], [eye, eye], 1),
                                ([0, 0], [eye, [[1.0, 0.0], [0.0, 1.0]]], 1), ([0, 0], [eye, [[1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 0, 0]]], 1),
                                ([0, 0], [eye, "abc"], 1), ([0, 0], [eye, nan], 1),
                                ([0], torch.tensor([[[1.0, 0.0, 0.0], [0.0, float("inf"), 0.0]]]), 0)):
        with pytest.raises(kb.PreprocessError) as e:
            pre.run_warps([frame], 64, 48, index, maps, dst)
        assert e.value.kind == "InvalidWarp", (index, maps)
        assert e.value.fields.get("region") == region, (index, maps, e.value.fields)
    lanczos = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).sampling(kb.InterpolationMode.Lanczos).build_cuda()
    with pytest.raises(kb.PreprocessError) as e:
        lanczos.run_warps([frame], 64, 48, [0], [eye], dst)
    assert e.value.kind == "UnsupportedSampling"
    with pytest.raises(kb.PreprocessError) as e:   # two maps, three outputs
        pre.run_warps([frame], 64, 48, [0, 0], [eye, eye], torch.zeros((3, 3, 8, 8)))
    assert e.value.kind == "BatchMismatch"
    with pytest.raises(kb.PreprocessError) as e:
        pre.run_warps([frame], 64, 48, [0], [eye], torch.zeros((1, 3, 8, 8), dtype=torch.float64))
    assert e.value.kind == "BadOutputShape"
    with pytest.raises(kb.PreprocessError) as e:   # a CPU destination is refused before the frames are looked at
        pre.run_warps([frame], 64, 48, [0], [eye], dst)
    assert e.value.kind == "NotDeviceTensor"


def test_sweep_coverage(kb):
    """Every format, both map kinds, both store paths, |w| < 1e-10 pads, off-frame pads, and samples that land exactly on 0,
    W - 1, the float below W and W."""
    lib = kb._lib.lib()
    cases = [wcase(i) for i in range(N_SWEEP)] + CHUNKS
    formats, kernels, persp_kinds, outs, samplers = set(), set(), set(), set(), set()
    wzero = offframe = 0
    landed = set()
    nmax = 0
    for wc in cases:
        c = wc.base
        formats.add(c.code)
        kernels.add((c.code, wc.kernel()))
        kernels.add((c.code, wc.kernel(ESZ[wc.out])))
        assert wc.kernel(ESZ[wc.out]) == GENERIC
        outs.add(wc.out)
        samplers.add(c.sampling)
        nmax = max(nmax, len(wc.warps))
        for k, fwd in wc.warps:
            inv, persp = inverse(lib, fwd)
            persp_kinds.add(persp)
            sx, sy, inside, small = warp_coords(inv, persp, c.dw, c.dh, c.w, c.h)
            wzero += int(small.any())
            offframe += int((~inside & ~small).any())
            for axis, s, n in (("x", sx, c.w), ("y", sy, c.h)):
                for name, v in (("0", F32(0)), ("W-1", F32(n - 1)), ("below W", np.nextafter(F32(n), F32(0))), ("W", F32(n))):
                    if (s == v).any():
                        landed.add((axis, name))
    assert formats == set(CODES)
    for code in CODES:
        assert (code, VECTOR) in kernels and (code, GENERIC) in kernels, FORMATS[code].name
    assert persp_kinds == {False, True} and outs == set(OUTS) and samplers == {NEAREST, BILINEAR}
    assert wzero > 20 and offframe > 100, (wzero, offframe)
    assert landed == {(a, n) for a in "xy" for n in ("0", "W-1", "below W", "W")}, landed
    assert nmax > CHUNK
    assert any(len({k for k, _ in wc.warps}) > 1 and [k for k, _ in wc.warps] != sorted(k for k, _ in wc.warps) for wc in cases)
    assert {o % 2 for wc in cases for o in wc.offsets} == {0, 1}   # frames at odd and even addresses
    assert any(wc.base.pitch > row_bytes(wc.base.fmt, wc.base.w, wc.base.bpp) for wc in cases)   # pitch padding
