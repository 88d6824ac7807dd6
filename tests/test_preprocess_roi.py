"""Camera preprocess: kb200_preprocess_rois, many regions of interest of a set of frames in one call, for every source format.

Region i = (k, x, y, w, h) must give:
  * for the whole frame (k, 0, 0, W, H), the bytes the batch entry gives frame k (test_whole_frame);
  * for any region, the bytes of the sweep's references (test_preprocess_sweep.reference's restatements: the oracle on the
    decoded RGB8 picture, or restate.preprocess_rgb16 on the decoded 16-bit picture) run on the w x h crop at (x, y)
    of frame k's decoded picture with kb200_preprocess_affine(mode, w, h, dst_w, dst_h) (test_sweep, `rcase(i)` a pure
    function of i); Lanczos within the sweep's tolerance.

Every sweep case that does not sample with Lanczos runs a second time into a destination one element past a 16-byte
boundary, which refuses the fast region kernels: the generic region kernel must give the same bits.  Destinations sit in
harness.Guarded with a 0xFF prefill; frames sit in one buffer with random bytes in their pitch padding, between them
and around them.  The CPU tests cover the host validation (no region outside its frame ever reaches a device), the
dispatch rule's coverage and run_rois' argument rules.
"""
import ctypes as C
from dataclasses import dataclass, replace

import numpy as np
import pytest
import torch

from harness import Guarded, compare_region, dev, lib, load_frames, roi_array
from restate import BILINEAR, CODES, Case, ESZ, FORMATS, LANCZOS, NEAREST, NORMS, OUTS, RCase, SAMPLING_NAME, pad_step, picture, place, region_reference, row_bytes, size_rule, src_bytes, yuv


BASE = 0x2011F000
CHUNK = 80   # regions per launch (preprocess_roi.cu ROI_CHUNK)
GENERIC = "preprocess_roi_generic_kernel"
INVALID, SLICE, INVALID_SOURCE = -1, -2, -8
F32 = np.float32


# ── the dispatch rule, restated (preprocess_roi.cu launch_rois) ──────────────────────────────────────────────────────
def fast_roi(f):
    return f.fast.replace("_kernel", "_roi_kernel") if f.fast else None


def expected_kernel(f, sampling, dw, dh, dst, frames):
    pair = f.family == "yuv420" and not f.words and f.layout in ("Nv12", "Nv21")
    if (sampling != LANCZOS and f.fast and dw % 4 == 0 and dst % 16 == 0 and dh <= 65535 * 8
            and (not pair or all(p % 2 == 0 for p in frames))):
        return fast_roi(f)
    return GENERIC


def roi_kernel(rc, dst=0):
    return expected_kernel(rc.base.fmt, rc.base.sampling, rc.base.dw, rc.base.dh, dst, rc.offsets)


def draw_rois(rng, w, h, n_frames, n):
    """n regions: the whole frame, 1x1, one row, one column, regions on every edge, odd origins, random ones, with
    repeated and out-of-order frame indices."""
    special = [(0, 0, w, h), (int(rng.integers(0, w)), int(rng.integers(0, h)), 1, 1), (0, int(rng.integers(0, h)), w, 1),
               (int(rng.integers(0, w)), 0, 1, h), (w - 1, h - 1, 1, 1), (0, h - 1, w, 1), (w - 1, 0, 1, h)]
    out = []
    for i in range(n):
        k = int(rng.integers(0, n_frames))
        if i < len(special) and rng.random() < 0.7:
            x, y, rw, rh = special[i]
        else:
            rw, rh = int(rng.integers(1, w + 1)), int(rng.integers(1, h + 1))
            x, y = int(rng.integers(0, w - rw + 1)), int(rng.integers(0, h - rh + 1))
            if rng.random() < 0.3 and x + rw < w:
                x |= 1
            if rng.random() < 0.3 and y + rh < h:
                y |= 1
        out.append((k, x, y, rw, rh))
    return tuple(out)


def rcase(i):
    """Case i of the sweep: a pure function of i.  Format i % 51; the first pass over the formats samples without Lanczos
    into a width the fast region kernels take, from even frame addresses."""
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
    sampling = int(rng.choice([NEAREST, BILINEAR]) if first else rng.choice([NEAREST, BILINEAR, LANCZOS], p=[0.3, 0.3, 0.4]))
    n_frames = int(rng.integers(1, 4))
    n = int(rng.choice([int(rng.integers(1, 8)), int(rng.integers(1, 41))]))
    base = Case(f"roi-{i}", BASE + i, f.code, (i % len(CODES) + 2 * (i // len(CODES))) % 4 if yuv(f) else 0, bpp, w, h, pitch, "roi", 1.0, 1.0, 0.0, 0.0, dw, dh,
                sampling, False, "table", n_frames, (), None, 0, str(rng.choice(list(NORMS))), float(rng.integers(0, 256)))
    offs = place(rng, f, src_bytes(f, w, h, pitch), n_frames, odd=not first and rng.random() < 0.3)
    return RCase(base, int(rng.integers(0, 2)), str(rng.choice(OUTS)), n_frames, offs, draw_rois(rng, w, h, n_frames, n))


N_SWEEP = 2 * len(CODES)


def chunk_cases():
    """n_rois around the launch chunk, with mixed frame indices: NV12 on its fast kernel, Bayer on the generic one."""
    out = []
    for j, n in enumerate((1, CHUNK - 1, CHUNK, CHUNK + 1, 300)):
        for code in (3, 17):
            rng = np.random.default_rng(BASE + 0x1000 + 16 * j + code)
            f = FORMATS[code]
            w, h = 24, 16
            base = Case(f"chunk-{n}-{f.name}", BASE + 0x1000 + n, code, 1 if code == 3 else 0, 1, w, h, row_bytes(f, w, 1), "roi", 1.0, 1.0,
                        0.0, 0.0, 8, 6, BILINEAR, False, "table", 3, (), None, 0, "imagenet", 114.0)
            rois = tuple((int(rng.integers(0, 3)),) + r[1:] for r in draw_rois(rng, w, h, 3, n))
            out.append(RCase(base, j % 2, OUTS[j % 3], 3, place(rng, f, src_bytes(f, w, h, base.pitch), 3), rois))
    return out


CHUNKS = chunk_cases()


def call(lib, c, mode, ptrs, lens, rois, dst_ptr, dst_len, out, stream=None):
    from kornia_rs_b200._lib import PreprocessDesc
    d = c.desc(PreprocessDesc)
    n = len(ptrs)
    return lib.kb200_preprocess_rois(stream, C.byref(d), mode, (C.c_void_p * max(1, n))(*ptrs), (C.c_size_t * max(1, n))(*lens), n,
                                     roi_array(rois), len(rois), dst_ptr, dst_len, OUTS.index(out))


def run_rcase(kb, lib, dev, rc):
    c = rc.base
    raws, src = load_frames(dev, rc)
    ptrs = [src.ptr + o for o in rc.offsets]
    lens = [c.need] * rc.n_frames
    m = len(rc.rois)
    elems = 3 * c.dw * c.dh
    nbytes = m * elems * ESZ[rc.out]
    outs = []
    for off in (0,) + ((ESZ[rc.out],) if c.sampling != LANCZOS else ()):
        dst = Guarded(dev, nbytes, min(nbytes, 1 << 16), off).fill(0xFF)
        st = call(lib, c, rc.mode, ptrs, lens, rc.rois, dst.ptr, m * elems, rc.out)
        assert st == 0, f"{rc}: status {st}: {kb._lib.last_error()}"
        ran = kb._lib.last_kernel()
        torch.cuda.synchronize()
        want = expected_kernel(c.fmt, c.sampling, c.dw, c.dh, dst.ptr, ptrs)
        assert ran == want == (roi_kernel(rc, off) if off else ran), f"{rc}: dst +{off} B ran {ran}, the dispatch mirror says {want}"
        for what, g in zip(("lead", "tail"), dst.guards()):
            assert (g == 0xFF).all(), f"{rc}: dst +{off} B: bytes written in the {what} guard"
        outs.append(dst.out())
    esz = ESZ[rc.out]
    ones = outs[0].view(np.uint16 if esz == 2 else np.uint32) == (0xFFFF if esz == 2 else 0xFFFFFFFF)
    assert not ones.any(), f"{rc}: {int(ones.sum())} output elements left unwritten"
    pics = {}
    fb = elems * esz
    for i, roi in enumerate(rc.rois):
        if roi[0] not in pics:
            pics[roi[0]] = picture(c, raws[roi[0]])
        compare_region(outs[0][i * fb:(i + 1) * fb], region_reference(rc, pics[roi[0]], roi), rc, f"{rc}: region {i} {roi}")
    if len(outs) == 2:
        bad = np.flatnonzero(outs[0] != outs[1])
        assert bad.size == 0, f"{rc}: {roi_kernel(rc)} and {GENERIC} differ in {bad.size} bytes"


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_SWEEP))
def test_sweep(kb, lib, dev, i):
    run_rcase(kb, lib, dev, rcase(i))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.base.name for c in CHUNKS])
def test_chunking(kb, lib, dev, name):
    run_rcase(kb, lib, dev, next(c for c in CHUNKS if c.base.name == name))


@pytest.mark.gpu
@pytest.mark.parametrize("code", CODES)
def test_whole_frame(kb, lib, dev, code):
    """Region (k, 0, 0, W, H) == the batch entry on frame k, for every sampler, mode and output type."""
    from kornia_rs_b200._lib import PreprocessDesc
    f = FORMATS[code]
    mw, mh, sw, sh = size_rule(f)
    w, h = max(mw, 20 // sw * sw), max(mh, 12 // sh * sh)
    for j, (samp, mode, out) in enumerate([(s, m, o) for s in (NEAREST, BILINEAR, LANCZOS) for m in (0, 1) for o in OUTS]):
        dw, dh = (16, 10) if j % 2 else (13, 9)
        c = Case(f"whole-{f.name}", BASE + 0x3000 + code, code, j % 4 if yuv(f) else 0, 3, w, h, row_bytes(f, w, 3), "roi", 1.0, 1.0, 0.0, 0.0,
                 dw, dh, samp, False, "table", 2, (), None, 0, "imagenet", 114.0)
        rc = RCase(c, mode, out, 2, (16, 16 + -(-c.need // 16) * 16), ((1, 0, 0, w, h), (0, 0, 0, w, h)))
        raws, src = load_frames(dev, rc)
        ptrs = [src.ptr + o for o in rc.offsets]
        got = torch.full((2 * 3 * dw * dh * ESZ[out],), 0xFF, dtype=torch.uint8, device=dev)
        assert call(lib, c, mode, ptrs, [c.need] * 2, rc.rois, got.data_ptr(), 2 * 3 * dw * dh, out) == 0, kb._lib.last_error()
        d = c.desc(PreprocessDesc)
        a = (C.c_float * 4)()
        lib.kb200_preprocess_affine(mode, w, h, dw, dh, a)
        d.scale_x, d.scale_y, d.pad_x, d.pad_y = a
        want = torch.full_like(got, 0)
        fn = getattr(lib, f"kb200_preprocess_{out}")
        assert fn(None, C.byref(d), (C.c_void_p * 2)(ptrs[1], ptrs[0]), (C.c_size_t * 2)(c.need, c.need), 2, want.data_ptr(), 2 * 3 * dw * dh) == 0
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"{f.name} {SAMPLING_NAME[samp]} mode {mode} {out}: whole-frame region differs from the batch entry"


@pytest.mark.gpu
@pytest.mark.parametrize("code", (0, 1, 2))
def test_interleaved_subrect_matches_pitched_view(kb, lib, dev, code):
    """RGB / BGR / Gray: a region == the batch entry on a view of the frame at the region's first byte, with its pitch."""
    from kornia_rs_b200._lib import PreprocessDesc
    f = FORMATS[code]
    w, h, bpp = 37, 23, 3 if code != 2 else 1
    c = Case(f"view-{f.name}", BASE + 0x4000 + code, code, 0, 3, w, h, row_bytes(f, w, 3) + 5, "roi", 1.0, 1.0, 0.0, 0.0, 20, 12, BILINEAR,
             False, "table", 1, (), None, 0, "imagenet", 114.0)
    rc = RCase(c, 0, "f32", 1, (16,), ())
    raws, src = load_frames(dev, rc)
    rng = np.random.default_rng(code)
    for samp in (NEAREST, BILINEAR, LANCZOS):
        for mode in (0, 1):
            rw, rh = int(rng.integers(1, w)), int(rng.integers(1, h))
            x, y = int(rng.integers(0, w - rw + 1)), int(rng.integers(0, h - rh + 1))
            cs = replace(c, sampling=samp)
            got = torch.empty((3 * 12 * 20,), dtype=torch.float32, device=dev)
            assert call(lib, cs, mode, [src.ptr + 16], [c.need], [(0, x, y, rw, rh)], got.data_ptr(), got.numel(), "f32") == 0
            d = replace(cs, w=rw, h=rh).desc(PreprocessDesc)
            a = (C.c_float * 4)()
            lib.kb200_preprocess_affine(mode, rw, rh, 20, 12, a)
            d.scale_x, d.scale_y, d.pad_x, d.pad_y = a
            d.src_bpp = 3 if code != 2 else 1
            want = torch.empty_like(got)
            first = src.ptr + 16 + y * c.pitch + x * (d.src_bpp if code != 2 else 1)
            assert lib.kb200_preprocess_f32(None, C.byref(d), (C.c_void_p * 1)(first), None, 1, want.data_ptr(), want.numel()) == 0
            torch.cuda.synchronize()
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), f"{f.name} ({x}, {y}, {rw}, {rh}) {SAMPLING_NAME[samp]} mode {mode}"


@pytest.mark.gpu
def test_graph_capture(kb, lib, dev):
    rc = CHUNKS[-2]   # 300 NV12 regions: four launches
    c = rc.base
    raws, src = load_frames(dev, rc)
    ptrs = [src.ptr + o for o in rc.offsets]
    n = len(rc.rois) * 3 * c.dw * c.dh
    eager = torch.empty(n, dtype=torch.float16, device=dev)
    replay = torch.zeros_like(eager)
    assert call(lib, c, rc.mode, ptrs, [c.need] * 3, rc.rois, eager.data_ptr(), n, "f16") == 0
    s = torch.cuda.Stream(dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            st = call(lib, c, rc.mode, ptrs, [c.need] * 3, rc.rois, replay.data_ptr(), n, "f16", stream=s.cuda_stream)
    assert st == 0, kb._lib.last_error()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.view(torch.int16), replay.view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ("Rgb8", "Bgra8", "Nv12", "Yuyv", "BayerGrbg12p", "P010", "I444"))
def test_python_run_rois(kb, lib, dev, fmt):
    """Preprocessor.run_rois == the C entry, for one format of each family and all three dtypes."""
    sf = kb.SourceFormat[fmt]
    w, h = 24, 18
    rng = np.random.default_rng(len(fmt))
    n = sf.buffer_len(w, h)
    frames = [torch.from_numpy(rng.integers(0, 256, n, dtype=np.int64).astype(np.uint8)).to(dev) for _ in range(2)]
    if sf.is_bayer16() or sf.is_yuv16() or (sf.is_yuv444() and sf.bit_depth() > 8):
        frames = [f.view(torch.int16).view(torch.uint8) for f in frames]
    rois = [(1, 3, 5, 11, 7), (0, 0, 0, w, h), (1, 23, 17, 1, 1)]
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        pre = (kb.Preprocessor.builder().source_format(sf).mode(kb.ResizeMode.Stretch).sampling(kb.InterpolationMode.Bilinear)
               .normalize(kb.Normalize.imagenet()).build_cuda())
        dst = torch.empty((3, 3, 8, 12), dtype=dtype, device=dev)
        pre.run_rois(frames, w, h, torch.tensor(rois, dtype=torch.int64), dst)
        dst2 = torch.empty_like(dst)
        pre.run_rois(frames, w, h, rois, dst2)
        desc = pre._desc(w, h, sf.pitch(w), sf.bpp(), sf.fmt_code(), 12, 8)
        want = torch.empty_like(dst)
        ptrs = (C.c_void_p * 2)(*[f.data_ptr() for f in frames])
        lens = (C.c_size_t * 2)(n, n)
        st = lib.kb200_preprocess_rois(None, C.byref(desc), 1, ptrs, lens, 2, roi_array(rois), 3, want.data_ptr(), want.numel(),
                                       (torch.float32, torch.float16, torch.bfloat16).index(dtype))
        assert st == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        assert torch.equal(dst.view(torch.uint8), want.view(torch.uint8)) and torch.equal(dst2.view(torch.uint8), want.view(torch.uint8)), (fmt, dtype)


# ── CPU: validation, dispatch coverage, Python argument rules ──────────────────────────────────────────────────────────
def _valid_case(code=3):
    f = FORMATS[code]
    return Case("valid", 1, code, 0, 3, 64, 48, row_bytes(f, 64, 3), "roi", 1.0, 1.0, 0.0, 0.0, 16, 16, BILINEAR, False, "table", 2, (), None, 0,
                "imagenet", 114.0)


FAKE = 0x7F0000000000   # never dereferenced: every call below is refused on the host


@pytest.mark.parametrize("roi, rule", [((2, 0, 0, 8, 8), "frame index"), ((-1, 0, 0, 8, 8), "frame index"), ((0, -1, 0, 8, 8), "negative"),
                                       ((0, 0, -3, 8, 8), "negative"), ((0, 0, 0, 0, 8), "empty"), ((0, 0, 0, 8, 0), "empty"),
                                       ((0, 0, 0, -5, 8), "empty"), ((0, 57, 0, 8, 8), "outside"), ((0, 0, 41, 8, 8), "outside"),
                                       ((0, 2 ** 31 - 1, 0, 1, 1), "outside"), ((0, 2 ** 31 - 8, 0, 16, 1), "outside"),
                                       ((0, 0, 2 ** 31 - 2, 1, 2 ** 31 - 1), "outside")])
def test_invalid_region_is_refused_on_the_host(kb, roi, rule):
    lib = kb._lib.lib()
    c = _valid_case()
    good = (1, 0, 0, 64, 48)
    st = call(lib, c, 0, [FAKE, FAKE + 8192], [c.need] * 2, [good, roi], FAKE, 2 * 3 * 16 * 16, "f32")
    msg = kb._lib.last_error()
    assert st == INVALID and msg.startswith("region 1:") and rule in msg, (st, msg)


def test_invalid_call_is_refused_on_the_host(kb):
    from kornia_rs_b200._lib import PreprocessDesc
    lib = kb._lib.lib()
    c = _valid_case()
    r = [(0, 1, 1, 9, 9)]
    ok = dict(mode=0, ptrs=[FAKE, FAKE + 8192], lens=[c.need] * 2, rois=r, dst_ptr=FAKE, dst_len=3 * 16 * 16, out="f32")

    def go(**kw):
        a = dict(ok, **kw)
        return call(lib, c, a["mode"], a["ptrs"], a["lens"], a["rois"], a["dst_ptr"], a["dst_len"], a["out"])

    assert go(rois=[]) == INVALID and "n_rois" in kb._lib.last_error()
    assert go(mode=2) == INVALID and "mode" in kb._lib.last_error()
    assert go(mode=-1) == INVALID
    d = c.desc(PreprocessDesc)
    assert lib.kb200_preprocess_rois(None, C.byref(d), 0, (C.c_void_p * 1)(FAKE), None, 1, roi_array(r), 1, FAKE, 768, 3) == INVALID
    assert "output format" in kb._lib.last_error()
    assert lib.kb200_preprocess_rois(None, C.byref(d), 0, None, None, 1, roi_array(r), 1, FAKE, 768, 0) == INVALID
    assert lib.kb200_preprocess_rois(None, C.byref(d), 0, (C.c_void_p * 1)(FAKE), None, 1, None, 1, FAKE, 768, 0) == INVALID
    assert lib.kb200_preprocess_rois(None, None, 0, (C.c_void_p * 1)(FAKE), None, 1, roi_array(r), 1, FAKE, 768, 0) == INVALID
    assert go(dst_len=3 * 16 * 16 - 1) == SLICE
    assert go(lens=[c.need, c.need - 1]) == INVALID_SOURCE
    assert go(ptrs=[FAKE, 0]) == INVALID
    # the descriptor's own rules still hold; its scale and pad are ignored
    bad = replace(c, w=63)   # odd NV12 width
    assert call(lib, bad, 0, ok["ptrs"], ok["lens"], r, FAKE, 768, "f32") == INVALID_SOURCE
    d = c.desc(PreprocessDesc)
    d.scale_x, d.pad_y = -1.0, float("nan")
    assert lib.kb200_preprocess_rois(None, C.byref(d), 0, (C.c_void_p * 2)(FAKE, FAKE), None, 2, roi_array([(0, 0, 0, 1, 1)]), 1, None, 48, 0) == INVALID
    assert "dst" in kb._lib.last_error()   # got past the descriptor: scale and pad were not checked


def test_dispatch_coverage():
    cases = [rcase(i) for i in range(N_SWEEP)] + CHUNKS
    kernels = {code: set() for code in CODES}
    samplers, modes, dw4, outs, matrices, nmax = set(), set(), set(), set(), {}, 0
    for rc in cases:
        c = rc.base
        kernels[c.code].add(roi_kernel(rc))
        kernels[c.code].add(roi_kernel(rc, ESZ[rc.out]))
        assert roi_kernel(rc, ESZ[rc.out]) == GENERIC
        samplers.add(c.sampling)
        modes.add(rc.mode)
        dw4.add(c.dw % 4)
        outs.add(rc.out)
        if yuv(c.fmt):
            matrices.setdefault(c.fmt.family, set()).add(c.matrix)
        nmax = max(nmax, len(rc.rois))
        assert all(0 <= k < rc.n_frames and x >= 0 and y >= 0 and w >= 1 and h >= 1 and x + w <= c.w and y + h <= c.h for k, x, y, w, h in rc.rois)
    for code, f in FORMATS.items():
        assert GENERIC in kernels[code], f.name
        if f.fast:
            assert fast_roi(f) in kernels[code], f.name
    assert samplers == {NEAREST, BILINEAR, LANCZOS} and modes == {0, 1} and dw4 == {0, 1, 2, 3} and outs == set(OUTS)
    assert all(m == {0, 1, 2, 3} for m in matrices.values()) and set(matrices) == {"yuv420", "yuv422", "yuv444"}, matrices
    assert nmax > CHUNK


def test_run_rois_argument_rules(kb):
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).build_cuda()
    frame = torch.zeros(64 * 48 * 3 // 2, dtype=torch.uint8)
    dst = torch.zeros((1, 3, 8, 8))
    for rois in (torch.zeros((1, 4), dtype=torch.int64), torch.zeros((1, 5), dtype=torch.float32), torch.zeros(5, dtype=torch.int32), [(0, 0, 0, 8)],
                 [(0, 0, 0, 8, 8.0)], [], [(0, 2 ** 31, 0, 1, 1)], [(1, 0, 0, 8, 8)], [(-1, 0, 0, 8, 8)], [(0, -2, 0, 8, 8)],
                 [(0, 0, 0, 0, 8)], [(0, 57, 0, 8, 8)], [(0, 0, 41, 8, 8)], [(0, 0, 0, 8, 8), (0, 63, 47, 2, 1)]):
        with pytest.raises(kb.PreprocessError) as e:
            pre.run_rois([frame], 64, 48, rois, dst)
        assert e.value.kind == "InvalidRoi", rois
    with pytest.raises(kb.PreprocessError) as e:   # two regions, three outputs
        pre.run_rois([frame], 64, 48, [(0, 0, 0, 8, 8)] * 2, torch.zeros((3, 3, 8, 8)))
    assert e.value.kind == "BatchMismatch"
    with pytest.raises(kb.PreprocessError) as e:
        pre.run_rois([frame], 64, 48, [(0, 0, 0, 8, 8)], torch.zeros((1, 3, 8, 8), dtype=torch.float64))
    assert e.value.kind == "BadOutputShape"
    with pytest.raises(kb.PreprocessError) as e:
        pre.run_rois([frame], 64, 48, [(0, 0, 0, 8, 8)], torch.zeros((1, 1, 8, 8)))
    assert e.value.kind == "BadOutputShape"
    with pytest.raises(kb.PreprocessError) as e:   # a CPU destination is refused before the frames are looked at
        pre.run_rois([frame], 64, 48, [(0, 0, 0, 8, 8)], dst)
    assert e.value.kind == "NotDeviceTensor"
