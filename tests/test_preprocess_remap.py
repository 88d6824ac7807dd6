"""Camera preprocess: kb200_preprocess_remap, a set of frames resampled through dense per-pixel coordinate maps, for every
source format, and kb200_generate_correction_map_polynomial_to, the undistortion map for an output camera of its own.

The reference (`remap_reference`) is test_preprocess_warp.warp_reference's numpy float32 sampler and normalisation, fed
with the map's coordinates and remap's inside rule (0 <= x < src_w, 0 <= y < src_h in f32; NaN is outside) in place of
warp_coords.

On the GPU:
  * twins, bit for bit: an identity map of a whole frame against the batch entry (every format, sampler and output type);
    the float32 coordinates warp_coords gives an affine or perspective map (NaN where it finds a pixel outside) against
    kb200_preprocess_warps on that map;
  * a seeded sweep (`mcase(i)`, a pure function of i, every format twice) of undistortion maps from the device generator
    (both entries), random smooth maps, per-pixel noise (NaN, +-inf, -0.0, 1e30, samples on 0, W - 1, the float below W
    and W) and constant maps against the reference, each run into a harness.Guarded destination with a 0xFF
    prefill, on the kernel a host mirror of the dispatch rule names, and again with dst and with the maps one element past
    a 16-byte boundary, where the generic kernel must give the same bytes;
  * several maps and an arbitrary (frame, map) table against one shared-map call per map, at region counts around the
    launch chunk; a captured graph; Preprocessor.run_remap with [H, W], [K, H, W] and Image maps;
  * the map generator: `_to` with new_intrinsic == intrinsic gives the existing entry's bits, and any other new_intrinsic a
    numpy float64 restatement of its expression, bit for bit (the library builds with -fmad=false);
  * an independent anchor: cv2.remap (INTER_LINEAR, BORDER_CONSTANT) on smooth RGB8 frames.
On the CPU: every host refusal, the header and binding symbols, run_remap's argument rules and what the sweep covers.
"""
import ctypes as C
import os
import re
from dataclasses import dataclass
from unittest import mock

import numpy as np
import pytest
import torch

from harness import Guarded, batch_entry, compare_region, dev, inverse, lib, load_frames, warp_array
from restate import BILINEAR, CODES, ESZ, FORMATS, LANCZOS, NEAREST, NORMS, OUTS, RCase, SAMPLING_NAME, draw_map, make_case, pad_step, picture, place, remap_reference, row_bytes, size_rule, smooth_rgb, src_bytes, warp_coords, yuv


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = 0x5E3A0000
CHUNK = 192   # regions per launch (preprocess_remap.cu REMAP_CHUNK)
VECTOR, GENERIC = "preprocess_remap_kernel", "preprocess_remap_generic_kernel"
INVALID, SLICE, UNSUPPORTED, INVALID_SOURCE = -1, -2, -4, -8
F32 = np.float32
KINDS = ("undistort", "undistort_to", "smooth", "noise", "constant")


# ── the dispatch rule, restated (preprocess_remap.cu remap_vector_ok) ────────────────────────────────────────────────
def expected_kernel(dw, out, dst, map_x, map_y):
    ok = dw % 4 == 0 and map_x % 16 == 0 and map_y % 16 == 0 and dst % (16 if out == "f32" else 8) == 0
    return VECTOR if ok else GENERIC


def distort_map(intr, dist, new, dw, dh):
    """distortion.cu correction_map_kernel restated in numpy float64, one rounding per operation in the kernel's order."""
    fx, fy, cx, cy = (np.float64(v) for v in intr)
    k1, k2, k3, k4, k5, k6, p1, p2 = (np.float64(v) for v in dist)
    nfx, nfy, ncx, ncy = (np.float64(v) for v in new)
    px = np.arange(dw, dtype=np.float64)[None, :]
    py = np.arange(dh, dtype=np.float64)[:, None]
    x = np.broadcast_to((px - ncx) / nfx, (dh, dw))
    y = np.broadcast_to((py - ncy) / nfy, (dh, dw))
    r2 = x * x + y * y
    r4 = r2 * r2
    r6 = r4 * r2
    kr = (((1.0 + k1 * r2) + k2 * r4) + k3 * r6) / (((1.0 + k4 * r2) + k5 * r4) + k6 * r6)
    x_2, y_2 = 2.0 * x, 2.0 * y
    xy_2 = x_2 * y
    xd = (x * kr + xy_2 * p1) + p2 * (r2 + x_2 * x)
    yd = (y * kr + p1 * (r2 + y_2 * y)) + xy_2 * p2
    return (fx * xd + cx).astype(F32), (fy * yd + cy).astype(F32)


def draw_camera(rng, w, h):
    """A camera for a w x h frame: (intrinsic, distortion) with barrel or pincushion distortion."""
    f = float(rng.uniform(0.6, 1.4)) * max(w, h)
    intr = (f * float(rng.uniform(0.9, 1.1)), f, w / 2 + float(rng.uniform(-2, 2)), h / 2 + float(rng.uniform(-2, 2)))
    dist = (float(rng.uniform(-0.4, 0.3)), float(rng.uniform(-0.1, 0.1)), float(rng.uniform(-0.02, 0.02)), float(rng.uniform(0, 0.05)),
            0.0, 0.0, float(rng.uniform(-0.01, 0.01)), float(rng.uniform(-0.01, 0.01)))
    return intr, dist


def edge_values(n):
    return [0.0, n - 1.0, float(np.nextafter(F32(n), F32(0))), float(n)]


def draw_map_pair(rng, kind, w, h, dw, dh):
    """One map of `kind` for a w x h frame and a dw x dh output: (map_x, map_y) float32 [dh, dw], or ("device", args) for
    the generator kinds, which the device builds."""
    if kind in ("undistort", "undistort_to"):
        intr, dist = draw_camera(rng, w, h)
        if kind == "undistort":
            return ("device", (intr, dist, None))
        s = float(rng.uniform(0.5, 1.5)) * min(dw / w, dh / h)   # letterboxed into the output, or cropped
        new = (intr[0] * s, intr[1] * s, dw / 2 + float(rng.uniform(-1, 1)), dh / 2 + float(rng.uniform(-1, 1)))
        return ("device", (intr, dist, new))
    v, u = np.mgrid[0:dh, 0:dw].astype(np.float64)
    if kind == "smooth":
        a = rng.uniform(-1.5, 1.5, (2, 3)) * ((1.0, w / max(dw, 1), w / max(dh, 1)), (1.0, h / max(dw, 1), h / max(dh, 1)))
        a[:, 0] = rng.uniform(-0.2, 1.0, 2) * (w, h)
        ph = rng.uniform(0, 6.3, 2)
        mx = a[0, 0] + a[0, 1] * u + a[0, 2] * v + 0.1 * w * np.sin(u / max(dw, 1) * 3 + ph[0])
        my = a[1, 0] + a[1, 1] * u + a[1, 2] * v + 0.1 * h * np.cos(v / max(dh, 1) * 3 + ph[1])
        return mx.astype(F32), my.astype(F32)
    if kind == "constant":
        x = float(rng.uniform(-0.2, 1.2) * w) if rng.random() < 0.7 else float(rng.choice(edge_values(w)))
        y = float(rng.uniform(-0.2, 1.2) * h) if rng.random() < 0.7 else float(rng.choice(edge_values(h)))
        return np.full((dh, dw), x, F32), np.full((dh, dw), y, F32)

    def noise(n, shape):
        specials = np.array([np.nan, np.inf, -np.inf, -0.0, 1e30, -1e30] + edge_values(n) + [n / 2 + 0.5, 0.5], F32)
        vals = rng.uniform(-0.3 * n, 1.3 * n, shape).astype(F32)
        pick = rng.random(shape) < 0.3
        vals[pick] = rng.choice(specials, int(pick.sum()))
        half = rng.random(shape) < 0.1   # nearest's ties
        vals[half] = (rng.integers(0, n, int(half.sum())) + 0.5).astype(F32)
        return vals
    return noise(w, (dh, dw)), noise(h, (dh, dw))


# ── the cases ──────────────────────────────────────────────────────────────────────────────────────────────────────────
@dataclass(frozen=True)
class MCase:
    base: object              # restate.Case: format, frame geometry, sampler, normalisation, pad value, dst size
    out: str
    n_frames: int
    offsets: tuple            # each frame's byte offset in one allocation (16-B aligned base)
    maps: tuple               # per map: (kind, drawn map)
    regions: tuple            # (frame k, map j)

    @property
    def rcase(self):
        return RCase(self.base, 1, self.out, self.n_frames, self.offsets, ())

    def __str__(self):
        c = self.base
        return (f"{c.name}: {c.fmt.name} matrix {c.matrix} bpp {c.bpp} {c.w}x{c.h} pitch {c.pitch} -> {c.dw}x{c.dh} {SAMPLING_NAME[c.sampling]} "
                f"{self.out} norm {c.norm} pad {c.pad_value} frames {self.offsets} maps {[k for k, _ in self.maps]} {len(self.regions)} regions")


def mcase(i):
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
    base = make_case(f"remap-{i}", BASE + i, f.code, (i % len(CODES) + 2 * (i // len(CODES))) % 4 if yuv(f) else 0, bpp, w, h, pitch, dw, dh,
                     sampling, str(rng.choice(list(NORMS))), float(rng.integers(0, 256)))
    offs = place(rng, f, src_bytes(f, w, h, pitch), n_frames, odd=not first and rng.random() < 0.3)
    n_maps = int(rng.integers(1, 5))
    kinds = [KINDS[(i + j) % len(KINDS)] if j < 2 else str(rng.choice(KINDS)) for j in range(n_maps)]
    maps = tuple((k, draw_map_pair(rng, k, w, h, dw, dh)) for k in kinds)
    n = int(rng.choice([int(rng.integers(1, 8)), int(rng.integers(1, 41))]))
    regions = tuple((int(rng.integers(0, n_frames)), int(rng.integers(0, n_maps))) for _ in range(n))
    return MCase(base, str(rng.choice(OUTS)), n_frames, offs, maps, regions)


N_SWEEP = 2 * len(CODES)


# ── the call ─────────────────────────────────────────────────────────────────────────────────────────────────────────
def region_array(regions):
    from kornia_rs_b200._lib import RemapRoi
    return (RemapRoi * max(1, len(regions)))(*[RemapRoi(k, j) for k, j in regions])


def call(lib, c, ptrs, lens, map_x, map_y, map_len, n_maps, regions, dst_ptr, dst_len, out, stream=None, desc=None):
    from kornia_rs_b200._lib import PreprocessDesc
    d = desc if desc is not None else c.desc(PreprocessDesc)
    n = len(ptrs)
    return lib.kb200_preprocess_remap(stream, C.byref(d), (C.c_void_p * max(1, n))(*ptrs), (C.c_size_t * max(1, n))(*lens) if lens is not None else None,
                                      n, map_x, map_y, map_len, n_maps, region_array(regions), len(regions), dst_ptr, dst_len, OUTS.index(out))


def generate(lib, dev, intr, dist, new, dw, dh):
    """The device generator's map (map_x, map_y) as float32 numpy arrays [dh, dw]: the `_to` entry when new is given."""
    mx = torch.empty((dh, dw), dtype=torch.float32, device=dev)
    my = torch.empty_like(mx)
    i4, d8 = (C.c_double * 4)(*intr), (C.c_double * 8)(*dist)
    if new is None:
        st = lib.kb200_generate_correction_map_polynomial(None, i4, d8, dw, dh, mx.data_ptr(), my.data_ptr(), mx.numel())
    else:
        st = lib.kb200_generate_correction_map_polynomial_to(None, i4, d8, (C.c_double * 4)(*new), dw, dh, mx.data_ptr(), my.data_ptr(), mx.numel())
    assert st == 0
    torch.cuda.synchronize()
    return mx.cpu().numpy(), my.cpu().numpy()


def resolve_maps(lib, dev, mc):
    """The case's maps as float32 numpy arrays [K, dh, dw], the generator kinds built on the device."""
    c = mc.base
    xs, ys = [], []
    for _, m in mc.maps:
        mx, my = generate(lib, dev, *m[1], c.dw, c.dh) if isinstance(m[0], str) else m
        xs.append(mx)
        ys.append(my)
    return np.stack(xs), np.stack(ys)


def map_buffer(dev, mx, my, shift):
    """map_x and map_y in one allocation, each starting `shift` bytes past a 16-B boundary, fenced by NaN."""
    k = mx.size
    span = -(-(k * 4 + 64) // 16) * 16
    buf = torch.full((2 * span + 64,), float("nan"), dtype=torch.float32, device=dev).view(torch.uint8)
    ox, oy = 16 + shift, 16 + span + shift
    buf[ox:ox + 4 * k].copy_(torch.from_numpy(mx.reshape(-1).view(np.uint8)))
    buf[oy:oy + 4 * k].copy_(torch.from_numpy(my.reshape(-1).view(np.uint8)))
    return buf, buf.data_ptr() + ox, buf.data_ptr() + oy


def run_mcase(kb, lib, dev, mc):
    c = mc.base
    raws, src = load_frames(dev, mc.rcase)
    ptrs = [src.ptr + o for o in mc.offsets]
    mx, my = resolve_maps(lib, dev, mc)
    m = len(mc.regions)
    elems = 3 * c.dw * c.dh
    esz = ESZ[mc.out]
    nbytes = m * elems * esz
    outs = []
    for dst_shift, map_shift in ((0, 0), (esz, 0), (0, 4)):
        buf, px, py = map_buffer(dev, mx, my, map_shift)
        dst = Guarded(dev, nbytes, min(nbytes, 1 << 16), dst_shift).fill(0xFF)
        st = call(lib, c, ptrs, [c.need] * mc.n_frames, px, py, mx.size, len(mc.maps), mc.regions, dst.ptr, m * elems, mc.out)
        assert st == 0, f"{mc}: status {st}: {kb._lib.last_error()}"
        ran = kb._lib.last_kernel()
        torch.cuda.synchronize()
        want = expected_kernel(c.dw, mc.out, dst.ptr, px, py)
        assert ran == want, f"{mc}: dst +{dst_shift} B, maps +{map_shift} B ran {ran}, the dispatch mirror says {want}"
        assert (dst_shift, map_shift) == (0, 0) or ran == GENERIC
        buf_after = dst.snapshot()
        for what, g in (("lead", buf_after[:dst.lead]), ("tail", buf_after[dst.lead + dst.n:])):
            assert (g == 0xFF).all(), f"{mc}: dst +{dst_shift} B: bytes written in the {what} guard"
        outs.append(buf_after[dst.lead:dst.lead + dst.n])
        del buf
    ones = outs[0].view(np.uint16 if esz == 2 else np.uint32) == (0xFFFF if esz == 2 else 0xFFFFFFFF)
    assert not ones.any(), f"{mc}: {int(ones.sum())} output elements left unwritten"
    pics = {}
    fb = elems * esz
    for i, (k, j) in enumerate(mc.regions):
        if k not in pics:
            pics[k] = picture(c, raws[k])
        want = remap_reference(pics[k], mx[j], my[j], c.sampling, c.norm, c.pad_value, mc.out)
        compare_region(outs[0][i * fb:(i + 1) * fb], want, mc.rcase, f"{mc}: region {i} frame {k} map {j} ({mc.maps[j][0]})")
    for o in outs[1:]:
        bad = np.flatnonzero(outs[0] != o)
        assert bad.size == 0, f"{mc}: the kernels differ in {bad.size} bytes"


# The GPU tests below loop over their cases inside one test each; every assertion message names its case.
@pytest.mark.gpu
def test_sweep(kb, lib, dev):
    for i in range(N_SWEEP):
        run_mcase(kb, lib, dev, mcase(i))


@pytest.mark.gpu
def test_identity_twin(kb, lib, dev):
    for code in CODES:
        identity_twin(kb, lib, dev, code)


def identity_twin(kb, lib, dev, code):
    """An identity map of each whole frame == the batch entry on that frame at dst = src_w x src_h (Stretch: scale 1, pad 0),
    for Nearest and Bilinear and every output type."""
    f = FORMATS[code]
    mw, mh, sw, sh = size_rule(f)
    w, h = max(mw, 20 // sw * sw), max(mh, 12 // sh * sh)
    v, u = np.mgrid[0:h, 0:w].astype(F32)
    mx, my = torch.from_numpy(u.copy()).to(dev), torch.from_numpy(v.copy()).to(dev)
    for j, (samp, out) in enumerate([(s, o) for s in (NEAREST, BILINEAR) for o in OUTS]):
        c = make_case(f"identity-{f.name}", BASE + 0x3000 + code, code, j % 4 if yuv(f) else 0, 3, w, h, row_bytes(f, w, 3), w, h, samp,
                      "imagenet", 114.0)
        mc = MCase(c, out, 2, (16, 16 + -(-c.need // 16) * 16), (), ())
        raws, src = load_frames(dev, mc.rcase)
        ptrs = [src.ptr + o for o in mc.offsets]
        got = torch.full((2 * 3 * w * h * ESZ[out],), 0xFF, dtype=torch.uint8, device=dev)
        assert call(lib, c, ptrs, [c.need] * 2, mx.data_ptr(), my.data_ptr(), w * h, 1, ((1, 0), (0, 0)), got.data_ptr(), 2 * 3 * w * h,
                    out) == 0, kb._lib.last_error()
        want = torch.zeros_like(got)
        assert batch_entry(lib, c, out, [ptrs[1], ptrs[0]], want) == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"{f.name} {SAMPLING_NAME[samp]} {out}: identity map differs from the batch entry"


def warp_twin_map(rng, kind, w, h, dw, dh, lib):
    """(forward map, map_x, map_y): warp_coords' float32 coordinates of a map without a degenerate axis, NaN outside."""
    while True:
        fwd = draw_map(rng, kind, w, h, dw, dh)
        inv, persp = inverse(lib, fwd)
        if persp or (abs(inv[0, 0]) >= 1e-6 and abs(inv[1, 0]) >= 1e-6):
            break
    sx, sy, inside, _ = warp_coords(inv, persp, dw, dh, w, h)
    return fwd, np.where(inside, sx, F32(np.nan)).astype(F32), np.where(inside, sy, F32(np.nan)).astype(F32)


@pytest.mark.gpu
def test_warp_twin(kb, lib, dev):
    for code in CODES:
        warp_twin(kb, lib, dev, code)


def warp_twin(kb, lib, dev, code):
    """Affine and perspective maps as dense maps (warp_coords' coordinates, NaN outside) == kb200_preprocess_warps on the
    same maps, bit for bit."""
    f = FORMATS[code]
    mw, mh, sw, sh = size_rule(f)
    w, h = max(mw, 36 // sw * sw), max(mh, 28 // sh * sh)
    rng = np.random.default_rng(BASE + 0x4000 + code)
    for j, (kind, samp, out, dw) in enumerate((("similarity", BILINEAR, "f32", 24), ("affine", NEAREST, "f16", 21), ("perspective", BILINEAR, "bf16", 20),
                                               ("perspective", NEAREST, "f32", 17))):
        dh = 18
        c = make_case(f"warp-twin-{f.name}", BASE + 0x4000 + code, code, j % 4 if yuv(f) else 0, 3, w, h, row_bytes(f, w, 3), dw, dh, samp,
                      "imagenet", float(rng.integers(0, 256)))
        mc = MCase(c, out, 2, (16, 16 + -(-c.need // 16) * 16), (), ())
        raws, src = load_frames(dev, mc.rcase)
        ptrs = [src.ptr + o for o in mc.offsets]
        fwds, xs, ys = zip(*[warp_twin_map(rng, kind, w, h, dw, dh, lib) for _ in range(3)])
        mx, my = torch.from_numpy(np.stack(xs)).to(dev), torch.from_numpy(np.stack(ys)).to(dev)
        regions = ((0, 2), (1, 0), (0, 1))
        n = 3 * 3 * dw * dh
        got = torch.full((n * ESZ[out],), 0xFF, dtype=torch.uint8, device=dev)
        assert call(lib, c, ptrs, [c.need] * 2, mx.data_ptr(), my.data_ptr(), mx.numel(), 3, regions, got.data_ptr(), n, out) == 0, kb._lib.last_error()
        want = torch.zeros_like(got)
        from kornia_rs_b200._lib import PreprocessDesc
        st = lib.kb200_preprocess_warps(None, C.byref(c.desc(PreprocessDesc)), (C.c_void_p * 2)(*ptrs), None, 2,
                                        warp_array([(k, fwds[q]) for k, q in regions]), 3, want.data_ptr(), n, OUTS.index(out))
        assert st == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"{f.name} {kind} {SAMPLING_NAME[samp]} {out}: differs from kb200_preprocess_warps"


def table_case(n, code, seed):
    """n regions over 3 frames and 4 maps of mixed kinds, in a frame and map order of no pattern."""
    rng = np.random.default_rng(seed)
    f = FORMATS[code]
    w, h, dw, dh = 24, 16, 8, 6
    base = make_case(f"table-{n}-{f.name}", seed, code, 1 if yuv(f) else 0, 1, w, h, row_bytes(f, w, 1), dw, dh, BILINEAR, "imagenet", 114.0)
    maps = tuple((k, draw_map_pair(rng, k, w, h, dw, dh)) for k in ("undistort_to", "smooth", "noise", "constant"))
    regions = tuple((int(rng.integers(0, 3)), int(rng.integers(0, 4))) for _ in range(n))
    return MCase(base, OUTS[n % 3], 3, place(rng, f, src_bytes(f, w, h, base.pitch), 3), maps, regions)


TABLES = [table_case(n, code, BASE + 0x1000 + 16 * n + code) for n in (CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 17) for code in (3, 18)]


@pytest.mark.gpu
def test_regions_and_maps(kb, lib, dev):
    for mc in TABLES:
        regions_and_maps(kb, lib, dev, mc)


def regions_and_maps(kb, lib, dev, mc):
    """Region counts around the launch chunk, several maps and an arbitrary (frame, map) table: the reference, and one
    shared-map call per map on that map's regions, bit for bit."""
    run_mcase(kb, lib, dev, mc)
    c = mc.base
    raws, src = load_frames(dev, mc.rcase)
    ptrs = [src.ptr + o for o in mc.offsets]
    mx, my = (torch.from_numpy(a).to(dev) for a in resolve_maps(lib, dev, mc))
    elems = 3 * c.dw * c.dh
    dt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[mc.out]
    whole = torch.empty((len(mc.regions), elems), dtype=dt, device=dev)
    assert call(lib, c, ptrs, [c.need] * 3, mx.data_ptr(), my.data_ptr(), mx.numel(), 4, mc.regions, whole.data_ptr(), whole.numel(), mc.out) == 0
    for j in range(4):
        idx = [i for i, (_, q) in enumerate(mc.regions) if q == j]
        part = torch.empty((len(idx), elems), dtype=dt, device=dev)
        assert call(lib, c, ptrs, [c.need] * 3, mx[j].data_ptr(), my[j].data_ptr(), mx[j].numel(), 1, [(mc.regions[i][0], 0) for i in idx],
                    part.data_ptr(), part.numel(), mc.out) == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        assert torch.equal(whole[idx].view(torch.uint8), part.view(torch.uint8)), f"{mc}: map {j} differs from its shared-map call"


@pytest.mark.gpu
def test_graph_capture(kb, lib, dev):
    mc = TABLES[-2]   # 401 NV12 regions: three launches
    c = mc.base
    raws, src = load_frames(dev, mc.rcase)
    ptrs = [src.ptr + o for o in mc.offsets]
    mx, my = (torch.from_numpy(a).to(dev) for a in resolve_maps(lib, dev, mc))
    n = len(mc.regions) * 3 * c.dw * c.dh
    eager = torch.empty(n, dtype=torch.float16, device=dev)
    replay = torch.zeros_like(eager)
    args = (ptrs, [c.need] * 3, mx.data_ptr(), my.data_ptr(), mx.numel(), 4, mc.regions)
    assert call(lib, c, *args, eager.data_ptr(), n, "f16") == 0
    s = torch.cuda.Stream(dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            st = call(lib, c, *args, replay.data_ptr(), n, "f16", stream=s.cuda_stream)
    assert st == 0, kb._lib.last_error()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.view(torch.int16), replay.view(torch.int16))


@pytest.mark.gpu
def test_python_run_remap(kb, lib, dev):
    for fmt in ("Rgb8", "Nv12", "Yuyv", "BayerGrbg12p", "P010", "I444"):
        python_run_remap(kb, lib, dev, fmt)


def python_run_remap(kb, lib, dev, fmt):
    """Preprocessor.run_remap == the C entry, with [H, W], [K, H, W] and Image maps, for all three dtypes."""
    sf = kb.SourceFormat[fmt]
    w, h, dw, dh = 24, 18, 12, 8
    rng = np.random.default_rng(len(fmt))
    n = sf.buffer_len(w, h)
    frames = [torch.from_numpy(rng.integers(0, 256, n, dtype=np.int64).astype(np.uint8)).to(dev) for _ in range(2)]
    intr, dist = draw_camera(rng, w, h)
    img_x, img_y = kb.imgproc.generate_correction_map_polynomial(intr, dist, kb.ImageSize(dw, dh), dev,
                                                                 new_intrinsic=(intr[0] / 2, intr[1] / 2, dw / 2, dh / 2))
    smooth = draw_map_pair(rng, "smooth", w, h, dw, dh)
    mx = torch.stack([img_x.data[..., 0], torch.from_numpy(smooth[0]).to(dev)]).contiguous()
    my = torch.stack([img_y.data[..., 0], torch.from_numpy(smooth[1]).to(dev)]).contiguous()
    regions = [(1, 0), (0, 1), (1, 1)]
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        pre = (kb.Preprocessor.builder().source_format(sf).sampling(kb.InterpolationMode.Bilinear).normalize(kb.Normalize.imagenet()).build_cuda())
        desc = pre._desc(w, h, sf.pitch(w), sf.bpp(), sf.fmt_code(), dw, dh)
        want = torch.empty((3, 3, dh, dw), dtype=dtype, device=dev)
        st = lib.kb200_preprocess_remap(None, C.byref(desc), (C.c_void_p * 2)(*[f.data_ptr() for f in frames]), (C.c_size_t * 2)(n, n), 2,
                                        mx.data_ptr(), my.data_ptr(), mx.numel(), 2, region_array(regions), 3, want.data_ptr(), want.numel(),
                                        (torch.float32, torch.float16, torch.bfloat16).index(dtype))
        assert st == 0, kb._lib.last_error()
        got = torch.empty_like(want)
        pre.run_remap(frames, w, h, mx, my, got, torch.tensor(regions))
        shared = torch.empty((2, 3, dh, dw), dtype=dtype, device=dev)   # regions None: (i, 0) for every frame, Image maps
        pre.run_remap(frames, w, h, img_x, img_y, shared)
        one = torch.empty((1, 3, dh, dw), dtype=dtype, device=dev)      # [H, W] maps
        pre.run_remap(frames, w, h, mx[1], my[1], one, [(0, 0)])
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), (fmt, dtype)
        assert torch.equal(shared[1].view(torch.uint8), want[0].view(torch.uint8)), (fmt, dtype)
        assert torch.equal(one[0].view(torch.uint8), want[1].view(torch.uint8)), (fmt, dtype)


@pytest.mark.gpu
def test_correction_map_to(kb, lib, dev):
    """`_to` with new_intrinsic == intrinsic gives the existing entry's bits; other new_intrinsics match the float64
    restatement bit for bit, at output sizes other than the frame's."""
    rng = np.random.default_rng(BASE + 0x7000)
    for t in range(6):
        w, h = int(rng.integers(40, 200)), int(rng.integers(30, 120))
        intr, dist = draw_camera(rng, w, h)
        dist = tuple(dist[:4]) + tuple(float(v) for v in rng.uniform(0, 0.05, 2)) + dist[6:]
        plain = generate(lib, dev, intr, dist, None, w, h)
        same = generate(lib, dev, intr, dist, intr, w, h)
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(plain, same)), t
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(plain, distort_map(intr, dist, intr, w, h))), t
        dw, dh = int(rng.integers(8, 160)), int(rng.integers(8, 160))
        new = (float(rng.uniform(0.3, 2.0)) * intr[0], float(rng.uniform(0.3, 2.0)) * intr[1], float(rng.uniform(0, dw)), float(rng.uniform(0, dh)))
        got = generate(lib, dev, intr, dist, new, dw, dh)
        want = distort_map(intr, dist, new, dw, dh)
        for a, b in zip(got, want):
            bad = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
            assert bad.size == 0, f"case {t}: {bad.size} map entries differ, first {a.reshape(-1)[bad[0]]} != {b.reshape(-1)[bad[0]]}"


@pytest.mark.gpu
def test_cv2_anchor(kb, lib, dev):
    """Bilinear f32 output x 255 (unit normalisation) against cv2.remap (INTER_LINEAR, BORDER_CONSTANT) on smooth RGB8
    frames, over the pixels whose sample lies at least one pixel inside the frame.  cv2 rounds each coordinate to 1/32 px
    (error <= 1/64 per axis), weighs the taps in 15-bit fixed point and rounds to u8, so
    |ours - cv2| <= 0.5 + 2 * G / 64 + 4 * 255 / 2^15, G the frame's largest difference between neighbouring pixels."""
    cv2 = pytest.importorskip("cv2")
    w, h, dw, dh = 96, 64, 80, 56
    rng = np.random.default_rng(BASE + 0x6000)
    for t in range(8):
        img = smooth_rgb(w, h, BASE + t)
        g = max(np.abs(np.diff(img.astype(np.int32), axis=0)).max(), np.abs(np.diff(img.astype(np.int32), axis=1)).max())
        tol = 0.5 + 2 * g / 64 + 4 * 255 / 2 ** 15
        while True:   # a map with at least a fifth of its output on interior samples
            m = draw_map_pair(rng, ("undistort_to", "smooth")[t % 2], w, h, dw, dh)
            mx, my = generate(lib, dev, *m[1], dw, dh) if isinstance(m[0], str) else m
            interior = (mx >= 1) & (mx <= w - 2) & (my >= 1) & (my <= h - 2)
            if interior.sum() > 0.2 * dw * dh:
                break
        c = make_case("cv2", 0, 0, 0, 3, w, h, 3 * w, dw, dh, BILINEAR, "unit", 0.0)
        src = torch.from_numpy(img.reshape(-1).copy()).to(dev)
        dmx, dmy = torch.from_numpy(mx).to(dev), torch.from_numpy(my).to(dev)
        out = torch.empty((3, dh, dw), dtype=torch.float32, device=dev)
        assert call(lib, c, [src.data_ptr()], [src.numel()], dmx.data_ptr(), dmy.data_ptr(), dmx.numel(), 1, [(0, 0)], out.data_ptr(), out.numel(),
                    "f32") == 0, kb._lib.last_error()
        torch.cuda.synchronize()
        ours = out.cpu().numpy().transpose(1, 2, 0) * 255.0
        ref = cv2.remap(img, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT).astype(np.float64)
        err = np.abs(ours - ref)[interior]
        assert err.max() <= tol, f"map {t}: max |ours - cv2| {err.max():.3f} > {tol:.3f}"


# ── CPU: validation, symbols, run_remap argument rules, coverage ─────────────────────────────────────────────────────
FAKE = 0x7F0000000000   # never dereferenced: every call below is refused on the host
MAP = FAKE + (1 << 24)


def _valid_case(code=3, sampling=BILINEAR):
    f = FORMATS[code]
    return make_case("valid", 1, code, 0, 3, 64, 48, row_bytes(f, 64, 3), 16, 16, sampling, "imagenet", 114.0)


REGION_RULES = [((2, 0), "frame index 2 is outside [0, 2)"), ((-1, 0), "frame index -1"), ((0, 2), "map index 2 is outside [0, 2)"),
                ((1, -1), "map index -1")]


def test_invalid_region_is_refused_on_the_host(kb):
    lib = kb._lib.lib()
    c = _valid_case()
    for region, rule in REGION_RULES:
        st = call(lib, c, [FAKE, FAKE + 8192], [c.need] * 2, MAP, MAP + 4096, 2 * 256, 2, [(1, 1), region], FAKE, 2 * 3 * 256, "f32")
        msg = kb._lib.last_error()
        assert st == INVALID and msg.startswith("region 1:") and rule in msg, (region, st, msg)


def test_invalid_call_is_refused_on_the_host(kb):
    from kornia_rs_b200._lib import PreprocessDesc
    lib = kb._lib.lib()
    c = _valid_case()
    ok = dict(ptrs=[FAKE, FAKE + 8192], lens=[c.need] * 2, map_x=MAP, map_y=MAP + 4096, map_len=256, n_maps=1, regions=[(0, 0)], dst_ptr=FAKE,
              dst_len=3 * 256, out="f32")

    def go(case=c, **kw):
        a = dict(ok, **kw)
        return call(lib, case, a["ptrs"], a["lens"], a["map_x"], a["map_y"], a["map_len"], a["n_maps"], a["regions"], a["dst_ptr"], a["dst_len"], a["out"])

    def err():
        return kb._lib.last_error()

    assert go(regions=[]) == INVALID and "n_regions" in err()
    assert go(n_maps=0) == INVALID and "n_maps" in err()
    assert go(case=_valid_case(sampling=LANCZOS)) == UNSUPPORTED and "Nearest or Bilinear" in err()
    d = c.desc(PreprocessDesc)
    regions = region_array([(0, 0)])
    frames = (C.c_void_p * 1)(FAKE)
    assert lib.kb200_preprocess_remap(None, C.byref(d), frames, None, 1, MAP, MAP, 256, 1, regions, 1, FAKE, 768, 3) == INVALID
    assert "output format" in err()
    assert lib.kb200_preprocess_remap(None, C.byref(d), None, None, 1, MAP, MAP, 256, 1, regions, 1, FAKE, 768, 0) == INVALID and "'frames'" in err()
    assert lib.kb200_preprocess_remap(None, C.byref(d), frames, None, 1, MAP, MAP, 256, 1, None, 1, FAKE, 768, 0) == INVALID and "'regions'" in err()
    assert lib.kb200_preprocess_remap(None, C.byref(d), frames, None, 1, None, MAP, 256, 1, regions, 1, FAKE, 768, 0) == INVALID and "'map_x'" in err()
    assert lib.kb200_preprocess_remap(None, C.byref(d), frames, None, 1, MAP, None, 256, 1, regions, 1, FAKE, 768, 0) == INVALID and "'map_y'" in err()
    assert lib.kb200_preprocess_remap(None, C.byref(d), frames, None, 1, MAP, MAP, 256, 1, regions, 1, None, 768, 0) == INVALID and "'dst'" in err()
    assert lib.kb200_preprocess_remap(None, None, frames, None, 1, MAP, MAP, 256, 1, regions, 1, FAKE, 768, 0) == INVALID
    for mx, my in ((MAP + 2, MAP), (MAP, MAP + 1)):
        assert go(map_x=mx, map_y=my) == INVALID and "4-byte aligned" in err()
    assert go(map_len=255) == SLICE and "'map'" in err()
    assert go(n_maps=2, regions=[(0, 1)], map_len=511) == SLICE and "'map'" in err()
    assert go(dst_len=3 * 256 - 1) == SLICE and "'dst'" in err()
    assert go(lens=[c.need, c.need - 1]) == INVALID_SOURCE
    assert go(ptrs=[FAKE, 0]) == INVALID and "null frame pointer at index 1" in err()
    p010 = _valid_case(code=80)
    assert go(case=p010, ptrs=[FAKE, FAKE + 1], lens=[p010.need] * 2) == INVALID_SOURCE and "2-byte aligned" in err()
    # the descriptor's own rules still hold; its scale and pad are ignored
    from dataclasses import replace
    assert go(case=replace(c, w=63)) == INVALID_SOURCE   # odd NV12 width
    d = c.desc(PreprocessDesc)
    d.scale_x, d.pad_y = -1.0, float("nan")
    assert lib.kb200_preprocess_remap(None, C.byref(d), (C.c_void_p * 2)(FAKE, FAKE), None, 2, MAP, MAP, 256, 1, regions, 1, FAKE, 10, 0) == SLICE
    # every refusal comes before anything is enqueued: a bad region after a short frame and a short map is still the region
    assert go(regions=[(0, 0), (0, 5)], lens=[1, 1], map_len=1) == INVALID and "region 1" in err()


def test_header_and_binding_symbols(kb):
    import __graft_entry__ as ge
    from kornia_rs_b200._lib import RemapRoi
    assert {"kb200_preprocess_remap", "kb200_generate_correction_map_polynomial_to"} <= set(ge.declared_symbols())
    assert C.sizeof(RemapRoi) == 8 and RemapRoi.map.offset == 4
    hdr = open(os.path.join(ROOT, "include", "kornia_b200.h")).read()
    assert re.search(r"typedef struct kb200_remap_roi \{\s*int32_t frame, map;\s*\} kb200_remap_roi;", hdr)
    rs = open(os.path.join(ROOT, "bindings", "rust", "src", "lib.rs")).read()
    assert "pub struct kb200_remap_roi" in rs and "pub fn kb200_preprocess_remap(" in rs and "pub fn launch_preprocess_remap(" in rs
    assert "pub fn kb200_generate_correction_map_polynomial_to(" in rs


def test_run_remap_argument_rules(kb):
    """run_remap's own checks, all of which come before any device is touched (every map here is a CPU tensor or fails
    before its device is looked at, except where the test says so)."""
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).build_cuda()
    frame = torch.zeros(64 * 48 * 3 // 2, dtype=torch.uint8)
    dst = torch.zeros((1, 3, 8, 8))
    m = torch.zeros((8, 8))
    for mx, my in ((m, m), (m.double(), m), (torch.zeros(8), m), (torch.zeros((1, 1, 8, 8)), m), ("abc", m), (m, None)):
        with pytest.raises(kb.PreprocessError) as e:   # a CPU map is refused like a map of the wrong shape or dtype
            pre.run_remap([frame], 64, 48, mx, my, dst)
        assert e.value.kind == "InvalidMap" and e.value.fields.get("region") is None, (mx, my)
    img = kb.Image(torch.zeros((8, 8, 3)))
    with pytest.raises(kb.PreprocessError) as e:
        pre.run_remap([frame], 64, 48, img, img, dst)
    assert e.value.kind == "InvalidMap"
    lanczos = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).sampling(kb.InterpolationMode.Lanczos).build_cuda()
    with pytest.raises(kb.PreprocessError) as e:
        lanczos.run_remap([frame], 64, 48, m, m, dst)
    assert e.value.kind == "UnsupportedSampling"


def test_run_remap_region_rules(kb, monkeypatch):
    """The region table's rules, with the maps' own checks passed (a device map is not needed to reach them)."""
    from kornia_rs_b200.preprocess import Preprocessor
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).build_cuda()
    maps = torch.zeros((2, 8, 8))
    monkeypatch.setattr(Preprocessor, "_remap_map", staticmethod(lambda name, m: m))
    frame = torch.zeros(64 * 48 * 3 // 2, dtype=torch.uint8)
    dst = torch.zeros((1, 3, 8, 8))
    for regions, region in (([], None), ([(1, 0)], 0), ([(0, 0), (0, 2)], 1), ([(0, 0), (-1, 0)], 1), ([(0, 0), (0, 0, 0)], 1),
                            ([(0, 0), (0.0, 0)], 1), ([(0, 0), "ab"], 1), ([(0, 0), (True, 0)], 1),
                            (torch.zeros((1, 2), dtype=torch.float32), None), (torch.zeros((1, 3), dtype=torch.int64), None),
                            (torch.tensor([[0, 0], [0, 5]]), 1)):
        with pytest.raises(kb.PreprocessError) as e:
            pre.run_remap([frame], 64, 48, maps, maps, dst, regions)
        assert e.value.kind == "InvalidMap", regions
        assert e.value.fields.get("region") == region, (regions, e.value.fields)
    with pytest.raises(kb.PreprocessError) as e:   # two regions, one output
        pre.run_remap([frame], 64, 48, maps, maps, dst, [(0, 0), (0, 1)])
    assert e.value.kind == "BatchMismatch"
    with pytest.raises(kb.PreprocessError) as e:
        pre.run_remap([frame], 64, 48, maps, maps, torch.zeros((1, 3, 8, 8), dtype=torch.float64), [(0, 0)])
    assert e.value.kind == "BadOutputShape"
    with pytest.raises(kb.PreprocessError) as e:   # a CPU destination
        pre.run_remap([frame], 64, 48, maps, maps, dst, [(0, 0)])
    assert e.value.kind == "NotDeviceTensor"


def test_sweep_coverage(kb):
    """Every format, every map kind, both store paths, NaN / inf / 1e30 / -0.0 pads, and samples that land exactly on 0,
    W - 1, the float below W and W."""
    cases = [mcase(i) for i in range(N_SWEEP)]
    formats, vec, kinds, outs, samplers = set(), set(), set(), set(), set()
    landed, specials = set(), set()
    for mc in cases + TABLES:
        c = mc.base
        formats.add(c.code)
        vec.add((c.code, c.dw % 4 == 0))
        outs.add(mc.out)
        samplers.add(c.sampling)
        used = {j for _, j in mc.regions}
        for j, (k, m) in enumerate(mc.maps):
            if j not in used:
                continue
            kinds.add(k)
            if isinstance(m[0], str):
                continue
            for axis, s, n in (("x", m[0], c.w), ("y", m[1], c.h)):
                for name, v in (("0", F32(0)), ("W-1", F32(n - 1)), ("below W", np.nextafter(F32(n), F32(0))), ("W", F32(n))):
                    if (s == v).any():
                        landed.add((axis, name))
                specials |= {name for name, hit in (("nan", np.isnan(s).any()), ("inf", np.isposinf(s).any()), ("-inf", np.isneginf(s).any()),
                                                    ("1e30", (s == F32(1e30)).any()), ("-0", (np.signbit(s) & (s == 0)).any()))
                             if hit}
    assert formats == set(CODES)
    for code in CODES:
        assert (code, True) in vec, FORMATS[code].name   # the vector kernel at the aligned run; the shifted runs take the generic one
    assert kinds == set(KINDS) and outs == set(OUTS) and samplers == {NEAREST, BILINEAR}
    assert landed == {(a, n) for a in "xy" for n in ("0", "W-1", "below W", "W")}, landed
    assert specials == {"nan", "inf", "-inf", "1e30", "-0"}, specials
    assert max(len(mc.regions) for mc in TABLES) > 2 * CHUNK
    assert any(len({k for k, _ in mc.regions}) > 1 and len({j for _, j in mc.regions}) > 1 for mc in cases)
    assert {o % 2 for mc in cases for o in mc.offsets} == {0, 1}   # frames at odd and even addresses
    assert any(mc.base.pitch > row_bytes(mc.base.fmt, mc.base.w, mc.base.bpp) for mc in cases)   # pitch padding
