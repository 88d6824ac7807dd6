"""Camera preprocess: a seeded sweep of random geometries and descriptors over every source format, kernel, sampler and
entry, against references that do not use the library's decoders.

`case(i)` is a pure function of its index (numpy.random.default_rng(BASE + i)): format i % 51, descriptor kind
(i // 51) % 9, and random source size, pitch padding, destination size, sampler, output type, entry, frame layout,
YUV matrix and normalisation.  Hand-picked edge cases (EDGES) run through the same machinery.  Each case:

  * runs through its entry (pointer table, strided, or host pipeline) into a destination prefilled with 0xFF bytes (NaN in
    f32 and f16) inside test_footprint.Guarded, whose guards must keep their fill;
  * must run the kernel that `expected_kernel`, a host mirror of launch_preprocess's dispatch rule, names for it;
  * is compared with a restatement the suite already trusts: the oracle's ko_preprocess_frame on the case's own
    descriptor (for YUV and Bayer frames on the restated RGB8 decode), or test_bayer16.preprocess_rgb16 on the restated
    16-bit RGB decode; bit for bit, Lanczos within the oracle tolerance (host sinf against CUDA's);
  * unless it samples with Lanczos, runs a second time into a destination one element past a 16-byte boundary, which
    refuses the identity and fast kernels: the generic kernel must then give the same bits.

test_sweep_coverage (CPU only) runs every case through the dispatch mirror and asserts what the sweep covers, so that a
change to the generator cannot silently shrink it.
"""
import ctypes as C
from collections import defaultdict
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from test_bayer import demosaic as demosaic8
from test_bayer16 import PATTERNS, demosaic as demosaic16, preprocess_rgb16
from test_bayer_packed import GROUP, unpack
from test_footprint import Guarded
from test_yuv16 import decode as decode_yuv16
from test_yuv444 import decode8 as decode_yuv444, decode16 as decode_yuv444_16
from test_yuv_layouts import to_twin
from test_yuv_matrix import MATRICES, decode as decode_yuv8

BASE = 0x5EED0000
GENERIC = "preprocess_generic_kernel"
NEAREST, BILINEAR, LANCZOS = 0, 1, 3
SAMPLING_NAME = {NEAREST: "Nearest", BILINEAR: "Bilinear", LANCZOS: "Lanczos"}
ENTRIES = ("table", "strided", "host")
KINDS = ("letterbox", "stretch", "identity", "identity-miss", "crop", "nonuniform", "fractional", "offedge", "boundary")
F32 = np.float32
IMAGENET_INV = tuple(float(F32(1.0) / F32(s)) for s in (0.229, 0.224, 0.225))
NORMS = {"imagenet": ((0.485, 0.456, 0.406), IMAGENET_INV), "unit": ((0.0,) * 3, (1.0,) * 3), "scale255": ((0.0,) * 3, (255.0,) * 3)}


# ── the source formats: preprocess.cu's SRC_FORMATS ──────────────────────────────────────────────────────────────────
@dataclass(frozen=True)
class Fmt:
    code: int
    name: str
    family: str               # rgb, gray, yuv420, yuv422, yuv444, bayer
    layout: str = ""          # the YUV layout in the test modules' spelling; the Bayer pattern
    bits: int = 8
    words: bool = False       # one 16-bit word per sample
    packed: bool = False      # MIPI CSI-2 packed samples
    identity: str | None = None
    fast: str | None = None


def _formats():
    f = [Fmt(0, "Rgb8", "rgb"), Fmt(1, "Bgr8", "rgb"), Fmt(2, "Gray8", "gray")]
    for code, lay in ((3, "Nv12"), (5, "Nv21"), (6, "I420"), (7, "Yv12")):
        f.append(Fmt(code, lay, "yuv420", lay, identity=f"preprocess_{lay.lower()}_identity_kernel", fast=f"preprocess_{lay.lower()}_kernel"))
    for code, lay in ((4, "Yuyv"), (8, "Uyvy"), (9, "Yvyu")):
        f.append(Fmt(code, lay, "yuv422", lay))
    f.append(Fmt(11, "I444", "yuv444", identity="preprocess_i444_identity_kernel", fast="preprocess_i444_kernel"))
    for p, pat in enumerate(PATTERNS):
        name = "Bayer" + pat.capitalize()
        f.append(Fmt(16 + p, name, "bayer", pat, identity=f"preprocess_bayer_{pat.lower()}_identity_kernel"))
        for k, bits in enumerate((10, 12, 14, 16)):
            f.append(Fmt(32 + 4 * k + p, f"{name}{bits}", "bayer", pat, bits, words=True, identity=f"preprocess_bayer16_{pat.lower()}_identity_kernel"))
        for k, bits in enumerate((10, 12, 14)):
            f.append(Fmt(64 + 4 * k + p, f"{name}{bits}p", "bayer", pat, bits, packed=True,
                         identity=f"preprocess_bayer{bits}p_{pat.lower()}_identity_kernel"))
    for code, name in ((80, "P010"), (81, "P012"), (82, "I010"), (83, "I012")):
        k = "p01x" if name[0] == "P" else "i01x"
        f.append(Fmt(code, name, "yuv420", "Nv12" if name[0] == "P" else "I420", int(name[2:]), words=True,
                     identity=f"preprocess_{k}_identity_kernel", fast=f"preprocess_{k}_kernel"))
    for code, name in ((85, "I410"), (86, "I412"), (87, "I410Msb"), (88, "I412Msb")):
        f.append(Fmt(code, name, "yuv444", "", int(name[2:4]), words=True, identity="preprocess_i41x_identity_kernel", fast="preprocess_i41x_kernel"))
    return {x.code: x for x in sorted(f, key=lambda x: x.code)}


FORMATS = _formats()
CODES = tuple(FORMATS)
assert len(CODES) == 51


def group(f):
    """The family a sampler (and, for YUV, a matrix) must be covered for."""
    if f.family == "bayer":
        return f"bayer{f.bits}p" if f.packed else "bayer16" if f.words else "bayer8"
    return f.family + ("-16" if f.words else "")


def yuv(f):
    return f.family.startswith("yuv")


def row_bytes(f, w, bpp):
    if f.packed:
        return w * f.bits // 8
    return w * (bpp if f.family == "rgb" else 2 if f.words or f.family == "yuv422" else 1)


def pad_step(f):
    """Pitch padding a format allows: 0 none (tight frames), else its granularity in bytes."""
    if f.family in ("yuv420", "yuv444"):
        return 0
    return 2 if f.words else 1


def src_bytes(f, w, h, pitch):   # kb200_preprocess_src_bytes
    if f.family == "yuv444":
        return pitch * h * 3
    if f.family == "yuv420":
        return pitch * h + (w * h if f.words else w * h // 2)
    return pitch * h


def id_align(f):   # the identity kernels' row and frame alignment
    return 16 if f.packed else 8 if f.words else 4


def elem_align(f):   # the frame alignment every entry requires
    return 2 if f.words else 1


def size_rule(f):
    """(min w, min h, w step, h step)."""
    if f.family == "yuv420":
        return 2, 2, 2, 2
    if f.family == "yuv422":
        return 2, 1, 2, 1
    if f.family == "bayer":
        return (4, 3, GROUP[f.bits], 1) if f.packed else (3, 3, 1, 1)
    return 1, 1, 1, 1


# ── the dispatch rule, restated (preprocess.cu launch_preprocess) ──────────────────────────────────────────────────────
def expected_kernel(d, frames, stride, dst, sampling):
    """The kernel launch_preprocess runs for descriptor `d` (fmt bits 0-7 the format) on frames at the addresses `frames`
    (pointer table: stride None; strided: [base] and `stride`) into `dst`."""
    f = FORMATS[d.fmt & 0xFF]
    lanczos = sampling == LANCZOS

    def aligned(a):
        return all(p % a == 0 for p in frames) and (stride is None or stride % a == 0)

    a = id_align(f)
    if (not lanczos and f.identity and d.scale_x == 1.0 and d.scale_y == 1.0 and d.pad_x == 0.0 and d.pad_y == 0.0 and d.dst_w == d.src_w
            and d.dst_h == d.src_h and d.src_w % 4 == 0 and d.src_pitch % a == 0 and dst % 16 == 0 and aligned(a)):
        return f.identity
    # the NV12 / NV21 fast kernel reads a chroma pair as one 16-bit word
    pair = f.family == "yuv420" and not f.words and f.layout in ("Nv12", "Nv21")
    if not lanczos and f.fast and d.dst_w % 4 == 0 and dst % 16 == 0 and d.dst_h <= 65535 * 8 and (not pair or aligned(2)):
        return f.fast
    return GENERIC


# ── the cases ──────────────────────────────────────────────────────────────────────────────────────────────────────────
@dataclass(frozen=True)
class Case:
    name: str
    seed: int                 # frame contents
    code: int
    matrix: int
    bpp: int
    w: int
    h: int
    pitch: int
    kind: str
    scale_x: float
    scale_y: float
    pad_x: float
    pad_y: float
    dw: int
    dh: int
    sampling: int
    f16: bool
    entry: str
    batch: int
    frames: tuple             # table: each frame's byte offset in one 16-B aligned allocation; strided / host: (base offset,)
    stride: int | None        # strided / host: bytes from one frame to the next
    chunk: int                # host: frames per staging chunk
    norm: str
    pad_value: float

    @property
    def fmt(self):
        return FORMATS[self.code]

    @property
    def need(self):
        return src_bytes(self.fmt, self.w, self.h, self.pitch)

    def desc(self, cls):
        d = cls()
        d.scale_x, d.scale_y, d.pad_x, d.pad_y = self.scale_x, self.scale_y, self.pad_x, self.pad_y
        d.src_w, d.src_h, d.src_pitch, d.src_bpp = self.w, self.h, self.pitch, self.bpp
        d.fmt = self.code | (self.matrix << 8)
        d.dst_w, d.dst_h = self.dw, self.dh
        mean, inv = NORMS[self.norm]
        d.mean, d.inv_std = (C.c_float * 3)(*mean), (C.c_float * 3)(*inv)
        d.pad_value, d.sampling = self.pad_value, self.sampling
        return d

    def planned(self, dst=0):
        """The kernel the case must run, its frames where the layout puts them (the allocation's base is 16-B aligned; the host
        pipeline stages frames 16-B aligned into its own 16-B aligned buffers)."""
        from oracle.oracle import PreprocessDesc
        if self.entry == "host":
            dev_stride = (self.need + 15) // 16 * 16
            return expected_kernel(self.desc(PreprocessDesc), [0], dev_stride, 0, self.sampling)
        return expected_kernel(self.desc(PreprocessDesc), list(self.frames), self.stride, dst, self.sampling)

    def __str__(self):
        fr = self.frames if len(self.frames) <= 4 else self.frames[:4] + ("...",)
        return (f"{self.name}: {self.fmt.name}(code {self.code}) matrix {self.matrix} bpp {self.bpp} {self.w}x{self.h} pitch {self.pitch} "
                f"kind {self.kind} scale ({self.scale_x!r}, {self.scale_y!r}) pad ({self.pad_x!r}, {self.pad_y!r}) -> {self.dw}x{self.dh} "
                f"{SAMPLING_NAME[self.sampling]} {'f16' if self.f16 else 'f32'} {self.entry} batch {self.batch} frames {fr} stride {self.stride} "
                f"chunk {self.chunk} norm {self.norm} pad_value {self.pad_value}")


def f32(v):
    return float(F32(v))


def layout(rng, f, entry, batch, need, align=None, miss=False):
    """Frame placement: (frames, stride).  `align`: every frame aligned to it; `miss`: one frame (or the stride) not aligned to it."""
    e = elem_align(f)
    if entry == "table":
        offs, at = [], 0
        for k in range(batch):
            if align:
                at = -(-at // align) * align + align * int(rng.integers(0, 3))
            else:
                at += e * int(rng.integers(0, 16 // e))
            offs.append(at)
            at += need + (e * int(rng.integers(0, 8)) if not align else 0)
        if miss:
            k = int(rng.integers(0, batch))
            offs[k] += e * int(rng.integers(1, align // e))
            for j in range(k + 1, batch):
                offs[j] = -(-(offs[j - 1] + need) // align) * align
        return tuple(offs), None
    if align:
        stride = -(-need // align) * align + align * int(rng.integers(0, 2))
        base = 0
        if miss:
            if batch > 1 and rng.random() < 0.5:
                stride += e * int(rng.integers(1, align // e))
            else:
                base = e * int(rng.integers(1, align // e))
        return (base,), stride
    return (e * int(rng.integers(0, 16 // e)),), need + e * int(rng.integers(0, 16 // e))


def host_chunk(c_need, dst_frame, batch):
    """Frames per staging chunk as the host pipeline sizes them (bytes rounded up to 256), for staging asked to hold
    max(1, batch - 1) frames: ragged chunks whenever a frame or its output is at least 256 bytes."""
    want = max(1, batch - 1)
    dev_stride = (c_need + 15) // 16 * 16
    src_b, dst_b = -(-want * dev_stride // 256) * 256, -(-want * dst_frame // 256) * 256
    return min(src_b // dev_stride, dst_b // dst_frame, 256), want * dev_stride, want * dst_frame


def draw_dim(rng, lo, step, hi):
    v = int(rng.integers(lo, 17)) if rng.random() < 0.5 else int(rng.integers(lo, hi + 1))
    return max(lo, v // step * step)


def dst_dim(rng):
    return int(rng.integers(1, 17)) if rng.random() < 0.4 else int(rng.integers(1, 257))


def boundary_axis(rng, n, dst):
    """(scale, pad, target): a pad that puts some destination pixel's source coordinate exactly on the target."""
    targets = {"0": 0.0, "last": float(n - 1), "below": float(np.nextafter(F32(n), F32(0))), "edge": float(n)}
    t = str(rng.choice(list(targets)))
    v = F32(targets[t])
    for scale in (float(rng.choice([1.0, 2.0, 0.5, 0.25, 4.0])), 1.0):
        for o in rng.permutation(dst)[:32]:
            pad = F32(F32(o) - v * F32(scale))
            if (F32(o) - pad) / F32(scale) == v:
                return scale, float(pad), t
    return 1.0, float(F32(F32(dst - 1) - F32(n))), "edge"   # (dst - 1 - pad) / 1 == n exactly


def case(i):
    """Case i of the sweep: a pure function of i."""
    from oracle.oracle import preprocess_affine
    rng = np.random.default_rng(BASE + i)
    f = FORMATS[CODES[i % len(CODES)]]
    kind = KINDS[(i // len(CODES)) % len(KINDS)]
    bpp = int(rng.choice([3, 4])) if f.family == "rgb" else 1
    mw, mh, sw, sh = size_rule(f)
    w, h = draw_dim(rng, mw, sw, 200), draw_dim(rng, mh, sh, 200)
    entry = str(rng.choice(ENTRIES))
    batch = int(rng.integers(1, 4))
    sampling = int(rng.choice([NEAREST, BILINEAR, LANCZOS], p=[0.35, 0.4, 0.25]))
    step = pad_step(f)
    pad_bytes = step * int(rng.integers(1, 24 // step + 1)) if step and rng.random() < 0.6 else 0
    align, miss = None, False
    if kind.startswith("identity"):   # sizes that qualify for the identity kernel, and sizes that just miss
        variant = "hit" if kind == "identity" else str(rng.choice(["width", "pitch", "frame"]))
        if variant == "width" and (f.packed and GROUP[f.bits] == 4):
            variant = "frame"
        if variant == "pitch" and not step:
            variant = "frame"
        if variant == "frame" and entry == "host":
            entry = str(rng.choice(["table", "strided"]))
        if variant == "width":
            w = max(4, w // 4 * 4) + int(rng.choice([r for r in (1, 2, 3) if r % sw == 0]))
        else:
            w = max(4, w // 4 * 4)
        a = id_align(f)
        row = row_bytes(f, w, bpp)
        if variant == "pitch":
            pad_bytes = next(p for p in range(step, 64, step) if (row + p) % a and p >= int(rng.integers(1, 9)))
        elif step:
            pad_bytes = -(-row // a) * a - row + a * int(rng.integers(0, 3))
        if variant in ("hit", "frame", "pitch"):
            align, miss = a, variant == "frame"
        if sampling == LANCZOS and (variant == "hit" or rng.random() < 0.7):
            sampling = int(rng.choice([NEAREST, BILINEAR]))
        dw, dh, sx, sy, px, py = w, h, 1.0, 1.0, 0.0, 0.0
    else:
        dw, dh = dst_dim(rng), dst_dim(rng)
        if rng.random() < 0.5:
            dw = max(4, dw // 4 * 4)
        if kind in ("letterbox", "stretch"):
            r = rng.random()
            if r < 0.15 and 8 * w <= 256 and 8 * h <= 256:
                dw, dh = 8 * w, 8 * h
            elif r < 0.25:
                dw, dh = 1, 1
            sx, sy, px, py = preprocess_affine(0 if kind == "letterbox" else 1, w, h, dw, dh)
        elif kind == "crop":
            s = f32(rng.uniform(1.05, 4.0))
            sx, sy = s, (s if rng.random() < 0.5 else f32(rng.uniform(1.05, 4.0)))
            px, py = -f32(rng.uniform(0.0, w * sx / 2)), -f32(rng.uniform(0.0, h * sy / 2))
        elif kind == "nonuniform":
            sx, sy = f32(np.exp(rng.uniform(np.log(0.1), np.log(8.0)))), f32(np.exp(rng.uniform(np.log(0.1), np.log(8.0))))
            px, py = f32(rng.uniform(-dw / 4, dw / 4)), f32(rng.uniform(-dh / 4, dh / 4))
        elif kind == "fractional":
            sx = sy = f32(rng.uniform(0.3, 3.0))
            px, py = (f32(int(rng.integers(-8, 9)) + float(rng.choice([0.25, 0.5, 0.75, rng.random()]))) for _ in range(2))
        elif kind == "offedge":
            px, py = f32(rng.uniform(0.2, 0.8) * dw), f32(rng.uniform(0.2, 0.8) * dh)
            sx, sy = f32((dw - px) / w * rng.uniform(1.1, 3.0)), f32((dh - py) / h * rng.uniform(1.1, 3.0))
            if rng.random() < 0.5:   # off one edge only
                if rng.random() < 0.5:
                    px, sx = 0.0, f32(dw / w)
                else:
                    py, sy = 0.0, f32(dh / h)
        else:
            (sx, px, tx), (sy, py, ty) = boundary_axis(rng, w, dw), boundary_axis(rng, h, dh)
            kind = f"boundary-{tx}-{ty}"
    pitch = row_bytes(f, w, bpp) + pad_bytes
    need = src_bytes(f, w, h, pitch)
    frames, stride = layout(rng, f, entry if entry != "host" else "strided", batch, need, align, miss)
    f16 = bool(rng.random() < 0.5)
    chunk = host_chunk(need, 3 * dw * dh * (2 if f16 else 4), batch)[0] if entry == "host" else 0
    return Case(f"sweep-{i}", BASE + i, f.code, int(rng.integers(0, 4)) if yuv(f) else 0, bpp, w, h, pitch, kind, f32(sx), f32(sy), f32(px),
                f32(py), dw, dh, sampling, f16, entry, batch, frames, stride, chunk, str(rng.choice(list(NORMS))), float(rng.integers(0, 256)))


N_SWEEP = len(CODES) * len(KINDS)


def edge(name, code, w, h, dw=None, dh=None, *, scale=(1.0, 1.0), pad=(0.0, 0.0), mode=None, sampling=BILINEAR, f16=False, entry="table",
         batch=1, pitch_pad=0, offset=0, gap=0, matrix=0, kind=None):
    """A hand-picked case: frames aligned to 16 bytes plus `offset`, `gap` bytes between them."""
    from oracle.oracle import preprocess_affine
    f = FORMATS[code]
    dw, dh = (w, h) if dw is None else (dw, dh)
    if mode is not None:
        scale, pad = preprocess_affine(mode, w, h, dw, dh)[:2], preprocess_affine(mode, w, h, dw, dh)[2:]
        kind = kind or ("letterbox", "stretch")[mode]
    kind = kind or ("identity" if (dw, dh, scale, pad) == (w, h, (1.0, 1.0), (0.0, 0.0)) else "crop")
    row = row_bytes(f, w, 3)
    pitch = (-(-row // id_align(f)) * id_align(f) if f.family == "bayer" else row) + pitch_pad   # Bayer rows aligned for the identity kernel
    need = src_bytes(f, w, h, pitch)
    stride = -(-need // 16) * 16 + gap
    frames = tuple(offset + k * stride for k in range(batch)) if entry == "table" else (offset,)
    seed = 0xED6E0000 + sum(ord(ch) * 131 ** k for k, ch in enumerate(name)) % 0xFFFF
    chunk = host_chunk(need, 3 * dw * dh * (2 if f16 else 4), batch)[0] if entry == "host" else 0
    return Case(name, seed, code, matrix, 3, w, h, pitch, kind, f32(scale[0]), f32(scale[1]), f32(pad[0]), f32(pad[1]), dw, dh, sampling, f16,
                entry, batch, frames, None if entry == "table" else stride, chunk, "imagenet", 114.0)


def _edges():
    e = []
    # Bayer identity: w = 4 (left and right edge in one thread), h = 3 / 4 / 5 / 9 (the ya == 1 row 0 store, both tails)
    for code in (16, 19, 36, 47, 64, 69, 74):
        for h in (3, 4, 5, 9):
            e.append(edge(f"bayer-identity-{FORMATS[code].name}-4x{h}", code, 4, h, f16=h == 5, entry=("table", "strided", "host")[h % 3]))
    # packed identity: widths whose threads straddle two 8-byte words (8, 24, 36) and do not (4), pitch paddings of 16 and 32
    for code in (65, 70, 75):
        for w, h, pp in ((8, 4, 0), (24, 7, 16), (36, 6, 32)):
            e.append(edge(f"packed-identity-{FORMATS[code].name}-{w}x{h}-p{pp}", code, w, h, pitch_pad=pp, entry="strided"))
    for code in (11, 85, 88):
        for h in (1, 2):
            e.append(edge(f"yuv444-identity-{FORMATS[code].name}-4x{h}", code, 4, h, f16=h == 2, matrix=h))
    e.append(edge("nv12-2x2-letterbox-641x479", 3, 2, 2, 641, 479, mode=0))
    for code in (0, 2, 3, 82, 4, 11, 86, 17, 41, 73):
        e.append(edge(f"one-pixel-{FORMATS[code].name}", code, 7 if FORMATS[code].family not in ("yuv420", "yuv422", "bayer") else 8, 6, 1, 1,
                      mode=1, sampling=(NEAREST, BILINEAR, LANCZOS)[code % 3]))
    # a crop whose sample coordinates hit w and h exactly: (18 + 6) / 1.5 == 16, (9 + 3) / 1.5 == 8
    for code in (3, 6, 80, 0):
        for samp in (NEAREST, BILINEAR):
            e.append(edge(f"crop-hits-edge-{FORMATS[code].name}-{SAMPLING_NAME[samp]}", code, 16, 8, 24, 12, scale=(1.5, 1.5), pad=(-6.0, -3.0),
                          sampling=samp))
    # NV12 / NV21 frames at odd addresses on a fast-kernel geometry: the generic kernel (the fast one reads 16-bit chroma pairs)
    for code in (3, 5):
        e.append(edge(f"odd-frame-{FORMATS[code].name}-table", code, 16, 8, 24, 12, mode=0, offset=1, batch=2))
        e.append(edge(f"odd-frame-{FORMATS[code].name}-strided", code, 16, 8, 24, 12, mode=1, gap=1, entry="strided", batch=3))
    # more than 256 frames: the second launch runs with frame0 > 0
    for name, code, w, h, dw, dh, entry, n in (("nv12-identity", 3, 8, 2, 8, 2, "table", 257), ("bayer8-identity", 18, 4, 3, 4, 3, "strided", 300),
                                               ("i410-identity", 85, 4, 2, 4, 2, "table", 258), ("i444-fast", 11, 4, 2, 8, 4, "table", 260),
                                               ("p010-fast", 80, 4, 2, 12, 3, "strided", 270), ("yv12-fast", 7, 6, 4, 4, 9, "table", 257),
                                               ("rgb-generic", 0, 5, 3, 7, 5, "table", 257), ("bayer12p-generic", 68, 4, 3, 6, 5, "strided", 280),
                                               ("yuyv-generic", 4, 6, 2, 3, 3, "strided", 261)):
        e.append(edge(f"batch{n}-{name}", code, w, h, dw, dh, mode=None if (w, h) == (dw, dh) else 1, entry=entry, batch=n))
    return e


EDGES = {c.name: c for c in _edges()}
assert len(EDGES) == len(_edges()), "edge case names must be unique"


# ── references ─────────────────────────────────────────────────────────────────────────────────────────────────────
def frame_bytes(c, k):
    """Frame k of case c: random bytes; 16-bit Bayer codes below 2^bits; random words (junk in the ignored bits) for 16-bit YUV."""
    f, need = c.fmt, c.need
    rng = np.random.default_rng([c.seed, k])
    if f.family == "bayer" and f.words:
        return rng.integers(0, 1 << f.bits, need // 2, dtype=np.int64).astype("<u2").view(np.uint8)
    return rng.integers(0, 256, need, dtype=np.int64).astype(np.uint8)


def oracle_rgb(c, src, fmt, bpp, pitch, f16):
    from oracle import oracle as o
    d = c.desc(o.PreprocessDesc)
    d.fmt, d.src_bpp, d.src_pitch = fmt, bpp, pitch
    return o.preprocess_frame_desc(src, d, f16)


def reference(c, raw):
    """(3, dh, dw) expected output of one frame: f16 bits, or f32 (Lanczos: always f32, compared within a tolerance)."""
    f, w, h = c.fmt, c.w, c.h
    h16 = c.f16 and c.sampling != LANCZOS
    m = MATRICES[c.matrix]
    rows = raw[:c.pitch * h].reshape(h, c.pitch)[:, :row_bytes(f, w, c.bpp)]
    if f.family in ("rgb", "gray"):
        return oracle_rgb(c, raw, c.code, c.bpp, c.pitch, h16)
    if f.family in ("yuv420", "yuv422") and not f.words:
        tight = raw if f.family == "yuv420" else np.ascontiguousarray(rows).reshape(-1)
        if c.matrix == 0:   # BT.601 limited: the oracle reads NV12 and YUYV itself
            twin = to_twin(tight, w, h, f.layout)
            return oracle_rgb(c, twin, 3 if f.family == "yuv420" else 4, 1 if f.family == "yuv420" else 2, w if f.family == "yuv420" else 2 * w, h16)
        rgb = decode_yuv8(tight, w, h, f.layout, m)
    elif f.code == 11:
        rgb = decode_yuv444(raw, w, h, m)
    elif f.family == "bayer" and not f.words and not f.packed:
        rgb = demosaic8(np.ascontiguousarray(rows), f.layout).astype(np.uint8)
    else:
        if f.family == "bayer":
            samples = np.ascontiguousarray(rows).view("<u2") if f.words else unpack(np.ascontiguousarray(rows), f.bits)
            rgb16 = demosaic16(np.asarray(samples).astype(np.uint16), f.layout)
        else:
            words = torch.from_numpy(raw.view("<u2").astype(np.int32))
            rgb16 = (decode_yuv16 if f.family == "yuv420" else decode_yuv444_16)(words, w, h, f.name, m).numpy()
        mean, inv = NORMS[c.norm]
        return preprocess_rgb16(np.asarray(rgb16).astype(np.uint16), f.bits, (c.scale_x, c.scale_y, c.pad_x, c.pad_y), c.dw, c.dh,
                                SAMPLING_NAME[c.sampling], mean, inv, c.pad_value, h16)
    return oracle_rgb(c, np.ascontiguousarray(rgb), 0, 3, 3 * w, h16)


def compare(got, want, c, what):
    if c.sampling == LANCZOS:
        # host sinf against CUDA's: the oracle's f32 tolerance, scaled with the normalisation's gain, plus for f16 output one
        # f16 step at the expected value (the kernel rounds its own f32 result, which may sit across a binade boundary from the
        # oracle's; Lanczos overshoot passes 256 at gain 255).  At ImageNet gain that is the oracle's 2e-3.
        g = got.view(np.float16 if c.f16 else np.float32).astype(np.float32)
        want = want.reshape(-1).astype(np.float32)
        tol = 1e-4 * max(1.0, max(NORMS[c.norm][1]) / max(IMAGENET_INV)) + (np.spacing(np.abs(want).astype(np.float16)).astype(np.float32)
                                                                             if c.f16 else 0.0)
        over = np.abs(g - want) - tol
        assert over.max() <= 0, f"{what}: error {float(np.abs(g - want)[over.argmax()])} at element {int(over.argmax())} exceeds {float(np.broadcast_to(tol, over.shape)[over.argmax()])}"
    else:
        w = np.ascontiguousarray(want).reshape(-1).view(np.uint8)
        bad = np.flatnonzero(got != w)
        assert bad.size == 0, f"{what}: {bad.size} bytes differ, first at byte {bad[0]}"


# ── the GPU run ─────────────────────────────────────────────────────────────────────────────────────────────────────
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lib(kb):
    return kb._lib.lib()


def run_case(kb, lib, dev, c):
    from kornia_rs_b200._lib import PreprocessDesc
    f = c.fmt
    d = c.desc(PreprocessDesc)
    need = c.need
    assert lib.kb200_preprocess_src_bytes(C.byref(d)) == need, str(c)
    if c.kind in ("letterbox", "stretch"):
        a = (C.c_float * 4)()
        lib.kb200_preprocess_affine(KINDS.index(c.kind), c.w, c.h, c.dw, c.dh, a)
        assert tuple(a) == (c.scale_x, c.scale_y, c.pad_x, c.pad_y), str(c)
    frames = [frame_bytes(c, k) for k in range(c.batch)]
    esz = 2 if c.f16 else 4
    out_elems = 3 * c.dw * c.dh
    nbytes = out_elems * esz * c.batch
    starts = list(c.frames) if c.entry == "table" else [c.frames[0] + k * c.stride for k in range(c.batch)]
    span = starts[-1] + need
    image = np.zeros(span, np.uint8)
    for s, fr in zip(starts, frames):
        image[s:s + need] = fr
    dev_src = Guarded(dev, span).load("u8", image)
    host_src = Guarded(dev, span, host=True).load("u8", image) if c.entry == "host" else None
    fn = {(e, h): getattr(lib, f"kb200_preprocess{'_strided' if e == 'strided' else ''}_{'f16' if h else 'f32'}") for e in ("table", "strided") for h in (0, 1)}

    def device_call(entry, dst):
        if entry == "table":
            ptrs = (C.c_void_p * c.batch)(*[dev_src.ptr + s for s in starts])
            lens = (C.c_size_t * c.batch)(*[need] * c.batch)
            st = fn["table", c.f16](None, C.byref(d), ptrs, lens, c.batch, dst.ptr, out_elems * c.batch)
            return st, expected_kernel(d, [dev_src.ptr + s for s in starts], None, dst.ptr, c.sampling)
        st = fn["strided", c.f16](None, C.byref(d), dev_src.ptr + c.frames[0], dev_src.n - c.frames[0], c.stride, c.batch, dst.ptr, out_elems * c.batch)
        return st, expected_kernel(d, [dev_src.ptr + c.frames[0]], c.stride, dst.ptr, c.sampling)

    outs = []
    runs = [(0, c.planned())] + ([(esz, GENERIC)] if c.sampling != LANCZOS else [])
    for off, want_kernel in runs:
        host = c.entry == "host" and off == 0
        dst = Guarded(dev, nbytes, min(nbytes, 1 << 16), off, host=host).fill(0xFF)
        if host:
            _, src_chunk, dst_chunk = host_chunk(need, out_elems * esz, c.batch)
            pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=src_chunk, dst_chunk_bytes=dst_chunk, depth=2)
            try:
                st = lib.kb200_preprocess_host(pipe._h, None, C.byref(d), host_src.ptr + c.frames[0], host_src.n - c.frames[0], c.stride, c.batch,
                                               dst.ptr, out_elems * c.batch, int(c.f16))
                mirror = c.planned()
                torch.cuda.synchronize()
            finally:
                pipe.close()
        else:
            st, mirror = device_call("table" if c.entry == "table" else "strided", dst)
        assert st == 0, f"{c}: status {st}: {kb._lib.last_error()}"
        ran = kb._lib.last_kernel()
        torch.cuda.synchronize()
        assert ran == want_kernel == mirror, f"{c}: dst +{off} B ran {ran}, the dispatch mirror says {mirror}, the case plans {want_kernel}"
        lead, tail = dst.guards()
        for what, g in (("lead", lead), ("tail", tail)):
            bad = np.flatnonzero(g != 0xFF)
            assert bad.size == 0, f"{c}: dst +{off} B: {bad.size} bytes written in the {what} guard"
        outs.append(dst.out())
    ones = outs[0].view(np.uint16 if c.f16 else np.uint32) == (0xFFFF if c.f16 else 0xFFFFFFFF)
    assert not ones.any(), f"{c}: {int(ones.sum())} output elements left unwritten (first {int(np.flatnonzero(ones)[0])})"
    fb = out_elems * esz
    check = range(c.batch) if c.batch <= 4 else sorted({0, 1, 255, 256, c.batch - 1})
    for k in check:
        compare(outs[0][k * fb:(k + 1) * fb], reference(c, frames[k]), c, f"{c}: frame {k} differs from the reference")
    if len(outs) == 2:
        bad = np.flatnonzero(outs[0] != outs[1])
        assert bad.size == 0, f"{c}: {c.planned()} and {GENERIC} differ in {bad.size} bytes, first at byte {bad[0]} (frame {bad[0] // fb})"


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_SWEEP))
def test_sweep(kb, lib, dev, i):
    run_case(kb, lib, dev, case(i))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGES))
def test_edge(kb, lib, dev, name):
    run_case(kb, lib, dev, EDGES[name])


# ── what the sweep covers (CPU) ─────────────────────────────────────────────────────────────────────────────────────
def straddles(bits, w):
    """A packed identity thread at column x reads bits / 2 bytes from x * bits / 8: past its 8-byte word at some x."""
    return any(((x * bits // 8) & 7) + bits // 2 > 8 for x in range(0, w, 4))


def test_sweep_coverage():
    cases = [case(i) for i in range(N_SWEEP)] + list(EDGES.values())
    assert len({c.name for c in cases}) == len(cases)
    kernels, samplers, matrices, kinds = defaultdict(set), defaultdict(set), defaultdict(set), set()
    entries, outs, dst_w4, fast_h8, split = set(), set(), set(), set(), set()
    bayer_id = defaultdict(set)
    for c in cases:
        f = c.fmt
        k = c.planned()
        assert c.planned(dst=16 + (2 if c.f16 else 4)) == GENERIC or c.entry == "host"
        kernels[c.code].add(k)
        samplers[group(f)].add(c.sampling)
        if yuv(f):
            matrices[group(f)].add(c.matrix)
        kinds.add(c.kind.split("-")[0])
        entries.add(c.entry)
        outs.add(c.f16)
        dst_w4.add(c.dw % 4)
        if k == f.fast:
            fast_h8.add(c.dh % 8)
        if c.batch > 256:
            split.add("identity" if k == f.identity else "fast" if k == f.fast else "generic")
        if f.family == "bayer" and k == f.identity:
            t = group(f)
            bayer_id[t] |= {f"h{c.h % 2}", *(["h=3"] if c.h == 3 else []), *(["w=4"] if c.w == 4 else [])}
            if f.packed and straddles(f.bits, c.w):
                bayer_id[t].add("straddle")
    for code, f in FORMATS.items():
        assert kernels[code] == {k for k in (f.identity, f.fast, GENERIC) if k}, f"{f.name}: ran {sorted(kernels[code])}"
    for g in {group(f) for f in FORMATS.values()}:
        assert samplers[g] == {NEAREST, BILINEAR, LANCZOS}, g
    for g in {group(f) for f in FORMATS.values() if yuv(f)}:
        assert matrices[g] == {0, 1, 2, 3}, g
    assert kinds == {k.split("-")[0] for k in KINDS}, kinds
    assert entries == set(ENTRIES) and outs == {False, True}
    assert dst_w4 == {0, 1, 2, 3}
    assert fast_h8 == set(range(8)), fast_h8
    assert split == {"identity", "fast", "generic"}, split
    for t in ("bayer8", "bayer16", "bayer10p", "bayer12p", "bayer14p"):
        want = {"h0", "h1", "h=3", "w=4"} | ({"straddle"} if t.endswith("p") else set())
        assert bayer_id[t] >= want, (t, bayer_id[t])
