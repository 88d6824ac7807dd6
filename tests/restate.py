"""The suite's independent restatements and format facts: pure numpy / torch, no device and no library handle.

The source-format table (preprocess.cu's SRC_FORMATS) and the preprocess sweep's cases, the Bayer demosaic and MIPI
packing, the YUV layouts and their Q20 / Q16 decodes, the f32 restatement of the oracle's preprocess for 16-bit RGB, the
region / warp / remap references, and the host mirrors of the dispatch rules the tests assert.  Every test module and
every tools/*_bench.py reads these from here; a helper that only one test module uses stays in that module.
"""
import ctypes as C
import math
from dataclasses import dataclass, replace

import numpy as np
import torch

# ── Bayer patterns ──
PATTERNS = ("RGGB", "BGGR", "GRBG", "GBRG")
PATTERN_CODE = {p: i for i, p in enumerate(PATTERNS)}                  # kb200_bayer_pattern
R_AT = {"RGGB": (0, 0), "BGGR": (1, 1), "GRBG": (1, 0), "GBRG": (0, 1)}   # (column, row) parity of the R site
DEPTHS = (10, 12, 14, 16)

# ── the preprocess sweep's vocabulary ──
BASE = 0x5EED0000
GENERIC = "preprocess_generic_kernel"
NEAREST, BILINEAR, LANCZOS = 0, 1, 3
SAMPLING_NAME = {NEAREST: "Nearest", BILINEAR: "Bilinear", LANCZOS: "Lanczos"}
ENTRIES = ("table", "strided", "host")
KINDS = ("letterbox", "stretch", "identity", "identity-miss", "crop", "nonuniform", "fractional", "offedge", "boundary")
F32 = np.float32
IMAGENET_INV = tuple(float(F32(1.0) / F32(s)) for s in (0.229, 0.224, 0.225))
NORMS = {"imagenet": ((0.485, 0.456, 0.406), IMAGENET_INV), "unit": ((0.0,) * 3, (1.0,) * 3), "scale255": ((0.0,) * 3, (255.0,) * 3)}


# ── the source formats: preprocess.cu's SRC_FORMATS ──
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


# ── the dispatch rule, restated (preprocess.cu launch_preprocess) ──
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


# ── the preprocess sweep's cases ──
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


# ── the sweep's frames and the oracle on a case's descriptor ──
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


# ── Bayer mosaics: 16-bit names, the demosaic, MIPI CSI-2 packing ──
def fmt_name(pattern, bits):
    return f"Bayer{pattern.capitalize()}{bits}"


def white(bits):
    return (1 << bits) - 1


def demosaic(raw, pattern):
    """bayer.cuh's demosaic (cv2's COLOR_Bayer??2RGB): numpy arrays or torch tensors [..., h, w] -> [..., h, w, 3] of the
    input's dtype.  The sums are int32: 4 * 65535 + 2 does not fit 16 bits."""
    is_t = isinstance(raw, torch.Tensor)
    h, w = raw.shape[-2:]
    p = raw.to(torch.int32) if is_t else raw.astype(np.int32)
    rx, ry = R_AT[pattern]
    ar = (lambda n: torch.arange(n, device=raw.device)) if is_t else np.arange
    cx, cy = ar(w).clip(1, w - 2), ar(h).clip(1, h - 2)

    def at(dy, dx):
        return p[..., cy + dy, :][..., cx + dx]

    c, n, s, wv, e = at(0, 0), at(-1, 0), at(1, 0), at(0, -1), at(0, 1)
    d = at(-1, -1) + at(-1, 1) + at(1, -1) + at(1, 1)
    g4, d4, h2, v2 = (n + s + wv + e + 2) >> 2, (d + 2) >> 2, (wv + e + 1) >> 1, (n + s + 1) >> 1
    px, py = (cx & 1)[None, :], (cy & 1)[:, None]
    rsite, bsite = (px == rx) & (py == ry), (px != rx) & (py != ry)
    grow = ~rsite & ~bsite & (py == ry)    # a G on an R row has R left and right
    where = torch.where if is_t else np.where
    r = where(rsite, c, where(bsite, d4, where(grow, h2, v2)))
    b = where(bsite, c, where(rsite, d4, where(grow, v2, h2)))
    g = where(rsite | bsite, g4, c)
    out = (torch.stack if is_t else np.stack)([r, g, b], -1)
    return out.to(raw.dtype) if is_t else out.astype(raw.dtype)


# ── the oracle's ko_preprocess_frame restated for interleaved 16-bit RGB with a white level ──
# Op for op in f32 (numpy rounds every operation; nothing is fused): plan_pixel, the three samplers, then
# o = (px / W - mean) * inv_std inside the content, (pad / 255 - mean) * inv_std on the pad.
def _lanczos_w(dd):
    ad = np.abs(dd)
    pd = F32(3.14159265358979) * dd
    with np.errstate(divide="ignore", invalid="ignore"):
        v = F32(3.0) * np.sin(pd) * np.sin(pd / F32(3.0)) / (pd * pd)
    return np.where(ad < F32(1e-6), F32(1.0), np.where(ad >= F32(3.0), F32(0.0), v)).astype(F32)


def preprocess_rgb16(rgb, bits, affine, dw, dh, sampling, mean, inv_std, pad_value, f16=False):
    """rgb: (h, w, 3) uint16 -> (3, dh, dw) f32 (or f16 bits rounded to nearest even)."""
    h, w = rgb.shape[:2]
    sxs, sys_, padx, pady = (F32(v) for v in affine)
    src = rgb.astype(F32)
    sx = np.broadcast_to((np.arange(dw, dtype=F32) - padx) / sxs, (dh, dw))
    sy = np.broadcast_to(((np.arange(dh, dtype=F32) - pady) / sys_)[:, None], (dh, dw))
    inside = ~((sx < 0) | (sy < 0) | (sx >= F32(w)) | (sy >= F32(h)))

    def tap(yi, xi):
        return src[np.clip(yi, 0, h - 1), np.clip(xi, 0, w - 1)]

    if sampling == "Nearest":
        def roundf(v):
            f = np.floor(v)
            return (f + (v - f >= F32(0.5))).astype(np.int64)
        px = tap(np.clip(roundf(sy), 0, h - 1), np.clip(roundf(sx), 0, w - 1))
    elif sampling == "Bilinear":
        x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
        ax, ay = (sx - x0.astype(F32))[..., None], (sy - y0.astype(F32))[..., None]
        x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
        x0, y0 = np.maximum(x0, 0), np.maximum(y0, 0)
        t00, t10, t01, t11 = tap(y0, x0), tap(y0, x1), tap(y1, x0), tap(y1, x1)
        top = t00 + (t10 - t00) * ax
        bot = t01 + (t11 - t01) * ax
        px = top + (bot - top) * ay
    else:
        x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
        acc = np.zeros((dh, dw, 3), F32)
        wsum = np.zeros((dh, dw), F32)
        for j in range(-2, 4):
            yj = y0 + j
            wy = _lanczos_w(sy - yj.astype(F32))
            for i in range(-2, 4):
                xi = x0 + i
                wt = wy * _lanczos_w(sx - xi.astype(F32))
                acc = acc + wt[..., None] * tap(yj, xi)
                wsum = wsum + wt
        with np.errstate(divide="ignore", invalid="ignore"):
            px = acc / wsum[..., None]
    q = np.where(inside[..., None], px / F32(white(bits)), F32(pad_value) / F32(255.0))
    o = ((q - np.asarray(mean, F32)) * np.asarray(inv_std, F32)).astype(F32).transpose(2, 0, 1)
    return np.ascontiguousarray(o.astype(np.float16) if f16 else o)


GROUP = {10: 4, 12: 2, 14: 4}          # samples per group
GROUP_BYTES = {10: 5, 12: 3, 14: 7}    # bytes per group


def pack(samples, bits):
    """[..., h, w] samples < 2^bits (numpy) -> [..., h, w*bits/8] uint8, each row packed on its own."""
    g, gb, lo = GROUP[bits], GROUP_BYTES[bits], bits - 8
    v = np.asarray(samples).astype(np.int64)
    *lead, w = v.shape
    assert w % g == 0
    v = v.reshape(*lead, w // g, g)
    field = np.zeros(v.shape[:-1], np.int64)
    for j in range(g):
        field |= (v[..., j] & ((1 << lo) - 1)) << (lo * j)
    lo_bytes = np.stack([(field >> (8 * i)) & 0xFF for i in range(gb - g)], -1)
    return np.concatenate([v >> lo, lo_bytes], -1).astype(np.uint8).reshape(*lead, w // g * gb)


def unpack(raw, bits):
    """[..., h, w*bits/8] uint8 (numpy array or torch tensor) -> [..., h, w] samples (int32)."""
    g, gb, lo = GROUP[bits], GROUP_BYTES[bits], bits - 8
    is_t = isinstance(raw, torch.Tensor)
    b = raw.to(torch.int32) if is_t else raw.astype(np.int32)
    *lead, nb = b.shape
    b = b.reshape(*lead, nb // gb, gb)
    field = b[..., g] * 0
    for i in range(gb - g):
        field = field | (b[..., g + i] << (8 * i))
    out = (torch.stack if is_t else np.stack)([(b[..., j] << lo) | ((field >> (lo * j)) & ((1 << lo) - 1)) for j in range(g)], -1)
    return out.reshape(*lead, nb // gb * g)


# ── YUV layouts: repacking to the NV12 / YUYV twin ──
L420 = ("Nv21", "I420", "Yv12")
L422 = ("Uyvy", "Yvyu")
# byte positions of (Y0, U, Y1, V) in a 4:2:2 word; YUYV is (0, 1, 2, 3)
WORD = {"Yuyv": (0, 1, 2, 3), "Uyvy": (1, 0, 3, 2), "Yvyu": (0, 3, 2, 1)}


def _cat(parts):
    return torch.cat(parts, -1) if isinstance(parts[0], torch.Tensor) else np.concatenate(parts, -1)


def _interleave(a, b):
    st = torch.stack((a, b), -1) if isinstance(a, torch.Tensor) else np.stack((a, b), -1)
    return st.reshape(*a.shape[:-1], -1)


def yuv420_to_nv12(raw, w, h, layout):
    """A 4:2:0 frame in `layout` -> its NV12 twin."""
    y, c, q = raw[..., :w * h], raw[..., w * h:], (w // 2) * (h // 2)
    if layout == "Nv12":
        return raw
    if layout == "Nv21":
        return _cat([y, _interleave(c[..., 1::2], c[..., 0::2])])
    u, v = (c[..., :q], c[..., q:]) if layout == "I420" else (c[..., q:], c[..., :q])
    return _cat([y, _interleave(u, v)])


def nv12_to_yuv420(nv12, w, h, layout):
    """An NV12 frame -> the same picture in `layout`."""
    y, u, v = nv12[..., :w * h], nv12[..., w * h::2], nv12[..., w * h + 1::2]
    if layout == "Nv21":
        return _cat([y, _interleave(v, u)])
    return _cat([y, u, v]) if layout == "I420" else _cat([y, v, u])


def yuv422_swap(raw, layout):
    """YUYV <-> `layout` (each permutation is its own inverse)."""
    words = raw.reshape(*raw.shape[:-1], -1, 4)
    idx = list(WORD[layout])
    return words[..., idx].reshape(raw.shape)


def to_twin(raw, w, h, layout):
    return yuv420_to_nv12(raw, w, h, layout) if layout in L420 + ("Nv12",) else yuv422_swap(raw, layout)


def layout_bytes(layout, w, h):
    return w * h * 3 // 2 if layout in L420 + ("Nv12",) else w * h * 2


def decode_direct(raw, w, h, layout):
    """One frame in `layout` -> [h, w, 3] RGB8 with the BT.601-limited decode of NV12 / YUYV, reading the layout directly."""
    return decode_yuv8(raw, w, h, layout, "Bt601Limited")


def expected_decode_kernel(layout, w, h, n, src_off, dst_off):
    name = layout.lower()
    aligned = src_off % 16 == 0 and dst_off % 16 == 0
    if layout in L420 + ("Nv12",):
        vec = w % 16 == 0 and aligned and (w * h * 3 // 2) % 16 == 0
    else:
        vec = aligned and (w * h * n) % 16 == 0   # otherwise the generic kernel runs last (for the tail, or for all)
    return f"rgb_from_{name}_{'vec16' if vec else 'generic'}"


# ── YUV matrices: Q20 for bytes, Q16 for 10- and 12-bit codes ──
MATRICES = ("Bt601Limited", "Bt601Full", "Bt709Limited", "Bt709Full")   # kb200_yuv_matrix order
YUV420 = ("Nv12",) + L420
TABLE = {
    "Bt601Limited": (16, 1220542, 1673527, 2116026, -409993, -852492),
    "Bt601Full": (0, 1048576, 1470104, 1858077, -360853, -748826),
    "Bt709Limited": (16, 1220945, 1879825, 2215014, -223607, -558796),
    "Bt709Full": (0, 1048576, 1651297, 1945738, -196424, -490864),
}


KR_KB = {"Bt601": (0.299, 0.114), "Bt709": (0.2126, 0.0722)}


def q20(y, u, v, m):
    """The Q20 decode of byte arrays y, u, v with matrix m -> [..., 3] RGB8."""
    yo, cy, cvr, cub, cug, cvg = TABLE[m]
    yy = np.maximum(y.astype(np.int64) - yo, 0) * cy
    u, v = u.astype(np.int64) - 128, v.astype(np.int64) - 128
    r = (yy + cvr * v + (1 << 19)) >> 20
    g = (yy + cug * u + cvg * v + (1 << 19)) >> 20
    b = (yy + cub * u + (1 << 19)) >> 20
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode_yuv8(raw, w, h, layout, m):
    """One frame in `layout` -> [h, w, 3] RGB8 through q20, reading the layout directly (chroma replicated)."""
    if layout in YUV420:
        y, c, q = raw[:w * h].reshape(h, w), raw[w * h:], (w // 2) * (h // 2)
        if layout in ("Nv12", "Nv21"):
            pairs = c.reshape(h // 2, w // 2, 2)
            u, v = (pairs[..., 0], pairs[..., 1]) if layout == "Nv12" else (pairs[..., 1], pairs[..., 0])
        else:
            first, second = c[:q].reshape(h // 2, w // 2), c[q:].reshape(h // 2, w // 2)
            u, v = (first, second) if layout == "I420" else (second, first)
        up = lambda a: np.repeat(np.repeat(a, 2, 0), 2, 1)
        return q20(y, up(u), up(v), m)
    words = raw.reshape(h, w // 2, 4)
    y0, u, y1, v = (words[..., i] for i in WORD.get(layout, (0, 1, 2, 3)))
    return q20(np.stack([y0, y1], -1).reshape(h, w), np.repeat(u, 2, 1), np.repeat(v, 2, 1), m)


TABLE16 = {
    10: {"Bt601Limited": (64, 76533, 104905, 132590, -25750, -53435), "Bt601Full": (0, 65536, 91881, 116130, -22553, -46802),
         "Bt709Limited": (64, 76533, 117835, 138846, -14017, -35027), "Bt709Full": (0, 65536, 103206, 121609, -12276, -30679)},
    12: {"Bt601Limited": (256, 76590, 104982, 132687, -25769, -53475), "Bt601Full": (0, 65536, 91881, 116130, -22553, -46802),
         "Bt709Limited": (256, 76590, 117921, 138947, -14027, -35053), "Bt709Full": (0, 65536, 103206, 121609, -12276, -30679)},
}


BITS = {"P010": 10, "P012": 12, "I010": 10, "I012": 12, "I444": 8, "I410": 10, "I412": 12, "I410Msb": 10, "I412Msb": 12}


def q16(y, u, v, m, bits):
    """The Q16 decode of n-bit code tensors y, u, v with matrix m -> [..., 3] int64 codes 0..W."""
    yo, cy, cvr, cub, cug, cvg = TABLE16[bits][m]
    half = 1 << (bits - 1)
    yy = (y - yo).clamp(min=0) * cy
    u, v = u - half, v - half
    r = (yy + cvr * v + (1 << 15)) >> 16
    g = (yy + cug * u + cvg * v + (1 << 15)) >> 16
    b = (yy + cub * u + (1 << 15)) >> 16
    return torch.stack([r, g, b], -1).clamp(0, white(bits))


def codes(words, fmt):
    """16-bit words -> their n-bit codes (int64): the high bits of a P01x or I41xMsb word, the low bits of an I01x or I41x
    word."""
    wd = words.to(torch.int32).to(torch.int64) & 0xFFFF
    bits = BITS[fmt]
    return wd >> (16 - bits) if fmt[0] == "P" or fmt.endswith("Msb") else wd & white(bits)


def decode_yuv16(raw, w, h, fmt, m):
    """Frames [..., w*h*3/2] of 16-bit words -> [..., h, w, 3] int64, reading the layout directly (chroma replicated)."""
    c = codes(raw, fmt)
    lead = c.shape[:-1]
    y, ch, q = c[..., :w * h].reshape(*lead, h, w), c[..., w * h:], (w // 2) * (h // 2)
    u, v = (ch[..., 0::2], ch[..., 1::2]) if fmt[0] == "P" else (ch[..., :q], ch[..., q:])

    def up(a):
        return a.reshape(*lead, h // 2, w // 2).repeat_interleave(2, -2).repeat_interleave(2, -1)

    return q16(y, up(u), up(v), m, BITS[fmt])


def decode_yuv444_16(raw, w, h, fmt, m):
    """Frames [..., 3*w*h] of 16-bit words -> [..., h, w, 3] int64, each pixel from its own Y, U, V."""
    c = codes(raw, fmt)
    lead = c.shape[:-1]
    y, u, v = (c[..., k * w * h:(k + 1) * w * h].reshape(*lead, h, w) for k in range(3))
    return q16(y, u, v, m, BITS[fmt])


def decode_yuv444(raw, w, h, m):
    """One I444 frame (numpy bytes, 3*w*h) -> [h, w, 3] RGB8."""
    y, u, v = (raw[k * w * h:(k + 1) * w * h].reshape(h, w) for k in range(3))
    return q20(y, u, v, m)


# ── region, warp and remap references ──
OUTS = ("f32", "f16", "bf16")
ESZ = {"f32": 4, "f16": 2, "bf16": 2}


@dataclass(frozen=True)
class RCase:
    base: Case                # format, frame geometry, sampler, normalisation, pad value, dst size (f16 unused)
    mode: int
    out: str
    n_frames: int
    offsets: tuple            # each frame's byte offset in one allocation (16-B aligned base)
    rois: tuple               # (k, x, y, w, h)

    def __str__(self):
        c = self.base
        r = self.rois if len(self.rois) <= 6 else self.rois[:6] + ("...",)
        return (f"{c.name}: {c.fmt.name} matrix {c.matrix} bpp {c.bpp} {c.w}x{c.h} pitch {c.pitch} -> {c.dw}x{c.dh} mode {self.mode} "
                f"{SAMPLING_NAME[c.sampling]} {self.out} norm {c.norm} pad {c.pad_value} frames {self.offsets} rois {r}")


def place(rng, f, need, n, odd=False):
    """Frame offsets: even (and element-aligned), gaps between frames; `odd`: one frame of a byte format at an odd address."""
    e = max(2, elem_align(f))
    offs, at = [], 16
    for _ in range(n):
        at = -(-at // e) * e + e * int(rng.integers(0, 8))
        offs.append(at)
        at += need + e * int(rng.integers(1, 8))
    if odd and elem_align(f) == 1:
        k = int(rng.integers(0, n))
        offs[k] += 1 - offs[k] % 2
    return tuple(offs)


def picture(c, raw):
    """Frame `raw` of case c decoded: (8, (h, w, 3) uint8) or (bits, (h, w, 3) uint16)."""
    f, w, h = c.fmt, c.w, c.h
    m = MATRICES[c.matrix]
    rows = raw[:c.pitch * h].reshape(h, c.pitch)[:, :row_bytes(f, w, c.bpp)]
    if f.family == "gray":
        return 8, np.repeat(np.ascontiguousarray(rows)[:, :, None], 3, axis=2)
    if f.family == "rgb":
        px = np.ascontiguousarray(rows).reshape(h, w, c.bpp)[:, :, :3]
        return 8, np.ascontiguousarray(px if f.code == 0 else px[:, :, ::-1])
    if f.family in ("yuv420", "yuv422") and not f.words:
        tight = raw if f.family == "yuv420" else np.ascontiguousarray(rows).reshape(-1)
        return 8, np.asarray(decode_yuv8(tight, w, h, f.layout, m)).astype(np.uint8).reshape(h, w, 3)
    if f.code == 11:
        return 8, np.asarray(decode_yuv444(raw, w, h, m)).astype(np.uint8).reshape(h, w, 3)
    if f.family == "bayer" and not f.words and not f.packed:
        return 8, demosaic(np.ascontiguousarray(rows), f.layout).astype(np.uint8)
    if f.family == "bayer":
        samples = np.ascontiguousarray(rows).view("<u2") if f.words else unpack(np.ascontiguousarray(rows), f.bits)
        return f.bits, np.asarray(demosaic(np.asarray(samples).astype(np.uint16), f.layout)).astype(np.uint16)
    words = torch.from_numpy(raw.view("<u2").astype(np.int32))
    rgb16 = (decode_yuv16 if f.family == "yuv420" else decode_yuv444_16)(words, w, h, f.name, m).numpy()
    return f.bits, np.asarray(rgb16).astype(np.uint16).reshape(h, w, 3)


def region_reference(rc, pic, roi):
    """(3, dh, dw) of region roi: f32, or f16 bits for f16 output (Lanczos: f32, compared within a tolerance)."""
    from oracle.oracle import preprocess_affine
    c = rc.base
    bits, arr = pic
    _, x, y, w, h = roi
    sx, sy, px, py = preprocess_affine(rc.mode, w, h, c.dw, c.dh)
    h16 = rc.out == "f16" and c.sampling != LANCZOS
    crop = np.ascontiguousarray(arr[y:y + h, x:x + w])
    if bits == 8:
        cc = replace(c, w=w, h=h, pitch=3 * w, scale_x=sx, scale_y=sy, pad_x=px, pad_y=py)
        return oracle_rgb(cc, crop.reshape(-1), 0, 3, 3 * w, h16)
    mean, inv = NORMS[c.norm]
    return preprocess_rgb16(crop, bits, (sx, sy, px, py), c.dw, c.dh, SAMPLING_NAME[c.sampling], mean, inv, c.pad_value, h16)


def forward_of(inv):
    """The forward map (float32, row-major 9) whose float64 inverse is `inv` (3x3)."""
    return tuple(float(v) for v in np.linalg.inv(np.asarray(inv, np.float64)).astype(F32).reshape(-1))


def draw_map(rng, kind, w, h, dw, dh):
    """One forward map of `kind` for a w x h frame and a dw x dh output."""
    if kind in ("similarity", "perspective", "rot90"):
        ang = float(rng.uniform(-np.pi, np.pi)) if kind != "rot90" else float(np.pi / 2 * rng.integers(1, 4))
        s = float(np.exp(rng.uniform(np.log(0.25), np.log(4.0))))
        # frame point the output centre lands on: usually inside, sometimes past an edge
        c = (float(rng.uniform(-0.3, 1.3) * w), float(rng.uniform(-0.3, 1.3) * h))
        if kind == "rot90":   # get_rotation_matrix2d's float cos / sin: a ~1e-8 step on the axis it turns away, the degenerate rule
            a, b = F32(np.cos(ang)) * F32(s), F32(np.sin(ang)) * F32(s)
            m = [a, b, F32(dw / 2) - a * F32(c[0]) - b * F32(c[1]), -b, a, F32(dh / 2) + b * F32(c[0]) - a * F32(c[1]), 0, 0, 1]
            return tuple(float(F32(v)) for v in m)
        r = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]]) / s   # output -> frame
        inv = np.eye(3)
        inv[:2, :2] = r
        inv[:2, 2] = np.array(c) - r @ np.array([dw / 2, dh / 2])
        if kind == "perspective":
            p = np.eye(3)
            p[2, :2] = rng.uniform(-0.03, 0.03, 2)
            inv = inv @ p
            if rng.random() < 0.2:   # an inverse of tiny scale: |w| < 1e-10 at every pixel, all pad
                return tuple(float(F32(v) * F32(1e12)) for v in forward_of(inv))
        return forward_of(inv)
    if kind == "affine":
        inv = np.eye(3)
        inv[:2, :2] = rng.uniform(-2.0, 2.0, (2, 2))
        while abs(np.linalg.det(inv[:2, :2])) < 0.05:
            inv[:2, :2] = rng.uniform(-2.0, 2.0, (2, 2))
        inv[:2, 2] = rng.uniform(-0.5, 1.5, 2) * (w, h)
        return forward_of(inv)
    if kind == "edges":
        # a translation (or an x2 upscale, half-integer samples: nearest's ties) that puts column / row 0 of the output on
        # 0, W - 1, the float below W or W
        tx = [0.0, w - 1.0, float(np.nextafter(F32(w), F32(0))), float(w)][int(rng.integers(0, 4))]
        ty = [0.0, h - 1.0, float(np.nextafter(F32(h), F32(0))), float(h)][int(rng.integers(0, 4))]
        if rng.random() < 0.5:
            tx, ty = (float(-rng.integers(0, dw)) + tx, ty) if rng.random() < 0.5 else (tx, float(-rng.integers(0, dh)) + ty)
        s = 2.0 if rng.random() < 0.3 else 1.0
        return (s, 0.0, -s * tx, 0.0, s, -s * ty, 0.0, 0.0, 1.0)
    if kind == "wzero":
        # w = x - c exactly (c a power of two): |w| < 1e-10 on column c, negative left of it
        c = float(2 ** int(rng.integers(0, max(1, int(np.log2(max(dw - 1, 1))) + 1))))
        t = rng.uniform(-0.5, 0.5, 2) * (w, h)
        return (1.0, 0.0, float(F32(t[0])), 0.0, 1.0, float(F32(t[1])), 1.0 / c, 0.0, -1.0 / c) if rng.random() < 0.5 else \
            (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 1.0 / c, 0.0, -1.0 / c)
    if kind == "wcross":
        inv = np.eye(3)
        inv[:2, :2] = rng.uniform(-1.5, 1.5, (2, 2))
        inv[:2, 2] = rng.uniform(0, 1, 2) * (w, h)
        gx, gy = rng.uniform(-2, 2, 2) / (dw, dh)
        inv[2] = (gx, gy, -(gx * rng.uniform(0, dw) + gy * rng.uniform(0, dh)) + rng.uniform(-1e-3, 1e-3))
        if abs(np.linalg.det(inv)) < 1e-6:
            inv[2, 2] += 0.5
        return forward_of(inv)
    # "tiny": a map whose output is a few frame pixels, and the frame's corner regions
    s = float(rng.choice([0.125, 0.25, 8.0]))
    return (s, 0.0, -s * float(rng.integers(-2, w + 2)), 0.0, s, -s * float(rng.integers(-2, h + 2)), 0.0, 0.0, 1.0)


def warp_coords(inv, persp, dw, dh, w, h):
    """warp_coord on inverse `inv` over a dw x dh output: (sx, sy, inside, |w| < 1e-10 mask), float32."""
    x = np.arange(dw, dtype=F32)[None, :]
    y = np.arange(dh, dtype=F32)[:, None]
    m = inv.reshape(-1)
    with np.errstate(all="ignore"):
        if persp:
            ww = (m[6] * x + m[7] * y) + m[8]
            small = np.abs(ww) < F32(1e-10)
            sx = ((m[0] * x + m[1] * y) + m[2]) / ww
            sy = ((m[3] * x + m[4] * y) + m[5]) / ww
            inside = ~small & (sx >= 0) & (sx < F32(w)) & (sy >= 0) & (sy < F32(h))
        else:
            sx0 = np.broadcast_to(m[1] * y + m[2], (dh, dw))
            sy0 = np.broadcast_to(m[4] * y + m[5], (dh, dw))
            sx = m[0] * x + sx0
            sy = m[3] * x + sy0
            ax = sx0 if abs(m[0]) < F32(1e-6) else sx
            ay = sy0 if abs(m[3]) < F32(1e-6) else sy
            inside = (ax >= 0) & (ax < F32(w)) & (ay >= 0) & (ay < F32(h))
            small = np.zeros((dh, dw), bool)
    return sx.astype(F32), sy.astype(F32), inside, small


def warp_reference(pic, inv, persp, dw, dh, sampling, norm, pad_value, out):
    """(3, dh, dw) of one region: f32, or f16 bits for f16 output."""
    h, w = pic[1].shape[:2]
    sx, sy, inside, _ = warp_coords(inv, persp, dw, dh, w, h)
    return sample_reference(pic, sx, sy, inside, sampling, norm, pad_value, out)


def sample_reference(pic, sx, sy, inside, sampling, norm, pad_value, out):
    """(3, dh, dw) sampled at frame coordinates (sx, sy) where `inside`, the pad value elsewhere."""
    bits, arr = pic
    h, w = arr.shape[:2]
    # the degenerate-axis clamp: [0, the float below W]; it moves no other inside coordinate
    sx = np.where(inside, np.minimum(np.maximum(sx, F32(0)), np.nextafter(F32(w), F32(0))), F32(0))
    sy = np.where(inside, np.minimum(np.maximum(sy, F32(0)), np.nextafter(F32(h), F32(0))), F32(0))
    t = arr.astype(F32)
    fx, fy = np.floor(sx), np.floor(sy)
    if sampling == NEAREST:   # roundf: half away from zero, here on s >= 0
        xn = np.clip(fx.astype(np.int64) + (sx - fx >= F32(0.5)), 0, w - 1)
        yn = np.clip(fy.astype(np.int64) + (sy - fy >= F32(0.5)), 0, h - 1)
        px = t[yn, xn]
    else:
        ax, ay = (sx - fx)[..., None], (sy - fy)[..., None]
        x0, y0 = np.maximum(fx.astype(np.int64), 0), np.maximum(fy.astype(np.int64), 0)
        x1, y1 = np.minimum(fx.astype(np.int64) + 1, w - 1), np.minimum(fy.astype(np.int64) + 1, h - 1)
        top = t[y0, x0] + (t[y0, x1] - t[y0, x0]) * ax   # a zero weight adds exactly 0: the tap not read
        bot = t[y1, x0] + (t[y1, x1] - t[y1, x0]) * ax
        px = top + (bot - top) * ay
    mean, inv_std = (np.array(v, F32) for v in NORMS[norm])
    q = px / F32(255 if bits == 8 else (1 << bits) - 1)
    o = (q - mean) * inv_std
    padv = (F32(pad_value) / F32(255) - mean) * inv_std
    o = np.where(inside[..., None], o, padv).astype(F32).transpose(2, 0, 1)
    return np.ascontiguousarray(o.astype(np.float16) if out == "f16" else o)


def make_case(name, seed, code, matrix, bpp, w, h, pitch, dw, dh, sampling, norm, pad_value):
    return Case(name, seed, code, matrix, bpp, w, h, pitch, "warp", 1.0, 1.0, 0.0, 0.0, dw, dh, sampling, False, "table", 1, (), None, 0, norm,
                pad_value)


def smooth_rgb(w, h, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    chans = []
    for _ in range(3):
        a, b, p, q = rng.uniform(0.02, 0.08, 4)
        chans.append(127.5 + 60 * np.sin(a * x + b * y + p * 10) + 50 * np.cos(q * x - a * y))
    return np.clip(np.rint(np.stack(chans, axis=2)), 0, 255).astype(np.uint8)


def inside_of(mx, my, w, h):
    with np.errstate(invalid="ignore"):
        return (mx >= 0) & (mx < F32(w)) & (my >= 0) & (my < F32(h))


def remap_reference(pic, mx, my, sampling, norm, pad_value, out):
    """(3, dh, dw) of one region through the map (mx, my) (float32 [dh, dw]): f32, or f16 bits for f16 output."""
    h, w = pic[1].shape[:2]
    with np.errstate(invalid="ignore"):
        return sample_reference(pic, mx, my, inside_of(mx, my, w, h), sampling, norm, pad_value, out)


# ── host mirrors of the dispatchers ──
@dataclass
class Schedule:
    mode: str             # fused: POINT / BOX / YZERO / GENERAL, or "gather" when the staged kernel declines
    npx: int = 0
    stages: int = 0
    per_sm: int = 0
    tiles_x: int = 0
    rows_per_chunk: int = 0
    chunks_y: int = 0
    nunits: int = 0
    grid: int = 0
    dtx: int = 0
    dcy: int = 0
    dimg: int = 0
    dh: int = 0

    @property
    def staged(self):
        return self.mode != "gather"

    @property
    def units_per_cta(self):
        return -(-self.nunits // self.grid)

    @property
    def ragged(self):
        """The last chunk of every image is shorter than the others."""
        return self.dh % self.rows_per_chunk != 0

    def regime(self):
        return {"mode": self.mode, "multi": self.nunits > self.grid, "dimg": self.dimg >= 1, "ragged": self.ragged}

    def __str__(self):
        if not self.staged:
            return "gather"
        return (f"{self.mode} npx={self.npx} stages={self.stages} per_sm={self.per_sm} tiles={self.tiles_x} rc={self.rows_per_chunk} "
                f"chunks={self.chunks_y} units={self.nunits} grid={self.grid} ({self.units_per_cta}/CTA) "
                f"stride=({self.dtx},{self.dcy},{self.dimg})")


def _lround(x):
    return int(math.floor(x + 0.5))


def _pick_npx(dw, order, tol):
    npx, best = 1, 1e30
    for o in order:
        tw = 128 * o
        waste = -(-dw // tw) * tw / dw
        if waste < best - tol:
            best, npx = waste, o
    return npx


def _walk(s, dh, batch, ctas, min_rc):
    total_rows = dh * batch * s.tiles_x
    s.rows_per_chunk = min(max(min_rc, total_rows // (ctas * 16)), dh)
    s.chunks_y = -(-dh // s.rows_per_chunk)
    s.nunits = s.tiles_x * s.chunks_y * batch
    s.grid = min(s.nunits, ctas)
    s.dtx = s.grid % s.tiles_x
    g = s.grid // s.tiles_x
    s.dcy, s.dimg = g % s.chunks_y, g // s.chunks_y
    s.dh = dh
    return s


def _axis_weights_all_zero(dst_len, src_len, scale):
    d = np.arange(dst_len, dtype=F32)
    f = np.maximum((d + F32(0.5)) * F32(scale) - F32(0.5), F32(0))
    a = np.minimum(f.astype(np.uint32), src_len - 1)
    b = np.minimum(a + 1, src_len - 1)
    return bool(np.all((b == a) | (f - a.astype(F32) == 0)))


def fused_schedule(sw, sh, dw, dh, batch, sm, npx_knob=0, stages_knob=0, ctas_knob=0):
    """launch_fused_resize_rows (csrc/resize_fused.cu) on the host.  The leaf and output type do not enter the schedule."""
    row_bytes = sw * 3
    sx, sy = F32(sw) / F32(dw), F32(sh) / F32(dh)
    if row_bytes % 16 or sx > 6 or sw < 16:
        return Schedule("gather")
    yz = _axis_weights_all_zero(dh, sh, sy)
    xz = yz and _axis_weights_all_zero(dw, sw, sx)
    mode = "BOX" if (sw == 2 * dw and sh == 2 * dh) else ("POINT" if xz else ("YZERO" if yz else "GENERAL"))
    npx = _pick_npx(dw, (2, 3, 1, 4, 5), 0.10 if mode == "GENERAL" else 0.02)
    if 1 <= npx_knob <= 5:
        npx = npx_knob
    tw = 128 * npx
    slot = int(((tw - 1) * float(sx) + 4.0) * 3.0) + 32
    slot = min((slot + 127) & ~127, (row_bytes + 16 + 127) & ~127)
    stage_bytes = slot * (2 if mode in ("GENERAL", "BOX") else 1)
    stages = stages_knob if 2 <= stages_knob <= 16 else 3
    per_sm = ctas_knob if ctas_knob > 0 else (4 if mode == "GENERAL" else _lround(36 * 1024 / (stages * stage_bytes)))
    per_sm = max(2, min(per_sm, 8))
    while per_sm > 2 and per_sm * (stages * stage_bytes + 1024) > 200 * 1024:
        per_sm -= 1
    if ctas_knob <= 0 and stages_knob <= 0 and per_sm == 2:
        stages = min(16, max(3, int(18 * 1024 / stage_bytes)))
    if stages < 3 or stage_bytes * stages > 200 * 1024:
        return Schedule("gather")
    s = Schedule(mode, npx=npx, stages=stages, per_sm=per_sm, tiles_x=-(-dw // tw))
    return _walk(s, dh, batch, sm * per_sm, 8)


NAMED_FUSED_MODES = {(384, 216, 128, 72): "POINT", (384, 216, 192, 108): "BOX", (384, 216, 160, 90): "GENERAL", (384, 216, 384, 72): "POINT",
                     (384, 216, 160, 72): "YZERO", (383, 216, 128, 72): "gather", (3840, 40, 512, 20): "gather"}


def _remap_maps(dw, dh, sw, sh, kind, rng):
    y, x = np.meshgrid(np.arange(dh, dtype=np.float32), np.arange(dw, dtype=np.float32), indexing="ij")
    if kind == "identity":
        return x * np.float32(sw / dw), y * np.float32(sh / dh)
    if kind == "swirl":   # smooth distortion that leaves the image on all sides, with NaN / inf holes
        cx, cy = np.float32(sw / 2), np.float32(sh / 2)
        r2 = ((x - dw / 2) ** 2 + (y - dh / 2) ** 2).astype(np.float32) / np.float32(dw * dw)
        mx = (cx + (x - dw / 2) * (1 + 1.5 * r2) * np.float32(sw / dw)).astype(np.float32)
        my = (cy + (y - dh / 2) * (1 + 1.5 * r2) * np.float32(sh / dh)).astype(np.float32)
        mx[0, 0] = np.nan; my[1, 1] = np.inf; mx[2, 2] = -np.inf; mx[3, 3] = sw - 0.25; my[3, 3] = sh - 0.25; mx[4, 4] = sw; my[5, 5] = -0.0
        return mx, my
    mx = rng.uniform(-3, sw + 3, (dh, dw)).astype(np.float32); my = rng.uniform(-3, sh + 3, (dh, dw)).astype(np.float32)
    return mx, my


def filter_kernel(w, c, op):
    """try_sep_stream (csrc/filter.cu): rows of a whole number of float4 (>= 16 floats) and a streaming instance for
    (C, K, sobel) -> the streaming kernel; everything else (and every kx != ky filter) -> the tile kernel."""
    k = int(op[-1]) if op != "sep" else 0
    inst = (op.startswith("gauss") and c in (1, 3, 4) and k in (3, 5, 7) and not (c == 4 and k == 7)) or \
           (op.startswith("sobel") and c in (1, 3) and k in (3, 5))
    return "sep_filter_stream2_kernel" if inst and (w * c) % 4 == 0 and w * c >= 16 else "sep_filter_fused_kernel"


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
