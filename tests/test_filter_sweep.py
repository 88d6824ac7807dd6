"""Separable filters and u8 blurs: a seeded sweep over every kernel instance the two dispatchers can pick, with taps that
tell the axes and the tap order apart, against the oracle; and a float64 restatement that pins the oracle's own
orientation and centre.

A gaussian with sigma_x == sigma_y has kx == ky, both palindromes, and sobel's magnitude does not change when the axes
are swapped or the derivative taps reversed.  A kernel that applied ky horizontally, or read kx[K-1-t], passes every test
that only runs those.  So here:

  * `case(i)` is a pure function of its index (numpy.random.default_rng(BASE + i)): the op (i % 5), and from the index
    within the op the channel count, tap length and row shape, so that every instance is reached; then random taps
    (separable_filter: equal lengths 3/5/7 with kx != ky and a non-palindromic kx, or random lengths 1-31, odd and even,
    mixed signs), sigma_x != sigma_y at equal sizes and (0, 0) auto sizes (gaussians), kx != ky (box), image size, batch,
    and buffers aligned or one element past a 16-byte boundary.  Hand-picked edge cases (EDGES) run the same way.
  * Each case calls the C ABI directly, src inside harness.Guarded poison, dst inside a Guarded region prefilled
    with NaN (f32) or 0xCD (u8).  The guards must keep their fill, no f32 output may be left at the fill, kb200_last_kernel()
    must be the kernel `plan` (a host mirror of launch_sep / launch_blur_u8) names, and every frame must equal the
    oracle bit for bit (f32: +0 / -0 and NaN payloads aside; infinities must match in sign).

test_sweep_coverage (CPU) runs every case through the mirror and asserts what the sweep reaches, so that a change to the
generator cannot silently shrink it.  test_oracle_float64_anchor (CPU) compares oracle.separable_filter with a numpy float64
restatement of the reference engine, so that the oracle's orientation and centre do not rest on the C++ code alone.
"""
import ctypes as C
from collections import defaultdict
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from harness import Guarded, assert_f32_bits_or_signed_zero, dev, knobs, lib
from restate import _q8_two_pass_numpy


BASE = 0x5F170000
F32 = np.float32
OPS = ("separable", "gaussian", "sobel", "gaussian_u8", "box_u8")
N_PER_OP = 80
N_SWEEP = len(OPS) * N_PER_OP
F32_SHAPES = ("stream", "interior", "offset", "partial", "small")
U8_SHAPES = ("stream", "word", "byte", "offset", "small")

STREAM_F32, TILE_F32 = "sep_filter_stream2_kernel", "sep_filter_fused_kernel"
STREAM_U8, WORD_U8, BYTE_U8 = "blur_u8_stream_kernel", "blur_u8_tile_w_kernel", "blur_u8_tile_kernel"
# try_sep_stream's instances (C, K, sobel), and the f32 tile kernel's (KX, KY, sobel) for every C = 1..4
SS_INST = {(3, 5, False), (3, 3, False), (3, 7, False), (1, 5, False), (1, 3, False), (1, 7, False), (4, 5, False), (4, 3, False),
           (3, 3, True), (3, 5, True), (1, 3, True), (1, 5, True)}
TILE_INST = {(k, k, False) for k in (3, 5, 7, 0)} | {(3, 3, True), (5, 5, True)}
SS_EW = 512                # floats per strip of sep_filter_stream2_kernel (SS2<1>::EW)
U8S_EB = 1024              # bytes per strip of blur_u8_stream_kernel (U8S_CT * NV * 4)
TILE_CAP = 100 * 1024      # launch_sep's shared-memory cap: min(max_smem_optin, 100 KiB), and an H100 allows 227 KiB
# Both stream launchers size a chunk as max(32, units / (CTAs * 12 or 4)) rows: 32 rows for every case here as long as the
# units stay below this on a GPU with at least 100 SMs (an H100 has 114 or 132).
SS_TOTAL_MAX, U8S_TOTAL_MAX = 33 * 12 * 100, 33 * 4 * 100


# ── the cases ──────────────────────────────────────────────────────────────────────────────────────────────────────────
@dataclass(frozen=True)
class Case:
    name: str
    seed: int                 # frame contents
    op: str
    C: int
    cols: int
    rows: int
    batch: int
    kx: tuple = ()            # separable_filter's taps
    ky: tuple = ()
    ksize: tuple = (0, 0)     # gaussian / box sizes; sobel (k, k)
    sigma: tuple = (0.0, 0.0)
    src_off: int = 0          # bytes past a 16-B boundary
    dst_off: int = 0
    knobs: tuple = ()         # ((name, value), ...)

    @property
    def u8(self):
        return self.op.endswith("_u8")

    def __str__(self):
        t = f"kx {list(self.kx)} ky {list(self.ky)}" if self.op == "separable" else f"ksize {self.ksize} sigma {self.sigma}"
        return (f"{self.name}: {self.op} C={self.C} {self.cols}x{self.rows} x{self.batch} {t} src +{self.src_off} B dst +{self.dst_off} B"
                + (f" knobs {dict(self.knobs)}" if self.knobs else ""))


def taps(c):
    """(kx, ky, binomial) as the entry point builds them: f32 arrays for the f32 ops, Q8 u8 arrays for the u8 blurs."""
    from oracle import oracle as o
    if c.op == "separable":
        return np.array(c.kx, F32), np.array(c.ky, F32), False
    if c.op == "sobel":
        return (*o.sobel_kernel_1d(c.ksize[0]), False)
    if c.op == "box_u8":
        return tuple(o.quantize_kernel_256(np.full(k, F32(1.0) / F32(k), F32)) for k in c.ksize) + (False,)
    kxn, kyn, sx, sy = o.gaussian_resolve(*c.ksize, *c.sigma)
    if c.op == "gaussian":
        return o.gaussian_kernel_1d(kxn, sx), o.gaussian_kernel_1d(kyn, sy), False
    if kxn == 3 and kyn == 3 and F32(0.6) <= sx <= F32(1.2) and F32(0.6) <= sy <= F32(1.2):   # blur_u8_path
        return np.zeros(3, np.uint8), np.zeros(3, np.uint8), True
    return o.quantize_kernel_256(o.gaussian_kernel_1d(kxn, sx)), o.quantize_kernel_256(o.gaussian_kernel_1d(kyn, sy)), False


def f32_taps(rng, k, avoid=None):
    """k random float32 taps, mixed signs, not a palindrome (k > 1), and not `avoid`."""
    while True:
        t = rng.uniform(-1.5, 1.5, k).astype(F32)
        t[rng.integers(0, k)] = F32(rng.uniform(0.5, 2.0))   # a positive tap of some size
        if (k == 1 or not np.array_equal(t, t[::-1])) and (avoid is None or not np.array_equal(t, avoid)):
            return tuple(float(v) for v in t)


def multiple_of(C, b):
    """The smallest m such that m * C is a multiple of b."""
    return b // np.gcd(C, b)


def f32_geometry(rng, shape, C):
    """(cols, rows, src_off, dst_off) for a row shape of the f32 dispatcher."""
    rows = int(rng.integers(1, 91))
    m = multiple_of(C, 4)
    if shape == "stream":       # whole float4s, 16 <= cols * C < 1032: edge strips only
        return m * int(rng.integers(-(-16 // (m * C)), 1028 // (m * C) + 1)), rows, 0, 0
    if shape == "interior":     # >= 1032 floats: interior strips where the halo allows
        return m * int(rng.integers(-(-1032 // (m * C)), 2600 // (m * C) + 1)), int(rng.integers(1, 41)), 0, 0
    if shape == "offset":       # a streamable row, src and / or dst one float past a 16-B boundary: the tile kernel
        so, do = ((4, 0), (0, 4), (4, 4))[int(rng.integers(0, 3))]
        return m * int(rng.integers(-(-16 // (m * C)), 700 // (m * C) + 1)), rows, so, do
    so, do = ((0, 0), (4, 0), (0, 4), (4, 4))[int(rng.integers(0, 4))] if rng.random() < 0.4 else (0, 0)
    if shape == "partial":      # a partial float4 at the end of each row (C = 4 has none: rows shorter than 16 floats)
        if C == 4:
            return int(rng.integers(1, 4)), rows, so, do
        cols = int(rng.integers(1, 600))
        while cols * C % 4 == 0:
            cols += 1
        return cols, rows, so, do
    return int(rng.integers(1, 41)), int(rng.integers(1, 41)), so, do


def u8_geometry(rng, shape, C):
    """(cols, rows, src_off, dst_off) for a row shape of the u8 dispatcher."""
    rows = int(rng.integers(1, 91))
    if shape in ("stream", "offset"):   # rows of whole 16-B words, at least 256 bytes
        m = multiple_of(C, 16)
        cols = m * int(rng.integers(-(-256 // (m * C)), 2200 // (m * C) + 1))
        if shape == "stream":
            return cols, rows, 0, 0
        return (cols, rows) + ((1, 0), (0, 1), (1, 1))[int(rng.integers(0, 3))]
    if shape == "word":        # whole 4-B words, but short of 256 bytes or not whole 16-B words
        m = multiple_of(C, 4)
        while True:
            cols = m * int(rng.integers(max(1, -(-4 // m)), 600 // (m * C) + 1))
            if cols >= 4 and (cols * C % 16 or cols * C < 256):
                return cols, rows, 0, 0
    so, do = ((0, 0), (1, 0), (0, 1), (1, 1))[int(rng.integers(0, 4))] if rng.random() < 0.4 else (0, 0)
    if shape == "byte":        # rows of a partial word (C = 4 has none: fewer than 4 columns)
        if C == 4:
            return int(rng.integers(1, 4)), rows, so, do
        cols = int(rng.integers(1, 700))
        while cols * C % 4 == 0:
            cols += 1
        return cols, rows, so, do
    return int(rng.integers(1, 41)), int(rng.integers(1, 41)), so, do


def sigma_pair(rng, k, u8):
    """sigma_x != sigma_y whose taps at size k differ (Q8 taps for u8; never both in the binomial range at k = 3)."""
    from oracle import oracle as o
    while True:
        sx, sy = (float(F32(rng.uniform(0.3, 3.0))) for _ in range(2))
        if u8 and k == 3 and F32(0.6) <= sx <= F32(1.2) and F32(0.6) <= sy <= F32(1.2):
            continue
        tx, ty = o.gaussian_kernel_1d(k, sx), o.gaussian_kernel_1d(k, sy)
        if u8:
            tx, ty = o.quantize_kernel_256(tx), o.quantize_kernel_256(ty)
        if not np.array_equal(tx, ty):
            return sx, sy


def odd(rng, lo=1, hi=31):
    return int(rng.integers(lo // 2, hi // 2 + 1)) * 2 + 1


def case(i):
    """Case i of the sweep: a pure function of i."""
    rng = np.random.default_rng(BASE + i)
    op, j = OPS[i % len(OPS)], i // len(OPS)
    batch = int(rng.integers(1, 4))
    kw = {}
    if op in ("separable", "gaussian", "sobel"):
        C = 1 + j % 4
        if op == "separable":
            # j < 60: every (C, K = 3/5/7, row shape) once with kx != ky and a non-palindromic kx; then random lengths 1-31
            shape = F32_SHAPES[(j // 12) % 5] if j < 60 else F32_SHAPES[j % 5]
            if j < 60:
                k = (3, 5, 7)[(j // 4) % 3]
                kx = f32_taps(rng, k)
                kw = dict(kx=kx, ky=f32_taps(rng, k, avoid=np.array(kx, F32)))
            else:
                kw = dict(kx=f32_taps(rng, int(rng.integers(1, 32))), ky=f32_taps(rng, int(rng.integers(1, 32))))
        elif op == "gaussian":
            # j < 60: sigma_x != sigma_y at equal sizes 3/5/7; then (0, 0) auto sizes, and unequal sizes
            shape = F32_SHAPES[(j // 4) % 5]
            if j < 60:
                k = (3, 5, 7)[(j // 20) % 3]
                kw = dict(ksize=(k, k), sigma=sigma_pair(rng, k, False))
            elif j < 70:
                kw = dict(ksize=(0, 0), sigma=(float(F32(rng.uniform(0.2, 3.6))), float(F32(rng.uniform(0.2, 3.6))) if j % 2 else 0.0))
            else:
                kw = dict(ksize=(odd(rng), odd(rng)), sigma=(float(F32(rng.uniform(0.0, 3.0))), float(F32(rng.uniform(0.0, 3.0)))))
        else:
            shape = F32_SHAPES[(j // 8) % 5]
            k = (3, 5)[(j // 4) % 2]
            kw = dict(ksize=(k, k))
        cols, rows, so, do = f32_geometry(rng, shape, C)
    else:
        C = (1, 3, 4)[j % 3]
        shape = U8_SHAPES[(j // 9) % 5]
        if op == "gaussian_u8":
            # j < 45: every (C, K = 3/5/7, row shape) with sigma_x != sigma_y at equal sizes; 45-53 the same on stream rows with
            # the stream kernel switched off (knob b = 3: the word kernel); 54-62 the binomial path; then auto and unequal sizes
            k = (3, 5, 7)[(j // 3) % 3]
            if j < 54:
                if j >= 45:
                    shape, kw = "stream", dict(knobs=(("b", 3),))
                kw.update(ksize=(k, k), sigma=sigma_pair(rng, k, True))
            elif j < 63:
                kw = dict(ksize=(3, 3), sigma=(float(F32(rng.uniform(0.6, 1.2))), float(F32(rng.uniform(0.6, 1.2))) if j % 2 else 0.0))
            elif j < 72:
                kw = dict(ksize=(0, 0), sigma=(float(F32(rng.uniform(0.2, 3.6))), float(F32(rng.uniform(0.2, 3.6))) if j % 2 else 0.0))
            else:
                kw = dict(ksize=(odd(rng), odd(rng)), sigma=(float(F32(rng.uniform(0.0, 3.0))), float(F32(rng.uniform(0.0, 3.0)))))
        else:
            # every fourth case kx == ky in 3/5/7 (the fixed instances), the rest kx != ky
            if j % 4 == 0:
                k = (3, 5, 7)[(j // 4) % 3]
                kw = dict(ksize=(k, k))
            else:
                kx = odd(rng)
                ky = kx
                while ky == kx:
                    ky = odd(rng)
                kw = dict(ksize=(kx, ky))
            if j >= 72:
                kw["knobs"] = (("b", 3),)
        cols, rows, so, do = u8_geometry(rng, shape, C)
    return Case(f"sweep-{i}", BASE + i, op, C, cols, rows, batch, src_off=so, dst_off=do, **kw)


# ── the dispatch rules, restated ───────────────────────────────────────────────────────────────────────────────────
@dataclass(frozen=True)
class Plan:
    kernel: str
    inst: tuple               # f32 stream (C, K, sobel); f32 tile (KX, KY, sobel, C); u8 (C, K), K = 0: run-time tap counts
    tile: tuple = ()          # f32 tile: ((tw, th) before the shared-memory shrink loop, (tw, th) after it)
    strips: frozenset = frozenset()   # f32 stream: "edge" / "interior" strips present
    ragged: bool = False      # stream: the last row chunk is short
    binomial: bool = False
    kx_ne_ky: bool = False
    kx_palindrome: bool = True


def tile_regime(C, kxn, kyn, sobel, cols, rows):
    """launch_sep's tile size: 64 x 32 pixels (32 wide for cols <= 32, 16 high for rows <= 16), halved until it fits."""
    tw, th = (32 if cols <= 32 else 64), (16 if rows <= 16 else 32)
    start = (tw, th)

    def smem(tw, th):
        return ((tw + kxn - 1) * C * (th + kyn - 1) + tw * C * (th + kyn - 1) * (2 if sobel else 1)) * 4

    while smem(tw, th) > TILE_CAP and (tw > 16 or th > 8):
        if th > 8 and th >= tw // 2:
            th //= 2
        else:
            tw //= 2
    assert smem(tw, th) <= TILE_CAP
    return start, (tw, th)


def plan(c):
    """The kernel launch_sep / launch_blur_u8 runs for case c, and what of it the case exercises."""
    kx, ky, binomial = taps(c)
    kxn, kyn = len(kx), len(ky)
    ne = kxn != kyn or not np.array_equal(kx, ky)
    pal = bool(np.array_equal(kx, kx[::-1]))
    src_al, dst_al = c.src_off % 16 == 0, c.dst_off % 16 == 0
    if not c.u8:
        sobel = c.op == "sobel"
        rowlen = c.cols * c.C
        finite = bool(np.isfinite(kx).all() and np.isfinite(ky).all())
        # try_sep_stream; taps with an inf or NaN skip it (see launch_sep)
        if finite and rowlen % 4 == 0 and src_al and dst_al and rowlen >= 16 and kxn == kyn and (c.C, kxn, sobel) in SS_INST:
            hx = kxn // 2
            hl, hr = (hx * c.C + 3) // 4 * 4, ((kxn - 1 - hx) * c.C + 3) // 4 * 4
            strips = -(-rowlen // SS_EW)
            kinds = frozenset("edge" if e0 - hl < 0 or e0 + SS_EW + hr > rowlen else "interior" for e0 in range(0, strips * SS_EW, SS_EW))
            assert strips * c.batch * c.rows < SS_TOTAL_MAX, str(c)
            rc = min(32, c.rows)
            return Plan(STREAM_F32, (c.C, kxn, sobel), strips=kinds, ragged=c.rows % rc != 0, kx_ne_ky=ne, kx_palindrome=pal)
        if sobel:
            inst = (kxn, kxn, True)
        elif finite and kxn == kyn and kxn in (3, 5, 7):
            inst = (kxn, kxn, False)
        else:
            inst = (0, 0, False)
        return Plan(TILE_F32, inst + (c.C,), tile=tile_regime(c.C, kxn, kyn, sobel, c.cols, c.rows), kx_ne_ky=ne, kx_palindrome=pal)
    rowb = c.cols * c.C
    b3 = dict(c.knobs).get("b") == 3
    word_ok = (rowb % 4 == 0 and c.src_off % 4 == 0 and c.dst_off % 4 == 0 and kxn == kyn
               and (binomial or (int(kx.astype(np.int64).sum()) <= 256 and int(ky.astype(np.int64).sum()) <= 256)) and c.cols >= 4)
    fixed = kxn in (3, 5, 7)
    if word_ok and fixed and rowb % 16 == 0 and rowb >= 256 and src_al and dst_al and (kxn // 2) * c.C <= 16 and not b3:
        assert -(-rowb // U8S_EB) * c.batch * c.rows < U8S_TOTAL_MAX, str(c)
        return Plan(STREAM_U8, (c.C, kxn), ragged=c.rows % min(32, c.rows) != 0, binomial=binomial, kx_ne_ky=ne, kx_palindrome=pal)
    if word_ok and fixed:
        return Plan(WORD_U8, (c.C, kxn), binomial=binomial, kx_ne_ky=ne, kx_palindrome=pal)
    return Plan(BYTE_U8, (c.C, kxn if kxn == kyn and fixed else 0), binomial=binomial, kx_ne_ky=ne, kx_palindrome=pal)


def reachable_tile_regimes():
    """Every (start, end) tile size of the shrink loop over all inputs launch_sep accepts."""
    out = set()
    for C in range(1, 5):
        for sobel, sizes in ((False, [(a, b) for a in range(1, 32) for b in range(1, 32)]), (True, [(3, 3), (5, 5)])):
            for kxn, kyn in sizes:
                for cols in (32, 33):
                    for rows in (16, 17):
                        out.add(tile_regime(C, kxn, kyn, sobel, cols, rows))
    return out


# ── hand-picked edges ───────────────────────────────────────────────────────────────────────────────────────────────
def edge(name, op, C, cols, rows, batch=1, **kw):
    seed = 0xED6F0000 + sum(ord(ch) * 131 ** k for k, ch in enumerate(name)) % 0xFFFF
    return Case(name, seed, op, C, cols, rows, batch, **kw)


INF, NAN = float("inf"), float("nan")
NEXT_BELOW_06, NEXT_ABOVE_12 = float(np.nextafter(F32(0.6), F32(0))), float(np.nextafter(F32(1.2), F32(2)))


def _edges():
    e = []
    a3, b3 = (0.25, -1.0, 1.5), (1.25, 0.5, -0.75)
    a5, b5 = (0.5, -0.25, 1.0, 0.125, -0.75), (-0.5, 1.5, 0.25, 0.75, -0.125)
    a7 = (0.1, -0.2, 0.3, 1.0, -0.4, 0.05, 0.6)
    # 1x1, 1xN and Nx1 images on every op
    for cols, rows in ((1, 1), (1, 23), (23, 1)):
        g = f"{cols}x{rows}"
        for C in (1, 3, 4):
            e.append(edge(f"tiny-{g}-separable5-C{C}", "separable", C, cols, rows, 2, kx=a5, ky=b5))
        e.append(edge(f"tiny-{g}-separable3-C2", "separable", 2, cols, rows, kx=a3, ky=b3))
        e.append(edge(f"tiny-{g}-gaussian5-C3", "gaussian", 3, cols, rows, ksize=(5, 5), sigma=(0.8, 1.7)))
        e.append(edge(f"tiny-{g}-sobel3-C1", "sobel", 1, cols, rows, ksize=(3, 3)))
        e.append(edge(f"tiny-{g}-sobel5-C4", "sobel", 4, cols, rows, ksize=(5, 5)))
        e.append(edge(f"tiny-{g}-gaussian-u8-C3", "gaussian_u8", 3, cols, rows, 2, ksize=(5, 5), sigma=(1.0, 2.0)))
        e.append(edge(f"tiny-{g}-binomial-u8-C4", "gaussian_u8", 4, cols, rows, ksize=(3, 3), sigma=(1.0, 1.0)))
        e.append(edge(f"tiny-{g}-box-u8-C1", "box_u8", 1, cols, rows, ksize=(3, 7)))
    # taps longer than the image
    long_x, long_y = f32_taps(np.random.default_rng(31), 31), f32_taps(np.random.default_rng(32), 31)
    for C in (1, 4):
        e.append(edge(f"long-taps-separable31-5x3-C{C}", "separable", C, 5, 3, 2, kx=long_x, ky=long_y))
    e.append(edge("long-taps-gaussian31-5x3", "gaussian", 3, 5, 3, ksize=(31, 31), sigma=(2.0, 5.0)))
    e.append(edge("long-taps-gaussian-auto29-5x3", "gaussian", 2, 5, 3, ksize=(0, 0), sigma=(3.6, 0.0)))
    e.append(edge("long-taps-gaussian-u8-31x29-5x3", "gaussian_u8", 3, 5, 3, ksize=(31, 29), sigma=(4.0, 3.0)))
    e.append(edge("long-taps-box-u8-31-5x3", "box_u8", 4, 5, 3, ksize=(31, 31)))
    e.append(edge("long-taps-box-u8-7x31-5x3", "box_u8", 1, 5, 3, ksize=(7, 31)))
    # the shortest streamable row (16 floats), one float4 less, and 1032 floats (one interior strip for short halos)
    e.append(edge("row16-separable3-C4", "separable", 4, 4, 37, kx=a3, ky=b3))
    e.append(edge("row16-separable7-C1", "separable", 1, 16, 41, 2, kx=a7, ky=a7[::-1]))
    e.append(edge("row16-sobel3-C1", "sobel", 1, 16, 9, ksize=(3, 3)))
    e.append(edge("row12-separable3-C3", "separable", 3, 4, 19, kx=a3, ky=b3))
    e.append(edge("row12-separable5-C1", "separable", 1, 12, 19, kx=a5, ky=b5))
    for C, cols, k in ((1, 1032, 3), (1, 1032, 7), (3, 344, 5), (4, 258, 5), (4, 258, 3)):
        kx, ky = {3: (a3, b3), 5: (a5, b5), 7: (a7, a5 + (1.0, 2.0))}[k]
        e.append(edge(f"row1032-separable{k}-C{C}", "separable", C, cols, 35, kx=kx, ky=ky[:k]))
    e.append(edge("row1032-sobel3-C3", "sobel", 3, 344, 33, ksize=(3, 3)))
    e.append(edge("row1032-gaussian7-C3", "gaussian", 3, 344, 40, ksize=(7, 7), sigma=(0.7, 2.5)))
    # u8 rows of exactly 256 bytes (the shortest stream row), and 240 (the word kernel)
    for C, cols, k, sg in ((1, 256, 3, (0.5, 2.0)), (1, 256, 5, (2.0, 0.9)), (1, 256, 7, (1.1, 3.0)), (4, 64, 7, (3.0, 0.8)), (4, 64, 3, (1.0, 2.5)),
                           (1, 240, 5, (0.9, 1.9)), (4, 60, 7, (1.5, 2.5))):
        e.append(edge(f"u8-row{cols * C}-gaussian{k}-C{C}", "gaussian_u8", C, cols, 45, 2, ksize=(k, k), sigma=sg))
    e.append(edge("u8-row256-box5-C4", "box_u8", 4, 64, 33, ksize=(5, 5)))
    # the binomial path at sigma exactly 0.6 and 1.2 and just outside, on stream, word and byte rows
    for sg, tag in (((0.6, 0.6), "0.6"), ((1.2, 1.2), "1.2"), ((0.6, 1.2), "0.6-1.2"), ((1.2, 0.0), "1.2-auto"),
                    ((NEXT_BELOW_06, 0.6), "below0.6"), ((1.2, NEXT_ABOVE_12), "above1.2"), ((NEXT_ABOVE_12, 0.0), "above1.2-auto")):
        for C, cols, shape in ((3, 256, "stream"), (4, 21, "word"), (1, 37, "byte")):
            e.append(edge(f"binomial-{tag}-{shape}", "gaussian_u8", C, cols, 34, ksize=(3, 3), sigma=sg))
    # pure shifts: a halo or centre off by one moves the whole image
    s0, s1 = (0.0, 0.0, 1.0), (1.0, 0.0, 0.0)
    for C, cols, rows, so, do, tag in ((1, 64, 20, 0, 0, "stream"), (3, 64, 20, 0, 0, "stream"), (4, 16, 20, 0, 0, "stream"),
                                       (1, 1100, 20, 0, 0, "interior"), (2, 33, 17, 0, 0, "tile"), (3, 64, 20, 4, 4, "offset")):
        e.append(edge(f"shift-{tag}-C{C}-right-up", "separable", C, cols, rows, kx=s0, ky=s1, src_off=so, dst_off=do))
        e.append(edge(f"shift-{tag}-C{C}-left-down", "separable", C, cols, rows, kx=s1, ky=s0, src_off=so, dst_off=do))
    e.append(edge("shift5-stream-C3", "separable", 3, 64, 20, kx=(0.0, 0.0, 0.0, 0.0, 1.0), ky=(0.0, 1.0, 0.0, 0.0, 0.0)))
    e.append(edge("shift7-tile-C4", "separable", 4, 3, 20, kx=(1.0,) + (0.0,) * 6, ky=(0.0,) * 5 + (1.0, 0.0)))
    # even lengths: the centre is k / 2
    for kxn, kyn in ((2, 2), (4, 4), (6, 6), (2, 6), (4, 1), (1, 2)):
        kx, ky = f32_taps(np.random.default_rng(kxn), kxn), f32_taps(np.random.default_rng(10 + kyn), kyn)
        for C, cols in ((1, 64), (3, 37), (4, 300)):
            e.append(edge(f"even-{kxn}x{kyn}-C{C}-{cols}", "separable", C, cols, 23, kx=kx, ky=ky))
    e.append(edge("even-shift-2", "separable", 3, 40, 12, kx=(0.0, 1.0), ky=(1.0, 0.0)))
    # the tile kernel's shrink loop: C = 4 with 31 x 31 taps ends at 32 x 16, C = 3 with 31-tap columns at 64 x 16
    for cols, rows in ((100, 40), (100, 12)):
        e.append(edge(f"tile-shrink-31x31-C4-{cols}x{rows}", "separable", 4, cols, rows, kx=long_x, ky=long_y))
        e.append(edge(f"tile-shrink-13x31-C4-{cols}x{rows}", "separable", 4, cols, rows, kx=long_x[:13], ky=long_y))
    e.append(edge("tile-shrink-11x31-C3-100x40", "separable", 3, 100, 40, kx=long_x[:11], ky=long_y))
    # non-finite taps that fall outside the image at a border: the reference skips such taps, so the border stays finite
    e.append(edge("nonfinite-last-column-stream-row", "separable", 3, 64, 20, kx=(0.5, 1.0, INF), ky=(0.25, 0.5, 0.25)))
    e.append(edge("nonfinite-first-column-C2", "separable", 2, 37, 9, kx=(NAN, 1.0, 0.5), ky=(1.0, -1.0, 2.0)))
    e.append(edge("nonfinite-last-row-C1", "separable", 1, 37, 11, kx=(1.0, 2.0, -1.0), ky=(1.0, -1.0, INF)))
    e.append(edge("nonfinite-first-row-offset", "separable", 3, 64, 13, kx=(0.5, 1.5, -0.5), ky=(-INF, 2.0, 1.0), src_off=4))
    e.append(edge("nonfinite-1x1", "separable", 3, 1, 1, kx=(INF, 1.0, INF), ky=(NAN, 1.0, NAN)))
    e.append(edge("nonfinite-column-image", "separable", 1, 1, 17, kx=(INF, NAN, 1.0, NAN, INF), ky=(1.0, 2.0, -3.0)))
    e.append(edge("nonfinite-even-first-column", "separable", 4, 20, 6, kx=(INF, 1.0), ky=(0.5, 1.0, 0.25, -1.0)))
    e.append(edge("nonfinite-31-taps-5x3", "separable", 3, 5, 3, kx=(INF,) + long_x[1:30] + (NAN,), ky=(-INF,) + long_y[1:30] + (INF,)))
    # a row the stream kernel would take with finite taps (interior strips included); rows = 3 keeps ky's end taps outside
    e.append(edge("nonfinite-7-taps-interior-row", "separable", 1, 1100, 3, 2, kx=a7, ky=(INF,) + a7[1:6] + (NAN,)))
    return e


EDGES = {c.name: c for c in _edges()}
assert len(EDGES) == len(_edges()), "edge case names must be unique"


# ── the GPU run ─────────────────────────────────────────────────────────────────────────────────────────────────────
def frame(c, k):
    rng = np.random.default_rng([c.seed, k])
    if c.u8:
        return rng.integers(0, 256, (c.rows, c.cols, c.C), dtype=np.int64).astype(np.uint8)
    return rng.uniform(-8.0, 8.0, (c.rows, c.cols, c.C)).astype(F32)


def reference(c, f):
    from oracle import oracle as o
    if c.op == "separable":
        return o.separable_filter(f, np.array(c.kx, F32), np.array(c.ky, F32))
    if c.op == "gaussian":
        return o.gaussian_blur(f, c.ksize, c.sigma)
    if c.op == "sobel":
        return o.sobel(f, c.ksize[0])
    if c.op == "gaussian_u8":
        return o.gaussian_blur_u8(f, c.ksize, c.sigma)
    return o.box_blur_u8(f, c.ksize)


def call(lib, c, src, dst, n):
    g = (c.cols, c.rows, c.C, c.batch)
    if c.op == "separable":
        kx, ky = np.array(c.kx, F32), np.array(c.ky, F32)
        fp = C.POINTER(C.c_float)
        return lib.kb200_separable_filter_f32(None, src, n, dst, n, None, kx.ctypes.data_as(fp), kx.size, ky.ctypes.data_as(fp), ky.size, *g)
    if c.op == "gaussian":
        return lib.kb200_gaussian_blur_f32(None, src, n, dst, n, *g, *c.ksize, *c.sigma)
    if c.op == "sobel":
        return lib.kb200_sobel_f32(None, src, n, dst, n, *g, c.ksize[0])
    if c.op == "gaussian_u8":
        return lib.kb200_gaussian_blur_u8(None, src, n, dst, n, *g, *c.ksize, *c.sigma)
    return lib.kb200_box_blur_u8(None, src, n, dst, n, *g, *c.ksize)


def assert_same_f32(got, want, what):
    """Bit for bit, as assert_f32_bits_or_signed_zero, where both are finite; elsewhere the same non-finite class (NaN, +inf or -inf)."""
    got, want = got.reshape(-1), want.reshape(-1)
    fin_g, fin_w = np.isfinite(got), np.isfinite(want)
    cls = lambda a: np.where(np.isnan(a), 2, np.sign(np.nan_to_num(a, nan=0.0, posinf=1.0, neginf=-1.0)))
    bad = np.flatnonzero((fin_g != fin_w) | (~fin_w & (cls(got) != cls(want))))
    if bad.size:
        raise AssertionError(f"{what}: {bad.size} elements differ in finiteness, first at element {bad[0]}: got {got[bad[0]]}, want {want[bad[0]]}")
    if fin_w.any():
        assert_f32_bits_or_signed_zero(got[fin_w], want[fin_w], what)


def run_case(kb, lib, dev, c):
    p = plan(c)
    frames = [frame(c, k) for k in range(c.batch)]
    n = c.cols * c.rows * c.C
    esz = 1 if c.u8 else 4
    fill = 0xCD if c.u8 else 0xFF
    src = Guarded(dev, n * esz * c.batch, offset=c.src_off).load("u8" if c.u8 else "f32", np.concatenate([f.reshape(-1) for f in frames]).view(np.uint8))
    dst = Guarded(dev, n * esz * c.batch, offset=c.dst_off).fill(fill)
    with knobs(kb, dict(c.knobs)):
        st = call(lib, c, src.ptr, dst.ptr, n * c.batch)
        ran = kb._lib.last_kernel()
    assert st == 0, f"{c}: status {st}: {kb._lib.last_error()}"
    torch.cuda.synchronize()
    assert ran == p.kernel, f"{c}: ran {ran}, the dispatch mirror says {p.kernel} ({p})"
    lead, tail = dst.guards()
    for what, g in (("lead", lead), ("tail", tail)):
        bad = np.flatnonzero(g != fill)
        assert bad.size == 0, f"{c}: {bad.size} bytes written in the {what} guard"
    out = dst.out()
    if not c.u8:
        out = out.view(np.uint32)
        left = np.flatnonzero(out == 0xFFFFFFFF)
        assert left.size == 0, f"{c}: {left.size} output elements left unwritten (first {left[0]})"
        out = out.view(F32)
    for k, f in enumerate(frames):
        got, want = out[k * n:(k + 1) * n], reference(c, f)
        what = f"{c}: frame {k} ({p.kernel} {p.inst})"
        if c.u8:
            bad = np.flatnonzero(got != want.reshape(-1))
            assert bad.size == 0, f"{what}: {bad.size} bytes differ from the oracle, first at byte {bad[0]}: got {got[bad[0]]}, want {want.reshape(-1)[bad[0]]}"
        else:
            assert_same_f32(got, want, what)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(N_SWEEP))
def test_sweep(kb, lib, dev, i):
    run_case(kb, lib, dev, case(i))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGES))
def test_edge(kb, lib, dev, name):
    run_case(kb, lib, dev, EDGES[name])


# ── what the sweep covers (CPU) ─────────────────────────────────────────────────────────────────────────────────────
def test_sweep_coverage(oracle):
    cases = [case(i) for i in range(N_SWEEP)] + list(EDGES.values())
    assert len({c.name for c in cases}) == len(cases)
    ops = {c.op for c in cases}
    assert ops == set(OPS)
    hit, ne, npal, regimes, strips, ragged, paths = defaultdict(set), defaultdict(set), defaultdict(set), set(), set(), set(), set()
    offset_paths, lengths, auto = set(), set(), set()
    for c in cases:
        p = plan(c)
        hit[p.kernel].add(p.inst)
        if p.kx_ne_ky:
            ne[p.kernel].add(p.inst)
            if not p.kx_palindrome:
                npal[p.kernel].add(p.inst)
        if p.kernel == TILE_F32:
            regimes.add(p.tile)
        strips |= p.strips
        if p.ragged:
            ragged.add(p.kernel)
        paths.add((p.kernel, "binomial" if p.binomial else "q8") if c.u8 else (p.kernel,))
        if c.src_off % 16 or c.dst_off % 16:
            offset_paths.add(p.kernel)
        if c.op == "separable":
            lengths |= {len(c.kx), len(c.ky)}
        if c.op.startswith("gaussian") and c.ksize == (0, 0):
            auto.add(c.op)
    f32_tile = {t + (C,) for t in TILE_INST for C in range(1, 5)}
    u8_fixed = {(C, k) for C in (1, 3, 4) for k in (3, 5, 7)}
    assert hit[STREAM_F32] == SS_INST, sorted(SS_INST - hit[STREAM_F32])
    assert hit[TILE_F32] == f32_tile, sorted(f32_tile - hit[TILE_F32])
    assert hit[STREAM_U8] == u8_fixed and hit[WORD_U8] == u8_fixed, (sorted(u8_fixed - hit[STREAM_U8]), sorted(u8_fixed - hit[WORD_U8]))
    assert hit[BYTE_U8] == {(C, k) for C in (1, 3, 4) for k in (3, 5, 7, 0)}, sorted(hit[BYTE_U8])
    # every fixed-size instance that filters with two tap vectors sees them differ (and, f32, with kx not a palindrome)
    for kern, want in ((STREAM_F32, {s for s in SS_INST if not s[2]}), (TILE_F32, {t for t in f32_tile if t[0] and not t[2]})):
        assert want <= ne[kern], (kern, sorted(want - ne[kern]))
        assert want <= npal[kern], (kern, sorted(want - npal[kern]))
    for kern, want in ((STREAM_U8, u8_fixed), (WORD_U8, u8_fixed), (BYTE_U8, u8_fixed)):
        assert want <= ne[kern], (kern, sorted(want - ne[kern]))
    assert regimes == reachable_tile_regimes(), sorted(reachable_tile_regimes() - regimes)
    assert strips == {"edge", "interior"} and ragged == {STREAM_F32, STREAM_U8}, (strips, ragged)
    assert {(k, b) for k in (STREAM_U8, WORD_U8, BYTE_U8) for b in ("binomial", "q8")} <= paths, sorted(paths)
    assert offset_paths == {TILE_F32, BYTE_U8}, offset_paths
    assert {1, 2, 4, 6, 31} <= lengths and {l % 2 for l in lengths if 7 < l < 31} == {0, 1}, sorted(lengths)
    assert auto == {"gaussian", "gaussian_u8"}, auto


# ── the oracle against a float64 restatement (CPU) ──────────────────────────────────────────────────────────────────
def separable_f64(src, kx, ky):
    """separable_filter.rs's engine in float64: correlation, taps ascending, taps outside the image skipped (zero border
    without 0 * k), H into a temporary image, then V."""
    def one_axis(a, k, axis):
        n, half, out = a.shape[axis], len(k) // 2, np.zeros_like(a)
        for t, kt in enumerate(np.asarray(k, np.float64)):
            d = t - half                      # output p reads input p + d
            lo, hi = max(0, -d), min(n, n - d)
            if lo < hi:
                sl_out, sl_in = [slice(None)] * 3, [slice(None)] * 3
                sl_out[axis], sl_in[axis] = slice(lo, hi), slice(lo + d, hi + d)
                out[tuple(sl_out)] += a[tuple(sl_in)] * kt
        return out
    return one_axis(one_axis(np.asarray(src, np.float64), kx, 1), ky, 0)


ANCHORS = {
    "k3": ((0.25, -1.0, 1.5), (1.25, 0.5, -0.75), 13, 11, 3),
    "k5": ((0.5, -0.25, 1.0, 0.125, -0.75), (-0.5, 1.5, 0.25, 0.75, -0.125), 9, 12, 1),
    "k7": ((0.1, -0.2, 0.3, 1.0, -0.4, 0.05, 0.6), (0.7, 0.0, -0.3, 0.2, 1.0, -0.6, 0.4), 17, 10, 4),
    "even2x4": ((1.0, -2.0), (0.5, 1.0, -1.0, 3.0), 8, 9, 2),
    "even6x6": ((0.3, -0.1, 0.9, 0.4, -0.7, 0.2), (-0.2, 0.6, 0.1, 1.1, -0.5, 0.3), 11, 7, 1),
    "shift": ((0.0, 0.0, 1.0), (1.0, 0.0, 0.0), 6, 5, 3),
    "unequal1x31": ((2.0,), tuple(float(v) for v in np.linspace(-1.0, 1.5, 31, dtype=F32)), 7, 40, 1),
    "longer-than-image": (tuple(float(v) for v in np.linspace(1.0, -0.5, 31, dtype=F32)), (0.5, -1.0, 0.25, 2.0, 0.75), 5, 3, 2),
}


@pytest.mark.parametrize("name", list(ANCHORS))
def test_oracle_float64_anchor(oracle, name):
    """oracle.separable_filter within 1e-5 of the float64 restatement, relative to the sum of |term|; the same restatement
    with the axes swapped or the taps reversed is far outside that, so the check decides orientation and centre."""
    kx, ky, w, h, c = ANCHORS[name]
    src = np.random.default_rng(len(name)).uniform(-4.0, 4.0, (h, w, c)).astype(F32)
    got = oracle.separable_filter(src, np.array(kx, F32), np.array(ky, F32)).astype(np.float64)
    mag = separable_f64(np.abs(src), np.abs(kx), np.abs(ky)) + 1e-30
    err = np.abs(got - separable_f64(src, kx, ky)) / mag
    assert err.max() <= 1e-5, f"{name}: relative error {err.max():.3g} at {np.unravel_index(err.argmax(), err.shape)}"
    for tag, (ax, ay) in (("swapped", (ky, kx)), ("reversed", (kx[::-1], ky[::-1]))):
        if (tuple(ax), tuple(ay)) != (tuple(kx), tuple(ky)):
            wrong = np.abs(got - separable_f64(src, ax, ay)) / mag
            assert wrong.max() > 1e-3, f"{name}: the {tag} taps are indistinguishable here"


def test_oracle_float64_anchor_skips_outside_taps(oracle):
    """Taps that only ever fall outside the image are skipped, whatever their value: a one-column image filtered with
    inf / NaN at every horizontal offset but 0 gives the vertical filter of the column alone."""
    src = np.random.default_rng(5).uniform(-4.0, 4.0, (9, 1, 2)).astype(F32)
    kx, ky = np.array([INF, NAN, 1.0, NAN, INF], F32), np.array([0.5, -1.0, 2.0], F32)
    got = oracle.separable_filter(src, kx, ky)
    want = separable_f64(src, [0.0, 0.0, 1.0, 0.0, 0.0], ky)
    assert np.isfinite(got).all()
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("k,sx,sy,c", [(3, 0.5, 2.0, 1), (5, 0.7, 2.5, 3), (7, 3.0, 1.0, 4), (5, 2.0, 0.9, 1)])
def test_oracle_u8_two_pass_kx_ne_ky(oracle, k, sx, sy, c):
    """gaussian_blur_u8 with equal sizes and different sigmas: the oracle applies kx along rows and ky along columns, as
    the independent numpy two-pass does, and the swapped taps give a different image."""
    img = np.random.default_rng(k * c).integers(0, 256, (23, 31, c), dtype=np.int64).astype(np.uint8)
    ikx = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(k, sx))
    iky = oracle.quantize_kernel_256(oracle.gaussian_kernel_1d(k, sy))
    got = oracle.gaussian_blur_u8(img, (k, k), (sx, sy))
    np.testing.assert_array_equal(got, _q8_two_pass_numpy(img, ikx, iky))
    assert not np.array_equal(got, _q8_two_pass_numpy(img, iky, ikx))
