"""Memory footprint of every entry point: what a call writes and reads AROUND its buffers, not only what it writes into them.

Every other GPU file compares the output tensor with the oracle.  A kernel that stores past its last row, leaves pixels
unwritten that a zero prefill happens to match, or taps the neighbouring frame at zero weight passes those comparisons.
Here each call gets its buffers inside one allocation laid out as [lead | region | tail] and is checked for:

  * writes outside the output: lead and tail (each one output row + 4 KiB or more) keep their prefill byte for byte;
  * unwritten output: the call runs once into 0x00 and once into 0xFF (NaN for f32 / f16 / bf16, 255 for u8), and the
    two regions must be bit-identical before they are compared with the oracle;
  * reads outside the input: the source region sits between poison (f32 NaN / +inf / -inf, u8 0xFF, u16 0xFFFF), and a
    batch of three tight frames has a poisoned middle frame; the outer frames must still give the oracle's bits.  The
    camera preprocess also gets poisoned pitch padding and poisoned gaps between strided frames;
  * the launcher's own length contract: every length passed is exactly the one computed here from the shapes, and the
    same call with one element less of `dst` or `src` is refused with the operand named, leaving every buffer untouched.

Every case asserts kb200_last_kernel(), so none passes on a path it does not claim.  The C ABI is called directly so
that every length is the test's own.

What poison cannot see: an out-of-bounds read whose value is masked out before it reaches a result.  The word-tap
windows of the u8 samplers and blurs read whole aligned words and discard the bytes they do not need, so a read of a
byte just past the source is invisible here; so is any read whose value is multiplied away by an integer zero weight.
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import Callable

import numpy as np
import pytest
import torch

from harness import FootprintCase, Guarded, OK, SLICE, as_bytes, assert_f32_bits_or_signed_zero, compare_to_oracle, dev, lib, neighbour_frames, poison, run_guarded
from restate import decode_direct, decode_yuv16, demosaic, filter_kernel, fused_schedule, pack, preprocess_rgb16, unpack


pytestmark = pytest.mark.gpu


# ── builders ────────────────────────────────────────────────────────────────────────────────────────────────────────
def o():
    from oracle import oracle
    return oracle


def pat_f32(n, seed):
    return o().pattern_f32(n, seed)


def pat_u8(n, seed):
    return o().pattern_u8(n, seed)


def img_f32(w, h, c, seed=1):
    return lambda k: pat_f32(w * h * c, seed + 31 * k).reshape(h, w, c)


def img_u8(w, h, c, seed=1):
    return lambda k: pat_u8(w * h * c, seed + 31 * k).reshape(h, w, c)


def f3(v):
    return (C.c_float * 3)(*[float(x) for x in v])


CASES = []


def add(*cases):
    CASES.extend(cases)


# fused u8 HWC -> CHW resize + normalize (f32 / f16 / bf16) ─────────────────────────────────────────────────────────
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
INV = tuple(float(np.float32(1.0) / np.float32(s)) for s in STD)   # Normalize::mean_inv_std


def fused_scale_bias():
    return o().normalize_params_from_mean_std(MEAN, STD)


def fused_oracle(dw, dh, out):
    def f(frame):
        sc, bi = fused_scale_bias()
        r = o().resize_normalize_u8_to_f32_chw(frame, dw, dh, sc, bi, 1)
        if out == "f32":
            return r
        return torch.from_numpy(r).to(torch.float16 if out == "f16" else torch.bfloat16).view(torch.uint16).numpy()
    return f


def fused_call(sw, sh, dw, dh, out, rows=None):
    def f(lib, s, sl, d, dl, n, aux):
        sc, bi = fused_scale_bias()
        if rows:
            return lib.kb200_resize_normalize_chw_u8_f32_rows(None, s, sl, d, dl, sw, sh, dw, dh, n, f3(sc), f3(bi), 1, *row_plan(sh, dh))
        fn = {"f32": lib.kb200_resize_normalize_chw_u8_f32, "f16": lib.kb200_resize_normalize_chw_u8_f16,
              "bf16": lib.kb200_resize_normalize_chw_u8_bf16}[out]
        return fn(None, s, sl, d, dl, sw, sh, dw, dh, n, f3(sc), f3(bi), 1)
    return f


def schedule_is(sw, sh, dw, dh, batch, mode):
    def check(dev):
        s = fused_schedule(sw, sh, dw, dh, batch, torch.cuda.get_device_properties(dev).multi_processor_count)
        assert s.mode == mode and s.ragged, f"{sw}x{sh}->{dw}x{dh}: {s}"
    return check


for out in ("f32", "f16", "bf16"):
    esz = 4 if out == "f32" else 2
    add(FootprintCase(f"fused-{out}-point-fullrow", "fused_rows_kernel", img_u8(384, 216, 3), fused_oracle(128, 72, out),
             fused_call(384, 216, 128, 72, out), 384 * 216 * 3, 3 * 128 * 72, knobs={"fr.rows": 2}, row=128 * esz))
    for mode, (sw, sh, dw, dh) in (("POINT", (384, 213, 128, 71)), ("BOX", (384, 142, 192, 71)), ("YZERO", (384, 213, 160, 71)),
                                   ("GENERAL", (384, 213, 160, 89))):
        add(FootprintCase(f"fused-{out}-tiled-{mode}", "fused_rows_kernel", img_u8(sw, sh, 3), fused_oracle(dw, dh, out),
                 fused_call(sw, sh, dw, dh, out), sw * sh * 3, 3 * dw * dh, batch=3, knobs={"fr.rows": 1}, row=dw * esz,
                 pre=schedule_is(sw, sh, dw, dh, 3, mode)))
    add(FootprintCase(f"fused-{out}-gather-unaligned-src", "fused_resize_gather_kernel", img_u8(384, 216, 3), fused_oracle(128, 72, out),
             fused_call(384, 216, 128, 72, out), 384 * 216 * 3, 3 * 128 * 72, offset=True, row=128 * esz))
add(FootprintCase("fused-f32-gather-row-bytes", "fused_resize_gather_kernel", img_u8(383, 216, 3), fused_oracle(128, 72, "f32"),
         fused_call(383, 216, 128, 72, "f32"), 383 * 216 * 3, 3 * 128 * 72, row=512))


def row_plan(sh, dh):
    """kb200_resize_row_plan: the periodic window of source rows the geometry taps."""
    from kornia_rs_b200 import _lib
    P, F, K = C.c_uint32(), C.c_uint32(), C.c_uint32()
    _lib.lib().kb200_resize_row_plan(sh, dh, C.byref(P), C.byref(F), C.byref(K))
    return P.value, F.value, K.value


def compacted(sw, sh, dh):
    def f(k):
        P, F, K = row_plan(sh, dh)
        assert (P, F, K) == (3, 1, 1), (P, F, K)   # 213 -> 71 is an exact 3:1 downscale: one row in three
        return img_u8(sw, sh, 3)(k).reshape(sh // P, P, sw, 3)[:, F:F + K].reshape(-1, sw, 3)
    return f


def _rows_case():
    sw, sh, dw, dh = 384, 213, 128, 71
    full = img_u8(sw, sh, 3)
    comp = compacted(sw, sh, dh)
    # the oracle needs the full frame: map a compacted frame back to the full one by its index
    lookup = {}

    def frame(k):
        c = comp(k)
        lookup[c.tobytes()[:64]] = k
        return c

    def oracle(c):
        k = lookup.get(c.tobytes()[:64])
        if k is None:   # a neighbour-test frame of constant bytes: every source row holds the same value
            f = np.broadcast_to(c.reshape(-1)[:1].reshape(1, 1, 1), (sh, sw, 3)).copy()
            return fused_oracle(dw, dh, "f32")(f)
        return fused_oracle(dw, dh, "f32")(full(k))

    return FootprintCase("fused-f32-rows-compacted", "fused_rows_kernel", frame, oracle, fused_call(sw, sh, dw, dh, "f32", rows=True),
                None, 3 * dw * dh, batch=3, row=dw * 4)


add(_rows_case())


# f32 resize ──────────────────────────────────────────────────────────────────────────────────────────────────────
def resize_oracle(dw, dh, mode=1):
    return lambda f: o().resize_f32(f, dw, dh, mode)


def resize_c3(fn, sw, sh, dw, dh):
    return lambda lib, s, sl, d, dl, n, aux: getattr(lib, fn)(None, s, sl, d, dl, sw, sh, dw, dh, n, 0)


add(FootprintCase("resize-rows-f32", "resize_rows_f32_kernel", img_f32(640, 360, 3), resize_oracle(212, 120),
         resize_c3("kb200_resize_bilinear_f32_c3", 640, 360, 212, 120), 640 * 360 * 3, 212 * 120 * 3, batch=3, row=212 * 12),
    FootprintCase("resize-rows-f32-ragged", "resize_rows_f32_kernel", img_f32(1280, 16, 3), resize_oracle(1000, 37),
         resize_c3("kb200_resize_bilinear_f32_c3", 1280, 16, 1000, 37), 1280 * 16 * 3, 1000 * 37 * 3, batch=3, row=12000),
    FootprintCase("resize-c3-gather", "resize_f32_c3_kernel", img_f32(129, 97, 3), resize_oracle(64, 48),
         resize_c3("kb200_resize_bilinear_f32_c3", 129, 97, 64, 48), 129 * 97 * 3, 64 * 48 * 3, row=64 * 12),
    FootprintCase("resize-c3-unaligned", "resize_f32_c3_kernel", img_f32(128, 96, 3), resize_oracle(64, 48),
         resize_c3("kb200_resize_bilinear_f32_c3", 128, 96, 64, 48), 128 * 96 * 3, 64 * 48 * 3, offset=True, row=64 * 12),
    FootprintCase("resize-nearest-c3", ("resize_f32_c3_kernel", "resize_rows_f32_kernel"), img_f32(129, 97, 3), resize_oracle(61, 45, 0),
         resize_c3("kb200_resize_nearest_f32_c3", 129, 97, 61, 45), 129 * 97 * 3, 61 * 45 * 3, row=61 * 12))
for c in (1, 2, 4):
    add(FootprintCase(f"resize-generic-c{c}", "resize_f32_generic_kernel", img_f32(131, 67, c), resize_oracle(70, 33),
             lambda lib, s, sl, d, dl, n, aux, c=c: lib.kb200_resize_f32(None, s, sl, d, dl, 131, 67, 70, 33, c, n, 1),
             131 * 67 * c, 70 * 33 * c, row=70 * 4 * c))
add(FootprintCase("resize-bicubic", "resize_bicubic_c3_kernel", img_f32(129, 97, 3), resize_oracle(61, 45, 2),
         lambda lib, s, sl, d, dl, n, aux: lib.kb200_resize_bicubic_f32_c3(None, s, sl, d, dl, 129, 97, 61, 45, n),
         129 * 97 * 3, 61 * 45 * 3, row=61 * 12))


def _lanczos():
    sw, sh, dw, dh = 129, 97, 61, 45

    def scratch_len(lib, b):   # floats, passed exactly
        return lib.kb200_resize_lanczos_scratch_len(sh, dw, dh, b)

    return FootprintCase("resize-lanczos", "resize_lanczos_kernels", img_f32(sw, sh, 3), resize_oracle(dw, dh, 3),
                lambda lib, s, sl, d, dl, b, aux: lib.kb200_resize_lanczos_f32_c3(None, s, sl, d, dl, aux["scratch"], scratch_len(lib, b),
                                                                                  sw, sh, dw, dh, b),
                sw * sh * 3, dw * dh * 3, aux={"scratch": lambda lib, b: 4 * scratch_len(lib, b)}, row=dw * 12)


def _bn_oracle(dw, dh):
    def f(frame):
        base = o().resize_f32(frame, dw, dh)
        inv = np.float32(1.0) / np.array(STD, np.float32)
        return ((base - np.array(MEAN, np.float32)) * inv).astype(np.float32)
    return f


add(FootprintCase("resize-bilinear-normalize", "resize_rows_f32_kernel", img_f32(640, 360, 3), _bn_oracle(320, 180),
         lambda lib, s, sl, d, dl, n, aux: lib.kb200_resize_bilinear_normalize_f32_c3(None, s, sl, d, dl, 640, 360, 320, 180, n, f3(MEAN), f3(STD), 0),
         640 * 360 * 3, 320 * 180 * 3, batch=3, row=320 * 12))


# u8 resize ───────────────────────────────────────────────────────────────────────────────────────────────────────
for c in (1, 3, 4):
    add(FootprintCase(f"resize-bilinear-u8-c{c}", ("resize_bilinear_u8_kernel", "resize_bilinear_u8_c3_3to1_kernel"), img_u8(101, 67, c),
             lambda f: o().resize_bilinear_u8(f, 45, 29),
             lambda lib, s, sl, d, dl, n, aux, c=c: lib.kb200_resize_bilinear_u8(None, s, sl, d, dl, 101, 67, 45, 29, c, n),
             101 * 67 * c, 45 * 29 * c, batch=3, row=45 * c))
for name, (sw, sh, dw, dh, interp, kern) in {
        "2to1": (202, 134, 101, 67, 1, ("pyrdown_2x_rgb_u8_w4_kernel", "pyrdown_2x_rgb_u8_kernel")),
        "2to1-odd": (198, 134, 99, 67, 1, ("pyrdown_2x_rgb_u8_w4_kernel", "pyrdown_2x_rgb_u8_kernel")),
        "up2": (101, 67, 202, 134, 1, "pyrup_2x_rgb_u8_kernel"),
        "3to1": (300, 201, 100, 67, 1, "resize_bilinear_u8_c3_3to1_kernel"),
        "nearest": (101, 67, 45, 29, 0, "resize_nearest_u8_kernel")}.items():
    add(FootprintCase(f"resize-fast-u8-{name}", kern, img_u8(sw, sh, 3), lambda f, dw=dw, dh=dh, i=interp: o().resize_fast_u8(f, dw, dh, i),
             lambda lib, s, sl, d, dl, n, aux, a=(sw, sh, dw, dh, interp): lib.kb200_resize_fast_u8(None, s, sl, d, dl, *a[:4], 3, n, a[4]),
             sw * sh * 3, dw * dh * 3, batch=3, row=dw * 3))


# f32 warps ───────────────────────────────────────────────────────────────────────────────────────────────────────
H_GENTLE = [1.02, 0.03, -7.0, -0.03, 1.01, 4.0, 1.2e-5, 7.0e-6, 1.0]
H_ZOOM_OUT = [0.6, 0.02, 30.0, -0.01, 0.7, 20.0, 0, 0, 1]       # the destination's border maps outside the source


def warp_f32(kind, m, sw, sh, dw, dh, interp=1):
    fn = "kb200_warp_affine_f32_c3" if kind == "affine" else "kb200_warp_perspective_f32_c3"
    n_m = 6 if kind == "affine" else 9
    return lambda lib, s, sl, d, dl, n, aux: getattr(lib, fn)(None, s, sl, d, dl, sw, sh, dw, dh, n, (C.c_float * n_m)(*m), interp)


def warp_oracle(kind, m, dw, dh, mode=1):
    fn = o().warp_affine_f32 if kind == "affine" else o().warp_perspective_f32
    return lambda f: fn(f, m, dw, dh, mode)


def _warps():
    sw, sh = 389, 211
    rot = o().get_rotation_matrix2d((sw / 2.0, sh / 2.0), 3.0, 0.8)
    aff = [float(v) for v in rot]
    aff_tiled = [float(v) for v in o().get_rotation_matrix2d((128.0, 96.0), 30.0, 1.0)]
    lean, gen = "warp_bilinear_lean_kernel", "warp_bilinear_lean_kernel/general"
    for kind, m in (("affine", aff), ("perspective", H_ZOOM_OUT)):
        # dw, dh % 32 != 0: 388x200 (dh % 8 == 0) stores through the 4-D map, 388x203 through four 1-D row copies, 333x203 with STG.
        # The 4-D map store and the row copies report the same kernel tag, and launch_lean falls back to the row copies when
        # the tensor map cannot be encoded, so for 388x200 the tag proves a TMA store ran, not which of the two.
        for dw, dh in ((388, 200), (388, 203), (333, 203)):
            tag = f"{kind}-{dw}x{dh}"
            stg = "" if dw % 4 == 0 else "/stg"
            for a, want in ((0, (lean + stg, gen + stg)), (7, (lean + stg, gen + stg)), (5, (lean + "/stg", gen + "/stg")),
                            (4, (gen + stg,))):
                add(FootprintCase(f"warp-{tag}-lean-a{a}", want, img_f32(sw, sh, 3), warp_oracle(kind, m, dw, dh), warp_f32(kind, m, sw, sh, dw, dh),
                         sw * sh * 3, dw * dh * 3, knobs={"warp.path": 1, "a": a}, row=dw * 12))
            add(FootprintCase(f"warp-{tag}-lean-unaligned", (lean + "/stg", gen + "/stg"), img_f32(sw, sh, 3), warp_oracle(kind, m, dw, dh),
                     warp_f32(kind, m, sw, sh, dw, dh), sw * sh * 3, dw * dh * 3, offset=True, knobs={"warp.path": 1}, row=dw * 12))
        # the streaming kernels take gentle maps only: a small rotation (affine) and a zoom-out (perspective), borders outside
        ssw, ssh, sdw, sdh = (512, 300, 480, 260) if kind == "affine" else (388, 211, 388, 211)
        sm = [float(v) for v in o().get_rotation_matrix2d((256.0, 150.0), -3.5, 0.9)] if kind == "affine" else H_ZOOM_OUT
        for interp, kern in ((1, "warp_stream2_kernel"), (0, "warp_stream_kernel")):
            add(FootprintCase(f"warp-{kind}-stream-i{interp}", kern, img_f32(ssw, ssh, 3), warp_oracle(kind, sm, sdw, sdh, interp),
                     warp_f32(kind, sm, ssw, ssh, sdw, sdh, interp), ssw * ssh * 3, sdw * sdh * 3, knobs={"warp.path": 3}, row=sdw * 12))
        add(FootprintCase(f"warp-{kind}-tiled", "warp_tiled_kernel", img_f32(256, 192, 3),
                 warp_oracle(kind, aff_tiled if kind == "affine" else [0.8, 0.45, -20.0, -0.5, 0.85, 60.0, 1.0e-4, -6.0e-5, 1.0], 227, 181),
                 warp_f32(kind, aff_tiled if kind == "affine" else [0.8, 0.45, -20.0, -0.5, 0.85, 60.0, 1.0e-4, -6.0e-5, 1.0], 256, 192, 227, 181),
                 256 * 192 * 3, 227 * 181 * 3, knobs={"warp.path": 2}, row=227 * 12))
        for interp, kern in ((2, "warp_bicubic_kernel"), (3, "warp_lanczos_kernel")):
            add(FootprintCase(f"warp-{kind}-hq{interp}", kern, img_f32(97, 61, 3), warp_oracle(kind, m if kind == "perspective" else
                                                                                        [float(v) for v in o().get_rotation_matrix2d((48.5, 30.5), 30.0, 0.9)], 80, 70, interp),
                     warp_f32(kind, m if kind == "perspective" else [float(v) for v in o().get_rotation_matrix2d((48.5, 30.5), 30.0, 0.9)], 97, 61, 80, 70, interp),
                     97 * 61 * 3, 80 * 70 * 3, row=80 * 12))


# u8 warps and remaps ─────────────────────────────────────────────────────────────────────────────────────────────
def _u8_warps():
    sw, sh, dw, dh = 131, 77, 121, 63      # frames of sw*sh*C bytes: not a multiple of 4 for C = 1, 3
    m = [float(v) for v in o().get_rotation_matrix2d((65.5, 38.5), 7.0, 0.8)]
    for c in (1, 3, 4):
        for b in (0, 1):
            kn = {"b": 1} if b else {}
            add(FootprintCase(f"warp-affine-u8-c{c}-b{b}", "warp_affine_u8_kernel", img_u8(sw, sh, c), lambda f: o().warp_affine_u8(f, dw, dh, m),
                     lambda lib, s, sl, d, dl, n, aux, c=c: lib.kb200_warp_affine_u8(None, s, sl, d, dl, sw, sh, dw, dh, c, n, (C.c_float * 6)(*m)),
                     sw * sh * c, dw * dh * c, batch=3, knobs=kn, row=dw * c))
            add(FootprintCase(f"warp-perspective-u8-c{c}-b{b}", "warp_perspective_u8_kernel", img_u8(sw, sh, c),
                     lambda f: o().warp_perspective_u8(f, dw, dh, H_ZOOM_OUT),
                     lambda lib, s, sl, d, dl, n, aux, c=c: lib.kb200_warp_perspective_u8(None, s, sl, d, dl, sw, sh, dw, dh, c, n, (C.c_float * 9)(*H_ZOOM_OUT)),
                     sw * sh * c, dw * dh * c, batch=3, knobs=kn, row=dw * c))


def radial(sw, sh, dw, dh):
    yy, xx = np.mgrid[0:dh, 0:dw].astype(np.float32)
    cx, cy = np.float32(dw / 2), np.float32(dh / 2)
    r = ((xx - cx) ** 2 + (yy - cy) ** 2) / np.float32(dw * dw)
    k = np.float32(1.0) + np.float32(0.3) * r
    mx = (cx + (xx - cx) * k) * np.float32(sw / dw)
    my = (cy + (yy - cy) * k) * np.float32(sh / dh)
    mx[0, 0], my[1, 1] = np.nan, -3.0        # a NaN coordinate and one left of the source: 0
    return mx.astype(np.float32), my.astype(np.float32)


def _remaps():
    sw, sh, dw, dh = 131, 77, 121, 63
    mx, my = radial(sw, sh, dw, dh)
    aux = {"mx": (mx, "f32"), "my": (my, "f32")}
    for interp, kerns in ((1, ("remap_lean_kernel", "remap_lean_kernel/general", "remap_lean_kernel/stg", "remap_lean_kernel/general/stg")),
                          (0, "remap_f32_c3_kernel")):
        add(FootprintCase(f"remap-f32-i{interp}", kerns, img_f32(sw, sh, 3), lambda f, i=interp: o().remap(f, mx, my, i),
                 lambda lib, s, sl, d, dl, n, aux, i=interp: lib.kb200_remap_f32_c3(None, s, sl, d, dl, aux["mx"], aux["my"], dw * dh, sw, sh, dw, dh, n, i),
                 sw * sh * 3, dw * dh * 3, aux=aux, row=dw * 12))
    add(FootprintCase("remap-f32-thread-per-pixel", "remap_f32_c3_kernel", img_f32(sw, sh, 3), lambda f: o().remap(f, mx, my, 1),
             lambda lib, s, sl, d, dl, n, aux: lib.kb200_remap_f32_c3(None, s, sl, d, dl, aux["mx"], aux["my"], dw * dh, sw, sh, dw, dh, n, 1),
             sw * sh * 3, dw * dh * 3, aux=aux, knobs={"a": 6}, row=dw * 12))
    for c in (1, 3, 4):
        for b in (0, 1, 2):
            add(FootprintCase(f"remap-u8-c{c}-b{b}", "remap_u8_kernel", img_u8(sw, sh, c), lambda f: o().remap(f, mx, my, 1),
                     lambda lib, s, sl, d, dl, n, aux, c=c: lib.kb200_remap_u8(None, s, sl, d, dl, aux["mx"], aux["my"], dw * dh, sw, sh, dw, dh, c, n, 1),
                     sw * sh * c, dw * dh * c, batch=3, aux=aux, knobs={"b": b} if b else {}, row=dw * c))


# filters ─────────────────────────────────────────────────────────────────────────────────────────────────────────
def _filters():
    for w, h, c in ((700, 37, 3), (97, 61, 3), (1100, 21, 1), (33, 50, 4)):
        add(FootprintCase(f"gaussian-f32-{w}x{h}x{c}", filter_kernel(w, c, "gauss5"), img_f32(w, h, c), lambda f: o().gaussian_blur(f, (5, 5), (1.5, 1.5)),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h, c): lib.kb200_gaussian_blur_f32(None, s, sl, d, dl, *a, n, 5, 5, 1.5, 1.5),
                 w * h * c, w * h * c, row=w * c * 4),
            FootprintCase(f"sobel-f32-{w}x{h}x{c}", filter_kernel(w, c, "sobel3"), img_f32(w, h, c), lambda f: o().sobel(f, 3),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h, c): lib.kb200_sobel_f32(None, s, sl, d, dl, *a, n, 3),
                 w * h * c, w * h * c, row=w * c * 4))
    kx = np.array([0.25, 0.5, 0.25, 0.125], np.float32)
    ky = np.array([-1.0, 0.0, 2.0], np.float32)
    for (w, h, c), off, kern in (((700, 37, 3), False, "sep_filter_fused_kernel"), ((700, 37, 3), True, "sep_filter_fused_kernel")):
        add(FootprintCase(f"separable-f32-{'unaligned' if off else 'aligned'}", kern, img_f32(w, h, c), lambda f: o().separable_filter(f, kx, ky),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h, c): lib.kb200_separable_filter_f32(
                     None, s, sl, d, dl, None, kx.ctypes.data_as(C.POINTER(C.c_float)), 4, ky.ctypes.data_as(C.POINTER(C.c_float)), 3, *a, n),
                 w * h * c, w * h * c, offset=off, row=w * c * 4))
    # u8 blurs: stream (16-B rows and bases), word (4-B), byte tile (odd row bytes), and the tile kernel forced (b = 3)
    for (w, h, c), off, kn, kern in (((320, 37, 3), False, {}, "blur_u8_stream_kernel"), ((320, 37, 3), False, {"b": 3}, "blur_u8_tile_w_kernel"),
                                     ((97, 33, 4), False, {}, "blur_u8_tile_w_kernel"), ((97, 33, 3), False, {}, "blur_u8_tile_kernel"),
                                     ((320, 37, 3), True, {}, "blur_u8_tile_kernel")):
        tag = f"{w}x{h}x{c}{'-unaligned' if off else ''}{'-b3' if kn else ''}"
        add(FootprintCase(f"gaussian-u8-{tag}", kern, img_u8(w, h, c), lambda f: o().gaussian_blur_u8(f, (5, 5), (1.5, 1.5)),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h, c): lib.kb200_gaussian_blur_u8(None, s, sl, d, dl, *a, n, 5, 5, 1.5, 1.5),
                 w * h * c, w * h * c, batch=3, offset=off, knobs=kn, row=w * c),
            FootprintCase(f"box-u8-{tag}", kern, img_u8(w, h, c), lambda f: o().box_blur_u8(f, (3, 3)),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h, c): lib.kb200_box_blur_u8(None, s, sl, d, dl, *a, n, 3, 3),
                 w * h * c, w * h * c, batch=3, offset=off, knobs=kn, row=w * c))


# colour ──────────────────────────────────────────────────────────────────────────────────────────────────────────
L420 = ("Nv12", "Nv21", "I420", "Yv12")
L422 = ("Yuyv", "Uyvy", "Yvyu")


def _colour():
    for i, lay in enumerate(L420):
        for (w, h), off, v in (((64, 48), False, "vec16"), ((70, 6), False, "generic"), ((64, 48), True, "generic")):
            add(FootprintCase(f"yuv420-{lay}-{w}x{h}{'-unaligned' if off else ''}", f"rgb_from_{lay.lower()}_{v}",
                     lambda k, w=w, h=h: pat_u8(w * h * 3 // 2, 40 + k), lambda f, w=w, h=h, lay=lay: decode_direct(f, w, h, lay),
                     lambda lib, s, sl, d, dl, n, aux, a=(w, h, i): lib.kb200_rgb_from_yuv420_u8(None, s, sl, d, dl, a[0], a[1], n, a[2]),
                     w * h * 3 // 2, w * h * 3, batch=3, offset=off, row=w * 3))
    for i, lay in enumerate(L422):
        # 64x48: whole vectors; 70x5 x3: the vec16 body and a generic tail (the generic kernel runs last); unaligned: generic
        for (w, h), off, v in (((64, 48), False, "vec16"), ((70, 5), False, "generic"), ((64, 48), True, "generic")):
            add(FootprintCase(f"yuv422-{lay}-{w}x{h}{'-unaligned' if off else ''}", f"rgb_from_{lay.lower()}_{v}",
                     lambda k, w=w, h=h: pat_u8(w * h * 2, 50 + k), lambda f, w=w, h=h, lay=lay: decode_direct(f, w, h, lay),
                     lambda lib, s, sl, d, dl, n, aux, a=(w, h, i): lib.kb200_rgb_from_yuv422_u8(None, s, sl, d, dl, a[0], a[1], n, a[2]),
                     w * h * 2, w * h * 3, batch=3, offset=off, row=w * 3))
    for (w, h), off, v in (((64, 48), False, "vec16"), ((70, 7), False, "generic"), ((64, 48), True, "generic")):
        add(FootprintCase(f"bayer-u8-{w}x{h}{'-unaligned' if off else ''}", (f"rgb_from_bayer_grbg_{v}",), lambda k, w=w, h=h: pat_u8(w * h, 60 + k).reshape(h, w),
                 lambda f: demosaic(f, "GRBG").astype(np.uint8),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h): lib.kb200_rgb_from_bayer_u8(None, s, sl, d, dl, a[0], a[1], n, 2),
                 w * h, w * h * 3, batch=3, offset=off, row=w * 3))
        add(FootprintCase(f"bayer-u16-{w}x{h}{'-unaligned' if off else ''}", f"rgb_from_bayer16_gbrg_{'vec' if v == 'vec16' else v}",
                 lambda k, w=w, h=h: (pat_u8(w * h * 2, 70 + k).view(np.uint16) & 0x0FFF).reshape(h, w),
                 lambda f: demosaic(f, "GBRG").astype(np.uint16),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h): lib.kb200_rgb_from_bayer_u16(None, s, sl, d, dl, a[0], a[1], n, 3),
                 w * h, w * h * 3, batch=3, offset=off, row=w * 6))
    for bits, (w, h), off, v in ((10, (128, 6), False, "vec"), (12, (36, 5), False, "generic"), (14, (128, 6), True, "generic")):
        rb = w * bits // 8
        add(FootprintCase(f"bayer-packed{bits}-{w}x{h}{'-unaligned' if off else ''}", f"rgb_from_bayer{bits}p_rggb_{v}",
                 lambda k, w=w, h=h, bits=bits: pack(np.random.default_rng(80 + k).integers(0, 1 << bits, (h, w)), bits),
                 lambda f, bits=bits: demosaic(unpack_np(f, bits), "RGGB").astype(np.uint16),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h, bits): lib.kb200_rgb_from_bayer_packed(None, s, sl, d, dl, a[0], a[1], n, 0, a[2]),
                 rb * h, w * h * 3, batch=3, offset=off, row=w * 6))
    for fmt, (w, h), off, v in (("P010", (64, 48), False, "vec"), ("I012", (70, 4), False, "generic"), ("P010", (64, 16), True, "generic")):
        lay, bits = (0, 10) if fmt == "P010" else (1, 12)
        add(FootprintCase(f"yuv420-u16-{fmt}-{w}x{h}{'-unaligned' if off else ''}", f"rgb_from_{fmt[0].lower()}01x_{v}",
                 lambda k, w=w, h=h: pat_u8(w * h * 3, 90 + k).view(np.uint16).copy(),
                 lambda f, w=w, h=h, fmt=fmt: decode_yuv16(torch.from_numpy(f.astype(np.int32)), w, h, fmt, "Bt601Limited").numpy().astype(np.uint16),
                 lambda lib, s, sl, d, dl, n, aux, a=(w, h, lay, bits): lib.kb200_rgb_from_yuv420_u16(None, s, sl, d, dl, a[0], a[1], n, a[2], a[3], 0),
                 w * h * 3 // 2, w * h * 3, batch=3, offset=off, row=w * 6))
    add(FootprintCase("nv12-from-rgb", "nv12_from_rgb_kernel", img_u8(70, 6, 3), lambda f: o().nv12_from_rgb(f),
             lambda lib, s, sl, d, dl, n, aux: lib.kb200_nv12_from_rgb_u8(None, s, sl, d, dl, 70, 6, n), 70 * 6 * 3, 70 * 6 * 3 // 2, batch=3, row=70),
        FootprintCase("yuyv-from-rgb", "yuyv_from_rgb_kernel", img_u8(70, 5, 3), lambda f: o().yuyv_from_rgb(f),
             lambda lib, s, sl, d, dl, n, aux: lib.kb200_yuyv_from_rgb_u8(None, s, sl, d, dl, 70, 5, n), 70 * 5 * 3, 70 * 5 * 2, batch=3, row=140))
    for off, kf, ku in ((False, "gray_from_rgb_f32_vec4", "gray_from_rgb_u8_vec16"), (True, "gray_from_rgb_f32_scalar", "gray_from_rgb_u8_scalar")):
        tag = "unaligned" if off else "aligned"
        add(FootprintCase(f"gray-f32-{tag}", kf, img_f32(64, 32, 3), lambda f: o().gray_from_rgb_f32(f, 1),
                 lambda lib, s, sl, d, dl, n, aux: lib.kb200_gray_from_rgb_f32(None, s, sl, d, dl, 64 * 32 * n, 1), 64 * 32 * 3, 64 * 32,
                 batch=3, offset=off, row=64 * 4),
            FootprintCase(f"gray-u8-{tag}", ku, img_u8(64, 32, 3), lambda f: o().gray_from_rgb_u8(f),
                 lambda lib, s, sl, d, dl, n, aux: lib.kb200_gray_from_rgb_u8(None, s, sl, d, dl, 64 * 32 * n), 64 * 32 * 3, 64 * 32,
                 batch=3, offset=off, row=64))


def unpack_np(raw, bits):
    return unpack(raw, bits).astype(np.int64)


# statistics (entry points without lengths: npixels) ──────────────────────────────────────────────────────────────
def _stats():
    for off, kern in ((False, "normalize_mean_std_c3_vec"), (True, "normalize_mean_std_generic")):
        add(FootprintCase(f"normalize-mean-std-{'unaligned' if off else 'aligned'}", kern, img_f32(64, 32, 3), lambda f: o().normalize_mean_std(f, MEAN, STD),
                 lambda lib, s, sl, d, dl, n, aux: lib.kb200_normalize_mean_std_f32(None, s, d, 64 * 32 * n, 3, f3(MEAN), f3(STD)),
                 64 * 32 * 3, 64 * 32 * 3, batch=3, offset=off, lengths=False, row=64 * 12))
    sc, bi = (0.017, 0.018, 0.019), (-2.1, -2.0, -1.8)
    for off, kern in ((False, "normalize_rgb_u8_vec"), (True, "normalize_rgb_u8_generic")):
        add(FootprintCase(f"normalize-rgb-u8-{'unaligned' if off else 'aligned'}", kern, img_u8(64, 32, 3), lambda f: o().normalize_rgb_u8(f, sc, bi, 1),
                 lambda lib, s, sl, d, dl, n, aux: lib.kb200_normalize_rgb_u8_f32(None, s, d, 64 * 32 * n, f3(sc), f3(bi), 1),
                 64 * 32 * 3, 64 * 32 * 3, batch=3, offset=off, lengths=False, row=64 * 12))
    measured = np.array(o().find_min_max(img_f32(64, 32, 3)(0)), np.float32)   # what find_min_max leaves in the device pair
    add(FootprintCase("normalize-min-max", "normalize_min_max_kernel", img_f32(64, 32, 3), lambda f: o().normalize_min_max(f, -1.0, 2.0),
             lambda lib, s, sl, d, dl, n, aux: lib.kb200_normalize_min_max_f32(None, s, d, 64 * 32 * 3 * n, -1.0, 2.0, aux["mm"]),
             64 * 32 * 3, 64 * 32 * 3, batch=1, lengths=False, aux={"mm": (measured, "f32")}, row=64 * 12))


# pyramids ────────────────────────────────────────────────────────────────────────────────────────────────────────
def _pyramids():
    for c in (1, 2, 3, 4):
        w, h = 53, 37
        dw, dh = (w + 1) // 2, (h + 1) // 2
        for dt, img in (("f32", img_f32), ("u8", img_u8)):
            esz = 4 if dt == "f32" else 1
            add(FootprintCase(f"pyrdown-{dt}-c{c}", f"pyrdown_{dt}_kernel", img(w, h, c), getattr(o(), f"pyrdown_{dt}"),
                     lambda lib, s, sl, d, dl, n, aux, c=c, dt=dt: getattr(lib, f"kb200_pyrdown_{dt}")(None, s, sl, d, dl, w, h, c, n),
                     w * h * c, dw * dh * c, batch=3, row=dw * c * esz),
                FootprintCase(f"pyrup-{dt}-c{c}", f"pyrup_{dt}_kernel", img(w, h, c), getattr(o(), f"pyrup_{dt}"),
                     lambda lib, s, sl, d, dl, n, aux, c=c, dt=dt: getattr(lib, f"kb200_pyrup_{dt}")(None, s, sl, d, dl, w, h, c, n),
                     w * h * c, 4 * w * h * c, batch=3, row=2 * w * c * esz))


def _fusion():
    sc, bi = fused_scale_bias()
    for sink, maps in ((0, 1), (1, 4)):
        add(FootprintCase(f"fused-pipeline-sink{sink}", "fused_pipeline_kernel", img_u8(131, 77, 3),
                 lambda f, sink=sink, maps=maps: o().fused_pipeline_u8(f, 61, 37, maps, sc, bi, sink),
                 lambda lib, s, sl, d, dl, n, aux, sink=sink, maps=maps: lib.kb200_fused_pipeline_u8_f32(None, s, sl, d, dl, 131, 77, 61, 37, n, maps,
                                                                                                       f3(sc), f3(bi), sink),
                 131 * 77 * 3, 61 * 37 * (3 if sink == 0 else 1), batch=3, row=61 * 4))


for build in (_warps, _u8_warps, _remaps, _filters, _colour, _stats, _pyramids, _fusion):
    build()
add(_lanczos())

IDS = [c.id for c in CASES]
assert len(set(IDS)) == len(IDS), "case ids must be unique"
BY_ID = {c.id: c for c in CASES}


@pytest.mark.parametrize("cid", IDS)
def test_footprint(kb, lib, dev, cid):
    """Guards, unwritten output, poisoned surroundings and the exact length contract, on a tight batch."""
    case = BY_ID[cid]
    if case.pre:
        case.pre(dev)
    frames = [case.frame(k) for k in range(case.batch)]
    run_guarded(kb, lib, dev, case, frames, range(case.batch), True)


NEIGHBOUR_IDS = [c.id for c in CASES if c.batch > 1]


@pytest.mark.parametrize("cid", NEIGHBOUR_IDS)
def test_poisoned_neighbour_frame(kb, lib, dev, cid):
    """Three tight frames, the middle one poisoned (f32 all NaN between finite frames; integer all max between all 0): the outer
    frames' results must not see it."""
    case = BY_ID[cid]
    run_guarded(kb, lib, dev, case, neighbour_frames(case), (0, 2), False)


# ── result buffers of the reductions and the map generator ─────────────────────────────────────────────────────────
def test_find_min_max_result_guards(kb, lib, dev):
    src = pat_f32(67 * 33 * 3, 5)
    g = Guarded(dev, src.nbytes).load("f32", as_bytes(src))
    for fill in (0x00, 0xFF):
        out = Guarded(dev, 8).fill(fill)
        assert lib.kb200_find_min_max_f32(None, g.ptr, src.size, out.ptr) == OK
        assert kb._lib.last_kernel() == "minmax_kernel"
        torch.cuda.synchronize()
        lead, tail = out.guards()
        assert np.all(lead == fill) and np.all(tail == fill)
        assert tuple(out.out().view(np.float32)) == tuple(np.float32(v) for v in o().find_min_max(src))


@pytest.mark.parametrize("off", [0, 1, 2, 3, 5])
def test_std_mean_result_guards(kb, lib, dev, off):
    npx = 4096 * 3 + 7
    src = pat_u8(npx * 3, 4242)
    g = Guarded(dev, src.nbytes, offset=off).load("u8", src)
    before = g.snapshot()
    for fill in (0x00, 0xFF):
        out = Guarded(dev, 48).fill(fill)
        assert lib.kb200_std_mean_u8_c3(None, g.ptr, npx, out.ptr) == OK
        assert kb._lib.last_kernel() == "std_mean_kernel"
        torch.cuda.synchronize()
        lead, tail = out.guards()
        assert np.all(lead == fill) and np.all(tail == fill)
        assert out.out().view(np.uint64).tolist() == [int(v) for v in o().std_mean(src.reshape(1, npx, 3))[2]]
    assert np.array_equal(g.snapshot(), before)


@pytest.mark.parametrize("w,h", [(8, 4), (641, 479)])
def test_correction_map_guards(kb, lib, dev, w, h):
    intr = (C.c_double * 4)(577.48583984375, 652.8748779296875, 577.48583984375, 386.1428833007813)
    dist = (C.c_double * 8)(1.75, 0.0098, -0.027, 2.1, 0.46, -0.082, -5.5e-5, 3.0e-5)
    ox, oy = o().generate_correction_map_polynomial(list(intr), list(dist), w, h)
    outs = []
    for fill in (0x00, 0xFF):
        mx, my = Guarded(dev, w * h * 4, w * 4).fill(fill), Guarded(dev, w * h * 4, w * 4).fill(fill)
        assert lib.kb200_generate_correction_map_polynomial(None, intr, dist, w, h, mx.ptr, my.ptr, w * h) == OK
        assert kb._lib.last_kernel() == "correction_map_kernel"
        torch.cuda.synchronize()
        for g in (mx, my):
            lead, tail = g.guards()
            assert np.all(lead == fill) and np.all(tail == fill)
        outs.append((mx.out(), my.out()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    assert_f32_bits_or_signed_zero(outs[0][0].view(np.float32), ox.reshape(-1), "map_x")
    assert_f32_bits_or_signed_zero(outs[0][1].view(np.float32), oy.reshape(-1), "map_y")
    mx.fill(0x5A)
    assert lib.kb200_generate_correction_map_polynomial(None, intr, dist, w, h, mx.ptr, my.ptr, w * h - 1) == SLICE
    assert "'map'" in kb._lib.last_error()


def test_gradient_magnitude_guards(kb, lib, dev):
    n = 67 * 33 * 3
    gx, gy = pat_f32(n, 1), pat_f32(n, 2)
    a, b = Guarded(dev, gx.nbytes).load("f32", as_bytes(gx)), Guarded(dev, gy.nbytes).load("f32", as_bytes(gy))
    want = np.sqrt(gx.astype(np.float32) * gx + gy * gy).astype(np.float32)
    outs = []
    for fill in (0x00, 0xFF):
        d = Guarded(dev, gx.nbytes).fill(fill)
        assert lib.kb200_gradient_magnitude_f32(None, a.ptr, b.ptr, d.ptr, n) == OK
        assert kb._lib.last_kernel() == "gradient_magnitude_kernel"
        torch.cuda.synchronize()
        lead, tail = d.guards()
        assert np.all(lead == fill) and np.all(tail == fill)
        outs.append(d.out())
    assert np.array_equal(outs[0], outs[1])
    assert_f32_bits_or_signed_zero(outs[0].view(np.float32), want, "gradient magnitude")


# ── camera preprocess: pitch padding, strided gaps, one guarded buffer per frame, and the host entries ─────────────
PP = {   # name -> (fmt code, src_bpp, w, h)
    "rgb": (0, 3, 64, 48), "gray": (2, 1, 64, 48), "nv12": (3, 1, 64, 48), "yuyv": (4, 2, 64, 48),
    "bayer8": (18, 1, 64, 48), "bayer16": (36, 2, 64, 48), "bayer12p": (68, 1, 64, 48), "p010": (80, 2, 64, 48),
}
TIGHT = ("nv12", "yuyv", "p010")        # frames that must be tightly packed (src_pitch == width * bpp)


def pp_desc(lib, name, mode, dw, dh, pitch_pad=0, sampling=1):
    fmt, bpp, w, h = PP[name]
    d = o().make_desc(o().PreprocessCfg(mode=mode, fmt=0, bpp=3, mean=MEAN, inv_std=INV), w, h, dw, dh)
    row = w * 12 // 8 if name == "bayer12p" else w * bpp
    d.fmt, d.src_bpp, d.src_pitch, d.sampling = fmt, bpp, row + (0 if name in TIGHT else pitch_pad), sampling
    from kornia_rs_b200._lib import PreprocessDesc
    k = PreprocessDesc()
    for f, _ in PreprocessDesc._fields_:
        setattr(k, f, getattr(d, f))
    return k


def pp_frame(name, d, k):
    """One frame's bytes, pitch padding included (filled later with poison)."""
    n = lib_src_bytes(d)
    return pat_u8(n, 0x7000 + 97 * k) if name not in ("bayer16", "p010") else (pat_u8(n, 0x7000 + 97 * k).view(np.uint16) & 0x0FFF).view(np.uint8)


def lib_src_bytes(d):
    from kornia_rs_b200 import _lib
    return _lib.lib().kb200_preprocess_src_bytes(C.byref(d))


def pp_poison_padding(frame, d):
    """The bytes between w*bpp and the pitch of every row -> 0xFF."""
    fmt, bpp, w = d.fmt, d.src_bpp, d.src_w
    row = w * 12 // 8 if fmt == 68 else w * bpp
    f = frame.copy()
    if d.src_pitch > row:
        rows = f[:d.src_pitch * d.src_h].reshape(d.src_h, d.src_pitch)
        rows[:, row:] = 0xFF
    return f


def pp_oracle(name, d, mode, frame, f16):
    """The oracle of one frame, (3, dh, dw): oracle.preprocess_frame for the formats it reads (RGB, Gray, NV12, YUYV) and, for
    Bayer 8-bit, on the demosaiced RGB twin; the float restatement of test_bayer16 on the decoded 16-bit RGB twin for 12-bit
    Bayer, packed 12-bit Bayer and P010.  Lanczos results are f32 (compared within a tolerance)."""

    lanczos = d.sampling == 3
    h16 = f16 and not lanczos
    w, h, dw, dh = d.src_w, d.src_h, d.dst_w, d.dst_h
    row = w * 12 // 8 if name == "bayer12p" else w * d.src_bpp
    tight = frame[:d.src_pitch * h].reshape(h, d.src_pitch)[:, :row].copy() if name not in TIGHT else frame
    cfg = dict(mode=mode, pitch=d.src_pitch, mean=MEAN, inv_std=INV, sampling=d.sampling)
    if name in ("rgb", "gray", "nv12", "yuyv"):
        fmt = {"rgb": o().FMT_RGB, "gray": o().FMT_GRAY, "nv12": o().FMT_NV12, "yuyv": o().FMT_YUYV}[name]
        return o().preprocess_frame(frame, o().PreprocessCfg(fmt=fmt, **cfg), w, h, dw, dh, f16=h16)
    if name == "bayer8":
        twin = demosaic(tight.reshape(h, w), "GRBG").astype(np.uint8)
        cfg["pitch"] = None
        return o().preprocess_frame(twin, o().PreprocessCfg(fmt=o().FMT_RGB, **cfg), w, h, dw, dh, f16=h16)
    if name == "bayer16":
        rgb, bits = demosaic(tight.view(np.uint16).reshape(h, w), "RGGB"), 12
    elif name == "bayer12p":
        rgb, bits = demosaic(unpack_np(tight, 12), "RGGB"), 12
    else:
        rgb = decode_yuv16(torch.from_numpy(frame.view(np.uint16).astype(np.int32)), w, h, "P010", "Bt601Limited").numpy()
        bits = 10
    affine = (d.scale_x, d.scale_y, d.pad_x, d.pad_y)
    return preprocess_rgb16(np.asarray(rgb).astype(np.uint16), bits, affine, dw, dh, "Lanczos" if lanczos else "Bilinear", MEAN, INV,
                            d.pad_value, h16)


def pp_compare(got, want, lanczos, f16, what):
    if lanczos:   # the oracle calls host sinf, the kernel the CUDA one: test_preprocess_lanczos_vs_oracle's tolerance
        g = got.view(np.float16 if f16 else np.float32).astype(np.float32)
        assert np.max(np.abs(g - want.reshape(-1).astype(np.float32))) <= (2e-3 if f16 else 1e-4), what
    else:
        assert np.array_equal(got, as_bytes(want)), what


PP_GEOMS = {   # mode 0 letterbox / 1 stretch; (dw, dh); sampling; expected kernel family
    "identity": (1, (64, 48), 1), "letterbox": (0, (40, 40), 1), "lanczos": (0, (40, 40), 3),
}


def pp_kernel(name, geom, d):
    if geom == "lanczos" or name in ("rgb", "gray", "yuyv"):
        return "preprocess_generic_kernel"
    if name in ("bayer8", "bayer16", "bayer12p"):
        s, p = {"bayer8": ("", "grbg"), "bayer16": ("16", "rggb"), "bayer12p": ("12p", "rggb")}[name]
        return f"preprocess_bayer{s}_{p}_identity_kernel" if geom == "identity" else "preprocess_generic_kernel"
    base = {"nv12": "nv12", "p010": "p01x"}[name]
    return f"preprocess_{base}{'_identity' if geom == 'identity' else ''}_kernel"


PP_CASES = [(n, g) for n in PP for g in PP_GEOMS]


@pytest.mark.parametrize("name,geom", PP_CASES)
@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_footprint(kb, lib, dev, name, geom, f16):
    """Both device entries: the strided one with poisoned pitch padding and a poisoned gap between frames, the pointer-table
    one with every frame in its own guarded allocation; exact lengths, guards, 0x00 / 0xFF runs."""
    mode, (dw, dh), sampling = PP_GEOMS[geom]
    d = pp_desc(lib, name, mode, dw, dh, 16, sampling)   # 16 bytes of padding keep every pitch a multiple of 16
    need = lib_src_bytes(d)
    n = 3
    frames = [pp_poison_padding(pp_frame(name, d, k), d) for k in range(n)]
    want = [pp_oracle(name, d, mode, f, f16) for f in frames]
    esz = 2 if f16 else 4
    out_elems = 3 * dw * dh
    kernel = pp_kernel(name, geom, d)
    gap = 48
    stride = need + gap
    ring = Guarded(dev, stride * (n - 1) + need, dw * esz)
    ring.load("u8", np.concatenate([np.concatenate([f, poison("u8", gap)]) for f in frames])[:stride * (n - 1) + need])
    ring_before = ring.snapshot()
    singles = [Guarded(dev, need, dw * esz).load("u8", frames[k]) for k in range(n)]
    singles_before = [g.snapshot() for g in singles]
    strided_fn = lib.kb200_preprocess_strided_f16 if f16 else lib.kb200_preprocess_strided_f32
    table_fn = lib.kb200_preprocess_f16 if f16 else lib.kb200_preprocess_f32
    ptrs = (C.c_void_p * n)(*[g.ptr for g in singles])
    lens = (C.c_size_t * n)(*[need] * n)
    calls = {
        "strided": lambda dst, dl, bl=ring.n: strided_fn(None, C.byref(d), ring.ptr, bl, stride, n, dst, dl),
        "table": lambda dst, dl, ln=lens: table_fn(None, C.byref(d), ptrs, ln, n, dst, dl),
    }
    for entry, call in calls.items():
        outs = []
        for fill in (0x00, 0xFF):
            dst = Guarded(dev, out_elems * esz * n, dw * esz).fill(fill)
            st = call(dst.ptr, out_elems * n)
            assert st == OK, f"{name} {geom} {entry}: {kb._lib.last_error()}"
            k = kb._lib.last_kernel()
            torch.cuda.synchronize()
            assert k == kernel, f"{name} {geom} {entry}: ran {k}"
            lead, tail = dst.guards()
            assert np.all(lead == fill) and np.all(tail == fill), f"{name} {geom} {entry}: write outside dst"
            outs.append(dst.out())
        assert np.array_equal(outs[0], outs[1]), f"{name} {geom} {entry}: output left unwritten"
        fb = out_elems * esz
        for j in range(n):
            pp_compare(outs[0][j * fb:(j + 1) * fb], want[j], sampling == 3, f16, f"{name} {geom} {entry}: frame {j} differs from the oracle")
        dst.fill(0x5A)
        before = dst.snapshot()
        assert call(dst.ptr, out_elems * n - 1) == SLICE and "'dst'" in kb._lib.last_error()
        if entry == "strided":
            assert call(dst.ptr, out_elems * n, ring.n - 1) == -8 and f"need {ring.n}" in kb._lib.last_error()
        else:
            short = (C.c_size_t * n)(need, need - 1, need)
            assert call(dst.ptr, out_elems * n, short) == -8 and f"need {need}" in kb._lib.last_error()
        torch.cuda.synchronize()
        assert np.array_equal(dst.snapshot(), before)
    assert np.array_equal(ring.snapshot(), ring_before)
    assert all(np.array_equal(g.snapshot(), b) for g, b in zip(singles, singles_before))


@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_batch_over_256_strided(kb, lib, dev, f16):
    """300 frames cross the 256-frame launch split; the gaps between frames and the padding of every row are poison."""
    name, n = "nv12", 300
    d = pp_desc(lib, name, 0, 40, 40)
    need = lib_src_bytes(d)
    gap = 16
    stride = need + gap
    frames = [pp_frame(name, d, k) for k in range(n)]
    ring = Guarded(dev, stride * (n - 1) + need, 160)
    ring.load("u8", np.concatenate([np.concatenate([f, poison("u8", gap)]) for f in frames])[:stride * (n - 1) + need])
    esz = 2 if f16 else 4
    out_elems = 3 * 40 * 40
    fn = lib.kb200_preprocess_strided_f16 if f16 else lib.kb200_preprocess_strided_f32
    outs = []
    for fill in (0x00, 0xFF):
        dst = Guarded(dev, out_elems * esz * n, 160).fill(fill)
        assert fn(None, C.byref(d), ring.ptr, ring.n, stride, n, dst.ptr, out_elems * n) == OK
        assert kb._lib.last_kernel() == "preprocess_nv12_kernel"
        torch.cuda.synchronize()
        lead, tail = dst.guards()
        assert np.all(lead == fill) and np.all(tail == fill)
        outs.append(dst.out())
    assert np.array_equal(outs[0], outs[1])
    cfg = o().PreprocessCfg(mode=0, fmt=o().FMT_NV12, mean=MEAN, inv_std=INV)
    fb = out_elems * esz
    for k in (0, 1, 255, 256, 257, n - 1):
        want = o().preprocess_frame(frames[k], cfg, 64, 48, 40, 40, f16=f16)
        assert np.array_equal(outs[0][k * fb:(k + 1) * fb], as_bytes(want)), f"frame {k}"


# ── host entries: pinned guarded destination, host source with poisoned gaps, several chunks and a ragged last one ──
def test_resize_normalize_host_guards(kb, lib, dev):
    sw, sh, dw, dh, n = 192, 108, 64, 36, 7
    sc, bi = fused_scale_bias()
    frames = [img_u8(sw, sh, 3, 11)(k) for k in range(n)]
    src = Guarded(dev, sw * sh * 3 * n, host=True).load("u8", np.concatenate([as_bytes(f) for f in frames]))
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * sw * sh * 3, dst_chunk_bytes=3 * 3 * dw * dh * 4, depth=2)
    try:
        for out, esz in ((0, 4), (1, 2)):
            outs = []
            for fill in (0x00, 0xFF):
                dst = Guarded(dev, 3 * dw * dh * esz * n, dw * esz, host=True).fill(fill)
                st = lib.kb200_resize_normalize_chw_u8_host(pipe._h, None, src.ptr, src.n, dst.ptr, 3 * dw * dh * n, sw, sh, dw, dh, n,
                                                            f3(sc), f3(bi), 1, out)
                assert st == OK, kb._lib.last_error()
                assert kb._lib.last_kernel() == "fused_rows_kernel"   # 192x108 -> 64x36: 3:1, the staged point mode
                torch.cuda.synchronize()
                lead, tail = dst.guards()
                assert np.all(lead == fill) and np.all(tail == fill)
                outs.append(dst.out())
            assert np.array_equal(outs[0], outs[1])
            fb = 3 * dw * dh * esz
            for k in range(n):
                w = fused_oracle(dw, dh, "f32" if out == 0 else "f16")(frames[k])
                compare_to_oracle(outs[0][k * fb:(k + 1) * fb], w, f"host out {out} frame {k}")
            dst.fill(0x5A)
            assert lib.kb200_resize_normalize_chw_u8_host(pipe._h, None, src.ptr, src.n, dst.ptr, 3 * dw * dh * n - 1, sw, sh, dw, dh, n,
                                                          f3(sc), f3(bi), 1, out) == SLICE
            assert lib.kb200_resize_normalize_chw_u8_host(pipe._h, None, src.ptr, src.n - 1, dst.ptr, 3 * dw * dh * n, sw, sh, dw, dh, n,
                                                          f3(sc), f3(bi), 1, out) == SLICE
            torch.cuda.synchronize()
            assert np.all(dst.snapshot() == 0x5A)
    finally:
        pipe.close()


@pytest.mark.parametrize("f16", [False, True])
def test_preprocess_host_guards(kb, lib, dev, f16):
    name, n = "nv12", 7
    d = pp_desc(lib, name, 0, 40, 40)
    need = lib_src_bytes(d)
    gap = 40
    stride = need + gap
    frames = [pp_frame(name, d, k) for k in range(n)]
    src = Guarded(dev, stride * (n - 1) + need, host=True)
    src.load("u8", np.concatenate([np.concatenate([f, poison("u8", gap)]) for f in frames])[:src.n])
    src_before = src.snapshot()
    esz = 2 if f16 else 4
    out_elems = 3 * 40 * 40
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=3 * ((need + 15) // 16 * 16), dst_chunk_bytes=3 * out_elems * 4, depth=2)
    try:
        outs = []
        for fill in (0x00, 0xFF):
            dst = Guarded(dev, out_elems * esz * n, 160, host=True).fill(fill)
            st = lib.kb200_preprocess_host(pipe._h, None, C.byref(d), src.ptr, src.n, stride, n, dst.ptr, out_elems * n, int(f16))
            assert st == OK, kb._lib.last_error()
            assert kb._lib.last_kernel() == "preprocess_nv12_kernel"
            torch.cuda.synchronize()
            lead, tail = dst.guards()
            assert np.all(lead == fill) and np.all(tail == fill)
            outs.append(dst.out())
        assert np.array_equal(outs[0], outs[1])
        cfg = o().PreprocessCfg(mode=0, fmt=o().FMT_NV12, mean=MEAN, inv_std=INV)
        fb = out_elems * esz
        for k in range(n):
            assert np.array_equal(outs[0][k * fb:(k + 1) * fb], as_bytes(o().preprocess_frame(frames[k], cfg, 64, 48, 40, 40, f16=f16))), k
        dst.fill(0x5A)
        assert lib.kb200_preprocess_host(pipe._h, None, C.byref(d), src.ptr, src.n, stride, n, dst.ptr, out_elems * n - 1, int(f16)) == SLICE
        assert lib.kb200_preprocess_host(pipe._h, None, C.byref(d), src.ptr, src.n - 1, stride, n, dst.ptr, out_elems * n, int(f16)) == -8
        torch.cuda.synchronize()
        assert np.all(dst.snapshot() == 0x5A)
        assert np.array_equal(src.snapshot(), src_before)
    finally:
        pipe.close()
