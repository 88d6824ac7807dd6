"""The camera source formats against each other: decode, camera preprocess and end to end, one table entry per set.

    python tools/format_bench.py --out DIR --set yuv16 [--set bayer_packed ...]

Sets: yuv (the 4:2:0 and 4:2:2 layouts against their NV12 / YUYV sibling), yuv_matrix (the four YUV matrices), yuv16
(P010, P012, I010, I012 against NV12 and 12-bit Bayer), yuv444 (I444, I410, I410Msb against NV12 and P010), bayer (the
four patterns against NV12), bayer16 (12-bit against 8-bit Bayer and NV12), bayer_packed (MIPI RAW10 / 12 / 14 against
unpacked 12-bit Bayer) and bf16 (bf16 CHW output against f32 and f16, per format).  The arms of a set carry one picture
where they can: the YUV layouts and depths are repackings of the same NV12 bytes, the packed mosaics of the same samples.

Decode: 1080p x 256 and 4K x 16, into RGB8, or RGB16 for sources deeper than 8 bits.  Preprocess: 256 frames of 1080p,
ImageNet normalisation, config 3a (1080p -> 1080p, the identity kernels) and 3b (1080p -> 640x640 letterbox), CHW out.
A *_generic arm runs its fast twin's frames from a source one byte, or into an output four bytes, off the alignment the
fast kernels need, to show what they buy.  A set launches its preprocess through the frame table or the strided entry;
the sets that time 3b's fast kernels use the strided entry, because building and checking 256 frame pointers in Python
takes longer than a 3b launch runs.  End to end: config 3a of --e2e-frames pinned host frames to a pinned host tensor
through a HostPipeline, recording the bytes each direction moved.

The arms of a section alternate in table order, each timed with CUDA events over --iters launches after --warmup, the
whole set repeated --reps times; a row has the times, their minimum and spread ((max - min) / min).  Bandwidth is
algorithmic bytes over the H100 SXM data-sheet 3.35 TB/s: the source frame (for 3b the distinct bytes the sampler taps,
counted by the oracle; a Bayer tap's 3x3 neighbourhood covers the whole mosaic at 3b's 3:1 ratio) plus the output.
Afterwards every arm runs once more into a poisoned destination and is checked bit for bit against its reference
(tests/restate.py, tests/harness.py, the oracle, a twin format on the device, or another arm of the run); the end to
end result against the device run.  Writes one JSON line per set to DIR/<set>_bench.jsonl (bf16:
preprocess_bf16_bench.jsonl) and stdout, with the card's name, power limit and max SM clock read in the same run.
"""
from __future__ import annotations

import sys
import time
from dataclasses import dataclass, replace
from functools import lru_cache
from types import SimpleNamespace
from typing import Callable

import numpy as np
import torch

from benchkit import PEAK_GBS, arg_parser, e2e_result, parse_args, row, start, time_arms, words, write_line
from harness import bayer16_identity, offset_buf, restated, yuv16_identity
from restate import FORMATS, NORMS, decode_yuv16, decode_yuv8, demosaic, nv12_to_yuv420, pack, row_bytes, src_bytes, unpack, yuv422_swap

FMT = {f.name: f for f in FORMATS.values()}
DECODE = (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16))
W, H, N = 1920, 1080, 256
CFGS = {"cfg3a": ("Stretch", W, H), "cfg3b": ("Letterbox", 640, 640)}
OUTS = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
RUN = {torch.float32: "run_raw_batch", torch.float16: "run_raw_batch_f16", torch.bfloat16: "run_raw_batch_bf16"}
CHUNK, STREAMS = 8, 3   # the end-to-end HostPipeline: frames per chunk, ring depth


def content(name, fn=None):
    """An arm's frames: the set's content `name`, through fn(frames, w, h) when given."""
    return lambda c, w, h: fn(c[name], w, h) if fn else c[name]


def packed(t, w, h, bits):
    """restate.pack, 16 frames at a time on the host: [n, w*h] samples -> [n, w*h*bits/8] bytes on t's device."""
    return torch.cat([torch.from_numpy(pack(c.view(-1, h, w).cpu().numpy(), bits)).reshape(len(c), -1) for c in t.split(16)]).to(t.device)


def i444(nv12, w, h):
    """The I444 frames of NV12 frames' pictures: each chroma sample replicated 2 x 2."""
    uv = nv12[:, w * h:].view(-1, h // 2, 1, w // 2, 1, 2).expand(-1, h // 2, 2, w // 2, 2, 2)
    return torch.cat([nv12[:, :w * h], uv[..., 0].reshape(-1, w * h), uv[..., 1].reshape(-1, w * h)], 1)


@dataclass(frozen=True)
class Arm:
    label: str
    fmt: str                      # a SourceFormat member; it also picks the decoder (decoder())
    frames: Callable              # (the set's content, w, h) -> [n, frame elements] on the device
    matrix: str | None = None     # the YuvMatrix of the decoder and the preprocessor; None: their default, BT.601 limited
    off: str | None = None        # "src": frames one byte past 16-B alignment; "dst": the output 4 bytes past it
    tap: tuple | None = None      # 3b source bytes: (oracle count "nv12" / "yuyv" / "px", bytes per count); None: the frame
    dec: str | None = None        # decode reference: "pic" (the restated picture) or an arm's label; None: unchecked
    pre: str | None = None        # preprocess reference: "rs16", "rgb8", "oracle", "oracle_rgb", "unpacked" or an arm's label
    cfgs: tuple = ("cfg3a", "cfg3b")
    sampling: str = "Bilinear"
    out: str | None = None        # an output type of the arm's own (bf16's arms); None: the section's


@dataclass(frozen=True)
class Set:
    seed: int
    content: dict                 # name -> (values, per pixel): random uint8 samples, or uint16 when values > 256
    decode: tuple = ()            # ((group, arms), ...): a group is one timed section per size, its name prefixing the key
    pre: tuple = ()               # ((group, arms), ...): per group, one timed section per config and output type
    pre_key: str = "{cfg}_{out}"
    outs: tuple = ("f32", "f16")
    table: bool = True            # preprocess through the frame table, else through the strided entry
    e2e: tuple = ()
    e2e_outs: tuple = ("f32",)
    file: str = ""                # the result file's name when it is not <set>_bench


NV12 = Arm("Nv12", "Nv12", content("nv12"), tap=("nv12", 1), dec="pic", pre="oracle")
YUYV = Arm("Yuyv", "Yuyv", content("yuyv"), tap=("yuyv", 1), dec="pic", pre="oracle")
YUV420 = [NV12] + [Arm(k, k, content("nv12", lambda t, w, h, k=k: nv12_to_yuv420(t, w, h, k)), tap=("nv12", 1), dec="Nv12", pre="Nv12")
                   for k in ("Nv21", "I420", "Yv12")]
YUV422 = [YUYV] + [Arm(k, k, content("yuyv", lambda t, w, h, k=k: yuv422_swap(t, k)), tap=("yuyv", 1), dec="Yuyv", pre="Yuyv")
                   for k in ("Uyvy", "Yvyu")]
MATRICES = ("Bt601Limited", "Bt601Full", "Bt709Limited", "Bt709Full")
YUV16 = [Arm(k, k, content("nv12", lambda t, w, h, k=k, s=s: words(nv12_to_yuv420(t, w, h, "I420") if k[0] == "I" else t, s)),
             "Bt709Limited", tap=("nv12", 2), dec="pic", pre="rs16") for k, s in (("P010", 8), ("P012", 8), ("I010", 2), ("I012", 4))]
BAYER12 = Arm("Bayer12", "BayerRggb12", content("bayer12"), dec="pic", pre="rs16")
BAYER8 = [Arm(p, "Bayer" + p.capitalize(), content("bayer8"), dec="pic", pre="rgb8") for p in ("RGGB", "BGGR", "GRBG", "GBRG")]
I444 = [Arm("I444", "I444", content("nv12", i444), "Bt709Limited", tap=("px", 3), dec="Nv12", pre="Nv12"),
        Arm("I410", "I410", content("nv12", lambda t, w, h: words(i444(t, w, h), 2)), "Bt709Limited", tap=("px", 6), dec="P010", pre="P010"),
        Arm("I410Msb", "I410Msb", content("nv12", lambda t, w, h: words(i444(t, w, h), 8)), "Bt709Limited", tap=("px", 6), dec="P010",
            pre="P010"),
        replace(NV12, matrix="Bt709Limited", pre="oracle_rgb"), YUV16[0]]
RAW = [Arm(f"Raw{b}p", f"BayerRggb{b}p", content("s10", lambda t, w, h, b=b: packed(t, w, h, b)), dec="Bayer12", pre="unpacked")
       for b in (10, 12, 14)] + [replace(BAYER12, frames=content("s10"), dec=None, pre=None)]
B16 = [BAYER12, replace(BAYER8[0], label="Bayer8"), NV12]


def by_out(fmt, tap, **kw):
    """One group of bf16's: the same preprocess of `fmt` into f32, f16 and bf16, the bf16 output checked against f32's."""
    return fmt, [Arm(k, fmt, content(fmt.lower()), tap=tap, pre="f32" if k == "bf16" else None, out=k, **kw) for k in OUTS]


SETS = {
    "yuv": Set(0x7E11, {"nv12": (256, 1.5), "yuyv": (256, 2)}, decode=(("yuv420", YUV420), ("yuv422", YUV422)),
               pre=(("yuv420", [YUV420[i] for i in (0, 2, 1, 3)]), ("yuv422", YUV422[:2])), pre_key="{cfg}_{group}", outs=("f32",)),
    "yuv_matrix": Set(0x709, {"nv12": (256, 1.5), "yuyv": (256, 2)},
                      decode=tuple((a.fmt.lower(), [replace(a, label=m, matrix=m) for m in MATRICES]) for a in (NV12, YUYV)),
                      pre=(("", [replace(NV12, label=m, matrix=m, pre="rgb8") for m in MATRICES]),)),
    "yuv16": Set(0x1016, {"nv12": (256, 1.5), "bayer12": (4096, 1), "coin": (2, 1)}, decode=(("", YUV16 + [NV12, BAYER12]),),
                 pre=(("", YUV16 + [NV12, BAYER12,
                                    replace(BAYER12, label="Bayer12_zeros", cfgs=("cfg3a",),   # zero dividends for __fdiv_rn
                                            frames=lambda c, w, h: words(torch.where(c["coin"] == 1, 0, c["bayer12"].to(torch.int32)), 0)),
                                    replace(YUV16[0], label="P010_generic", off="dst", pre="P010", cfgs=("cfg3b",))]),),
                 table=False, e2e=tuple(YUV16 + [NV12, BAYER12])),
    "yuv444": Set(0x444, {"nv12": (256, 1.5)}, decode=(("", I444),),
                  pre=(("", I444 + [replace(I444[0], label="I444_generic", off="dst", cfgs=("cfg3b",))]),), table=False, e2e=tuple(I444)),
    "bayer": Set(0xBA7E, {"bayer8": (256, 1), "nv12": (256, 1.5)}, decode=(("", [NV12] + BAYER8),), pre=(("", [NV12] + BAYER8),),
                 pre_key="{cfg}", outs=("f32",), e2e=(NV12, BAYER8[0])),
    "bayer16": Set(0xB16, {"bayer12": (4096, 1), "bayer8": (256, 1), "nv12": (256, 1.5)}, decode=(("", B16),), pre=(("", B16),), e2e=tuple(B16)),
    "bayer_packed": Set(0xBAC, {"s10": (1024, 1)}, decode=(("", RAW + [replace(RAW[1], label="Raw12p_generic", off="src")]),),
                        pre=(("", RAW + [replace(RAW[1], label="Raw12p_generic", off="src", cfgs=("cfg3a",))]),), e2e=tuple(RAW),
                        e2e_outs=("f32", "f16")),
    "bf16": Set(0xBF16, {"nv12": (256, 1.5), "p010": (65536, 1.5), "bayerrggb12": (4096, 1), "i444": (256, 3), "yuyv": (256, 2)},
                pre=(by_out("Nv12", ("nv12", 1)), by_out("P010", ("nv12", 2)), by_out("BayerRggb12", ("px", 2)), by_out("I444", ("px", 3)),
                     by_out("Yuyv", ("px", 2)), by_out("Nv12", None, sampling="Lanczos", cfgs=("cfg3b",))),
                pre_key="{group}_{cfg}", outs=("f32",), table=False, e2e=tuple(by_out("Nv12", None)[1]), file="preprocess_bf16_bench"),
}


def decoder(f):
    """The name of format f's decoder in kornia_rs_b200.imgproc."""
    if f.family == "bayer":
        return "rgb_from_bayer_packed" if f.packed else "rgb_from_bayer16" if f.words else "rgb_from_bayer"
    return f"rgb_from_{f.name.lower()}"


def frame_bytes(a, w, h):
    f = FMT[a.fmt]
    return src_bytes(f, w, h, row_bytes(f, w, 1))


@lru_cache(None)
def tapped(kind):
    """Config 3b's distinct tapped bytes of an NV12 or a YUYV frame, or its tapped pixels ("px"), counted by the oracle."""
    from oracle import oracle as o

    fmt, per_px = {"nv12": (o.FMT_NV12, 1.5), "yuyv": (o.FMT_YUYV, 2), "px": (o.FMT_RGB, 3)}[kind]
    mean, inv = NORMS["imagenet"]
    cfg = o.PreprocessCfg(mode=o.LETTERBOX, fmt=fmt, mean=mean, inv_std=inv)
    _, dw, dh = CFGS["cfg3b"]
    count = o.preprocess_frame(np.zeros(int(W * H * per_px), np.uint8), cfg, W, H, dw, dh, count_touched=True)[1]
    return count // 3 if kind == "px" else count


def decode_bytes(a, w, h, n):
    return n * (frame_bytes(a, w, h) + (6 if FMT[a.fmt].bits > 8 else 3) * w * h)


def pre_bytes(a, cfg, out):
    _, dw, dh = CFGS[cfg]
    src = frame_bytes(a, W, H) if cfg == "cfg3a" or a.tap is None else tapped(a.tap[0]) * a.tap[1]
    return N * (src + 3 * OUTS[a.out or out].itemsize * dw * dh)


def decode_sections(s):
    """(section key, w, h, frames, arms) of the set's decode, in run order."""
    for tag, w, h, n in DECODE:
        for g, arms in s.decode:
            yield (f"{g}_{tag}" if g else tag), w, h, n, arms


def pre_sections(s, group, arms):
    """(section key, config, output type, arms) of one preprocess group, in run order."""
    for cfg in CFGS:
        arms_c = [a for a in arms if cfg in a.cfgs]
        for out in s.outs if arms_c else ():
            yield s.pre_key.format(cfg=cfg, group=group, out=out) + ("_lanczos" if arms_c[0].sampling == "Lanczos" else ""), cfg, out, arms_c


# ── on the device ──
def make_content(x, s, n, w, h):
    return {k: torch.randint(0, hi, (n, int(w * h * per)), dtype=torch.int32 if hi > 256 else torch.uint8, device=x.dev, generator=x.gen)
            .to(torch.uint16 if hi > 256 else torch.uint8) for k, (hi, per) in s.content.items()}


def frames_of(x, arms, c, w, h):
    """{label: the arm's frames [n, elements]}, each distinct repacking made once."""
    made, src = {}, {}
    for a in arms:
        if a.frames not in made:
            made[a.frames] = a.frames(c, w, h).contiguous()
        t = made[a.frames]
        src[a.label] = offset_buf(x.dev, t.numel(), 1, t.dtype).view(t.shape).copy_(t) if a.off == "src" else t
    return src


def preprocessor(kb, a, mode):
    b = (kb.Preprocessor.builder().source_format(kb.SourceFormat[a.fmt]).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet())
         .sampling(kb.InterpolationMode[a.sampling]))
    return (b.yuv_matrix(kb.YuvMatrix[a.matrix]) if a.matrix else b).build_cuda()


def launcher(pre, frames, w, h, dst, table):
    """One launch of `pre` over frames [n, elements] into dst, through the frame table or the strided entry."""
    if table:
        fr, fn = list(frames.unbind()), getattr(pre, RUN[dst.dtype])
        return lambda: fn(fr, w, h, dst)
    stride = frames.shape[1] * frames.element_size()
    return lambda: pre.run_raw_strided(frames.view(-1), stride, len(frames), w, h, dst, dtype=dst.dtype)


def same(got, want):
    """Bit-for-bit equality: float outputs by their bits after rounding `want` to got's type, integers by value."""
    want = torch.as_tensor(want).to(got.device).reshape(got.shape)
    if got.is_floating_point():
        bits = torch.int32 if got.element_size() == 4 else torch.int16
        return bool(torch.equal(got.view(bits), want.to(got.dtype).contiguous().view(bits)))
    return bool(torch.equal(got.to(torch.int32), want.to(torch.int32)))


def reference(x, a, r, s):
    """What arm a's output for frames s must equal under reference r (see Arm.dec and Arm.pre)."""
    from oracle import oracle as o

    f, m = FMT[a.fmt], a.matrix or "Bt601Limited"
    if r == "pic":
        if f.family == "bayer":
            return demosaic(s.view(-1, x.h, x.w), f.layout)
        if f.words:
            return decode_yuv16(s, x.w, x.h, a.fmt, m)
        return np.stack([decode_yuv8(t.cpu().numpy(), x.w, x.h, a.fmt, m) for t in s])
    if r == "identity":
        if f.family == "bayer":
            return bayer16_identity(s.view(-1, x.h, x.w), f.layout, f.bits, x.kb)
        return yuv16_identity(s, x.w, x.h, a.fmt, m, x.kb)
    if r == "restated":
        rgb = torch.as_tensor(reference(x, a, "pic", s))[0].to(torch.int32).cpu().numpy().astype(np.uint16)
        return restated(x.kb, rgb, f.bits, x.mode, a.sampling, x.dw, x.dh, x.dt == torch.float16)
    if r in ("oracle", "oracle_rgb"):
        src = reference(x, a, "pic", s)[0] if r == "oracle_rgb" else s[0].cpu().numpy()
        inv = tuple(float(np.float32(1.0) / np.float32(v)) for v in x.kb.IMAGENET_STD)
        cfg = o.PreprocessCfg(mode=o.LETTERBOX if x.mode == "Letterbox" else o.STRETCH, mean=x.kb.IMAGENET_MEAN, inv_std=inv,
                              fmt=o.FMT_RGB if r == "oracle_rgb" else {"Nv12": o.FMT_NV12, "Yuyv": o.FMT_YUYV}[a.fmt])
        return o.preprocess_frame(src.reshape(-1), cfg, x.w, x.h, x.dw, x.dh, f16=x.dt == torch.float16)
    # a twin on the device: the restated picture as RGB8, or the packed samples unpacked into the 16-bit format of their depth
    if r == "rgb8":
        twin, fr = "Rgb8", torch.as_tensor(reference(x, a, "pic", s)).to(x.dev)
    else:
        twin, fr = f"Bayer{f.layout.capitalize()}{f.bits}", unpack(s.view(len(s), x.h, -1), f.bits).to(torch.uint16)
    want = torch.empty((len(s), 3, x.dh, x.dw), dtype=x.dt, device=x.dev)
    launcher(preprocessor(x.kb, replace(a, fmt=twin, matrix=None), x.mode), fr.reshape(len(s), -1), x.w, x.h, want, True)()
    return want


def check(x, arms, src, outs, fns, refs):
    """Runs every arm once more into its destination, poisoned first, and checks it against refs[label]: {label: bool or None}.
    A device reference is checked on every frame, a host one on the first, middle and last."""
    wanted = {r for r in refs.values() if r in outs}
    kept, ok = {}, {}
    for a in sorted(arms, key=lambda a: a.label not in wanted):   # the arms others are checked against first
        dst, r = outs[a.label], refs[a.label]
        dst.view(torch.uint8).fill_(0xFF)   # NaN in every float type
        fns[a.label]()
        if a.label in wanted:
            kept[a.label] = dst.clone()
        if r is None or r in kept:
            ok[a.label] = None if r is None else same(dst, kept[r])
            continue
        host = r in ("restated", "oracle", "oracle_rgb") or r in ("pic", "rgb8") and FMT[a.fmt].family != "bayer" and not FMT[a.fmt].words
        n = len(dst)
        frames = [slice(i, i + 1) for i in sorted({0, n // 2, n - 1})] if host else [slice(i, i + 8) for i in range(0, n, 8)]
        ok[a.label] = all(same(dst[i], reference(x, a, r, src[a.label][i])) for i in frames)
    return {a.label: ok[a.label] for a in arms}


def timed(x, name, key, arms, fns, alg, outs, src, refs):
    """Times the arms, checks them, and returns benchkit.row with each arm's spread ((max - min) / min) added."""
    times, kernels = time_arms(x.bench, fns, x.args.iters, x.args.warmup, x.args.reps, x.st, x.kb)
    r = row(times, kernels, alg, check(x, arms, src, outs, fns, refs), "output_checked")
    for k, t in times.items():
        r[k]["spread"] = round((max(t) - min(t)) / min(t), 4)
    print(f"[{name}] {key}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
    return r


def run_decode(x, name, s):
    res = {}
    for key, w, h, n, arms in decode_sections(s):
        x2 = SimpleNamespace(**{**vars(x), "w": w, "h": h})
        src = frames_of(x, arms, make_content(x, s, n, w, h), w, h)
        dts = {a.label: torch.uint16 if FMT[a.fmt].bits > 8 else torch.uint8 for a in arms}
        imgs = {dt: x.kb.Image.zeros_cuda(x.kb.ImageSize(w, h), 3, dt, x.dev, batch=n) for dt in set(dts.values())}
        img = {k: imgs[dt] for k, dt in dts.items()}
        ip = x.kb.imgproc

        def fn(a):
            f = FMT[a.fmt]
            args = (ip.BayerPattern[f.layout],) + ((f.bits,) if f.packed else ()) if f.family == "bayer" else ()
            kw = {"matrix": x.kb.YuvMatrix[a.matrix]} if a.matrix else {}
            return lambda: getattr(ip, decoder(f))(src[a.label], img[a.label], *args, **kw)

        alg = {a.label: decode_bytes(a, w, h, n) for a in arms}
        res[key] = {"batch": n, "src": [w, h], **timed(x2, name, f"decode {key}", arms, {a.label: fn(a) for a in arms}, alg,
                                                        {k: v.data for k, v in img.items()}, src, {a.label: a.dec for a in arms})}
        del src, imgs, img
        torch.cuda.empty_cache()
    return res


def run_preprocess(x, name, s):
    res = {}
    for group, arms in s.pre:
        src = frames_of(x, arms, make_content(x, s, N, W, H), W, H)
        for key, cfg, out, arms_c in pre_sections(s, group, arms):
            mode, dw, dh = CFGS[cfg]
            pres = {a.label: preprocessor(x.kb, a, mode) for a in arms_c}
            flat = {dt: torch.empty(N * 3 * dh * dw + 8, dtype=dt, device=x.dev) for dt in {OUTS[a.out or out] for a in arms_c}}
            outs = {}
            for a in arms_c:
                buf = flat[OUTS[a.out or out]]
                k = 4 // buf.element_size() if a.off == "dst" else 0   # 4 bytes off 16-B alignment: the fast kernels refuse it
                outs[a.label] = buf[k:k + N * 3 * dh * dw].view(N, 3, dh, dw)
            fns = {a.label: launcher(pres[a.label], src[a.label], W, H, outs[a.label], s.table) for a in arms_c}
            refs = {a.label: ("identity" if cfg == "cfg3a" else "restated") if a.pre == "rs16" else a.pre for a in arms_c}
            x2 = SimpleNamespace(**{**vars(x), "w": W, "h": H, "dw": dw, "dh": dh, "mode": mode, "dt": OUTS[out]})
            res[key] = {"batch": N, "src": [W, H], "dst": [dw, dh],
                        **timed(x2, name, key, arms_c, fns, {a.label: pre_bytes(a, cfg, out) for a in arms_c}, outs, src, refs)}
            del flat, outs, fns
            torch.cuda.empty_cache()
        del src
        torch.cuda.empty_cache()
    return res


def run_e2e(x, s):
    n = x.args.e2e_frames
    host = {}
    for a, t in zip(s.e2e, frames_of(x, s.e2e, make_content(x, s, n, W, H), W, H).values()):
        if a.fmt not in host:   # bf16's arms share one source and one pipeline
            host[a.fmt] = t.cpu().pin_memory()
    torch.cuda.empty_cache()
    pres = {a.label: preprocessor(x.kb, a, "Stretch") for a in s.e2e}
    pipes = {f: x.kb.imgproc.HostPipeline(x.dev, src_chunk_bytes=CHUNK * ((t.shape[1] * t.element_size() + 15) // 16 * 16),
                                          dst_chunk_bytes=CHUNK * 12 * W * H, depth=STREAMS) for f, t in host.items()}
    fmt = {a.label: a.fmt for a in s.e2e}
    res = {}
    for out in s.e2e_outs:
        dts = {a.label: OUTS[a.out or out] for a in s.e2e}
        outs = {k: torch.empty((n, 3, H, W), dtype=dt, pin_memory=True) for k, dt in dts.items()}
        fns = {k: (lambda k=k: pres[k].run_raw_host(host[fmt[k]], W, H, (W, H), out=outs[k], pipeline=pipes[fmt[k]], dtype=dts[k]))
               for k in dts}
        steps, transfer = time_arms(x.bench, fns, x.args.e2e_steps, 1, x.args.reps, x.st, x.kb, probe=lambda k: pipes[fmt[k]].last_transfer())
        res[out] = {}
        for a in s.e2e:
            want = torch.empty((n, 3, H, W), dtype=dts[a.label], device=x.dev)
            launcher(pres[a.label], host[a.fmt].to(x.dev), W, H, want, True)()
            got = outs[a.label].to(x.dev)
            ok = same(got, want) and (a.pre not in outs or same(got, outs[a.pre]))
            res[out][a.label] = e2e_result(steps[a.label], transfer[a.label], ok)
            print(f"[e2e cfg3a {out}] {a.label}: {res[out][a.label]['ms_per_step']} ms/step", file=sys.stderr, flush=True)
            del want
            torch.cuda.empty_cache()
    for p in pipes.values():
        p.close()
    return {"batch": n, "chunk_frames": CHUNK, "streams": STREAMS, "steps_per_rep": x.args.e2e_steps,
            **(res[s.e2e_outs[0]] if len(s.e2e_outs) == 1 else res)}


def main():
    ap = arg_parser(__doc__, "<set>_bench")
    ap.add_argument("--set", action="append", required=True, choices=list(SETS), help="a set to run (repeatable)")
    ap.add_argument("--e2e-frames", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=5)
    args = parse_args(ap)

    import kornia_rs_b200 as kb

    bench, facts = start("format_bench")
    dev = torch.device("cuda:0")
    for name in args.set:
        s = SETS[name]
        x = SimpleNamespace(kb=kb, bench=bench, args=args, dev=dev, st=torch.cuda.current_stream(dev),
                            gen=torch.Generator(device=dev).manual_seed(s.seed))
        line = {"tool": "tools/format_bench.py", "set": name, "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters,
                "warmup": args.warmup, "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s"}
        if s.decode:
            line["decode"] = run_decode(x, name, s)
        line["preprocess"] = run_preprocess(x, name, s)
        if s.e2e:
            line["e2e_cfg3a"] = run_e2e(x, s)
        write_line(args.out, s.file or f"{name}_bench", line)


if __name__ == "__main__":
    main()
