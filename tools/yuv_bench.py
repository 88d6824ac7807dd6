"""The YUV layouts beyond NV12 / YUYV against their NV12 / YUYV siblings, decode and camera preprocess, in one run.

    python tools/yuv_bench.py --out DIR

Decode (RGB8 HWC out), 1080p x 256 and 4K x 16: NV21, I420 and YV12 against NV12; UYVY and YVYU against YUYV.
Preprocess (f32 CHW out, ImageNet normalisation), 256 frames: config 3a (1080p -> 1080p) and 3b (1080p -> 640x640
letterbox), I420, NV21 and YV12 against NV12, UYVY against YUYV.

Each layout's frames are the sibling's frames byte-repacked, so every arm computes the same picture; the line records
whether each arm's output equals its sibling's bit for bit.  Every arm is timed with CUDA events over --iters launches
after warm-up, the arms alternating, the whole set repeated --reps times to show the spread.  Bandwidth uses algorithmic
bytes over the H100 SXM data-sheet 3.35 TB/s: frame bytes (4:2:0 1.5 B/px, 4:2:2 2 B/px; for 3b the distinct bytes the
sampler taps, counted by the oracle) plus the output (3 B/px RGB8, 12 B/px f32 CHW).

Writes one JSON line to DIR/yuv_bench.jsonl (and stdout), with the card's name, power limit and max SM clock read in the
same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, parse_args, row, start, time_arms, write_line

FAMILIES = {"yuv420": ("Nv12", ("Nv21", "I420", "Yv12")), "yuv422": ("Yuyv", ("Uyvy", "Yvyu"))}


def from_sibling(t, w, h, layout):
    """Frames [N, bytes] of the NV12 / YUYV sibling -> the same pictures in `layout` (torch, on the device)."""
    import torch

    if layout in ("Nv12", "Yuyv"):
        return t
    if layout in ("Uyvy", "Yvyu"):
        idx = [1, 0, 3, 2] if layout == "Uyvy" else [0, 3, 2, 1]
        return t.view(t.shape[0], -1, 4)[..., idx].reshape(t.shape).contiguous()
    y, u, v = t[:, :w * h], t[:, w * h::2], t[:, w * h + 1::2]
    if layout == "Nv21":
        return torch.cat([y, torch.stack([v, u], -1).reshape(t.shape[0], -1)], 1).contiguous()
    return torch.cat([y, u, v] if layout == "I420" else [y, v, u], 1).contiguous()


def main():
    args = parse_args(arg_parser(__doc__, "yuv_bench"))

    import numpy as np
    import torch

    import kornia_rs_b200 as kb
    from oracle import oracle as o

    bench, facts = start("yuv_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0x7E11)

    # ── decode ──
    decode = {}
    for tag, w, h, n in (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16)):
        for fam, (sib, others) in FAMILIES.items():
            fb = w * h * 3 // 2 if fam == "yuv420" else w * h * 2
            base = torch.randint(0, 256, (n, fb), dtype=torch.uint8, device=dev, generator=gen)
            srcs = {k: from_sibling(base, w, h, k) for k in (sib,) + others}
            outs = {k: kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n) for k in srcs}
            fns = {k: (lambda k=k: getattr(kb.imgproc, f"rgb_from_{k.lower()}")(srcs[k], outs[k])) for k in srcs}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            same = {k: bool(torch.equal(outs[k].data, outs[sib].data)) for k in srcs}
            decode[f"{fam}_{tag}"] = {"batch": n, "src": [w, h],
                                      **row(times, kernels, {k: n * (fb + 3 * w * h) for k in srcs}, same, "bit_identical_to_sibling")}
            print(f"[yuv_bench] decode {fam} {tag}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
            del base, srcs, outs
            torch.cuda.empty_cache()

    # ── camera preprocess, configs 3a / 3b ──
    w, h, n = 1920, 1080, 256
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    preprocess = {}
    arms = {"yuv420": ("Nv12", ("I420", "Nv21", "Yv12")), "yuv422": ("Yuyv", ("Uyvy",))}
    for fam, (sib, others) in arms.items():
        fb = w * h * 3 // 2 if fam == "yuv420" else w * h * 2
        base = torch.randint(0, 256, (n, fb), dtype=torch.uint8, device=dev, generator=gen)
        srcs = {k: from_sibling(base, w, h, k) for k in (sib,) + others}
        for cfg, mode, (dw, dh) in (("cfg3a", "Stretch", (w, h)), ("cfg3b", "Letterbox", (640, 640))):
            pres = {k: kb.Preprocessor.builder().source_format(kb.SourceFormat[k]).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda()
                    for k in srcs}
            if cfg == "cfg3a":
                src_bytes = fb
            else:   # distinct tapped bytes of one frame, the sibling's layout (the same count in every layout of the family)
                ocfg = o.PreprocessCfg(mode=o.LETTERBOX, fmt=o.FMT_NV12 if sib == "Nv12" else o.FMT_YUYV, mean=kb.IMAGENET_MEAN, inv_std=inv)
                src_bytes = o.preprocess_frame(base[0].cpu().numpy(), ocfg, w, h, dw, dh, count_touched=True)[1]
            dst = torch.empty((n, 3, dh, dw), dtype=torch.float32, device=dev)
            frames = {k: [srcs[k][i] for i in range(n)] for k in srcs}
            fns = {k: (lambda k=k: pres[k].run_raw_batch(frames[k], w, h, dst)) for k in srcs}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            pres[sib].run_raw_batch(frames[sib], w, h, dst)
            want = dst.clone()
            same = {}
            for k in srcs:
                dst.fill_(float("nan"))
                pres[k].run_raw_batch(frames[k], w, h, dst)
                same[k] = bool(torch.equal(dst.view(torch.int32), want.view(torch.int32)))
            preprocess[f"{cfg}_{fam}"] = {"batch": n, "src": [w, h], "dst": [dw, dh], "src_bytes_per_frame": src_bytes,
                                          **row(times, kernels, {k: n * (src_bytes + 12 * dw * dh) for k in srcs}, same,
                                                "bit_identical_to_sibling")}
            print(f"[yuv_bench] {cfg} {fam}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
            del dst, want, frames
            torch.cuda.empty_cache()
        del base, srcs

    line = {"tool": "tools/yuv_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "decode": decode, "preprocess": preprocess}
    write_line(args.out, "yuv_bench", line)


if __name__ == "__main__":
    main()
