"""The four YUV colour matrices against each other, decode and camera preprocess, in one run.

    python tools/yuv_matrix_bench.py --out DIR

Decode (RGB8 HWC out), 1080p x 256 and 4K x 16, NV12 and YUYV.  Preprocess (CHW out, ImageNet normalisation), NV12
1080p x 256: config 3a (1080p -> 1080p, the identity kernel) and 3b (1080p -> 640x640 letterbox), f32 and f16.

The same frames go through every matrix; the matrices are the arms.  Every arm is timed with CUDA events over --iters
launches after warm-up, the arms alternating, the whole set repeated --reps times; the line records each arm's times,
their minimum and their spread ((max - min) / min).  Every arm's output is checked: decodes against the numpy
restatement of the Q20 arithmetic on the first and last frame, preprocess runs against the device preprocess of the
first and last frame's RGB8 twin (the restatement's decode of it), bit for bit.  Bandwidth uses algorithmic bytes over
the H100 SXM data-sheet 3.35 TB/s.

Writes one JSON line to DIR/yuv_matrix_bench.jsonl (and stdout), with the card's name, power limit and max SM clock read
in the same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, parse_args, start, time_arms, write_line

MATRICES = ("Bt601Limited", "Bt601Full", "Bt709Limited", "Bt709Full")


def row_for(times, kernels, alg_bytes, ok):
    row = {}
    for k in times:
        best = min(times[k])
        gbs = alg_bytes / (best * 1e-3) / 1e9
        row[k] = {"ms": [round(t, 4) for t in times[k]], "ms_min": round(best, 4), "spread": round((max(times[k]) - best) / best, 4),
                  "gbs": round(gbs, 1), "frac_of_3350": round(gbs / PEAK_GBS, 3), "kernel": kernels[k], "output_checked": ok[k]}
    return row


def main():
    args = parse_args(arg_parser(__doc__, "yuv_matrix_bench"))

    import torch

    import numpy as np

    import kornia_rs_b200 as kb
    from oracle import oracle as o
    from restate import decode_yuv8

    bench, facts = start("yuv_matrix_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0x709)

    # ── decode ──
    decode_rows = {}
    for tag, w, h, n in (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16)):
        for layout, fb in (("Nv12", w * h * 3 // 2), ("Yuyv", w * h * 2)):
            src = torch.randint(0, 256, (n, fb), dtype=torch.uint8, device=dev, generator=gen)
            outs = {m: kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n) for m in MATRICES}
            op = getattr(kb.imgproc, f"rgb_from_{layout.lower()}")
            fns = {m: (lambda m=m: op(src, outs[m], matrix=kb.YuvMatrix[m])) for m in MATRICES}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            ok = {}
            for m in MATRICES:
                ok[m] = all(bool((outs[m].data[k].cpu().numpy() == decode_yuv8(src[k].cpu().numpy(), w, h, layout, m)).all()) for k in (0, n - 1))
            decode_rows[f"{layout.lower()}_{tag}"] = {"batch": n, "src": [w, h], **row_for(times, kernels, n * (fb + 3 * w * h), ok)}
            print(f"[yuv_matrix_bench] decode {layout} {tag}: " + "  ".join(f"{m} {min(times[m]):.4f}" for m in MATRICES), file=sys.stderr, flush=True)
            del src, outs
            torch.cuda.empty_cache()

    # ── camera preprocess, configs 3a / 3b, NV12 ──
    w, h, n = 1920, 1080, 256
    fb = w * h * 3 // 2
    frames_t = torch.randint(0, 256, (n, fb), dtype=torch.uint8, device=dev, generator=gen)
    frames = [frames_t[i] for i in range(n)]
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    preprocess = {}
    for cfg, mode, (dw, dh) in (("cfg3a", "Stretch", (w, h)), ("cfg3b", "Letterbox", (640, 640))):
        if cfg == "cfg3a":
            src_bytes = fb
        else:   # distinct tapped bytes of one frame, counted by the oracle (as tools/yuv_bench.py counts them)
            ocfg = o.PreprocessCfg(mode=o.LETTERBOX, fmt=o.FMT_NV12, mean=kb.IMAGENET_MEAN, inv_std=inv)
            src_bytes = o.preprocess_frame(frames_t[0].cpu().numpy(), ocfg, w, h, dw, dh, count_touched=True)[1]
        for f16 in (False, True):
            dt, it = (torch.float16, torch.int16) if f16 else (torch.float32, torch.int32)
            build = lambda fmt, m=None: ((lambda b: (b.yuv_matrix(kb.YuvMatrix[m]) if m else b).build_cuda())(
                kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet())))
            pres = {m: build("Nv12", m) for m in MATRICES}
            dsts = {m: torch.empty((n, 3, dh, dw), dtype=dt, device=dev) for m in MATRICES}
            run = (lambda p, fr, d: p.run_raw_batch_f16(fr, w, h, d)) if f16 else (lambda p, fr, d: p.run_raw_batch(fr, w, h, d))
            fns = {m: (lambda m=m: run(pres[m], frames, dsts[m])) for m in MATRICES}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            twin_pre = build("Rgb8")
            ok = {}
            for m in MATRICES:
                good = True
                for k in (0, n - 1):
                    twin = torch.from_numpy(decode_yuv8(frames_t[k].cpu().numpy(), w, h, "Nv12", m).reshape(-1)).to(dev)
                    want = torch.full((1, 3, dh, dw), float("nan"), dtype=dt, device=dev)
                    run(twin_pre, [twin], want)
                    good = good and bool(torch.equal(dsts[m][k:k + 1].view(it), want.view(it)))
                ok[m] = good
            out_bytes = 3 * dw * dh * (2 if f16 else 4)
            key = f"{cfg}_{'f16' if f16 else 'f32'}"
            preprocess[key] = {"batch": n, "src": [w, h], "dst": [dw, dh], "src_bytes_per_frame": src_bytes,
                               **row_for(times, kernels, n * (src_bytes + out_bytes), ok)}
            print(f"[yuv_matrix_bench] {key}: " + "  ".join(f"{m} {min(times[m]):.4f}" for m in MATRICES), file=sys.stderr, flush=True)
            del dsts, pres
            torch.cuda.empty_cache()

    line = {"tool": "tools/yuv_matrix_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "decode": decode_rows,
            "preprocess": preprocess}
    write_line(args.out, "yuv_matrix_bench", line)


if __name__ == "__main__":
    main()
