"""Bayer mosaics against NV12, decode and camera preprocess, in one run.

    python tools/bayer_bench.py --out DIR

Decode (RGB8 HWC out), 1080p x 256 and 4K x 16: each Bayer pattern against rgb_from_nv12 at the same size.
Preprocess (f32 CHW out, ImageNet normalisation), 256 frames: config 3a (1080p -> 1080p, the identity kernels) and 3b
(1080p -> 640x640 letterbox, the generic kernel for Bayer), each pattern against NV12.
End to end: config 3a from pinned host frames to a pinned host tensor through a HostPipeline, RGGB against NV12,
recording the bytes each direction moved.

Every arm is timed with CUDA events over --iters launches after warm-up, the arms alternating, the whole set repeated
--reps times to show the spread.  Bandwidth uses algorithmic bytes over the H100 SXM data-sheet 3.35 TB/s: the frame
(Bayer 1 B/px; NV12 1.5 B/px, for 3b the distinct bytes its sampler taps, counted by the oracle — at 3b's exact 3:1
ratio a Bayer tap's 3x3 neighbourhood covers every source byte) plus the output (3 B/px RGB8, 12 B/px f32 CHW).
Every Bayer output is checked: decode against restate.demosaic (on the device), preprocess
against the run on its RGB twin (the checked decode's output as SourceFormat.Rgb8), end to end against the device run.

Writes one JSON line to DIR/bayer_bench.jsonl (and stdout), with the card's name, power limit and max SM clock read in
the same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, e2e_result, parse_args, row, start, time_arms, write_line

PATTERNS = ("RGGB", "BGGR", "GRBG", "GBRG")


def main():
    ap = arg_parser(__doc__, "bayer_bench")
    ap.add_argument("--e2e-frames", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=5)
    args = parse_args(ap)

    import numpy as np
    import torch

    import kornia_rs_b200 as kb
    from oracle import oracle as o
    from restate import demosaic

    bench, facts = start("bayer_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0xBA7E)
    fmt = {p: kb.SourceFormat["Bayer" + p.capitalize()] for p in PATTERNS}

    def decode_into(p, src, img):
        kb.imgproc.rgb_from_bayer(src, img, kb.imgproc.BayerPattern[p])

    # ── decode ──
    decode = {}
    for tag, w, h, n in (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16)):
        bayer = torch.randint(0, 256, (n, w * h), dtype=torch.uint8, device=dev, generator=gen)
        nv12 = torch.randint(0, 256, (n, w * h * 3 // 2), dtype=torch.uint8, device=dev, generator=gen)
        outs = {k: kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n) for k in ("Nv12",) + PATTERNS}
        fns = {"Nv12": lambda: kb.imgproc.rgb_from_nv12(nv12, outs["Nv12"])}
        fns.update({p: (lambda p=p: decode_into(p, bayer, outs[p])) for p in PATTERNS})
        times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
        same = {"Nv12": None}
        for p in PATTERNS:
            same[p] = all(bool(torch.equal(outs[p].data[k0:k0 + 16], demosaic(bayer[k0:k0 + 16].view(-1, h, w), p))) for k0 in range(0, n, 16))
        alg = {"Nv12": n * (w * h * 3 // 2 + 3 * w * h), **{p: n * (w * h + 3 * w * h) for p in PATTERNS}}
        decode[tag] = {"batch": n, "src": [w, h], **row(times, kernels, alg, same, "output_checked")}
        print(f"[bayer_bench] decode {tag}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
        del bayer, nv12, outs
        torch.cuda.empty_cache()

    # ── camera preprocess, configs 3a / 3b ──
    w, h, n = 1920, 1080, 256
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    bayer = torch.randint(0, 256, (n, w * h), dtype=torch.uint8, device=dev, generator=gen)
    nv12 = torch.randint(0, 256, (n, w * h * 3 // 2), dtype=torch.uint8, device=dev, generator=gen)
    frames = {"Nv12": [nv12[i] for i in range(n)], **{p: [bayer[i] for i in range(n)] for p in PATTERNS}}
    preprocess = {}
    for cfg, mode, (dw, dh) in (("cfg3a", "Stretch", (w, h)), ("cfg3b", "Letterbox", (640, 640))):
        def builder(f):
            return kb.Preprocessor.builder().source_format(f).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda()

        pres = {"Nv12": builder(kb.SourceFormat.Nv12), **{p: builder(fmt[p]) for p in PATTERNS}}
        ocfg = o.PreprocessCfg(mode=o.LETTERBOX if mode == "Letterbox" else o.STRETCH, fmt=o.FMT_NV12, mean=kb.IMAGENET_MEAN, inv_std=inv)
        nv12_bytes = w * h * 3 // 2 if cfg == "cfg3a" else o.preprocess_frame(nv12[0].cpu().numpy(), ocfg, w, h, dw, dh, count_touched=True)[1]
        outs = {k: torch.empty((n, 3, dh, dw), dtype=torch.float32, device=dev) for k in pres}
        fns = {k: (lambda k=k: pres[k].run_raw_batch(frames[k], w, h, outs[k])) for k in pres}
        times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
        same = {"Nv12": None}
        twin_pre = builder(kb.SourceFormat.Rgb8)
        rgb = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=32)
        want = torch.empty((32, 3, dh, dw), dtype=torch.float32, device=dev)
        for p in PATTERNS:
            ok = True
            for k0 in range(0, n, 32):
                decode_into(p, bayer[k0:k0 + 32], rgb)
                ok = ok and bool(torch.equal(rgb.data, demosaic(bayer[k0:k0 + 32].view(-1, h, w), p)))
                twin_pre.run_raw_batch([rgb.data[i].view(-1) for i in range(32)], w, h, want)
                ok = ok and bool(torch.equal(outs[p][k0:k0 + 32].view(torch.int32), want.view(torch.int32)))
            same[p] = ok
        alg = {"Nv12": n * (nv12_bytes + 12 * dw * dh), **{p: n * (w * h + 12 * dw * dh) for p in PATTERNS}}
        preprocess[cfg] = {"batch": n, "src": [w, h], "dst": [dw, dh], "nv12_src_bytes_per_frame": nv12_bytes,
                           **row(times, kernels, alg, same, "output_checked")}
        print(f"[bayer_bench] {cfg}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
        del outs, want, rgb
        torch.cuda.empty_cache()
    del frames, bayer, nv12
    torch.cuda.empty_cache()

    # ── end to end, config 3a from host frames ──
    n = args.e2e_frames
    chunk, nstreams = 8, 3
    host = {"Nv12": torch.empty((n, w * h * 3 // 2), dtype=torch.uint8, pin_memory=True),
            "RGGB": torch.empty((n, w * h), dtype=torch.uint8, pin_memory=True)}
    for t in host.values():
        t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device=dev, generator=gen).cpu())
    pres = {"Nv12": kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda(),
            "RGGB": kb.Preprocessor.builder().source_format(fmt["RGGB"]).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda()}
    outs = {k: torch.empty((n, 3, h, w), dtype=torch.float32, pin_memory=True) for k in host}
    pipes = {k: kb.imgproc.HostPipeline(dev, src_chunk_bytes=chunk * ((host[k].shape[1] + 15) // 16 * 16), dst_chunk_bytes=chunk * 12 * w * h,
                                        depth=nstreams) for k in host}
    fns = {k: (lambda k=k: pres[k].run_raw_host(host[k], w, h, (w, h), out=outs[k], pipeline=pipes[k])) for k in host}
    steps, _ = time_arms(bench, fns, args.e2e_steps, 1, args.reps, st, kb)
    e2e = {}
    for k in host:
        transfer = pipes[k].last_transfer()
        pipes[k].close()
        want = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
        dev_frames = host[k].to(dev)
        pres[k].run_raw_batch([dev_frames[i] for i in range(n)], w, h, want)
        e2e[k] = e2e_result(steps[k], transfer, bool(torch.equal(outs[k].to(dev).view(torch.int32), want.view(torch.int32))))
        print(f"[bayer_bench] e2e cfg3a {k}: {e2e[k]['ms_per_step']} ms/step", file=sys.stderr, flush=True)
        del want, dev_frames
        torch.cuda.empty_cache()

    line = {"tool": "tools/bayer_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "decode": decode, "preprocess": preprocess,
            "e2e_cfg3a": {"batch": n, "chunk_frames": chunk, "streams": nstreams, "steps_per_rep": args.e2e_steps, **e2e}}
    write_line(args.out, "bayer_bench", line)


if __name__ == "__main__":
    main()
