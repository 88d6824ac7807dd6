"""12-bit Bayer against 8-bit Bayer and NV12, decode and camera preprocess, in one run.

    python tools/bayer16_bench.py --out DIR

Decode, 1080p x 256 and 4K x 16: rgb_from_bayer16 (BayerRggb12 content, RGB16 HWC out) against rgb_from_bayer (RGGB,
RGB8 out) and rgb_from_nv12 (RGB8 out) at the same size.
Preprocess, 256 frames, ImageNet normalisation, f32 and f16 CHW out: config 3a (1080p -> 1080p, the identity kernels)
and 3b (1080p -> 640x640 letterbox; the generic kernel for both Bayer depths), BayerRggb12 against BayerRggb and NV12.
End to end: config 3a from pinned host frames to a pinned host f32 tensor through a HostPipeline, 64 frames, the three
formats, recording the bytes each direction moved.

Every arm is timed with CUDA events over --iters launches after warm-up, the arms alternating, the whole set repeated
--reps times to show the spread.  Bandwidth uses algorithmic bytes over the H100 SXM data-sheet 3.35 TB/s: the frame
(Bayer12 2 B/px, Bayer8 1 B/px, NV12 1.5 B/px; for 3b NV12 counts the distinct bytes its sampler taps, as in
tools/bayer_bench.py, while a Bayer tap's 3x3 neighbourhood covers every source sample at 3b's exact 3:1 ratio) plus the
output (6 / 3 / 3 B/px RGB for the decodes, 12 / 6 B/px for f32 / f16 CHW).
Every Bayer output is checked on the device: the 12-bit decode against restate.demosaic, the 12-bit 3a preprocess
against that demosaic normalised in torch (harness.bayer16_identity: separate IEEE f32 operations), the 12-bit 3b
preprocess against the f32 restatement of the oracle (harness.restated) on three frames, the 8-bit arms as
tools/bayer_bench.py checks them, and end to end against the device run.

Writes one JSON line to DIR/bayer16_bench.jsonl (and stdout), with the card's name, power limit and max SM clock read
in the same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, e2e_result, parse_args, row, start, time_arms, write_line

ARMS = ("Bayer12", "Bayer8", "Nv12")


def main():
    ap = arg_parser(__doc__, "bayer16_bench")
    ap.add_argument("--e2e-frames", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=5)
    args = parse_args(ap)

    import numpy as np
    import torch

    import kornia_rs_b200 as kb
    from oracle import oracle as o
    from harness import bayer16_identity, restated, to_np16
    from restate import demosaic

    bench, facts = start("bayer16_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0xB16)
    fmt = {"Bayer12": kb.SourceFormat.BayerRggb12, "Bayer8": kb.SourceFormat.BayerRggb, "Nv12": kb.SourceFormat.Nv12}
    bpp = {"Bayer12": 2.0, "Bayer8": 1.0, "Nv12": 1.5}

    def frames_for(n, w, h):
        return {"Bayer12": torch.randint(0, 4096, (n, w * h), dtype=torch.int32, device=dev, generator=gen).to(torch.uint16),
                "Bayer8": torch.randint(0, 256, (n, w * h), dtype=torch.uint8, device=dev, generator=gen),
                "Nv12": torch.randint(0, 256, (n, w * h * 3 // 2), dtype=torch.uint8, device=dev, generator=gen)}

    # ── decode ──
    decode = {}
    for tag, w, h, n in (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16)):
        src = frames_for(n, w, h)
        outs = {"Bayer12": kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint16, dev, batch=n),
                "Bayer8": kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n),
                "Nv12": kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n)}
        fns = {"Bayer12": lambda: kb.imgproc.rgb_from_bayer16(src["Bayer12"], outs["Bayer12"], kb.imgproc.BayerPattern.RGGB),
               "Bayer8": lambda: kb.imgproc.rgb_from_bayer(src["Bayer8"], outs["Bayer8"], kb.imgproc.BayerPattern.RGGB),
               "Nv12": lambda: kb.imgproc.rgb_from_nv12(src["Nv12"], outs["Nv12"])}
        times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
        same = {"Nv12": None,
                "Bayer12": all(bool(torch.equal(outs["Bayer12"].data[k:k + 16].view(torch.int16),
                                                demosaic(src["Bayer12"][k:k + 16].view(-1, h, w), "RGGB").view(torch.int16))) for k in range(0, n, 16)),
                "Bayer8": all(bool(torch.equal(outs["Bayer8"].data[k:k + 16], demosaic(src["Bayer8"][k:k + 16].view(-1, h, w), "RGGB")))
                              for k in range(0, n, 16))}
        alg = {k: int(n * w * h * (bpp[k] + (6 if k == "Bayer12" else 3))) for k in ARMS}
        decode[tag] = {"batch": n, "src": [w, h], **row(times, kernels, alg, same, "output_checked")}
        print(f"[bayer16_bench] decode {tag}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
        del src, outs
        torch.cuda.empty_cache()

    # ── camera preprocess, configs 3a / 3b, f32 and f16 ──
    w, h, n = 1920, 1080, 256
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    src = frames_for(n, w, h)
    frames = {k: [src[k][i] for i in range(n)] for k in ARMS}
    preprocess = {}
    for cfg, mode, (dw, dh) in (("cfg3a", "Stretch", (w, h)), ("cfg3b", "Letterbox", (640, 640))):
        def builder(f):
            return kb.Preprocessor.builder().source_format(f).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda()

        pres = {k: builder(fmt[k]) for k in ARMS}
        ocfg = o.PreprocessCfg(mode=o.LETTERBOX if mode == "Letterbox" else o.STRETCH, fmt=o.FMT_NV12, mean=kb.IMAGENET_MEAN, inv_std=inv)
        nv12_bytes = w * h * 3 // 2 if cfg == "cfg3a" else o.preprocess_frame(src["Nv12"][0].cpu().numpy(), ocfg, w, h, dw, dh, count_touched=True)[1]
        for f16 in (False, True):
            dt, it, out_b = (torch.float16, torch.int16, 6) if f16 else (torch.float32, torch.int32, 12)
            outs = {k: torch.empty((n, 3, dh, dw), dtype=dt, device=dev) for k in ARMS}
            fns = {k: (lambda k=k: (pres[k].run_raw_batch_f16 if f16 else pres[k].run_raw_batch)(frames[k], w, h, outs[k])) for k in ARMS}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            same = {"Nv12": None}
            if cfg == "cfg3a":
                same["Bayer12"] = all(bool(torch.equal(outs["Bayer12"][k:k + 16].view(it),
                                                       bayer16_identity(src["Bayer12"][k:k + 16].view(-1, h, w), "RGGB", 12, kb).to(dt).contiguous().view(it)))
                                      for k in range(0, n, 16))
            else:
                same["Bayer12"] = all(np.array_equal(outs["Bayer12"][k].cpu().numpy().view(np.uint16 if f16 else np.uint32),
                                                     restated(kb, demosaic(to_np16(src["Bayer12"][k]).reshape(h, w), "RGGB"), 12, mode, "Bilinear",
                                                              dw, dh, f16).view(np.uint16 if f16 else np.uint32)) for k in (0, n // 2, n - 1))
            twin_pre = builder(kb.SourceFormat.Rgb8)
            rgb = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=32)
            want = torch.empty((32, 3, dh, dw), dtype=dt, device=dev)
            ok = True
            for k0 in range(0, n, 32):
                kb.imgproc.rgb_from_bayer(src["Bayer8"][k0:k0 + 32], rgb, kb.imgproc.BayerPattern.RGGB)
                ok = ok and bool(torch.equal(rgb.data, demosaic(src["Bayer8"][k0:k0 + 32].view(-1, h, w), "RGGB")))
                (twin_pre.run_raw_batch_f16 if f16 else twin_pre.run_raw_batch)([rgb.data[i].view(-1) for i in range(32)], w, h, want)
                ok = ok and bool(torch.equal(outs["Bayer8"][k0:k0 + 32].view(it), want.view(it)))
            same["Bayer8"] = ok
            src_b = {"Bayer12": 2 * w * h, "Bayer8": w * h, "Nv12": nv12_bytes}
            alg = {k: n * (src_b[k] + out_b * dw * dh) for k in ARMS}
            key = f"{cfg}_{'f16' if f16 else 'f32'}"
            preprocess[key] = {"batch": n, "src": [w, h], "dst": [dw, dh], "nv12_src_bytes_per_frame": nv12_bytes,
                               **row(times, kernels, alg, same, "output_checked")}
            print(f"[bayer16_bench] {key}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
            del outs, want, rgb
            torch.cuda.empty_cache()
    del frames, src
    torch.cuda.empty_cache()

    # ── end to end, config 3a from host frames ──
    n = args.e2e_frames
    chunk, nstreams = 8, 3
    host = {"Bayer12": torch.empty((n, w * h), dtype=torch.uint16, pin_memory=True),
            "Bayer8": torch.empty((n, w * h), dtype=torch.uint8, pin_memory=True),
            "Nv12": torch.empty((n, w * h * 3 // 2), dtype=torch.uint8, pin_memory=True)}
    host["Bayer12"].copy_(torch.randint(0, 4096, (n, w * h), dtype=torch.int32, device=dev, generator=gen).to(torch.uint16).cpu())
    for k in ("Bayer8", "Nv12"):
        host[k].copy_(torch.randint(0, 256, host[k].shape, dtype=torch.uint8, device=dev, generator=gen).cpu())
    pres = {k: kb.Preprocessor.builder().source_format(fmt[k]).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda() for k in ARMS}
    outs = {k: torch.empty((n, 3, h, w), dtype=torch.float32, pin_memory=True) for k in ARMS}
    frame_bytes = {k: host[k].shape[1] * host[k].element_size() for k in ARMS}
    pipes = {k: kb.imgproc.HostPipeline(dev, src_chunk_bytes=chunk * ((frame_bytes[k] + 15) // 16 * 16), dst_chunk_bytes=chunk * 12 * w * h,
                                        depth=nstreams) for k in ARMS}
    fns = {k: (lambda k=k: pres[k].run_raw_host(host[k], w, h, (w, h), out=outs[k], pipeline=pipes[k])) for k in ARMS}
    steps, _ = time_arms(bench, fns, args.e2e_steps, 1, args.reps, st, kb)
    e2e = {}
    for k in ARMS:
        transfer = pipes[k].last_transfer()
        pipes[k].close()
        want = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
        dev_frames = host[k].to(dev)
        pres[k].run_raw_batch([dev_frames[i] for i in range(n)], w, h, want)
        e2e[k] = e2e_result(steps[k], transfer, bool(torch.equal(outs[k].to(dev).view(torch.int32), want.view(torch.int32))))
        print(f"[bayer16_bench] e2e cfg3a {k}: {e2e[k]['ms_per_step']} ms/step", file=sys.stderr, flush=True)
        del want, dev_frames
        torch.cuda.empty_cache()

    line = {"tool": "tools/bayer16_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "decode": decode, "preprocess": preprocess,
            "e2e_cfg3a": {"batch": n, "chunk_frames": chunk, "streams": nstreams, "steps_per_rep": args.e2e_steps, **e2e}}
    write_line(args.out, "bayer16_bench", line)


if __name__ == "__main__":
    main()
