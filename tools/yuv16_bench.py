"""10- and 12-bit 4:2:0 video (P010, P012, I010, I012) against NV12 and 12-bit Bayer, decode and camera preprocess, in one run.

    python tools/yuv16_bench.py --out DIR

Every arm carries the same picture: random NV12 bytes, repacked as P010 / P012 words (byte << 8: NV12's layout, the
code in the high bits) and I010 / I012 words (byte << 2 / byte << 4: I420's layout, the code in the low bits), so the
8-bit content is identical; the BayerRggb12 arm is random 12-bit samples.
Decode, 1080p x 256 and 4K x 16: rgb_from_p010 / _p012 / _i010 / _i012 (RGB16 out), rgb_from_nv12 (RGB8 out),
rgb_from_bayer16 (RGB16 out).
Preprocess, 256 frames, ImageNet normalisation, f32 and f16 CHW out: config 3a (1080p -> 1080p, the identity kernels)
and 3b (1080p -> 640x640 letterbox), plus for 3b the P010 frames on the generic kernel (an output 4 bytes off 16-byte
alignment, which the fast kernel refuses) to show what the fast kernel buys, and for 3a the Bayer12 frames with half the
samples 0 (the 16-bit Bayer identity kernel divides by W with a plain __fdiv_rn, so this arm shows what zero dividends
cost it).  Preprocess launches go through the strided entry (one ring of 256 frames): the pointer-table entry builds and
checks 256 frame pointers in Python per launch, which takes longer than a 3b launch runs, so it would time the host.
End to end: config 3a from pinned host frames to a pinned host f32 tensor through a HostPipeline, 64 frames, recording
the bytes each direction moved.

Every arm is timed with CUDA events over --iters launches after warm-up, the arms alternating, the whole set repeated
--reps times; the minimum is reported.  Bandwidth uses algorithmic bytes over the H100 SXM data-sheet 3.35 TB/s: the
frame (P01x / I01x 3 B/px, NV12 1.5 B/px, Bayer12 2 B/px; for 3b the 4:2:0 arms count the distinct bytes their sampler
taps, the NV12 count from the oracle doubled for 16-bit words) plus the output (6 / 3 / 6 B/px RGB for the decodes,
12 / 6 B/px for f32 / f16 CHW).  The timed launches of an arm set share one output buffer; afterwards every arm runs
once more and its output is checked bit for bit: the 16-bit YUV arms against restate.decode_yuv16 (decode and 3a
on every frame, 3b on three frames through harness.restated, the f32 restatement of the oracle), the generic 3b arm
against the fast one, NV12 against restate.decode_yuv8 and the oracle on three frames, Bayer12 as
tools/bayer16_bench.py checks it, and end to end against the device run.

Writes one JSON line to DIR/yuv16_bench.jsonl (and stdout), with the card's name, power limit and max SM clock read
in the same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, e2e_result, parse_args, row, start, time_arms, write_line

YUV16 = ("P010", "P012", "I010", "I012")
ARMS = YUV16 + ("Nv12", "Bayer12")
MATRIX = "Bt709Limited"   # the matrix of HD video; NV12 keeps the reference's BT.601 limited


def main():
    ap = arg_parser(__doc__, "yuv16_bench")
    ap.add_argument("--e2e-frames", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=5)
    args = parse_args(ap)

    import numpy as np
    import torch

    import kornia_rs_b200 as kb
    from oracle import oracle as o
    from harness import bayer16_identity, restated, to_np16, yuv16_identity
    from restate import BITS, decode_yuv16, decode_yuv8, demosaic

    bench, facts = start("yuv16_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0x1016)
    ym = kb.YuvMatrix[MATRIX]
    fmt = {"P010": kb.SourceFormat.P010, "P012": kb.SourceFormat.P012, "I010": kb.SourceFormat.I010, "I012": kb.SourceFormat.I012,
           "Nv12": kb.SourceFormat.Nv12, "Bayer12": kb.SourceFormat.BayerRggb12}
    src_bpp = {**{k: 3.0 for k in YUV16}, "Nv12": 1.5, "Bayer12": 2.0}

    def frames_for(n, w, h):
        nv12 = torch.randint(0, 256, (n, w * h * 3 // 2), dtype=torch.uint8, device=dev, generator=gen)
        b16 = nv12.to(torch.int32)
        planar = torch.cat([b16[:, :w * h], b16[:, w * h::2], b16[:, w * h + 1::2]], 1)   # the I420 repack
        return {"P010": (b16 << 8).to(torch.uint16), "P012": (b16 << 8).to(torch.uint16), "I010": (planar << 2).to(torch.uint16),
                "I012": (planar << 4).to(torch.uint16), "Nv12": nv12,
                "Bayer12": torch.randint(0, 4096, (n, w * h), dtype=torch.int32, device=dev, generator=gen).to(torch.uint16)}

    def decode_call(k, src, out):
        if k == "Nv12":
            return kb.imgproc.rgb_from_nv12(src, out)
        if k == "Bayer12":
            return kb.imgproc.rgb_from_bayer16(src, out, kb.imgproc.BayerPattern.RGGB)
        return getattr(kb.imgproc, f"rgb_from_{k.lower()}")(src, out, matrix=ym)

    # ── decode ──
    decode = {}
    for tag, w, h, n in (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16)):
        src = frames_for(n, w, h)
        out16 = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint16, dev, batch=n)
        out8 = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n)
        outs = {k: out8 if k == "Nv12" else out16 for k in ARMS}
        fns = {k: (lambda k=k: decode_call(k, src[k], outs[k])) for k in ARMS}
        times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
        same = {}
        for k in ARMS:
            fns[k]()
            got = outs[k].data
            if k in YUV16:
                same[k] = all(bool(torch.equal(got[i:i + 8].to(torch.int32).to(torch.int64), decode_yuv16(src[k][i:i + 8], w, h, k, MATRIX)))
                              for i in range(0, n, 8))
            elif k == "Bayer12":
                same[k] = all(bool(torch.equal(got[i:i + 16].view(torch.int16), demosaic(src[k][i:i + 16].view(-1, h, w), "RGGB").view(torch.int16)))
                              for i in range(0, n, 16))
            else:
                same[k] = all(np.array_equal(got[i].cpu().numpy(), decode_yuv8(src[k][i].cpu().numpy(), w, h, "Nv12", "Bt601Limited"))
                              for i in sorted({0, n // 2, n - 1}))
        alg = {k: int(n * w * h * (src_bpp[k] + (3 if k == "Nv12" else 6))) for k in ARMS}
        decode[tag] = {"batch": n, "src": [w, h], **row(times, kernels, alg, same, "output_checked")}
        print(f"[yuv16_bench] decode {tag}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
        del src, outs, out16, out8
        torch.cuda.empty_cache()

    # ── camera preprocess, configs 3a / 3b, f32 and f16 ──
    w, h, n = 1920, 1080, 256
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    src = frames_for(n, w, h)
    # the Bayer12 frames with half the samples 0: the 16-bit Bayer identity kernel (plain __fdiv_rn) on zero dividends
    src["Bayer12_zeros"] = torch.where(torch.rand(src["Bayer12"].shape, device=dev, generator=gen) < 0.5, 0, src["Bayer12"].to(torch.int32)).to(torch.uint16)
    preprocess = {}
    for cfg, mode, (dw, dh) in (("cfg3a", "Stretch", (w, h)), ("cfg3b", "Letterbox", (640, 640))):
        def builder(k):
            b = kb.Preprocessor.builder().source_format(fmt[k]).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet())
            return (b.yuv_matrix(ym) if k in YUV16 else b).build_cuda()

        pres = {k: builder(k) for k in ARMS}
        ocfg = o.PreprocessCfg(mode=o.LETTERBOX if mode == "Letterbox" else o.STRETCH, fmt=o.FMT_NV12, mean=kb.IMAGENET_MEAN, inv_std=inv)
        nv12_bytes = w * h * 3 // 2 if cfg == "cfg3a" else o.preprocess_frame(src["Nv12"][0].cpu().numpy(), ocfg, w, h, dw, dh, count_touched=True)[1]
        arms = ARMS + (("P010_generic",) if cfg == "cfg3b" else ("Bayer12_zeros",))
        for f16 in (False, True):
            dt, it, out_b = (torch.float16, torch.int16, 6) if f16 else (torch.float32, torch.int32, 12)
            flat = torch.empty(n * 3 * dh * dw + 8, dtype=dt, device=dev)
            out = flat[:n * 3 * dh * dw].view(n, 3, dh, dw)
            k4 = 4 // flat.element_size()   # an output 4 bytes off 16-byte alignment: the fast kernels refuse it
            off = flat[k4:k4 + n * 3 * dh * dw].view(n, 3, dh, dw)

            def run(k, dst):   # the strided entry: a 256-frame pointer table costs more host time than a 3b launch takes
                p = pres[{"P010_generic": "P010", "Bayer12_zeros": "Bayer12"}.get(k, k)]
                s = src[{"P010_generic": "P010"}.get(k, k)]
                p.run_raw_strided(s.view(-1), s.shape[1] * s.element_size(), n, w, h, dst, f16=f16)

            fns = {k: (lambda k=k: run(k, off if k == "P010_generic" else out)) for k in arms}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            same = {}
            for k in arms:
                if k == "P010_generic":
                    continue
                run(k, out)
                if k in YUV16 and cfg == "cfg3a":
                    same[k] = all(bool(torch.equal(out[i:i + 8].view(it), yuv16_identity(src[k][i:i + 8], w, h, k, MATRIX, kb).to(dt).contiguous().view(it)))
                                  for i in range(0, n, 8))
                elif k in YUV16:
                    same[k] = all(np.array_equal(out[i].cpu().numpy().view(np.uint16 if f16 else np.uint32),
                                                 restated(kb, decode_yuv16(src[k][i].cpu(), w, h, k, MATRIX).numpy().astype(np.uint16), BITS[k], mode,
                                                          "Bilinear", dw, dh, f16).view(np.uint16 if f16 else np.uint32)) for i in (0, n // 2, n - 1))
                elif k in ("Bayer12", "Bayer12_zeros") and cfg == "cfg3a":
                    same[k] = all(bool(torch.equal(out[i:i + 16].view(it), bayer16_identity(src[k][i:i + 16].view(-1, h, w), "RGGB", 12, kb).to(dt).contiguous().view(it)))
                                  for i in range(0, n, 16))
                elif k == "Bayer12":
                    same[k] = all(np.array_equal(out[i].cpu().numpy().view(np.uint16 if f16 else np.uint32),
                                                 restated(kb, demosaic(to_np16(src[k][i]).reshape(h, w), "RGGB"), 12, mode, "Bilinear", dw, dh,
                                                          f16).view(np.uint16 if f16 else np.uint32)) for i in (0, n // 2, n - 1))
                else:
                    same[k] = all(np.array_equal(out[i].cpu().numpy().view(np.uint16 if f16 else np.uint32),
                                                 o.preprocess_frame(src[k][i].cpu().numpy(), ocfg, w, h, dw, dh, f16=f16).view(np.uint16 if f16 else np.uint32))
                                  for i in (0, n - 1))
                if k == "P010" and cfg == "cfg3b":
                    fast = out.clone()
                    run("P010_generic", off)
                    same["P010_generic"] = bool(torch.equal(off.view(it), fast.view(it)))
                    del fast
            src_b = {**{k: 2 * nv12_bytes for k in YUV16}, "P010_generic": 2 * nv12_bytes, "Nv12": nv12_bytes, "Bayer12": 2 * w * h,
                     "Bayer12_zeros": 2 * w * h}
            alg = {k: n * (src_b[k] + out_b * dw * dh) for k in arms}
            key = f"{cfg}_{'f16' if f16 else 'f32'}"
            preprocess[key] = {"batch": n, "src": [w, h], "dst": [dw, dh], "nv12_src_bytes_per_frame": nv12_bytes,
                               **row(times, kernels, alg, same, "output_checked")}
            print(f"[yuv16_bench] {key}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
            del out, off, flat
            torch.cuda.empty_cache()
    del src
    torch.cuda.empty_cache()

    # ── end to end, config 3a from host frames ──
    n = args.e2e_frames
    chunk, nstreams = 8, 3
    dsrc = frames_for(n, w, h)
    host = {k: torch.empty(dsrc[k].shape, dtype=dsrc[k].dtype, pin_memory=True) for k in ARMS}
    for k in ARMS:
        host[k].copy_(dsrc[k].cpu())
    del dsrc
    pres = {}
    for k in ARMS:
        b = kb.Preprocessor.builder().source_format(fmt[k]).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet())
        pres[k] = (b.yuv_matrix(ym) if k in YUV16 else b).build_cuda()
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
        print(f"[yuv16_bench] e2e cfg3a {k}: {e2e[k]['ms_per_step']} ms/step", file=sys.stderr, flush=True)
        del want, dev_frames
        torch.cuda.empty_cache()

    line = {"tool": "tools/yuv16_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "matrix_yuv16": MATRIX, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "decode": decode,
            "preprocess": preprocess, "e2e_cfg3a": {"batch": n, "chunk_frames": chunk, "streams": nstreams, "steps_per_rep": args.e2e_steps, **e2e}}
    write_line(args.out, "yuv16_bench", line)


if __name__ == "__main__":
    main()
