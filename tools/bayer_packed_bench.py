"""MIPI-packed Bayer (RAW10, RAW12, RAW14) against unpacked 12-bit Bayer, decode and camera preprocess, in one run.

    python tools/bayer_packed_bench.py --out DIR

Every arm carries the same samples (10-bit content, so every depth holds it): RAW10P, RAW12P and RAW14P packed frames
of the RGGB format, and the unpacked 12-bit frame (BayerRggb12, one 16-bit word per sample).  A further arm,
RAW12P_generic, runs the RAW12P frames from base addresses one byte off 16-B alignment, which sends them to the generic
kernels: the fast kernels must beat it on their own workloads.
Decode, 1080p x 256 and 4K x 16: rgb_from_bayer_packed against rgb_from_bayer16 (RGB16 HWC out for every arm).
Preprocess, 256 frames, ImageNet normalisation, f32 and f16 CHW out: config 3a (1080p -> 1080p, the identity kernels)
and 3b (1080p -> 640x640 letterbox, the generic kernel for every arm).
End to end: config 3a from pinned host frames to a pinned host tensor through a HostPipeline, 64 frames, f32 and f16,
recording the bytes each direction moved.

Every arm is timed with CUDA events over --iters launches after warm-up, the arms alternating, the whole set repeated
--reps times to show the spread.  Bandwidth uses algorithmic bytes over the H100 SXM data-sheet 3.35 TB/s: the frame
(1.25 / 1.5 / 1.75 B/px packed, 2 B/px unpacked; at 3b's exact 3:1 ratio a Bayer tap's 3x3 neighbourhood covers every
source sample) plus the output (6 B/px RGB16 for the decodes, 12 / 6 B/px for f32 / f16 CHW).
Every packed output is checked on the device, bit for bit: the decodes against the unpacked arm's output (the same
samples give the same RGB), the preprocess against the same samples run unpacked in the 16-bit format of the packed
depth (for RAW12P that is the unpacked arm itself), and end to end against the device run.

Writes one JSON line to DIR/bayer_packed_bench.jsonl (and stdout), with the card's name, power limit and max SM clock
read in the same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, e2e_result, parse_args, row, start, time_arms, write_line

PACKED = {"Raw10p": 10, "Raw12p": 12, "Raw14p": 14}
ARMS = ("Raw10p", "Raw12p", "Raw14p", "Bayer12", "Raw12p_generic")


def main():
    ap = arg_parser(__doc__, "bayer_packed_bench")
    ap.add_argument("--e2e-frames", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=5)
    args = parse_args(ap)

    import torch

    import kornia_rs_b200 as kb
    from restate import unpack

    bench, facts = start("bayer_packed_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0xBAC)
    SF = kb.SourceFormat
    fmt = {"Raw10p": SF.BayerRggb10p, "Raw12p": SF.BayerRggb12p, "Raw14p": SF.BayerRggb14p, "Bayer12": SF.BayerRggb12,
           "Raw12p_generic": SF.BayerRggb12p}
    twin_fmt = {"Raw10p": SF.BayerRggb10, "Raw12p": SF.BayerRggb12, "Raw14p": SF.BayerRggb14, "Raw12p_generic": SF.BayerRggb12}
    bpp = {"Raw10p": 1.25, "Raw12p": 1.5, "Raw14p": 1.75, "Bayer12": 2.0, "Raw12p_generic": 1.5}

    def pack_dev(samples, bits):
        """[n, h, w] int32 samples -> [n, h * w * bits / 8] uint8 on the device (the inverse of restate.unpack)."""
        g, gb, lo = (2, 3, 4) if bits == 12 else (4, bits // 2, bits - 8)
        n, h, w = samples.shape
        v = samples.view(n, h, w // g, g)
        field = torch.zeros_like(v[..., 0])
        for j in range(g):
            field |= (v[..., j] & ((1 << lo) - 1)) << (lo * j)
        parts = [v >> lo] + [((field >> (8 * i)) & 0xFF).unsqueeze(-1) for i in range(gb - g)]
        return torch.cat(parts, -1).to(torch.uint8).reshape(n, -1)

    def frames_for(n, w, h):
        """The same 10-bit samples in every arm; the generic arm's frames start one byte past a 16-B boundary."""
        s = torch.randint(0, 1024, (n, h, w), dtype=torch.int32, device=dev, generator=gen)
        out = {k: pack_dev(s, b) for k, b in PACKED.items()}
        out["Bayer12"] = s.to(torch.uint16).view(n, h * w)
        fb = out["Raw12p"].shape[1]
        slot = (fb + 1 + 15) // 16 * 16
        ring = torch.empty(n * slot + 16, dtype=torch.uint8, device=dev)
        mis = ring[1:1 + n * slot].view(n, slot)[:, :fb]
        mis.copy_(out["Raw12p"])
        out["Raw12p_generic"] = mis
        assert all(v.data_ptr() % 16 for v in mis[:4])
        return out

    def frame_bytes(k, w, h):
        return w * h * 2 if k == "Bayer12" else w * h * PACKED[k.split("_")[0]] // 8

    # ── decode ──
    decode = {}
    for tag, w, h, n in (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16)):
        src = frames_for(n, w, h)
        outs = {k: kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint16, dev, batch=n) for k in ARMS}

        def fn(k):
            if k == "Bayer12":
                return lambda: kb.imgproc.rgb_from_bayer16(src[k], outs[k], kb.imgproc.BayerPattern.RGGB)
            return lambda: kb.imgproc.rgb_from_bayer_packed(src[k], outs[k], kb.imgproc.BayerPattern.RGGB, PACKED[k])

        fns = {k: fn(k) for k in ARMS if k != "Raw12p_generic"}
        # the generic arm: the decoder takes tight frames, so its frames are the RAW12P ones copied one byte past alignment
        gsrc = torch.empty(n * frame_bytes("Raw12p", w, h) + 1, dtype=torch.uint8, device=dev)[1:]
        gsrc.copy_(src["Raw12p"].reshape(-1))
        fns["Raw12p_generic"] = lambda: kb.imgproc.rgb_from_bayer_packed(gsrc, outs["Raw12p_generic"], kb.imgproc.BayerPattern.RGGB, 12)
        times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
        same = {k: bool(torch.equal(outs[k].data.view(torch.int16), outs["Bayer12"].data.view(torch.int16))) for k in ARMS if k != "Bayer12"}
        same["Bayer12"] = None
        alg = {k: int(n * (frame_bytes(k, w, h) + 6 * w * h)) for k in ARMS}
        decode[tag] = {"batch": n, "src": [w, h], **row(times, kernels, alg, same, "output_checked")}
        print(f"[bayer_packed_bench] decode {tag}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
        del src, outs, gsrc
        torch.cuda.empty_cache()

    # ── camera preprocess, configs 3a / 3b, f32 and f16 ──
    w, h, n = 1920, 1080, 256
    src = frames_for(n, w, h)
    frames = {k: [src[k][i] for i in range(n)] for k in ARMS}
    preprocess = {}
    for cfg, mode, (dw, dh) in (("cfg3a", "Stretch", (w, h)), ("cfg3b", "Letterbox", (640, 640))):
        def builder(f):
            return kb.Preprocessor.builder().source_format(f).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet()).build_cuda()

        pres = {k: builder(fmt[k]) for k in ARMS}
        arms = ARMS if cfg == "cfg3a" else ARMS[:4]   # 3b takes the generic kernel for every arm
        for f16 in (False, True):
            dt, it, out_b = (torch.float16, torch.int16, 6) if f16 else (torch.float32, torch.int32, 12)
            outs = {k: torch.empty((n, 3, dh, dw), dtype=dt, device=dev) for k in arms}
            fns = {k: (lambda k=k: (pres[k].run_raw_batch_f16 if f16 else pres[k].run_raw_batch)(frames[k], w, h, outs[k])) for k in arms}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            same = {"Bayer12": None}
            want = torch.empty((32, 3, dh, dw), dtype=dt, device=dev)
            for k in arms:
                if k == "Bayer12":
                    continue
                twin = builder(twin_fmt[k])
                ok = True
                for k0 in range(0, n, 32):
                    (twin.run_raw_batch_f16 if f16 else twin.run_raw_batch)([src["Bayer12"][i] for i in range(k0, k0 + 32)], w, h, want)
                    ok = ok and bool(torch.equal(outs[k][k0:k0 + 32].view(it), want.view(it)))
                same[k] = ok
            alg = {k: n * (frame_bytes(k, w, h) + out_b * dw * dh) for k in arms}
            key = f"{cfg}_{'f16' if f16 else 'f32'}"
            preprocess[key] = {"batch": n, "src": [w, h], "dst": [dw, dh], **row(times, kernels, alg, same, "output_checked")}
            print(f"[bayer_packed_bench] {key}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
            del outs, want
            torch.cuda.empty_cache()
    del frames, src
    torch.cuda.empty_cache()

    # ── end to end, config 3a from host frames, f32 and f16 ──
    n = args.e2e_frames
    chunk, nstreams = 8, 3
    e2e_arms = ARMS[:4]
    s = frames_for(n, w, h)
    host = {k: s[k].cpu().pin_memory() for k in e2e_arms}
    del s
    pres = {k: kb.Preprocessor.builder().source_format(fmt[k]).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda()
            for k in e2e_arms}
    pipes = {k: kb.imgproc.HostPipeline(dev, src_chunk_bytes=chunk * ((frame_bytes(k, w, h) + 15) // 16 * 16), dst_chunk_bytes=chunk * 12 * w * h,
                                        depth=nstreams) for k in e2e_arms}
    e2e = {}
    for f16 in (False, True):
        dt, it = (torch.float16, torch.int16) if f16 else (torch.float32, torch.int32)
        outs = {k: torch.empty((n, 3, h, w), dtype=dt, pin_memory=True) for k in e2e_arms}
        fns = {k: (lambda k=k: pres[k].run_raw_host(host[k], w, h, (w, h), out=outs[k], f16=f16, pipeline=pipes[k])) for k in e2e_arms}
        steps, _ = time_arms(bench, fns, args.e2e_steps, 1, args.reps, st, kb)
        res = {}
        for k in e2e_arms:
            transfer = pipes[k].last_transfer()
            want = torch.empty((n, 3, h, w), dtype=dt, device=dev)
            dev_frames = host[k].to(dev)
            (pres[k].run_raw_batch_f16 if f16 else pres[k].run_raw_batch)([dev_frames[i] for i in range(n)], w, h, want)
            res[k] = e2e_result(steps[k], transfer, bool(torch.equal(outs[k].to(dev).view(it), want.view(it))))
            print(f"[bayer_packed_bench] e2e cfg3a {'f16' if f16 else 'f32'} {k}: {res[k]['ms_per_step']} ms/step", file=sys.stderr, flush=True)
            del want, dev_frames
            torch.cuda.empty_cache()
        e2e["f16" if f16 else "f32"] = res
        del outs
    for p in pipes.values():
        p.close()

    line = {"tool": "tools/bayer_packed_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "decode": decode, "preprocess": preprocess,
            "e2e_cfg3a": {"batch": n, "chunk_frames": chunk, "streams": nstreams, "steps_per_rep": args.e2e_steps, **e2e}}
    write_line(args.out, "bayer_packed_bench", line)


if __name__ == "__main__":
    main()
