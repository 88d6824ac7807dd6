"""4:4:4 video (I444, I410, I410Msb) against its 4:2:0 siblings (NV12, P010), decode and camera preprocess, in one run.

    python tools/yuv444_bench.py --out DIR

Every arm carries the same picture: random I420 bytes.  I444 is that frame with its chroma replicated 2x2, I410 /
I410Msb the I444 bytes as 10-bit codes in the low / high bits of 16-bit words (byte << 2 / byte << 8); NV12 is the I420
frame repacked, P010 the NV12 bytes as words (byte << 8).  So every 8-bit arm decodes to the same RGB8 picture and every
16-bit arm to the same RGB16 picture, whatever the matrix (BT.709 limited throughout).
Decode, 1080p x 256 and 4K x 16: rgb_from_i444 / rgb_from_nv12 (RGB8 out), rgb_from_i410 / _i410msb / _p010 (RGB16 out).
Preprocess, 256 frames, ImageNet normalisation, f32 and f16 CHW out: config 3a (1080p -> 1080p, the identity kernels)
and 3b (1080p -> 640x640 letterbox), plus for 3b the I444 frames on the generic kernel (an output 4 bytes off 16-byte
alignment, which the fast kernel refuses) to show what the fast kernel buys.  Preprocess launches go through the strided
entry (one ring of 256 frames), as tools/yuv16_bench.py does.
End to end: config 3a from pinned host frames to a pinned host f32 tensor through a HostPipeline, 64 frames, recording
the bytes each direction moved.

Every arm is timed with CUDA events over --iters launches after warm-up, the arms alternating, the whole set repeated
--reps times; the minimum is reported.  Bandwidth uses algorithmic bytes over the H100 SXM data-sheet 3.35 TB/s: the
frame (I444 3 B/px, I41x 6 B/px, NV12 1.5 B/px, P010 3 B/px; for 3b the distinct bytes the sampler taps, counted by the
oracle on the RGB8 twin for 4:4:4 and on the NV12 frame for 4:2:0, doubled for 16-bit words) plus the output (3 / 6 B/px
RGB for the decodes, 12 / 6 B/px for f32 / f16 CHW).  Afterwards every arm runs once more and its output is checked bit
for bit: the 4:4:4 arms against their 4:2:0 sibling on every frame (the twin identity), NV12 and P010 against
restate.decode_yuv8, restate.decode_yuv16 and the oracle, the generic 3b arm against the fast one,
and end to end against the device run.

Writes one JSON line to DIR/yuv444_bench.jsonl (and stdout), with the card's name, power limit and max SM clock read in
the same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, e2e_result, parse_args, row, start, time_arms, write_line

ARMS = ("I444", "I410", "I410Msb", "Nv12", "P010")
SIBLING = {"I444": "Nv12", "I410": "P010", "I410Msb": "P010"}   # the 4:2:0 arm each 4:4:4 arm must equal bit for bit
WORDS = ("I410", "I410Msb", "P010")
MATRIX = "Bt709Limited"


def main():
    ap = arg_parser(__doc__, "yuv444_bench")
    ap.add_argument("--e2e-frames", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=5)
    args = parse_args(ap)

    import numpy as np
    import torch

    import kornia_rs_b200 as kb
    from oracle import oracle as o
    from harness import restated, yuv16_identity
    from restate import decode_yuv16, decode_yuv8

    bench, facts = start("yuv444_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0x444)
    ym = kb.YuvMatrix[MATRIX]
    src_bpp = {"I444": 3.0, "I410": 6.0, "I410Msb": 6.0, "Nv12": 1.5, "P010": 3.0}

    def frames_for(n, w, h):
        i420 = torch.randint(0, 256, (n, w * h * 3 // 2), dtype=torch.uint8, device=dev, generator=gen)
        q = (w // 2) * (h // 2)
        u, v = i420[:, w * h:w * h + q], i420[:, w * h + q:]
        up = lambda a: a.view(n, h // 2, 1, w // 2, 1).expand(n, h // 2, 2, w // 2, 2).reshape(n, w * h)
        i444 = torch.cat([i420[:, :w * h], up(u), up(v)], 1)
        nv12 = torch.cat([i420[:, :w * h], torch.stack([u, v], -1).reshape(n, 2 * q)], 1)
        b444 = i444.to(torch.int32)
        return {"I444": i444, "I410": (b444 << 2).to(torch.uint16), "I410Msb": (b444 << 8).to(torch.uint16), "Nv12": nv12,
                "P010": (nv12.to(torch.int32) << 8).to(torch.uint16)}

    # ── decode ──
    decode = {}
    for tag, w, h, n in (("1080p_x256", 1920, 1080, 256), ("4k_x16", 3840, 2160, 16)):
        src = frames_for(n, w, h)
        outs = {k: kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint16 if k in WORDS else torch.uint8, dev, batch=n) for k in ARMS}
        fns = {k: (lambda k=k: getattr(kb.imgproc, f"rgb_from_{k.lower()}")(src[k], outs[k], matrix=ym)) for k in ARMS}
        times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
        for k in ARMS:
            fns[k]()
        torch.cuda.synchronize()
        same = {"Nv12": all(np.array_equal(outs["Nv12"].data[i].cpu().numpy(), decode_yuv8(src["Nv12"][i].cpu().numpy(), w, h, "Nv12", MATRIX))
                            for i in sorted({0, n // 2, n - 1})),
                "P010": all(bool(torch.equal(outs["P010"].data[i:i + 8].to(torch.int32).to(torch.int64), decode_yuv16(src["P010"][i:i + 8], w, h, "P010", MATRIX)))
                            for i in range(0, n, 8))}
        for k, sib in SIBLING.items():
            same[k] = bool(torch.equal(outs[k].data, outs[sib].data))
        alg = {k: int(n * w * h * (src_bpp[k] + (6 if k in WORDS else 3))) for k in ARMS}
        decode[tag] = {"batch": n, "src": [w, h], **row(times, kernels, alg, same, "output_checked")}
        print(f"[yuv444_bench] decode {tag}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
        del src, outs
        torch.cuda.empty_cache()

    # ── camera preprocess, configs 3a / 3b, f32 and f16 ──
    w, h, n = 1920, 1080, 256
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)
    src = frames_for(n, w, h)
    preprocess = {}
    for cfg, mode, (dw, dh) in (("cfg3a", "Stretch", (w, h)), ("cfg3b", "Letterbox", (640, 640))):
        pres = {k: kb.Preprocessor.builder().source_format(kb.SourceFormat[k]).mode(kb.ResizeMode[mode]).normalize(kb.Normalize.imagenet())
                .yuv_matrix(ym).build_cuda() for k in ARMS}
        ocfg = o.PreprocessCfg(mode=o.LETTERBOX if mode == "Letterbox" else o.STRETCH, fmt=o.FMT_NV12, mean=kb.IMAGENET_MEAN, inv_std=inv)
        rcfg = o.PreprocessCfg(mode=o.LETTERBOX if mode == "Letterbox" else o.STRETCH, fmt=o.FMT_RGB, mean=kb.IMAGENET_MEAN, inv_std=inv)
        if cfg == "cfg3a":
            nv12_bytes, rgb_bytes = w * h * 3 // 2, 3 * w * h
        else:
            nv12_bytes = o.preprocess_frame(src["Nv12"][0].cpu().numpy(), ocfg, w, h, dw, dh, count_touched=True)[1]
            rgb_bytes = o.preprocess_frame(np.zeros(3 * w * h, np.uint8), rcfg, w, h, dw, dh, count_touched=True)[1]
        arms = ARMS + (("I444_generic",) if cfg == "cfg3b" else ())
        for f16 in (False, True):
            dt, it, out_b = (torch.float16, torch.int16, 6) if f16 else (torch.float32, torch.int32, 12)
            flat = torch.empty(n * 3 * dh * dw + 8, dtype=dt, device=dev)
            out = flat[:n * 3 * dh * dw].view(n, 3, dh, dw)
            k4 = 4 // flat.element_size()   # an output 4 bytes off 16-byte alignment: the fast kernels refuse it
            off = flat[k4:k4 + n * 3 * dh * dw].view(n, 3, dh, dw)

            def run(k, dst):
                kk = "I444" if k == "I444_generic" else k
                s = src[kk]
                pres[kk].run_raw_strided(s.view(-1), s.shape[1] * s.element_size(), n, w, h, dst, f16=f16)

            fns = {k: (lambda k=k: run(k, off if k == "I444_generic" else out)) for k in arms}
            times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
            same, ref = {}, {}
            for k in ("Nv12", "P010"):
                run(k, out)
                if k == "P010" and cfg == "cfg3a":
                    same[k] = all(bool(torch.equal(out[i:i + 8].view(it), yuv16_identity(src[k][i:i + 8], w, h, k, MATRIX, kb).to(dt).contiguous().view(it)))
                                  for i in range(0, n, 8))
                elif k == "P010":
                    same[k] = all(np.array_equal(out[i].cpu().numpy().view(np.uint16 if f16 else np.uint32),
                                                 restated(kb, decode_yuv16(src[k][i].cpu(), w, h, k, MATRIX).numpy().astype(np.uint16), 10, mode,
                                                          "Bilinear", dw, dh, f16).view(np.uint16 if f16 else np.uint32)) for i in (0, n // 2, n - 1))
                else:   # the oracle on the RGB8 twin of the BT.709 picture
                    same[k] = all(np.array_equal(out[i].cpu().numpy().view(np.uint16 if f16 else np.uint32),
                                                 o.preprocess_frame(decode_yuv8(src[k][i].cpu().numpy(), w, h, "Nv12", MATRIX).reshape(-1), rcfg, w, h, dw, dh,
                                                                    f16=f16).view(np.uint16 if f16 else np.uint32)) for i in (0, n - 1))
                ref[k] = out.clone()
            for k in arms:
                if k in SIBLING or k == "I444_generic":
                    dst = off if k == "I444_generic" else out
                    run(k, dst)
                    same[k] = bool(torch.equal(dst.view(it), ref[SIBLING.get(k, "Nv12")].view(it)))
            del ref
            src_b = {"I444": rgb_bytes, "I444_generic": rgb_bytes, "I410": 2 * rgb_bytes, "I410Msb": 2 * rgb_bytes, "Nv12": nv12_bytes,
                     "P010": 2 * nv12_bytes}
            alg = {k: n * (src_b[k] + out_b * dw * dh) for k in arms}
            key = f"{cfg}_{'f16' if f16 else 'f32'}"
            preprocess[key] = {"batch": n, "src": [w, h], "dst": [dw, dh], "i444_src_bytes_per_frame": rgb_bytes, "nv12_src_bytes_per_frame": nv12_bytes,
                               **row(times, kernels, alg, same, "output_checked")}
            print(f"[yuv444_bench] {key}: " + "  ".join(f"{k} {min(times[k]):.4f}" for k in times), file=sys.stderr, flush=True)
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
    pres = {k: kb.Preprocessor.builder().source_format(kb.SourceFormat[k]).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet())
            .yuv_matrix(ym).build_cuda() for k in ARMS}
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
        print(f"[yuv444_bench] e2e cfg3a {k}: {e2e[k]['ms_per_step']} ms/step", file=sys.stderr, flush=True)
        del want, dev_frames
        torch.cuda.empty_cache()

    line = {"tool": "tools/yuv444_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "matrix": MATRIX, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "decode": decode,
            "preprocess": preprocess, "e2e_cfg3a": {"batch": n, "chunk_frames": chunk, "streams": nstreams, "steps_per_rep": args.e2e_steps, **e2e}}
    write_line(args.out, "yuv444_bench", line)


if __name__ == "__main__":
    main()
