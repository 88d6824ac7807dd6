"""Camera preprocess with bfloat16 output against f32 and f16, kernel by kernel and end to end, in one run.

    python tools/preprocess_bf16_bench.py --out DIR

Arms: the same call into an f32, an f16 and a bf16 destination (Preprocessor.run_raw_strided(..., dtype=...)), the
three alternating.  256 frames, ImageNet normalisation, BT.601 limited:
  * fast kernels, config 3a (1080p -> 1080p: the identity kernels) and 3b (1080p -> 640x640 letterbox): NV12, P010,
    BayerRggb12 and I444 (3b for BayerRggb12 is the generic kernel: the Bayer formats have no letterbox fast kernel);
  * the generic kernel: YUYV 3a and 3b, and NV12 3b with Lanczos sampling;
  * end to end: config 3a x 64 NV12 frames from pinned host memory to a pinned host tensor through a HostPipeline,
    with the bytes each direction moved (kb200_host_pipeline_last_transfer).
Every arm is timed with CUDA events over --iters launches after warm-up, the whole set repeated --reps times; minima
are reported.  Bandwidth: algorithmic bytes over the H100 SXM data-sheet 3.35 TB/s, as DESIGN §4 counts them: the
source bytes the sampler taps (3a: the whole frame; 3b: the tapped pixels the oracle counts on the NV12 frame and on
the RGB8 twin, at the format's bytes per pixel; Lanczos: the whole frame) plus the output, 4 B (f32) or 2 B (f16, bf16)
per value.  Every bf16 output of the run is checked bit for bit against the f32 arm's output of the same call rounded
by torch's .to(torch.bfloat16).

Writes one JSON line to DIR/preprocess_bf16_bench.jsonl (and stdout), with the card's name, power limit and max SM
clock read in the same run.
"""
from __future__ import annotations

import sys
import time

from benchkit import PEAK_GBS, arg_parser, e2e_result, parse_args, start, time_arms, write_line

OUTS = ("f32", "f16", "bf16")
FAST = ("Nv12", "P010", "BayerRggb12", "I444")
SRC_BPP = {"Nv12": 1.5, "P010": 3.0, "BayerRggb12": 2.0, "I444": 3.0, "Yuyv": 2.0}   # frame bytes per pixel
TAP_BPP = {"Nv12": None, "P010": None, "BayerRggb12": 2, "I444": 3, "Yuyv": 2}         # 3b: bytes per tapped pixel (None: the NV12 count)


def main():
    ap = arg_parser(__doc__, "preprocess_bf16_bench")
    ap.add_argument("--e2e-frames", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=5)
    args = parse_args(ap)

    import numpy as np
    import torch

    import kornia_rs_b200 as kb
    from oracle import oracle as o

    bench, facts = start("preprocess_bf16_bench")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    gen = torch.Generator(device=dev).manual_seed(0xBF16)
    dtypes = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
    esz = {"f32": 4, "f16": 2, "bf16": 2}
    w, h, n = 1920, 1080, 256
    inv = tuple(float(np.float32(1.0) / np.float32(s)) for s in kb.IMAGENET_STD)

    def frames(fmt, count):
        if fmt == "BayerRggb12":
            return torch.randint(0, 4096, (count, w * h), dtype=torch.int32, device=dev, generator=gen).to(torch.uint16)
        if fmt == "P010":   # 10-bit codes in the high bits, junk in the low 6
            return torch.randint(0, 65536, (count, w * h * 3 // 2), dtype=torch.int32, device=dev, generator=gen).to(torch.uint16)
        nbytes = int(w * h * SRC_BPP[fmt])
        return torch.randint(0, 256, (count, nbytes), dtype=torch.uint8, device=dev, generator=gen)

    # tapped source pixels of config 3b (1080p -> 640x640 letterbox, bilinear), counted by the oracle
    lb = o.PreprocessCfg(mode=o.LETTERBOX, fmt=o.FMT_NV12, mean=kb.IMAGENET_MEAN, inv_std=inv)
    nv12_3b = o.preprocess_frame(np.zeros(w * h * 3 // 2, np.uint8), lb, w, h, 640, 640, count_touched=True)[1]
    rgb_cfg = o.PreprocessCfg(mode=o.LETTERBOX, fmt=o.FMT_RGB, mean=kb.IMAGENET_MEAN, inv_std=inv)
    px_3b = o.preprocess_frame(np.zeros(3 * w * h, np.uint8), rgb_cfg, w, h, 640, 640, count_touched=True)[1] // 3

    def src_bytes(fmt, cfg, lanczos=False):
        if cfg == "cfg3a" or lanczos:
            return int(w * h * SRC_BPP[fmt])
        if TAP_BPP[fmt] is None:
            return nv12_3b * (2 if fmt == "P010" else 1)
        return px_3b * TAP_BPP[fmt]

    preprocess = {}
    plan = [(fmt, cfg, "Bilinear") for fmt in FAST + ("Yuyv",) for cfg in ("cfg3a", "cfg3b")] + [("Nv12", "cfg3b", "Lanczos")]
    for fmt, cfg, samp in plan:
        dw, dh = (w, h) if cfg == "cfg3a" else (640, 640)
        pre = (kb.Preprocessor.builder().source_format(kb.SourceFormat[fmt]).mode(kb.ResizeMode.Stretch if cfg == "cfg3a" else kb.ResizeMode.Letterbox)
               .normalize(kb.Normalize.imagenet()).sampling(kb.InterpolationMode[samp]).build_cuda())
        src = frames(fmt, n)
        stride = src.shape[1] * src.element_size()
        outs = {k: torch.empty((n, 3, dh, dw), dtype=dtypes[k], device=dev) for k in OUTS}
        fns = {k: (lambda k=k: pre.run_raw_strided(src.view(-1), stride, n, w, h, outs[k], dtype=dtypes[k])) for k in OUTS}
        times, kernels = time_arms(bench, fns, args.iters, args.warmup, args.reps, st, kb)
        for k in OUTS:
            fns[k]()
        torch.cuda.synchronize()
        want = outs["f32"].to(torch.bfloat16)
        ok = bool(torch.equal(torch.isnan(want), torch.isnan(outs["bf16"]))
                  and torch.equal(outs["bf16"].view(torch.int16)[~torch.isnan(want)], want.view(torch.int16)[~torch.isnan(want)]))
        del want
        sb = src_bytes(fmt, cfg, samp == "Lanczos")
        row = {}
        for k in OUTS:
            best = min(times[k])
            alg = n * (sb + 3 * dw * dh * esz[k])
            gbs = alg / (best * 1e-3) / 1e9
            row[k] = {"ms": [round(t, 4) for t in times[k]], "ms_min": round(best, 4), "spread": round((max(times[k]) - best) / best, 4),
                      "alg_bytes": alg, "gbs": round(gbs, 1), "frac_of_3350": round(gbs / PEAK_GBS, 3), "kernel": kernels[k]}
        row["bf16"]["equals_f32_rounded"] = ok
        row["bf16_over_f16"] = round(row["bf16"]["ms_min"] / row["f16"]["ms_min"], 3)
        key = f"{fmt}_{cfg}" + ("_lanczos" if samp == "Lanczos" else "")
        preprocess[key] = {"batch": n, "src": [w, h], "dst": [dw, dh], "src_bytes_per_frame": sb, **row}
        print(f"[preprocess_bf16_bench] {key}: " + "  ".join(f"{k} {row[k]['ms_min']:.4f} ms ({row[k]['frac_of_3350']})" for k in OUTS)
              + f"  bf16 == f32 rounded: {ok}", file=sys.stderr, flush=True)
        del src, outs
        torch.cuda.empty_cache()

    # ── end to end, config 3a from host frames ──
    ne = args.e2e_frames
    chunk, nstreams = 8, 3
    host = torch.empty((ne, w * h * 3 // 2), dtype=torch.uint8, pin_memory=True)
    host.copy_(frames("Nv12", ne).cpu())
    pre = kb.Preprocessor.builder().source_format(kb.SourceFormat.Nv12).mode(kb.ResizeMode.Stretch).normalize(kb.Normalize.imagenet()).build_cuda()
    outs = {k: torch.empty((ne, 3, h, w), dtype=dtypes[k], pin_memory=True) for k in OUTS}
    pipe = kb.imgproc.HostPipeline(dev, src_chunk_bytes=chunk * ((host.shape[1] + 15) // 16 * 16), dst_chunk_bytes=chunk * 12 * w * h, depth=nstreams)
    steps, transfer = {k: [] for k in OUTS}, {}
    for _ in range(args.reps):   # one pipeline for the three arms: each arm's link bytes are read right after its turn
        for k in OUTS:
            fn = lambda k=k: pre.run_raw_host(host, w, h, (w, h), out=outs[k], pipeline=pipe, dtype=dtypes[k])
            steps[k].append(bench.time_launches(fn, args.e2e_steps, 1, st))
            transfer[k] = pipe.last_transfer()
    pipe.close()
    want = outs["f32"].to(torch.bfloat16)
    e2e_ok = bool(torch.equal(outs["bf16"].view(torch.int16), want.view(torch.int16)))
    e2e = {}
    for k in OUTS:
        e2e[k] = e2e_result(steps[k], transfer[k])
        print(f"[preprocess_bf16_bench] e2e cfg3a {k}: {e2e[k]['ms_per_step']} ms/step, {transfer[k][0]} B up, {transfer[k][1]} B down",
              file=sys.stderr, flush=True)
    e2e["bf16"]["equals_f32_rounded"] = e2e_ok

    line = {"tool": "tools/preprocess_bf16_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "preprocess": preprocess,
            "e2e_cfg3a": {"batch": ne, "chunk_frames": chunk, "streams": nstreams, "steps_per_rep": args.e2e_steps, **e2e}}
    write_line(args.out, "preprocess_bf16_bench", line)


if __name__ == "__main__":
    main()
