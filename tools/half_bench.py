"""f32 vs f16 vs bf16 output of the fused u8 -> CHW resize+normalize, device and end to end, in one run.

    python tools/half_bench.py --out DIR

Device: config 2 (64 x 4K -> 1280x720, FR_POINT), 16 x 4K -> 1920x1080 (FR_BOX) and 16 x 4K -> 1600x900 (FR_GENERAL),
timed with CUDA events over --iters launches after warm-up, the three output types alternating, the whole set repeated
--reps times to show the spread.  Bandwidth uses algorithmic bytes: distinct tapped source bytes + 4 or 2 bytes per
output value, over the H100 SXM data-sheet 3.35 TB/s.

End to end: config 2 from pinned host buffers to a pinned host tensor through a HostPipeline with bench.py's e2e
chunking (8 frames per chunk, a 3-stream ring), f32 vs f16 vs bf16 alternating, ms per step and link bytes.

Writes one JSON line to DIR/half_bench.jsonl (and stdout), with the card's name, power limit and max SM clock read in the
same run.
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0   # H100 SXM data sheet HBM3


def _bench_module():
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def gpu_facts() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def tapped_pixels(sw, sh, dw, dh):
    """Distinct source pixels addressed by >= 1 tap of the fused sampler (resize/fused.rs:196-201), as bench.py counts them."""
    import numpy as np

    def axis(s_len, d_len):
        i = np.arange(d_len, dtype=np.float32)
        f = np.maximum((i + np.float32(0.5)) * (np.float32(s_len) / np.float32(d_len)) - np.float32(0.5), np.float32(0))
        i0 = np.minimum(f.astype(np.int64), s_len - 1)
        return len(np.union1d(i0, np.minimum(i0 + 1, s_len - 1)))
    return axis(sw, dw) * axis(sh, dh)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for half_bench.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=10)
    args = ap.parse_args()
    if args.iters < 20 or args.reps < 3:
        ap.error("--iters >= 20 and --reps >= 3: fewer cannot show the spread")

    import torch

    import kornia_rs_b200 as kb

    if not torch.cuda.is_available():
        raise SystemExit("half_bench.py needs a CUDA device")
    bench = _bench_module()
    facts = gpu_facts()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    p = kb.imgproc.NormalizeParams.from_mean_std(bench.IMAGENET_MEAN, bench.IMAGENET_STD)
    scale, bias = p.scale, p.bias
    SW, SH, N = bench.SW, bench.SH, bench.BATCH
    src = torch.empty((N, SH, SW, 3), dtype=torch.uint8, device=dev)
    gen = bench.LcgPattern(SW * SH * 3, dev)
    for i in range(N):
        gen.frame(0x12345678 + i, src[i].view(-1))   # bench.py's headline frames
    del gen
    dtypes = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
    esize = {"f32": 4, "f16": 2, "bf16": 2}
    op = kb.imgproc.resize_normalize_to_tensor_u8_bilinear

    # ── device ──
    workloads = [("cfg2_point_4k_to_720p", 1280, 720, N), ("box_4k_to_1080p", 1920, 1080, 16), ("general_4k_to_1600x900", 1600, 900, 16)]
    device = {}
    for tag, dw, dh, n in workloads:
        s = src[:n]
        outs = {k: torch.empty((n, 3, dh, dw), dtype=t, device=dev) for k, t in dtypes.items()}
        fns = {k: (lambda k=k: op(s, dw, dh, scale, bias, dtypes[k], out=outs[k])) for k in dtypes}
        times = {k: [] for k in dtypes}
        kernels = {}
        for _ in range(args.reps):
            for k in dtypes:
                times[k].append(bench.time_launches(fns[k], args.iters, args.warmup, st))
                kernels[k] = kb._lib.last_kernel()
        same = {k: bool(torch.equal(outs[k].view(torch.int16), outs["f32"].to(dtypes[k]).view(torch.int16))) for k in ("f16", "bf16")}
        tapped = tapped_pixels(SW, SH, dw, dh)
        row = {"batch": n, "dst": [dw, dh], "tapped_src_bytes_per_frame": tapped * 3, "bit_identical_to_f32_cast": same}
        for k in dtypes:
            alg = n * (tapped * 3 + esize[k] * 3 * dw * dh)
            best = min(times[k])
            row[k] = {"ms": [round(t, 4) for t in times[k]], "ms_min": round(best, 4), "gpix_s": round(n * dw * dh / (best * 1e-3) / 1e9, 2),
                      "alg_bytes": alg, "gbs": round(alg / (best * 1e-3) / 1e9, 1), "frac_of_3350": round(alg / (best * 1e-3) / 1e9 / PEAK_GBS, 3),
                      "kernel": kernels[k]}
        device[tag] = row
        print(f"[half_bench] {tag}: " + "  ".join(f"{k} {row[k]['ms']} ms" for k in dtypes), file=sys.stderr, flush=True)
        del outs

    # ── end to end: host buffers, bench.py's e2e chunking ──
    DW, DH = bench.DW, bench.DH
    chunk, nstreams = 8, 3
    host_src = torch.empty((N, SH, SW, 3), dtype=torch.uint8, pin_memory=True)
    host_src.copy_(src)
    ref = {k: op(src, DW, DH, scale, bias, dtypes[k]) for k in dtypes}
    del src
    e2e = {}
    pipes, hosts = {}, {}
    for k in dtypes:
        pipes[k] = kb.imgproc.HostPipeline(dev, src_chunk_bytes=chunk * SW * SH * 3, dst_chunk_bytes=chunk * 3 * DW * DH * esize[k], depth=nstreams)
        hosts[k] = torch.empty((N, 3, DH, DW), dtype=dtypes[k], pin_memory=True)
    steps = {k: [] for k in dtypes}
    for _ in range(args.reps):
        for k in dtypes:
            fn = lambda: op(host_src, DW, DH, scale, bias, dtypes[k], out=hosts[k], pipeline=pipes[k])
            fn(); fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.e2e_steps):
                fn()
            e1.record(st)
            torch.cuda.synchronize()
            steps[k].append(e0.elapsed_time(e1) / args.e2e_steps)
    for k in dtypes:
        up, down = pipes[k].last_transfer()
        best = min(steps[k])
        e2e[k] = {"ms_per_step": [round(t, 3) for t in steps[k]], "ms_min": round(best, 3), "h2d_bytes": up, "d2h_bytes": down,
                  "h2d_gbs": round(up / (best * 1e-3) / 1e9, 1), "d2h_gbs": round(down / (best * 1e-3) / 1e9, 1),
                  "gpix_s": round(N * DW * DH / (best * 1e-3) / 1e9, 3),
                  "matches_device_result": bool(torch.equal(hosts[k].to(dev).view(torch.int16 if esize[k] == 2 else torch.int32),
                                                            ref[k].view(torch.int16 if esize[k] == 2 else torch.int32)))}
        pipes[k].close()
        print(f"[half_bench] e2e {k}: {e2e[k]['ms_per_step']} ms/step", file=sys.stderr, flush=True)

    line = {"tool": "tools/half_bench.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "reps": args.reps, "peak_gbs": PEAK_GBS, "peak_source": "H100 SXM data sheet, 3.35 TB/s", "device": device,
            "e2e_cfg2": {"batch": N, "chunk_frames": chunk, "streams": nstreams, "steps_per_rep": args.e2e_steps, **e2e}}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "half_bench.jsonl"), "a") as f:
        f.write(json.dumps(line) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
