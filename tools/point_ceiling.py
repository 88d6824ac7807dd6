"""What HBM gives for the fused resize headline's own traffic, next to the kernels that move it.

    python tools/point_ceiling.py --out DIR [--rounds 5] [--iters 20] [--half]

The headline (bench.py) resizes 64 frames 3840x2160 -> 1280x720, u8 HWC -> f32 CHW, in the point mode: it reads 1 of
every 3 source rows whole (11,520 B: the 9-byte tap stride puts a tap in every 32-B sector) and writes three f32 planes.
On the headline's own buffers ([64,2160,3840,3] u8, [64,3,720,1280] f32) this times:

  a  read     a read-only pass over exactly the tapped rows (y = 3d + 1)                          530,841,600 B
  b  write    a write-only pass over the destination                                             707,788,800 B
  c  twin     reads the tapped rows, writes every destination value as (float)byte: the headline's traffic with no
              arithmetic; one CTA per (image, destination row), LDG.128 / lane-contiguous STG.128   1,238,630,400 B
  d  memcpy   cudaMemcpyAsync device to device of 619,315,200 B (1,238,630,400 B moved)
  e  tiled    the headline launch on the tiled point schedule (knob fr.rows = 1)
  f  rows     the headline launch on the full-row point schedule (knob fr.rows = 2)
  --half      e and f again with f16 output (1,238,630,400 - 353,894,400 B)

Each round times every arm once, in turn (CUDA events around --iters launches after --warmup); --rounds rounds.  The
probes a-d are compiled from tools/point_ceiling.cu with nvcc into a temporary directory.  Writes one JSON line to
DIR/point_ceiling.jsonl (and stdout), with the card's name, power limit and max SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

from benchkit import ROOT, start, write_line

PERIOD, FIRST = 3, 1          # the headline's tapped rows and columns: 3d + 1


def build_probes(tmp: str) -> C.CDLL:
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(tmp, "point_ceiling.so")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
           os.path.join(ROOT, "tools", "point_ceiling.cu"), "-o", so]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    subprocess.run(cmd, check=True)
    lib = C.CDLL(so)
    u32, vp = C.c_uint32, C.c_void_p
    lib.probe_read.argtypes = [vp, vp, u32, u32, u32, u32, u32, u32, vp]
    lib.probe_write.argtypes = [vp, u32, u32, u32, vp]
    lib.probe_twin.argtypes = [vp, vp, u32, u32, u32, u32, u32, u32, u32, vp]
    lib.probe_memcpy.argtypes = [vp, vp, C.c_size_t, vp]
    return lib


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="directory for point_ceiling.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--half", action="store_true", help="also time the tiled and full-row launches with f16 output")
    args = ap.parse_args()
    if args.iters < 20 or args.rounds < 3:
        ap.error("--iters >= 20 and --rounds >= 3: fewer cannot show the spread")

    import torch

    import kornia_rs_b200 as kb

    bench, facts = start("point_ceiling")
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev)
    sp = C.c_void_p(st.cuda_stream)
    tmp = tempfile.mkdtemp(prefix="point_ceiling_")
    lib = build_probes(tmp)

    SW, SH, DW, DH, N = bench.SW, bench.SH, bench.DW, bench.DH, bench.BATCH
    assert SH == PERIOD * DH and SW == PERIOD * DW
    row_bytes = SW * 3
    src = torch.empty((N, SH, SW, 3), dtype=torch.uint8, device=dev)
    gen = bench.LcgPattern(SW * SH * 3, dev)
    for i in range(N):
        gen.frame(0x12345678 + i, src[i].view(-1))   # bench.py's headline frames
    del gen
    dst = torch.empty((N, 3, DH, DW), dtype=torch.float32, device=dev)
    dst16 = torch.empty((N, 3, DH, DW), dtype=torch.float16, device=dev) if args.half else None
    sink = torch.zeros(1, dtype=torch.int32, device=dev)
    p = kb.imgproc.NormalizeParams.from_mean_std(bench.IMAGENET_MEAN, bench.IMAGENET_STD)
    op = kb.imgproc.resize_normalize_to_tensor_u8_bilinear

    read_b = N * DH * row_bytes
    write_b = N * 3 * DW * DH * 4
    both = read_b + write_b
    copy_b = both // 2

    def check(rc):
        if rc != 0:
            raise RuntimeError(f"probe launch failed: CUDA error {rc}")

    def fused(dtype, out):
        return lambda: op(src, DW, DH, p.scale, p.bias, dtype, out=out)

    def with_knobs(fn, values):
        """Runs fn (a whole timed window) with the developer knobs set, then resets them to 0 (the dispatcher's choice)."""
        for k, v in values.items():
            kb._lib.set_knob(k, v)
        try:
            return fn()
        finally:
            for k in values:
                kb._lib.set_knob(k, 0)

    # name -> (launch, bytes moved, knobs)
    arms = {
        "a_read": (lambda: check(lib.probe_read(src.data_ptr(), sink.data_ptr(), N, SH, row_bytes, DH, PERIOD, FIRST, sp)), read_b, {}),
        "b_write": (lambda: check(lib.probe_write(dst.data_ptr(), N, DW, DH, sp)), write_b, {}),
        "c_twin": (lambda: check(lib.probe_twin(src.data_ptr(), dst.data_ptr(), N, SH, row_bytes, DW, DH, PERIOD, FIRST, sp)), both, {}),
        "d_memcpy": (lambda: check(lib.probe_memcpy(dst.data_ptr(), src.data_ptr(), copy_b, sp)), 2 * copy_b, {}),
        "e_tiled": (fused(torch.float32, dst), both, {"fr.rows": 1}),
        "f_rows": (fused(torch.float32, dst), both, {"fr.rows": 2}),
    }
    if args.half:
        half_b = read_b + write_b // 2
        arms["e_tiled_f16"] = (fused(torch.float16, dst16), half_b, {"fr.rows": 1})
        arms["f_rows_f16"] = (fused(torch.float16, dst16), half_b, {"fr.rows": 2})

    # correctness of what is timed: the twin writes (float)byte of the point taps; both schedules give the same bits
    check(lib.probe_twin(src.data_ptr(), dst.data_ptr(), N, SH, row_bytes, DW, DH, PERIOD, FIRST, sp))
    twin_ok = bool(torch.equal(dst[0], src[0, FIRST::PERIOD, FIRST::PERIOD, :].permute(2, 0, 1).float()))
    outs = {}
    for name in [k for k in arms if k.startswith(("e_", "f_"))]:
        with_knobs(arms[name][0], arms[name][2])
        outs[name] = (dst16 if name.endswith("f16") else dst).clone()
    same = {k: bool(torch.equal(v.view(torch.int16 if v.dtype == torch.float16 else torch.int32),
                                outs["e_tiled_f16" if k.endswith("f16") else "e_tiled"].view(torch.int16 if v.dtype == torch.float16 else torch.int32)))
            for k, v in outs.items() if k.startswith("f_")}
    del outs
    torch.cuda.synchronize()

    times = {k: [] for k in arms}
    for r in range(args.rounds):
        for k, (fn, _, kn) in arms.items():
            times[k].append(with_knobs(lambda: bench.time_launches(fn, args.iters, args.warmup, st), kn))
        print(f"[point_ceiling] round {r}: " + "  ".join(f"{k} {times[k][-1]:.4f}" for k in arms), file=sys.stderr, flush=True)
    shutil.rmtree(tmp, ignore_errors=True)

    res = {}
    for k, (_, nbytes, _) in arms.items():
        t = times[k]
        mean = statistics.fmean(t)
        res[k] = {"ms": [round(x, 4) for x in t], "ms_mean": round(mean, 4), "spread": round((max(t) - min(t)) / mean, 4),
                  "bytes": nbytes, "tbs": round(nbytes / (mean * 1e-3) / 1e12, 3)}
    ratio = {k: round(res["c_twin"]["ms_mean"] / res[k]["ms_mean"], 4) for k in res if k.startswith(("e_", "f_")) and not k.endswith("f16")}
    line = {"tool": "tools/point_ceiling.py", "gpu": facts, "date": time.strftime("%Y-%m-%d"), "iters": args.iters, "warmup": args.warmup,
            "rounds": args.rounds, "shape": {"src": [N, SH, SW, 3], "dst": [N, 3, DH, DW]}, "arms": res,
            "twin_ms_over_arm_ms": ratio,
            "twin_faster_than_tiled": round(1.0 - res["c_twin"]["ms_mean"] / res["e_tiled"]["ms_mean"], 4),
            "rows_faster_than_tiled": round(1.0 - res["f_rows"]["ms_mean"] / res["e_tiled"]["ms_mean"], 4),
            "twin_output_ok": twin_ok, "rows_bits_equal_tiled": same}
    write_line(args.out, "point_ceiling", line)


if __name__ == "__main__":
    main()
