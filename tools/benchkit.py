"""What the benchmarks under tools/ share: the card's facts, bench.py's timer, the two timing procedures, result rows,
the command line and the JSON-line writer, and the byte counts of the camera preprocess's region benchmarks.

Every tool takes shared code from here, tests/restate.py, tests/harness.py, the oracle and the library, never from
another tool, so changing one benchmark cannot change another's results.  Importing this module puts the repository
root and tests/ on sys.path.
"""
from __future__ import annotations

import argparse
import ctypes as C
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

PEAK_GBS = 3350.0   # H100 SXM data sheet HBM3


def gpu_facts() -> dict:
    """The card's name, power limit and max SM clock, read now."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def bench_module():
    """bench.py, loaded by path: its time_launches, its headline shapes and frames."""
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def arg_parser(doc: str, name: str) -> argparse.ArgumentParser:
    """The command line every DIR-writing benchmark takes: --out DIR, --iters, --warmup, --reps.  A tool adds its own
    flags to it, then calls parse_args."""
    ap = argparse.ArgumentParser(description=doc.split("\n\n")[0])
    ap.add_argument("--out", required=True, help=f"directory for {name}.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    return ap


def parse_args(ap: argparse.ArgumentParser):
    args = ap.parse_args()
    if args.iters < 20 or args.reps < 3:
        ap.error("--iters >= 20 and --reps >= 3: fewer cannot show the spread")
    return args


def start(name: str):
    """Refuses to run without a CUDA device; returns (bench.py as a module, the card's facts)."""
    import torch

    if not torch.cuda.is_available():
        raise SystemExit(f"{name}.py needs a CUDA device")
    return bench_module(), gpu_facts()


def append_lines(path: str, lines: list) -> None:
    """Appends one JSON line per dict in `lines` to the file `path`."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "a") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


def write_line(out_dir: str, name: str, line: dict) -> None:
    """Appends `line` to out_dir/<name>.jsonl and prints it."""
    append_lines(os.path.join(out_dir, f"{name}.jsonl"), [line])
    print(json.dumps(line))


def time_arms(bench, fns, iters, warmup, reps, stream, kb, probe=None):
    """{arm: fn}, the arms alternating, the set repeated `reps` times; each arm's turn is bench.time_launches (`warmup`
    calls, a synchronise, CUDA events around `iters` calls, a synchronise).  Returns ({arm: [ms per call, one per rep]},
    {arm: probe(arm) after its last turn}); the default probe is the kernel the arm's last call launched."""
    times = {k: [] for k in fns}
    probed = {}
    for _ in range(reps):
        for k, fn in fns.items():
            times[k].append(bench.time_launches(fn, iters, warmup, stream))
            probed[k] = probe(k) if probe else kb._lib.last_kernel()
    return times, probed


def time_alternating(arms, iters, repeats):
    """{arm: fn}: two warm-up calls per arm, then `repeats` rounds of `iters` calls per arm in turn, CUDA events on the
    current stream; {arm: (min, max)} of the ms per call over the rounds."""
    import torch

    for fn in arms.values():
        fn(); fn()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(repeats):
        for k, fn in arms.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            res[k].append(s.elapsed_time(e) / iters)
    return {k: (min(v), max(v)) for k, v in res.items()}


def row(times, kernels, alg_bytes, checks, check_key):
    """One result per arm from time_arms' output: the times, their minimum, the algorithmic bytes and the rate they give
    at that minimum, the kernel, and the outcome of the arm's output check under `check_key`."""
    r = {}
    for k in times:
        best = min(times[k])
        gbs = alg_bytes[k] / (best * 1e-3) / 1e9
        r[k] = {"ms": [round(t, 4) for t in times[k]], "ms_min": round(best, 4), "alg_bytes": alg_bytes[k], "gbs": round(gbs, 1),
                "frac_of_3350": round(gbs / PEAK_GBS, 3), "kernel": kernels[k], check_key: checks[k]}
    return r


def e2e_result(steps, transfer, matches=None, pixels=None):
    """One host-pipeline arm: its ms per step (one per rep) and their minimum, the bytes the last step moved each way
    (HostPipeline.last_transfer()) and their rates at that minimum, Gpix/s when `pixels` (per step) is given, and
    whether the host result matched the device run when `matches` is given."""
    best = min(steps)
    up, down = transfer
    r = {"ms_per_step": [round(t, 3) for t in steps], "ms_min": round(best, 3), "h2d_bytes": up, "d2h_bytes": down,
         "h2d_gbs": round(up / (best * 1e-3) / 1e9, 1), "d2h_gbs": round(down / (best * 1e-3) / 1e9, 1)}
    if pixels is not None:
        r["gpix_s"] = round(pixels / (best * 1e-3) / 1e9, 3)
    if matches is not None:
        r["matches_device_result"] = matches
    return r


def words(t, shift):
    """Samples as 16-bit words, each shifted left by `shift` bits: a P01x / I41xMsb code in the high bits, an I01x / I41x
    code in the low ones."""
    import torch

    return (t.to(torch.int32) << shift).to(torch.uint16)


# ── the region benchmarks (preprocess_roi / _warp / _remap_bench) ──

OUT_CODES = {"f32": 0, "bf16": 2}
FORMATS = {"NV12": (3, 1), "P010": (80, 2), "RGGB": (16, 1), "RGGB12": (36, 2)}   # format code, bytes per sample


def frame_len(fmt, w, h):
    """Bytes of one tight w x h frame: a 4:2:0 frame's 1.5 samples per pixel, a Bayer mosaic's one."""
    bps = FORMATS[fmt][1]
    return w * h * bps if fmt.startswith("RGGB") else w * h * 3 // 2 * bps


def stream():
    """The current CUDA stream's handle, for the library's C entries."""
    import torch

    return torch.cuda.current_stream().cuda_stream


def preprocess_desc(code, sample_bytes, w, h, dw, dh, affine=(1.0, 1.0, 0.0, 0.0), bpp=1):
    """kb200_preprocess_desc: a w x h source of format `code` with rows of w * sample_bytes bytes (`bpp`: bytes per pixel
    of an RGB source) to dw x dh through `affine` (scale_x, scale_y, pad_x, pad_y), ImageNet normalisation, pad 114,
    bilinear."""
    import kornia_rs_b200 as kb
    from kornia_rs_b200._lib import PreprocessDesc

    inv_std = tuple(float(np.float32(1) / np.float32(s)) for s in kb.IMAGENET_STD)
    d = PreprocessDesc()
    d.scale_x, d.scale_y, d.pad_x, d.pad_y = affine
    d.src_w, d.src_h, d.src_pitch, d.src_bpp, d.fmt = w, h, w * sample_bytes, bpp, code
    d.dst_w, d.dst_h = dw, dh
    d.mean, d.inv_std = (C.c_float * 3)(*kb.IMAGENET_MEAN), (C.c_float * 3)(*inv_std)
    d.pad_value, d.sampling = 114.0, 1
    return d


def tap_mask(sx, sy, w, h, m=None):
    """Marks in the h x w mask `m` (a new one when None) the pixels the bilinear sampler taps at the in-frame float32
    coordinates (sx, sy): (x0, y0) = floor, and x0 + 1 / y0 + 1 (clamped to the frame) only where its weight is not zero."""
    if m is None:
        m = np.zeros((h, w), bool)
    x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
    nx, ny = sx != x0, sy != y0
    x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
    m[y0, x0] = True
    m[y0[nx], x1[nx]] = True
    m[y1[ny], x0[ny]] = True
    m[y1[nx & ny], x1[nx & ny]] = True
    return m


def mask_bytes(fmt, m):
    """Distinct source bytes of one frame behind its tapped pixels `m`: per tapped Bayer pixel its 3 x 3 demosaic
    neighbourhood, per tapped luma pixel of a 4:2:0 frame the chroma pair it decodes with; at the format's bytes per
    sample."""
    h, w = m.shape
    bps = FORMATS[fmt][1]
    if fmt.startswith("RGGB"):
        p = np.pad(m, 1)
        m = np.zeros_like(m)
        for dy in range(3):
            for dx in range(3):
                m |= p[dy:dy + h, dx:dx + w]
        return int(m.sum()) * bps
    ys, xs = np.nonzero(m)
    chroma = np.zeros((h // 2, w // 2), bool)
    chroma[ys >> 1, xs >> 1] = True
    return (int(m.sum()) + 2 * int(chroma.sum())) * bps
