"""Knob sweeps on the GPU box: python tools/sweep.py <what> — prints one line per configuration (ms, GB/s, frac of peak).

  warp      config 5 (4K f32 warp_perspective, 16 images) through the row-streaming kernel: ws.npx x ws.stages x ws.ctas x ws.rc
  resize    f32 resize 4K -> 720p / 1080p / 1600x900 through resize_rows: rs.npx x rs.stages x rs.ctas
  fused     fused u8 resize, general mode 4K -> 1600x900: fr.npx x fr.stages x fr.ctas
"""
import itertools
import json
import os
import sys

from benchkit import PEAK_GBS, ROOT, bench_module
import torch

import kornia_rs_b200 as kb

PEAK = PEAK_GBS
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass
dev = torch.device("cuda:0")
st = torch.cuda.current_stream(dev)
time_launches = bench_module().time_launches


def timeit(fn):
    return time_launches(fn, 10, 3, st)


def setk(**kw):
    for k, v in kw.items():
        kb._lib.set_knob(k.replace("_", "."), v)


what = sys.argv[1]
g = torch.Generator(device=dev).manual_seed(3)
w, h = 3840, 2160
if what == "warp":
    n = 16
    src = kb.Image(torch.rand((n, h, w, 3), dtype=torch.float32, device=dev, generator=g))
    dst = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.float32, dev, batch=n)
    H = [1.02, 0.03, -40.0, -0.03, 1.01, 25.0, 2.0e-6, 1.2e-6, 1.0]
    fn = lambda: kb.imgproc.warp_perspective(src, dst, H, kb.InterpolationMode.Bilinear)
    alg = n * w * h * 24
    setk(warp_path=1)
    for a in (1, 0):      # a = 1: two __fdiv_rn; a = 0: shared reciprocal
        for pf in (0, 96, -1):
            setk(a=a, warp_pf=pf)
            ms = timeit(fn)
            print(f"gather pf_all={a} pf={pf:3d} {kb._lib.last_kernel():28s} {ms:.4f} ms  frac {alg / ms / 1e6 / PEAK:.3f}", flush=True)
    setk(a=0, warp_pf=0)
    if len(sys.argv) > 2 and sys.argv[2] == "gather":
        sys.exit(0)
    setk(warp_path=3)
    for npx, stages, ctas, rc in itertools.product((1,), (0, 8, 32), (3, 4, 6, 8), (0, 136, 540)):
        setk(ws_npx=npx, ws_stages=stages, ws_ctas=ctas, ws_rc=rc)
        try:
            ms = timeit(fn)
            print(f"npx={npx} stages={stages:2d} ctas={ctas} rc={rc:3d} {kb._lib.last_kernel():22s} {ms:.4f} ms  frac {alg / ms / 1e6 / PEAK:.3f}", flush=True)
        except Exception as ex:
            print(f"npx={npx} stages={stages} ctas={ctas} rc={rc}: {ex}")
elif what == "resize":
    n = 16
    src = kb.Image(torch.rand((n, h, w, 3), dtype=torch.float32, device=dev, generator=g))
    for dw, dh, tapped in ((1280, 720, 2560 * 1440), (1920, 1080, w * h), (1600, 900, None)):
        dst = kb.Image.zeros_cuda(kb.ImageSize(dw, dh), 3, torch.float32, dev, batch=n)
        fn = lambda: kb.imgproc.resize(src, dst, kb.InterpolationMode.Bilinear)
        tp = tapped if tapped else int(w * h * 0.98)
        alg = n * (tp * 12 + dw * dh * 12)
        for npx, stages, ctas in itertools.product((1, 2, 3), (0, 2, 4, 6), (0, 2, 3, 4, 6, 8)):
            setk(rs_npx=npx, rs_stages=stages, rs_ctas=ctas)
            ms = timeit(fn)
            print(f"{dw}x{dh} npx={npx} stages={stages} ctas={ctas} {kb._lib.last_kernel():24s} {ms:.4f} ms  frac~{alg / ms / 1e6 / PEAK:.3f}", flush=True)
elif what == "fused":
    n = 16
    src = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=dev, generator=g)
    p = kb.imgproc.NormalizeParams.from_mean_std(kb.IMAGENET_MEAN, kb.IMAGENET_STD)
    for dw, dh in ((1600, 900), (1920, 1080), (1280, 720)):
        dst = torch.empty((n, 3, dh, dw), dtype=torch.float32, device=dev)
        fn = lambda: kb.imgproc.resize_normalize_to_tensor_u8_to_f32_bilinear(src, dw, dh, p.scale, p.bias, out=dst)
        for npx, stages, ctas in itertools.product((0, 1, 2, 3, 4), (0, 3, 4, 6), (0, 2, 4, 6, 8)):
            setk(fr_npx=npx, fr_stages=stages, fr_ctas=ctas)
            ms = timeit(fn)
            print(f"{dw}x{dh} npx={npx} stages={stages} ctas={ctas} {kb._lib.last_kernel():24s} {ms:.4f} ms  {n * dw * dh / ms / 1e3:.0f} Mpix/s", flush=True)
