"""A/B timings on the GPU box: python tools/ab_bench.py — the lean bilinear warp against the round-2 x4 kernel (knob a),
the u8 blur's row-streaming kernel against the tile kernel (knob b = 3) with its CTA / chunk knobs (c, d)."""
import sys
from benchkit import PEAK_GBS, bench_module
import torch
import kornia_rs_b200 as kb
dev = torch.device("cuda:0"); st = torch.cuda.current_stream(dev)
time_launches = bench_module().time_launches
def timeit(fn): return time_launches(fn, 10, 3, st)
w, h, n = 3840, 2160, 16
g = torch.Generator(device=dev).manual_seed(1)
what = sys.argv[1:] or ["warp", "u8", "blur"]
if "warp" in what:
    s = kb.Image(torch.rand((n, h, w, 3), dtype=torch.float32, device=dev, generator=g))
    d_ = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.float32, dev, batch=n)
    H = [1.02, 0.03, -40.0, -0.03, 1.01, 25.0, 2.0e-6, 1.2e-6, 1.0]
    M = kb.imgproc.get_rotation_matrix2d((w / 2, h / 2), 3.0, 1.0)
    # a: 0 lean + TMA tile stores, 5 lean + STG, 3 round-2 x4
    for a, pf in ((0, 0), (7, 0), (0, -1), (5, 0), (3, 0)):     # 0: one 4-D tensor-map store per warp, 7: four 1-D row copies per warp
        kb._lib.set_knob("a", a); kb._lib.set_knob("warp.pf", pf)
        ms = timeit(lambda: kb.imgproc.warp_perspective(s, d_, H, kb.InterpolationMode.Bilinear))
        print(f"warp_perspective a={a} pf={pf} {kb._lib.last_kernel():36s} {ms:.4f} ms frac {n*w*h*24/ms/1e6/PEAK_GBS:.3f}", flush=True)
        ms = timeit(lambda: kb.imgproc.warp_affine(s, d_, M, kb.InterpolationMode.Bilinear))
        print(f"warp_affine rot3 a={a} pf={pf} {kb._lib.last_kernel():36s} {ms:.4f} ms frac {n*w*h*24/ms/1e6/PEAK_GBS:.3f}", flush=True)
    kb._lib.set_knob("a", 0); kb._lib.set_knob("warp.pf", 0)
    for ang in (30.0, 45.0, 10.0):
        M30 = kb.imgproc.get_rotation_matrix2d((w / 2, h / 2), ang, 1.0)
        for c in (0,):
            kb._lib.set_knob("c", c)
            ms = timeit(lambda: kb.imgproc.warp_affine(s, d_, M30, kb.InterpolationMode.Bilinear))
            print(f"warp_affine rot{ang:g} box={c} {kb._lib.last_kernel():36s} {ms:.4f} ms frac {n*w*h*24/ms/1e6/PEAK_GBS:.3f}", flush=True)
        kb._lib.set_knob("c", 0)
    yy, xx = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32), torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
    r2 = ((xx - w / 2) ** 2 + (yy - h / 2) ** 2) / float(w * w)
    mx = kb.Image((w / 2 + (xx - w / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous()); my = kb.Image((h / 2 + (yy - h / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous())
    for a, pf in ((0, 0), (7, 0), (5, 0), (6, 0)):       # lean + tensor-map / 1-D TMA tile stores, lean + STG, thread-per-pixel kernel
        kb._lib.set_knob("a", a); kb._lib.set_knob("warp.pf", pf)
        ms = timeit(lambda: kb.imgproc.remap(s, d_, mx, my, kb.InterpolationMode.Bilinear))
        print(f"remap_f32 a={a} pf={pf} {kb._lib.last_kernel():28s} {ms:.4f} ms frac {n*w*h*24.5/ms/1e6/PEAK_GBS:.3f}", flush=True)
    kb._lib.set_knob("a", 0); kb._lib.set_knob("warp.pf", 0)
    del s, d_
if "u8" in what:
    s8 = kb.Image(torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=dev, generator=g))
    d8 = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n)
    H = [1.02, 0.03, -40.0, -0.03, 1.01, 25.0, 2.0e-6, 1.2e-6, 1.0]
    M = kb.imgproc.get_rotation_matrix2d((w / 2, h / 2), 30.0, 1.0)
    yy, xx = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32), torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
    r2 = ((xx - w / 2) ** 2 + (yy - h / 2) ** 2) / float(w * w)
    mx = kb.Image((w / 2 + (xx - w / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous()); my = kb.Image((h / 2 + (yy - h / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous())
    ops = {"warp_perspective_u8": lambda: kb.imgproc.warp_perspective_u8(s8, d8, H), "warp_affine_u8_rot30": lambda: kb.imgproc.warp_affine_u8(s8, d8, M),
           "remap_u8": lambda: kb.imgproc.remap_u8(s8, d8, mx, my, kb.InterpolationMode.Bilinear)}
    for b in (0, 1):          # 0: interior fast path (word taps), 1: the clamped byte sampler everywhere (round-1 form)
        kb._lib.set_knob("b", b)
        for name, fn in ops.items():
            ms = timeit(fn)
            print(f"{name:24s} b={b} {kb._lib.last_kernel():32s} {ms:.4f} ms frac {n*w*h*6/ms/1e6/PEAK_GBS:.3f}", flush=True)
    kb._lib.set_knob("b", 0)
    M3 = kb.imgproc.get_rotation_matrix2d((w / 2, h / 2), 3.0, 1.0)
    ops2 = dict(ops); ops2["warp_affine_u8_rot3"] = lambda: kb.imgproc.warp_affine_u8(s8, d8, M3); del ops2["remap_u8"]
    for c in (8, 16, 32, 64, 128):      # 32-pixel segments of a row per warp
        kb._lib.set_knob("c", c)
        for name, fn in ops2.items():
            ms = timeit(fn)
            print(f"{name:24s} segs={c} {ms:.4f} ms frac {n*w*h*6/ms/1e6/PEAK_GBS:.3f}", flush=True)
    kb._lib.set_knob("c", 0)
    del s8, d8
if "blur" in what:
    s8 = kb.Image(torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=dev, generator=g))
    d8 = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n)
    for b, c, dd in ((3, 0, 0), (0, 0, 0), (0, 2, 0), (0, 3, 0), (0, 4, 0), (0, 6, 0), (0, 4, 64), (0, 4, 128), (0, 8, 128)):
        kb._lib.set_knob("b", b); kb._lib.set_knob("c", c); kb._lib.set_knob("d", dd)
        ms = timeit(lambda: kb.imgproc.gaussian_blur_u8(s8, d8, (5, 5), (1.5, 1.5)))
        print(f"gaussian_blur_u8 b={b} c={c} d={dd} {kb._lib.last_kernel():28s} {ms:.4f} ms frac {n*w*h*6/ms/1e6/PEAK_GBS:.3f}", flush=True)
    for k in "bcd": kb._lib.set_knob(k, 0)
