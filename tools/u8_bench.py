"""u8 twins quick timing (GPU box): python tools/u8_bench.py — word-granular sampler on/off (knob b=1 disables)."""
from benchkit import PEAK_GBS, bench_module
import torch
import kornia_rs_b200 as kb
dev = torch.device("cuda:0"); st = torch.cuda.current_stream(dev)
time_launches = bench_module().time_launches
w, h, n = 3840, 2160, 16
g = torch.Generator(device=dev).manual_seed(1)
s8 = kb.Image(torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=dev, generator=g))
d8 = kb.Image.zeros_cuda(kb.ImageSize(w, h), 3, torch.uint8, dev, batch=n)
H = [1.02, 0.03, -40.0, -0.03, 1.01, 25.0, 2.0e-6, 1.2e-6, 1.0]
M = kb.imgproc.get_rotation_matrix2d((w / 2, h / 2), 30.0, 1.0)
yy, xx = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32), torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
r2 = ((xx - w / 2) ** 2 + (yy - h / 2) ** 2) / float(w * w)
mx = kb.Image((w / 2 + (xx - w / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous()); my = kb.Image((h / 2 + (yy - h / 2) * (1 + 0.05 * r2)).unsqueeze(-1).contiguous())
ops = {"warp_perspective_u8": lambda: kb.imgproc.warp_perspective_u8(s8, d8, H), "warp_affine_u8_rot30": lambda: kb.imgproc.warp_affine_u8(s8, d8, M),
       "remap_u8": lambda: kb.imgproc.remap_u8(s8, d8, mx, my, kb.InterpolationMode.Bilinear), "gaussian_blur_u8": lambda: kb.imgproc.gaussian_blur_u8(s8, d8, (5, 5), (1.5, 1.5))}
for b in (1, 0):
    kb._lib.set_knob("b", b)
    for name, fn in ops.items():
        ms = time_launches(fn, 10, 3, st)
        print(f"words={'off' if b else 'on '} {name:24s} {ms:.4f} ms  {n*w*h/ms/1e6:.0f} Gpix/s  frac {n*w*h*6/ms/1e6/PEAK_GBS:.3f}", flush=True)
