"""GPU baseline: the reference's OWN CUDA kernels, run the way the reference runs them, on the same GPU.

`baseline/extract_ref_kernels.py` (run at build time when $KORNIA_RS_SRC names a kornia-rs checkout) extracted every NVRTC translation
unit of the §8 path verbatim and compiled it with the reference's NVRTC options (`compute_90`, `--fmad=false`,
crates/kornia-tensor/src/cuda.rs:675-718) into `baseline/_ref/ptx/`.  This module loads that PTX through the CUDA
driver API — the reference's own path: NVRTC PTX -> cuModuleLoadData -> cuLaunchKernel (cudarc) — and launches each
kernel with the reference's launch geometry:

  * 2-D image kernels: 32x8 blocks, grid = ceil(w/32) x ceil(h/8)             (cuda/mod.rs:73-90 make_config)
  * 1-D map kernels:   256-thread blocks, grid = ceil(n/256)                  (kornia-tensor/src/cuda.rs:794-802)
  * ONE launch per image / per frame: the reference has no batch dimension on this path
    (preprocess.rs:1277-1280 run_raw_batch loops over frames; the imgproc launchers take one image)
  * separable filters: H pass into a scratch image, V pass into dst (cuda/filter.rs:361-385);
    sobel = 2 separable filters + magnitude = 5 launches (filter/cuda.rs:185-232)
  * L1-preferred cache config, best effort (try_compile_with_l1 / prefer_l1_cache)

Measurement and cross-check infrastructure only (bench.py's `vs_ref_gpu` column, tests/test_ref_gpu_kernels.py): the
product library never sees this file.  Nothing here reads the reference's sources at run time.
"""
from __future__ import annotations

import ctypes as C
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
REFDIR = os.path.join(HERE, "_ref")


def available() -> bool:
    return os.path.exists(os.path.join(REFDIR, "manifest.json"))


class RefGpu:
    def __init__(self, device_index: int = 0):
        import torch
        from cuda.bindings import driver

        self.drv = driver
        self.torch = torch
        self.dev = torch.device("cuda", device_index)
        torch.zeros(1, device=self.dev)   # make torch create / retain the primary context
        self._ck(driver.cuInit(0))
        cudev = self._ck(driver.cuDeviceGet(device_index))
        self.ctx = self._ck(driver.cuDevicePrimaryCtxRetain(cudev))
        self._ck(driver.cuCtxSetCurrent(self.ctx))
        self.manifest = json.load(open(os.path.join(REFDIR, "manifest.json")))["units"]
        self._unit_of = {k: u for u, m in self.manifest.items() for k in m["kernels"]}
        self._mods, self._funcs = {}, {}
        self._taps = {}

    def _ck(self, r):
        if int(r[0]) != 0:
            raise RuntimeError(f"CUDA driver error {r[0]}")
        return r[1] if len(r) == 2 else (r[1:] if len(r) > 2 else None)

    def func(self, kernel: str):
        if kernel not in self._funcs:
            unit = self._unit_of[kernel]
            if unit not in self._mods:
                ptx = open(os.path.join(REFDIR, "ptx", unit + ".ptx"), "rb").read().rstrip(b" \0") + b"\0"
                self._ck(self.drv.cuCtxSetCurrent(self.ctx))
                self._mods[unit] = self._ck(self.drv.cuModuleLoadData(ptx))
            f = self._ck(self.drv.cuModuleGetFunction(self._mods[unit], kernel.encode()))
            try:
                self.drv.cuFuncSetCacheConfig(f, self.drv.CUfunc_cache.CU_FUNC_CACHE_PREFER_L1)
            except Exception:
                pass
            self._funcs[kernel] = f
        return self._funcs[kernel]

    def launch(self, kernel: str, grid, block, args) -> None:
        """args: list of ctypes values (c_void_p for device pointers)."""
        ptrs = (C.c_void_p * len(args))(*[C.cast(C.pointer(a), C.c_void_p) for a in args])
        stream = self.torch.cuda.current_stream(self.dev).cuda_stream
        r = self.drv.cuLaunchKernel(self.func(kernel), grid[0], grid[1], 1, block[0], block[1], 1, 0, stream, C.addressof(ptrs), 0)
        if int(r[0]) != 0:
            raise RuntimeError(f"cuLaunchKernel({kernel}) failed: {r[0]}")

    # launch geometry of the reference
    @staticmethod
    def cfg2d(w: int, h: int):
        bw, bh = min(32, w), min(8, h)                                   # cuda/mod.rs:78-90
        return ((w + bw - 1) // bw, (h + bh - 1) // bh), (bw, bh)

    @staticmethod
    def cfg1d(n: int):
        return ((n + 255) // 256, 1), (256, 1)

    @staticmethod
    def _p(t):
        return C.c_void_p(t.data_ptr())

    @staticmethod
    def _coeffs(src_len: int, dst_len: int):
        """PixelMapping::HalfPixel.coeffs (cuda/resize.rs:462-478) in f32."""
        import numpy as np

        a = np.float32(src_len) / np.float32(dst_len)
        return float(a), float(np.float32(0.5) * a - np.float32(0.5))

    # ── ops: one call = what the reference's adapter enqueues for the whole batch ────────────────
    def resize_bilinear(self, src, dst, kernel="resize_bilinear_downscale_3c"):
        n, sh, sw, _ = src.shape
        _, dh, dw, _ = dst.shape
        ax, bx = self._coeffs(sw, dw)
        ay, by = self._coeffs(sh, dh)
        grid, block = self.cfg2d(dw, dh)
        for i in range(n):
            self.launch(kernel, grid, block, [self._p(src[i]), self._p(dst[i]), C.c_uint(sw), C.c_uint(sh), C.c_uint(dw), C.c_uint(dh),
                                              C.c_float(ax), C.c_float(bx), C.c_float(ay), C.c_float(by)])

    def resize_lanczos(self, src, dst, inter, x0s, wx, y0s, wy):
        """cuda/resize.rs:823-905 — host-built per-axis tables (lanczos_axis) uploaded by the caller, H pass into the
        dst_w x src_h intermediate, then V pass; per image."""
        n, sh, sw, _ = src.shape
        _, dh, dw, _ = dst.shape
        gh, bh = self.cfg2d(dw, sh)
        gv, bv = self.cfg2d(dw, dh)
        for i in range(n):
            self.launch("resize_lanczos_h_3c", gh, bh, [self._p(src[i]), self._p(inter), self._p(x0s), self._p(wx), C.c_uint(sw), C.c_uint(sh), C.c_uint(dw)])
            self.launch("resize_lanczos_v_3c", gv, bv, [self._p(inter), self._p(dst[i]), self._p(y0s), self._p(wy), C.c_uint(dw), C.c_uint(sh), C.c_uint(dh)])

    def warp(self, kind: str, interp: str, src, dst, minv):
        """kind 'affine' (6 inverse coefficients) or 'perspective' (9); interp bilinear|nearest|bicubic|lanczos."""
        n, sh, sw, _ = src.shape
        _, dh, dw, _ = dst.shape
        grid, block = self.cfg2d(dw, dh)
        for i in range(n):
            self.launch(f"warp_{kind}_{interp}_3c", grid, block,
                        [self._p(src[i]), self._p(dst[i]), C.c_uint(sw), C.c_uint(sh), C.c_uint(dw), C.c_uint(dh)] + [C.c_float(float(v)) for v in minv])

    def taps(self, k):
        key = tuple(float(v) for v in k)
        if key not in self._taps:
            self._taps[key] = self.torch.tensor(key, dtype=self.torch.float32, device=self.dev)
        return self._taps[key]

    def separable_filter(self, src, dst, scratch, kx, ky):
        """cuda/filter.rs:361-385 — H pass into scratch, V pass into dst, per image."""
        n, rows, cols, c = src.shape
        tx, ty = self.taps(kx), self.taps(ky)
        grid, block = self.cfg2d(cols, rows)
        for i in range(n):
            self.launch(f"sep_filter_f32_h_c{c}_k{len(kx)}", grid, block, [self._p(src[i]), self._p(scratch), self._p(tx), C.c_uint(len(kx)), C.c_uint(cols), C.c_uint(rows)])
            self.launch(f"sep_filter_f32_v_c{c}_k{len(ky)}", grid, block, [self._p(scratch), self._p(dst[i]), self._p(ty), C.c_uint(len(ky)), C.c_uint(cols), C.c_uint(rows)])

    def sobel(self, src, dst, scratch, gx, gy, ksize=3):
        """filter/cuda.rs:185-232 — gx = sep(d, s), gy = sep(s, d), magnitude: 5 launches per image."""
        d, s = ((-1.0, 0.0, 1.0), (1.0, 2.0, 1.0)) if ksize == 3 else ((-1.0, -2.0, 0.0, 2.0, 1.0), (1.0, 4.0, 6.0, 4.0, 1.0))
        n, rows, cols, c = src.shape
        cnt = rows * cols * c
        for i in range(n):
            self.separable_filter(src[i:i + 1], gx, scratch, d, s)
            self.separable_filter(src[i:i + 1], gy, scratch, s, d)
            grid, block = self.cfg1d(cnt)
            self.launch("gradient_magnitude_f32", grid, block, [self._p(gx), self._p(gy), self._p(dst[i]), C.c_uint(cnt)])

    def gray_f32(self, src, dst):
        n = src.shape[0]
        npx = src.shape[1] * src.shape[2]
        grid, block = self.cfg1d(npx)
        for i in range(n):
            self.launch("gray_from_rgb_f32", grid, block, [self._p(src[i]), self._p(dst[i]), C.c_uint(npx)])

    def gray_u8(self, src, dst):
        n = src.shape[0]
        npx = src.shape[1] * src.shape[2]
        grid, block = self.cfg1d((npx + 3) // 4)                          # PxPerThread::Four
        for i in range(n):
            self.launch("gray_from_rgb_u8", grid, block, [self._p(src[i]), self._p(dst[i]), C.c_uint(npx)])

    def rgb_from_nv12(self, raw, dst, w, h):
        """cuda/color/video.rs:328-375 — thread per 2x2 block, NV12: u = plane+0, v = plane+1, step 2."""
        n = raw.shape[0]
        ylen = w * h
        grid, block = self.cfg2d(w // 2, h // 2)
        block = (32, 8)
        grid = ((w // 2 + 31) // 32, (h // 2 + 7) // 8)                   # config_2d: fixed 32x8
        for i in range(n):
            base = raw[i].data_ptr()
            self.launch("rgb_from_planar420_u8", grid, block, [C.c_void_p(base), C.c_void_p(base + ylen), C.c_void_p(base + ylen + 1), self._p(dst[i]),
                                                                C.c_uint(w), C.c_uint(w // 2), C.c_uint(h // 2), C.c_uint(2)])

    def preprocess(self, frames, sw, sh, dst, affine, mean, inv_std, pad_value=114.0, fmt=3, bpp=1, sampler="bilinear", f16=False):
        """preprocess.rs:1277-1372 — one launch per frame, 256-thread 1-D grid over dst pixels."""
        n, _, dh, dw = dst.shape
        name = f"resize_normalize_to_chw_{sampler}" + ("_f16" if f16 else "")
        grid, block = self.cfg1d(dw * dh)
        sx, sy, px, py = (float(v) for v in affine)
        pitch = sw * bpp
        for i in range(n):
            self.launch(name, grid, block, [self._p(frames[i]), self._p(dst[i]), C.c_float(sx), C.c_float(sy), C.c_float(px), C.c_float(py),
                                            C.c_int(sw), C.c_int(sh), C.c_int(pitch), C.c_int(bpp), C.c_int(fmt), C.c_int(dw), C.c_int(dh),
                                            C.c_float(mean[0]), C.c_float(mean[1]), C.c_float(mean[2]),
                                            C.c_float(inv_std[0]), C.c_float(inv_std[1]), C.c_float(inv_std[2]), C.c_float(pad_value)])

    def remap(self, src, dst, map_x, map_y, interp="bilinear"):
        n, sh, sw, _ = src.shape
        _, dh, dw, _ = dst.shape
        grid, block = self.cfg2d(dw, dh)
        for i in range(n):
            self.launch(f"remap_{interp}_3c", grid, block, [self._p(src[i]), self._p(map_x), self._p(map_y), self._p(dst[i]),
                                                            C.c_uint(sw), C.c_uint(sh), C.c_uint(dw), C.c_uint(dh)])
