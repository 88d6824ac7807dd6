"""kb200_preprocess_remap on an H100: lens undistortion of whole frames, undistortion fitted to a model input, and a camera
rig with one map per camera.  Appends one JSON line per workload, source format and output type to
results/h100_preprocess_remap_bench.jsonl (or --out).

  R1  256 NV12 1080p frames through one shared full-resolution undistortion map (kb200_generate_correction_map_polynomial)
      to 1920 x 1080, f32 and bf16.  Arms: `remap` (this entry); `existing` (today's path: kb200_rgb_from_nv12_u8, then
      kb200_remap_u8 of the RGB8 frames through the same map, then kb200_preprocess_strided_* to normalise them to CHW; its
      u8 remap uses Q10 arithmetic, so it is for timing only); `remap_region_major`, when --region-major-lib names a build
      of the library whose remap kernels take the region as the slowest-varying part of the block index (not a library
      option: a scratch build for this comparison only).  A second R1 row runs identity maps against the batch entry
      (kb200_preprocess_strided_* at scale 1, its identity kernel); the outputs must be identical.
  R2  64 NV12, P010 and 12-bit RGGB 1080p frames undistorted and fitted to 640 x 640 through one map from
      kb200_generate_correction_map_polynomial_to, f32 and bf16.
  R3  a rig of 6 cameras x 16 NV12 1080p frames, each camera with its own 640 x 384 map, f32: one call (96 regions,
      6 maps) against 6 shared-map calls (`per_map`).

Three regions of every output are checked in the same run against restate.remap_reference.
Arms alternate: 20 launches after warm-up, 3 repeats, minima given with the repeat spread.  Algorithmic bytes: the
distinct source bytes the bilinear taps read in each frame (per tapped luma pixel of NV12 / P010 the chroma pair it decodes
with, per tapped Bayer pixel its 3 x 3 demosaic neighbourhood), each distinct map once (8 bytes per output pixel) and the
output bytes.
"""
import argparse
import ctypes as C
import json
import os
import zlib

import numpy as np
import torch

from benchkit import (FORMATS, OUT_CODES, PEAK_GBS, ROOT, append_lines, frame_len, gpu_facts, mask_bytes, preprocess_desc, stream,
                      tap_mask, time_alternating)

F32 = np.float32
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}


def tapped_bytes(fmt, w, h, mx, my):
    """Distinct source bytes of one frame the bilinear sampler reads through the map (mx, my): see the module docstring."""
    with np.errstate(invalid="ignore"):
        inside = (mx >= 0) & (mx < F32(w)) & (my >= 0) & (my < F32(h))
    return mask_bytes(fmt, tap_mask(mx[inside], my[inside], w, h))


def camera(w, h, rng):
    """A 1080p-class camera with visible barrel distortion: (intrinsic, distortion)."""
    f = float(rng.uniform(0.9, 1.1)) * w * 0.6
    return (f, f, w / 2 + float(rng.uniform(-8, 8)), h / 2 + float(rng.uniform(-8, 8))), \
        (float(rng.uniform(-0.3, -0.2)), float(rng.uniform(0.03, 0.08)), 0.0, 0.0, 0.0, 0.0, float(rng.uniform(-1e-3, 1e-3)), float(rng.uniform(-1e-3, 1e-3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_preprocess_remap_bench.jsonl"))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--region-major-lib", default=None, help="a scratch build whose remap kernels walk regions slowest (R1 only)")
    a = ap.parse_args()
    import kornia_rs_b200 as kb
    from kornia_rs_b200._lib import RemapRoi
    from harness import compare_region
    from restate import Case, RCase, picture, remap_reference

    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    lib = kb._lib.lib()
    alt = None
    if a.region_major_lib:
        alt = C.CDLL(os.path.abspath(a.region_major_lib))
        alt.kb200_preprocess_remap.argtypes = lib.kb200_preprocess_remap.argtypes
        alt.kb200_preprocess_remap.restype = C.c_int
    dev = torch.device("cuda:0")
    facts = dict(zip(("gpu", "power_limit", "max_sm_clock"), gpu_facts().values()))

    def gen_map(intr, dist, new, dw, dh):
        mx = torch.empty((dh, dw), dtype=torch.float32, device=dev)
        my = torch.empty_like(mx)
        i4, d8 = (C.c_double * 4)(*intr), (C.c_double * 8)(*dist)
        if new is None:
            assert lib.kb200_generate_correction_map_polynomial(stream(), i4, d8, dw, dh, mx.data_ptr(), my.data_ptr(), mx.numel()) == 0
        else:
            assert lib.kb200_generate_correction_map_polynomial_to(stream(), i4, d8, (C.c_double * 4)(*new), dw, dh, mx.data_ptr(), my.data_ptr(),
                                                                  mx.numel()) == 0
        return mx, my

    def remap_call(fn, d, ptrs, lens, n, mx, my, n_maps, regs, dst, out):
        rois = (RemapRoi * len(regs))(*[RemapRoi(k, j) for k, j in regs])
        plane = mx.numel() // n_maps

        def run():
            st = fn(stream(), C.byref(d), ptrs, lens, n, mx.data_ptr(), my.data_ptr(), n_maps * plane, n_maps, rois, len(regs), dst.data_ptr(),
                    dst.numel(), OUT_CODES[out])
            assert st == 0, kb._lib.last_error()
        return run

    def check_regions(wl, fmt, w, h, dw, dh, out, base, need, regs, maps_x, maps_y, dst):
        torch.cuda.synchronize()
        c = Case(wl, 0, FORMATS[fmt][0], 0, 1, w, h, w * FORMATS[fmt][1], "remap", 1.0, 1.0, 0.0, 0.0, dw, dh, 1, False, "table", 1, (), None, 0,
                 "imagenet", 114.0)
        rc = RCase(c, 1, out, 1, (), ())
        picked = [0, len(regs) // 2, len(regs) - 1]
        for i in picked:
            k, j = regs[i]
            raw = base[k * need:(k + 1) * need].cpu().numpy()
            want = remap_reference(picture(c, raw), maps_x[j], maps_y[j], 1, "imagenet", 114.0, out)
            compare_region(dst[i].contiguous().view(torch.uint8).cpu().numpy().reshape(-1), want, rc, f"{wl} {fmt} {out} region {i}")
        return picked

    def frames_of(fmt, w, h, n, key):
        need = frame_len(fmt, w, h)
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(key.encode()))
        base = torch.randint(0, 256, (n * need,), dtype=torch.uint8, device=dev, generator=g)
        if fmt == "P010":   # codes in the high 10 bits
            base.view(torch.int16).bitwise_and_(-64)
        elif fmt == "RGGB12":   # codes below 2^12
            base.view(torch.int16).bitwise_and_(0x0FFF)
        ptrs = (C.c_void_p * n)(*[base.data_ptr() + k * need for k in range(n)])
        lens = (C.c_size_t * n)(*[need] * n)
        return base, need, ptrs, lens

    def emit(row, t, nbytes, main_arm, check):
        for k, (lo, hi) in t.items():
            row[f"{k}_ms_min"], row[f"{k}_ms_max"] = round(lo, 4), round(hi, 4)
        row["algorithmic_bytes"] = nbytes
        for k in t:
            if k in (main_arm, "batch_entry", "remap_region_major"):
                row[f"{k}_share_of_3.35TBps"] = round(nbytes / (t[k][0] * 1e-3) / (PEAK_GBS * 1e9), 3)
        row.update(iters=a.iters, repeats=a.repeats, **check, **facts)
        print(json.dumps(row), flush=True)
        lines.append(row)

    lines = []
    w, h = 1920, 1080

    # ── R1: 256 NV12 1080p frames, one shared full-resolution undistortion map ─────────────────────────────────────────
    n = 256
    base, need, ptrs, lens = frames_of("NV12", w, h, n, "R1")
    intr, dist = camera(w, h, np.random.default_rng(1))
    mx, my = gen_map(intr, dist, None, w, h)
    hx, hy = mx.cpu().numpy(), my.cpu().numpy()
    src_bytes = tapped_bytes("NV12", w, h, hx, hy) * n
    regs = [(k, 0) for k in range(n)]
    d = preprocess_desc(*FORMATS["NV12"], w, h, w, h)
    rgb = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
    rgb2 = torch.empty_like(rgb)
    dn = preprocess_desc(0, 3, w, h, w, h, bpp=3)   # RGB8
    for out in ("f32", "bf16"):
        dst = torch.empty((n, 3, h, w), dtype=DTYPES[out], device=dev)
        run = remap_call(lib.kb200_preprocess_remap, d, ptrs, lens, n, mx, my, 1, regs, dst, out)
        run()
        kern = kb._lib.last_kernel()
        check = {"regions_checked_against_reference": check_regions("R1", "NV12", w, h, w, h, out, base, need, regs, [hx], [hy], dst)}
        arms = {"remap": run}
        if alt is not None:
            adst = torch.empty_like(dst)
            arun = remap_call(alt.kb200_preprocess_remap, d, ptrs, lens, n, mx, my, 1, regs, adst, out)
            arun()
            torch.cuda.synchronize()
            check["region_major_identical"] = bool(torch.equal(adst.view(torch.uint8), dst.view(torch.uint8)))
            assert check["region_major_identical"], "the region-major build differs"
            arms["remap_region_major"] = arun
        entry = getattr(lib, f"kb200_preprocess_strided_{out}")
        edst = torch.empty_like(dst)

        def existing():
            s = stream()
            assert lib.kb200_rgb_from_nv12_u8(s, base.data_ptr(), base.numel(), rgb.data_ptr(), rgb.numel(), w, h, n) == 0
            assert lib.kb200_remap_u8(s, rgb.data_ptr(), rgb.numel(), rgb2.data_ptr(), rgb2.numel(), mx.data_ptr(), my.data_ptr(), mx.numel(), w, h, w, h,
                                      3, n, 1) == 0
            assert entry(s, C.byref(dn), rgb2.data_ptr(), rgb2.numel(), w * h * 3, n, edst.data_ptr(), edst.numel()) == 0

        arms["existing"] = existing
        t = time_alternating(arms, a.iters, a.repeats)
        nbytes = src_bytes + 8 * w * h + dst.numel() * dst.element_size()
        row = {"workload": "R1", "src": f"NV12 {w}x{h}", "out": out, "frames": n, "regions": n, "maps": 1, "dst": [3, h, w], "sampling": "Bilinear",
               "kernel": kern, "launches": -(-n // 192), "tapped_src_bytes": src_bytes}
        emit(row, t, nbytes, "remap", check)
        del dst, edst
        torch.cuda.empty_cache()

    # R1 identity twin: identity maps against the batch entry's identity kernel
    v, u = torch.meshgrid(torch.arange(h, dtype=torch.float32, device=dev), torch.arange(w, dtype=torch.float32, device=dev), indexing="ij")
    ix, iy = u.contiguous(), v.contiguous()
    for out in ("f32", "bf16"):
        dst = torch.empty((n, 3, h, w), dtype=DTYPES[out], device=dev)
        ref = torch.empty_like(dst)
        run = remap_call(lib.kb200_preprocess_remap, d, ptrs, lens, n, ix, iy, 1, regs, dst, out)
        run()
        kern = kb._lib.last_kernel()
        entry = getattr(lib, f"kb200_preprocess_strided_{out}")

        def batch():
            assert entry(stream(), C.byref(d), base.data_ptr(), base.numel(), need, n, ref.data_ptr(), ref.numel()) == 0

        batch()
        torch.cuda.synchronize()
        check = {"batch_entry_kernel": kb._lib.last_kernel(), "identical_to_batch_entry": bool(torch.equal(dst.view(torch.uint8), ref.view(torch.uint8)))}
        assert check["identical_to_batch_entry"], "R1 identity differs from the batch entry"
        t = time_alternating({"remap": run, "batch_entry": batch}, a.iters, a.repeats)
        src_b = (w * h * 3 // 2) * n
        nbytes = src_b + 8 * w * h + dst.numel() * dst.element_size()
        row = {"workload": "R1-identity", "src": f"NV12 {w}x{h}", "out": out, "frames": n, "regions": n, "maps": 1, "dst": [3, h, w],
               "sampling": "Bilinear", "kernel": kern, "tapped_src_bytes": src_b}
        emit(row, t, nbytes, "remap", check)
        del dst, ref
        torch.cuda.empty_cache()
    del base, rgb, rgb2
    torch.cuda.empty_cache()

    # ── R2: 64 1080p frames undistorted and fitted to 640 x 640 ─────────────────────────────────────────────────────────
    n, dw, dh = 64, 640, 640
    intr, dist = camera(w, h, np.random.default_rng(2))
    s = dw / w   # the whole frame's width across the output: a letterbox, the rows above and below are pad
    mx, my = gen_map(intr, dist, (intr[0] * s, intr[1] * s, dw / 2, dh / 2), dw, dh)
    hx, hy = mx.cpu().numpy(), my.cpu().numpy()
    regs = [(k, 0) for k in range(n)]
    for fmt in ("NV12", "P010", "RGGB12"):
        base, need, ptrs, lens = frames_of(fmt, w, h, n, "R2" + fmt)
        d = preprocess_desc(*FORMATS[fmt], w, h, dw, dh)
        src_bytes = tapped_bytes(fmt, w, h, hx, hy) * n
        for out in ("f32", "bf16"):
            dst = torch.empty((n, 3, dh, dw), dtype=DTYPES[out], device=dev)
            run = remap_call(lib.kb200_preprocess_remap, d, ptrs, lens, n, mx, my, 1, regs, dst, out)
            run()
            kern = kb._lib.last_kernel()
            check = {"regions_checked_against_reference": check_regions("R2", fmt, w, h, dw, dh, out, base, need, regs, [hx], [hy], dst)}
            t = time_alternating({"remap": run}, a.iters, a.repeats)
            nbytes = src_bytes + 8 * dw * dh + dst.numel() * dst.element_size()
            row = {"workload": "R2", "src": f"{fmt} {w}x{h}", "out": out, "frames": n, "regions": n, "maps": 1, "dst": [3, dh, dw],
                   "sampling": "Bilinear", "kernel": kern, "tapped_src_bytes": src_bytes}
            emit(row, t, nbytes, "remap", check)
        del base
        torch.cuda.empty_cache()

    # ── R3: a rig of 6 cameras x 16 frames, one 640 x 384 map per camera ────────────────────────────────────────────────
    cams, per, dw, dh = 6, 16, 640, 384
    n = cams * per
    base, need, ptrs, lens = frames_of("NV12", w, h, n, "R3")
    rng = np.random.default_rng(3)
    maps = []
    for q in range(cams):
        intr, dist = camera(w, h, rng)
        s = dw / w * float(rng.uniform(1.0, 1.3))
        maps.append(gen_map(intr, dist, (intr[0] * s, intr[1] * s, dw / 2, dh / 2), dw, dh))
    mx = torch.stack([m[0] for m in maps]).contiguous()
    my = torch.stack([m[1] for m in maps]).contiguous()
    hx, hy = mx.cpu().numpy(), my.cpu().numpy()
    regs = [(k, k % cams) for k in range(n)]   # frame k comes from camera k % 6
    d = preprocess_desc(*FORMATS["NV12"], w, h, dw, dh)
    src_bytes = sum(tapped_bytes("NV12", w, h, hx[k % cams], hy[k % cams]) for k in range(n))
    out = "f32"
    dst = torch.empty((n, 3, dh, dw), dtype=DTYPES[out], device=dev)
    run = remap_call(lib.kb200_preprocess_remap, d, ptrs, lens, n, mx, my, cams, regs, dst, out)
    run()
    kern = kb._lib.last_kernel()
    check = {"regions_checked_against_reference": check_regions("R3", "NV12", w, h, dw, dh, out, base, need, regs, hx, hy, dst)}
    pdst = torch.empty((cams, per, 3, dh, dw), dtype=DTYPES[out], device=dev)
    per_map = []
    for q in range(cams):
        fp = (C.c_void_p * per)(*[base.data_ptr() + k * need for k in range(q, n, cams)])
        fl = (C.c_size_t * per)(*[need] * per)
        per_map.append(remap_call(lib.kb200_preprocess_remap, d, fp, fl, per, mx[q], my[q], 1, [(i, 0) for i in range(per)], pdst[q], out))

    def six_calls():
        for fn in per_map:
            fn()

    six_calls()
    torch.cuda.synchronize()
    check["identical_to_per_map_calls"] = bool(torch.equal(pdst.transpose(0, 1).reshape(n, 3, dh, dw).view(torch.uint8), dst.view(torch.uint8)))
    assert check["identical_to_per_map_calls"], "R3 differs from the per-map calls"
    t = time_alternating({"remap": run, "per_map": six_calls}, a.iters, a.repeats)
    nbytes = src_bytes + 8 * dw * dh * cams + dst.numel() * dst.element_size()
    row = {"workload": "R3", "src": f"NV12 {w}x{h}", "out": out, "frames": n, "regions": n, "maps": cams, "dst": [3, dh, dw], "sampling": "Bilinear",
           "kernel": kern, "tapped_src_bytes": src_bytes}
    emit(row, t, nbytes, "remap", check)

    append_lines(a.out, lines)


if __name__ == "__main__":
    main()
