"""kb200_preprocess_warps on an H100: rotated face crops, oriented 4K tiles, perspective plate crops and identity maps of
whole frames.  Appends one JSON line per workload, source format and output type to results/h100_preprocess_warp_bench.jsonl
(or --out).

  W1  faces: 256 similarity maps (angle within +-45 degrees, source faces 48-320 px) from 8 1080p frames to 112 x 112,
      f32 and bf16, on NV12, P010 and 8-bit RGGB frames.  Arms: `warps` (this entry); `rois` (kb200_preprocess_rois on each
      map's axis-aligned bounding box in the frame, Stretch: the same crops without the rotation); `existing` (today's
      path: the frames decoded to RGB8 by kb200_rgb_from_nv12_u8 / kb200_rgb_from_bayer_u8, one kb200_warp_affine_u8 per
      region, then kb200_preprocess_strided_* on the 256 RGB8 crops to normalise them to CHW; its u8 warp uses Q10
      arithmetic, so it is for timing only; there is no 8-bit path for P010, so that arm is not run there).
  W2  oriented tiles: 128 crops of 640 x 640 at 30 degrees from 16 NV12 4K frames, f32 (the frames do not fit in L2).
  W3  plates: 512 perspective crops of 192 x 64 from 16 NV12 1080p frames, bf16.
  W4  identity: 256 NV12 1080p frames through identity maps to 1920 x 1080, f32, against the batch entry
      (kb200_preprocess_strided_f32 at scale 1, its identity kernel) in the same run: the outputs must be identical.

W1-W3 check three regions of each `warps` output in the same run against restate.warp_reference.
Arms alternate: 20 launches after warm-up, 3 repeats, minima given with the repeat spread.  Algorithmic bytes: the distinct
source bytes the sampler taps in each frame over the union of its regions plus the output bytes.  The taps come from the
same float32 coordinate rule as the reference (warp_coords): for each inside pixel the tap (x0, y0), and x0 + 1 / y0 + 1
only where its weight is not zero; per tapped luma pixel of NV12 / P010 the chroma pair it decodes with (2 / 4 bytes per
(y / 2, x / 2)), per tapped Bayer pixel its 3 x 3 demosaic neighbourhood.
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


def tapped_bytes(fmt, w, h, regions, inverse, dw, dh):
    """Distinct source bytes the bilinear sampler reads over `regions` ([(k, forward map)]): see the module docstring."""
    from restate import warp_coords
    per_frame = {}
    for k, fwd in regions:
        inv, persp = inverse(fwd)
        sx, sy, inside, _ = warp_coords(inv, persp, dw, dh, w, h)
        sx = np.minimum(np.maximum(sx[inside], F32(0)), np.nextafter(F32(w), F32(0)))
        sy = np.minimum(np.maximum(sy[inside], F32(0)), np.nextafter(F32(h), F32(0)))
        tap_mask(sx, sy, w, h, per_frame.setdefault(k, np.zeros((h, w), bool)))
    return sum(mask_bytes(fmt, m) for m in per_frame.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_preprocess_warp_bench.jsonl"))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import kornia_rs_b200 as kb
    from kornia_rs_b200._lib import Roi, WarpRoi
    from harness import compare_region, inverse
    from restate import Case, RCase, forward_of, picture, warp_reference

    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    lib = kb._lib.lib()
    dev = torch.device("cuda:0")
    facts = dict(zip(("gpu", "power_limit", "max_sm_clock"), gpu_facts().values()))

    def lib_inverse(fwd):
        return inverse(lib, fwd)

    lines = []

    def similarity(w, h, dw, dh, side, ang, cx, cy):
        """Forward map taking a side x side square centred at (cx, cy), turned by ang, onto the dw x dh output."""
        r = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]]) * (side / dw)
        inv = np.eye(3)
        inv[:2, :2] = r
        inv[:2, 2] = np.array([cx, cy]) - r @ np.array([dw / 2, dh / 2])
        return forward_of(inv)

    def bbox(fwd, w, h, dw, dh):
        """The output rectangle's corners mapped into the frame: their axis-aligned bounding box, clipped to the frame."""
        inv = np.linalg.inv(np.array(fwd, np.float64).reshape(3, 3))
        pts = inv @ np.array([[0, dw, 0, dw], [0, 0, dh, dh], [1, 1, 1, 1]], np.float64)
        xs, ys = pts[0] / pts[2], pts[1] / pts[2]
        x0, y0 = int(max(0, np.floor(xs.min()))), int(max(0, np.floor(ys.min())))
        x1, y1 = int(min(w, np.ceil(xs.max()))), int(min(h, np.ceil(ys.max())))
        return x0, y0, max(1, x1 - x0), max(1, y1 - y0)

    plan = []
    for fmt in ("NV12", "P010", "RGGB"):
        for out in ("f32", "bf16"):
            plan.append(("W1", fmt, out))
    plan += [("W2", "NV12", "f32"), ("W3", "NV12", "bf16"), ("W4", "NV12", "f32")]
    cache = {}
    for wl, fmt, out in plan:
        if wl == "W1":
            w, h, n, dw, dh, m = 1920, 1080, 8, 112, 112, 256
        elif wl == "W2":
            w, h, n, dw, dh, m = 3840, 2160, 16, 640, 640, 128
        elif wl == "W3":
            w, h, n, dw, dh, m = 1920, 1080, 16, 192, 64, 512
        else:
            w, h, n, dw, dh, m = 1920, 1080, 256, 1920, 1080, 256
        key = (wl, fmt)
        if key not in cache:
            r = np.random.default_rng(zlib.crc32("/".join(key).encode()))
            if wl == "W1":
                regs = []
                for i in range(m):
                    side = float(r.uniform(48, 320))
                    regs.append((i % n, similarity(w, h, dw, dh, side, float(np.deg2rad(r.uniform(-45, 45))), float(r.uniform(side, w - side)),
                                                   float(r.uniform(side, h - side)))))
            elif wl == "W2":
                regs = [(i % n, similarity(w, h, dw, dh, 640.0, float(np.deg2rad(30)), float(r.uniform(500, w - 500)), float(r.uniform(500, h - 500))))
                        for i in range(m)]
            elif wl == "W3":
                regs = []
                for i in range(m):
                    inv = np.eye(3)
                    inv[:2, :2] = np.array([[1.0, 0.15], [0.05, 1.0]]) * r.uniform(0.8, 1.6)
                    inv[:2, 2] = (r.uniform(100, w - 400), r.uniform(100, h - 200))
                    inv[2, :2] = r.uniform(-1e-3, 1e-3, 2)
                    regs.append((i % n, forward_of(inv)))
            else:
                regs = [(i, (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)) for i in range(m)]
            need = frame_len(fmt, w, h)
            base = torch.randint(0, 256, (n * need,), dtype=torch.uint8, device=dev)
            if fmt == "P010":   # codes in the high 10 bits
                base.view(torch.int16).bitwise_and_(-64)
            one = tapped_bytes(fmt, w, h, regs[:1], lib_inverse, dw, dh) if wl == "W4" else None
            src_bytes = one * n if wl == "W4" else tapped_bytes(fmt, w, h, regs, lib_inverse, dw, dh)
            cache[key] = (regs, need, base, src_bytes)
        regs, need, base, src_bytes = cache[key]
        frames = [base[k * need:(k + 1) * need] for k in range(n)]
        ptrs = (C.c_void_p * n)(*[f.data_ptr() for f in frames])
        lens = (C.c_size_t * n)(*[need] * n)
        warps = (WarpRoi * m)(*[WarpRoi(k, (C.c_float * 9)(*f)) for k, f in regs])
        d = preprocess_desc(*FORMATS[fmt], w, h, dw, dh)
        dst = torch.empty((m, 3, dh, dw), dtype=DTYPES[out], device=dev)

        def run_warps():
            st = lib.kb200_preprocess_warps(stream(), C.byref(d), ptrs, lens, n, warps, m, dst.data_ptr(), dst.numel(), OUT_CODES[out])
            assert st == 0, kb._lib.last_error()

        run_warps()
        kern = kb._lib.last_kernel()
        arms = {"warps": run_warps}
        check = {}
        if wl == "W4":
            ref = torch.empty_like(dst)
            entry = getattr(lib, f"kb200_preprocess_strided_{out}")

            def batch():
                assert entry(stream(), C.byref(d), base.data_ptr(), base.numel(), need, n, ref.data_ptr(), ref.numel()) == 0

            batch()
            arms["batch_entry"] = batch
            torch.cuda.synchronize()
            check["batch_entry_kernel"] = kb._lib.last_kernel()
            check["identical_to_batch_entry"] = bool(torch.equal(dst.view(torch.int32), ref.view(torch.int32)))
            assert check["identical_to_batch_entry"], "W4 differs from the batch entry"
        else:
            torch.cuda.synchronize()
            host = base.cpu().numpy()
            c = Case(wl, 0, FORMATS[fmt][0], 0, 1, w, h, w * FORMATS[fmt][1], "warp", 1.0, 1.0, 0.0, 0.0, dw, dh, 1, False, "table", n, (), None, 0,
                     "imagenet", 114.0)
            rc = RCase(c, 1, out, n, (), ())
            picked = [0, m // 2, m - 1]
            for i in picked:
                k, fwd = regs[i]
                inv, persp = inverse(lib, fwd)
                got = dst[i].contiguous().view(torch.uint8).cpu().numpy().reshape(-1)
                compare_region(got, warp_reference(picture(c, host[k * need:(k + 1) * need]), inv, persp, dw, dh, 1, "imagenet", 114.0, out), rc,
                        f"{wl} {fmt} region {i}")
            check["regions_checked_against_reference"] = picked
        if wl == "W1":
            boxes = [(k,) + bbox(f, w, h, dw, dh) for k, f in regs]
            rois = (Roi * m)(*[Roi(*b) for b in boxes])
            rdst = torch.empty_like(dst)

            def run_rois():
                st = lib.kb200_preprocess_rois(stream(), C.byref(d), 1, ptrs, lens, n, rois, m, rdst.data_ptr(), rdst.numel(), OUT_CODES[out])
                assert st == 0, kb._lib.last_error()

            arms["rois"] = run_rois
            if fmt != "P010":
                rgb = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
                crops = torch.empty((m, dh, dw, 3), dtype=torch.uint8, device=dev)
                ms = [(C.c_float * 6)(*f[:6]) for _, f in regs]
                dn = preprocess_desc(0, 3, dw, dh, dw, dh, bpp=3)   # RGB8
                entry = getattr(lib, f"kb200_preprocess_strided_{out}")
                edst = torch.empty_like(dst)

                def existing():
                    s = stream()
                    if fmt == "NV12":
                        assert lib.kb200_rgb_from_nv12_u8(s, base.data_ptr(), base.numel(), rgb.data_ptr(), rgb.numel(), w, h, n) == 0
                    else:
                        assert lib.kb200_rgb_from_bayer_u8(s, base.data_ptr(), base.numel(), rgb.data_ptr(), rgb.numel(), w, h, n, 0) == 0
                    fb, cb = w * h * 3, dw * dh * 3
                    for i, (k, _) in enumerate(regs):
                        assert lib.kb200_warp_affine_u8(s, rgb.data_ptr() + k * fb, fb, crops.data_ptr() + i * cb, cb, w, h, dw, dh, 3, 1, ms[i]) == 0
                    assert entry(s, C.byref(dn), crops.data_ptr(), crops.numel(), cb, m, edst.data_ptr(), edst.numel()) == 0

                arms["existing"] = existing
        t = time_alternating(arms, a.iters, a.repeats)
        nbytes = src_bytes + dst.numel() * dst.element_size()
        row = {"workload": wl, "src": f"{fmt} {w}x{h}", "out": out, "frames": n, "regions": m, "dst": [3, dh, dw], "sampling": "Bilinear",
               "kernel": kern, "launches": -(-m // 72), "tapped_src_bytes": src_bytes, "algorithmic_bytes": nbytes}
        for k, (lo, hi) in t.items():
            row[f"{k}_ms_min"], row[f"{k}_ms_max"] = round(lo, 4), round(hi, 4)
        row["warps_share_of_3.35TBps"] = round(nbytes / (t["warps"][0] * 1e-3) / (PEAK_GBS * 1e9), 3)
        if "batch_entry" in t:
            row["batch_entry_share_of_3.35TBps"] = round(nbytes / (t["batch_entry"][0] * 1e-3) / (PEAK_GBS * 1e9), 3)
        row.update(iters=a.iters, repeats=a.repeats, **check, **facts)
        print(json.dumps(row), flush=True)
        lines.append(row)
        del dst
        torch.cuda.empty_cache()
    append_lines(a.out, lines)


if __name__ == "__main__":
    main()
