"""kb200_preprocess_rois on an H100: whole frames against the batch entry, detection crops and 4K tiles, against one
preprocess call per region.  Appends one JSON line per workload and output type to results/h100_preprocess_roi_bench.jsonl
(or --out).

  W1  256 NV12 1080p frames, one region (k, 0, 0, 1920, 1080) each, Letterbox to 640x640 Bilinear, against
      kb200_preprocess_strided_* on the same frames; the outputs must be identical.
  W2  8 NV12 1080p frames, 32 seeded regions each (sides 32-512, random positions, odd origins) -> 256 x [3, 224, 224],
      Letterbox, Bilinear.
  W3  16 NV12 4K frames, 7 x 4 overlapping 640x640 tiles each -> 448 x [3, 640, 640], Stretch (identity-scale regions).

The W2 / W3 comparison arm is one kb200_preprocess_* call per region with a zoom descriptor over the whole frame (the only
way to crop a YUV frame without this entry).  Its taps clamp at the frame's edges, not the region's, so its outputs differ
at region borders: it is for timing only.  Three regions of each W2 / W3 output are checked in the same run against the
crop reference restate.region_reference (the oracle on the w x h crop of the decoded frame).

W1 has a third arm: the batch entry called once per 80 frames (80, 80, 80, 16), the launches the region entry makes for 256
regions, which tells the cost of that split from the rest of the gap.

Arms alternate: 20 launches after warm-up, 3 repeats, minima given with the repeat spread.  Algorithmic bytes: the distinct
source bytes the bilinear sampler taps per frame over the union of its regions (taps_1d: the tap rows and columns of each
region, the x1 / y1 tap only where its weight is not zero, and the chroma pairs those luma taps use), plus the output
bytes.
"""
import argparse
import ctypes as C
import json
import os

import numpy as np
import torch

from benchkit import FORMATS, OUT_CODES, PEAK_GBS, ROOT, append_lines, gpu_facts, preprocess_desc, stream, time_alternating

DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}


def taps_1d(n_out, scale, pad, n, origin):
    """Frame coordinates the bilinear sampler taps along one axis of a region of n samples at `origin`: for each output
    coordinate inside the region, s = (o - pad) / scale (f32, IEEE), the tap floor(s), and floor(s) + 1 (clamped to the
    region) only where the weight s - floor(s) is not zero."""
    s = (np.arange(n_out, dtype=np.float32) - np.float32(pad)) / np.float32(scale)
    s = s[(s >= 0) & (s < n)]
    x0 = np.floor(s)
    x1 = np.minimum(x0[s != x0] + 1, n - 1)
    return origin + np.unique(np.concatenate([x0, x1]).astype(np.int64))


def src_bytes_tapped(w, h, rois_per_frame, dw, dh, mode, affine):
    """Distinct NV12 bytes the bilinear sampler reads for the regions of each frame: the union over the frame's regions of
    the luma samples it taps (the tap rows x the tap columns of each region) and of the chroma pairs those taps decode
    with (2 bytes per (y / 2, x / 2))."""
    total = 0
    for rois in rois_per_frame:
        luma = np.zeros((h, w), bool)
        for _, x, y, rw, rh in rois:
            sx, sy, px, py = affine(mode, rw, rh, dw, dh)
            luma[np.ix_(taps_1d(dh, sy, py, rh, y), taps_1d(dw, sx, px, rw, x))] = True
        ys, xs = np.nonzero(luma)
        chroma = np.zeros((h // 2, w // 2), bool)
        chroma[ys >> 1, xs >> 1] = True
        total += int(luma.sum()) + 2 * int(chroma.sum())
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "h100_preprocess_roi_bench.jsonl"))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import kornia_rs_b200 as kb
    from kornia_rs_b200._lib import Roi
    from oracle.oracle import preprocess_affine
    from harness import compare_region
    from restate import Case, RCase, picture, region_reference

    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    lib = kb._lib.lib()
    dev = torch.device("cuda:0")
    facts = dict(zip(("gpu", "power_limit", "max_sm_clock"), gpu_facts().values()))

    def roi_call(d, mode, ptrs, lens, rois, dst, out):
        st = lib.kb200_preprocess_rois(stream(), C.byref(d), mode, ptrs, lens, len(lens), rois, len(rois),
                                       dst.data_ptr(), dst.numel(), OUT_CODES[out])
        assert st == 0, kb._lib.last_error()
        return lib.kb200_last_kernel().decode()

    lines = []
    rng = np.random.default_rng(2026)
    for wl in ("W1", "W2", "W3"):
        if wl == "W1":
            w, h, n, dw, dh, mode = 1920, 1080, 256, 640, 640, 0
            per = [[(k, 0, 0, w, h)] for k in range(n)]
        elif wl == "W2":
            w, h, n, dw, dh, mode = 1920, 1080, 8, 224, 224, 0
            per = []
            for k in range(n):
                rs = []
                for _ in range(32):
                    rw, rh = int(rng.integers(32, 513)), int(rng.integers(32, 513))
                    x, y = int(rng.integers(0, (w - rw) // 2)) * 2 + 1, int(rng.integers(0, (h - rh) // 2)) * 2 + 1
                    rs.append((k, min(x, w - rw), min(y, h - rh), rw, rh))
                per.append(rs)
        else:
            w, h, n, dw, dh, mode = 3840, 2160, 16, 640, 640, 1
            xs = [round(i * (w - 640) / 6) for i in range(7)]
            ys = [round(j * (h - 640) / 3) for j in range(4)]
            per = [[(k, x, y, 640, 640) for y in ys for x in xs] for k in range(n)]
        need = w * h * 3 // 2
        base = torch.randint(0, 256, (n * need,), dtype=torch.uint8, device=dev)
        frames = [base[k * need:(k + 1) * need] for k in range(n)]
        ptrs = (C.c_void_p * n)(*[f.data_ptr() for f in frames])
        lens = (C.c_size_t * n)(*[need] * n)
        flat = [r for rs in per for r in rs]
        rois = (Roi * len(flat))(*[Roi(*r) for r in flat])
        d = preprocess_desc(*FORMATS["NV12"], w, h, dw, dh)
        m = len(flat)
        for out in ("f32", "bf16"):
            dst = torch.empty((m, 3, dh, dw), dtype=DTYPES[out], device=dev)
            ref = torch.empty_like(dst)
            kern = roi_call(d, mode, ptrs, lens, rois, dst, out)
            entry = getattr(lib, f"kb200_preprocess_strided_{out}")
            if wl == "W1":
                dfull = preprocess_desc(*FORMATS["NV12"], w, h, dw, dh, preprocess_affine(mode, w, h, dw, dh))

                def other():
                    assert entry(stream(), C.byref(dfull), base.data_ptr(), base.numel(), need, n, ref.data_ptr(),
                                 ref.numel()) == 0
            else:
                # one call per region: a zoom descriptor on the whole frame (taps clamp at the frame's edges)
                calls = []
                for i, (k, x, y, rw, rh) in enumerate(flat):
                    sx, sy, px, py = preprocess_affine(mode, rw, rh, dw, dh)
                    dz = preprocess_desc(*FORMATS["NV12"], w, h, dw, dh, (sx, sy, px - x * sx, py - y * sy))
                    calls.append((dz, frames[k].data_ptr(), ref[i].data_ptr()))

                def other():
                    s = stream()
                    for dz, fp, op in calls:
                        entry(s, C.byref(dz), fp, need, need, 1, op, 3 * dw * dh)
            other()
            torch.cuda.synchronize()
            check = {}
            if wl == "W1":
                check["identical_to_batch_entry"] = bool(torch.equal(dst.view(torch.int16 if out == "bf16" else torch.int32),
                                                                     ref.view(torch.int16 if out == "bf16" else torch.int32)))
                assert check["identical_to_batch_entry"], "W1 differs from the batch entry"
            else:
                host = base.cpu().numpy()
                c = Case(wl, 0, 3, 0, 1, w, h, w, "roi", 1.0, 1.0, 0.0, 0.0, dw, dh, 1, False, "table", n, (), None, 0, "imagenet", 114.0)
                rc = RCase(c, mode, out, n, tuple(k * need for k in range(n)), tuple(flat))
                picked = [0, len(flat) // 2, len(flat) - 1]
                for i in picked:
                    k = flat[i][0]
                    pic = picture(c, host[k * need:(k + 1) * need])
                    got = dst[i].contiguous().view(torch.uint8).cpu().numpy().reshape(-1)
                    compare_region(got, region_reference(rc, pic, flat[i]), rc, f"{wl} region {i}")
                check["regions_checked_against_crop_reference"] = picked
            arms = {"rois": lambda: roi_call(d, mode, ptrs, lens, rois, dst, out), "existing": other}
            if wl == "W1":   # the batch entry in the region entry's launches: 80 frames per call
                def split():
                    st = stream()
                    for f0 in range(0, n, 80):
                        nb = min(80, n - f0)
                        assert entry(st, C.byref(dfull), base.data_ptr() + f0 * need, nb * need, need, nb,
                                     ref.data_ptr() + f0 * 3 * dw * dh * ref.element_size(), nb * 3 * dw * dh) == 0
                arms["existing_80_per_launch"] = split
            t = time_alternating(arms, a.iters, a.repeats)
            esz = dst.element_size()
            nbytes = src_bytes_tapped(w, h, per, dw, dh, mode, preprocess_affine) + dst.numel() * esz
            row = {"workload": wl, "out": out, "frames": n, "regions": m, "src": f"NV12 {w}x{h}", "dst": [3, dh, dw], "mode": ["Letterbox", "Stretch"][mode],
                   "sampling": "Bilinear", "kernel": kern, "launches": -(-m // 80),
                   "rois_ms_min": round(t["rois"][0], 4), "rois_ms_max": round(t["rois"][1], 4),
                   "existing_arm": "kb200_preprocess_strided (one call)" if wl == "W1" else f"{m} x kb200_preprocess_strided (zoom descriptor, timing only)",
                   "existing_ms_min": round(t["existing"][0], 4), "existing_ms_max": round(t["existing"][1], 4),
                   "algorithmic_bytes": nbytes, "rois_share_of_3.35TBps": round(nbytes / (t["rois"][0] * 1e-3) / (PEAK_GBS * 1e9), 3),
                   "existing_share_of_3.35TBps": round(nbytes / (t["existing"][0] * 1e-3) / (PEAK_GBS * 1e9), 3),
                   **({"existing_80_per_launch_ms_min": round(t["existing_80_per_launch"][0], 4),
                       "existing_80_per_launch_ms_max": round(t["existing_80_per_launch"][1], 4)} if wl == "W1" else {}),
                   "iters": a.iters, "repeats": a.repeats, **check, **facts}
            print(json.dumps(row), flush=True)
            lines.append(row)
    append_lines(a.out, lines)


if __name__ == "__main__":
    main()
