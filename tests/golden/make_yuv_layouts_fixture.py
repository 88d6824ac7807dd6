"""Generates tests/golden/yuv_layouts_cv2.npz.  Needs only numpy and cv2 (which the tests may not depend on at run
time), so it runs on its own:

    python tests/golden/make_yuv_layouts_fixture.py

yuv_layouts_cv2.npz — raw frames + cv2.cvtColor(COLOR_YUV2RGB_<layout>) outputs for the YUV layouts beyond NV12 / YUYV
(NV21, I420, YV12, UYVY, YVYU), the cv2 anchor of tests/test_yuv_layouts.py; nv12_cv2.npz / yuyv_cv2.npz
(make_fixtures.py) are the same for NV12 / YUYV.  Keys: `<layout>_<case>_{raw,rgb,wh}`.  4:2:0 cases cover the
reference's generators (yuv/kernels.rs:2078-2081, :2112-2122, here in each layout's byte order), odd chroma widths
(w = 70, 130), a 2-row frame and random bytes; 4:2:2 cases the known gray (:2068), odd pair counts (w = 70, 130), a
1-row frame and random bytes.
"""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def cases() -> dict:
    import cv2

    rng = np.random.default_rng(20261015)
    codes = {"nv21": cv2.COLOR_YUV2RGB_NV21, "i420": cv2.COLOR_YUV2RGB_I420, "yv12": cv2.COLOR_YUV2RGB_YV12,
             "uyvy": cv2.COLOR_YUV2RGB_UYVY, "yvyu": cv2.COLOR_YUV2RGB_YVYU}
    out = {}
    for layout in ("nv21", "i420", "yv12"):
        for name, (w, h) in {"a": (4, 4), "b": (64, 6), "c": (70, 4), "d": (130, 2), "e": (128, 96)}.items():
            if name == "a":
                raw = np.concatenate([np.array([(v * 9 + 16) & 0xFF for v in range(w * h)], np.uint8),
                                      np.array([(v * 5 + 100) & 0xFF for v in range(w * h // 2)], np.uint8)])
            elif name in ("b", "c"):
                raw = np.concatenate([np.array([(i * 7 + 16) % 240 for i in range(w * h)], np.uint8),
                                      np.array([(i * 5 + 90) % 250 for i in range(w * h // 2)], np.uint8)])
            else:
                raw = rng.integers(0, 256, w * h * 3 // 2, dtype=np.uint8)
            out[f"{layout}_{name}_raw"] = raw
            out[f"{layout}_{name}_rgb"] = cv2.cvtColor(raw.reshape(h * 3 // 2, w), codes[layout])
            out[f"{layout}_{name}_wh"] = np.array([w, h])
    for layout in ("uyvy", "yvyu"):
        for name, (w, h) in {"a": (2, 1), "b": (64, 5), "c": (130, 7), "d": (70, 1)}.items():
            raw = rng.integers(0, 256, w * h * 2, dtype=np.uint8)
            if name == "a":
                raw = np.array([128, 16, 128, 16] if layout == "uyvy" else [16, 128, 16, 128], np.uint8)
            out[f"{layout}_{name}_raw"] = raw
            out[f"{layout}_{name}_rgb"] = cv2.cvtColor(raw.reshape(h, w, 2), codes[layout])
            out[f"{layout}_{name}_wh"] = np.array([w, h])
    return out


def main():
    np.savez_compressed(os.path.join(HERE, "yuv_layouts_cv2.npz"), **cases())
    print("yuv_layouts_cv2.npz written to", HERE)


if __name__ == "__main__":
    main()
