"""Writes tests/golden/bayer_cv2.npz: seeded raw Bayer frames and cv2's bilinear demosaic of each.

    python tests/golden/make_bayer_fixture.py

Needs numpy and cv2 only.  A pattern is named by its 2x2 quad read row-major (top-left, top-right, bottom-left,
bottom-right): RGGB means the top-left pixel is R.  cv2's conversion codes name the pattern by the second row's
middle pair, so they are offset from these names:

    RGGB <-> cv2.COLOR_BayerBG2RGB        BGGR <-> cv2.COLOR_BayerRG2RGB
    GRBG <-> cv2.COLOR_BayerGB2RGB        GBRG <-> cv2.COLOR_BayerGR2RGB

Keys per case `<pattern>_<w>x<h>`: `_raw` (h, w) uint8, `_rgb` (h, w, 3) uint8, `_wh` (w, h).
"""
import os

import cv2
import numpy as np

CV2_CODE = {"rggb": cv2.COLOR_BayerBG2RGB, "bggr": cv2.COLOR_BayerRG2RGB, "grbg": cv2.COLOR_BayerGB2RGB,
            "gbrg": cv2.COLOR_BayerGR2RGB}
SIZES = [(3, 3), (5, 5), (6, 8), (7, 9), (16, 34), (64, 130)]   # (w, h): odd sizes and the 3x3 minimum included


def main():
    out = {}
    for pattern, code in CV2_CODE.items():
        for w, h in SIZES:
            raw = np.random.default_rng(w * 1009 + h * 17 + len(out)).integers(0, 256, (h, w), dtype=np.uint8)
            name = f"{pattern}_{w}x{h}"
            out[f"{name}_raw"] = raw
            out[f"{name}_rgb"] = cv2.cvtColor(raw, code)
            out[f"{name}_wh"] = np.array([w, h], np.int32)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bayer_cv2.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out) // 3} cases, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
