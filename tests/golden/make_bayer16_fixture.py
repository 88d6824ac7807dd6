"""Writes tests/golden/bayer16_cv2.npz: seeded 16-bit-sample Bayer frames and cv2's bilinear demosaic of each.

    python tests/golden/make_bayer16_fixture.py

Needs numpy and cv2 only.  The samples are LSB-aligned 16-bit words (V4L2's unpacked SRGGB10 ... SGBRG16): 10-bit,
12-bit and full-range 16-bit content, plus an all-65535 frame, the largest sums the arithmetic meets.  Patterns are
named as in make_bayer_fixture.py (the 2x2 quad read row-major; cv2's codes are offset from these names):

    RGGB <-> cv2.COLOR_BayerBG2RGB        BGGR <-> cv2.COLOR_BayerRG2RGB
    GRBG <-> cv2.COLOR_BayerGB2RGB        GBRG <-> cv2.COLOR_BayerGR2RGB

Keys per case `<pattern>_<bits>_<w>x<h>` (bits 10, 12, 16, or `max` for the all-65535 frame): `_raw` (h, w) uint16,
`_rgb` (h, w, 3) uint16, `_wh` (w, h).
"""
import os

import cv2
import numpy as np

CV2_CODE = {"rggb": cv2.COLOR_BayerBG2RGB, "bggr": cv2.COLOR_BayerRG2RGB, "grbg": cv2.COLOR_BayerGB2RGB,
            "gbrg": cv2.COLOR_BayerGR2RGB}
SIZES = [(3, 3), (6, 8), (7, 9), (16, 34), (53, 37)]   # (w, h): odd and even sizes and the 3x3 minimum
DEPTHS = (10, 12, 16)


def main():
    out = {}
    for pattern, code in CV2_CODE.items():
        for bits in DEPTHS:
            for w, h in SIZES:
                raw = np.random.default_rng(w * 1009 + h * 17 + bits * 7 + len(out)).integers(0, 1 << bits, (h, w), dtype=np.uint16)
                name = f"{pattern}_{bits}_{w}x{h}"
                out[f"{name}_raw"] = raw
                out[f"{name}_rgb"] = cv2.cvtColor(raw, code)
                out[f"{name}_wh"] = np.array([w, h], np.int32)
        raw = np.full((9, 7), 65535, np.uint16)
        name = f"{pattern}_max_7x9"
        out[f"{name}_raw"] = raw
        out[f"{name}_rgb"] = cv2.cvtColor(raw, code)
        out[f"{name}_wh"] = np.array([7, 9], np.int32)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bayer16_cv2.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out) // 3} cases, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
