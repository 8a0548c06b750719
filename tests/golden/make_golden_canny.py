"""Writes tests/golden/canny_cv2.npz (python tests/golden/make_golden_canny.py, needs cv2): input images, thresholds and
cv2.Canny's outputs, so that the restatement oracle/canny.py is pinned to OpenCV where cv2 is not installed.  Random, blurred
and structured images of odd and non-square shapes, thresholds reversed, equal, fractional, zero and above 2040."""
import os

import cv2
import numpy as np
from scipy import ndimage

HERE = os.path.dirname(os.path.abspath(__file__))
THRESHOLDS = [(100, 200), (200, 100), (60, 60), (50.7, 120.2), (0, 0), (30, 2100), (-3, 75.9)]


def images():
    rng = np.random.default_rng(1234)
    out = []
    for i, (h, w) in enumerate([(37, 53), (64, 64), (29, 97), (80, 41), (1, 17), (33, 1)]):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if i % 3 == 1:
            img = ndimage.gaussian_filter(img.astype(np.float64), (1.3, 1.3, 0)).clip(0, 255).astype(np.uint8)
        elif i % 3 == 2:   # structured: discs and bars with per-channel offsets
            yy, xx = np.mgrid[:h, :w]
            base = ((yy - h / 2) ** 2 + (xx - w / 3) ** 2 < (min(h, w) / 3) ** 2) * 170 + ((xx // 7) % 2) * 60
            img = np.stack([base, np.roll(base, 2, 1), base // 2 + 40], -1).clip(0, 255).astype(np.uint8)
        out.append(img)
    return out


def main():
    arrays = {}
    for i, img in enumerate(images()):
        arrays[f"img{i}"] = img
        for j, (lo, hi) in enumerate(THRESHOLDS):
            arrays[f"edge{i}_{j}"] = cv2.Canny(img, lo, hi)
    arrays["thresholds"] = np.array(THRESHOLDS, dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, "canny_cv2.npz"), **arrays)


if __name__ == "__main__":
    main()
