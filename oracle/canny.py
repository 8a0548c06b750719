"""Integer numpy restatement of controlnet_aux's `CannyDetector` at its defaults: cv2.Canny(HWC3(img), 100, 200) with aperture
3 and the L1 gradient.  Pinned bit for bit to cv2.Canny by tests/test_canny.py (golden fixtures written by
tests/golden/make_golden_canny.py, and cv2 itself where it is installed).

  * each channel's 3x3 Sobel (cv2.Sobel, ksize 3, BORDER_REPLICATE) in integers; per pixel the channel of largest
    |dx| + |dy| supplies dx, dy and the magnitude, the first channel on ties;
  * non-maximum suppression as cv::Canny: |dy| << 15 against |dx| * TG22 (TG22 = round(tan 22.5deg * 2^15)) and
    tg67x = tg22x + (|dx| << 16) pick horizontal / vertical / diagonal; '>' against one neighbour and '>=' against the other
    across horizontal and vertical gradients, '>' against both across diagonal ones; neighbours outside the image count 0;
  * thresholds swapped when low > high and floored; candidate m > low, strong m > high;
  * hysteresis: 255 on each candidate whose 8-connected component of candidates holds a strong pixel, 0 elsewhere;
  * the control image: the u8 map replicated to 3 channels, / 255.

Canny runs at the engine's resolution on the frame after the engine's nearest resize (as HED, oracle/hed.py); float frames
become u8 as rint(clamp(x, 0, 1) * 255) in fp32.  Test infrastructure only (see oracle/__init__)."""
from __future__ import annotations

import math

import numpy as np
from scipy import ndimage

CANNY_SHIFT = 15
TG22 = int(0.4142135623730950488016887242097 * (1 << CANNY_SHIFT) + 0.5)


def thresholds(low: float, high: float):
    """cv::Canny's integer thresholds: swapped when low > high, floored"""
    if low > high:
        low, high = high, low
    return math.floor(low), math.floor(high)


def to_u8(frame) -> np.ndarray:
    """(H, W, 3) u8, or a (3, H, W) float frame in [0, 1] (fp32 or fp16) -> (H, W, 3) u8 as the engine reads it"""
    a = np.asarray(frame)
    if a.dtype == np.uint8:
        return a
    x = np.fmin(np.fmax(a.astype(np.float32), np.float32(0)), np.float32(1)) * np.float32(255)
    return np.rint(x).astype(np.uint8).transpose(1, 2, 0)


def gradients(img: np.ndarray):
    """(H, W, 3) u8 -> dx, dy, mag (H, W) int32: the Sobels of the channel of largest |dx| + |dy| (first on ties)"""
    p = np.pad(img.astype(np.int32), ((1, 1), (1, 1), (0, 0)), mode="edge")
    dx = (p[:-2, 2:] - p[:-2, :-2]) + 2 * (p[1:-1, 2:] - p[1:-1, :-2]) + (p[2:, 2:] - p[2:, :-2])
    dy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    mag = np.abs(dx) + np.abs(dy)
    best = np.zeros(mag.shape[:2], dtype=np.int64)
    for c in range(1, mag.shape[2]):
        best = np.where(mag[..., c] > np.take_along_axis(mag, best[..., None], 2)[..., 0], c, best)
    pick = lambda a: np.take_along_axis(a, best[..., None], 2)[..., 0]
    return pick(dx), pick(dy), pick(mag)


def classes(img: np.ndarray, low: float = 100, high: float = 200) -> np.ndarray:
    """(H, W) u8: 0 none, 1 candidate (kept by non-maximum suppression, m > low), 2 strong (also m > high)"""
    lo, hi = thresholds(low, high)
    dx, dy, m = gradients(img)
    H, W = m.shape
    mp = np.pad(m, 1)   # magnitude 0 outside the image
    nb = lambda oy, ox: mp[1 + oy:1 + oy + H, 1 + ox:1 + ox + W]
    ax = np.abs(dx).astype(np.int64)
    ay = np.abs(dy).astype(np.int64) << CANNY_SHIFT
    tg22x = ax * TG22
    tg67x = tg22x + (ax << (CANNY_SHIFT + 1))
    horiz = ay < tg22x
    vert = ~horiz & (ay > tg67x)
    diag = ~horiz & ~vert
    s = np.where((dx ^ dy) < 0, -1, 1)
    keep_h = (m > nb(0, -1)) & (m >= nb(0, 1))
    keep_v = (m > nb(-1, 0)) & (m >= nb(1, 0))
    # diagonal: row above at x - s, row below at x + s
    keep_d = np.where(s < 0, (m > nb(-1, 1)) & (m > nb(1, -1)), (m > nb(-1, -1)) & (m > nb(1, 1)))
    keep = (m > lo) & ((horiz & keep_h) | (vert & keep_v) | (diag & keep_d))
    return np.where(keep, np.where(m > hi, 2, 1), 0).astype(np.uint8)


def hysteresis(cls: np.ndarray) -> np.ndarray:
    """(H, W) class map -> (H, W) u8 edge map: 255 on the candidates of 8-connected components with a strong pixel"""
    lab, n = ndimage.label(cls > 0, structure=np.ones((3, 3), dtype=bool))
    strong = np.zeros(n + 1, dtype=bool)
    strong[lab[cls == 2]] = True
    strong[0] = False
    return np.where(strong[lab], 255, 0).astype(np.uint8)


def canny(img: np.ndarray, low: float = 100, high: float = 200) -> np.ndarray:
    """cv2.Canny(img, low, high) for an (H, W, 3) u8 image: (H, W) u8"""
    return hysteresis(classes(img, low, high))


def control_image(frame, low: float = 100, high: float = 200) -> np.ndarray:
    """The frame's control image, (H, W, 3) u8 (0 / 255): CannyDetector's output, HWC3 of the edge map"""
    e = canny(to_u8(frame), low, high)
    return np.repeat(e[..., None], 3, axis=2)
