"""A numpy / scipy restatement of the VideoComposer canny annotator (tools/annotator/canny/__init__.py CannyDetector),
written from OpenCV's documented behaviour and needing no cv2: the oracle of vgen_b200/canny.py at any size.

* `quantise`: cv2.convertScaleAbs(img * 255.) of an fp32 (h, w, c) frame: the fp32 product, |x|, round to nearest even,
  saturate to uint8.
* `thresholds`: the reference's threshold choice from the frame's median (np.median over all h * w * c bytes).
* `canny`: cv2.Canny(img, low, high) with aperture 3 and the L1 gradient: thresholds swapped if low > high and floored;
  3x3 Sobel with replicated borders; for several channels the channel with the strictly largest |dx| + |dy|;
  non-maximum suppression with the Q15 tan(22.5 deg) direction test (magnitude outside the image is 0); candidates
  m > low, strong pixels m > high; hysteresis: a candidate is an edge when it is 8-connected through candidates to a
  strong pixel (scipy.ndimage.label).
"""
from __future__ import annotations

import math

import numpy as np
from scipy import ndimage

TG22 = 13573  # round(tan(22.5 deg) * 2^15)


def quantise(img):
    """convertScaleAbs(img * 255.) of an fp32 array."""
    x = np.abs(np.asarray(img, dtype=np.float32) * np.float32(255.0))
    return np.clip(np.rint(np.nan_to_num(x, nan=0.0)), 0, 255).astype(np.uint8)


def thresholds(img_u8, low=None, high=None, random_threshold=True, r=None):
    """The (low, high) the reference passes to cv2.Canny.  With both None: from m = np.median(img_u8), either
    (1 -/+ 0.33) * m (random_threshold is False) or (1 - r) * m and twice that, r the reference's
    np.random.uniform(0.1, 0.4) draw (pass it, or leave it None to draw it here from numpy's global stream)."""
    if low is None and high is None:
        m = np.median(img_u8)
        if random_threshold is False:
            return int(max(0, (1 - 0.33) * m)), int(min(255, (1 + 0.33) * m))
        if r is None:
            r = np.random.uniform(0.1, 0.4)
        low = int(max(0, (1 - r) * m))
        return low, 2 * low
    return low, high


def cv_thresholds(low, high):
    """cv2.Canny's integer thresholds: swapped if low > high, then floored."""
    low, high = float(low), float(high)
    if low > high:
        low, high = high, low
    return math.floor(low), math.floor(high)


def sobel(b):
    """3x3 Sobel dx, dy (int32) of one uint8 channel, replicated borders."""
    p = np.pad(b.astype(np.int32), 1, mode="edge")
    dx = (p[:-2, 2:] + 2 * p[1:-1, 2:] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[1:-1, :-2] + p[2:, :-2])
    dy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    return dx, dy


def classify(img_u8, low, high):
    """Per pixel 0 (no edge), 1 (candidate) or 2 (strong) after non-maximum suppression; low / high are the integer
    thresholds of cv_thresholds."""
    img = np.asarray(img_u8)
    if img.ndim == 2:
        img = img[:, :, None]
    dx, dy = sobel(img[:, :, 0])
    mag = np.abs(dx) + np.abs(dy)
    for ch in range(1, img.shape[2]):
        cx, cy = sobel(img[:, :, ch])
        cm = np.abs(cx) + np.abs(cy)
        sel = cm > mag
        dx, dy, mag = np.where(sel, cx, dx), np.where(sel, cy, dy), np.where(sel, cm, mag)
    h, w = mag.shape
    M = np.pad(mag, 1)                                     # magnitude outside the image is 0

    def nb(oy, ox):
        return M[1 + oy:1 + oy + h, 1 + ox:1 + ox + w]

    ax = np.abs(dx).astype(np.int64)
    ay = np.abs(dy).astype(np.int64) << 15
    tg22 = ax * TG22
    horiz = ay < tg22
    vert = ~horiz & (ay > tg22 + (ax << 16))
    diag = ~horiz & ~vert
    s = np.where((dx ^ dy) < 0, -1, 1)
    # the diagonal neighbours along the gradient: (y - 1, x - s) and (y + 1, x + s)
    d_prev = np.where(s < 0, nb(-1, 1), nb(-1, -1))
    d_next = np.where(s < 0, nb(1, -1), nb(1, 1))
    peak = ((horiz & (mag > nb(0, -1)) & (mag >= nb(0, 1)))
            | (vert & (mag > nb(-1, 0)) & (mag >= nb(1, 0)))
            | (diag & (mag > d_prev) & (mag > d_next)))
    cand = peak & (mag > low)
    return np.where(cand, np.where(mag > high, 2, 1), 0).astype(np.uint8)


def hysteresis(cls):
    """Candidates 8-connected through candidates to a strong pixel."""
    lab, _ = ndimage.label(cls > 0, structure=np.ones((3, 3), dtype=bool))
    strong = np.unique(lab[cls == 2])
    return np.isin(lab, strong[strong > 0])


def canny(img_u8, low, high):
    """cv2.Canny(img_u8, low, high) (aperture 3, L1 gradient) as uint8 0 / 255."""
    lo, hi = cv_thresholds(low, high)
    return hysteresis(classify(img_u8, lo, hi)).astype(np.uint8) * np.uint8(255)


def detect(img, low_threshold=None, high_threshold=None, random_threshold=True, r=None):
    """CannyDetector()(img, ...) as a float32 (h, w, 1) array of 0 / 1: img is fp32 (h, w, c) in [0, 1] (quantised) or
    uint8 (taken as it is)."""
    img_np = img if np.asarray(img).dtype == np.uint8 else quantise(img)
    low, high = thresholds(img_np, low_threshold, high_threshold, random_threshold, r)
    return (canny(img_np, low, high)[:, :, None] / np.float32(255.0)).astype(np.float32)
