"""The VideoComposer canny annotator on the device: a drop-in for tools/annotator/canny/__init__.py `CannyDetector`, and
`canny_video` for whole videos.

The reference copies each frame to the host, runs cv2.convertScaleAbs, np.median and cv2.Canny there, and copies the map
back.  Here the frames stay where they are: one call quantises them, takes each frame's median from a histogram,
computes its thresholds in float64, runs Sobel, non-maximum suppression and hysteresis (connected-component labelling),
and writes the maps (csrc/canny.cu, `vgen_canny`).  Nothing is read back to the host.

The thresholds follow the reference exactly, including its use of numpy's global stream: with both thresholds None and
`random_threshold` not `False`, every frame draws one `np.random.uniform(0.1, 0.4)`, in the order the reference would
draw them.  There is no CPU fallback: CPU tensors raise `VgenError`.
"""
from __future__ import annotations

import math
import numbers

import numpy as np
import torch

from . import lib as _l
from . import ops


def threshold_plan(n, low_threshold=None, high_threshold=None, random_threshold=True):
    """(mode, r, low, high) of ops.canny for n frames: r is the list of the reference's np.random.uniform(0.1, 0.4) draws,
    one per frame in order, when it would draw (mode 2), else None."""
    if low_threshold is None and high_threshold is None:
        if random_threshold is False:                      # the reference tests identity with False
            return 1, None, 0.0, 0.0
        return 2, [np.random.uniform(0.1, 0.4) for _ in range(n)], 0.0, 0.0
    if low_threshold is None or high_threshold is None:
        raise ValueError("canny: give both thresholds or neither")
    for t in (low_threshold, high_threshold):
        if isinstance(t, bool) or not isinstance(t, numbers.Real) or math.isnan(t):
            raise ValueError(f"canny: thresholds must be real numbers, got {t!r}")
    return 0, None, float(low_threshold), float(high_threshold)


def _run(frames, out, low_threshold, high_threshold, random_threshold):
    mode, r, low, high = threshold_plan(frames.shape[0], low_threshold, high_threshold, random_threshold)
    rand = None
    if r is not None:                                      # pinned, so the upload is asynchronous
        rand = torch.tensor(r, dtype=torch.float64).pin_memory().to(frames.device, non_blocking=True)
    return ops.canny(frames, mode, rand, low, high, out=out)


class CannyDetector:
    """`CannyDetector()(img, low_threshold=None, high_threshold=None, random_threshold=True)` as the reference: img is a
    CUDA fp32 tensor (h, w, c) in [0, 1] (c = 1 or 3; quantised as cv2.convertScaleAbs(img * 255.)) or a uint8
    np.ndarray (h, w) / (h, w, c) taken as it is.  Returns the edge map as a CUDA fp32 tensor (h, w, 1) of 0.0 / 1.0."""

    def __call__(self, img, low_threshold=None, high_threshold=None, random_threshold=True):
        if isinstance(img, torch.Tensor):
            if not img.is_cuda or img.dtype != torch.float32:
                raise _l.VgenError(f"CannyDetector: expected a CUDA fp32 tensor, got {img.dtype} on {img.device}")
            if img.dim() != 3 or img.shape[2] not in (1, 3):
                raise ValueError(f"CannyDetector: expected an (h, w, c) tensor with c = 1 or 3, got {tuple(img.shape)}")
            frames = img.permute(2, 0, 1).unsqueeze(0)
        elif isinstance(img, np.ndarray):
            if img.dtype != np.uint8 or img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] not in (1, 3)):
                raise ValueError(f"CannyDetector: expected a uint8 (h, w) or (h, w, c) array with c = 1 or 3, got "
                                 f"{img.dtype} {img.shape}")
            a = img if img.ndim == 3 else img[:, :, None]
            frames = torch.from_numpy(np.ascontiguousarray(a)).cuda().permute(2, 0, 1).unsqueeze(0)
        else:
            raise ValueError(f"CannyDetector: expected a torch.Tensor or np.ndarray, got {type(img).__name__}")
        h, w = frames.shape[2:]
        out = torch.empty(h, w, 1, device=frames.device, dtype=torch.float32)
        return _run(frames, out, low_threshold, high_threshold, random_threshold)


def canny_video(frames, low_threshold=None, high_threshold=None, random_threshold=True):
    """The canny condition of videos: frames CUDA fp32 [b, f, c, h, w] in [0, 1] (c = 1 or 3) -> fp32 [b, 1, f, h, w] of
    0.0 / 1.0, equal to stacking CannyDetector()(frames[i, j].permute(1, 2, 0), ...) over (i, j) in that order (one
    np.random draw per frame when the reference draws), in one set of launches."""
    if not isinstance(frames, torch.Tensor) or not frames.is_cuda or frames.dtype != torch.float32:
        what = f"{frames.dtype} on {frames.device}" if isinstance(frames, torch.Tensor) else type(frames).__name__
        raise _l.VgenError(f"canny_video: expected a CUDA fp32 tensor, got {what}")
    if frames.dim() != 5 or frames.shape[2] not in (1, 3):
        raise ValueError(f"canny_video: expected [b, f, c, h, w] with c = 1 or 3, got {tuple(frames.shape)}")
    b, f, _, h, w = frames.shape
    out = torch.empty(b, 1, f, h, w, device=frames.device, dtype=torch.float32)
    return _run(frames.flatten(0, 1), out, low_threshold, high_threshold, random_threshold)
