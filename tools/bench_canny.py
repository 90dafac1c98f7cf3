"""Time the canny annotator on one 16-frame video at 448 x 256 and at 1280 x 704.

    python tools/bench_canny.py [--rounds 5] [--iters 20]

native: `canny_video` on fp32 CUDA frames [1, 16, 3, h, w] (random thresholds, seeded), timed with CUDA events over
--iters calls per round.  reference: where OpenCV is installed, the reference detector's per-frame path on the same
frames: per frame `.cpu().numpy()`, cv2.convertScaleAbs(x * 255.), np.median, np.random.uniform, cv2.Canny and the map's
copy back to the device, then the stack into [1, 1, 16, h, w]; host clock around work that ends in a device synchronise.
Each line gives the median and range over the rounds, the two maps' agreement, and the card's name, power limit and
maximum SM clock.  A time that was not taken is printed as "not measured".
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from vgen_b200.canny import canny_video  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _frames(f, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(f, 3, h // 8, w // 8, device="cuda", generator=g)
    x = torch.nn.functional.interpolate(x, size=(h, w), mode="bicubic", align_corners=False).clamp_(0, 1)
    return x[None]


def _reference_path(frames):
    import cv2
    b, f = frames.shape[:2]
    maps = []
    for i in range(b):
        for j in range(f):
            img = frames[i, j].permute(1, 2, 0).cpu().numpy()
            img_np = cv2.convertScaleAbs(img * 255.)
            m = np.median(img_np)
            low = int(max(0, (1 - np.random.uniform(0.1, 0.4)) * m))
            edge = cv2.Canny(img_np, low, 2 * low)
            maps.append(torch.from_numpy(edge.copy()).unsqueeze(-1).float().cuda() / 255.0)
    return torch.stack(maps).reshape(b, f, *maps[0].shape[:2]).unsqueeze(1)


def _stats(xs):
    return f"{np.median(xs):.3f} ms ({min(xs):.3f}-{max(xs):.3f})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_canny needs a CUDA device")
    card = _card()
    try:
        import cv2  # noqa: F401
        have_cv2 = True
    except ImportError:
        have_cv2 = False
    for w, h in ((448, 256), (1280, 704)):
        frames = _frames(16, h, w, seed=w)
        np.random.seed(0)
        canny_video(frames)                                # warm-up: module load, allocator
        torch.cuda.synchronize()
        nat, ref, agree = [], [], "not compared"
        for _ in range(a.rounds):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            np.random.seed(0)
            s.record()
            for _ in range(a.iters):
                out = canny_video(frames)
            e.record()
            e.synchronize()
            nat.append(s.elapsed_time(e) / a.iters)
            if have_cv2:
                np.random.seed(a.iters - 1)                # any seed: the agreement check below reseeds
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                _reference_path(frames)
                torch.cuda.synchronize()
                ref.append((time.perf_counter() - t0) * 1e3)
        if have_cv2:
            np.random.seed(1)
            want = _reference_path(frames)
            np.random.seed(1)
            out = canny_video(frames)
            agree = f"{int((out != want).sum())} of {out.numel()} pixels differ"
        ref_s = _stats(ref) if ref else "not measured (OpenCV is not installed)"
        speed = f", {np.median(ref) / np.median(nat):.1f}x" if ref else ""
        print(f"canny 16 frames {w}x{h}: native {_stats(nat)} per video; reference per-frame path {ref_s}{speed}; "
              f"{agree}; card: {card}", flush=True)


if __name__ == "__main__":
    main()
