"""Time the colour-palette annotator and the 'histogram' composition.

    python tools/bench_histogram.py [--rounds 5] [--iters 20] [--steps 10]

annotator: `histogram_video` on one fp32 CUDA video [1, 16, 3, h, w] at 448 x 256 and 1280 x 704 (CUDA events over
--iters calls per round), against the reference procedure: per frame `.cpu().numpy()`, then the oracle's numpy restatement
of Palette.histogram (rgb2lab, sklearn's euclidean_distances, argmin, bincount, smoothing), and the stack moved back to
the device; host clock around work that ends in a device synchronise.  Rounds alternate between the two.
UNet: the graphed full-size VideoComposer forward (tests/_vcomp.py FULL_VCOMP_CASES["full_vcomposer"], synthetic
weights) with 'histogram' added to the compositions, called with and without a histogram, in alternating rounds of
--steps forwards.  Each line gives the median and range over the rounds and the card's name, power limit and maximum SM
clock.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from vgen_b200.palette import histogram_video  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _stats(xs):
    return f"{np.median(xs):.3f} ms ({min(xs):.3f}-{max(xs):.3f})"


def _frames(f, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(f, 3, h // 8, w // 8, device="cuda", generator=g)
    return torch.nn.functional.interpolate(x, size=(h, w), mode="bicubic", align_corners=False).clamp_(0, 1)[None]


def bench_annotator(a, card):
    from oracle.palette_oracle import PaletteOracle
    ora = PaletteOracle()

    def reference(frames):
        out = [ora.histogram(frames[0, j].permute(1, 2, 0).cpu().numpy().astype(np.float64)) for j in range(frames.shape[1])]
        return torch.from_numpy(np.stack(out)).float().cuda()[None]

    for w, h in ((448, 256), (1280, 704)):
        frames = _frames(16, h, w, seed=w)
        histogram_video(frames)
        torch.cuda.synchronize()
        nat, ref = [], []
        for _ in range(a.rounds):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.iters):
                out = histogram_video(frames)
            e.record()
            e.synchronize()
            nat.append(s.elapsed_time(e) / a.iters)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            want = reference(frames)
            torch.cuda.synchronize()
            ref.append((time.perf_counter() - t0) * 1e3)
        diff = float((out - want).abs().max())
        print(f"palette histogram 16 frames {w}x{h}: native {_stats(nat)} per video; reference per-frame numpy path "
              f"{_stats(ref)}, {np.median(ref) / np.median(nat):.0f}x; max |diff| {diff:.1e} (fp32 output); card: {card}",
              flush=True)


def bench_unet(a, card):
    from oracle import synth
    from _histogram import FULL_HIST, config_of, make_inputs, call_kwargs, product_spec
    import vgen_b200
    case = FULL_HIST
    m = getattr(vgen_b200, case["cls"])(config=config_of(case), **case["ctor"], enable_histogram=True)
    m.load_state_dict(synth.state_dict(product_spec(case["cls"], case["comps"], case["resolution"], case["ctor"]),
                                       seed=case["seed"]), strict=True)
    m = m.cuda().eval()
    inp = {k: v.cuda() for k, v in make_inputs(dict(case, b=1)).items()}
    kw = call_kwargs(case, inp)
    modes = {"with histogram": kw, "without": {k: v for k, v in kw.items() if k != "histogram"}}
    with torch.no_grad():
        for k in modes.values():
            for _ in range(3):                                 # eager, capture, replay
                m(inp["x"], inp["t"], **k)
        torch.cuda.synchronize()
        times = {n: [] for n in modes}
        for _ in range(a.rounds):
            for n, k in modes.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.steps):
                    m(inp["x"], inp["t"], **k)
                e.record()
                e.synchronize()
                times[n].append(s.elapsed_time(e) / a.steps)
    res = ", ".join(f"{n} {_stats(v)}" for n, v in times.items())
    print(f"graphed full_vcomposer forward (1 x 16 x 256 x 448, compositions + 'histogram'): {res}; card: {card}",
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_histogram needs a CUDA device")
    card = _card()
    bench_annotator(a, card)
    bench_unet(a, card)


if __name__ == "__main__":
    main()
