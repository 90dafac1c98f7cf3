"""Time the sketch annotators the way the VideoComposer engines call them: a 16-frame video as 8 chunks of n = 2 frames,
each `sketch = pidinet(misc_imgs.sub(pidi_mean).div_(pidi_std)); sketch = 1.0 - cleaner(1.0 - sketch)` in fp32, at
448 x 256 (cfg.resolution) and 896 x 512.

    python tools/bench_sketch.py [--rounds 3] [--window 1.0] [--out results.json]

Native (vgen_b200.sketch, CUDA-graphed) against the oracle in fp32 with cuDNN's TF32 convolutions (oracle/sketch_oracle.py,
the engines' arithmetic in PyTorch), with synthetic full-size weights (tests/_sketch.full_state_dict).  PiDiNet (with the
engine's normalisation) and the cleaner (with the engine's 1 - x on both sides) are timed separately; each round times each
side over a window of at least --window seconds, the sides alternating.  Medians over rounds are reported as ms per video
and as TFLOP/s from the FLOP count of one video (torch.utils.flop_counter on the oracle, on meta tensors).  Outputs are
compared at the timed sizes against the fp32 oracle (TF32 off).  The card's name, power limit and max SM clock are read in
the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

import _sketch as sk  # noqa: E402
from oracle import sketch_oracle  # noqa: E402
from vgen_b200.sketch import pidinet_bsd, sketch_simplification_gan  # noqa: E402

FRAMES, CHUNK = 16, 2
SHAPES = [(256, 448), (512, 896)]
PIDI_MEAN, PIDI_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def video_flops(net, H, W):
    from torch.utils.flop_counter import FlopCounterMode
    which = "pidinet_full" if net == "pidinet" else "cleaner"
    sd = {k: torch.empty(s, device="meta") for k, s in sk.product_spec(which)}
    with FlopCounterMode(display=False) as fc:
        if net == "pidinet":
            sketch_oracle.pidinet_forward(sd, torch.empty(1, 3, H, W, device="meta"))
        else:
            sketch_oracle.cleaner_forward(sd, torch.empty(1, 1, H, W, device="meta"), sk.GAN_MEAN, sk.GAN_STD)
    return fc.get_total_flops() * FRAMES


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _time(fn, chunks, window):
    torch.cuda.synchronize()
    t0, videos = time.perf_counter(), 0
    while True:
        for c in chunks:
            fn(c)
        videos += 1
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= window:
            return 1e3 * dt / videos


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sketch needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    gold = os.path.join(ROOT, "tests", "golden")
    sp = sk.full_state_dict(sk.load_spec(gold, "pidinet_full"), "pidinet")
    sc = sk.full_state_dict(sk.load_spec(gold, "cleaner"), "cleaner")
    p, c = pidinet_bsd(), sketch_simplification_gan()
    p.load_state_dict(sp, strict=True)
    c.load_state_dict(sc, strict=True)
    p, c = (m.eval().requires_grad_(False).to(dev) for m in (p, c))
    sp, sc = ({k: v.to(dev) for k, v in d.items()} for d in (sp, sc))
    mean = torch.tensor(PIDI_MEAN, device=dev).view(1, 3, 1, 1)
    std = torch.tensor(PIDI_STD, device=dev).view(1, 3, 1, 1)

    def tf32(flag, fn):
        def run(x):
            torch.backends.cudnn.allow_tf32 = flag
            return fn(x)
        return run

    sides = {
        "pidinet": {"native": tf32(False, lambda x: p(x.sub(mean).div_(std))),
                    "oracle_tf32": tf32(True, lambda x: sketch_oracle.pidinet_forward(sp, x.sub(mean).div_(std)))},
        "cleaner": {"native": tf32(False, lambda s: 1.0 - c(1.0 - s)),
                    "oracle_tf32": tf32(True, lambda s: 1.0 - sketch_oracle.cleaner_forward(sc, 1.0 - s, sk.GAN_MEAN, sk.GAN_STD))},
    }
    truth_fn = {"pidinet": tf32(False, lambda x: sketch_oracle.pidinet_forward(sp, x.sub(mean).div_(std))),
                "cleaner": tf32(False, lambda s: 1.0 - sketch_oracle.cleaner_forward(sc, 1.0 - s, sk.GAN_MEAN, sk.GAN_STD))}
    res = {"card": card(), "frames": FRAMES, "chunk": CHUNK, "rounds": a.rounds, "window_s": a.window, "shapes": {}}
    for H, W in SHAPES:
        frames = [(sk.make_input("pidinet", CHUNK, H, W, 100 + i).to(dev) * std + mean).clamp_(0, 1)
                  for i in range(FRAMES // CHUNK)]
        sketches = [truth_fn["pidinet"](f) for f in frames]      # the cleaner's input: the engine's PiDiNet output
        out = {}
        for net, chunks in (("pidinet", frames), ("cleaner", sketches)):
            for fn in sides[net].values():                          # warm-up: pack, capture, cuDNN algorithm choice
                for _ in range(2):
                    for ch in chunks:
                        fn(ch)
            times = {k: [] for k in sides[net]}
            for _ in range(a.rounds):
                for k, fn in sides[net].items():
                    times[k].append(_time(fn, chunks, a.window))
            flops = video_flops(net, H, W)
            truth = truth_fn[net](chunks[0]).float()
            r = {"tflop_per_video": flops / 1e12}
            for k, v in times.items():
                med = statistics.median(v)
                r[k] = {"ms_per_video": med, "rounds_ms": v, "tflops": flops / (med * 1e-3) / 1e12}
            r["speedup"] = r["oracle_tf32"]["ms_per_video"] / r["native"]["ms_per_video"]
            r["rel_l2_vs_fp32"] = {k: rel_l2(fn(chunks[0]), truth) for k, fn in sides[net].items()}
            out[net] = r
            print(f"[bench_sketch] {W}x{H} {net}: native {r['native']['ms_per_video']:.1f} ms/video "
                  f"({r['native']['tflops']:.0f} TFLOP/s), oracle TF32 {r['oracle_tf32']['ms_per_video']:.1f} ms/video "
                  f"({r['oracle_tf32']['tflops']:.0f} TFLOP/s), x{r['speedup']:.2f}; rel-L2 vs fp32 {r['rel_l2_vs_fp32']}; "
                  f"rounds {times}", flush=True)
        res["shapes"][f"{W}x{H}"] = out
    torch.backends.cudnn.allow_tf32 = True
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
