"""Time the depth annotator (MiDaS v3 DPT-Large) the way the VideoComposer engines call it: a 16-frame video as 8 calls of
n = 2 frames (chunk_size 2), input fp16 channels_last, at 448 x 256 (cfg.resolution) and 896 x 512.

    python tools/bench_depth.py [--rounds 3] [--window 1.0] [--out results.json]

Native (vgen_b200.midas_v3, CUDA-graphed) against the oracle in fp16 channels_last (oracle/depth_oracle.py, the engines'
arithmetic in PyTorch), with synthetic full-size weights (tests/_depth.full_state_dict).  Each round times each side over
a window of at least --window seconds, the sides alternating; the medians over rounds are reported as ms per video and as
TFLOP/s from the FLOP count of one video (torch.utils.flop_counter on the oracle, on meta tensors).  Outputs are compared
at the timed sizes against the fp32 oracle (TF32 off).  The card's name, power limit and max SM clock are read in the
same run.
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

import _depth as dp  # noqa: E402
from oracle import depth_oracle  # noqa: E402
from vgen_b200.depth import MiDaS  # noqa: E402

FRAMES, CHUNK = 16, 2
SHAPES = [(256, 448), (512, 896)]


def video_flops(H, W):
    """FLOPs of one 16-frame video through the reference arithmetic (counted on meta tensors)."""
    from torch.utils.flop_counter import FlopCounterMode
    sd = {k: torch.empty(s, device="meta") for k, s in dp.product_spec(dp.FULL)}
    with FlopCounterMode(display=False) as fc:
        depth_oracle.midas_forward(sd, torch.empty(1, 3, H, W, device="meta"), **dp.oracle_kw(dp.FULL))
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
        raise SystemExit("bench_depth needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.set_grad_enabled(False)
    dev = torch.device("cuda")
    sd = dp.full_state_dict(dp.load_spec(os.path.join(ROOT, "tests", "golden"), "full"))
    m = MiDaS(**dp.FULL)
    m.load_state_dict(sd, strict=True)
    m = m.eval().requires_grad_(False).to(memory_format=torch.channels_last).half().to(dev)
    sd16 = depth_oracle._params(sd, True, dev)         # the engine's module state: fp16, 4-D weights channels_last
    sd32 = {k: v.to(dev) for k, v in sd.items()}
    kw = dp.oracle_kw(dp.FULL)
    native = lambda x: m(x)                                                            # noqa: E731
    oracle = lambda x: depth_oracle.midas_forward(sd16, x, half=True, **kw)             # noqa: E731
    res = {"card": card(), "frames": FRAMES, "chunk": CHUNK, "rounds": a.rounds, "window_s": a.window, "shapes": {}}
    for H, W in SHAPES:
        chunks = [dp.make_input(CHUNK, H, W, 100 + i).to(dev).half().contiguous(memory_format=torch.channels_last)
                  for i in range(FRAMES // CHUNK)]
        for fn in (native, oracle):                      # warm-up: pack, capture, cuDNN algorithm choice
            for _ in range(2):
                for c in chunks:
                    fn(c)
        times = {"native": [], "oracle_fp16": []}
        for _ in range(a.rounds):
            times["native"].append(_time(native, chunks, a.window))
            times["oracle_fp16"].append(_time(oracle, chunks, a.window))
        flops = video_flops(H, W)
        x32 = chunks[0].float().contiguous()
        truth = depth_oracle.midas_forward(sd32, x32, **kw).float()
        mine, yard = native(chunks[0]), oracle(chunks[0])
        r = {"tflop_per_video": flops / 1e12}
        for k, v in times.items():
            med = statistics.median(v)
            r[k] = {"ms_per_video": med, "rounds_ms": v, "tflops": flops / (med * 1e-3) / 1e12}
        r["speedup"] = r["oracle_fp16"]["ms_per_video"] / r["native"]["ms_per_video"]
        r["rel_l2_vs_fp32"] = {"native": rel_l2(mine, truth), "oracle_fp16": rel_l2(yard, truth),
                               "native_vs_oracle_fp16": rel_l2(mine, yard)}
        r["positive_share"] = float((truth > 0).float().mean())
        res["shapes"][f"{W}x{H}"] = r
        print(f"[bench_depth] {W}x{H}: native {r['native']['ms_per_video']:.1f} ms/video "
              f"({r['native']['tflops']:.0f} TFLOP/s), oracle fp16 {r['oracle_fp16']['ms_per_video']:.1f} ms/video "
              f"({r['oracle_fp16']['tflops']:.0f} TFLOP/s), x{r['speedup']:.2f}; rel-L2 vs fp32 {r['rel_l2_vs_fp32']}",
              flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
