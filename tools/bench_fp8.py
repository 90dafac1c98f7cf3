"""FP8 (fp8_linear=True) against fp16 UNet forwards at the BASELINE configs 2 (I2VGen-XL, 16 frames at 1280 x 704, the
CFG pair as one batch of 2) and 3 (VideoLCM, 16 frames at 448 x 256), same weights, alternating in one process.

    python tools/bench_fp8.py [--reps 5] [--iters 5] [--workloads i2vgen,videolcm]

Per workload it prints the graphed forward time of both modes (median and range over the alternating repetitions), the
speedup, the per-family kernel times of one instrumented (eager) forward of each mode, the FP8 GEMMs' achieved TFLOP/s
next to the H100 SXM data-sheet figure for dense FP8 (1979 TFLOP/s, not a measured number), the packed arena bytes, and
the FP8 output's relative L2 distance to the fp16 output.  The card's name, power limit and maximum SM clock are printed
with the numbers.  Weights are random (bench.py's build_model recipe); nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from vgen_b200 import ops, registry  # noqa: E402
from vgen_b200.diffusion import cfg_forward  # noqa: E402

FP8_DATASHEET_TFLOPS = 1979.0   # H100 SXM data sheet, dense FP8, 700 W (not measured)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def arena_bytes(m):
    return sum(t.numel() * t.element_size() for _, t in m.packed_tensors())


def forward_fn(wl, m, cond, x, t):
    if wl["kind"] == "i2vgen":
        kw = dict(image=cond["image"], local_image=cond["local_image"], fps=cond["fps"])
        pair = [dict(y=cond["y"], **kw), dict(y=cond["y_neg"], **kw)]
        return lambda: cfg_forward(m, x, t, pair)
    return lambda: m(x, t, y=cond["y"])


def time_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def families(fn):
    ops.PROF = ops.KernelProfile()
    try:
        fn()
        return ops.PROF.summary()
    finally:
        ops.PROF = None


def run(wl_key, reps, iters):
    wl = bench.WORKLOADS[wl_key]
    dev = torch.device("cuda")
    model_reg, _, _ = registry.register(force_local=True)
    models = {}
    for mode in ("fp16", "fp8"):
        m = bench.build_model(wl, model_reg, 0, dev)
        m.fp8_linear = mode == "fp8"
        m.offload_masters()
        models[mode] = m
    cond = bench.synth_conditioning(wl, 7, dev)
    x = cond["noise"]
    t = torch.tensor([751], device=dev)
    fns = {mode: forward_fn(wl, m, cond, x, t) for mode, m in models.items()}
    with torch.no_grad():
        outs = {}
        for mode, fn in fns.items():
            for _ in range(3):                     # eager + pack, capture, replay
                o = fn()
            outs[mode] = torch.cat(o) if isinstance(o, tuple) else o
        err = float((outs["fp8"].float() - outs["fp16"].float()).norm() / outs["fp16"].float().norm())
        times = {"fp16": [], "fp8": []}
        for _ in range(reps):                      # alternate the modes so drift hits both alike
            for mode in ("fp16", "fp8"):
                times[mode].append(time_ms(fns[mode], iters))
        fam = {mode: families(fn) for mode, fn in fns.items()}
    res = {"workload": wl["name"], "card": card(), "reps": reps, "iters_per_rep": iters, "fp8_vs_fp16_rel_l2": err}
    for mode in ("fp16", "fp8"):
        ts = times[mode]
        res[mode] = {"forward_ms_median": statistics.median(ts), "forward_ms_min": min(ts), "forward_ms_max": max(ts),
                     "arena_bytes": arena_bytes(models[mode]),
                     "families_ms_eager": {k: round(v["ms"], 3) for k, v in sorted(fam[mode].items(), key=lambda kv: -kv[1]["ms"])}}
    res["speedup_fp8"] = res["fp16"]["forward_ms_median"] / res["fp8"]["forward_ms_median"]
    g8 = fam["fp8"].get("tapgemm_fp8")
    if g8:
        tf = g8["flops"] / (g8["ms"] * 1e-3) / 1e12
        res["fp8_gemm"] = {"launches": g8["launches"], "ms": g8["ms"], "tflop": g8["flops"] / 1e12, "tflops": tf,
                           "share_of_datasheet_1979": tf / FP8_DATASHEET_TFLOPS}
    g16 = fam["fp16"].get("tapgemm")
    if g16:
        res["fp16_tapgemm_tflops"] = g16["flops"] / (g16["ms"] * 1e-3) / 1e12
    del models
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--workloads", default="i2vgen,videolcm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a GPU")
    for key in args.workloads.split(","):
        r = run(key, args.reps, args.iters)
        print(f"== {r['workload']} on {r['card']}")
        for mode in ("fp16", "fp8"):
            d = r[mode]
            print(f"  {mode}: forward {d['forward_ms_median']:.2f} ms (range {d['forward_ms_min']:.2f}-{d['forward_ms_max']:.2f} "
                  f"over {r['reps']} x {r['iters_per_rep']}), arena {d['arena_bytes'] / 2**30:.3f} GiB")
        print(f"  speedup fp8 / fp16: {r['speedup_fp8']:.3f}x; fp8 vs fp16 output rel L2 {r['fp8_vs_fp16_rel_l2']:.3e}")
        if "fp8_gemm" in r:
            g = r["fp8_gemm"]
            print(f"  FP8 GEMMs: {g['launches']} launches, {g['tflop']:.2f} TFLOP in {g['ms']:.2f} ms = {g['tflops']:.0f} TFLOP/s "
                  f"({100 * g['share_of_datasheet_1979']:.0f}% of the 1979 TFLOP/s data-sheet figure, dense FP8)")
        print("  per-family ms (one eager forward each): fp16", r["fp16"]["families_ms_eager"])
        print("                                          fp8 ", r["fp8"]["families_ms_eager"])
        print(json.dumps(r))


if __name__ == "__main__":
    main()
