"""Where the tap-GEMM's N tile matters: every tap-GEMM shape of one eager denoise step of bench.py's workloads, timed at
each N tile.

    python tools/bench_tapgemm_wide.py [--workloads i2vgen,videolcm,sr600,higen] [--rounds 3] [--ms 30] [--out DIR]

1. Enumeration: one eager step of each workload (bench.py's build_model / Stepper recipe, random weights) under
   ops.KernelProfile; by_shape() lists every tap-GEMM shape with its launches per step and device time.
2. Per shape: the same GEMM on random inputs, with the N tile the launcher picks (bn = 0) and forced to each tile the
   plain epilogue offers, alternating all of them in every round; median and min-max of the per-launch time over the
   rounds.  GEGLU and folded-LayerNorm projections are listed but not swept (their tile is fixed at pack time or by
   another epilogue).
3. Fill rate for each (shape, tile): bytes the TMA brings into shared memory (A box + W tile per k-iteration, for every
   output tile) over the kernel time, next to the TFLOP/s: a kernel bound by L2-to-SM delivery keeps the fill rate flat
   while the TFLOP/s follows the FLOP per byte of the tile.

Prints one JSON line per shape and writes everything to DIR/tapgemm_wide.json.  The card's name, power limit and maximum
SM clock go with the numbers.  Without a CUDA device it stops after parsing and checking the shape arithmetic.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

BK = 64          # K per pipeline stage (tapgemm_sm90.cu kBK)
A_BYTES = 128 * BK * 2
SWEEP_BN = (96, 128, 160, 192, 224, 256)

_TAG = [
    ("linear", re.compile(r"^linear m(\d+) k(\d+) n(\d+)(.*)$")),
    ("conv3x3", re.compile(r"^conv3x3 (\d+)x(\d+)x(\d+) c(\d+) n(\d+)$")),
    ("tconv3", re.compile(r"^tconv3 b(\d+) f(\d+) hw(\d+) c(\d+) n(\d+)$")),
]


def parse_tag(tag):
    """'linear m.. k.. n..[ geglu][ res][ ln]' / 'conv3x3 NxHxW c.. n..' / 'tconv3 b.. f.. hw.. c.. n..' -> dict or None."""
    for kind, rx in _TAG:
        m = rx.match(tag)
        if not m:
            continue
        g = m.groups()
        if kind == "linear":
            flags = g[3].split()
            return dict(kind=kind, m=int(g[0]), k=int(g[1]), n=int(g[2]), geglu="geglu" in flags, res="res" in flags,
                        ln="ln" in flags)
        if kind == "conv3x3":
            return dict(kind=kind, nimg=int(g[0]), h=int(g[1]), w=int(g[2]), c=int(g[3]), n=int(g[4]))
        return dict(kind=kind, b=int(g[0]), f=int(g[1]), hw=int(g[2]), c=int(g[3]), n=int(g[4]))
    return None


def _pick_box(d1, d2):
    """api_tapgemm.cu pick_box: the (box1, box2) output tile (<= 128 positions) that wastes the fewest MMA rows."""
    best, bb = -1.0, (1, 1)
    for x in range(min(d1, 128), 0, -1):
        y = min(128 // x, d2, 256)
        tiles = math.ceil(d1 / x) * math.ceil(d2 / y)
        eff = d1 * d2 / (tiles * 128.0)
        if eff > best + 1e-9:
            best, bb = eff, (x, y)
    return bb


def geometry(s):
    """(m_tiles, rows per A box, k_iters, flop) of a parsed shape, as the launcher tiles it."""
    if s["kind"] == "linear":
        return math.ceil(s["m"] / 128), min(s["m"], 128), s["k"] // BK, 2.0 * s["m"] * s["n"] * s["k"]
    if s["kind"] == "conv3x3":
        b1, b2 = _pick_box(s["w"], s["h"])
        mt = s["nimg"] * math.ceil(s["w"] / b1) * math.ceil(s["h"] / b2)
        return mt, b1 * b2, 9 * s["c"] // BK, 2.0 * s["nimg"] * s["h"] * s["w"] * s["n"] * 9 * s["c"]
    hw, f = s["hw"], s["f"]
    b1 = min(hw, 128)
    b2 = min(128 // hw, f) if hw < 128 else 1
    mt = s["b"] * math.ceil(f / b2) * math.ceil(hw / b1)
    return mt, b1 * b2, 3 * s["c"] // BK, 2.0 * s["b"] * f * hw * s["n"] * 3 * s["c"]


def fill_bytes(s, bn):
    """Bytes the TMA lands in shared memory for the whole GEMM at N tile bn (zero-filled rows count: they are written)."""
    mt, rows, kit, _ = geometry(s)
    return mt * math.ceil(s["n"] / bn) * kit * (rows * BK * 2 + bn * BK * 2)


def sweepable(s):
    return s["kind"] != "linear" or not (s["geglu"] or s["ln"])


def make_call(s, dev, ops):
    """Random inputs of the shape and a function bn -> one launch of the same GEMM with that N tile."""
    g = torch.Generator(device=dev).manual_seed(7)
    rnd = lambda *sh: torch.randn(*sh, generator=g, device=dev)   # noqa: E731
    n = s["n"]
    bias = rnd(n)
    if s["kind"] == "linear":
        a = rnd(s["m"], s["k"]).half()
        w = (rnd(n, s["k"]) * s["k"] ** -0.5).half()
        r = rnd(s["m"], n).half() if s["res"] else None
        out = torch.empty(s["m"], n, device=dev, dtype=torch.float16)
        return lambda bn: ops.linear(a, w, bias=bias, residual=r, out=out, bn=bn)
    if s["kind"] == "conv3x3":
        x = rnd(s["nimg"], s["h"], s["w"], s["c"]).half()
        w = (rnd(n, 9 * s["c"]) * (9 * s["c"]) ** -0.5).half()
        out = torch.empty(s["nimg"], s["h"], s["w"], n, device=dev, dtype=torch.float16)
        return lambda bn: ops.conv2d_3x3(x, w, bias=bias, out=out, bn=bn)
    x = rnd(s["b"], s["f"], s["hw"], s["c"]).half()
    w = (rnd(n, 3 * s["c"]) * (3 * s["c"]) ** -0.5).half()
    out = torch.empty(s["b"], s["f"], s["hw"], n, device=dev, dtype=torch.float16)
    return lambda bn: ops.tconv3(x, w, bias=bias, out=out, bn=bn)


def time_launch(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def enumerate_step(wl_key, dev):
    """{tag: {launches, ms}} of the tap-GEMM launches of one eager denoise step of the workload."""
    import bench
    from vgen_b200 import ops, registry
    wl = bench.WORKLOADS[wl_key]
    model_reg, diff_reg, _ = registry.register(force_local=True)
    model = bench.build_model(wl, model_reg, 0, dev)
    cond = bench.synth_conditioning(wl, 8888, dev)
    stepper = bench.Stepper(wl_key, model, dev, cond, diff_reg)
    xt = cond["noise"].clone()
    xt = stepper.step(xt, 0)          # warm: packs the weights, loads the modules
    torch.cuda.synchronize()
    ops.PROF = ops.KernelProfile()
    stepper.step(xt, 1)
    shapes = ops.PROF.by_shape()
    ops.PROF = None
    del model, stepper, cond, xt
    torch.cuda.empty_cache()
    return {k.split(":", 1)[1]: {"launches": v["launches"], "ms": v["ms"]} for k, v in shapes.items()
            if k.startswith("tapgemm:")}


def sweep(shapes, dev, rounds, window_ms):
    from vgen_b200 import ops
    rows = []
    for tag, st in sorted(shapes.items(), key=lambda kv: -kv[1]["ms"]):
        s = parse_tag(tag)
        row = dict(tag=tag, launches=st["launches"], step_ms=round(st["ms"], 3))
        if s is None or not sweepable(s) or s["n"] <= 96:   # n <= 96: one tile of ceil(n / 32) * 32, nothing to choose
            rows.append(row)
            print(json.dumps(row), flush=True)
            continue
        fn = make_call(s, dev, ops)
        bns = [0] + [bn for bn in SWEEP_BN if bn < s["n"] + 32]
        for bn in bns:
            fn(bn)
        torch.cuda.synchronize()
        one = time_launch(lambda: fn(0), 3)
        reps = max(3, int(window_ms / max(one, 1e-3)))
        t = {bn: [] for bn in bns}
        for r in range(rounds):
            for bn in (bns if r % 2 == 0 else bns[::-1]):
                t[bn].append(time_launch(lambda: fn(bn), reps))
        _, _, _, flop = geometry(s)
        res = {}
        for bn in bns:
            med = statistics.median(t[bn])
            ent = {"ms": round(med, 4), "min": round(min(t[bn]), 4), "max": round(max(t[bn]), 4),
                   "tflops": round(flop / med / 1e9, 1)}
            if bn:
                ent["fill_tbs"] = round(fill_bytes(s, bn) / med / 1e9, 2)
                ent["flop_per_fill_byte"] = round(flop / fill_bytes(s, bn), 1)
            res[str(bn)] = ent
        best = min((bn for bn in bns if bn), key=lambda b: res[str(b)]["ms"])
        row.update(flop=flop, reps=reps, by_bn=res, best_bn=best,
                   pick_vs_best=round(res["0"]["ms"] / res[str(best)]["ms"], 4))
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="i2vgen,videolcm,sr600,higen")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ms", type=float, default=30.0, help="timing window per (shape, tile, round)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    # the shape arithmetic, checked without a device
    s = parse_tag("conv3x3 32x22x40 c1280 n1280")
    assert s and geometry(s)[2] == 9 * 1280 // BK and parse_tag("linear m28160 k1280 n1280 res")["res"]
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: nothing to time", "parsed": s, "geometry": geometry(s)}))
        return 1
    dev = torch.device("cuda", 0)
    result = {"card": card(), "rounds": args.rounds, "workloads": {}}
    print(json.dumps({"card": result["card"]}), flush=True)
    for wl in args.workloads.split(","):
        shapes = enumerate_step(wl, dev)
        print(json.dumps({"workload": wl, "tapgemm_shapes": len(shapes),
                          "tapgemm_ms": round(sum(v["ms"] for v in shapes.values()), 2)}), flush=True)
        result["workloads"][wl] = sweep(shapes, dev, args.rounds, args.ms)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "tapgemm_wide.json"), "w") as f:
            json.dump(result, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
