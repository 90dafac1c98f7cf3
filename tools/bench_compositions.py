"""Time the VideoComposer condition path of UNetSD_TFT2V at the released shape (configs/tft2v_vcomposer_infer.yaml:
16 frames, 448 x 256, six spatial conditions + image tokens) with a CFG batch (b = 2), on the GPU.

    python tools/bench_compositions.py [--window 1.0] [--repeats 5] [--json OUT]

Reports, with the card's name and power limit read in the same run:
  1. the six spatial encoders of one forward: the fused ops.cond_stem chain against the same chain with the stem composed
     from existing ops (cp_to_pc to 8 channels -> 72-wide im2col -> GEMM -> adaptive_avgpool with SiLU);
  2. the UNet forward (CUDA-graphed) with and without the conditions;
  3. cond_stem's achieved bytes/s (one read of the condition, one write of the pooled map) against the H100 SXM data
     sheet's 3.35 TB/s HBM3 bandwidth.
Every variant is warmed up, timed over windows of at least --window seconds with CUDA events, and the variants alternate
for --repeats rounds; the median and the spread are printed.  Synthetic weights (oracle/synth.py); nothing is written
into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

from oracle import synth  # noqa: E402
from vgen_b200 import arch, ops  # noqa: E402
from vgen_b200.unet import _pack_conv3x3  # noqa: E402
import _vcomp as vc  # noqa: E402

HBM_DATASHEET = 3.35e12   # bytes/s, NVIDIA H100 SXM data sheet


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        dev = torch.cuda.current_device()
        return q[dev] if dev < len(q) else (q[0] if q else "unknown")
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (power limit unreadable: {e})"


def _time(fn, window):
    """Mean ms per call over a window of at least `window` seconds (CUDA events)."""
    fn()
    torch.cuda.synchronize()
    n = 1
    while True:
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        e.synchronize()
        ms = s.elapsed_time(e)
        if ms >= window * 1e3:
            return ms / n
        n = max(n * 2, int(n * window * 1e3 * 1.2 / max(ms, 1e-3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_compositions: no CUDA device")
    torch.set_grad_enabled(False)
    card = _card()
    print(f"card: {card}")

    case = dict(vc.FULL_VCOMP_CASES["full_vcomposer"], b=2, t=[721, 721])       # the CFG pair as one batch
    spec = vc.load_spec(os.path.join(ROOT, "tests", "golden"), "full_vcomposer", vc.FULL_VCOMP_CASES)
    m = vc.build_product(case)
    m.load_state_dict(synth.state_dict(spec, seed=case["seed"]), strict=True)
    m = m.cuda().eval()
    inp = {k: v.cuda() for k, v in vc.make_inputs(case).items()}
    kw = vc.call_kwargs(case, inp)
    W = m._packed or m._pack()
    b, f, h, w = case["b"], case["f"], case["h"], case["w"]
    oh, ow = case["resolution"][1] // 2, case["resolution"][0] // 2
    spatial = [k for k in arch.VCOMP_SUM_ORDER if k in case["conds"]]

    # baseline stem weights: [32, 9*8] packed for im2col + GEMM
    base_w = {k: _pack_conv3x3(W[m._spatial[k][0] + "0.w"].cpu(), "cuda", cin_pad=8) for k in spatial}

    def stem_base(k):
        v = kw[k]
        _, cin, _, H, Wd = v.shape
        x8 = ops.cp_to_pc(v.contiguous(), b, cin, f * H * Wd, c_pad=8).view(b * f, H, Wd, 8)
        wt = base_w[k]
        col = ops.im2col(x8, 3, 3, 1, 1, 1, H, Wd, wt.shape[1])
        y = ops.linear(col, wt, bias=W[m._spatial[k][0] + "0.b"]).view(b * f, H, Wd, wt.shape[0])
        return ops.adaptive_avgpool(y, oh, ow, silu_in=True)

    def stem_fused(k):
        enc = m._spatial[k][0]
        return ops.cond_stem(kw[k], W[enc + "0.w"], W[enc + "0.b"], oh, ow)

    def encoders(stem):
        def run():
            for k in spatial:
                enc, after, _ = m._spatial[k]
                s = m._conv3x3_s2(stem(k), W, enc + "3.")
                s = m._conv3x3_s2(s, W, enc + "5.", act_silu=True)
                m._frame_transformer(s, W, after, b, f)
        return run

    def stems_only():
        for k in spatial:
            stem_fused(k)

    # the two stems compute the same map (the baseline rounds the full-resolution conv output to fp16 once more)
    for k in spatial:
        d = (stem_fused(k).float() - stem_base(k).float()).norm() / stem_base(k).float().norm()
        assert float(d) < 2e-3, (k, float(d))

    xin, tin = inp["x"], inp["t"]
    bare = {"y": kw["y"]}
    variants = {
        "encoders_fused": encoders(stem_fused),
        "encoders_baseline": encoders(stem_base),
        "unet_with_conditions": lambda: m(xin, tin, **kw),
        "unet_without_conditions": lambda: m(xin, tin, **bare),
        "cond_stem_x6": stems_only,
    }
    for fn in variants.values():          # warm-up: packs, sets attributes, captures the graphs
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.repeats):
        for k, fn in variants.items():
            times[k].append(_time(fn, args.window))

    stem_bytes = sum(kw[k].numel() * kw[k].element_size() + b * f * oh * ow * 32 * 2 for k in spatial)
    res = {"card": card, "shape": dict(b=b, f=f, H=case["H"], W=case["W"], latent=[h, w], conditions=spatial),
           "ms": {k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()}}
    stem_ms = res["ms"]["cond_stem_x6"]["median"]
    res["cond_stem_bytes"] = stem_bytes
    res["cond_stem_bytes_per_s"] = stem_bytes / (stem_ms * 1e-3)
    res["cond_stem_fraction_of_datasheet_hbm"] = res["cond_stem_bytes_per_s"] / HBM_DATASHEET
    for k, v in res["ms"].items():
        print(f"{k:26s} median {v['median']:9.3f} ms  (min {v['min']:.3f}, max {v['max']:.3f}, {args.repeats} alternating rounds)")
    print(f"cond_stem: {stem_bytes / 1e6:.1f} MB per forward in {stem_ms:.3f} ms = {res['cond_stem_bytes_per_s'] / 1e12:.2f} TB/s "
          f"({100 * res['cond_stem_fraction_of_datasheet_hbm']:.1f}% of the data sheet's 3.35 TB/s)")
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
