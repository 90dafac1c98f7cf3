"""Time UNetSD_LoRA's runtime LoRA against the merged model at InstructVideo's eval shape: the released UNet (rank-4 LoRA on
the 66 attentions), the CFG pair as one batch of 2, 16 frames, 32 x 32 latent, 77 tokens, synthetic weights (LoRA up
weights non-zero), CUDA-graphed forwards.

    python tools/bench_lora.py [--repeats 5] [--iters 5] [--json OUT]

Variants (one model each, same weights):
  merged         the default: the LoRA folded into the weights at pack time
  runtime_1      runtime mode, the model's own set at strength 1
  runtime_cfg    runtime mode, per-branch strengths [1, 0] (tuned conditional, base unconditional branch)
  runtime_2sets  runtime mode, the own set and a second rank-4 set at [1, 0.5]
  composed       the same LoRA from existing ops: projection GEMM, a linear down projection, a linear up projection taking
                 the projection's output as its residual (strength 1, alpha / rank folded into the down weights)
Each round times --iters forwards of every variant in alternating order; medians and spreads over --repeats rounds are
printed with the card's name and power limit read in the same run.  Also timed: what a strength change costs in merged
mode (merged_state_dict and the re-pack).  Nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

import torch  # noqa: E402

from vgen_b200 import ops  # noqa: E402
from bench_compositions import _card  # noqa: E402
import _instructvideo as iv  # noqa: E402
from _lora_runtime import lora_pairs  # noqa: E402


def _composed_lora_linear(self, x, W, key, lo, **kw):
    """The LoRA of one projection from existing ops (strength 1): y = proj(x); y + U (D x) with D pre-scaled and padded."""
    c = self._composed.get(key)
    if c is None:
        d = torch.zeros(lo["rpad"], lo["d"].shape[1], device=x.device, dtype=torch.float32)
        d[:lo["d"].shape[0]] = lo["d"].float() * lo["scale"][:, None]
        c = self._composed[key] = d.half()
    y = ops.linear(x, W[key], **kw)
    return ops.linear(ops.linear(x, c), lo["u"], residual=y)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lora: no CUDA device")
    torch.set_grad_enabled(False)
    card = _card()
    print(f"card: {card}")
    golden = os.path.join(ROOT, "tests", "golden")
    case = iv.FULL_IV_CASES["full_iv_lora"]
    sd = iv.weights(iv.load_spec(golden, "full_iv_lora", iv.FULL_IV_CASES), case["seed"])
    second = lora_pairs(case["ctor"], seed=91)

    def model():
        m = iv.build_product(case)
        m.load_state_dict(sd, strict=True)
        return m.cuda().eval().offload_masters()

    inp = {k: v.cuda() for k, v in iv.make_inputs(case).items()}
    x, t, y = torch.cat([inp["x"]] * 2), torch.cat([inp["t"]] * 2), torch.cat([inp["y"], inp["y_neg"]])
    models = {name: model() for name in ("merged", "runtime_1", "runtime_cfg", "runtime_2sets", "composed")}
    models["runtime_2sets"].add_lora("second", second)
    comp = models["composed"]
    comp._composed = {}
    comp._lora_linear = types.MethodType(_composed_lora_linear, comp)
    cfg = torch.tensor([1.0, 0.0], device="cuda")
    calls = {
        "merged": lambda: models["merged"](x, t, y),
        "runtime_1": lambda: models["runtime_1"](x, t, y, lora_strength=1.0),
        "runtime_cfg": lambda: models["runtime_cfg"](x, t, y, lora_strength=cfg),
        "runtime_2sets": lambda: models["runtime_2sets"](x, t, y, lora_strength=torch.tensor([[1.0, 0.5]] * 2, device="cuda")),
        "composed": lambda: models["composed"](x, t, y, lora_strength=1.0),
    }
    outs = {}
    for k, fn in calls.items():       # eager (packs), capture, replay
        for _ in range(3):
            outs[k] = fn()
    torch.cuda.synchronize()
    rel = lambda a, b: float((a.float() - b.float()).norm() / b.float().norm())  # noqa: E731
    agree = {k: rel(outs[k], outs["merged"]) for k in ("runtime_1", "composed")}
    print(f"rel L2 against merged: {agree}")
    times = {k: [] for k in calls}
    for r in range(args.repeats):
        order = list(calls) if r % 2 == 0 else list(calls)[::-1]
        for k in order:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            for _ in range(args.iters):
                calls[k]()
            e.record()
            torch.cuda.synchronize()
            times[k].append(s.elapsed_time(e) / args.iters)
    # a strength change in merged mode: merge on the host, re-pack the arena (the graphs are dropped with it)
    m = models["merged"]
    repack = []
    for i in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.lora_scale = 1.0 + 0.5 * (i + 1)
        m.invalidate_packed()
        m._pack()
        torch.cuda.synchronize()
        repack.append((time.perf_counter() - t0) * 1e3)
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"card": card, "workload": dict(batch=2, frames=case["f"], latent=[case["h"], case["w"]], tokens=case["ntok"], rank=4),
           "ms_per_forward": {k: dict(median=med[k], min=min(v), max=max(v), runs=v) for k, v in times.items()},
           "overhead_vs_merged_pct": {k: 100.0 * (med[k] / med["merged"] - 1) for k in med if k != "merged"},
           "merged_strength_change_ms": dict(median=statistics.median(repack), runs=repack),
           "rel_l2_vs_merged": agree}
    for k, v in res["ms_per_forward"].items():
        print(f"{k:14s} median {v['median']:8.2f} ms/forward (min {v['min']:.2f}, max {v['max']:.2f}; "
              f"{args.repeats} alternating rounds of {args.iters})")
    print(f"merged-mode strength change (merge + re-pack): median {res['merged_strength_change_ms']['median']:.0f} ms")
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
