"""Time the DreamVideo adapters of UNetSD_DreamVideo at the released shape (the joint flavour of configs/dreamvideo/infer:
32 frames, 256 x 256 pixels = 32 x 32 latent, 77 tokens, y_image [b, 1, 1024]) with the CFG pair as one batch (b = 2,
ag_strength 1 / 0), on the GPU.

    python tools/bench_dreamvideo.py [--window 1.0] [--repeats 5] [--json OUT]

Reports, with the card's name and power limit read in the same run, the CUDA-graphed UNet forward
  1. with the adapters as built (down projection with GELU and condition term in one GEMM, up projection fused into the
     sublayer's output projection, one condition launch per forward);
  2. with the same adapters composed from existing ops: per adapter a linear_small for condition_linear, a broadcast copy
     and an axpy for x + lambda * condition, the down ops.linear, eltwise gelu and the up ops.linear with the residual x,
     which the sublayer's own output projection then takes as its residual;
  3. of the same weights with the adapters removed (the base flavour),
and checks that 1 and 2 agree.  Every variant is warmed up, timed over windows of at least --window seconds with CUDA
events, and the variants alternate for --repeats rounds; the median and the spread are printed.  Synthetic weights
(oracle/synth.py); nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

import torch  # noqa: E402

from oracle import synth  # noqa: E402
from vgen_b200 import arch, ops  # noqa: E402
from vgen_b200.unet import UNetSD_DreamVideo  # noqa: E402
from bench_compositions import _card, _time  # noqa: E402
import _dreamvideo as dv  # noqa: E402


class _ComposedAdapters(UNetSD_DreamVideo):
    """The same model with every adapter composed from existing ops (the measurement baseline; parallel positions only)."""

    def attach(self, sd):
        dev = torch.device("cuda")
        self._plain = {}
        for k, v in sd.items():
            for _name, mod, _i, out in arch.ADAPTER_SITES:
                if k.endswith(f".{mod}.down_linear.weight"):
                    q = k[:-len(f"{mod}.down_linear.weight")]
                    a = q + mod + "."
                    self._plain[q + mod] = {
                        "out.w": sd[q + out + "weight"].reshape(sd[q + out + "weight"].shape[0], -1).half().to(dev),
                        "out.b": sd[q + out + "bias"].float().to(dev),
                        "down.w": v.half().to(dev), "down.b": sd[a + "down_linear.bias"].float().to(dev),
                        "up.w": sd[a + "up_linear.weight"].half().to(dev), "up.b": sd[a + "up_linear.bias"].float().to(dev),
                        "cond.w": sd[a + "condition_linear.weight"].half().to(dev) if a + "condition_linear.weight" in sd else None,
                        "cond.b": sd[a + "condition_linear.bias"].float().to(dev) if a + "condition_linear.weight" in sd else None}

    def _sublayer_out(self, t, W, p, mod, out, width, hw, produce):
        pl = self._plain.get(p + mod) if W.get(p + mod) is not None else None
        if pl is None:
            return super()._sublayer_out(t, W, p, mod, out, width, hw, produce)
        x = t
        if pl["cond.w"] is not None and self._bench_cond is not None:
            c16, lams, rows_per_video = self._bench_cond
            cond = ops.linear_small(c16, pl["cond.w"], pl["cond.b"])                    # [b, C]
            x = torch.empty_like(t)
            for bi, lam in enumerate(lams):
                rows = slice(bi * rows_per_video * hw, (bi + 1) * rows_per_video * hw)
                ops.copy2d(cond[bi].view(1, -1).expand(rows_per_video * hw, -1), x[rows])    # broadcast (row stride 0)
                ops.eltwise("axpy", t[rows].contiguous(), x[rows].contiguous(), s=lam, out=x[rows])
        h = ops.eltwise("gelu", ops.linear(x, pl["down.w"], bias=pl["down.b"]))
        ad = ops.linear(h, pl["up.w"], bias=pl["up.b"], residual=t)
        return ops.linear(produce(None).view(-1, width), pl["out.w"], bias=pl["out.b"], residual=ad)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dreamvideo: no CUDA device")
    torch.set_grad_enabled(False)
    card = _card()
    print(f"card: {card}")

    case = dict(dv.FULL_DV_CASES["full_dv_joint"], b=2, t=[721, 721])
    spec = dv.load_spec(os.path.join(ROOT, "tests", "golden"), "full_dv_joint", dv.FULL_DV_CASES)
    sd = synth.state_dict(spec, seed=case["seed"])
    inp = {k: v.cuda() for k, v in dv.make_inputs(case).items()}
    b, f = case["b"], case["f"]
    y_image = inp["y_image"][:1].expand(b, -1, -1).contiguous()     # y_visual and the zero feature of the CFG pair
    y_image[1:].zero_()
    ag = torch.tensor([1.0, 0.0], device="cuda")
    kw = {"y": inp["y"], "y_image": y_image, "ag_strength": ag}

    built = dv.build_product(case)
    built.load_state_dict(sd, strict=True)
    built = built.cuda().eval()
    composed = _ComposedAdapters(**case["ctor"])
    composed.load_state_dict(sd, strict=True)
    composed = composed.cuda().eval()
    composed.attach(sd)
    composed._bench_cond = (built._to_f16_rows(y_image).view(b, -1), [1.0, 0.0], f)
    base_ctor = {k: v for k, v in case["ctor"].items() if "adapter" not in k}
    base = UNetSD_DreamVideo(**base_ctor)
    base.load_state_dict({k: v for k, v in sd.items() if "_adapter." not in k}, strict=True)
    base = base.cuda().eval()
    del sd

    x, t = inp["x"], inp["t"]
    a = built(x, t, **kw)
    c = composed(x, t, **kw)
    agree = float((a.float() - c.float()).norm() / c.float().norm())
    print(f"adapters as built vs composed from existing ops: rel-L2 {agree:.2e}")
    assert agree < 5e-3, agree

    variants = {
        "unet_adapters_built": lambda: built(x, t, **kw),
        "unet_adapters_composed": lambda: composed(x, t, **kw),
        "unet_base": lambda: base(x, t, y=kw["y"]),
    }
    for fn in variants.values():          # warm-up: packs, sets attributes, captures the graphs
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.repeats):
        for k, fn in variants.items():
            times[k].append(_time(fn, args.window))
    res = {"card": card, "shape": dict(b=b, f=f, latent=[case["h"], case["w"]], tokens=case["ntok"]),
           "adapters_built_vs_composed_rel_l2": agree,
           "ms": {k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()}}
    for k, v in res["ms"].items():
        print(f"{k:24s} median {v['median']:9.3f} ms  (min {v['min']:.3f}, max {v['max']:.3f}, {args.repeats} alternating rounds)")
    ms = {k: v["median"] for k, v in res["ms"].items()}
    print(f"adapter overhead: built {ms['unet_adapters_built'] - ms['unet_base']:.2f} ms "
          f"({100 * (ms['unet_adapters_built'] / ms['unet_base'] - 1):.1f}%), composed "
          f"{ms['unet_adapters_composed'] - ms['unet_base']:.2f} ms ({100 * (ms['unet_adapters_composed'] / ms['unet_base'] - 1):.1f}%)")
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
