"""Time long clips on the GPU at the 32-frame TF-T2V / DreamVideo shape: the T2V trunk (full_t2v architecture), a 32 x 32
latent, 77 tokens, and the CFG pair as one batch of 2.

    python tools/bench_longclip.py [--window 1.0] [--repeats 5] [--json OUT]

Reports, with the card's name and power limit read in the same run:
  1. the attention_temporal kernel at the top level's shape (2 x 1024 = 2048 pixels x 5 heads of 64) for
     f in 32, 48, 64, 128, 256, against PyTorch SDPA with the '(b h w) f c' permute copies (the reference's route), and
     the achieved bytes/s from the q/k/v/out bytes against the H100 SXM data sheet's 3.35 TB/s;
  2. the CUDA-graphed UNet forward and the time per frame at f in 32, 64, 128.
Attention calls are captured into a CUDA graph of --chain calls so host overhead is not timed; every variant is warmed
up, timed over windows of at least --window seconds with CUDA events, and the variants alternate for --repeats rounds;
the median and the spread are printed.  Synthetic weights (oracle/synth.py); nothing is written into the tree.
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
import torch.nn.functional as F  # noqa: E402

from oracle import synth  # noqa: E402
from oracle.cases import FULL_CASES, make_inputs  # noqa: E402
from vgen_b200 import ops  # noqa: E402
from bench_compositions import _card, _time  # noqa: E402
from _helpers import build_product  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
ATTN_FRAMES = (32, 48, 64, 128, 256)
UNET_FRAMES = (32, 64, 128)


def _graphed(fn, chain):
    """A CUDA graph of `chain` back-to-back calls of fn; returns its replay (ms per call = replay time / chain)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(chain):
            fn()

    def replay():
        g.replay()
    # the graph holds raw addresses of the tensors fn closes over, and every later capture empties the allocator's
    # cache: keep fn (and with it those tensors) alive as long as the graph can be replayed
    replay.keep = (g, fn)
    return replay


def _attention_variants(f, b=2, npix=1024, heads=5, chain=20):
    inner = heads * 64
    qkv = torch.randn(b, f, npix, 3 * inner, device="cuda").half()
    q, k, v = qkv[..., :inner], qkv[..., inner:2 * inner], qkv[..., 2 * inner:]
    out = torch.empty(b, f, npix, inner, device="cuda", dtype=torch.float16)

    def native():
        ops.attention_temporal(q, k, v, heads, 64, out=out)

    def sdpa():
        t = lambda x: x.permute(0, 2, 1, 3).reshape(b * npix, f, heads, 64).transpose(1, 2)  # noqa: E731
        o = F.scaled_dot_product_attention(t(q), t(k), t(v))
        out.copy_(o.transpose(1, 2).reshape(b, npix, f, inner).permute(0, 2, 1, 3))

    native()
    mine = out.clone()
    sdpa()
    agree = float((mine.float() - out.float()).abs().max() / out.float().abs().max())
    assert agree < 3e-3, (f, agree)
    nbytes = 4 * b * f * npix * inner * 2
    return {"native": _graphed(native, chain), "sdpa": _graphed(sdpa, chain)}, nbytes, chain, agree


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_longclip: no CUDA device")
    torch.set_grad_enabled(False)
    card = _card()
    print(f"card: {card}")
    res = {"card": card, "attention": {}, "unet": {}}

    # ---- 1. the kernel
    variants, meta = {}, {}
    for f in ATTN_FRAMES:
        vs, nbytes, chain, agree = _attention_variants(f)
        for k, fn in vs.items():
            variants[(f, k)] = fn
        meta[f] = (nbytes, chain, agree)
    times = {key: [] for key in variants}
    for _ in range(args.repeats):
        for key, fn in variants.items():
            times[key].append(_time(fn, args.window) / meta[key[0]][1])
    for f in ATTN_FRAMES:
        nbytes, _, agree = meta[f]
        row = {"bytes": nbytes, "native_vs_sdpa_max_rel": agree}
        for k in ("native", "sdpa"):
            t = times[(f, k)]
            med = statistics.median(t)
            row[k] = dict(median_us=1e3 * med, min_us=1e3 * min(t), max_us=1e3 * max(t),
                          tb_per_s=nbytes / (med * 1e-3) / 1e12)
        row["native_share_of_3.35TBps"] = row["native"]["tb_per_s"] * 1e12 / HBM_BYTES_PER_S
        row["sdpa_over_native"] = row["sdpa"]["median_us"] / row["native"]["median_us"]
        res["attention"][f] = row
        print(f"attention f{f:4d}: native {row['native']['median_us']:9.1f} us ({row['native']['tb_per_s']:.2f} TB/s, "
              f"{100 * row['native_share_of_3.35TBps']:.0f}% of 3.35), SDPA+permutes {row['sdpa']['median_us']:9.1f} us "
              f"({row['sdpa_over_native']:.2f}x)  [min/max native {row['native']['min_us']:.1f}/{row['native']['max_us']:.1f}]")
    del variants

    # ---- 2. the graphed UNet forward
    case0 = dict(FULL_CASES["full_t2v"], b=2, t=[721, 721])
    spec = [(k, tuple(s)) for k, s in json.load(open(os.path.join(ROOT, "tests", "golden", "full_t2v.spec.json")))]
    m = build_product(case0)
    m.load_state_dict(synth.state_dict(spec, seed=case0["seed"]), strict=True)
    m = m.cuda().eval()
    fwd = {}
    for f in UNET_FRAMES:
        inp = {k: v.cuda() for k, v in make_inputs(dict(case0, f=f)).items()}
        fwd[f] = (lambda inp=inp: m(inp["x"], inp["t"], y=inp["y"]))
        for _ in range(3):                 # warm-up: packs, captures the graph
            fwd[f]()
    torch.cuda.synchronize()
    ut = {f: [] for f in UNET_FRAMES}
    for _ in range(args.repeats):
        for f in UNET_FRAMES:
            ut[f].append(_time(fwd[f], args.window))
    for f in UNET_FRAMES:
        med = statistics.median(ut[f])
        res["unet"][f] = dict(median_ms=med, min_ms=min(ut[f]), max_ms=max(ut[f]), ms_per_frame=med / f)
        print(f"unet forward f{f:4d} (b=2, 32x32): median {med:9.2f} ms  ({med / f:.3f} ms/frame; "
              f"min {min(ut[f]):.2f}, max {max(ut[f]):.2f}, {args.repeats} alternating rounds)")
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
