"""Time InstructVideo's segmental HPSv2 reward per 16-frame 256 x 256 video: the native SegmentalReward.score_latents
against the reference procedure on the same GPU.

    python tools/bench_reward.py [--batches 1 8] [--frames 16] [--segments 4] [--rounds 5]

Both procedures score the same latents [b, 4, 16, 32, 32] with synthetic full-size weights (HPSv2 = open_clip ViT-H/14,
the VAE of the released configs) and the same TSN frame draw:
  native     vgen_b200.reward: decode of the selected frames only, the frame kernel, the graphed image tower, the text
             tower, the score kernel
  reference  reward_scorer's steps (utils/reward/reward.py:134-192) on the oracle at the reference's precision: the VAE
             decode of every frame (in chunks of 16 frames) and the HPS towers with fp16 weights, both under fp16
             autocast, torchvision's Resize + Normalize of every frame, then the selection and the scores
Rounds alternate the two procedures; each timed call ends in a device synchronise.  The algorithmic FLOP of each
procedure is counted from shapes by the library's per-op counters (ops.KernelProfile) over one instrumented native call
and one instrumented single-frame decode.  Prints one JSON line per batch size with the medians (and min / max), the
speed-up, the FLOP, the largest score difference and the card's name, power limit and maximum SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import reward_oracle as ro, synth  # noqa: E402
from oracle.cases import FULL_CTORS  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _fill_(module, seed):
    """Synthetic weights drawn on the device (fan-in scaled matrices, unit norm weights, small biases)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    for name, p in module.named_parameters():
        if p.dim() >= 2:
            p.copy_(torch.randn(p.shape, device="cuda", generator=g) / float(np.sqrt(np.prod(p.shape[1:]))))
        elif name.endswith("weight"):
            p.copy_(1.0 + 0.1 * torch.randn(p.shape, device="cuda", generator=g))
        else:
            p.copy_(0.05 * torch.randn(p.shape, device="cuda", generator=g))
    for k in ("positional_embedding", "visual.positional_embedding", "visual.class_embedding", "token_embedding.weight"):
        if hasattr(module, "get_parameter") and k in dict(module.named_parameters()):
            module.get_parameter(k).mul_(0.02 * float(np.sqrt(module.get_parameter(k).shape[-1])))


def _flop(fn):
    from vgen_b200 import ops
    ops.PROF = ops.KernelProfile()
    try:
        fn()
        return sum(d["flops"] for d in ops.PROF.summary().values())
    finally:
        ops.PROF = None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--segments", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_reward: no CUDA device (the timings are only meaningful on the GPU)")
    os.environ.setdefault("VGEN_CLIP_BPE", os.path.join(ROOT, "tests", "golden", "clip_bpe_merges_head.txt.gz"))
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_grad_enabled(False)
    card = _card()

    from vgen_b200.autoencoder import AutoencoderKL
    from vgen_b200.clip import ARCHS, ClipModel
    from vgen_b200.clip_tokenizer import tokenize
    from vgen_b200.reward import SegmentalReward

    hps = ClipModel(ARCHS["ViT-H-14"]).cuda().eval()
    _fill_(hps, 1)
    vae = AutoencoderKL(**FULL_CTORS["full_vae"][1]).cuda().eval()
    _fill_(vae, 2)
    hsd16 = {k: v.half() for k, v in hps.state_dict().items()}
    vsd = dict(vae.state_dict())
    scorer = SegmentalReward(hps, vae, segments=args.segments)
    f, s = args.frames, args.segments

    for b in args.batches:
        caps = [f"a video of scene {i}, highly detailed" for i in range(b)]
        x0 = synth.tensor(f"bench_reward_x0_b{b}", (b, 4, f, 32, 32), 1.0, 3).cuda()
        tokens = tokenize(caps).cuda()

        def native(seed=0):
            return scorer.score_latents(caps, x0, torch.Generator().manual_seed(seed)).tolist()

        def reference(seed=0):
            idx = scorer.indices(b, f, torch.Generator().manual_seed(seed))
            z = (1.0 / 0.18215 * x0).permute(0, 2, 1, 3, 4).reshape(b * f, 4, 32, 32)
            with torch.autocast("cuda", dtype=torch.float16):
                video = torch.cat([ro.vgen_oracle.vae_decode(vsd, c) for c in z.split(16)]).float()
            video = video.view(b, f, *video.shape[1:]).permute(0, 2, 1, 3, 4)
            x = ro.preprocess(video, False)
            sel = x[torch.arange(b)[:, None], idx.cuda()].reshape(b * s, *x.shape[2:])
            with torch.autocast("cuda", dtype=torch.float16):
                img, txt = ro.features(hsd16, sel.half(), tokens, 80, 16)
            return ro.reward_scores(img.float(), txt.float(), idx.cuda(), f, True).tolist()

        for fn in (native, reference, native, reference):            # warm-up: packing, graph capture, module loads
            fn()
        torch.cuda.synchronize()
        times = {"native": [], "reference": []}
        for r in range(args.rounds):
            for name, fn in (("native", native), ("reference", reference)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(r)
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3)
        a, c = native(), reference()
        flop_native = _flop(native)
        flop_frame = _flop(lambda: vae.decode(torch.zeros(1, 4, 32, 32, device="cuda")))
        flop_ref = flop_native + flop_frame * b * (f - s)
        med = {k: float(np.median(v)) for k, v in times.items()}
        print(json.dumps({
            "workload": f"b={b} videos of {f} frames at 256x256 (latents 32x32), {s} TSN segments with TAR; "
                        "synthetic full-size HPSv2 ViT-H/14 + VAE",
            "native_ms_median": round(med["native"], 2), "reference_ms_median": round(med["reference"], 2),
            "native_ms_per_video": round(med["native"] / b, 2), "reference_ms_per_video": round(med["reference"] / b, 2),
            "native_ms_min_max": [round(min(times["native"]), 2), round(max(times["native"]), 2)],
            "reference_ms_min_max": [round(min(times["reference"]), 2), round(max(times["reference"]), 2)],
            "speedup": round(med["reference"] / med["native"], 2), "rounds": args.rounds,
            "tflop_native": round(flop_native / 1e12, 3), "tflop_reference": round(flop_ref / 1e12, 3),
            "tflop_decode_per_frame": round(flop_frame / 1e12, 4),
            "native_tflops_achieved": round(flop_native / 1e12 / (med["native"] / 1e3), 1),
            "max_score_diff": float(np.max(np.abs(np.asarray(a) - np.asarray(c)))), "gpu": card}), flush=True)


if __name__ == "__main__":
    main()
