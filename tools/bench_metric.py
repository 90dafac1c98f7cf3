"""Time DreamVideo's evaluation metric for one video: the native calculate_metric against the reference procedure.

    python tools/bench_metric.py [--frames 32] [--size 256] [--targets 6] [--rounds 7]

The workload is one DreamVideo video (32 frames at 256 x 256 by default) plus 6 reference images of other sizes, scored
with synthetic full-size ViT-B/32 and ViT-S/16 weights.  Both procedures start from the same decoded host data (the
video's RGB frames and the decoded images), so video / JPEG decoding is outside the window:
  native     vgen_b200.metric: one upload of the frames, the resize kernel, both towers, the score kernel
  reference  cal_metric_DreamVideo.py's steps on the GPU: the oracle CLIP in fp16 weights (what clip.load runs) and the
             oracle DINO in fp32, T.ToPILImage + the torchvision transforms per frame and per image, F.normalize and the
             score arithmetic
Rounds alternate the two procedures; each timed call ends in a device synchronise (the scores are read back as floats).
Prints the medians (and min / max) per procedure, the speed-up, the card's name and power limit, and the largest score
difference between the two as one JSON line.
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
import torch.nn.functional as F  # noqa: E402
import torchvision.transforms as T  # noqa: E402

import _metric as mt  # noqa: E402
from oracle import metric_oracle as mo  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        return out
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--targets", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metric: no CUDA device (the timings are only meaningful on the GPU)")
    os.environ.setdefault("VGEN_CLIP_BPE", os.path.join(ROOT, "tests", "golden", "clip_bpe_merges_head.txt.gz"))
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_grad_enabled(False)

    from vgen_b200.clip import OpenAIClipModel
    from vgen_b200.clip_tokenizer import tokenize
    from vgen_b200.dino import vit_small
    from vgen_b200.metric import clip_transform, dino_transform, score_video

    # inputs: a smooth moving video and reference images of several sizes (decoded host data)
    mt.METRIC_CASES["bench"] = dict(H=args.size, W=args.size, frames=args.frames, seed=90, prompt="", targets=[
        (h, w, "RGB") for h, w in [(512, 512), (480, 640), (640, 480), (300, 400), (1024, 768), (256, 256)][:args.targets]])
    frames = mt.make_frames("bench")
    targets = [a for a, _ in mt.make_targets("bench")]
    prompt = "a photo of sks dog running on the beach, highly detailed"

    # models: synthetic full-size weights
    csd = mt.clip_state_dict(mt.product_spec("clip_full"), 71, qk_gain=1.0)
    dsd = mt.dino_state_dict(mt.product_spec("dino_full"), 72, qk_gain=1.0)
    clip_m = OpenAIClipModel(mt.FULL_CLIP)
    clip_m.load_state_dict(csd, strict=True)
    clip_m = clip_m.eval().cuda()
    dino_m = vit_small()
    dino_m.load_state_dict(dsd, strict=True)
    dino_m = dino_m.eval().cuda()
    ctf, dtf = clip_transform(), dino_transform()
    csd16 = {k: v.cuda().half() for k, v in csd.items()}
    dsd32 = {k: v.cuda() for k, v in dsd.items()}
    heads = mt.FULL_DINO["num_heads"]
    ref_ctf = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(),
                         T.Normalize(mo.OPENAI_MEAN, mo.OPENAI_STD)])
    ref_dtf = T.Compose([T.Resize(256, interpolation=3), T.CenterCrop(224), T.ToTensor(),
                         T.Normalize(mo.IMAGENET_MEAN, mo.IMAGENET_STD)])
    from PIL import Image
    target_pils = [Image.fromarray(a) for a in targets]

    def native():
        s = score_video(torch.from_numpy(frames).cuda(), prompt, targets, clip_m, ctf, dino_m, dtf)
        return s.tolist()

    def reference():
        to_pil = T.ToPILImage()
        video = torch.from_numpy(frames).cuda().permute(0, 3, 1, 2)              # 'n f h w c -> (n f) c h w' on the GPU
        text = tokenize([prompt], truncate=False).cuda()
        t_feature = F.normalize(mo.clip_encode_text(csd16, text), p=2, dim=1)
        images = torch.cat([ref_ctf(to_pil(img)).unsqueeze(0) for img in video]).cuda()
        gen = F.normalize(mo.clip_encode_image(csd16, images.half()), p=2, dim=1)
        timg = torch.cat([ref_ctf(im).unsqueeze(0) for im in target_pils]).cuda()
        images_d = torch.cat([ref_dtf(to_pil(img)).unsqueeze(0) for img in video]).cuda()
        gen_d = F.normalize(mo.dino_forward(dsd32, images_d, heads), p=2, dim=1)
        timg_d = torch.cat([ref_dtf(im).unsqueeze(0) for im in target_pils]).cuda()
        tf = F.normalize(mo.clip_encode_image(csd16, timg.half()), p=2, dim=1)
        tdf = F.normalize(mo.dino_forward(dsd32, timg_d, heads), p=2, dim=1)
        gm, gdm = gen.mean(0), gen_d.mean(0)
        clip_t = (t_feature[0] * gm).sum()
        clip_i = (tf * gm).sum(1).mean()
        dino_i = (tdf * gdm).sum(1).mean()
        tc = (gen[:-1] * gen[1:]).sum(1).mean()
        return [float(clip_t), float(clip_i), float(dino_i), float(tc)]

    for fn in (native, reference, native, reference):                # warm-up: packing, graph capture, module loads
        fn()
    torch.cuda.synchronize()
    times = {"native": [], "reference": []}
    for _ in range(args.rounds):
        for name, fn in (("native", native), ("reference", reference)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
    a, b = native(), reference()
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({
        "workload": f"1 video, {args.frames} frames at {args.size}x{args.size}, {args.targets} reference images; "
                    "synthetic full-size ViT-B/32 + ViT-S/16",
        "native_ms_median": round(med["native"], 2), "reference_ms_median": round(med["reference"], 2),
        "native_ms_min_max": [round(min(times["native"]), 2), round(max(times["native"]), 2)],
        "reference_ms_min_max": [round(min(times["reference"]), 2), round(max(times["reference"]), 2)],
        "speedup": round(med["reference"] / med["native"], 2), "rounds": args.rounds,
        "scores_native": [round(v, 5) for v in a], "scores_reference": [round(v, 5) for v in b],
        "max_score_diff": float(np.nanmax(np.abs(np.asarray(a) - np.asarray(b)))), "gpu": _card()}))


if __name__ == "__main__":
    main()
