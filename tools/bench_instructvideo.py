"""Time one InstructVideo eval video end to end (configs/instructvideo/eval, the LoRA UNet): b = 1 with the CFG pair as one
batch of 2, 16 frames at 256 x 256 pixels (32 x 32 latent), 77 tokens, 20 DDIM steps of DiffusionDDIMReward
(linear_sd, eps, guide scale 9), the decode in chunks of decoder_bs = 4 frames, then save_video_local.

    python tools/bench_instructvideo.py [--repeats 3] [--json OUT]

Two pipelines on the same synthetic weights (oracle/synth.py, LoRA up weights non-zero):
  native   UNetSD_LoRA (LoRA merged at pack time, CUDA-graphed forward), DiffusionDDIMReward, AutoencoderKL,
           video_io.save_video_local;
  oracle   the reference's arithmetic in PyTorch under fp16 autocast, as the engine runs it: the model
           get_lora_merged_model returns (the merged weights through oracle/vgen_oracle.py's UNet, CFG as two calls),
           the oracle DDIM loop and VAE decode, frames made on the host, the same encoder.
Each round runs both once, in alternating order; the median and the spread over --repeats rounds are printed with the
card's name and power limit read in the same run.  The native video is compared with the oracle's.  Files go to a
temporary directory; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import synth, video_oracle, vgen_oracle as vo  # noqa: E402
from oracle.cases import _FULL_VAE  # noqa: E402
import vgen_b200  # noqa: E402
from vgen_b200 import video_io  # noqa: E402
from bench_compositions import _card  # noqa: E402
import _instructvideo as iv  # noqa: E402

STEPS, GUIDE, DECODER_BS, SCALE = 20, 9.0, 4, 0.18215
MEAN = STD = [0.5, 0.5, 0.5]


def _events(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    r = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), r


def _latent_to_frames(lat, decode):
    """1 / scale_factor, '(b f) c h w', decoder_bs chunks (inference_instructvideo_entrance.py:246-255)."""
    b, c, f, h, w = lat.shape
    z = (lat / SCALE).permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    z = torch.nan_to_num(z).clamp(-10, 10)      # random weights: keep the decoder's input bounded
    out = torch.cat([decode(z[i:i + DECODER_BS]) for i in range(0, b * f, DECODER_BS)])
    return out.reshape(b, f, *out.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_instructvideo: no CUDA device")
    torch.set_grad_enabled(False)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    card = _card()
    print(f"card: {card}")

    golden = os.path.join(ROOT, "tests", "golden")
    case = iv.FULL_IV_CASES["full_iv_lora"]
    spec = iv.load_spec(golden, "full_iv_lora", iv.FULL_IV_CASES)
    sd = iv.weights(spec, case["seed"])
    unet = iv.build_product(case)
    unet.load_state_dict(sd, strict=True)
    unet = unet.cuda().eval()
    merged = {k: v.cuda() for k, v in unet.merged_state_dict().items()}   # what get_lora_merged_model loads
    del sd
    vae = vgen_b200.AutoencoderKL(**_FULL_VAE)
    vsd = synth.state_dict([(k, tuple(v.shape)) for k, v in vae.state_dict().items()], seed=7)
    vae.load_state_dict(vsd, strict=True)
    vae = vae.cuda().eval()
    vsd = {k: v.cuda() for k, v in vsd.items()}
    diff = vgen_b200.DiffusionDDIMReward(**{k: v for k, v in iv.RELEASED_DIFFUSION.items() if k != "type"})
    betas = vo.make_betas("linear_sd", 1000, False, init_beta=0.00085, last_beta=0.0120)

    inp = {k: v.cuda() for k, v in iv.make_inputs(case).items()}
    noise, y, y0 = inp["x"], inp["y"], inp["y_neg"]
    kw = [{"y": y}, {"y": y0}]
    tmp = tempfile.mkdtemp(prefix="bench_instructvideo_")

    def native():
        lat = diff.ddim_sample_loop(noise, unet, kw, guide_scale=GUIDE, ddim_timesteps=STEPS, eta=0.0)
        video = _latent_to_frames(lat, vae.decode)
        return video_io.save_video_local(os.path.join(tmp, "native.mp4"), video, MEAN, STD)

    def oracle():
        fn = lambda xt, t, **k: vo.unet_t2v_forward(merged, xt, t, k["y"])  # noqa: E731
        with torch.autocast("cuda", dtype=torch.float16):
            lat = vo.ddim_sample_loop(noise.clone(), fn, kw, betas, GUIDE, STEPS, mean_type="eps", autocast_cfg=True)
            video = _latent_to_frames(lat.float(), lambda z: vo.vae_decode(vsd, z))
        frames = video_oracle.frames_uint8(video.float().cpu().numpy(), MEAN, STD)
        video_io._encode(os.path.join(tmp, "oracle.mp4"), np.stack(frames), 8, video=True)
        return frames

    variants = {"native": native, "oracle_autocast": oracle}
    results = {k: None for k in variants}
    for fn in variants.values():          # warm-up: packs, sets attributes, captures the graphs
        fn()
    times = {k: [] for k in variants}
    for r in range(args.repeats):
        order = list(variants) if r % 2 == 0 else list(variants)[::-1]
        for k in order:
            ms, results[k] = _events(variants[k])
            times[k].append(ms)
    a, b = np.stack(results["native"]).astype(np.int16), np.stack(results["oracle_autocast"]).astype(np.int16)
    diff_px = np.abs(a - b)
    res = {"card": card, "workload": dict(b=1, cfg_batch=2, frames=case["f"], pixels=[256, 256], latent=[case["h"], case["w"]],
                                          tokens=case["ntok"], ddim_steps=STEPS, decoder_bs=DECODER_BS),
           "video_vs_oracle": dict(frames=len(results["native"]), mean_abs_u8=float(diff_px.mean()), max_abs_u8=int(diff_px.max())),
           "ms": {k: dict(median=statistics.median(v), min=min(v), max=max(v), runs=v) for k, v in times.items()}}
    for k, v in res["ms"].items():
        print(f"{k:16s} median {v['median']:10.1f} ms  (min {v['min']:.1f}, max {v['max']:.1f}, {args.repeats} alternating rounds)")
    print(f"speed-up {res['ms']['oracle_autocast']['median'] / res['ms']['native']['median']:.2f}x; video vs oracle: "
          f"mean |du8| {res['video_vs_oracle']['mean_abs_u8']:.3f}, max {res['video_vs_oracle']['max_abs_u8']}")
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
