"""DreamVideo evaluation-metric parity cases: the tiny OpenAI-format CLIP and DINO configurations, synthetic weights,
synthetic videos and reference images, and the parameter lists checked against the reference's frozen digests.

tools/make_golden_metric.py runs the reference's own calculate_metric on these cases and freezes into
tests/golden/metric_<case>.npz the frames and the decoded target images (delta-coded along the rows, which lets them
compress), both transforms' fp32 outputs per image (as sha256 digests of their bytes: the suite checks bit-identity), the
features and the four scores; and into tests/golden/metric_specs.json the digests of the tiny and full-size parameter
lists.
"""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np
import torch

from oracle import synth
from _sketch import spec_digest  # noqa: F401  (re-exported for the metric tests)

# ViT-B/32 and ViT-S/16 shapes narrowed to 2 layers and 2 heads of head_dim 64, at 224 px
TINY_CLIP = dict(embed_dim=64, act="quick_gelu",
                 vision_cfg=dict(image_size=224, layers=2, width=128, head_width=64, patch_size=32),
                 text_cfg=dict(context_length=77, vocab_size=49408, width=128, heads=2, layers=2))
FULL_CLIP = dict(embed_dim=512, act="quick_gelu",
                 vision_cfg=dict(image_size=224, layers=12, width=768, head_width=64, patch_size=32),
                 text_cfg=dict(context_length=77, vocab_size=49408, width=512, heads=8, layers=12))
TINY_DINO = dict(patch_size=16, embed_dim=128, depth=2, num_heads=2, mlp_ratio=4, qkv_bias=True)
FULL_DINO = dict(patch_size=16, embed_dim=384, depth=12, num_heads=6, mlp_ratio=4, qkv_bias=True)

METRIC_CASES = {
    # a square video with reference images of other sizes and aspect ratios (one stored as a grayscale image)
    "square_targets": dict(H=256, W=256, frames=4, seed=51, prompt="a photo of sks dog running on the beach",
                           targets=[(300, 200, "RGB"), (180, 320, "L"), (260, 240, "RGB")]),
    # a non-square video with no reference images: CLIP-I = DINO-I = 0
    "wide_no_targets": dict(H=240, W=320, frames=3, seed=52, prompt="An astronaut riding a horse on Mars, oil painting",
                            targets=[]),
}

# Synthetic-weight calibration (measured on these cases, see the non-vacuity checks): at fan-in scale the attention of the
# class token is nearly uniform, so it carries the mean of the patches and every frame gets almost the same feature
# (consecutive-frame cosines above 0.99).  The tiny cases scale the query and key rows of the image towers' qkv projections
# by QK_GAIN, which sharpens the attention: the cosines drop to about 0.6-0.9.  The text tower keeps fan-in scale, and so
# do the full-size models (qk_gain=1), whose checks are about arithmetic, not about the scores.
QK_GAIN = 3.0


def _smooth_rgb(name, h, w, seed, t=0.0):
    """A smooth colour image with moving structure: a few sinusoids and gaussian blobs whose phases / centres move with t."""
    r = np.random.Generator(np.random.PCG64([sum(map(ord, name)), seed]))
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.zeros((h, w, 3))
    for c in range(3):
        for _ in range(3):
            fy, fx, ph, sp = r.uniform(0.5, 6, 2).tolist() + [r.uniform(0, 6.3), r.uniform(0.5, 1.5)]
            img[..., c] += np.sin(2 * np.pi * (fy * yy / h + fx * xx / w) + ph + sp * t)
    for _ in range(4):
        cy, cx, vy, vx, rad = r.uniform(0, h), r.uniform(0, w), r.uniform(-40, 40), r.uniform(-40, 40), r.uniform(15, 50)
        col = r.uniform(-2, 2, 3)
        g = np.exp(-(((yy - cy - vy * t) ** 2 + (xx - cx - vx * t) ** 2) / (2 * rad ** 2)))
        img += g[..., None] * col
    img = 127.5 + 40.0 * img
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def make_frames(name):
    """RGB frames uint8 [f, H, W, 3] of a case."""
    c = METRIC_CASES[name]
    return np.stack([_smooth_rgb(name, c["H"], c["W"], c["seed"], t=1.5 * i) for i in range(c["frames"])])


def make_targets(name):
    """[(uint8 [h, w] or [h, w, 3] array, PIL mode)] of a case's reference images, before any RGB conversion."""
    out = []
    for j, (h, w, mode) in enumerate(METRIC_CASES[name]["targets"]):
        a = _smooth_rgb(f"{name}_target{j}", h, w, METRIC_CASES[name]["seed"])
        out.append((a if mode == "RGB" else a[..., 1].copy(), mode))
    return out


def clip_state_dict(spec, seed, qk_gain=QK_GAIN):
    """OpenAI-format CLIP weights: synth.state_dict with open_clip's 0.02 scale for the embeddings, rounded to fp16 (an
    OpenAI checkpoint stores fp16 weights), logit_scale ln(1 / 0.07)."""
    sd = synth.state_dict([s for s in spec if len(s[1]) > 0], seed=seed)
    for k in ("positional_embedding", "visual.positional_embedding", "visual.class_embedding", "token_embedding.weight"):
        sd[k] = synth.tensor(k, dict(spec)[k], 0.02, seed)
    for k in sd:
        if k.startswith("visual.") and k.endswith("attn.in_proj_weight"):
            sd[k][: 2 * sd[k].shape[1]] *= qk_gain
    sd["logit_scale"] = torch.tensor(4.6052)
    return {k: sd[k].half().float() for k, _ in spec}


def dino_state_dict(spec, seed, qk_gain=QK_GAIN):
    sd = synth.state_dict(spec, seed=seed)
    for k in ("cls_token", "pos_embed"):
        sd[k] = synth.tensor(k, dict(spec)[k], 0.02, seed)
    for k in sd:
        if k.endswith("attn.qkv.weight"):
            sd[k][: 2 * sd[k].shape[1]] *= qk_gain
    return sd


def product_spec(which):
    from vgen_b200.clip import clip_spec
    from vgen_b200.dino import VisionTransformer, dino_spec
    if which in ("clip_tiny", "clip_full"):
        return [(k, tuple(s)) for k, s in clip_spec(TINY_CLIP if which == "clip_tiny" else FULL_CLIP)]
    kw = TINY_DINO if which == "dino_tiny" else FULL_DINO
    with torch.device("meta"):
        m = VisionTransformer(**kw)
    spec = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert spec == [(k, tuple(s)) for k, s in dino_spec(224, kw["patch_size"], 3, 0, kw["embed_dim"], kw["depth"],
                                                         kw["mlp_ratio"], kw["qkv_bias"])]
    return spec


def load_spec(golden_dir, which):
    """which: clip_tiny / clip_full / dino_tiny / dino_full; the product's list, checked against the reference's digest."""
    spec = product_spec(which)
    want = json.load(open(os.path.join(golden_dir, "metric_specs.json")))[which]
    assert spec_digest(spec) == want, f"{which}: parameter list differs from the reference's"
    return spec


def delta_encode(a):
    """uint8 [..., w, c] -> its differences along w, mod 256 (what the fixtures store of images)."""
    return np.diff(a.astype(np.int16), axis=-2, prepend=0).astype(np.uint8)


def delta_decode(d):
    return np.cumsum(d.astype(np.int64), axis=-2).astype(np.uint8)


def tensor_sha(t):
    """sha256 of a tensor's fp32 bytes in its contiguous layout."""
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().float().numpy()).tobytes()).hexdigest()


def load_case(golden_dir, name):
    """The frozen values of a case: a dict of numpy arrays with the frames decoded and the targets as a list."""
    z = dict(np.load(os.path.join(golden_dir, f"metric_{name}.npz")))
    z["frames"] = delta_decode(z.pop("frames_delta"))
    z["targets"] = [delta_decode(z.pop(f"target{j}_delta")) for j in range(len(METRIC_CASES[name]["targets"]))]
    return z
