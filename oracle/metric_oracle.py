"""TEST INFRASTRUCTURE ONLY -- CPU restatement of DreamVideo's evaluation metric (metric/cal_metric_DreamVideo.py):

  * Pillow's 8-bit bicubic resample (ImagingResample, libImaging/Resample.c: precompute_coeffs, normalize_coeffs_8bpc,
    ImagingResampleHorizontal_8bpc / Vertical_8bpc) in numpy integer arithmetic, and the torchvision transforms built on
    it (Resize(short side) -> CenterCrop -> ToTensor -> Normalize) in numpy float32;
  * OpenAI's CLIP (the open_clip CLIP built by build_model_from_openai_state_dict: QuickGELU in both towers), from an
    OpenAI-format state dict: oracle/clip_oracle.py's towers with QuickGELU and head width 64;
  * DINO's VisionTransformer (metric/dino/vision_transformer.py): clip_oracle's block with DINO's names and eps;
  * the four scores of calculate_metric.

tools/make_golden_metric.py checks it against the reference's own calculate_metric and freezes the results.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import clip_oracle

PRECISION_BITS = 32 - 8 - 2
OPENAI_MEAN, OPENAI_STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


# ---- Pillow ------------------------------------------------------------------------------------------------------------
def _bicubic(x):
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(in_size, out_size):
    """precompute_coeffs + normalize_coeffs_8bpc for the bicubic filter: -> (bounds int [out, 2] = (xmin, count),
    weights int64 [out, ksize] holding the int32 fixed-point coefficients)."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int64)
    kk = np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        for x, v in enumerate(w):
            kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _pass(img, axis, out_size):
    """One 8-bit pass along `axis` (0 rows, 1 columns) of a uint8 [H, W, C] image; int32 sums as in Resample.c."""
    bounds, kk = coeffs(img.shape[axis], out_size)
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((out_size,) + src.shape[1:], np.int64)
    for o in range(out_size):
        xmin, n = bounds[o]
        ss = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        for x in range(n):
            ss += src[xmin + x] * kk[o, x]
        assert ss.max() < 2 ** 31 and ss.min() >= -2 ** 31
        out[o] = np.clip(ss >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis).astype(np.uint8)


def pillow_resize(img, out_w, out_h):
    """Image.resize((out_w, out_h), BICUBIC) of a uint8 [H, W, C] array: horizontal pass first, an axis whose size does
    not change is not resampled.  (Restricting the horizontal pass to the rows the vertical pass reads, as Pillow does,
    leaves every value unchanged.)"""
    if img.shape[1] != out_w:
        img = _pass(img, 1, out_w)
    if img.shape[0] != out_h:
        img = _pass(img, 0, out_h)
    return img


def resized_size(h, w, size):
    """torchvision's Resize(int) output (h, w): the short side becomes `size`, the long one int(size * long / short)."""
    if w <= h:
        return int(size * h / w), size
    return size, int(size * w / h)


def transform(img, resize, crop, mean, std):
    """Resize(resize, BICUBIC) -> CenterCrop(crop) -> ToTensor -> Normalize(mean, std) of a uint8 [H, W, 3] array, in
    the float32 arithmetic torchvision runs on the CPU -> float32 [3, crop, crop]."""
    h, w = img.shape[:2]
    rh, rw = resized_size(h, w, resize)
    if (rh, rw) != (h, w):
        img = pillow_resize(img, rw, rh)
    top, left = int(round((rh - crop) / 2.0)), int(round((rw - crop) / 2.0))
    img = img[top:top + crop, left:left + crop]
    x = img.transpose(2, 0, 1).astype(np.float32) / np.float32(255)
    m = np.asarray(mean, np.float32).reshape(3, 1, 1)
    s = np.asarray(std, np.float32).reshape(3, 1, 1)
    return (x - m) / s


def clip_transform(img, size=224):
    return transform(img, size, size, OPENAI_MEAN, OPENAI_STD)


def dino_transform(img):
    return transform(img, 256, 224, IMAGENET_MEAN, IMAGENET_STD)


# ---- OpenAI CLIP -------------------------------------------------------------------------------------------------------
def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


def clip_encode_text(sd, tokens):
    """CLIP.encode_text: [b, 77] ids -> [b, E] (heads = width // 64, as build_model_from_openai_state_dict derives)."""
    return clip_oracle.encode_text(sd, tokens, sd["ln_final.weight"].shape[0] // 64, "last", quick_gelu)[0]


def clip_encode_image(sd, image):
    """CLIP.encode_image: [b, 3, H, W] -> [b, E]."""
    return clip_oracle.encode_image(sd, image, 64, quick_gelu)


# ---- DINO ViT ----------------------------------------------------------------------------------------------------------
DINO_BLOCK = ("norm1.", "attn.qkv.", "attn.proj.", "norm2.", "mlp.fc1.", "mlp.fc2.")


def dino_forward(sd, image, heads, eps=1e-6):
    """VisionTransformer.forward at the trained grid: patch embed, [CLS], + pos_embed, pre-LN blocks (qkv bias, GELU MLP),
    norm, class token -> [b, D]."""
    w = sd["patch_embed.proj.weight"]
    x = F.conv2d(image, w, sd["patch_embed.proj.bias"], stride=w.shape[-1]).flatten(2).transpose(1, 2)
    b, _, D = x.shape
    x = torch.cat([sd["cls_token"].expand(b, -1, -1), x], dim=1) + sd["pos_embed"]
    for i in range(clip_oracle._n_layers(sd, "blocks.")):
        x = clip_oracle._block(x, sd, f"blocks.{i}.", heads, False, eps=eps, names=DINO_BLOCK)
    return F.layer_norm(x, (D,), sd["norm.weight"], sd["norm.bias"], eps)[:, 0]


# ---- scores ------------------------------------------------------------------------------------------------------------
def scores(clip_frames, text, clip_targets, dino_frames, dino_targets):
    """calculate_metric's arithmetic for one video: -> (CLIP-T, CLIP-I, DINO-I, temporal consistency) as floats.  No
    targets: CLIP-I = DINO-I = 0; one frame: the temporal mean over an empty tensor is NaN."""
    g = F.normalize(clip_frames, p=2, dim=1)
    t = F.normalize(text.reshape(1, -1), p=2, dim=1)
    gd = F.normalize(dino_frames, p=2, dim=1)
    gm, gdm = g.mean(dim=0), gd.mean(dim=0)
    clip_t = float((t[0] * gm).sum())
    tc = float((g[:-1] * g[1:]).sum(dim=1).mean())
    if clip_targets is None or len(clip_targets) == 0:
        return clip_t, 0.0, 0.0, tc
    ti = F.normalize(clip_targets, p=2, dim=1)
    td = F.normalize(dino_targets, p=2, dim=1)
    return clip_t, float((ti * gm).sum(dim=1).mean()), float((td * gdm).sum(dim=1).mean()), tc
