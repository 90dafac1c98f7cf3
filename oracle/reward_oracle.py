"""TEST INFRASTRUCTURE ONLY -- CPU restatement of InstructVideo's segmental HPSv2 reward
(utils/reward/reward.py DiffRewardModel.reward_scorer :128-197) on top of the fp32 CLIP towers (oracle/clip_oracle.py) and
the VAE decoder (oracle/vgen_oracle.py vae_decode).  tools/make_golden_reward.py checks it against the reference's own
reward_scorer, run unmodified; tests/golden/reward_*.npz freeze what the reference computed.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import clip_oracle, vgen_oracle

OPENAI_MEAN, OPENAI_STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)


def resized_size(h, w, size):
    """torchvision's Resize(int) output size: the short side becomes `size`, the long one int(size * long / short)."""
    if w <= h:
        return int(size * h / w), size
    return size, int(size * w / h)


def decode(vae_sd, x0, scale_factor=0.18215):
    """reward.py:134-145: x0 [b, 4, f, h, w] -> video [b, 3, f, H, W] (every frame through the decoder)."""
    b, c, f, h, w = x0.shape
    z = (1. / scale_factor * x0).permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    v = vgen_oracle.vae_decode(vae_sd, z)
    return v.reshape(b, f, *v.shape[1:]).permute(0, 2, 1, 3, 4)


def preprocess(video, antialias, size=224):
    """reward.py:147-152: [b, 3, f, H, W] in [-1, 1] -> x * 0.5 + 0.5, clamp(0, 1), Resize(size) (bilinear), Normalize
    -> [b, f, 3, rh, rw]."""
    b, c, f, H, W = video.shape
    x = (video * 0.5 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4).reshape(b * f, c, H, W)
    x = F.interpolate(x, size=resized_size(H, W, size), mode="bilinear", align_corners=False, antialias=antialias)
    mean = torch.tensor(OPENAI_MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(OPENAI_STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    x = (x - mean) / std
    return x.reshape(b, f, c, *x.shape[2:])


def features(sd, images, tokens, head_width, text_heads):
    """open_clip CLIP.forward with output_dict (model.py:246-255): L2-normalised image features of images [n, 3, S, S] and
    text features of tokens [b, 77]."""
    img = clip_oracle.encode_image(sd, images, head_width)
    txt = clip_oracle.encode_text(sd, tokens, text_heads, layer="last")[0]
    return F.normalize(img, dim=-1), F.normalize(txt, dim=-1)


def reward_scores(img, txt, idx, f, tar, lambda_tar=1.0):
    """reward.py:174-192: img [b * s, E], txt [b, E] (normalised), idx [b, s] frame indices -> [b]."""
    b, s = idx.shape
    diag = (img.view(b, s, -1) * txt[:, None]).sum(-1)
    if tar:
        diag = torch.exp(-torch.abs(idx - f // 2) * lambda_tar).to(diag.dtype) * diag
    return diag.mean(1)


def score_latents(vae_sd, clip_sd, tokens, x0, idx, tar, lambda_tar, antialias, head_width, text_heads):
    """The whole reward_scorer up to reward_scores, with the frame indices given."""
    video = decode(vae_sd, x0)
    x = preprocess(video, antialias)
    b, s = idx.shape
    sel = x[torch.arange(b)[:, None], idx].reshape(b * s, *x.shape[2:])
    img, txt = features(clip_sd, sel, tokens, head_width, text_heads)
    return reward_scores(img, txt, idx, x0.shape[2], tar, lambda_tar)
