"""H100-native InstructVideo reward scoring: the Segmental Video Reward with HPSv2 and the Temporally Attenuated Reward
(TAR) of utils/reward/reward.py `DiffRewardModel.reward_scorer` (:128-197; RWRRewardModel and DDPORewardModel compute the
same `reward_scores`).

Given latents x0 [b, 4, f, h, w] and b captions, the reference decodes every frame, maps it to [0, 1], resizes it with
torchvision's Resize(224) (bilinear; short side 224), normalises it with the OpenAI mean / std, keeps `segments` frames per
video (`fixed_first`: every (f // segments)-th; `TSN`: one random frame per span, drawn with torch.randint on the global
CPU generator), scores them with HPSv2 (open_clip ViT-H/14) and averages the per-segment cosines of image and caption,
each weighted by exp(-|g - f // 2| * lambda_TAR) with TAR.

Here the frame indices are drawn first, so `score_latents` decodes only the selected frames (the decoder works frame by
frame, so the values are the same).  Then one kernel turns the selected frames into the tower's fp16 input
(`ops.reward_frames`), the image tower runs CUDA-graphed, the text tower runs, and one kernel computes the scores of all
videos (`ops.segment_reward`).  The reference's chunking by `decoder_bs` changes no values and is not reproduced.

    python -m vgen_b200.reward --videos DIR --captions FILE --hps HPS_v2.pt [--segments 4 --selection TSN --seed 0]
scores the mp4 files of DIR (decoded with cv2, as metric.read_video_rgb does); FILE holds one `<file name>|||<caption>`
line per video.
"""
from __future__ import annotations

import argparse
import os

import numpy as np
import torch

from . import ops
from .clip import ARCHS, ClipModel
from .clip_tokenizer import tokenize
from .metric import OPENAI_MEAN, OPENAI_STD, resized_size

_TILE_ROWS = 16                              # output rows per block of the frame kernel
SELECTION_METHODS = ("TSN", "fixed_first")


# ---- F.interpolate's bilinear taps -------------------------------------------------------------------------------------
def bilinear_taps(n_in, n_out, antialias):
    """The weights F.interpolate(mode='bilinear', align_corners=False) applies along one axis of size n_in -> n_out:
    (bounds int32 [n_out, 2] = (first input index, taps), weights fp32 [n_out, k]).  An index past n_in - 1 is read as
    n_in - 1 (the frame kernel clamps it).  The arithmetic is PyTorch's, in fp32, so the weights are its weights."""
    f32 = np.float32
    scale = f32(n_in) / f32(n_out)
    if not antialias:
        # upsample_bilinear2d: src = max(scale * (o + 0.5) - 0.5, 0) as one fused multiply-add (exact in fp64, rounded
        # once to fp32), i0 = (int)src, l1 = src - i0
        src = np.maximum((float(scale) * (np.arange(n_out, dtype=np.float64) + 0.5) - 0.5).astype(f32), f32(0))
        i0 = src.astype(np.int64)
        l1 = (src - i0.astype(f32)).astype(f32)
        bounds = np.stack([i0, np.full(n_out, 2)], 1).astype(np.int32)
        return bounds, np.stack([f32(1) - l1, l1], 1).astype(f32)
    # _upsample_bilinear2d_aa (its CPU kernel's order of operations): the triangle filter, stretched by the scale when
    # downsampling, weights normalised
    support = scale if scale >= 1 else f32(1)
    invscale = f32(1) / scale if scale >= 1 else f32(1)
    bounds = np.zeros((n_out, 2), np.int32)
    kk = np.zeros((n_out, int(np.ceil(support)) * 2 + 1), f32)
    for i in range(n_out):
        center = scale * (f32(i) + f32(0.5))
        xmin = max(int(center - support + f32(0.5)), 0)
        xsize = min(int(center + support + f32(0.5)), n_in) - xmin
        w = [max(f32(0), f32(1) - abs((f32(j + xmin) - center + f32(0.5)) * invscale)) for j in range(xsize)]
        total = f32(0)
        for v in w:
            total = f32(total + v)
        kk[i, :xsize] = [v / total if total != 0 else v for v in w]
        bounds[i] = (xmin, xsize)
    return bounds, kk


class BilinearPlan:
    """Resize(to oh x ow, bilinear, antialias) -> Normalize(mean, std) of h x w frames: the taps of both axes (host, once
    per size), moved to a device on first use."""

    def __init__(self, h, w, oh, ow, antialias, mean=OPENAI_MEAN, std=OPENAI_STD):
        self.h, self.w, self.oh, self.ow, self.antialias, self.mean, self.std = h, w, oh, ow, bool(antialias), mean, std
        self.hb, self.hk = bilinear_taps(w, ow, antialias)
        self.vb, self.vk = bilinear_taps(h, oh, antialias)
        starts = range(0, oh, _TILE_ROWS)
        self.tile_rows = max(int(self.vb[min(r + _TILE_ROWS, oh) - 1].sum() - self.vb[r, 0]) for r in starts)
        self._dev = {}

    def tables(self, device):
        t = self._dev.get(device)
        if t is None:
            t = self._dev[device] = tuple(torch.from_numpy(a).to(device) for a in (self.hb, self.hk, self.vb, self.vk))
        return t


# ---- frame selection ---------------------------------------------------------------------------------------------------
def segment_indices(b, f, segments, selection_method, generator=None, *, exponential_TSN=False):
    """The frames reward_scorer keeps (reward.py:155-165) -> int64 [b, segments] frame indices (CPU).

    `TSN` makes the reference's exact draw, torch.randint(f // segments, (b, segments)) (on the global CPU generator unless
    `generator` is given), plus segment * span; `fixed_first` takes frames 0, span, 2 span, ...  Raises ValueError where the
    reference fails or silently mis-groups: f < segments, a fixed_first stride that yields a number of frames other than
    `segments`, and fixed_first with exponential_TSN (the reference's TAR needs the TSN indices: NameError there)."""
    if selection_method not in SELECTION_METHODS:
        raise ValueError(f"vgen_b200 reward: selection_method must be one of {SELECTION_METHODS}, got {selection_method!r}")
    if segments < 1 or f < segments:
        raise ValueError(f"vgen_b200 reward: {f} frames cannot be split into {segments} segments")
    span = f // segments
    if selection_method == "fixed_first":
        if exponential_TSN:
            raise ValueError("vgen_b200 reward: exponential_TSN (the temporally attenuated reward) needs "
                             "selection_method='TSN'; the reference raises NameError with 'fixed_first'")
        idx = torch.arange(0, f, span)
        if idx.numel() != segments:
            raise ValueError(f"vgen_b200 reward: fixed_first over {f} frames with stride {span} selects {idx.numel()} "
                             f"frames, not {segments} segments")
        return idx[None].expand(b, segments).clone()
    local = torch.randint(span, (b, segments), generator=generator)
    return local + torch.arange(segments)[None] * span


# ---- the model ------------------------------------------------------------------------------------------------------------
def load_hps(path, device="cuda"):
    """HPSv2 (open_clip ViT-H/14 with the HPS_v2.pt weights) from a local file: {'state_dict': ...} as released, or a plain
    state dict; loaded with strict=True.  Nothing is downloaded."""
    ckpt = torch.load(path, map_location="cpu")
    sd = ckpt["state_dict"] if isinstance(ckpt, dict) and "state_dict" in ckpt else ckpt
    model = ClipModel(ARCHS["ViT-H-14"])
    model.load_state_dict(sd, strict=True)
    return model.eval().requires_grad_(False).to(device)


class SegmentalReward:
    """reward_scores of InstructVideo's segmental HPSv2 reward.  The defaults are the released training config's
    effective values (segments 4, TSN, exponential_TSN, lambda_TAR 1.0).  `antialias` selects torchvision's Resize
    behaviour: off is torchvision < 0.17 on tensors (the reference's pinned 0.15.2), on is 0.17 and later."""

    def __init__(self, hps, autoencoder=None, segments=4, selection_method="TSN", exponential_TSN=True, lambda_TAR=1.0,
                 scale_factor=0.18215, antialias=False):
        if selection_method not in SELECTION_METHODS:
            raise ValueError(f"vgen_b200 reward: selection_method must be one of {SELECTION_METHODS}, got {selection_method!r}")
        if selection_method == "fixed_first" and exponential_TSN:
            raise ValueError("vgen_b200 reward: exponential_TSN (the temporally attenuated reward) needs "
                             "selection_method='TSN'; the reference raises NameError with 'fixed_first'")
        self.hps, self.autoencoder = hps, autoencoder
        self.segments, self.selection_method = int(segments), selection_method
        self.exponential_TSN, self.lambda_TAR = bool(exponential_TSN), float(lambda_TAR)
        self.scale_factor, self.antialias = float(scale_factor), bool(antialias)
        self.image_size = hps.cfg["vision_cfg"]["image_size"]
        self._plans = {}

    def plan(self, h, w):
        """The frame plan of h x w frames; raises ValueError unless Resize(image_size) makes them image_size square."""
        p = self._plans.get((h, w))
        if p is None:
            rh, rw = resized_size(h, w, self.image_size)
            if (rh, rw) != (self.image_size, self.image_size):
                raise ValueError(f"vgen_b200 reward: {h}x{w} frames resize to {rh}x{rw}; the HPS image tower takes "
                                 f"{self.image_size}x{self.image_size} (the reference fails on the positional embedding)")
            p = self._plans[(h, w)] = BilinearPlan(h, w, rh, rw, self.antialias)
        return p

    def indices(self, b, f, generator=None):
        return segment_indices(b, f, self.segments, self.selection_method, generator, exponential_TSN=self.exponential_TSN)

    @torch.no_grad()
    def _score(self, captions, src, frame_idx, idx, f, h, w):
        """src: the frames; frame_idx: the flat source frame of each tower input; idx: int64 [b, s] segment frames."""
        dev = self.hps.device
        x = ops.reward_frames(src, frame_idx.to(dev, torch.int32), self.plan(h, w))
        img = self.hps.encode_image_nhwc(x)
        txt = self.hps.encode_text(tokenize(list(captions)).to(dev), 0)[0].contiguous()
        return ops.segment_reward(img, txt, idx.to(dev, torch.int32), f, self.exponential_TSN, self.lambda_TAR)

    def _check(self, captions, b, x, what):
        if not torch.is_tensor(x) or not x.is_cuda:
            raise ops._l.VgenError(f"vgen_b200 reward: {what} must be a CUDA tensor (no CPU path exists)")
        if isinstance(captions, str) or len(captions) != b:
            raise ValueError(f"vgen_b200 reward: {b} videos need {b} captions, got {1 if isinstance(captions, str) else len(captions)}")

    def score_latents(self, captions, x0, generator=None):
        """reward_scorer's reward_scores of latents x0 [b, 4, f, h, w] (CUDA): fp32 [b].  The frame indices are drawn
        first (as the reference draws them, on `generator` or the global CPU generator) and only the selected frames are
        decoded with the autoencoder."""
        if self.autoencoder is None:
            raise ValueError("vgen_b200 reward: score_latents needs the autoencoder")
        if x0.dim() != 5:
            raise ValueError(f"vgen_b200 reward: x0 must be [b, c, f, h, w], got {tuple(x0.shape)}")
        b, c, f, h, w = x0.shape
        self._check(captions, b, x0, "x0")
        idx = self.indices(b, f, generator)
        sel = idx.to(x0.device)
        z = x0.float().permute(0, 2, 1, 3, 4)[torch.arange(b, device=x0.device)[:, None], sel].reshape(-1, c, h, w)
        z = ops.lincomb_f32([(1.0 / self.scale_factor, z.contiguous())])
        video = self.autoencoder.decode(z)                                                  # fp32 [b * s, 3, H, W]
        n = video.shape[0]
        return self._score(captions, video, torch.arange(n), idx, f, video.shape[2], video.shape[3])

    def score_frames(self, captions, video, generator=None):
        """reward_scores of decoded video [b, 3, f, H, W] in [-1, 1] (fp32, CUDA; the engines' video_data): fp32 [b]."""
        if video.dim() != 5 or video.shape[1] != 3 or video.dtype != torch.float32:
            raise ValueError(f"vgen_b200 reward: video must be fp32 [b, 3, f, H, W], got {video.dtype} {tuple(video.shape)}")
        b, _, f, h, w = video.shape
        self._check(captions, b, video, "video")
        idx = self.indices(b, f, generator)
        return self._score(captions, video, (idx + torch.arange(b)[:, None] * f).view(-1), idx, f, h, w)

    def score_rgb8(self, captions, frames, generator=None):
        """reward_scores of videos stored as bytes, uint8 RGB [b, f, H, W, 3] (CUDA), each byte read as x / 255: fp32 [b].
        The reference has no counterpart (it scores decoder output); this is the entry point for saved videos."""
        if frames.dim() != 5 or frames.shape[4] != 3 or frames.dtype != torch.uint8:
            raise ValueError(f"vgen_b200 reward: frames must be uint8 [b, f, H, W, 3], got {frames.dtype} {tuple(frames.shape)}")
        b, f, h, w, _ = frames.shape
        self._check(captions, b, frames, "frames")
        idx = self.indices(b, f, generator)
        return self._score(captions, frames.flatten(0, 1), (idx + torch.arange(b)[:, None] * f).view(-1), idx, f, h, w)


def main(argv=None):
    from .metric import read_video_rgb
    p = argparse.ArgumentParser("vgen_b200.reward", description="InstructVideo's segmental HPSv2 reward of saved videos")
    p.add_argument("--videos", required=True, help="directory of .mp4 files")
    p.add_argument("--captions", required=True, help="file of '<file name>|||<caption>' lines")
    p.add_argument("--hps", required=True, help="HPS_v2.pt")
    p.add_argument("--segments", type=int, default=4)
    p.add_argument("--selection", choices=SELECTION_METHODS, default="TSN")
    p.add_argument("--no_tar", action="store_true", help="plain segment mean (exponential_TSN off)")
    p.add_argument("--lambda_tar", type=float, default=1.0)
    p.add_argument("--antialias", action="store_true", help="torchvision >= 0.17's antialiased Resize")
    p.add_argument("--seed", type=int, default=0, help="seed of the TSN frame draw")
    a = p.parse_args(argv)
    captions = {}
    with open(a.captions, encoding="utf-8") as fh:
        for line in fh:
            if line.strip():
                name, cap = line.rstrip("\n").split("|||", 1)
                captions[name.strip()] = cap.strip()
    files = sorted(f for f in os.listdir(a.videos) if f.endswith(".mp4"))
    missing = [f for f in files if f not in captions]
    if missing:
        raise SystemExit(f"vgen_b200 reward: no caption for {missing}")
    scorer = SegmentalReward(load_hps(a.hps), segments=a.segments, selection_method=a.selection,
                             exponential_TSN=not a.no_tar, lambda_TAR=a.lambda_tar, antialias=a.antialias)
    gen = torch.Generator().manual_seed(a.seed)
    scores = []
    for f in files:
        frames = read_video_rgb(os.path.join(a.videos, f)).cuda()
        s = float(scorer.score_rgb8([captions[f]], frames[None], gen)[0])
        scores.append(s)
        print(f"{f}: {s:.6f}", flush=True)
    print(f"mean over {len(scores)} videos: {sum(scores) / max(len(scores), 1):.6f}")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
