"""H100-native DreamVideo evaluation metric: a drop-in for metric/cal_metric_DreamVideo.py.

The paper's four scores of a generated video:
  CLIP-T                cosine of the prompt's CLIP text feature with the mean of the frames' CLIP image features
  CLIP-I                the same against the CLIP features of the subject's reference images, averaged over them
  DINO-I                CLIP-I with DINO ViT-S/16 features
  temporal consistency  mean CLIP cosine of consecutive frames

`calculate_metric` keeps the reference's signature, return value and printed line.  The models come from `load_clip`
(OpenAI's CLIP in the checkpoint format `clip.load` reads, without the `clip` package) and `vgen_b200.dino.vit_small`;
the preprocess arguments are the transform objects `load_clip` and `dino_transform()` return.  Videos are decoded with
cv2 and reference images with PIL on the host, as in the reference, and uploaded once as bytes; after that everything
runs on libvgen_b200.so kernels: the resize / crop / normalise of every frame and image (bit-exact with the reference's
PIL + torchvision transforms, metric.cu), both ViTs, and the scores (one launch per video).  `score_video` takes frames
that are already on the GPU, e.g. `ops.video_to_rgb8`'s output, so a generated clip can be scored without writing it.

    python -m vgen_b200.metric --videos_dir_path DIR --prompts_path FILE --clip_checkpoint ViT-B-32.pt \\
        --dino_checkpoint dino_deitsmall16_pretrain.pth
mirrors the reference's __main__; only the two checkpoint paths are arguments.
"""
from __future__ import annotations

import argparse
import math
import os
import time

import numpy as np
import torch

from . import ops
from .clip import OpenAIClipModel, openai_cfg
from .clip_tokenizer import tokenize

OPENAI_MEAN, OPENAI_STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
_PRECISION_BITS = 22                          # Pillow's 8-bit resample: 32 - 8 - 2 fractional bits
_TILE_ROWS = 16                               # output rows per block of the resize kernel


# ---- Pillow's bicubic coefficients (libImaging/Resample.c precompute_coeffs + normalize_coeffs_8bpc) -----------------
def _bicubic(x):
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def pillow_bicubic_coeffs(in_size, out_size):
    """Fixed-point bicubic weights of an in_size -> out_size resample, computed in double precision exactly as Pillow
    does: -> (bounds int32 [out, 2] = (first input index, taps), weights int32 [out, ksize])."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    one, ss = 1 << _PRECISION_BITS, 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)                 # C (int) truncation
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x, v in enumerate(w):
            v = v / ww if ww != 0.0 else v
            kk[xx, x] = int(-0.5 + v * one) if v < 0 else int(0.5 + v * one)   # round half away from zero
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def resized_size(h, w, size):
    """torchvision's Resize(int) output (h, w): the short side becomes `size`, the long one int(size * long / short)."""
    if w <= h:
        return int(size * h / w), size
    return size, int(size * w / h)


class ResizePlan:
    """Resize(resize, BICUBIC) -> CenterCrop(crop) -> Normalize(mean, std) of h x w images: Pillow's tables for the crop's
    rows and columns (host, once per size), moved to a device on first use."""

    def __init__(self, h, w, resize, crop, mean, std):
        self.h, self.w, self.mean, self.std = h, w, mean, std
        rh, rw = resized_size(h, w, resize)
        if rh < crop or rw < crop:
            raise ValueError(f"vgen_b200 metric: a {h}x{w} image resized to {rh}x{rw} is smaller than the {crop} crop")
        self.crop_h = self.crop_w = crop
        top, left = int(round((rh - crop) / 2.0)), int(round((rw - crop) / 2.0))
        self.hb, self.hk = self._axis(w, rw, left, crop)
        self.vb, self.vk = self._axis(h, rh, top, crop)
        last = [min(r + _TILE_ROWS, crop) - 1 for r in range(0, crop, _TILE_ROWS)]
        self.tile_rows = max(int(self.vb[e, 0] + self.vb[e, 1] - self.vb[r, 0]) for r, e in zip(range(0, crop, _TILE_ROWS), last))
        self._dev = {}

    @staticmethod
    def _axis(n_in, n_out, off, crop):
        if n_in == n_out:                     # Pillow does not resample an axis whose size is unchanged: identity taps
            b = np.stack([np.arange(off, off + crop), np.ones(crop, np.int64)], 1).astype(np.int32)
            return b, np.full((crop, 1), 1 << _PRECISION_BITS, np.int32)
        b, k = pillow_bicubic_coeffs(n_in, n_out)
        return np.ascontiguousarray(b[off:off + crop]), np.ascontiguousarray(k[off:off + crop])

    def tables(self, device):
        t = self._dev.get(device)
        if t is None:
            t = self._dev[device] = tuple(torch.from_numpy(a).to(device) for a in (self.hb, self.hk, self.vb, self.vk))
        return t


class ImageTransform:
    """The preprocess object of the metric: Resize(resize, BICUBIC) -> CenterCrop(crop) -> ToTensor -> Normalize(mean,
    std), bit-exact with torchvision on PIL images, run by the resize kernel.  Calling it on one image (PIL, or a uint8
    [H, W, 3] array / tensor) returns the fp32 [3, crop, crop] tensor torchvision returns, on `device`."""

    def __init__(self, resize, crop, mean, std, device="cuda"):
        self.resize, self.crop, self.mean, self.std, self.device = int(resize), int(crop), tuple(mean), tuple(std), device
        self._plans = {}

    def __repr__(self):
        return (f"ImageTransform(Resize({self.resize}, BICUBIC), CenterCrop({self.crop}), ToTensor(), "
                f"Normalize({self.mean}, {self.std}))")

    def plan(self, h, w):
        p = self._plans.get((h, w))
        if p is None:
            p = self._plans[(h, w)] = ResizePlan(h, w, self.resize, self.crop, self.mean, self.std)
        return p

    def batch(self, images, out_f32=False, out=None):
        """uint8 [n, H, W, 3] CUDA -> fp16 channels-last [n, crop, crop, 3] (the towers' input) or fp32 [n, 3, crop, crop]
        (into `out` if given)."""
        images = images.contiguous()
        return ops.resize_crop_normalize(images, self.plan(images.shape[1], images.shape[2]), out_f32, out)

    def images(self, images, device, out_f32=False):
        """A list of RGB images of any sizes (PIL, or uint8 [H_i, W_i, 3] arrays / tensors) -> one batch in list order on
        `device`: each image is uploaded as bytes and transformed by its own launch."""
        c = self.crop
        shape = (len(images), 3, c, c) if out_f32 else (len(images), c, c, 3)
        out = torch.empty(shape, device=device, dtype=torch.float32 if out_f32 else torch.float16)
        for i, im in enumerate(images):
            self.batch(_to_device_u8(im, device)[None], out_f32, out[i:i + 1])
        return out

    def __call__(self, img):
        return self.batch(_to_device_u8(img, self.device)[None], out_f32=True)[0]


def _to_device_u8(img, device):
    if torch.is_tensor(img):
        t = img
    else:
        if hasattr(img, "mode") and img.mode != "RGB":
            img = img.convert("RGB")
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(img)))
    if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
        raise ValueError(f"vgen_b200 metric: expected an RGB image as uint8 [H, W, 3], got {t.dtype} {tuple(t.shape)}")
    return t.to(device).contiguous()


def clip_transform(image_size=224, device="cuda"):
    """OpenAI CLIP's _transform(n_px): Resize(n_px, BICUBIC), CenterCrop(n_px), ToTensor, Normalize(OpenAI mean / std)."""
    return ImageTransform(image_size, image_size, OPENAI_MEAN, OPENAI_STD, device)


def dino_transform(device="cuda"):
    """The metric's DINO preprocess: Resize(256, interpolation=3 = BICUBIC), CenterCrop(224), ToTensor,
    Normalize(ImageNet mean / std)."""
    return ImageTransform(256, 224, IMAGENET_MEAN, IMAGENET_STD, device)


# ---- CLIP checkpoints -----------------------------------------------------------------------------------------------------
_OPENAI_FILES = {"ViT-B/32": "ViT-B-32.pt", "ViT-B/16": "ViT-B-16.pt", "ViT-L/14": "ViT-L-14.pt",
                 "ViT-L/14@336px": "ViT-L-14-336px.pt"}
_OPENAI_RESNETS = ("RN50", "RN101", "RN50x4", "RN50x16", "RN50x64")
_TORCHSCRIPT_EXTRA = ("input_resolution", "context_length", "vocab_size")


def _read_state_dict(path):
    try:                                               # OpenAI's released files are TorchScript archives
        return torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        return torch.load(path, map_location="cpu")


def load_clip(name_or_path, device="cuda"):
    """Replaces clip.load: -> (model, transform).  name_or_path is a checkpoint path (OpenAI's TorchScript file or a plain
    state dict) or a model name, which resolves to ~/.cache/clip/<file> if that file exists.  Nothing is downloaded."""
    if name_or_path in _OPENAI_RESNETS:
        raise NotImplementedError(f"vgen_b200 CLIP: {name_or_path} is a ModifiedResNet model; only the ViT models are supported")
    if name_or_path in _OPENAI_FILES:
        path = os.path.join(os.path.expanduser("~/.cache/clip"), _OPENAI_FILES[name_or_path])
        if not os.path.isfile(path):
            raise FileNotFoundError(f"vgen_b200 CLIP: {name_or_path} needs its checkpoint at {path} (nothing is downloaded)")
    elif os.path.isfile(name_or_path):
        path = name_or_path
    else:
        raise FileNotFoundError(f"vgen_b200 CLIP: {name_or_path} is neither a checkpoint file nor one of {sorted(_OPENAI_FILES)}")
    sd = {k: v for k, v in _read_state_dict(path).items() if k not in _TORCHSCRIPT_EXTRA}
    cfg = openai_cfg(sd)
    model = OpenAIClipModel(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.eval().requires_grad_(False).to(device)
    return model, clip_transform(cfg["vision_cfg"]["image_size"], device)


# ---- scores ---------------------------------------------------------------------------------------------------------------
def _check_preprocess(clip_preprocess, dino_preprocess):
    for nm, t in (("clip_preprocess", clip_preprocess), ("dino_preprocess", dino_preprocess)):
        if not isinstance(t, ImageTransform):
            raise TypeError(f"vgen_b200 metric: {nm} must be the transform vgen_b200.metric.load_clip / dino_transform() "
                            f"returns (its resize runs on the GPU), got {type(t).__name__}")


@torch.no_grad()
def score_video(frames, prompt, target_images, clip_model, clip_preprocess, dino_model, dino_preprocess):
    """The four scores of one video whose RGB frames are already on the GPU.

    frames: uint8 CUDA [f, H, W, 3]; prompt: str; target_images: list of RGB images (PIL, or uint8 [H, W, 3] arrays /
    tensors), may be empty.  -> CUDA fp32 [4] = (CLIP-T, CLIP-I, DINO-I, temporal consistency), nothing synchronised."""
    _check_preprocess(clip_preprocess, dino_preprocess)
    if not torch.is_tensor(frames) or not frames.is_cuda:
        raise ops._l.VgenError("vgen_b200 metric: frames must be a CUDA tensor (no CPU path exists)")
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3 or frames.shape[0] < 1:
        raise ValueError(f"vgen_b200 metric: frames must be uint8 [f >= 1, H, W, 3], got {frames.dtype} {tuple(frames.shape)}")
    dev = frames.device
    text = clip_model.encode_text(tokenize([prompt], truncate=False))[0]
    clip_f = clip_model.encode_image_nhwc(clip_preprocess.batch(frames))
    dino_f = dino_model.forward_nhwc(dino_preprocess.batch(frames))
    clip_t = dino_t = None
    if len(target_images):
        clip_t = clip_model.encode_image_nhwc(clip_preprocess.images(target_images, dev))
        dino_t = dino_model.forward_nhwc(dino_preprocess.images(target_images, dev))
    return ops.video_scores(clip_f, text, clip_t, dino_f, dino_t)


def read_video_rgb(path):
    """All frames of a video as uint8 [f, H, W, 3] RGB, decoded with cv2 as the reference does."""
    import cv2
    cap = cv2.VideoCapture(path)
    frames = []
    while True:
        ret, frame = cap.read()
        if (not ret) or (frame is None):
            break
        frames.append(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB))
    if not frames:
        raise ValueError(f"vgen_b200 metric: no frames could be read from {path}")
    return torch.from_numpy(np.stack(frames))


def read_image_rgb(path):
    from PIL import Image
    image = Image.open(path)
    if image.mode != "RGB":
        image = image.convert("RGB")
    return np.asarray(image)


def calculate_metric(videos_path, prompt, target_img_files, clip_model, clip_preprocess, dino_model, dino_preprocess,
                     chunk_size=1):
    """cal_metric_DreamVideo.py:22-142: -> (CLIP-T, CLIP-I, DINO-I, temporal consistency) of one video file; CLIP-I and
    DINO-I are 0 without target images, the temporal consistency of a one-frame video is NaN."""
    _check_preprocess(clip_preprocess, dino_preprocess)
    if chunk_size != 1:
        raise ValueError("vgen_b200 metric: calculate_metric scores one video; chunk_size must be 1")
    frames = read_video_rgb(videos_path)
    targets = [read_image_rgb(f) for f in target_img_files]
    dev = clip_model.device
    s = score_video(frames.to(dev), prompt, targets, clip_model, clip_preprocess, dino_model, dino_preprocess).tolist()
    clip_t, tc = s[0], s[3]
    clip_i, dino_i = (s[1], s[2]) if targets else (0, 0)
    print(f'CLIP-T: {clip_t:.4f}, CLIP-I: {clip_i:.4f}, DINO-I: {dino_i:.4f}, TemporalConsistency: {tc:.4f}')
    return clip_t, clip_i, dino_i, tc


def main(argv=None):
    from .dino import vit_small
    parser = argparse.ArgumentParser("Important args")
    parser.add_argument("--videos_dir_path", type=str, help="")
    parser.add_argument("--prompts_path", type=str, help="path of the prompts file")
    parser.add_argument("--clip_checkpoint", type=str, default="ViT-B/32", help="OpenAI CLIP checkpoint or model name")
    parser.add_argument("--dino_checkpoint", type=str, required=True, help="dino_deitsmall16_pretrain.pth")
    args = parser.parse_args(argv)

    clip_model, clip_preprocess = load_clip(args.clip_checkpoint, device="cuda")
    dino_vits16 = vit_small()
    dino_vits16.load_state_dict(torch.load(args.dino_checkpoint, map_location="cpu"))
    dino_vits16 = dino_vits16.eval().cuda()
    dino_preprocess = dino_transform()

    video_files = [os.path.join(args.videos_dir_path, f) for f in os.listdir(args.videos_dir_path)
                   if f.endswith(".mp4") or f.endswith(".gif")]
    prompts_dict = {}
    with open(args.prompts_path, "r", encoding="utf-8") as prompts_file:
        for line in prompts_file:
            parts = line.strip().split("|||")
            prompts_dict[parts[0]] = (parts[1], parts[2])
    print(f"-----------------test {len(video_files)} videos for video customization!---------------")
    if len(video_files) != len(prompts_dict):
        print(f"The number of videos {len(video_files)} and text prompts {len(prompts_dict)} are inconsistent!!")
        return 1
    lists = ([], [], [], [])
    for idx, video in enumerate(video_files):
        video_name = video.split("/")[-1]
        image_dir, prompt = prompts_dict[video_name]
        image_name = image_dir.split("/")[-1]
        target_img_files = [os.path.join(image_dir, f) for f in os.listdir(image_dir) if f.endswith(".jpg")]
        print(f"test {idx}th video {video_name}---{image_name}---{prompt}")
        for lst, v in zip(lists, calculate_metric(video, prompt, target_img_files, clip_model, clip_preprocess, dino_vits16,
                                                  dino_preprocess)):
            lst.append(v)
    m = [sum(lst) / len(lst) for lst in lists]
    print(time.strftime("%Y-%m-%d %H:%M:%S", time.localtime()),
          f"Final CLIP-T: {m[0]:.4f}, CLIP-I: {m[1]:.4f}, DINO-I: {m[2]:.4f},  TemporalConsistency: {m[3]:.4f}")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
