"""InstructVideo segmental-reward parity cases: a tiny ViT-H/14-shaped HPS model, the tiny VAE decoder, synthetic
latents and captions.

tools/make_golden_reward.py runs the reference's own DiffRewardModel.reward_scorer on these cases and freezes into
tests/golden/reward_<case>.npz the token ids, the selected frame indices, a subsample of the resized and
normalised selected frames (every 8th row and column) with their sum, the image and text features, and reward_scores;
and into tests/golden/reward_specs.json the digests of the tiny and full-size HPS parameter lists.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from oracle import synth
from _sketch import spec_digest  # noqa: F401  (re-exported for the reward tests)

# ViT-H/14 shapes (224 px, patch 14, vision head width 80, text head dim 64) narrowed to 2 layers
TINY_HPS = dict(embed_dim=64, vision_cfg=dict(image_size=224, layers=2, width=320, head_width=80, patch_size=14),
                text_cfg=dict(context_length=77, vocab_size=49408, width=128, heads=2, layers=2))
# the VAE narrowed to 32 channels and one block per level, with the real model's 8x upsampling (4 levels), so that 256 x 256
# frames come from 32 x 32 latents as in training
VAE_TINY = dict(ddconfig=dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=32, ch_mult=[1, 1, 1, 1],
                              num_res_blocks=1, attn_resolutions=[], dropout=0.0), embed_dim=4)
HPS_SEED, VAE_SEED = 81, 82
SUB = 8                                     # the fixtures keep every SUB-th row and column of the tower's input

REWARD_CASES = {
    # the released training config's selection: TSN with the temporally attenuated reward, 16 frames in 4 segments,
    # 256 x 256 frames, torchvision 0.15's un-antialiased Resize
    "tsn_tar": dict(b=2, f=16, h=32, w=32, segments=4, selection="TSN", tar=True, antialias=False, seed=91,
                    captions=["a corgi running on the beach, oil painting", "an astronaut riding a horse"]),
    # fixed_first without TAR, 8 segments, torchvision >= 0.17's antialiased Resize
    "fixed_first": dict(b=2, f=16, h=32, w=32, segments=8, selection="fixed_first", tar=False, antialias=True, seed=92,
                        captions=["a red car driving through a snowy forest", "fireworks over a city at night"]),
    # 96 x 96 frames (upsampled to 224), TSN with TAR, antialias on
    "small_frames": dict(b=2, f=8, h=12, w=12, segments=4, selection="TSN", tar=True, antialias=True, seed=93,
                         captions=["a cat playing piano", "waves crashing on rocks at sunset"]),
}


def make_latents(name):
    c = REWARD_CASES[name]
    return synth.tensor(f"reward_{name}_x0", (c["b"], 4, c["f"], c["h"], c["w"]), 1.0, c["seed"])


def product_spec(which):
    from vgen_b200.clip import ARCHS, clip_spec
    return [(k, tuple(s)) for k, s in clip_spec(TINY_HPS if which == "hps_tiny" else ARCHS["ViT-H-14"])]


def hps_state_dict(spec, seed=HPS_SEED):
    """open_clip-format weights: synth.state_dict with open_clip's 0.02 scale for the embeddings."""
    sd = synth.state_dict([s for s in spec if len(s[1]) > 0], seed=seed)
    for k in ("positional_embedding", "visual.positional_embedding", "visual.class_embedding", "token_embedding.weight"):
        sd[k] = synth.tensor(k, dict(spec)[k], 0.02, seed)
    sd["logit_scale"] = torch.tensor(4.6052)
    return {k: sd[k] for k, _ in spec}


def vae_product():
    """The product's tiny AutoencoderKL and its synthetic weights (names as the reference's, so the same values)."""
    from vgen_b200.autoencoder import AutoencoderKL
    m = AutoencoderKL(**VAE_TINY)
    spec = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    return m, spec, synth.state_dict(spec, seed=VAE_SEED)


def load_spec(golden_dir, which):
    """which: hps_tiny / hps_full / vae_tiny; the product's list, checked against the reference's digest."""
    spec = vae_product()[1] if which == "vae_tiny" else product_spec(which)
    want = json.load(open(os.path.join(golden_dir, "reward_specs.json")))[which]
    assert spec_digest(spec) == want, f"{which}: parameter list differs from the reference's"
    return spec


def load_case(golden_dir, name):
    return dict(np.load(os.path.join(golden_dir, f"reward_{name}.npz")))
