"""DreamVideo's text path (FrozenOpenCLIPCustomEmbedder + EmbeddingManager) and DDIM inversion: cases, the tiny CLIP and
the learned vectors, shared by tools/make_golden_dreamvideo_text.py and the tests.

The tiny CLIP is the one of tests/golden/clip_tiny.* (oracle/make_golden_clip.py: text width 128, 3 blocks).  Each case
builds a manager with the reference's constructor arguments and then overwrites every placeholder's vectors with
`learned_vectors(...)`, so the substitution is seen with vectors unlike any vocabulary row.
"""
from __future__ import annotations

import json
import os

import torch

from oracle import synth

GOLDEN = "dreamvideo_text.npz"
CKPT = "dreamvideo_text_ckpt.pt"        # written by the reference's EmbeddingManager.save (case "two_placeholders")
CKPT_CASE = "two_placeholders"
WIDTH = 128

TEXT_CASES = {
    "single": dict(prompts=["a * running on the road"], placeholders=["*"], init=["dog"], per_image=False, nv=1,
                   layer="penultimate"),
    "twice_b2": dict(prompts=["a * and a * on the grass", "a photo of *"], placeholders=["*"], init=["dog"],
                     per_image=False, nv=1, layer="last"),
    # three vectors per token; the second prompt's insertion pushes the end-of-text token past position 76
    "multi3": dict(prompts=["a * with a * friend", "a " * 73 + "*"], placeholders=["*"], init=["dog"], per_image=False,
                   nv=3, layer="penultimate"),
    "two_placeholders": dict(prompts=["a * chasing a @ in the park", "@ and *"], placeholders=["*", "@"],
                             init=["dog", "cat"], per_image=False, nv=2, layer="last"),
    # the 22 Hebrew-letter placeholders all start with the same BPE piece: the last one wins
    "per_image": dict(prompts=["a * and a א near a ת"], placeholders=["*"], init=["dog"], per_image=True, nv=1,
                      layer="penultimate"),
    "no_placeholder": dict(prompts=["a photo of a dog"], placeholders=["*"], init=["dog"], per_image=False, nv=1,
                           layer="last"),
}

# the DDIM inversion pin: the t2v_tiny UNet (oracle/cases.py) under DreamVideo's Diffusion section
# (configs/dreamvideo/*: linear_sd, eps, fixed_small), x0 = the case's x, context = the case's y_neg
REVERSE_CASE = "t2v_tiny"
REVERSE_STEPS = (4, 20)
REVERSE_DIFFUSION = dict(schedule="linear_sd", schedule_param=dict(num_timesteps=1000, init_beta=0.00085, last_beta=0.012,
                                                                   zero_terminal_snr=False),
                         mean_type="eps", var_type="fixed_small")

# the released step-2 subject config's embedder / embedmanager sections
# (configs/dreamvideo/subjectLearning/dog2_subjectLearning_step2.yaml:18-31)
RELEASED_EMBEDDER = {"type": "FrozenOpenCLIPCustomEmbedder", "layer": "penultimate", "vit_resolution": [224, 224],
                     "pretrained": "models/open_clip_pytorch_model.bin"}
RELEASED_EMBEDMANAGER = {"type": "EmbeddingManager", "placeholder_strings": ["*"], "initializer_words": ["dog"],
                         "per_image_tokens": False, "num_vectors_per_token": 1, "progressive_words": False}


def placeholder_list(case):
    from vgen_b200.embedding_manager import PER_IMG_TOKEN_LIST
    return list(case["placeholders"]) + (list(PER_IMG_TOKEN_LIST) if case["per_image"] else [])


def learned_vectors(name, case):
    """[n_placeholders, nv, WIDTH] fp32, in the manager's dict order."""
    return synth.tensor(f"dreamvideo_text:{name}", (len(placeholder_list(case)), case["nv"], WIDTH), 0.05, 7)


def tiny_clip_state_dict(golden_dir):
    """The tiny CLIP's weights exactly as tests/test_oracle_golden.py makes them."""
    spec = [(k, tuple(s)) for k, s in json.load(open(os.path.join(golden_dir, "clip_tiny.spec.json")))]
    sd = synth.state_dict([s for s in spec if len(s[1]) > 0], seed=31)
    for k in ("positional_embedding", "visual.positional_embedding", "visual.class_embedding", "token_embedding.weight"):
        sd[k] = synth.tensor(k, dict(spec)[k], 0.02, 31)
    sd["logit_scale"] = torch.tensor(2.6592)
    return sd


def use_golden_tokenizer(golden_dir, monkeypatch):
    """Point vgen_b200.clip_tokenizer at the committed merge list (the suite needs no open_clip)."""
    from vgen_b200 import clip_tokenizer as ct
    monkeypatch.setenv("VGEN_CLIP_BPE", os.path.join(golden_dir, "clip_bpe_merges_head.txt.gz"))
    monkeypatch.setattr(ct, "_DEFAULT", None)
