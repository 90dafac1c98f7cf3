"""Freeze the reference's InstructVideo reward (utils/reward/reward.py DiffRewardModel.reward_scorer, run unmodified) for
the cases of tests/_reward.py into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it):
    python tools/make_golden_reward.py
What the module needs is provided on the CPU as follows:
  * open_clip's `create_model_and_transforms`: returns the vendored open_clip `CLIP` built at the tiny ViT-H/14 shape of
    tests/_reward.py (output_dict=True) instead of downloading ViT-H-14; `get_tokenizer` returns the vendored tokenizer;
  * `torch.load('models/HPS_v2.pt')`: returns {'state_dict': the synthetic weights};
  * the `piq` and `skimage` imports, which reward_scorer does not use: empty modules;
  * the autoencoder: the reference's AutoencoderKL at tests/_reward.py's tiny configuration with synthetic weights;
  * `Resize(224)`: its `antialias` attribute is set per case (torchvision 0.15 leaves tensors un-antialiased, 0.17 and
    later antialias them).
The model runs in fp32 (the reference's fp16 HPS needs a GPU).  The tower's inputs, the TSN draw, the features and
reward_scores are recorded around the calls reward_scorer makes; the oracle (oracle/reward_oracle.py) is checked against
every one of them.  Only new files are written.
"""
from __future__ import annotations

import functools
import importlib
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _reward as rw  # noqa: E402
from oracle import refload, reward_oracle as ro, synth  # noqa: E402
from oracle.make_golden_clip import load_reference_open_clip  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _reference_reward_module(model_mod, tok_mod):
    for name in ("piq", "skimage", "skimage.metrics"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["piq"].ssim = sys.modules["piq"].SSIMLoss = None
    sys.modules["skimage.metrics"].structural_similarity = None
    oc = sys.modules["utils.reward.open_clip"]
    oc.create_model_and_transforms = None              # replaced per case below
    oc.get_tokenizer = lambda name: tok_mod.tokenize
    return importlib.import_module("utils.reward.reward")


def _cfg(case):
    return types.SimpleNamespace(
        reward_precision="fp16", selection_method=case["selection"], exponential_TSN=case["tar"], lambda_TAR=1.0,
        temporal_reward_type="", adv_clip_max=5.0, reward_weights={"reward": 1.0}, ST_reward_weights={"spatial": 1.0, "temporal": 0.0},
        motion_rep=None, low_penal_threshold=None, scale_factor=0.18215, decoder_bs=1, use_fp16=False, data_align_method=None)


def _recording(fn, sink, pick=lambda o: o):
    @functools.wraps(fn)
    def run(*a, **k):
        out = fn(*a, **k)
        sink.append(pick(out))
        return out
    return run


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


def main():
    torch.set_grad_enabled(False)
    refload.require_root()
    ref = refload.load()
    model_mod, tok_mod = load_reference_open_clip()
    reward_mod = _reference_reward_module(model_mod, tok_mod)

    def build_clip(cfg):
        v, t = cfg["vision_cfg"], cfg["text_cfg"]
        return model_mod.CLIP(cfg["embed_dim"], model_mod.CLIPVisionCfg(**v), model_mod.CLIPTextCfg(**t), output_dict=True)

    from vgen_b200.clip import ARCHS
    with torch.device("meta"):
        full = build_clip(ARCHS["ViT-H-14"])
    specs = {"hps_full": synth.spec_of(full), "hps_tiny": synth.spec_of(build_clip(rw.TINY_HPS))}
    digests = {k: rw.spec_digest(v) for k, v in specs.items()}
    hsd = rw.hps_state_dict(specs["hps_tiny"])
    vae = ref.AutoencoderKL(**rw.VAE_TINY).eval()
    vsd = synth.state_dict(synth.spec_of(vae), seed=rw.VAE_SEED)
    specs["vae_tiny"] = synth.spec_of(vae)
    digests["vae_tiny"] = rw.spec_digest(specs["vae_tiny"])
    vae.load_state_dict(vsd, strict=True)

    for name, case in rw.REWARD_CASES.items():
        clip = build_clip(rw.TINY_HPS)
        clip.load_state_dict(hsd, strict=True)
        reward_mod.create_model_and_transforms = lambda *a, **k: (clip, None, None)
        load = torch.load
        torch.load = lambda path, *a, **k: {"state_dict": hsd} if str(path).endswith("HPS_v2.pt") else load(path, *a, **k)
        try:
            scorer = reward_mod.DiffRewardModel("HPSv2", _cfg(case), vae, segments=case["segments"], reward_normalization=False)
        finally:
            torch.load = load
        scorer.diff_resize.antialias = case["antialias"]
        rec = {k: [] for k in ("norm", "randint", "feat", "cat")}
        scorer.diff_normalize = _recording(scorer.diff_normalize, rec["norm"])
        clip.forward = _recording(clip.forward, rec["feat"], lambda o: (o["image_features"], o["text_features"]))
        x0 = rw.make_latents(name)
        randint, cat = torch.randint, torch.cat
        torch.randint, torch.cat = _recording(randint, rec["randint"]), _recording(cat, rec["cat"])
        try:
            torch.manual_seed(case["seed"])
            loss = scorer.reward_scorer(case["captions"], x0, None, 0)
        finally:
            torch.randint, torch.cat = randint, cat
        scores = rec["cat"][-1]
        b, f, s = case["b"], case["f"], case["segments"]
        assert scores.shape == (b,) and abs(float(loss) - float((1 - scores).mean())) < 1e-6
        span = f // s
        if case["selection"] == "TSN":
            assert len(rec["randint"]) == 1
            idx = rec["randint"][0] + torch.arange(s)[None] * span
        else:
            idx = torch.arange(0, f, span)[None].expand(b, s)
        pre = rec["norm"][0].reshape(b, f, *rec["norm"][0].shape[1:])
        sel = pre[torch.arange(b)[:, None], idx].reshape(b * s, *pre.shape[2:])
        img = torch.cat([o[0] for o in rec["feat"]])
        txt = torch.cat([o[1] for o in rec["feat"]])
        tokens = tok_mod.tokenize(case["captions"])
        out = {"tokens": tokens.numpy(), "idx": idx.numpy(), "pre_sub": sel[:, :, ::rw.SUB, ::rw.SUB].numpy(),
               "pre_sum": sel.double().sum((1, 2, 3)).numpy(), "image_features": img.numpy(), "text_features": txt.numpy(),
               "reward_scores": scores.numpy()}
        # the oracle against every recorded value
        video = ro.decode(vsd, x0)
        clamped = float(((video * 0.5 + 0.5 < 0) | (video * 0.5 + 0.5 > 1)).float().mean())
        o_pre = ro.preprocess(video, case["antialias"])
        o_sel = o_pre[torch.arange(b)[:, None], idx].reshape(b * s, *o_pre.shape[2:])
        o_img, o_txt = ro.features(hsd, o_sel, tokens.long(), rw.TINY_HPS["vision_cfg"]["head_width"], rw.TINY_HPS["text_cfg"]["heads"])
        o_scores = ro.reward_scores(o_img, o_txt, idx, f, case["tar"])
        rep = {"pre": _rel(o_sel, sel), "img": _rel(o_img, img), "txt": _rel(o_txt, txt), "scores": _rel(o_scores, scores)}
        assert max(rep.values()) < 1e-5, (name, rep)
        print(f"{name}: idx {idx.tolist()}, reward_scores {scores.tolist()}, {clamped:.1%} of samples clamped, "
              f"oracle vs reference {rep}", flush=True)
        np.savez_compressed(os.path.join(GOLD, f"reward_{name}.npz"), **out)
    with open(os.path.join(GOLD, "reward_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)
    for k in ("hps_full", "hps_tiny"):
        print(f"{k}: {digests[k]['parameters']} parameters in {digests[k]['tensors']} tensors")


if __name__ == "__main__":
    main()
