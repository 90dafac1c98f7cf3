"""Freeze the reference's outputs for the InstructVideo cases (tests/_instructvideo.py) into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it, see oracle/refload.py):
    python tools/make_golden_instructvideo.py
For each case it builds the reference UNetSD_LoRA on CPU, loads synthetic weights (oracle/synth.py) and runs it in fp32:
  * use_lora=True with lora_alpha None: the unmerged forward (LoRA.forward raises when lora_alpha is set, unet_lora.py:128-130);
  * lora_alpha set: the forward of the model get_lora_merged_model returns.  That function is lifted out of
    inference_instructvideo_entrance.py with `ast` (importing the entrance pulls in the whole engine stack) and run with
    a MODEL stand-in that builds the reference class;
  * use_lora=False: the plain forward.
The oracle restatement is checked against each output before anything is written: <case>.npz holds the output under the
case's weight seed, instructvideo_pin.npz the outputs under a second seed.  instructvideo_specs.json holds the digests of
the reference's parameter lists (tensor count, parameter count, sha256) for the cases and the released eval UNet with and
without LoRA.  instructvideo_video.npz holds the frames utils/video_op.py:save_video_local returns for fixed videos, with
os.system and cv2.imwrite stubbed (no file is written).
"""
from __future__ import annotations

import ast
import contextlib
import copy
import importlib
import io
import json
import logging
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import refload, synth  # noqa: E402
import _instructvideo as iv  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
PIN_SEED = 83


def _maxrel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def lift_get_lora_merged_model(ref_cls):
    src = os.path.join(refload.REF_ROOT, "tools/inferences/inference_instructvideo_entrance.py")
    tree = ast.parse(open(src).read())
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "get_lora_merged_model"]
    assert len(keep) == 1
    model_reg = types.SimpleNamespace(build=lambda cfg: ref_cls(**{k: v for k, v in cfg.items() if k != "type"}))
    ns = {"torch": torch, "deepcopy": copy.deepcopy, "logging": logging, "MODEL": model_reg}
    exec(compile(ast.Module(body=keep, type_ignores=[]), src, "exec"), ns)
    return ns["get_lora_merged_model"]


def reference_video_frames():
    """save_video_local's returned frames, with the encoder calls stubbed."""
    import cv2
    sys.modules.setdefault("imageio", types.ModuleType("imageio"))
    from utils import video_op
    real_system, real_imwrite = os.system, cv2.imwrite
    os.system = lambda cmd: 0
    cv2.imwrite = lambda path, img, *a: True
    out = {}
    try:
        for name in iv.VIDEOS:
            v, mean, std = iv.make_video(name)
            frames = video_op.save_video_local(f"/nonexistent/{name}.mp4", v.clone(), mean, std)
            out[name] = np.stack(frames)
    finally:
        os.system, cv2.imwrite = real_system, real_imwrite
    return out


def main():
    torch.set_grad_enabled(False)
    refload.load()
    ref_cls = importlib.import_module("tools.modules.unet.unet_lora").UNetSD_LoRA
    merge = lift_get_lora_merged_model(ref_cls)
    quiet = contextlib.redirect_stdout(io.StringIO())     # the reference prints one line per attention module
    pin, digests = {}, {}
    for name, case in iv.IV_CASES.items():
        with quiet:
            m = ref_cls(**case["ctor"]).eval()
        spec = synth.spec_of(m)
        assert spec == iv.product_spec(case["ctor"]), f"{name}: the product's parameter list differs from the reference's"
        inp = iv.make_inputs(case)
        for seed in (case["seed"], PIN_SEED):
            sd = iv.weights(spec, seed)
            m.load_state_dict(sd, strict=True)
            run = m
            if case.get("merged"):
                with quiet:
                    run = merge(model=m, cfg_UNet=dict(case["ctor"], type="UNetSD_LoRA"), gpu="cpu").eval()
                assert not run.use_lora
            out = run(inp["x"], inp["t"], inp["y"])
            err = _maxrel(iv.oracle_call(case, sd, inp), out)
            assert err < 2e-5, (name, seed, err)
            if case["ctor"]["use_lora"]:
                base = iv.unet_lora_forward({k: v for k, v in sd.items() if "_lora." not in k}, inp["x"], inp["t"], inp["y"])
                assert _maxrel(base, out) > 0.1, (name, seed, "the LoRA must move the output")
            print(f"{name} seed {seed}: oracle vs reference maxrel {err:.2e}")
            if seed == case["seed"]:
                np.savez_compressed(os.path.join(GOLD, name + ".npz"), out=out.numpy())
            else:
                pin[f"{name}_seed{seed}"] = out.numpy()
        digests[name] = iv.spec_digest(spec)
    np.savez_compressed(os.path.join(GOLD, "instructvideo_pin.npz"), **pin)
    for name, ctor in iv.RELEASED.items():
        with quiet, torch.device("meta"):
            m = ref_cls(**ctor)
        digests[name] = iv.spec_digest(synth.spec_of(m))
        assert (digests[name]["tensors"], digests[name]["parameters"]) == iv.RELEASED_COUNTS[name], (name, digests[name])
        print(f"{name}: {digests[name]}")
    with open(os.path.join(GOLD, "instructvideo_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)
    frames = reference_video_frames()
    np.savez_compressed(os.path.join(GOLD, "instructvideo_video.npz"), **frames)
    print({k: v.shape for k, v in frames.items()})


if __name__ == "__main__":
    main()
