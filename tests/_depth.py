"""Depth-annotator (MiDaS v3) parity cases: a tiny constructor at three input shapes, the inputs, and the parameter lists
checked against the reference's frozen digests.

tools/make_golden_depth.py freezes the reference's fp32 outputs for these cases into tests/golden/depth_<case>.npz and the
digests of its parameter lists (the tiny constructor and the full-size midas_v3()) into tests/golden/depth_specs.json.
"""
from __future__ import annotations

import hashlib
import json
import os

import torch

from oracle import synth

TINY = dict(image_size=64, patch_size=16, dim=128, neck_dims=[64, 64, 128, 128], fusion_dim=128, num_heads=2, num_layers=4)
FULL = dict(image_size=384, patch_size=16, dim=1024, neck_dims=[256, 512, 1024, 1024], fusion_dim=256, num_heads=16,
            num_layers=24)

DEPTH_CASES = {
    # 64 x 64 is the constructor's image_size: the position table is used at its own 4 x 4 grid
    "tiny_64": dict(ctor=TINY, seed=65, n=1, H=64, W=64),
    "tiny_64x96_b2": dict(ctor=TINY, seed=69, n=2, H=64, W=96),
    "tiny_96x160_b2": dict(ctor=TINY, seed=63, n=2, H=96, W=160),
}


def make_input(n, H, W, seed):
    """Images as the engines feed them: normalised to [-1, 1] (mean 0.5, std 0.5), fp32 NCHW."""
    return synth.tensor(f"depth_x_{n}x{H}x{W}", (n, 3, H, W), 0.6, seed).clamp(-1.0, 1.0)


def spec_digest(spec):
    """{tensors, parameters, sha256} of a (name, shape) list, as frozen in tests/golden/depth_specs.json."""
    canon = json.dumps([[k, [int(d) for d in s]] for k, s in spec])
    params = sum(int(torch.Size(s).numel()) for _, s in spec)
    return {"tensors": len(spec), "parameters": params, "sha256": hashlib.sha256(canon.encode()).hexdigest()}


def product_spec(ctor):
    from vgen_b200.depth import MiDaS
    with torch.device("meta"):
        m = MiDaS(**ctor)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def load_spec(golden_dir, which):
    """which: "tiny" or "full".  The product's parameter list, checked against the reference's frozen digest."""
    spec = product_spec(TINY if which == "tiny" else FULL)
    want = json.load(open(os.path.join(golden_dir, "depth_specs.json")))[which]
    assert spec_digest(spec) == want, f"{which}: parameter list differs from the reference's"
    return spec


def state_dict(spec, seed):
    """Synthetic weights (oracle/synth.py); a tensor that comes out all zero is drawn again under another name."""
    sd = synth.state_dict(spec, seed=seed)
    for k, v in sd.items():
        if not v.abs().max() > 0:
            sd[k] = synth.tensor(k + "#redraw", v.shape, 0.05, seed)
    return sd


def full_state_dict(spec, seed=64):
    """Synthetic weights for the full-size midas_v3(): as state_dict(), with head.4's weight negated.  Drawn as they come,
    the 32 -> 1 output projection sends all but a fraction of a percent of the pixels below zero, and the final ReLU
    would leave a map of zeros to compare."""
    sd = state_dict(spec, seed)
    sd["head.4.weight"] = -sd["head.4.weight"]
    return sd


def oracle_kw(ctor):
    return {k: ctor[k] for k in ("image_size", "patch_size", "num_heads", "num_layers")}
