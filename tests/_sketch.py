"""Sketch-annotator (PiDiNet + sketch-simplification GAN) parity cases: tiny constructors and shapes, the inputs, synthetic
weights and the parameter lists checked against the reference's frozen digests.

tools/make_golden_sketch.py freezes the reference's fp32 outputs for these cases into tests/golden/sketch_<case>.npz, and
into tests/golden/sketch_specs.json the digests of the tiny and full-size parameter lists and of the reference's PDC ->
vanilla conversion of a synthetic PDC-format state dict.
"""
from __future__ import annotations

import hashlib
import json
import math
import os

import numpy as np
import torch

from oracle import synth

CARV4 = ["cd", "ad", "rd", "cv"] * 4
TINY_PIDINET = dict(inplane=8, pdcs=CARV4, dil=4, sa=True, convert=True)
FULL_PIDINET = dict(inplane=60, pdcs=CARV4, dil=24, sa=True, convert=True)
GAN_MEAN, GAN_STD = 0.9664114577640158, 0.0858381272736797

SKETCH_CASES = {
    "pidinet_64x96": dict(net="pidinet", seed=31, n=1, H=64, W=96),
    "pidinet_60x100_b2": dict(net="pidinet", seed=37, n=2, H=60, W=100),     # odd sizes: every max-pool floors
    "cleaner_32x48": dict(net="cleaner", seed=41, n=1, H=32, W=48),
    "cleaner_64x96_b2": dict(net="cleaner", seed=43, n=2, H=64, W=96),
}


def make_input(net, n, H, W, seed):
    """PiDiNet: frames normalised with the ImageNet mean / std, as the engines feed them.  Cleaner: 1 - an edge map, as the
    engines feed it (a light background with darker strokes), in [0, 1]."""
    if net == "pidinet":
        return synth.tensor(f"sketch_x_{n}x{H}x{W}", (n, 3, H, W), 1.0, seed).clamp(-2.1, 2.6)
    t = synth.tensor(f"sketch_c_{n}x{H}x{W}", (n, 1, H, W), 1.0, seed)
    return (1.0 - 0.5 * torch.sigmoid(3.0 * t - 2.0)).clamp(0.0, 1.0)


def spec_digest(spec):
    """{tensors, parameters, sha256} of a (name, shape) list, as frozen in tests/golden/sketch_specs.json."""
    canon = json.dumps([[k, [int(d) for d in s]] for k, s in spec])
    params = sum(int(torch.Size(s).numel()) for _, s in spec)
    return {"tensors": len(spec), "parameters": params, "sha256": hashlib.sha256(canon.encode()).hexdigest()}


def tensor_digest(sd):
    """sha256 over the names, shapes and fp32 bytes of a state dict, in its order."""
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(json.dumps(list(v.shape)).encode())
        h.update(np.ascontiguousarray(v.detach().float().numpy()).tobytes())
    return h.hexdigest()


def product_spec(which):
    from vgen_b200.sketch import PiDiNet, SketchSimplification
    with torch.device("meta"):
        m = {"pidinet_tiny": lambda: PiDiNet(**TINY_PIDINET), "pidinet_full": lambda: PiDiNet(**FULL_PIDINET),
             "cleaner": lambda: SketchSimplification(GAN_MEAN, GAN_STD)}[which]()
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def load_spec(golden_dir, which):
    """which: "pidinet_tiny", "pidinet_full" or "cleaner"; the product's list, checked against the reference's digest."""
    spec = product_spec(which)
    want = json.load(open(os.path.join(golden_dir, "sketch_specs.json")))[which]
    assert spec_digest(spec) == want, f"{which}: parameter list differs from the reference's"
    return spec


# Synthetic weights (oracle/synth.py).  The cleaner's convs are He-scaled, so activations keep their scale through its depth.
# The last layers are scaled so the pre-sigmoid logits spread over the sigmoid's slope instead of saturating or collapsing;
# the factors were calibrated by measuring the outputs' spread on the tiny cases (see the non-vacuity checks).
PIDINET_GAIN = 0.7   # PiDiNet's residual stream adds every block's output: at He scale it outgrows fp16 by the last stage
PIDINET_OUT_SCALE = 4.0
CLEANER_OUT_SCALE = 10.0


def state_dict(spec, seed, net):
    sd = synth.state_dict(spec, seed=seed, gain=PIDINET_GAIN if net == "pidinet" else math.sqrt(2.0))
    if net == "pidinet":
        for k in sd:
            if k.startswith("conv_reduces.") or k.startswith("classifier."):
                sd[k] = sd[k] * PIDINET_OUT_SCALE
    else:
        last = max(int(k.split(".")[1]) for k in sd)
        sd[f"layers.{last}.weight"] = sd[f"layers.{last}.weight"] * CLEANER_OUT_SCALE
        sd[f"layers.{last}.bias"] = sd[f"layers.{last}.bias"] * CLEANER_OUT_SCALE
    return sd


def pdc_state_dict(spec, seed=5):
    """A synthetic checkpoint in the reference's pretrained format: 3x3 PDC weights where the converted model has 5x5 ones,
    every key prefixed with 'module.'."""
    sd = {}
    for k, s in spec:
        if s[-1] == 5:
            s = (*s[:-2], 3, 3)
        sd["module." + k] = synth.tensor("pdc:" + k, s, 0.3, seed)
    return sd


def non_vacuous(out):
    """(std, share of pixels below 0.01 or above 0.99) of a sigmoid output."""
    o = out.float()
    return float(o.std()), float(((o < 0.01) | (o > 0.99)).float().mean())



def full_state_dict(spec, net, seed=64):
    """Synthetic weights for pidinet_bsd() / sketch_simplification_gan(), drawn as state_dict() draws the tiny cases'."""
    return state_dict(spec, seed, net)
