"""Long-clip parity cases: the tiny UNets at frame counts past 32 (and past 64), inputs, product and oracle calls.

Every temporal attention of these cases runs over more frames than the register-resident kernel takes: the head_dim-64
TemporalTransformers go through the flash-style kernel, the 4- and 8-channel frame transformers (I2VGen's local temporal
encoder, the VideoComposer condition encoders) through the scalar kernel past 64 frames.  tools/make_golden_longclip.py
freezes the reference's outputs for these cases into tests/golden/longclip_<case>.npz and the digests of its parameter
lists into tests/golden/longclip_specs.json.  Spatial sizes stay small (4 x 6 latents) so the CPU reference run is quick.
"""
from __future__ import annotations

import json
import os

import torch

import _helpers
import _vcomp as vc
from oracle import synth
from oracle.cases import CASES, make_inputs as _base_inputs

LONG_CASES = {
    "t2v_f48": dict(kind="t2v", ctor=CASES["t2v_tiny"]["ctor"], seed=41, b=1, f=48, h=4, w=6, ntok=5, t=[613]),
    "t2v_b2_f80": dict(kind="t2v", ctor=CASES["t2v_tiny"]["ctor"], seed=42, b=2, f=80, h=4, w=6, ntok=5, t=[877, 143],
                       ddim=dict(steps=4, guide_scale=9.0)),
    "i2vgen_f72": dict(kind="i2vgen", ctor=CASES["i2vgen_tiny"]["ctor"], seed=43, b=1, f=72, h=4, w=6, ntok=5, t=[961]),
    # built like tests/_vcomp.py's cases: a 32 x 48 depth map pools 2 x 2 to resolution / 2 = 16 x 24, then two stride-2
    # convs reach the 4 x 6 latent
    "vcomp_f70": dict(kind="vcomp", cls="UNetSD_VideoLCM", ctor=CASES["videolcm_tiny"]["ctor"], comps=["text", "depthmap"],
                      resolution=[48, 32], seed=44, b=1, f=70, h=4, w=6, H=32, W=48, ntok=5, t=[259], conds=["depth"],
                      image=False),
}


def make_inputs(case):
    return vc.make_inputs(case) if case["kind"] == "vcomp" else _base_inputs(case)


def build_product(case):
    return vc.build_product(case) if case["kind"] == "vcomp" else _helpers.build_product(case)


def product_call(case, m, inp):
    if case["kind"] == "vcomp":
        return m(inp["x"], inp["t"], **vc.call_kwargs(case, inp))
    return _helpers.product_call(case, m, inp)


def oracle_call(case, sd, inp):
    return vc.oracle_call(case, sd, inp) if case["kind"] == "vcomp" else _helpers.oracle_call(case, sd, inp)


def product_spec(case):
    """(name, shape) list of the vgen_b200 class of a case (built on the meta device: nothing is allocated)."""
    if case["kind"] == "vcomp":
        return vc.product_spec(case["cls"], case["comps"], case["resolution"], case["ctor"])
    with torch.device("meta"):
        m = build_product(case)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def load_spec(golden_dir, name):
    """The parameter list of a case, checked against the reference's frozen digest before any weights are made from it."""
    spec = product_spec(LONG_CASES[name])
    want = json.load(open(os.path.join(golden_dir, "longclip_specs.json")))[name]
    assert vc.spec_digest(spec) == want, f"{name}: parameter list differs from the reference's"
    return spec


def state_dict(golden_dir, name):
    return synth.state_dict(load_spec(golden_dir, name), seed=LONG_CASES[name]["seed"])
