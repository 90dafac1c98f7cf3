"""VideoComposer compositions of UNetSD_VideoLCM / UNetSD_TFT2V: parity cases, inputs and the oracle call.

The oracle of these cases is oracle/vgen_oracle.py's unet_videolcm_forward with the conditions, the image embedding and
the resolution, which restates the reference's condition encoders and image tokens (tools/modules/unet/unet_videolcm.py:
283-372, :598-745; unet_tf2tv.py is the same forward).  tools/make_golden_vcomp.py
freezes the reference's own outputs for these cases into tests/golden/ (vcomp_*.npz, tft2v_tiny.npz, vcomp_pin.npz) and
the reference's parameter lists as digests (vcomp_specs.json: tensor count, parameter count, sha256 of the list).
"""
from __future__ import annotations

import hashlib
import json
import os

import torch

from oracle import synth, vgen_oracle as vo
from oracle.vgen_oracle import ENCODERS, SUM_ORDER
from oracle.cases import CASES, FULL_CTORS, make_inputs as _base_inputs

RELEASED = ["text", "mask", "depthmap", "sketch", "motion", "image", "local_image", "single_sketch"]
EVERY = RELEASED + ["canny"]

_TINY = CASES["videolcm_tiny"]["ctor"]

VCOMP_CASES = {
    # every composition; conditions at 70 x 100 pool unevenly to resolution/2 = 32 x 48
    "vcomp_lcm_tiny": dict(cls="UNetSD_VideoLCM", ctor=_TINY, comps=EVERY, resolution=[96, 64], seed=31, b=1, f=4,
                           h=8, w=12, H=70, W=100, ntok=5, t=[377], conds=list(SUM_ORDER), image=True),
    # two videos, exact 2 x 2 pooling
    "vcomp_tft2v_tiny_b2": dict(cls="UNetSD_TFT2V", ctor=_TINY, comps=["text", "depthmap", "motion", "image"],
                                resolution=[96, 64], seed=32, b=2, f=3, h=8, w=12, H=64, W=96, ntok=5, t=[811, 95],
                                conds=["depth", "motion"], image=True),
    # the text-to-video call of inference_tft2v_entrance.py:204-207: y only
    "tft2v_tiny": dict(cls="UNetSD_TFT2V", ctor=_TINY, comps=["text", "image"], resolution=[96, 64], seed=33, b=1, f=4,
                       h=8, w=12, H=64, W=96, ntok=5, t=[505], conds=[], image=False),
}

# configs/tft2v_vcomposer_infer.yaml: the released composition list, 16 frames at 448 x 256
FULL_VCOMP_CASES = {
    "full_vcomposer": dict(cls="UNetSD_TFT2V", ctor=dict(FULL_CTORS["full_videolcm"][1]), comps=RELEASED,
                           resolution=[448, 256], seed=34, b=1, f=16, h=32, w=56, H=256, W=448, ntok=77, t=[721],
                           conds=["depth", "local_image", "motion", "sketch", "single_sketch", "masked"], image=True),
}
# the UNet section of configs/tft2v_vcomposer_infer.yaml, tft2v_t2v_infer.yaml and videolcm_vcomposer_infer.yaml as
# MODEL.build receives it (attn_scales is commented out there, so the class default [1/2, 1/4, 1/8] applies)
RELEASED_UNET = {"in_dim": 4, "dim": 320, "y_dim": 1024, "context_dim": 1024, "out_dim": 4, "dim_mult": [1, 2, 4, 4],
                 "num_heads": 8, "head_dim": 64, "num_res_blocks": 2, "dropout": 0.1, "temporal_attention": True,
                 "num_tokens": 4, "temporal_attn_times": 1, "use_checkpoint": True, "use_fps_condition": False,
                 "use_sim_mask": False}
# spec file -> (video_compositions, constructor kwargs)
FULL_SPECS = {"full_tft2v": (["text", "image"], FULL_VCOMP_CASES["full_vcomposer"]["ctor"]),
              "full_vcomposer": (RELEASED, FULL_VCOMP_CASES["full_vcomposer"]["ctor"]),
              "released_tft2v": (["text", "image"], RELEASED_UNET),
              "released_vcomposer": (RELEASED, RELEASED_UNET)}


def config_of(case):
    return dict(video_compositions=list(case["comps"]), resolution=list(case["resolution"]))


def make_inputs(case):
    """x / t / y / y_neg as oracle.cases.make_inputs, plus the case's pixel-space conditions and the image embedding."""
    base = dict(kind="videolcm", **{k: case[k] for k in ("seed", "b", "f", "h", "w", "ntok", "t")})
    d = _base_inputs(base)
    s = case["seed"] + 1000
    b, f = case["b"], case["f"]
    for kw in case["conds"]:
        d[kw] = synth.tensor("cond_" + kw, (b, ENCODERS[kw][2], f, case["H"], case["W"]), 0.5, s)
    if case["image"]:
        d["image"] = synth.tensor("image", (b, 1, 1024), 1.0, s)
    return d


def call_kwargs(case, inp):
    """Keyword arguments of the model call (the engines' names)."""
    kw = {"y": inp["y"]}
    for k in case["conds"]:
        kw[k] = inp[k]
    if case["image"]:
        kw["image"] = inp["image"]
    return kw


def spec_digest(spec):
    """{tensors, parameters, sha256} of a (name, shape) list, as frozen in tests/golden/vcomp_specs.json."""
    canon = json.dumps([[k, [int(d) for d in s]] for k, s in spec])
    params = sum(int(torch.Size(s).numel()) for _, s in spec)
    return {"tensors": len(spec), "parameters": params, "sha256": hashlib.sha256(canon.encode()).hexdigest()}


def reference_digest(golden_dir, name):
    return json.load(open(os.path.join(golden_dir, "vcomp_specs.json")))[name]


def product_spec(cls, comps, resolution, ctor):
    """(name, shape) list of the vgen_b200 class built with these arguments (on the meta device: nothing is allocated)."""
    import vgen_b200
    with torch.device("meta"):
        m = getattr(vgen_b200, cls)(config=dict(video_compositions=list(comps), resolution=list(resolution)), **ctor)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def load_spec(golden_dir, name, cases=None):
    """The parameter list of a case, checked against the reference's frozen digest before any weights are made from it."""
    case = (cases or VCOMP_CASES)[name]
    spec = product_spec(case["cls"], case["comps"], case["resolution"], case["ctor"])
    assert spec_digest(spec) == reference_digest(golden_dir, name), f"{name}: parameter list differs from the reference's"
    return spec


def oracle_call(case, sd, inp):
    kw = call_kwargs(case, inp)
    return vo.unet_videolcm_forward(sd, inp["x"], inp["t"], kw.pop("y"), resolution=case["resolution"], **kw)


def build_product(case):
    import vgen_b200
    return getattr(vgen_b200, case["cls"])(config=config_of(case), **case["ctor"])
