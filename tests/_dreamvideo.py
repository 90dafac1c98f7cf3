"""DreamVideo (UNetSD_DreamVideo): parity cases, inputs and the oracle call.

The oracle of these cases is oracle/vgen_oracle.py's unet_dreamvideo_forward, which restates
tools/modules/unet/unet_dreamvideo.py:225-290 and the adapters of util.py:499-519,603-672 (BasicTransformerBlockWithAdapter,
SpatialTransformerWithAdapter, TemporalTransformerWithAdapter) in the shared trunk.  It takes ag_strength per sample, which the
reference does not; tools/make_golden_dreamvideo.py therefore freezes the reference's outputs of a multi-lambda batch by
running it one video at a time (videos never interact).
Parameter lists of the reference are frozen as digests in tests/golden/dreamvideo_specs.json.
"""
from __future__ import annotations

import json
import os

import torch

from oracle import synth, vgen_oracle as vo
from oracle.cases import _T2V_TINY, make_inputs as _base_inputs
from _vcomp import spec_digest  # noqa: F401  (same digest format as vcomp_specs.json)

MOTION = ["self_attention", "cross_attention", "feedforward"]
SUBJECT = ["cross_attention"]

# ctor: the reference's constructor kwargs; ag: ag_strength per video; yi_frames: 1 ([b, 1, C]) or f ([b, f, C]) or None
DV_CASES = {
    "dv_subject_tiny": dict(ctor=dict(_T2V_TINY, spatial_adapter_list=SUBJECT), seed=41, b=1, f=4, h=8, w=12, ntok=5,
                            t=[613], yi_frames=None, ag=None),
    "dv_motion_tiny": dict(ctor=dict(_T2V_TINY, temporal_adapter_list=MOTION, temporal_adapter_condition_dim=1024), seed=42,
                           b=1, f=4, h=8, w=12, ntok=5, t=[377], yi_frames=1, ag=[1.0]),
    "dv_motion_frames_tiny": dict(ctor=dict(_T2V_TINY, temporal_adapter_list=MOTION, temporal_adapter_condition_dim=1024),
                                  seed=43, b=1, f=3, h=6, w=10, ntok=5, t=[95], yi_frames=3, ag=[0.7]),
    "dv_joint_tiny_b2": dict(ctor=dict(_T2V_TINY, spatial_adapter_list=SUBJECT, temporal_adapter_list=MOTION,
                                       temporal_adapter_condition_dim=1024), seed=44, b=2, f=3, h=8, w=6, ntok=7,
                             t=[811, 95], yi_frames=1, ag=[1.0, 0.5]),
    # serial positions, every site, a given hidden width (48 -> padded 64)
    "dv_serial_tiny": dict(ctor=dict(_T2V_TINY, spatial_adapter_list=MOTION, spatial_adapter_position_list=["serial", "parallel", "serial"],
                                     spatial_adapter_hidden_dim=48, temporal_adapter_list=["self_attention", "feedforward"],
                                     temporal_adapter_position_list=["serial", "parallel", "serial"],
                                     temporal_adapter_condition_dim=1024), seed=45, b=1, f=4, h=8, w=12, ntok=5, t=[500],
                           yi_frames=1, ag=[1.0]),
}

# the UNet section of configs/dreamvideo/{subjectLearning/*_step2, motionLearning/*}.yaml merged into
# tools/modules/config.py's cfg.UNet as the entrance does (so dim = 320 and attn_scales = [1, 1/2, 1/4] come from there)
RELEASED_UNET = {"in_dim": 4, "dim": 320, "y_dim": 1024, "upper_len": 128, "context_dim": 1024, "out_dim": 4,
                 "dim_mult": [1, 2, 4, 4], "num_heads": 8, "default_fps": 8, "head_dim": 64, "num_res_blocks": 2,
                 "attn_scales": [1 / 1, 1 / 2, 1 / 4], "dropout": 0.1, "misc_dropout": 0.4, "temporal_attention": True,
                 "temporal_attn_times": 1, "use_checkpoint": True, "use_fps_condition": False, "use_sim_mask": False}
RELEASED_ADAPTERS = {
    "released_base": {},
    "released_subject": {"spatial_adapter_list": SUBJECT},
    "released_motion": {"temporal_adapter_list": MOTION, "temporal_adapter_condition_dim": 1024},
    "released_joint": {"spatial_adapter_list": SUBJECT, "temporal_adapter_list": MOTION, "temporal_adapter_condition_dim": 1024},
}
RELEASED_COUNTS = {"released_base": (1480, 1411233860), "released_subject": (1544, 1423642980),
                   "released_motion": (1786, 1489200356), "released_joint": (1850, 1501609476)}

# the joint flavour at the released shape: 32 frames, 256 x 256 pixels (32 x 32 latent), 77 tokens
FULL_DV_CASES = {
    "full_dv_joint": dict(ctor=dict(RELEASED_UNET, **RELEASED_ADAPTERS["released_joint"]), seed=46, b=1, f=32, h=32, w=32,
                          ntok=77, t=[721], yi_frames=1, ag=[1.0], spec="released_joint"),
}


def make_inputs(case):
    """x / t / y / y_neg as oracle.cases.make_inputs, plus y_image and ag_strength (fp32 [b]) when the case has them."""
    d = _base_inputs(dict(kind="t2v", **{k: case[k] for k in ("seed", "b", "f", "h", "w", "ntok", "t")}))
    if case["yi_frames"]:
        d["y_image"] = synth.tensor("y_image", (case["b"], case["yi_frames"], 1024), 1.0, case["seed"] + 1000)
        d["ag_strength"] = torch.tensor(case["ag"], dtype=torch.float32)
    return d


def call_kwargs(case, inp):
    """Keyword arguments of the model call: ag_strength a float when the batch shares it, the [b] tensor otherwise."""
    kw = {"y": inp["y"]}
    if "y_image" in inp:
        kw["y_image"] = inp["y_image"]
        ag = inp["ag_strength"]
        kw["ag_strength"] = float(ag[0]) if len(set(case["ag"])) == 1 else ag
    return kw


def reference_digest(golden_dir, name):
    return json.load(open(os.path.join(golden_dir, "dreamvideo_specs.json")))[name]


def product_spec(ctor):
    import vgen_b200
    with torch.device("meta"):
        m = vgen_b200.UNetSD_DreamVideo(**ctor)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def load_spec(golden_dir, name, cases=None):
    """The parameter list of a case, checked against the reference's frozen digest before any weights are made from it."""
    case = (cases or DV_CASES)[name]
    spec = product_spec(case["ctor"])
    assert spec_digest(spec) == reference_digest(golden_dir, case.get("spec", name)), f"{name}: parameter list differs"
    return spec


def build_product(case):
    import vgen_b200
    return vgen_b200.UNetSD_DreamVideo(**case["ctor"])


def oracle_call(case, sd, inp):
    return vo.unet_dreamvideo_forward(sd, case["ctor"], inp["x"], inp["t"], inp["y"], inp.get("y_image"),
                                      inp.get("ag_strength"))
