"""InstructVideo (UNetSD_LoRA): parity cases, inputs and the oracle call.

The oracle of these cases is oracle/vgen_oracle.py's unet_lora_forward, which restates tools/modules/unet/unet_lora.py:134-195
(MemoryEfficientCrossAttention with its LoRA pairs) in the shared T2V trunk.  It never merges: every adapted projection is
x W^T + s (x D^T) U^T, computed as two thin GEMMs next to the base one, so it cannot share the product's shortcut (the merge
in the pack).
tools/make_golden_instructvideo.py freezes the reference's outputs for the cases and digests of its parameter lists
(tests/golden/instructvideo_specs.json).
"""
from __future__ import annotations

import json
import os

import torch

from oracle import synth
from oracle.vgen_oracle import unet_lora_forward
from oracle.cases import _FULL_UNET, _T2V_TINY, make_inputs as _base_inputs
from _vcomp import spec_digest  # noqa: F401  (same digest format as vcomp_specs.json)

# (a) the reference's unmerged forward; (b) the model get_lora_merged_model returns for lora_alpha 8 (s = 2);
# (c) use_lora=False (lora_rank is set, as in the released ModelScope-base configs, and ignored)
IV_CASES = {
    "iv_lora_tiny": dict(ctor=dict(_T2V_TINY, use_lora=True, lora_rank=4), seed=51, b=1, f=4, h=8, w=12, ntok=5, t=[613]),
    "iv_lora_alpha_tiny_b2": dict(ctor=dict(_T2V_TINY, use_lora=True, lora_rank=4, lora_alpha=8), seed=52, b=2, f=3, h=8,
                                  w=6, ntok=7, t=[811, 95], merged=True),
    "iv_nolora_tiny": dict(ctor=dict(_T2V_TINY, use_lora=False, lora_rank=4), seed=53, b=1, f=4, h=8, w=12, ntok=5, t=[377]),
}
# the released eval UNet dicts (configs/instructvideo/eval/*.yaml; lora_alpha is empty there, i.e. None)
RELEASED_UNET = dict(_FULL_UNET, lora_rank=4, lora_alpha=None)
RELEASED = {"released_lora": dict(RELEASED_UNET, use_lora=True), "released_base": dict(RELEASED_UNET, use_lora=False)}
RELEASED_COUNTS = {"released_lora": (2008, 1412895300), "released_base": (1480, 1411233860)}   # LoRA: 1 661 440 parameters
# their Diffusion dict and the ddim_steps list of the 20-step configs
RELEASED_DIFFUSION = {"type": "DiffusionDDIMReward", "schedule": "linear_sd",
                      "schedule_param": {"num_timesteps": 1000, "init_beta": 0.00085, "last_beta": 0.0120,
                                         "zero_terminal_snr": False},
                      "mean_type": "eps", "loss_type": "mse", "var_type": "fixed_small", "rescale_timesteps": False,
                      "noise_strength": 0}
DDIM20_STEPS = [951, 901, 851, 801, 751, 701, 651, 601, 551, 501, 451, 401, 351, 301, 251, 201, 151, 101, 51, 1]

# the eval shape: CFG pair as one batch of 2, 16 frames, 256 x 256 pixels (32 x 32 latent), 77 tokens
FULL_IV_CASES = {
    "full_iv_lora": dict(ctor=RELEASED["released_lora"], seed=54, b=1, f=16, h=32, w=32, ntok=77, t=[751], spec="released_lora"),
}


# save_video_local write-out: name -> (shape [b, 3, f, h, w], scale, mean, std); the first ends with a grey frame, which
# save_video_local keeps (save_i2vgen_video_safe would drop it)
VIDEOS = {
    "iv_video": ((2, 3, 5, 6, 10), 1.5, [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]),
    "iv_video_single": ((1, 3, 1, 4, 4), 1.0, [0.5, 0.5, 0.5], [0.5, 0.5, 0.5]),
}


def make_video(name):
    shape, scale, mean, std = VIDEOS[name]
    v = synth.tensor("iv_" + name, shape, scale, 9)
    if shape[2] > 1:
        v[:, :, -1] = 0.01 * v[:, :, -1]
    return v, mean, std


def make_inputs(case):
    """x / t / y / y_neg as oracle.cases.make_inputs."""
    return _base_inputs(dict(kind="t2v", **{k: case[k] for k in ("seed", "b", "f", "h", "w", "ntok", "t")}))


# The reference initialises the LoRA up weights to zero (unet_lora.py:122), which would make every LoRA test vacuous.
# Here they are synth's N(0, 1/sqrt(rank)) times this gain: the LoRA then moves the tiny cases' output by ~90 % of its
# maximum, while the network stays well conditioned (at gain 1 with s = 2 an fp32 and an fp64 forward differ by 5e-4).
LORA_UP_GAIN = 0.5


def weights(spec, seed):
    """Synthetic weights (oracle/synth.py) with the LoRA up weights scaled by LORA_UP_GAIN."""
    sd = synth.state_dict(spec, seed=seed)
    for k in sd:
        if k.endswith("_lora.up_linear.weight"):
            sd[k] = sd[k] * LORA_UP_GAIN
    return sd


def lora_scale(ctor):
    """get_lora_merged_model's alpha (inference_instructvideo_entrance.py:315)."""
    return 1.0 if ctor.get("lora_alpha") is None else ctor["lora_alpha"] / ctor["lora_rank"]


def reference_digest(golden_dir, name):
    return json.load(open(os.path.join(golden_dir, "instructvideo_specs.json")))[name]


def product_spec(ctor):
    import vgen_b200
    with torch.device("meta"):
        m = vgen_b200.UNetSD_LoRA(**ctor)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def load_spec(golden_dir, name, cases=None):
    """The parameter list of a case, checked against the reference's frozen digest before any weights are made from it."""
    case = (cases or IV_CASES)[name]
    spec = product_spec(case["ctor"])
    assert spec_digest(spec) == reference_digest(golden_dir, case.get("spec", name)), f"{name}: parameter list differs"
    return spec


def build_product(case):
    import vgen_b200
    return vgen_b200.UNetSD_LoRA(**case["ctor"])


def oracle_call(case, sd, inp, y_key="y"):
    return unet_lora_forward(sd, inp["x"], inp["t"], inp[y_key], lora_scale(case["ctor"]))
