"""VideoComposer compositions of UNetSD_VideoLCM / UNetSD_TFT2V: parity cases, inputs and a plain-torch oracle.

The oracle restates the reference's condition encoders and image tokens (tools/modules/unet/unet_videolcm.py:283-372,
:598-745; unet_tf2tv.py is the same forward) on top of oracle/vgen_oracle.py's trunk.  tools/make_golden_vcomp.py
freezes the reference's own outputs for these cases into tests/golden/ (vcomp_*.npz, tft2v_tiny.npz, vcomp_pin.npz) and
the reference's parameter lists as digests (vcomp_specs.json: tensor count, parameter count, sha256 of the list).
"""
from __future__ import annotations

import hashlib
import json
import os

import torch
import torch.nn.functional as F

from oracle import synth, vgen_oracle as vo
from oracle.cases import CASES, FULL_CTORS, make_inputs as _base_inputs

RELEASED = ["text", "mask", "depthmap", "sketch", "motion", "image", "local_image", "single_sketch"]
EVERY = RELEASED + ["canny"]

# forward keyword -> (encoder prefix, frame-transformer prefix, input channels), unet_videolcm.py:295-372
ENCODERS = {
    "depth": ("depth_embedding", "depth_embedding_after", 1),
    "motion": ("motion_embedding", "motion_embedding_after", 2),
    "canny": ("canny_embedding", "canny_embedding_after", 1),
    "masked": ("masked_embedding", "mask_embedding_after", 4),
    "sketch": ("sketch_embedding", "sketch_embedding_after", 1),
    "single_sketch": ("single_sketch_embedding", "single_sketch_embedding_after", 1),
    "local_image": ("local_image_embedding", "local_image_embedding_after", 3),
}
SUM_ORDER = ("depth", "local_image", "motion", "canny", "sketch", "single_sketch", "masked")   # :599-699

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


def _encode(v, sd, kw, b, oh, ow):
    """<kw>_embedding -> <kw>_embedding_after, unet_videolcm.py:599-607 -> [b, cd, f, h, w]."""
    enc, after, _ = ENCODERS[kw]
    s = vo._SD(sd).sub(enc)
    f = v.shape[2]
    z = v.permute(0, 2, 1, 3, 4).reshape(b * f, v.shape[1], v.shape[3], v.shape[4])
    z = F.silu(F.conv2d(z, s["0.weight"], s["0.bias"], padding=1))
    z = F.adaptive_avg_pool2d(z, (oh, ow))
    z = F.silu(F.conv2d(z, s["3.weight"], s["3.bias"], stride=2, padding=1))
    z = F.conv2d(z, s["5.weight"], s["5.bias"], stride=2, padding=1)
    cd, h, w = z.shape[1:]
    tok = z.reshape(b, f, cd, h, w).permute(0, 3, 4, 1, 2).reshape(b * h * w, f, cd)
    tok = vo._local_temporal_encoder(tok, vo._SD(sd).sub(after))
    return tok.reshape(b, h, w, f, cd).permute(0, 4, 3, 1, 2)


def unet_vcomp_forward(sd, x, t, y, resolution, image=None, fps=None, head_dim=64, use_fps_condition=False, **conds):
    """UNetSD_VideoLCM / UNetSD_TFT2V.forward in eval() (unet_videolcm.py:541-784): conditions summed into `concat`
    in the forward's order, image tokens appended after the text tokens."""
    b, c, f, h, w = x.shape
    dim = sd["time_embed.0.weight"].shape[1]
    root = vo._SD(sd)
    concat_dim = sd["input_blocks.0.0.weight"].shape[1] - c
    concat = x.new_zeros(b, concat_dim, f, h, w)
    for kw in SUM_ORDER:
        if conds.get(kw) is not None:
            concat = concat + _encode(conds[kw].to(x.dtype), sd, kw, b, resolution[1] // 2, resolution[0] // 2)
    xx = torch.cat([x, concat], dim=1)
    emb = vo._mlp(vo.sinusoidal_embedding(t, dim).to(x.dtype), root.sub("time_embed"))
    if use_fps_condition and fps is not None:
        emb = emb + vo._mlp(vo.sinusoidal_embedding(fps, dim).to(x.dtype), root.sub("fps_embedding"))
    emb = emb.repeat_interleave(f, dim=0)
    ctx = y
    if image is not None:
        ctx = torch.cat([ctx, vo._mlp(image, root.sub("pre_image_condition")).view(b, -1, y.shape[-1])], dim=1)
    ctx = ctx.repeat_interleave(f, dim=0)
    xx = xx.permute(0, 2, 1, 3, 4).reshape(b * f, c + concat_dim, h, w)
    out = vo._unet_trunk(sd, xx, emb, ctx, head_dim, b)
    return out.reshape(b, f, -1, h, w).permute(0, 2, 1, 3, 4)


def oracle_call(case, sd, inp):
    kw = call_kwargs(case, inp)
    return unet_vcomp_forward(sd, inp["x"], inp["t"], kw.pop("y"), case["resolution"], **kw)


def build_product(case):
    import vgen_b200
    return getattr(vgen_b200, case["cls"])(config=config_of(case), **case["ctor"])
