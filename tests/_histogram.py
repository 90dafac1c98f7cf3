"""The 'histogram' composition of UNetSD_VideoLCM / UNetSD_TFT2V and the colour-palette annotator: parity cases, inputs,
the UNet oracle and the frozen fixtures.

The UNet oracle is oracle/vgen_oracle.py's trunk with a per-frame context, as the reference builds it
(tools/modules/unet/unet_videolcm.py:713-759): [y tokens | image tokens] repeated over the frames, then each frame's
hist_context_embedding(histogram) token appended.  The palette oracle is oracle/palette_oracle.py.
tools/make_golden_histogram.py freezes the reference's own outputs (its UNet classes and its palette.py) into
tests/golden/histogram_*.npz and the parameter-list digests into tests/golden/histogram_specs.json.
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from oracle import synth, vgen_oracle as vo
from oracle.cases import FULL_CTORS
from _vcomp import EVERY, RELEASED, VCOMP_CASES, FULL_VCOMP_CASES, spec_digest
from _vcomp import call_kwargs as _vcomp_kwargs, make_inputs as _vcomp_inputs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_TINY = VCOMP_CASES["vcomp_lcm_tiny"]["ctor"]

HIST_CASES = {
    # every composition plus 'histogram', with the image tokens: the context is [y | image | histogram token]
    "histogram_lcm_tiny": dict(cls="UNetSD_VideoLCM", ctor=_TINY, comps=EVERY + ["histogram"], resolution=[96, 64],
                               seed=41, b=1, f=4, h=8, w=12, H=70, W=100, ntok=5, t=[377],
                               conds=list(vo.SUM_ORDER), image=True),
    # two videos, 'histogram' alone: the context is [y | histogram token]
    "histogram_tft2v_tiny_b2": dict(cls="UNetSD_TFT2V", ctor=_TINY, comps=["text", "histogram"], resolution=[96, 64],
                                    seed=42, b=2, f=3, h=8, w=12, H=64, W=96, ntok=5, t=[811, 95], conds=[],
                                    image=False),
}
FULL_HIST = dict(FULL_VCOMP_CASES["full_vcomposer"], comps=RELEASED + ["histogram"])
# spec name -> (class, video_compositions, constructor kwargs), digests in histogram_specs.json
HIST_SPECS = {"full_vcomposer_histogram": ("UNetSD_TFT2V", RELEASED + ["histogram"], FULL_CTORS["full_videolcm"][1]),
              "full_videolcm_histogram": ("UNetSD_VideoLCM", ["text", "histogram"], FULL_CTORS["full_videolcm"][1])}

# palette fixtures: name -> (height, width, uint8?)
FRAMES = {"u8_61x97": (61, 97, True), "f32_64x96": (64, 96, False), "u8_32x48_flat": (32, 48, True)}
SIGMAS = (20, 0, 5)
NEAREST_BOUND = 1e-9   # see tests/test_gpu_histogram.py::test_nearest_index_every_uint8_colour


def make_inputs(case):
    d = _vcomp_inputs(case)
    d["histogram"] = synth.tensor("histogram", (case["b"], case["f"], 156), 1.0, case["seed"] + 1000).abs()
    return d


def call_kwargs(case, inp):
    kw = _vcomp_kwargs(case, inp)
    kw["histogram"] = inp["histogram"]
    return kw


def config_of(case):
    return dict(video_compositions=list(case["comps"]), resolution=list(case["resolution"]))


def unet_forward(sd, x, t, y, histogram, image=None, resolution=None, **conds):
    """UNetSD_VideoLCM / UNetSD_TFT2V.forward in eval() with a histogram [b, f, hist_dim]
    (unet_videolcm.py:541-784): the shared context repeated per frame, then each frame's histogram token."""
    b, c, f, h, w = x.shape
    root = vo._SD(sd)
    concat = x.new_zeros(b, sd["input_blocks.0.0.weight"].shape[1] - c, f, h, w)
    for kw in vo.SUM_ORDER:
        if conds.get(kw) is not None:
            concat = concat + vo._encode_condition(conds[kw].to(x.dtype), sd, kw, b, resolution[1] // 2, resolution[0] // 2)
    ctx = y
    if image is not None:
        ctx = torch.cat([ctx, vo._mlp(image, root.sub("pre_image_condition")).view(b, -1, y.shape[-1])], dim=1)
    dim = sd["time_embed.0.weight"].shape[1]
    emb = vo._mlp(vo.sinusoidal_embedding(t, dim).to(x.dtype), root.sub("time_embed")).repeat_interleave(f, dim=0)
    hist = vo._mlp(histogram.to(x.dtype), root.sub("hist_context_embedding")).reshape(b * f, 1, -1)
    ctx = torch.cat([ctx.repeat_interleave(f, dim=0), hist], dim=1)
    xx = torch.cat([x, concat], dim=1).permute(0, 2, 1, 3, 4).reshape(b * f, -1, h, w)
    out = vo._unet_trunk(sd, xx, emb, ctx, 64, b)
    return out.reshape(b, f, -1, h, w).permute(0, 2, 1, 3, 4)


def oracle_call(case, sd, inp):
    kw = call_kwargs(case, inp)
    return unet_forward(sd, inp["x"], inp["t"], kw.pop("y"), kw.pop("histogram"), resolution=case["resolution"], **kw)


def product_spec(cls, comps, resolution, ctor):
    import vgen_b200
    with torch.device("meta"):
        m = getattr(vgen_b200, cls)(config=dict(video_compositions=list(comps), resolution=list(resolution)), **ctor,
                                    enable_histogram="histogram" in comps)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def reference_digest(name):
    return json.load(open(os.path.join(GOLD, "histogram_specs.json")))[name]


def load_spec(name):
    """The case's parameter list, checked against the reference's frozen digest."""
    case = HIST_CASES[name]
    spec = product_spec(case["cls"], case["comps"], case["resolution"], case["ctor"])
    assert spec_digest(spec) == reference_digest(name), f"{name}: parameter list differs from the reference's"
    return spec


def build_product(case, **kw):
    import vgen_b200
    return getattr(vgen_b200, case["cls"])(config=config_of(case), **case["ctor"],
                                           enable_histogram="histogram" in case["comps"], **kw)


def make_frame(name):
    """The fixture frame `name` (h, w, 3): uint8, or float32 in [0, 1]; the flat one has a few large single-colour areas."""
    h, w, u8 = FRAMES[name]
    g = np.random.Generator(np.random.PCG64(sum(map(ord, name))))
    if name.endswith("_flat"):
        img = np.zeros((h, w, 3), np.uint8)
        img[: h // 2, : w // 3] = (255, 255, 255)
        img[: h // 2, w // 3:] = (12, 200, 37)
        img[h // 2:] = g.integers(0, 256, size=(h - h // 2, w, 3), dtype=np.uint8)
        return img
    if u8:
        return g.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    return g.random(size=(h, w, 3), dtype=np.float32)


def load_palette_golden():
    return np.load(os.path.join(GOLD, "histogram_palette.npz"))
