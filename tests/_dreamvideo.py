"""DreamVideo (UNetSD_DreamVideo): parity cases, inputs and a plain-torch oracle of the adapted trunk.

The oracle restates tools/modules/unet/unet_dreamvideo.py:225-290 and the adapters of util.py:499-519,603-672
(BasicTransformerBlockWithAdapter, SpatialTransformerWithAdapter, TemporalTransformerWithAdapter) on top of
oracle/vgen_oracle.py's pieces.  It takes ag_strength per sample, which the reference does not; tools/make_golden_dreamvideo.py
therefore freezes the reference's outputs of a multi-lambda batch by running it one video at a time (videos never interact).
Parameter lists of the reference are frozen as digests in tests/golden/dreamvideo_specs.json.
"""
from __future__ import annotations

import json
import os

import torch
import torch.nn.functional as F

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


# ------------------------------------------------------------------------------------------------ oracle
_SITES = (("attn_adapter", 0), ("cross_attn_adapter", 1), ("ff_adapter", 2))


def _adapter(x, s, cond, lam):
    """Adapter.forward, util.py:510-517 (lam broadcasts over the rows of x)."""
    x_in = x
    if cond is not None and s.has("condition_linear.weight"):
        x = x + lam * vo._lin(cond, s.sub("condition_linear"))
    return vo._lin(F.gelu(vo._lin(x, s.sub("down_linear"))), s.sub("up_linear")) + x_in


def _block(x, ctx, s, heads, positions, cond, lam):
    """BasicTransformerBlockWithAdapter.forward, util.py:649-672."""
    def ff(z):
        val, gate = vo._lin(z, s.sub("ff.net.0.proj")).chunk(2, dim=-1)
        return vo._lin(val * F.gelu(gate), s.sub("ff.net.2"))
    subs = (lambda z: vo._attention(vo._ln(z, s.sub("norm1")), None, s.sub("attn1"), heads),
            lambda z: vo._attention(vo._ln(z, s.sub("norm2")), ctx, s.sub("attn2"), heads),
            lambda z: ff(vo._ln(z, s.sub("norm3"))))
    for (mod, idx), sub in zip(_SITES, subs):
        if not s.has(mod + ".down_linear.weight"):
            x = sub(x) + x
        elif positions[idx] == "parallel":
            x = sub(x) + _adapter(x, s.sub(mod), cond, lam)
        else:
            x = _adapter(sub(x) + x, s.sub(mod), cond, lam)
    return x


def _spatial(x, ctx, s, head_dim, positions):
    bf, c, hh, ww = x.shape
    h = vo._gn(x, s.sub("norm"), 1e-6).permute(0, 2, 3, 1).reshape(bf, hh * ww, c)
    h = vo._lin(h, s.sub("proj_in"))
    h = _block(h, ctx, s.sub("transformer_blocks.0"), h.shape[-1] // head_dim, positions, None, None)
    h = vo._lin(h, s.sub("proj_out"))
    return h.reshape(bf, hh, ww, c).permute(0, 3, 1, 2) + x


def _temporal(x, s, head_dim, batch, positions, cond, lam):
    """TemporalTransformerWithAdapter.forward, util.py:1340-1380: the condition [b, f, C] is broadcast over the pixels."""
    bf, c, hh, ww = x.shape
    f = bf // batch
    x5 = x.reshape(batch, f, c, hh, ww).permute(0, 2, 1, 3, 4)
    h = F.group_norm(x5, 32, s["norm.weight"], s["norm.bias"], 1e-6)
    h = h.permute(0, 3, 4, 2, 1).reshape(batch * hh * ww, f, c)
    h = F.linear(h, s["proj_in.weight"][:, :, 0], s["proj_in.bias"])
    cnd = lr = None
    if cond is not None:
        cnd = cond[:, None, None].expand(batch, hh, ww, f, cond.shape[-1]).reshape(batch * hh * ww, f, cond.shape[-1])
        lr = lam.repeat_interleave(hh * ww).view(-1, 1, 1)
    h = _block(h, None, s.sub("transformer_blocks.0"), h.shape[-1] // head_dim, positions, cnd, lr)
    h = F.linear(h, s["proj_out.weight"][:, :, 0], s["proj_out.bias"])
    return h.reshape(batch, hh, ww, f, c).permute(0, 3, 4, 1, 2).reshape(bf, c, hh, ww) + x


def _run(x, s, emb, ctx, head_dim, batch, ctor, cond, lam):
    if s.has("transformer_blocks.0.norm1.weight"):
        if s["proj_in.weight"].ndim == 2:
            return _spatial(x, ctx, s, head_dim, ctor.get("spatial_adapter_position_list", ["", "parallel", ""]))
        return _temporal(x, s, head_dim, batch, ctor.get("temporal_adapter_position_list", ["parallel"] * 3), cond, lam)
    return vo._run_block(x, s, emb, ctx, head_dim, batch)


def unet_dreamvideo_forward(sd, ctor, x, t, y, y_image=None, ag_strength=None, head_dim=64):
    """UNetSD_DreamVideo.forward in eval() (unet_dreamvideo.py:225-290); ag_strength: fp32 [b] (or None with y_image None)."""
    b, c, f, h, w = x.shape
    dim = sd["time_embed.0.weight"].shape[1]
    root = vo._SD(sd)
    emb = vo._mlp(vo.sinusoidal_embedding(t, dim).to(x.dtype), root.sub("time_embed")).repeat_interleave(f, dim=0)
    ctx = y.repeat_interleave(f, dim=0)
    cond = lam = None
    if y_image is not None and ctor.get("temporal_adapter_condition_dim"):
        cond = y_image.repeat_interleave(f, dim=1) if y_image.shape[1] == 1 else y_image
        cond, lam = cond.to(x.dtype), ag_strength.to(x.device, x.dtype)
    xx = x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    skips = []
    for i in vo._children(sd, "input_blocks."):
        blk = root.sub(f"input_blocks.{i}")
        if blk.has("op.weight"):
            xx = vo._run_block(xx, blk, emb, ctx, head_dim, b)
        else:
            for j in vo._children(sd, blk.p):
                xx = _run(xx, blk.sub(str(j)), emb, ctx, head_dim, b, ctor, cond, lam)
        skips.append(xx)
    for j in vo._children(sd, "middle_block."):
        xx = _run(xx, root.sub(f"middle_block.{j}"), emb, ctx, head_dim, b, ctor, cond, lam)
    for i in vo._children(sd, "output_blocks."):
        xx = torch.cat([xx, skips.pop()], dim=1)
        blk = root.sub(f"output_blocks.{i}")
        for j in vo._children(sd, blk.p):
            xx = _run(xx, blk.sub(str(j)), emb, ctx, head_dim, b, ctor, cond, lam)
    out = F.conv2d(F.silu(vo._gn(xx, root.sub("out.0"), 1e-5)), sd["out.2.weight"], sd["out.2.bias"], padding=1)
    return out.reshape(b, f, -1, h, w).permute(0, 2, 1, 3, 4)


def oracle_call(case, sd, inp):
    return unet_dreamvideo_forward(sd, case["ctor"], inp["x"], inp["t"], inp["y"], inp.get("y_image"), inp.get("ag_strength"))
