"""UNetSD_LoRA's runtime LoRA: extra LoRA sets for the tiny InstructVideo cases and the oracle of several sets at per-sample
strengths.

The oracle restates the reference's _proj with several sets through the single-pair oracle (oracle/vgen_oracle.py's
unet_lora_forward): for one sample, the sets' pairs at strengths s_j and scales c_j act like ONE pair
    D = [s_1 c_1 D_1; s_2 c_2 D_2; ...],  U = [U_1 | U_2 | ...]   at scale 1,
since U D x = sum_j s_j c_j U_j D_j x exactly (a concatenation, no approximation).  Batch entries never interact in the
UNet, so a batch with per-sample strengths is the concatenation of one such forward per sample.
"""
from __future__ import annotations

import torch

from oracle.vgen_oracle import unet_lora_forward
from _instructvideo import product_spec, weights

MODS = ("to_q_lora", "to_k_lora", "to_v_lora", "to_out_lora")


def lora_pairs(ctor, seed, rank=4):
    """A LoRA-only state dict for the model built from ctor (any use_lora), rank `rank`, made like the cases' own pairs
    (synth weights with the up weights scaled by LORA_UP_GAIN)."""
    spec = product_spec(dict(ctor, use_lora=True, lora_rank=rank))
    sd = weights(spec, seed)
    return {k: v for k, v in sd.items() if "_lora." in k}


def sites(sd):
    return sorted({k[:-len(".down_linear.weight")] for k in sd if k.endswith("_lora.down_linear.weight")})


def combined_pairs(sets, strengths):
    """sets: [(LoRA dict, scale)], strengths: one float per set -> one LoRA dict of the concatenated pairs (see above)."""
    out = {}
    for site in sites(sets[0][0]):
        d = torch.cat([float(s) * c * p[site + ".down_linear.weight"].double() for (p, c), s in zip(sets, strengths)])
        u = torch.cat([p[site + ".up_linear.weight"].double() for p, _ in sets], dim=1)
        out[site + ".down_linear.weight"], out[site + ".up_linear.weight"] = d, u
    return out


def oracle_multi(base, sets, x, t, y, strength):
    """unet_lora_forward with several LoRA sets: base = the state dict without LoRA keys, sets = [(LoRA dict, scale)],
    strength [b, len(sets)] (host values).  fp32 (or autocast) like the single-set oracle."""
    outs = []
    for i in range(x.shape[0]):
        comb = combined_pairs(sets, [float(v) for v in strength[i]])
        sd = dict(base)
        sd.update({k: v.to(device=x.device, dtype=torch.float32) for k, v in comb.items()})
        outs.append(unet_lora_forward(sd, x[i:i + 1], t[i:i + 1], y[i:i + 1], 1.0))
    return torch.cat(outs)
