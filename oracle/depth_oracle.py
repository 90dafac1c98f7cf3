"""Plain-PyTorch restatement of the MiDaS v3.0 DPT-Large depth annotator (tools/annotator/depth/__init__.py:162-293),
driven by a reference-format state dict (names as in MiDaS.state_dict()).

Two arithmetics:
  * half=False: fp32 throughout (the truth the parity tests compare against, with TF32 off);
  * half=True:  what the VideoComposer engines run -- the model `.to(memory_format=torch.channels_last).half()`, the input
    fp16 channels_last, so every op computes in fp16 with PyTorch's own accumulation; the attention softmax is fp32 as the
    reference's SelfAttention does it.
Every op is a torch.nn.functional call in the reference's order (the fusion blocks interpolate BEFORE conv_out, as the
reference does).  Runs on CPU or GPU.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _params(sd, half, device):
    out = {}
    for k, v in sd.items():
        t = v.detach().to(device=device, dtype=torch.float16 if half else torch.float32)
        out[k] = t.contiguous(memory_format=torch.channels_last) if (half and t.dim() == 4) else t
    return out


def _block(P, b, x, heads):
    n, L, d = x.shape
    hd = d // heads
    h = F.layer_norm(x, (d,), P[b + "norm1.weight"], P[b + "norm1.bias"])
    qkv = F.linear(h, P[b + "attn.to_qkv.weight"], P[b + "attn.to_qkv.bias"]).view(n, L, 3, heads, hd)
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))       # [n, heads, L, hd]
    s = (hd ** -0.5) * torch.matmul(q, k.transpose(-1, -2))
    a = torch.softmax(s.float(), dim=-1).to(s.dtype)
    o = torch.matmul(a, v).permute(0, 2, 1, 3).reshape(n, L, d)
    x = x + F.linear(o, P[b + "attn.proj.weight"], P[b + "attn.proj.bias"])
    h = F.layer_norm(x, (d,), P[b + "norm2.weight"], P[b + "norm2.bias"])
    h = F.gelu(F.linear(h, P[b + "mlp.0.weight"], P[b + "mlp.0.bias"]))
    return x + F.linear(h, P[b + "mlp.2.weight"], P[b + "mlp.2.bias"])


def _conv(P, nm, x, stride=1, padding=0, bias=True):
    return F.conv2d(x, P[nm + ".weight"], P[nm + ".bias"] if bias else None, stride=stride, padding=padding)


def _residual(P, q, x):
    t = F.conv2d(F.relu(x), P[q + ".residual.1.weight"], P[q + ".residual.1.bias"], padding=1)
    return x + F.conv2d(F.relu(t), P[q + ".residual.3.weight"], P[q + ".residual.3.bias"], padding=1)


def _fusion(P, s, x0, x1=None):
    q = f"fusion{s}."
    x = _residual(P, q + "layer2", x0 if x1 is None else x0 + _residual(P, q + "layer1", x1))
    x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
    return _conv(P, q + "conv_out", x)


def midas_forward(sd, x, image_size=384, patch_size=16, num_heads=16, num_layers=24, half=False):
    """depth [n, 1, H, W] of images x [n, 3, H, W] (fp32 for half=False, fp16 channels_last for half=True)."""
    P = _params(sd, half, x.device)
    x = x.to(torch.float16).contiguous(memory_format=torch.channels_last) if half else x.float()
    n, _, H, W = x.shape
    p, grid = patch_size, image_size // patch_size
    hp, wp = H // p, W // p
    pos = P["pos_embedding"]
    d = pos.shape[-1]
    grid_pos = F.interpolate(pos[:, 1:].reshape(1, grid, grid, d).permute(0, 3, 1, 2), size=(hp, wp), mode="bilinear",
                             align_corners=False).permute(0, 2, 3, 1).reshape(1, hp * wp, d)
    t = F.conv2d(x, P["patch_embedding.weight"], P["patch_embedding.bias"], stride=p).flatten(2).permute(0, 2, 1)
    t = torch.cat([P["cls_embedding"].expand(n, 1, d), t], dim=1) + torch.cat([pos[:, :1], grid_pos], dim=1)

    per = num_layers // 4
    stages = []
    for s in range(1, 5):
        for i in range((s - 1) * per, s * per):
            t = _block(P, f"blocks.{i}.", t, num_heads)
        r = torch.cat([t[:, 1:], t[:, :1].expand(n, hp * wp, d)], dim=-1)
        r = F.gelu(F.linear(r, P[f"fc{s}.0.weight"], P[f"fc{s}.0.bias"])).permute(0, 2, 1).reshape(n, d, hp, wp)
        y = _conv(P, f"conv{s}.0", r)
        if s in (1, 2):
            k = 4 if s == 1 else 2
            y = F.conv_transpose2d(y, P[f"conv{s}.1.weight"], P[f"conv{s}.1.bias"], stride=k)
            y = _conv(P, f"conv{s}.2", y, padding=1, bias=False)
        elif s == 3:
            y = _conv(P, "conv3.1", y, padding=1, bias=False)
        else:
            y = _conv(P, "conv4.1", y, stride=2, padding=1)
            y = _conv(P, "conv4.2", y, padding=1, bias=False)
        stages.append(y)

    y = _fusion(P, 4, stages[3])
    for s in (3, 2, 1):
        y = _fusion(P, s, y, stages[s - 1])
    y = _conv(P, "head.0", y, padding=1)
    y = F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=True)
    y = F.relu(_conv(P, "head.2", y, padding=1))
    return F.relu(F.conv_transpose2d(y, P["head.4.weight"], P["head.4.bias"]))
