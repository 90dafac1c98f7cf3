"""The pre-LN ViT trunk shared by the CLIP towers (clip.py), DINO (dino.py) and MiDaS's ViT-L/16 (depth.py): plain
functions over a model's packed-weight dict.

  pack_block / pack_patch   state-dict tensors -> packed keys (fp16 GEMM weights, fp32 biases and LayerNorm affines)
  embed                     im2col + patch linear -> [CLS] row, patch rows -> + fp32 position rows
  block                     x + proj(attn(LN1(x))), then x + fc2(act(fc1(LN2(x)))), residuals in the GEMM epilogues

Each model keeps its own state-dict names (given to pack_block as the six sublayer prefixes), its input checks and
layout conversion, and whatever runs before and after the blocks.  Packed keys stay flat in the model's dict, so
packed_tensors(), offload_masters() and parallel.broadcast_packed see them like any other.
"""
from __future__ import annotations

import torch

from . import ops


def f16(t, dev):
    """A GEMM weight as the tap-GEMM reads it: contiguous fp16 on dev."""
    return t.detach().to(device=dev, dtype=torch.float16).contiguous()


def f32(t, dev):
    """A bias, LayerNorm affine or embedding table: contiguous fp32 on dev."""
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def pack_block(W, sd, p, names, dev):
    """Pack block `p` of state dict `sd` into W under p + ln1.g / ln1.b / qkv.w / qkv.b / proj.* / ln2.* / fc1.* / fc2.*.
    names: the state-dict prefixes of LN1, qkv, proj, LN2, fc1 and fc2 within the block, to which "weight" / "bias" are
    appended (open_clip's qkv is "attn.in_proj_").  A missing bias (DINO's qkv_bias=False) packs as None."""
    ln1, qkv, proj, ln2, fc1, fc2 = (p + n for n in names)
    for key, src in (("ln1", ln1), ("ln2", ln2)):
        W[p + key + ".g"], W[p + key + ".b"] = f32(sd[src + "weight"], dev), f32(sd[src + "bias"], dev)
    for key, src in (("qkv", qkv), ("proj", proj), ("fc1", fc1), ("fc2", fc2)):
        b = sd.get(src + "bias")
        W[p + key + ".w"], W[p + key + ".b"] = f16(sd[src + "weight"], dev), None if b is None else f32(b, dev)


def pack_patch(w, dev):
    """Patch-embedding conv weight [D, c, p, p] -> fp16 [D, (ky, kx, c)] (im2col's column order), K zero-padded to a
    multiple of 64."""
    d, k = w.shape[0], w[0].numel()
    wp = torch.zeros(d, (k + 63) // 64 * 64)
    wp[:, :k] = w.detach().float().cpu().permute(0, 2, 3, 1).reshape(d, k)
    return f16(wp, dev)


def embed(img, patch, w, b, cls, pos):
    """img fp16 channels-last [n, H, W, c] -> tokens fp16 [n, 1 + (H/patch)(W/patch), D]: the [CLS] row cls (fp16 [1, D])
    then the patch rows (linear of the im2col columns with w from pack_patch and bias b, or None), plus the fp32
    position rows pos (one per token, any shape of that size)."""
    n, H, Wd, _ = img.shape
    gh, gw = H // patch, Wd // patch
    D, L = w.shape[0], gh * gw + 1
    col = ops.im2col(img, patch, patch, patch, 0, 0, gh, gw, w.shape[1])
    patches = ops.linear(col, w, bias=b)
    x = torch.empty(n, L, D, device=img.device, dtype=torch.float16)
    xr = x.view(n, L * D)
    ops.copy2d(cls.expand(n, D), xr[:, :D])
    ops.copy2d(patches.view(n, gh * gw * D), xr[:, D:])
    return ops.add_rows_f32_(x, pos)


def block(x, W, p, heads, eps=1e-5, act="gelu", attention="cross_small", scale=None, causal=False):
    """One pre-LN block on x fp16 [b, L, D] -> [b, L, D].
    act: "gelu" (erf) runs in fc1's GEMM epilogue (fp32, one rounding); "quick_gelu" (OpenAI CLIP) is a separate
    elementwise kernel, as the tap-GEMM has no QuickGELU epilogue.
    attention: "cross_small" (the small-problem kernel: any head_dim, optionally causal) or "d64" (the head_dim-64 flash
    kernel with softmax scale `scale`, None for 64 ** -0.5)."""
    b, L, D = x.shape
    x2 = x.view(b * L, D)
    h = ops.layer_norm(x2, W[p + "ln1.g"], W[p + "ln1.b"], eps)
    qkv = ops.linear(h, W[p + "qkv.w"], bias=W[p + "qkv.b"]).view(b, L, 3 * D)
    q, k, v = qkv[:, :, :D], qkv[:, :, D:2 * D], qkv[:, :, 2 * D:]
    if attention == "d64":
        a = ops.attention_d64(q, k, v, heads, scale=scale)
    else:
        a = ops.attention_cross_small(q, k, v, heads, causal=causal)
    x2 = ops.linear(a.view(b * L, D), W[p + "proj.w"], bias=W[p + "proj.b"], residual=x2)
    h = ops.layer_norm(x2, W[p + "ln2.g"], W[p + "ln2.b"], eps)
    if act == "gelu":
        h = ops.linear_gelu_rowbias(h, W[p + "fc1.w"], bias=W[p + "fc1.b"])
    else:
        h = ops.eltwise(act, ops.linear(h, W[p + "fc1.w"], bias=W[p + "fc1.b"]))
    return ops.linear(h, W[p + "fc2.w"], bias=W[p + "fc2.b"], residual=x2).view(b, L, D)
