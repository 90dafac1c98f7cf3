"""H100-native DINO ViT: a drop-in for DreamVideo's metric/dino/vision_transformer.py (`VisionTransformer`, `vit_tiny`,
`vit_small`, `vit_base`), the DINO-I feature extractor of metric/cal_metric_DreamVideo.py.

Same constructor arguments and state-dict names, so `dino_deitsmall16_pretrain.pth` loads into `vit_small()` with
`strict=True`.  The forward is the reference's at its trained grid:

  patch embedding (conv p x p, stride p, with bias) -> [CLS] + pos_embed -> depth x pre-LN blocks (LayerNorm eps of the
  norm_layer, qkv with bias, softmax attention, proj; fc1 -> GELU(erf) -> fc2) -> norm -> class token

and returns fp32 [n, embed_dim].  The patch embedding and the blocks are the shared ViT trunk (vgen_b200.vit): every op is
a kernel of libvgen_b200.so, im2col + the wgmma tap-GEMM for the patch embedding and the linears (bias, GELU and residual
in the epilogue), LayerNorm, the head_dim-64 flash attention.  Activations are fp16 with fp32 accumulation and
statistics; the forward is CUDA-graphed per input signature (n, H, W).

Not provided: inputs whose patch grid differs from the trained one (interpolate_pos_encoding), get_last_selfattention,
get_intermediate_layers and DINOHead raise NotImplementedError.  There is no CPU path: a CPU tensor or a CPU-resident
model raises VgenError.
"""
from __future__ import annotations

import functools

import torch
import torch.nn as nn

from . import ops, vit
from .graph import graphed
from .params import SpecModule
from .vit import f16, f32

# the reference's Block: the state-dict prefixes of LN1, qkv, proj, LN2, fc1, fc2 (vit.pack_block)
_BLOCK = ("norm1.", "attn.qkv.", "attn.proj.", "norm2.", "mlp.fc1.", "mlp.fc2.")


def _ln_eps(norm_layer):
    if norm_layer is nn.LayerNorm:
        return 1e-5
    if isinstance(norm_layer, functools.partial) and norm_layer.func is nn.LayerNorm and not norm_layer.args:
        return float(norm_layer.keywords.get("eps", 1e-5))
    raise NotImplementedError(f"vgen_b200 DINO: norm_layer must be nn.LayerNorm or a partial of it, got {norm_layer!r}")


def dino_spec(img_size, patch_size, in_chans, num_classes, embed_dim, depth, mlp_ratio, qkv_bias):
    """(name, shape) in the order of the reference VisionTransformer's state_dict()."""
    D, hid = embed_dim, int(embed_dim * mlp_ratio)
    n = (img_size // patch_size) ** 2
    spec = [("cls_token", (1, 1, D)), ("pos_embed", (1, n + 1, D)),
            ("patch_embed.proj.weight", (D, in_chans, patch_size, patch_size)), ("patch_embed.proj.bias", (D,))]
    for i in range(depth):
        p = f"blocks.{i}."
        spec += [(p + "norm1.weight", (D,)), (p + "norm1.bias", (D,)), (p + "attn.qkv.weight", (3 * D, D))]
        if qkv_bias:
            spec += [(p + "attn.qkv.bias", (3 * D,))]
        spec += [(p + "attn.proj.weight", (D, D)), (p + "attn.proj.bias", (D,)), (p + "norm2.weight", (D,)),
                 (p + "norm2.bias", (D,)), (p + "mlp.fc1.weight", (hid, D)), (p + "mlp.fc1.bias", (hid,)),
                 (p + "mlp.fc2.weight", (D, hid)), (p + "mlp.fc2.bias", (D,))]
    spec += [("norm.weight", (D,)), ("norm.bias", (D,))]
    if num_classes > 0:
        spec += [("head.weight", (num_classes, D)), ("head.bias", (num_classes,))]
    return spec


class VisionTransformer(SpecModule):
    """metric/dino/vision_transformer.py VisionTransformer (inference forward only)."""

    def __init__(self, img_size=(224,), patch_size=16, in_chans=3, num_classes=0, embed_dim=768, depth=12, num_heads=12,
                 mlp_ratio=4., qkv_bias=False, qk_scale=None, drop_rate=0., attn_drop_rate=0., drop_path_rate=0.,
                 norm_layer=nn.LayerNorm, **kwargs):
        super().__init__()
        if embed_dim % num_heads or embed_dim // num_heads != 64:
            raise NotImplementedError(f"vgen_b200 DINO: head_dim {embed_dim / num_heads:g} (the attention kernel serves "
                                      "head_dim 64, as in vit_tiny / vit_small / vit_base)")
        self.num_features = self.embed_dim = embed_dim
        self.img_size, self.patch_size, self.in_chans = int(img_size[0]), int(patch_size), int(in_chans)
        self.depth, self.num_heads, self.mlp_ratio, self.qkv_bias = depth, num_heads, mlp_ratio, qkv_bias
        self.scale = qk_scale or (embed_dim // num_heads) ** -0.5
        self.eps = _ln_eps(norm_layer)
        self.num_patches = (self.img_size // self.patch_size) ** 2
        self._build_params(dino_spec(self.img_size, self.patch_size, in_chans, num_classes, embed_dim, depth, mlp_ratio,
                                     qkv_bias))
        with torch.no_grad():
            self.cls_token.normal_(std=0.02, generator=torch.Generator().manual_seed(1))
            self.pos_embed.normal_(std=0.02, generator=torch.Generator().manual_seed(2))

    # ---- packing -------------------------------------------------------------------------------
    def _pack(self):
        dev = self.device
        if dev.type != "cuda":
            raise ops._l.VgenError("vgen_b200 DINO forward needs the model on a CUDA device (no CPU path exists)")
        sd = self.state_dict()
        W = {"patch.w": vit.pack_patch(sd["patch_embed.proj.weight"], dev), "patch.b": f32(sd["patch_embed.proj.bias"], dev),
             "cls": f16(sd["cls_token"].reshape(1, -1), dev), "pos": f32(sd["pos_embed"].reshape(-1), dev)}
        for i in range(self.depth):
            vit.pack_block(W, sd, f"blocks.{i}.", _BLOCK, dev)
        W["norm.g"], W["norm.b"] = f32(sd["norm.weight"], dev), f32(sd["norm.bias"], dev)
        self._packed = W
        return W

    # ---- forward -------------------------------------------------------------------------------
    def _check_grid(self, H, Wd):
        p = self.patch_size
        if H != Wd or (H // p) * (Wd // p) != self.num_patches:
            raise NotImplementedError(f"vgen_b200 DINO: a {H}x{Wd} input has a different patch grid from the trained "
                                      f"{self.img_size}x{self.img_size} one (interpolate_pos_encoding is not provided)")

    def forward(self, x):
        """x [n, in_chans, H, W] (CUDA; H = W at the trained grid) -> fp32 [n, embed_dim]."""
        if not torch.is_tensor(x) or x.dim() != 4 or x.shape[1] != self.in_chans:
            raise ValueError(f"vgen_b200 DINO: expected a tensor [n, {self.in_chans}, H, W], got {getattr(x, 'shape', x)}")
        self._check_grid(x.shape[2], x.shape[3])
        if not x.is_cuda:
            raise ops._l.VgenError("vgen_b200 DINO: input must be a CUDA tensor (no CPU path exists)")
        return self._forward_nchw(x.float().contiguous())

    def forward_nhwc(self, img):
        """img fp16 channels-last [n, H, W, in_chans] (CUDA, e.g. ops.resize_crop_normalize's output) -> fp32 [n, D]."""
        if not img.is_cuda or img.dtype != torch.float16 or img.dim() != 4 or img.shape[3] != self.in_chans:
            raise ops._l.VgenError(f"vgen_b200 DINO: expected a CUDA fp16 tensor [n, H, W, {self.in_chans}]")
        self._check_grid(img.shape[1], img.shape[2])
        return self._forward_nhwc(img.contiguous())

    @graphed
    @torch.no_grad()
    def _forward_nchw(self, x):
        self._packed or self._pack()
        n, c, H, Wd = x.shape
        return self._tower(ops.cp_to_pc(x, n, c, H * Wd).view(n, H, Wd, c))

    @graphed
    @torch.no_grad()
    def _forward_nhwc(self, img):
        self._packed or self._pack()
        return self._tower(img)

    def _tower(self, img):
        W = self._packed
        x = vit.embed(img, self.patch_size, W["patch.w"], W["patch.b"], W["cls"], W["pos"])
        for i in range(self.depth):
            x = vit.block(x, W, f"blocks.{i}.", self.num_heads, self.eps, attention="d64", scale=self.scale)
        n, L, D = x.shape
        y = ops.layer_norm(x.view(n, L * D)[:, :D], W["norm.g"], W["norm.b"], self.eps)     # the class tokens
        return ops.pc_to_cp(y.view(n, 1, D), n, D, 1, torch.float32).view(n, D)

    # ---- not provided ---------------------------------------------------------------------------
    def get_last_selfattention(self, x):
        raise NotImplementedError("vgen_b200 DINO: get_last_selfattention is not provided (the metric uses forward only)")

    def get_intermediate_layers(self, x, n=1):
        raise NotImplementedError("vgen_b200 DINO: get_intermediate_layers is not provided (the metric uses forward only)")

    def interpolate_pos_encoding(self, x, w, h):
        raise NotImplementedError("vgen_b200 DINO: interpolate_pos_encoding is not provided (inputs must be at the trained grid)")


def vit_tiny(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=192, depth=12, num_heads=3, mlp_ratio=4, qkv_bias=True,
                             norm_layer=functools.partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_small(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=384, depth=12, num_heads=6, mlp_ratio=4, qkv_bias=True,
                             norm_layer=functools.partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_base(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True,
                             norm_layer=functools.partial(nn.LayerNorm, eps=1e-6), **kwargs)


class DINOHead(nn.Module):
    """The self-distillation projection head (training only): not provided."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("vgen_b200 DINO: DINOHead (training / evaluation head) is not provided")
