"""H100-native MiDaS v3.0 DPT-Large, the depth annotator of the VideoComposer engines: a drop-in for `MiDaS` / `midas_v3`
of tools/annotator/depth/__init__.py:162-309 (inference_{tft2v,videolcm}_vcomposer_entrance.py build it for every video
whose config lists 'depthmap').

  patch embedding (im2col + tap-GEMM) -> cls token + position rows (resampled to the input's patch grid on the host)
  -> 24 pre-LN blocks in four slices; after each slice the readout gelu(fc_i(cat[token, cls])) and the stage's neck
  -> four FusionBlocks (ReLU'd residual conv units, 1x1 conv_out, bilinear x2) -> head (conv3x3, bilinear x2, conv3x3,
  ReLU -> 32 -> 1 -> ReLU).

Same constructor, parameter names, shapes and order as the reference, so `midas_v3_dpt_large.pth` loads with
`strict=True`.  The forward takes [n, 3, H, W] on the GPU (NCHW-contiguous or channels_last) in the module's parameter
dtype and returns [n, 1, H, W] in that dtype.  Every op is a kernel of libvgen_b200.so; activations are fp16 channels-last
with fp32 accumulation, fp32 LayerNorm / softmax statistics.  The patch embedding and the blocks are the shared ViT
trunk (vgen_b200.vit).  Kernel-level notes are in DESIGN.md section 3.
No CPU path: a CPU input or a CPU-resident model raises VgenError.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ops, vit
from .graph import graphed
from .params import SpecModule
from .vit import f16, f32

__all__ = ["MiDaS", "midas_v3"]

# AttentionBlock (depth/__init__.py:57-76): the state-dict prefixes of LN1, qkv, proj, LN2, fc1, fc2 (vit.pack_block)
_BLOCK = ("norm1.", "attn.to_qkv.", "attn.proj.", "norm2.", "mlp.0.", "mlp.2.")


def midas_spec(image_size=384, patch_size=16, dim=1024, neck_dims=(256, 512, 1024, 1024), fusion_dim=256, num_layers=24):
    """(name, shape) in the order of the reference MiDaS.state_dict()."""
    p, f = patch_size, fusion_dim

    def conv(nm, co, ci, k, bias=True):
        return [(nm + ".weight", (co, ci, k, k))] + ([(nm + ".bias", (co,))] if bias else [])

    spec = [("cls_embedding", (1, 1, dim)), ("pos_embedding", (1, (image_size // p) ** 2 + 1, dim))]
    spec += conv("patch_embedding", dim, 3, p)
    for i in range(num_layers):
        b = f"blocks.{i}."
        spec += [(b + "norm1.weight", (dim,)), (b + "norm1.bias", (dim,)), (b + "attn.to_qkv.weight", (3 * dim, dim)),
                 (b + "attn.to_qkv.bias", (3 * dim,)), (b + "attn.proj.weight", (dim, dim)), (b + "attn.proj.bias", (dim,)),
                 (b + "norm2.weight", (dim,)), (b + "norm2.bias", (dim,)), (b + "mlp.0.weight", (4 * dim, dim)),
                 (b + "mlp.0.bias", (4 * dim,)), (b + "mlp.2.weight", (dim, 4 * dim)), (b + "mlp.2.bias", (dim,))]
    for k in range(1, 5):
        c = neck_dims[k - 1]
        spec += [(f"fc{k}.0.weight", (dim, 2 * dim)), (f"fc{k}.0.bias", (dim,))]
        spec += conv(f"conv{k}.0", c, dim, 1)
        if k in (1, 2):
            s = 4 if k == 1 else 2
            spec += [(f"conv{k}.1.weight", (c, c, s, s)), (f"conv{k}.1.bias", (c,))]
            spec += conv(f"conv{k}.2", f, c, 3, bias=False)
        elif k == 3:
            spec += conv("conv3.1", f, c, 3, bias=False)
        else:
            spec += conv("conv4.1", c, c, 3) + conv("conv4.2", f, c, 3, bias=False)
        for layer in ("layer1", "layer2"):
            spec += conv(f"fusion{k}.{layer}.residual.1", f, f, 3) + conv(f"fusion{k}.{layer}.residual.3", f, f, 3)
        spec += conv(f"fusion{k}.conv_out", f, f, 1)
    spec += conv("head.0", f // 2, f, 3) + conv("head.2", 32, f // 2, 3)
    spec += [("head.4.weight", (32, 1, 1, 1)), ("head.4.bias", (1,))]
    return spec


class MiDaS(SpecModule):
    r"""MiDaS v3.0 DPT-Large (depth/__init__.py:162-293) on the native path."""

    def __init__(self, image_size=384, patch_size=16, dim=1024, neck_dims=[256, 512, 1024, 1024], fusion_dim=256,  # noqa: B006
                 num_heads=16, num_layers=24):
        super().__init__()
        if image_size % patch_size != 0 or num_layers % 4 != 0 or dim % num_heads != 0:
            raise ValueError(f"MiDaS: image_size {image_size} must be a multiple of patch_size {patch_size}, num_layers "
                             f"{num_layers} a multiple of 4 and dim {dim} a multiple of num_heads {num_heads}")
        if len(neck_dims) != 4 or any(c % 64 for c in neck_dims) or fusion_dim % 128:
            raise NotImplementedError(f"vgen_b200 MiDaS: neck_dims {list(neck_dims)} must be multiples of 64 and fusion_dim "
                                      f"{fusion_dim} a multiple of 128 (every neck / head conv runs on the wgmma tap-GEMM)")
        self.image_size, self.patch_size, self.dim = image_size, patch_size, dim
        self.neck_dims, self.fusion_dim, self.num_heads, self.num_layers = neck_dims, fusion_dim, num_heads, num_layers
        self.num_patches = (image_size // patch_size) ** 2
        stride = num_layers // 4
        self.slices = [slice(i * stride, (i + 1) * stride) for i in range(4)]
        self._build_params(midas_spec(image_size, patch_size, dim, neck_dims, fusion_dim, num_layers),
                           zero_init=lambda nm: nm == "cls_embedding")

    # ---- packing -------------------------------------------------------------------------------
    def _pack(self):
        dev = self.device
        if dev.type != "cuda":
            raise ops._l.VgenError("vgen_b200 MiDaS forward needs the model on a CUDA device (no CPU path exists)")
        sd = self.state_dict()
        # conv weight [co, ci, kh, kw] -> [co, (ky, kx, ci)], the tap-GEMM's K order
        taps = lambda w: f16(w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1), dev)  # noqa: E731
        d = self.dim
        W = {"pe.w": vit.pack_patch(sd["patch_embedding.weight"], dev), "pe.b": f32(sd["patch_embedding.bias"], dev),
             "cls": f16(sd["cls_embedding"].reshape(1, d), dev),
             "pos_src": sd["pos_embedding"].detach().to(device="cpu", dtype=torch.float32).reshape(-1, d)}
        for i in range(self.num_layers):
            vit.pack_block(W, sd, f"blocks.{i}.", _BLOCK, dev)
        for s in range(1, 5):
            w = sd[f"fc{s}.0.weight"]
            W[f"fc{s}.tok"], W[f"fc{s}.cls"], W[f"fc{s}.b"] = f16(w[:, :d], dev), f16(w[:, d:], dev), f32(sd[f"fc{s}.0.bias"], dev)
            W[f"conv{s}.0.w"], W[f"conv{s}.0.b"] = f16(sd[f"conv{s}.0.weight"].flatten(1), dev), f32(sd[f"conv{s}.0.bias"], dev)
            if s in (1, 2):
                W[f"conv{s}.1.w"] = f16(ops.pack_conv_transpose_weight(sd[f"conv{s}.1.weight"]), dev)
                W[f"conv{s}.1.b"] = f32(sd[f"conv{s}.1.bias"], dev)
                W[f"conv{s}.2.w"] = taps(sd[f"conv{s}.2.weight"])
            elif s == 3:
                W["conv3.1.w"] = taps(sd["conv3.1.weight"])
            else:
                W["conv4.1.w"], W["conv4.1.b"] = taps(sd["conv4.1.weight"]), f32(sd["conv4.1.bias"], dev)
                W["conv4.2.w"] = taps(sd["conv4.2.weight"])
            for nm in ("layer1.residual.1", "layer1.residual.3", "layer2.residual.1", "layer2.residual.3"):
                q = f"fusion{s}.{nm}"
                W[q + ".w"], W[q + ".b"] = taps(sd[q + ".weight"]), f32(sd[q + ".bias"], dev)
            q = f"fusion{s}.conv_out"
            W[q + ".w"], W[q + ".b"] = f16(sd[q + ".weight"].flatten(1), dev), f32(sd[q + ".bias"], dev)
        for nm in ("head.0", "head.2"):
            W[nm + ".w"], W[nm + ".b"] = taps(sd[nm + ".weight"]), f32(sd[nm + ".bias"], dev)
        W["head.4.w"], W["head.4.b"] = f32(sd["head.4.weight"].reshape(-1), dev), f32(sd["head.4.bias"], dev)
        self._packed = W
        return W

    def _pos(self, W, hp, wp):
        """Position rows for an hp x wp patch grid: the cls row, then the grid x grid table resampled bilinearly
        (align_corners=False, as depth/__init__.py:250-256 does per call) -- on the host in fp32, once per grid."""
        key = f"pos@{hp}x{wp}"
        if key not in W:
            src, grid = W["pos_src"], self.image_size // self.patch_size
            g = F.interpolate(src[1:].reshape(1, grid, grid, -1).permute(0, 3, 1, 2), size=(hp, wp), mode="bilinear",
                              align_corners=False).permute(0, 2, 3, 1).reshape(hp * wp, -1)
            W[key] = torch.cat([src[:1], g]).contiguous().to(W["cls"].device)
        return W[key]

    # ---- forward ---------------------------------------------------------------------------------
    def forward(self, x):
        """x [n, 3, H, W] CUDA, NCHW-contiguous or channels_last, in the parameter dtype -> depth [n, 1, H, W], x's dtype."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"MiDaS: expected [n, 3, H, W], got {tuple(x.shape)}")
        n, _, H, Wd = x.shape
        m = 2 * self.patch_size
        if H % m or Wd % m:
            raise ValueError(f"MiDaS: H and W must be multiples of {m} (the fusion adds stage maps of H/{self.patch_size} "
                             f"and its half), got {H} x {Wd}")
        if self.dim != 64 * self.num_heads:
            raise NotImplementedError(f"vgen_b200 MiDaS: head_dim {self.dim // self.num_heads} (the attention kernel serves 64)")
        if not x.is_cuda:
            raise ops._l.VgenError("vgen_b200 MiDaS: x must be a CUDA tensor (no CPU path exists)")
        dt = next(self.parameters()).dtype
        if x.dtype not in (torch.float16, torch.float32) or x.dtype != dt:
            raise TypeError(f"MiDaS: x is {x.dtype}, the module's parameters are {dt}")
        if x.is_contiguous():
            img = ops.cp_to_pc(x, n, 3, H * Wd)
        elif x.is_contiguous(memory_format=torch.channels_last):
            nhwc = x.permute(0, 2, 3, 1)
            img = nhwc if x.dtype == torch.float16 else ops.cp_to_pc(nhwc, n * H * Wd, 3, 1)
        else:
            raise ValueError("MiDaS: x must be NCHW-contiguous or channels_last")
        W = self._packed or self._pack()
        self._pos(W, H // self.patch_size, Wd // self.patch_size)
        return self._forward_nhwc(img.reshape(n, H, Wd, 3), x.dtype == torch.float32)

    @graphed
    @torch.no_grad()
    def _forward_nhwc(self, img, out_f32):
        W = self._packed
        n, H, Wd, _ = img.shape
        p = self.patch_size
        hp, wp = H // p, Wd // p
        x = vit.embed(img, p, W["pe.w"], W["pe.b"], W["cls"], self._pos(W, hp, wp))
        feats = []
        for s, sl in enumerate(self.slices, 1):
            for i in range(sl.start, sl.stop):
                x = vit.block(x, W, f"blocks.{i}.", self.num_heads, attention="d64")
            feats.append(self._neck(s, self._readout(x, W, s, hp, wp), W, n, hp, wp))
        y = self._fusion(W, 4, feats[3])
        for s in (3, 2, 1):
            y = self._fusion(W, s, y, feats[s - 1])
        h = ops.conv2d_3x3(y, W["head.0.w"], bias=W["head.0.b"])
        h = ops.conv2d_3x3(ops.upsample_bilinear2x(h), W["head.2.w"], bias=W["head.2.b"])
        out = ops.dpt_head_out(h, W["head.4.w"], W["head.4.b"], torch.float32 if out_f32 else torch.float16)
        return out.view(n, 1, H, Wd)

    @staticmethod
    def _readout(x, W, s, hp, wp):
        """gelu(fc_s(cat[token, cls])) = gelu(token W_tok^T + (cls W_cls^T + b)): the cls half is one fp32 row bias per
        image, added in the GEMM epilogue.  -> [n*hp*wp, d]."""
        n, L, d = x.shape
        xr = x.view(n, L * d)
        tok = torch.empty(n, hp * wp * d, device=x.device, dtype=torch.float16)
        ops.copy2d(xr[:, d:], tok)
        cls = ops.adapter_condition(xr[:, :d], W[f"fc{s}.cls"], W[f"fc{s}.b"])
        return ops.linear_gelu_rowbias(tok.view(n * hp * wp, d), W[f"fc{s}.tok"], row_bias=cls, rows_per_group=hp * wp)

    @staticmethod
    def _neck(s, t, W, n, hp, wp):
        """conv_s (depth/__init__.py:200-232) on the readout tokens -> fusion_dim channels at 4, 2, 1, 1/2 x the patch grid."""
        y = ops.linear(t, W[f"conv{s}.0.w"], bias=W[f"conv{s}.0.b"])
        y = y.view(n, hp, wp, y.shape[-1])
        if s in (1, 2):
            y = ops.conv_transpose_stride(y, W[f"conv{s}.1.w"], W[f"conv{s}.1.b"], 4 if s == 1 else 2)
            return ops.conv2d_3x3(y, W[f"conv{s}.2.w"])
        if s == 3:
            return ops.conv2d_3x3(y, W["conv3.1.w"])
        c = y.shape[-1]
        col = ops.im2col(y, 3, 3, 2, 1, 1, hp // 2, wp // 2, 9 * c)
        y = ops.linear(col, W["conv4.1.w"], bias=W["conv4.1.b"]).view(n, hp // 2, wp // 2, c)
        return ops.conv2d_3x3(y, W["conv4.2.w"])

    @staticmethod
    def _residual(x, W, q):
        """ResidualBlock (depth/__init__.py:125-139): x + conv(relu(conv(relu(x))))."""
        t = ops.conv2d_3x3(ops.eltwise("relu", x), W[q + ".residual.1.w"], bias=W[q + ".residual.1.b"])
        t = ops.eltwise("relu", t, out=t)
        return ops.conv2d_3x3(t, W[q + ".residual.3.w"], bias=W[q + ".residual.3.b"], residual=x)

    def _fusion(self, W, s, x0, x1=None):
        """FusionBlock (depth/__init__.py:141-160).  conv_out (1x1 + bias) runs BEFORE the bilinear x2: the interpolation
        weights sum to one, so the two commute, and the conv then costs a quarter of the FLOPs."""
        q = f"fusion{s}."
        x = x0 if x1 is None else ops.eltwise("add", x0, self._residual(x1, W, q + "layer1"))
        x = self._residual(x, W, q + "layer2")
        n, h, w, c = x.shape
        x = ops.linear(x.view(n * h * w, c), W[q + "conv_out.w"], bias=W[q + "conv_out.b"]).view(n, h, w, c)
        return ops.upsample_bilinear2x(x)


def midas_v3(pretrained=False, **kwargs):
    """depth/__init__.py:295-309: MiDaS v3.0 DPT-Large; pretrained=True loads models/midas_v3_dpt_large.pth relative to the
    working directory, as the reference does."""
    cfg = dict(image_size=384, patch_size=16, dim=1024, neck_dims=[256, 512, 1024, 1024], fusion_dim=256, num_heads=16,
               num_layers=24)
    cfg.update(**kwargs)
    model = MiDaS(**cfg)
    if pretrained:
        model.load_state_dict(torch.load("models/midas_v3_dpt_large.pth", map_location="cpu"))
    return model
