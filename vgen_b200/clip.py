"""H100-native CLIP conditioning (SURVEY.md section 8f-4): drop-ins for the reference's `FrozenOpenCLIPEmbedder`,
`FrozenOpenCLIPVisualEmbedder` and `FrozenOpenCLIPTextVisualEmbedder` (tools/modules/clip_embedder.py:10-245), i.e. the
ViT-H/14 text and image towers of open_clip's `CLIP` driven as those classes drive them:

  text   tokenize -> token + positional embedding -> the first (24 - layer_idx) causal pre-LN blocks -> ln_final
         -> (pooled @ text_projection, tokens [b, 77, 1024])                                          (:189-212)
  image  14x14 patch embedding -> class token + positional embedding -> ln_pre -> 32 blocks -> ln_post(class) @ proj
         (open_clip VisionTransformer.forward; the reference vendors a copy: utils/reward/open_clip/transformer.py:455-520)

Same constructor arguments; `.model` holds the parameters under open_clip's state_dict names, so
`open_clip_pytorch_model.bin` (a plain state_dict) loads with `strict=True`; `pretrained=None` leaves random weights.
Every op is a kernel of libvgen_b200.so: wgmma tap-GEMMs for the projections / MLPs (bias, residual in the epilogue),
LayerNorm, the small-attention kernel (77 causal tokens at head_dim 64; 257 tokens at head_dim 80), embedding gather.
The reference runs CLIP in fp32; here activations are fp16 with fp32 accumulation / statistics (the UNet consumes the
tokens as fp16 anyway), embeddings are summed in fp32.  Tokenisation is `vgen_b200.clip_tokenizer` (bit-exact ids).
No CPU path: a CPU-resident model raises.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .clip_tokenizer import tokenize
from .graph import graphed
from .params import SpecModule

ARCHS = {
    # utils/reward/open_clip/model_configs/ViT-H-14.json (the only arch the released configs use)
    "ViT-H-14": dict(embed_dim=1024, vision_cfg=dict(image_size=224, layers=32, width=1280, head_width=80, patch_size=14),
                     text_cfg=dict(context_length=77, vocab_size=49408, width=1024, heads=16, layers=24)),
}


def _block_spec(p, w):
    return [(p + "ln_1.weight", (w,)), (p + "ln_1.bias", (w,)), (p + "attn.in_proj_weight", (3 * w, w)),
            (p + "attn.in_proj_bias", (3 * w,)), (p + "attn.out_proj.weight", (w, w)), (p + "attn.out_proj.bias", (w,)),
            (p + "ln_2.weight", (w,)), (p + "ln_2.bias", (w,)), (p + "mlp.c_fc.weight", (4 * w, w)), (p + "mlp.c_fc.bias", (4 * w,)),
            (p + "mlp.c_proj.weight", (w, 4 * w)), (p + "mlp.c_proj.bias", (w,))]


def clip_spec(cfg, text=True, visual=True):
    """(name, shape) in the order of open_clip's CLIP.state_dict()."""
    E, v, t = cfg["embed_dim"], cfg["vision_cfg"], cfg["text_cfg"]
    spec = []
    if text:
        spec += [("positional_embedding", (t["context_length"], t["width"])), ("text_projection", (t["width"], E))]
    spec += [("logit_scale", ())]
    if visual:
        wv, grid = v["width"], v["image_size"] // v["patch_size"]
        spec += [("visual.class_embedding", (wv,)), ("visual.positional_embedding", (grid * grid + 1, wv)), ("visual.proj", (wv, E)),
                 ("visual.conv1.weight", (wv, 3, v["patch_size"], v["patch_size"])), ("visual.ln_pre.weight", (wv,)),
                 ("visual.ln_pre.bias", (wv,))]
        for i in range(v["layers"]):
            spec += _block_spec(f"visual.transformer.resblocks.{i}.", wv)
        spec += [("visual.ln_post.weight", (wv,)), ("visual.ln_post.bias", (wv,))]
    if text:
        for i in range(t["layers"]):
            spec += _block_spec(f"transformer.resblocks.{i}.", t["width"])
        spec += [("token_embedding.weight", (t["vocab_size"], t["width"])), ("ln_final.weight", (t["width"],)),
                 ("ln_final.bias", (t["width"],))]
    return spec


class ClipModel(SpecModule):
    """Parameter holder + forward of the two towers (the object the reference's embedders keep as `.model`)."""

    def __init__(self, cfg, text=True, visual=True):
        super().__init__()
        self.cfg, self.has_text, self.has_visual = cfg, text, visual
        self._build_params(clip_spec(cfg, text, visual))
        with torch.no_grad():
            self.logit_scale.fill_(2.6592)

    # ---- packing -------------------------------------------------------------------------------
    def _pack(self):
        sd = self.state_dict()
        dev = self.device
        if dev.type != "cuda":
            raise ops._l.VgenError("vgen_b200 CLIP forward needs the model on a CUDA device (no CPU path exists)")
        f16 = lambda t: t.detach().to(device=dev, dtype=torch.float16).contiguous()  # noqa: E731
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()  # noqa: E731
        W = {}

        def block(p):
            for ln in ("ln_1.", "ln_2."):
                W[p + ln + "g"], W[p + ln + "b"] = f32(sd[p + ln + "weight"]), f32(sd[p + ln + "bias"])
            W[p + "qkv.w"], W[p + "qkv.b"] = f16(sd[p + "attn.in_proj_weight"]), f32(sd[p + "attn.in_proj_bias"])
            W[p + "out.w"], W[p + "out.b"] = f16(sd[p + "attn.out_proj.weight"]), f32(sd[p + "attn.out_proj.bias"])
            W[p + "fc.w"], W[p + "fc.b"] = f16(sd[p + "mlp.c_fc.weight"]), f32(sd[p + "mlp.c_fc.bias"])
            W[p + "proj.w"], W[p + "proj.b"] = f16(sd[p + "mlp.c_proj.weight"]), f32(sd[p + "mlp.c_proj.bias"])

        if self.has_text:
            W["tok"], W["pos"] = f32(sd["token_embedding.weight"]), f32(sd["positional_embedding"])
            for i in range(self.cfg["text_cfg"]["layers"]):
                block(f"transformer.resblocks.{i}.")
            W["ln_final.g"], W["ln_final.b"] = f32(sd["ln_final.weight"]), f32(sd["ln_final.bias"])
            W["text_projection.w"] = f16(sd["text_projection"].t())                  # x @ P == linear(x, P^T)
        if self.has_visual:
            v = self.cfg["vision_cfg"]
            w = sd["visual.conv1.weight"]                                           # [wv, 3, p, p] -> [wv, (ky, kx, c)] K-padded
            k = w.shape[2] * w.shape[3] * 3
            kpad = ((k + 63) // 64) * 64
            wp = torch.zeros(w.shape[0], kpad)
            wp[:, :k] = w.detach().float().cpu().permute(0, 2, 3, 1).reshape(w.shape[0], k)
            W["visual.conv1.w"] = f16(wp)
            W["visual.cls"], W["visual.pos"] = f16(sd["visual.class_embedding"].reshape(1, -1)), f32(sd["visual.positional_embedding"])
            for nm in ("ln_pre.", "ln_post."):
                W["visual." + nm + "g"], W["visual." + nm + "b"] = f32(sd["visual." + nm + "weight"]), f32(sd["visual." + nm + "bias"])
            for i in range(v["layers"]):
                block(f"visual.transformer.resblocks.{i}.")
            W["visual.proj.w"] = f16(sd["visual.proj"].t())
        self._packed = W
        return W

    # ---- one residual block (ResidualAttentionBlock.forward) -------------------------------------
    @staticmethod
    def _block(x, W, p, heads, causal):
        b, L, w = x.shape
        x2 = x.view(b * L, w)
        h = ops.layer_norm(x2, W[p + "ln_1.g"], W[p + "ln_1.b"])
        qkv = ops.linear(h, W[p + "qkv.w"], bias=W[p + "qkv.b"]).view(b, L, 3 * w)
        a = ops.attention_cross_small(qkv[:, :, :w], qkv[:, :, w:2 * w], qkv[:, :, 2 * w:], heads, causal=causal)
        x2 = ops.linear(a.view(b * L, w), W[p + "out.w"], bias=W[p + "out.b"], residual=x2)
        h = ops.layer_norm(x2, W[p + "ln_2.g"], W[p + "ln_2.b"])
        h = ops.eltwise("gelu", ops.linear(h, W[p + "fc.w"], bias=W[p + "fc.b"]))
        return ops.linear(h, W[p + "proj.w"], bias=W[p + "proj.b"], residual=x2).view(b, L, w)

    # ---- towers ----------------------------------------------------------------------------------
    @graphed
    @torch.no_grad()
    def text_tokens(self, tokens, layer_idx=0):
        """tokens int64 [b, 77] (CUDA) -> ln_final(tokens after the first n - layer_idx blocks), fp16 [b, 77, W]."""
        W = self._packed or self._pack()
        t = self.cfg["text_cfg"]
        x = ops.embed_tokens(tokens.contiguous(), W["tok"], W["pos"])
        for i in range(t["layers"] - int(layer_idx)):
            x = self._block(x, W, f"transformer.resblocks.{i}.", t["heads"], True)
        b, L, w = x.shape
        return ops.layer_norm(x.view(b * L, w), W["ln_final.g"], W["ln_final.b"]).view(b, L, w)

    @torch.no_grad()
    def encode_text(self, tokens, layer_idx=0):
        """-> (xt fp32 [b, E], x fp32 [b, 77, W]) like clip_embedder.py:204-212 (fp32 out: the reference's CLIP is fp32)."""
        x = self.text_tokens(tokens, layer_idx)
        eot = tokens.argmax(dim=-1)                                           # index math, as in the reference
        pooled = x[torch.arange(x.shape[0], device=x.device), eot].contiguous()
        xt = ops.linear_small(pooled, self._packed["text_projection.w"])
        return xt.float(), x.float()

    @graphed
    @torch.no_grad()
    def encode_image(self, image):
        """image [b, 3, H, W] (preprocessed, CUDA) -> fp32 [b, E]."""
        if not image.is_cuda:
            raise ops._l.VgenError("vgen_b200 CLIP: image must be a CUDA tensor (no CPU path exists)")
        W = self._packed or self._pack()
        v = self.cfg["vision_cfg"]
        b, c, H, Wd = image.shape
        ps, wv = v["patch_size"], v["width"]
        gh, gw = H // ps, Wd // ps
        img = ops.cp_to_pc(image.float().contiguous(), b, c, H * Wd).view(b, H, Wd, c)              # channels-last fp16
        col = ops.im2col(img, ps, ps, ps, 0, 0, gh, gw, W["visual.conv1.w"].shape[1])
        patches = ops.linear(col, W["visual.conv1.w"]).view(b, gh * gw, wv)
        L = gh * gw + 1
        x = torch.empty(b, L, wv, device=image.device, dtype=torch.float16)
        xr = x.view(b, L * wv)
        ops.copy2d(W["visual.cls"].expand(b, wv), xr[:, :wv])
        ops.copy2d(patches.view(b, gh * gw * wv), xr[:, wv:])
        ops.add_rows_f32_(x, W["visual.pos"])
        x = ops.layer_norm(x.view(b * L, wv), W["visual.ln_pre.g"], W["visual.ln_pre.b"]).view(b, L, wv)
        heads = wv // v["head_width"]
        for i in range(v["layers"]):
            x = self._block(x, W, f"visual.transformer.resblocks.{i}.", heads, False)
        pooled = ops.layer_norm(x[:, 0].contiguous(), W["visual.ln_post.g"], W["visual.ln_post.b"])
        return ops.linear_small(pooled, W["visual.proj.w"]).float()


class _EmbedderBase(nn.Module):
    LAYERS = ["last", "penultimate"]
    TEXT, VISUAL = True, True

    def __init__(self, pretrained=None, vit_resolution=(224, 224), arch="ViT-H-14", device="cuda", max_length=77, freeze=True,
                 layer="last", **kwargs):
        super().__init__()
        assert layer in self.LAYERS
        cfg = arch if isinstance(arch, dict) else ARCHS.get(arch)
        if cfg is None:
            raise NotImplementedError(f"vgen_b200 CLIP: arch '{arch}' (the released configs use ViT-H-14)")
        self.model = ClipModel(cfg, text=self.TEXT, visual=self.VISUAL)
        if pretrained is not None:
            sd = torch.load(pretrained, map_location="cpu")
            sd = sd.get("state_dict", sd)
            keep = {k for k, _ in clip_spec(cfg, self.TEXT, self.VISUAL)}
            self.model.load_state_dict({k: v for k, v in sd.items() if k in keep}, strict=True)
        self.device, self.max_length, self.layer = device, max_length, layer
        self.layer_idx = {"last": 0, "penultimate": 1}[layer]
        self.vit_resolution = tuple(vit_resolution)
        if freeze:
            self.freeze()

    def freeze(self):
        self.model = self.model.eval()
        for p in self.parameters():
            p.requires_grad = False

    def _dev(self):
        return self.model.device


class FrozenOpenCLIPEmbedder(_EmbedderBase):
    """clip_embedder.py:10-77: text tokens only."""
    VISUAL = False

    def forward(self, text):
        return self.model.encode_text(tokenize(text).to(self._dev()), self.layer_idx)[1]

    encode = forward


class FrozenOpenCLIPEmbedderZero(FrozenOpenCLIPEmbedder):
    """clip_embedder.py:230-300 (InstructVideo's embedder): forward(text) is the same text tower as FrozenOpenCLIPEmbedder.
    The reference's white_image, zero_feature and forward_image (image features for reward training) need the visual tower
    and are not provided: they raise NotImplementedError.  The inference entrance reads zero_feature once without using it
    (inference_instructvideo_entrance.py:145); INTEGRATION.md says to drop that line."""

    def __init__(self, pretrained, vit_resolution=(224, 224), arch="ViT-H-14", device="cuda", max_length=77, freeze=True,
                 layer="last"):
        super().__init__(pretrained=pretrained, vit_resolution=vit_resolution, arch=arch, device=device,
                         max_length=max_length, freeze=freeze, layer=layer)

    @staticmethod
    def _training_only(name):
        raise NotImplementedError(f"vgen_b200 FrozenOpenCLIPEmbedderZero.{name}: the image features of InstructVideo's reward "
                                  "training are not provided (text tower only)")

    @property
    def white_image(self):
        self._training_only("white_image")

    @property
    def zero_feature(self):
        self._training_only("zero_feature")

    def forward_image(self, image):
        self._training_only("forward_image")


class FrozenOpenCLIPVisualEmbedder(_EmbedderBase):
    """clip_embedder.py:80-143: image embedding only."""
    TEXT = False

    def forward(self, image):
        return self.model.encode_image(image.to(self._dev()))

    encode = forward


class FrozenOpenCLIPTextVisualEmbedder(_EmbedderBase):
    """clip_embedder.py:146-217: (image embedding | None, pooled text embedding, text tokens)."""

    def forward(self, image=None, text=None):
        xi = self.model.encode_image(image.to(self._dev())) if image is not None else None
        xt, x = self.model.encode_text(tokenize(text).to(self._dev()), self.layer_idx)
        return xi, xt, x

    def encode_image(self, image):
        return self.model.encode_image(image)

    def encode(self, text):
        return self(text=text)
