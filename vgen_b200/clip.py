"""H100-native CLIP conditioning (SURVEY.md section 8f-4): drop-ins for the reference's `FrozenOpenCLIPEmbedder`,
`FrozenOpenCLIPVisualEmbedder`, `FrozenOpenCLIPTextVisualEmbedder` and `FrozenOpenCLIPCustomEmbedder`
(tools/modules/clip_embedder.py:10-370; the last takes DreamVideo's textual-inversion manager), i.e. the
ViT-H/14 text and image towers of open_clip's `CLIP` driven as those classes drive them:

  text   tokenize -> token + positional embedding -> the first (24 - layer_idx) causal pre-LN blocks -> ln_final
         -> (pooled @ text_projection, tokens [b, 77, 1024])                                          (:189-212)
  image  14x14 patch embedding -> class token + positional embedding -> ln_pre -> 32 blocks -> ln_post(class) @ proj
         (open_clip VisionTransformer.forward; the reference vendors a copy: utils/reward/open_clip/transformer.py:455-520)

Same constructor arguments; `.model` holds the parameters under open_clip's state_dict names, so
`open_clip_pytorch_model.bin` (a plain state_dict) loads with `strict=True`; `pretrained=None` leaves random weights.
Every op is a kernel of libvgen_b200.so: wgmma tap-GEMMs for the projections / MLPs (bias, residual in the epilogue),
LayerNorm, the small-attention kernel (77 causal tokens at head_dim 64; 257 tokens at head_dim 80), embedding gather.
The patch embedding and the blocks are the shared ViT trunk (vgen_b200.vit).
The reference runs CLIP in fp32; here activations are fp16 with fp32 accumulation / statistics (the UNet consumes the
tokens as fp16 anyway), embeddings are summed in fp32.  Tokenisation is `vgen_b200.clip_tokenizer` (bit-exact ids).
No CPU path: a CPU-resident model raises.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops, vit
from .clip_tokenizer import tokenize
from .graph import graphed
from .params import SpecModule
from .vit import f16, f32

ARCHS = {
    # utils/reward/open_clip/model_configs/ViT-H-14.json (the only arch the released configs use)
    "ViT-H-14": dict(embed_dim=1024, vision_cfg=dict(image_size=224, layers=32, width=1280, head_width=80, patch_size=14),
                     text_cfg=dict(context_length=77, vocab_size=49408, width=1024, heads=16, layers=24)),
}

# open_clip ResidualAttentionBlock: the state-dict prefixes of LN1, qkv, proj, LN2, fc1, fc2 (vit.pack_block)
_BLOCK = ("ln_1.", "attn.in_proj_", "attn.out_proj.", "ln_2.", "mlp.c_fc.", "mlp.c_proj.")


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
        self.act = cfg.get("act", "gelu")            # MLP activation: "gelu" (open_clip ViT-H) or "quick_gelu" (OpenAI)
        if self.act not in ("gelu", "quick_gelu"):
            raise ValueError(f"vgen_b200 CLIP: act must be 'gelu' or 'quick_gelu', got {self.act!r}")
        self._build_params(clip_spec(cfg, text, visual))
        with torch.no_grad():
            self.logit_scale.fill_(2.6592)

    # ---- packing -------------------------------------------------------------------------------
    def _pack(self):
        sd = self.state_dict()
        dev = self.device
        if dev.type != "cuda":
            raise ops._l.VgenError("vgen_b200 CLIP forward needs the model on a CUDA device (no CPU path exists)")
        W = {}
        if self.has_text:
            W["tok"], W["pos"] = f32(sd["token_embedding.weight"], dev), f32(sd["positional_embedding"], dev)
            for i in range(self.cfg["text_cfg"]["layers"]):
                vit.pack_block(W, sd, f"transformer.resblocks.{i}.", _BLOCK, dev)
            W["ln_final.g"], W["ln_final.b"] = f32(sd["ln_final.weight"], dev), f32(sd["ln_final.bias"], dev)
            W["text_projection.w"] = f16(sd["text_projection"].t(), dev)             # x @ P == linear(x, P^T)
        if self.has_visual:
            W["visual.conv1.w"] = vit.pack_patch(sd["visual.conv1.weight"], dev)
            W["visual.cls"] = f16(sd["visual.class_embedding"].reshape(1, -1), dev)
            W["visual.pos"] = f32(sd["visual.positional_embedding"], dev)
            for nm in ("visual.ln_pre.", "visual.ln_post."):
                W[nm + "g"], W[nm + "b"] = f32(sd[nm + "weight"], dev), f32(sd[nm + "bias"], dev)
            for i in range(self.cfg["vision_cfg"]["layers"]):
                vit.pack_block(W, sd, f"visual.transformer.resblocks.{i}.", _BLOCK, dev)
            W["visual.proj.w"] = f16(sd["visual.proj"].t(), dev)
        self._packed = W
        return W

    # ---- towers ----------------------------------------------------------------------------------
    def text_tokens(self, tokens, layer_idx=0, extra=None):
        """tokens int64 [b, 77] (CUDA) -> ln_final(tokens after the first n - layer_idx blocks), fp16 [b, 77, W].
        extra (fp32 [n_extra, W], CUDA): learned embeddings; an id >= vocab embeds row id - vocab of it (textual
        inversion, see embedding_manager.py), and every id must then be below vocab + n_extra (checked here, before
        the possibly graph-replayed forward)."""
        if extra is None:
            return self._text_tokens(tokens, layer_idx)
        ops.check_token_ids(tokens, self.cfg["text_cfg"]["vocab_size"] + extra.shape[0])
        return self._text_tokens(tokens, layer_idx, extra.contiguous())

    @graphed
    @torch.no_grad()
    def _text_tokens(self, tokens, layer_idx=0, extra=None):
        W = self._packed or self._pack()
        t = self.cfg["text_cfg"]
        if extra is None:
            x = ops.embed_tokens(tokens.contiguous(), W["tok"], W["pos"])
        else:
            x = ops.embed_tokens_extra(tokens.contiguous(), W["tok"], extra, W["pos"], check=False)
        for i in range(t["layers"] - int(layer_idx)):
            x = vit.block(x, W, f"transformer.resblocks.{i}.", t["heads"], act=self.act, causal=True)
        b, L, w = x.shape
        return ops.layer_norm(x.view(b * L, w), W["ln_final.g"], W["ln_final.b"]).view(b, L, w)

    @torch.no_grad()
    def encode_text(self, tokens, layer_idx=0, extra=None, pool_tokens=None):
        """-> (xt fp32 [b, E], x fp32 [b, 77, W]) like clip_embedder.py:204-212 (fp32 out: the reference's CLIP is fp32).
        With textual inversion `tokens` are the gather ids and `extra` the learned rows (text_tokens), and the pooled
        end-of-text position is taken from `pool_tokens`, the rewritten ids (clip_embedder.py:358)."""
        x = self.text_tokens(tokens, layer_idx, extra)
        eot = (tokens if pool_tokens is None else pool_tokens).argmax(dim=-1)  # index math, as in the reference
        pooled = x[torch.arange(x.shape[0], device=x.device), eot].contiguous()
        xt = ops.linear_small(pooled, self._packed["text_projection.w"])
        return xt.float(), x.float()

    @graphed
    @torch.no_grad()
    def encode_image(self, image):
        """image [b, 3, H, W] (preprocessed, CUDA) -> fp32 [b, E]."""
        if not image.is_cuda:
            raise ops._l.VgenError("vgen_b200 CLIP: image must be a CUDA tensor (no CPU path exists)")
        self._packed or self._pack()
        b, c, H, Wd = image.shape
        img = ops.cp_to_pc(image.float().contiguous(), b, c, H * Wd).view(b, H, Wd, c)              # channels-last fp16
        return self._image_tower(img).float()

    @graphed
    @torch.no_grad()
    def encode_image_nhwc(self, image):
        """image fp16 channels-last [b, H, W, 3] (preprocessed, CUDA; e.g. ops.resize_crop_normalize) -> fp32 [b, E]."""
        if not image.is_cuda or image.dtype != torch.float16 or image.dim() != 4 or image.shape[3] != 3:
            raise ops._l.VgenError("vgen_b200 CLIP: image must be a CUDA fp16 tensor [b, H, W, 3] (no CPU path exists)")
        self._packed or self._pack()
        y = self._image_tower(image.contiguous())
        return ops.pc_to_cp(y.view(y.shape[0], 1, y.shape[1]), y.shape[0], y.shape[1], 1, torch.float32).view(y.shape)

    def _image_tower(self, img):
        W = self._packed
        v = self.cfg["vision_cfg"]
        x = vit.embed(img, v["patch_size"], W["visual.conv1.w"], None, W["visual.cls"], W["visual.pos"])
        b, L, wv = x.shape
        x = ops.layer_norm(x.view(b * L, wv), W["visual.ln_pre.g"], W["visual.ln_pre.b"]).view(b, L, wv)
        heads = wv // v["head_width"]
        for i in range(v["layers"]):
            x = vit.block(x, W, f"visual.transformer.resblocks.{i}.", heads, act=self.act)
        pooled = ops.layer_norm(x.view(b, L * wv)[:, :wv], W["visual.ln_post.g"], W["visual.ln_post.b"])   # class tokens
        return ops.linear_small(pooled, W["visual.proj.w"])


def openai_cfg(sd):
    """The cfg of an OpenAI-format CLIP state dict, derived as build_model_from_openai_state_dict does
    (utils/reward/open_clip/model.py:354-397): widths, layer counts, patch size, grid, context length and vocabulary from
    the tensor shapes, heads = width // 64 in both towers, QuickGELU.  ModifiedResNet checkpoints raise."""
    if "visual.proj" not in sd:
        raise NotImplementedError("vgen_b200 CLIP: only the ViT CLIP models are supported; this state dict is a "
                                  "ModifiedResNet one (RN50, RN101, ...)")
    vw, ps = sd["visual.conv1.weight"].shape[0], sd["visual.conv1.weight"].shape[-1]
    grid = round((sd["visual.positional_embedding"].shape[0] - 1) ** 0.5)
    tw = sd["ln_final.weight"].shape[0]
    return dict(embed_dim=sd["text_projection"].shape[1], act="quick_gelu",
                vision_cfg=dict(image_size=ps * grid, patch_size=ps, width=vw, head_width=64,
                                layers=len([k for k in sd if k.startswith("visual.") and k.endswith(".attn.in_proj_weight")])),
                text_cfg=dict(context_length=sd["positional_embedding"].shape[0], vocab_size=sd["token_embedding.weight"].shape[0],
                              width=tw, heads=tw // 64,
                              layers=len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks")})))


class OpenAIClipModel(ClipModel):
    """OpenAI's CLIP as `clip.load` returns it (vgen_b200.metric.load_clip builds it): encode_text(ids [b, 77]) and
    encode_image(images [b, 3, H, W]) -> fp32 [b, E]."""

    def __init__(self, cfg):
        super().__init__(cfg, text=True, visual=True)

    @torch.no_grad()
    def encode_text(self, tokens):
        """The pooled end-of-text position is found on the host (ids are host data), so the device runs library kernels
        only: the text tower, one row copy per prompt, the projection and the fp32 conversion."""
        ids = tokens.detach().to("cpu", torch.int64)
        eot = ids.argmax(dim=-1).tolist()
        x = self.text_tokens(ids.to(self.device))
        b, L, w = x.shape
        pooled = torch.empty(b, w, device=x.device, dtype=torch.float16)
        for i, e in enumerate(eot):
            ops.copy2d(x[i, e:e + 1], pooled[i:i + 1])
        xt = ops.linear_small(pooled, self._packed["text_projection.w"])
        return ops.pc_to_cp(xt.view(b, 1, -1), b, xt.shape[1], 1, torch.float32).view(b, -1)


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


OPENAI_DATASET_MEAN = (0.48145466, 0.4578275, 0.40821073)      # utils/reward/open_clip/constants.py
OPENAI_DATASET_STD = (0.26862954, 0.26130258, 0.27577711)


def white_image(image_size):
    """open_clip's eval transform (resize, centre crop, normalise with the OpenAI mean / std) of an all-255 RGB image:
    the resize and crop leave a constant image constant, so it is (1 - mean) / std per channel, [1, 3, S, S] fp32."""
    mean = torch.tensor(OPENAI_DATASET_MEAN, dtype=torch.float32).view(3, 1, 1)
    std = torch.tensor(OPENAI_DATASET_STD, dtype=torch.float32).view(3, 1, 1)
    return ((torch.ones(3, image_size, image_size) - mean) / std).unsqueeze(0)


class FrozenOpenCLIPCustomEmbedder(_EmbedderBase):
    """clip_embedder.py:306-370 (DreamVideo's embedder): both towers, and text through an optional textual-inversion
    `EmbeddingManager` (vgen_b200.embedding_manager).  forward(image, text, embedding_manager) -> (xi | None, xt, x).
    The manager's substitution runs on the host over the ids (EmbeddingManager.plan); the learned vectors enter in
    the token-gather kernel, and the pooled end-of-text position follows the rewritten ids like the reference's."""

    @property
    def white_image(self):
        """The open_clip eval transform of a white image (the reference builds it at vit_resolution; the transform
        resizes and crops to the tower's input size, clip_embedder.py:323-324)."""
        return white_image(self.model.cfg["vision_cfg"]["image_size"])

    def forward(self, image=None, text=None, embedding_manager=None):
        xi = self.model.encode_image(image.to(self._dev())) if image is not None else None
        xt, x = self.encode_with_transformer(tokenize(text), embedding_manager)
        return xi, xt, x

    def encode_with_transformer(self, tokens, embedding_manager=None):
        """tokens int64 [b, 77] -> (xt fp32 [b, E], x fp32 [b, 77, W]) (clip_embedder.py:348-358)."""
        dev = self._dev()
        if embedding_manager is None:
            return self.model.encode_text(tokens.to(dev), self.layer_idx)
        from .embedding_manager import EmbeddingManager
        if not isinstance(embedding_manager, EmbeddingManager):
            raise TypeError(f"vgen_b200 FrozenOpenCLIPCustomEmbedder: embedding_manager must be a "
                            f"vgen_b200.embedding_manager.EmbeddingManager, got {type(embedding_manager).__name__} "
                            "(build it after vgen_b200.register())")
        ids, gather, extra = embedding_manager.plan(tokens, self.model.cfg["text_cfg"]["vocab_size"])
        if extra is None:
            return self.model.encode_text(ids.to(dev), self.layer_idx)
        return self.model.encode_text(gather.to(dev), self.layer_idx, extra=extra.to(dev), pool_tokens=ids.to(dev))

    def encode_image(self, image):
        return self.model.encode_image(image)

    def encode(self, text):
        return self(text=text)
