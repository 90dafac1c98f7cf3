"""H100-native UNetSD_T2VBase / UNetSD_I2VGen / UNetSD_VideoLCM / UNetSD_TFT2V / UNetSD_DreamVideo / UNetSD_LoRA /
UNetSD_SR600 / UNetSD_HiGen: same constructor arguments, state_dict keys and forward signatures as the reference classes
(tools/modules/unet/unet_t2v.py:19-277, unet_i2vgen.py:19-346, unet_videolcm.py:188-760, unet_tf2tv.py:188-753,
unet_dreamvideo.py:19-290, unet_lora.py:1091-1409, unet_sr600.py:52-299, unet_higen.py:175-467), but
the forward is a fixed-layout graph of libvgen_b200.so kernels.

Design (not a port of the reference's module tree):
  * activations stay fp16 channels-last [(b f), h, w, C] for the whole forward; the reference's dozens
    of '(b f) c h w <-> b c f h w' / '(b h w) f c' permute+contiguous copies (unet_t2v.py:294-296,
    util.py:1251-1280,923-926) do not exist: temporal kernels address frames by stride.
  * weights are repacked once per load into GEMM-ready fp16 [out][taps*in] matrices; q/k/v projections
    are fused into one GEMM; GEGLU value/gate rows are interleaved for the fused epilogue; the cross
    attention K/V of the (frame-invariant) context are computed once per video, not once per frame.
  * bias, timestep-embedding add, residual adds and GEGLU run in the GEMM epilogues.
Numerics follow the reference under fp16 autocast: fp16 operands, fp32 accumulation and fp32
norm/softmax statistics, fp16 rounding where the reference materialises an fp16 tensor.
"""
from __future__ import annotations

import os

import torch

from . import arch, ops
from .graph import graphed
from .params import SpecModule


def _f16(t, dev):
    return t.detach().to(device=dev, dtype=torch.float16).contiguous()


def _f32(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def _pack_conv3x3(w, dev, cin_pad=None):
    """[n, c, 3, 3] -> [n, 9*c'] with k = (ky*3+kx)*c' + ci (c' = c or the padded channel count),
    K padded with zeros to a multiple of 64 for the tap-GEMM."""
    n, c = w.shape[0], w.shape[1]
    cp = cin_pad or c
    wp = torch.zeros(n, 3, 3, cp, dtype=torch.float32)
    wp[..., :c] = w.detach().float().cpu().permute(0, 2, 3, 1)
    wp = wp.reshape(n, 9 * cp)
    kpad = ((9 * cp + 63) // 64) * 64
    if kpad != 9 * cp:
        wp = torch.cat([wp, torch.zeros(n, kpad - 9 * cp)], dim=1)
    return wp.to(device=dev, dtype=torch.float16).contiguous()


def _geglu_bn(n):
    for bn in (256, 192, 128, 64):
        if n % bn == 0:
            return bn
    raise ValueError(f"GEGLU width {n} is not a multiple of 64")


class _UNetBase(SpecModule):
    KIND = "t2v"
    cfg_batch = True  # samplers may evaluate the cond / uncond CFG branches as one batch-2b forward (diffusion.cfg_forward)
    WOIMG = False     # HiGen: temporal branches contribute 0 when a single frame is sampled
    SR600 = False     # SR600: (2,1)-padded downsampling, row-cropped upsampling, filtered skips
    # nn.LayerNorm folded into the projection that follows it (vgen_row_stats + vgen_epilogue.row_stats / col_sum: the normalised
    # tokens are never written).  OFF by default: it halves the LayerNorm work but the k = 320 projections that consume it pay for
    # the extra per-column terms in their epilogue; the balance has not been measured on the H100.  VGEN_LN_FOLD=1, or
    # FOLD_LN = True on a module followed by invalidate_packed(), turns it on; parity is the same (tests/test_gpu_parity.py).
    FOLD_LN = os.environ.get("VGEN_LN_FOLD", "0") == "1"
    _adapter_rows = None   # DreamVideo: (fp32 condition terms [groups, sum of hidden widths], frames per group) of the running forward

    def __init__(self, config=None, in_dim=4, dim=512, y_dim=512, context_dim=512, hist_dim=156, dim_condition=4,
                 out_dim=6, num_tokens=4, dim_mult=[1, 2, 3, 4], num_heads=None, head_dim=64, num_res_blocks=3,
                 attn_scales=[1 / 2, 1 / 4, 1 / 8], use_scale_shift_norm=True, dropout=0.1, temporal_attn_times=1,
                 temporal_attention=True, use_checkpoint=False, use_image_dataset=False, use_sim_mask=False,
                 training=True, inpainting=True, use_fps_condition=False, p_all_zero=0.1, p_all_keep=0.1, zero_y=None,
                 adapter_transformer_layers=1, concat_dim=8, context_embedding_depth=4, **kwargs):
        super().__init__()
        self.cfg = config
        if head_dim != 64:
            raise NotImplementedError("vgen_b200: head_dim must be 64 (all released VGen checkpoints)")
        if use_image_dataset:
            raise NotImplementedError("vgen_b200: use_image_dataset (training-time flag) is not supported")
        if adapter_transformer_layers != 1:
            raise NotImplementedError("vgen_b200: adapter_transformer_layers != 1 is not supported")
        # arguments that would change the reference's graph must not be swallowed silently (dropout / use_checkpoint /
        # training / inpainting / p_all_* only matter for training and are accepted as no-ops)
        if temporal_attn_times != 1:
            raise NotImplementedError("vgen_b200: temporal_attn_times != 1 (extra TemporalTransformers per block) is not "
                                      "used by any released config and is not supported")
        if use_sim_mask:
            raise NotImplementedError("vgen_b200: use_sim_mask=True (masked temporal attention) is not supported")
        self.plan = arch.unet_plan(self.KIND, in_dim=in_dim, dim=dim, y_dim=y_dim, context_dim=context_dim, out_dim=out_dim,
                                   num_tokens=num_tokens, dim_mult=tuple(dim_mult), num_heads=num_heads, head_dim=head_dim,
                                   num_res_blocks=num_res_blocks, attn_scales=tuple(attn_scales),
                                   temporal_attention=temporal_attention, use_fps_condition=use_fps_condition,
                                   concat_dim=concat_dim, context_embedding_depth=context_embedding_depth,
                                   **self._plan_kwargs(config))
        # attributes the reference exposes and engines read
        self.in_dim, self.dim, self.y_dim, self.context_dim, self.out_dim = in_dim, dim, y_dim, context_dim, out_dim
        self.embed_dim, self.num_tokens, self.head_dim = dim * 4, num_tokens, head_dim
        self.zero_y = zero_y
        self.use_fps_condition = self.plan.use_fps_condition
        self._build_params(arch.unet_spec(self.plan), arch.unet_zero_init)

    def _plan_kwargs(self, config):
        """Extra unet_plan arguments a subclass reads from `config`."""
        return {}

    # ------------------------------------------------------------------------------ weight packing
    def _pack_state_dict(self):
        """The state dict the packed weights are built from (UNetSD_LoRA: with the LoRA merged in)."""
        return {k: v for k, v in self.state_dict().items()}

    def _pack(self):
        sd = self._pack_state_dict()
        dev = self.device
        if dev.type != "cuda":
            raise ops._l.VgenError("vgen_b200 UNet forward needs the module on a CUDA device (no CPU path exists)")
        W = {}

        def lin(p, bias=True):
            w = sd[p + "weight"]
            W[p + "w"] = _f16(w.reshape(w.shape[0], -1), dev)
            if bias:
                W[p + "b"] = _f32(sd[p + "bias"], dev)

        def norm(p):
            W[p + "g"] = _f32(sd[p + "weight"], dev)
            W[p + "b"] = _f32(sd[p + "bias"], dev)

        def conv3(p, cin_pad=None):
            W[p + "w"] = _pack_conv3x3(sd[p + "weight"], dev, cin_pad)
            W[p + "b"] = _f32(sd[p + "bias"], dev)

        def tconv(p):
            w = sd[p + "weight"]  # [n, c, 3, 1, 1] -> [n, 3*c], k = kt*c + ci
            W[p + "w"] = _f16(w[:, :, :, 0, 0].permute(0, 2, 1).reshape(w.shape[0], -1), dev)
            W[p + "b"] = _f32(sd[p + "bias"], dev)

        def transformer_v2(p):
            e = p + "layers.0."
            norm(e + "0.norm."), lin(e + "0.fn.to_qkv.", bias=False), lin(e + "0.fn.to_out.0.")
            lin(e + "1.net.0.0."), lin(e + "1.net.2.")

        def fold(key, wmat, bias, nrm):
            """LayerNorm `nrm` folded into the linear `key` that consumes it (ops.fold_layer_norm)."""
            wf, cs, lb = ops.fold_layer_norm(wmat, bias, sd[nrm + "weight"], sd[nrm + "bias"])
            W[key], W[key + ".cs"], W[key + ".lb"] = _f16(wf, dev), _f32(cs, dev), _f32(lb, dev)

        def block(p, cross, cross1=False):
            a1, a2 = p + "attn1.", p + "attn2."
            ln_fold = self.FOLD_LN and not cross1
            if cross1:   # disable_self_attn=True: attn1 attends to the context as well (util.py:700-702)
                W[a1 + "q"] = _f16(sd[a1 + "to_q.weight"], dev)
                W[a1 + "kv"] = _f16(torch.cat([sd[a1 + "to_k.weight"], sd[a1 + "to_v.weight"]], 0), dev)
            else:
                W[a1 + "qkv"] = _f16(torch.cat([sd[a1 + "to_q.weight"], sd[a1 + "to_k.weight"], sd[a1 + "to_v.weight"]], 0), dev)
            lin(a1 + "to_out.0.")
            if cross:
                W[a2 + "q"] = _f16(sd[a2 + "to_q.weight"], dev)
                W[a2 + "kv"] = _f16(torch.cat([sd[a2 + "to_k.weight"], sd[a2 + "to_v.weight"]], 0), dev)
            else:
                W[a2 + "qkv"] = _f16(torch.cat([sd[a2 + "to_q.weight"], sd[a2 + "to_k.weight"], sd[a2 + "to_v.weight"]], 0), dev)
            lin(a2 + "to_out.0.")
            for nm in ("norm1.", "norm2.", "norm3."):
                norm(p + nm)
            gw, gb = sd[p + "ff.net.0.proj.weight"].detach().float(), sd[p + "ff.net.0.proj.bias"].detach().float()
            bn = _geglu_bn(gw.shape[0])
            if ln_fold:
                # norm1 -> attn1.qkv, norm2 -> attn2.q (cross) / attn2.qkv, norm3 -> GEGLU projection
                fold(a1 + "qkv", torch.cat([sd[a1 + "to_q.weight"], sd[a1 + "to_k.weight"], sd[a1 + "to_v.weight"]], 0), None, p + "norm1.")
                if cross:
                    fold(a2 + "q", sd[a2 + "to_q.weight"], None, p + "norm2.")
                else:
                    fold(a2 + "qkv", torch.cat([sd[a2 + "to_q.weight"], sd[a2 + "to_k.weight"], sd[a2 + "to_v.weight"]], 0), None, p + "norm2.")
                g3, b3 = sd[p + "norm3.weight"].detach().float(), sd[p + "norm3.bias"].detach().float()
                gb = gb + gw @ b3
                gw = gw * g3[None, :]
            wp, bp = ops.pack_geglu_weight(gw, gb, bn)
            W[p + "ff.geglu.w"], W[p + "ff.geglu.b"], W[p + "ff.geglu.bn"] = _f16(wp, dev), _f32(bp, dev), bn
            if ln_fold:
                W[p + "ff.geglu.cs"] = _f32(W[p + "ff.geglu.w"].double().sum(1), dev)
            lin(p + "ff.net.2.")

        cond_w, cond_v = [], []   # conditioned adapters: stacked down.W @ condition_linear.W / down.W @ condition_linear.b

        def adapters(q, names, positions):
            """DreamVideo adapters of the block at q (util.py:499-519,649-670).  The hidden width is padded to a multiple of 64
            (zero rows of down, zero columns of up) so every adapter GEMM takes the wgmma path.  Parallel: the sublayer's output
            projection and the up projection become one GEMM over the concatenated K [W_out | W_up] with b_out + b_up.  The
            condition term is composed here: down(x + lam (Wc c + bc)) = down(x) + lam (Wd Wc c + Wd bc)."""
            for name, mod, idx, out in arch.ADAPTER_SITES:
                if name not in names:
                    continue
                a = q + mod + "."
                wd, bd = sd[a + "down_linear.weight"].detach().double().cpu(), sd[a + "down_linear.bias"].detach().double().cpu()
                wu, bu = sd[a + "up_linear.weight"].detach().double().cpu(), sd[a + "up_linear.bias"].detach().double().cpu()
                hid, c = wd.shape
                hp = ((hid + 63) // 64) * 64
                wd_p, bd_p, wu_p = torch.zeros(hp, c, dtype=torch.float64), torch.zeros(hp, dtype=torch.float64), \
                    torch.zeros(c, hp, dtype=torch.float64)
                wd_p[:hid], bd_p[:hid], wu_p[:, :hid] = wd, bd, wu
                ad = {"pos": positions[idx], "hp": hp, "down.w": _f16(wd_p, dev), "down.b": _f32(bd_p, dev), "off": None}
                if positions[idx] == "parallel":
                    wo = sd[q + out + "weight"].detach().double().cpu()
                    W[q + out + "w"] = _f16(torch.cat([wo, wu_p], dim=1), dev)
                    W[q + out + "b"] = _f32(sd[q + out + "bias"].detach().double().cpu() + bu, dev)
                else:
                    ad["up.w"], ad["up.b"] = _f16(wu_p, dev), _f32(bu, dev)
                if a + "condition_linear.weight" in sd:
                    wc = sd[a + "condition_linear.weight"].detach().double().cpu()
                    bc = sd[a + "condition_linear.bias"].detach().double().cpu()
                    ad["off"] = sum(m.shape[0] for m in cond_w)
                    cond_w.append(torch.cat([wd @ wc, torch.zeros(hp - hid, wc.shape[1], dtype=torch.float64)]))
                    cond_v.append(torch.cat([wd @ bc, torch.zeros(hp - hid, dtype=torch.float64)]))
                W[q + mod] = ad

        def layer(L):
            p = L.prefix
            if L.kind == "conv_in":
                conv3(p, cin_pad=((L.cin + 7) // 8) * 8)
            elif L.kind == "res":
                norm(p + "in_layers.0."), conv3(p + "in_layers.2.")
                lin(p + "emb_layers.1.")
                norm(p + "out_layers.0."), conv3(p + "out_layers.3.")
                if L.cin != L.cout:
                    lin(p + "skip_connection.")
                for name, widx in (("conv1", 2), ("conv2", 3), ("conv3", 3), ("conv4", 3)):
                    q = f"{p}temopral_conv.{name}."
                    norm(q + "0."), tconv(f"{q}{widx}.")
            elif L.kind == "spatial":
                norm(p + "norm."), lin(p + "proj_in."), block(p + "transformer_blocks.0.", True), lin(p + "proj_out.")
                adapters(p + "transformer_blocks.0.", self.plan.spatial_adapters, self.plan.spatial_adapter_positions)
            elif L.kind == "temporal":
                norm(p + "norm."), lin(p + "proj_in."), block(p + "transformer_blocks.0.", False), lin(p + "proj_out.")
                adapters(p + "transformer_blocks.0.", self.plan.temporal_adapters, self.plan.temporal_adapter_positions)
            elif L.kind == "down":
                conv3(p + "op.")
            elif L.kind == "up":
                conv3(p + "conv.")

        for pre in ("time_embed.0.", "time_embed.2."):
            lin(pre)
        if self.plan.use_fps_condition:
            lin("fps_embedding.0."), lin("fps_embedding.2.")
        if self.KIND == "i2vgen":
            lin("context_embedding.0."), lin("context_embedding.2.")
            conv3("local_image_concat.0.", cin_pad=8), conv3("local_image_concat.2."), conv3("local_image_concat.4.")
            transformer_v2("local_temporal_encoder.")
            conv3("local_image_embedding.0.", cin_pad=8), conv3("local_image_embedding.3."), conv3("local_image_embedding.5.")
        if self.KIND == "videolcm":
            comps = self.plan.video_compositions
            if "image" in comps:
                lin("pre_image_condition.0."), lin("pre_image_condition.2.")
            for name, _kw, enc, after, _cin in arch.VCOMP_SPATIAL:
                if name in comps:
                    # the stem conv stays fp32 [cout][cin][3][3] (ops.cond_stem); the stride-2 convs are tap-GEMM packed
                    W[enc + "0.w"], W[enc + "0.b"] = _f32(sd[enc + "0.weight"], dev), _f32(sd[enc + "0.bias"], dev)
                    conv3(enc + "3."), conv3(enc + "5.")
                    transformer_v2(after)
        if self.KIND == "higen":
            W["context_embedding.tokens"] = _f16(sd["context_embedding.tokens"][0], dev)
            for d in range(self.plan.context_embedding_depth):
                block(f"context_embedding.context_transformer.{d}.", True, cross1=True)
            lin("context_embedding.input_mapping."), lin("context_embedding.output_mapping.")
            for pre in ("asim_embedding.", "msim_embedding."):
                lin(pre + "0."), lin(pre + "2.")
            conv3("img_embedding.", cin_pad=8)
        for blk in self.plan.input_blocks:
            for L in blk:
                layer(L)
        for L in self.plan.middle:
            layer(L)
        for blk in self.plan.output_blocks:
            for L in blk:
                layer(L)
        norm("out.0."), conv3("out.2.")
        if cond_w:
            W["adapter.cond.w"], W["adapter.cond.v"] = _f16(torch.cat(cond_w), dev), _f32(torch.cat(cond_v), dev)
        self._packed = W
        return W

    # ------------------------------------------------------------------------------ building blocks
    def _conv3x3_any(self, x, W, p, **epi):
        """3x3 stride-1 conv: TMA tap-GEMM when C % 64 == 0, otherwise im2col + GEMM."""
        n, h, w, c = x.shape
        wt = W[p + "w"]
        if c % 64 == 0 and wt.shape[1] == 9 * c:
            return ops.conv2d_3x3(x, wt, bias=W[p + "b"], **epi)
        col = ops.im2col(x, 3, 3, 1, 1, 1, h, w, wt.shape[1], act_silu=epi.pop("act_silu", False))
        out = ops.linear(col, wt, bias=W[p + "b"], residual=epi.get("residual"))
        return out.view(n, h, w, wt.shape[0])

    def _conv3x3_s2(self, x, W, p, act_silu=False, pad_h=1):
        n, h, w, c = x.shape
        ho, wo = (h + 2 * pad_h - 3) // 2 + 1, (w - 1) // 2 + 1
        wt = W[p + "w"]
        col = ops.im2col(x, 3, 3, 2, pad_h, 1, ho, wo, wt.shape[1], act_silu=act_silu)
        return ops.linear(col, wt, bias=W[p + "b"]).view(n, ho, wo, wt.shape[0])

    def _res_block(self, x, emb, L, W, b, f):
        """ResBlock._forward + TemporalConvBlock_v2 (util.py:900-927,1686-1697)."""
        p = L.prefix
        n, h, w, _ = x.shape
        # emb is [b, E] (one embedding per video) or [b*f, E] (HiGen: one per frame, unet_higen.py:440-443)
        e = ops.linear_small(emb, W[p + "emb_layers.1.w"], W[p + "emb_layers.1.b"], silu_in=True)  # [b | b*f, cout]
        g = ops.group_norm(x, W[p + "in_layers.0.g"], W[p + "in_layers.0.b"], 1e-5, True)
        hcur = ops.conv2d_3x3(g, W[p + "in_layers.2.w"], bias=W[p + "in_layers.2.b"], group_bias=e,
                              group_div=(b * f) // emb.shape[0])
        g = ops.group_norm(hcur, W[p + "out_layers.0.g"], W[p + "out_layers.0.b"], 1e-5, True)
        if L.cin != L.cout:
            skip = ops.linear(x.view(-1, L.cin), W[p + "skip_connection.w"], bias=W[p + "skip_connection.b"])
        else:
            skip = x
        hcur = ops.conv2d_3x3(g, W[p + "out_layers.3.w"], bias=W[p + "out_layers.3.b"], residual=skip.view(-1, L.cout))
        if self.WOIMG and f == 1:
            return hcur  # TemporalConvBlock_v2WoImg: identity + 0.0 * branch (unet_higen.py:80-83)
        # temporal conv: GroupNorm statistics over all frames of a video, 3-tap conv over frames
        t = hcur
        names = (("conv1", 2), ("conv2", 3), ("conv3", 3), ("conv4", 3))
        for i, (name, widx) in enumerate(names):
            q = f"{p}temopral_conv.{name}."
            g = ops.group_norm(t, W[q + "0.g"], W[q + "0.b"], 1e-5, True, n=b)
            last = i == len(names) - 1
            # all videos of the batch in one launch (the frame taps are zero-padded per video)
            t = ops.tconv3(g.view(b, f, h * w, L.cout), W[f"{q}{widx}.w"], bias=W[f"{q}{widx}.b"],
                           residual=hcur.view(b, f, h * w, L.cout) if last else None).view(hcur.shape)
        return t

    @staticmethod
    def _ln_linear(t, W, key, nrm):
        """nn.LayerNorm `nrm` followed by the bias-free projection `key` (util.py:694-704): when the pack folded the norm into
        the weights (key.cs present) only the row statistics are computed and the GEMM epilogue applies them."""
        if key + ".cs" in W:
            return ops.linear(t, W[key], bias=W[key + ".lb"], ln=(ops.row_stats(t), W[key + ".cs"]))
        return ops.linear(ops.layer_norm(t, W[nrm + "g"], W[nrm + "b"]), W[key])

    def _self_attn_qkv_spatial(self, t, W, p, nrm, n, hw, inner):
        qkv = self._ln_linear(t, W, p + "qkv", nrm)             # [M, 3*inner]
        v3 = qkv.view(n, hw, 3 * inner)
        return v3[:, :, :inner], v3[:, :, inner:2 * inner], v3[:, :, 2 * inner:]

    def _sublayer_out(self, t, W, p, mod, out, width, hw, produce):
        """t + sublayer(t) through the output projection W[p + out]; produce(buf) writes the sublayer's [M, width] input of
        that projection into the 2-D view buf (or returns a new tensor when buf is None).  With a DreamVideo adapter at
        p + mod (util.py:649-670) the parallel form is ONE GEMM [sublayer | h] . [W_out | W_up]^T + (b_out + b_up) + t, h =
        gelu(down(t) + condition term) written into the K tail of the same buffer; the serial form adds up(h(t')) + t' to
        t' = t + sublayer(t).  Without one it is the plain projection with the residual."""
        ad = W.get(p + mod)
        if ad is None:
            return ops.linear(produce(None).view(-1, width), W[p + out + "w"], bias=W[p + out + "b"], residual=t)
        if ad["pos"] == "serial":
            t = ops.linear(produce(None).view(-1, width), W[p + out + "w"], bias=W[p + out + "b"], residual=t)
            h = self._adapter_down(t, ad, hw)
            return ops.linear(h, ad["up.w"], bias=ad["up.b"], residual=t)
        buf = torch.empty(t.shape[0], width + ad["hp"], device=t.device, dtype=torch.float16)
        produce(buf[:, :width])
        self._adapter_down(t, ad, hw, out=buf[:, width:])
        return ops.linear(buf, W[p + out + "w"], bias=W[p + out + "b"], residual=t)

    def _adapter_down(self, t, ad, hw, out=None):
        """gelu(down(x + lam condition_linear(c))) of Adapter.forward (util.py:510-515) in one GEMM: the condition term is the
        fp32 row bias of this forward's adapter_condition launch (one row per video or per frame)."""
        g = None
        cond = self._adapter_rows
        if ad["off"] is not None and cond is not None:
            g = cond[0][:, ad["off"]:ad["off"] + ad["hp"]]
        return ops.linear_gelu_rowbias(t, ad["down.w"], bias=ad["down.b"], row_bias=g,
                                       rows_per_group=(cond[1] * hw if g is not None else 1), out=out)

    def _basic_block_spatial(self, t, ctx_tokens, W, p, heads, n, hw, inner, f):
        """BasicTransformerBlock on tokens t [M, inner] (M = n*hw); ctx_tokens [b, L, ctx_dim] fp16."""
        t = self._sublayer_out(t, W, p, "attn_adapter", "attn1.to_out.0.", inner, hw, lambda o: ops.attention_d64(
            *self._self_attn_qkv_spatial(t, W, p + "attn1.", p + "norm1.", n, hw, inner), heads,
            out=None if o is None else o.view(n, hw, inner)))
        q = self._ln_linear(t, W, p + "attn2.q", p + "norm2.").view(n, hw, inner)
        bctx, lctx, cdim = ctx_tokens.shape
        kv = ops.linear(ctx_tokens.view(-1, cdim), W[p + "attn2.kv"]).view(bctx, lctx, 2 * inner)
        t = self._sublayer_out(t, W, p, "cross_attn_adapter", "attn2.to_out.0.", inner, hw, lambda o: ops.attention_d64(
            q, kv[:, :, :inner], kv[:, :, inner:], heads, kv_batch_div=f, out=None if o is None else o.view(n, hw, inner)))
        return self._feed_forward(t, W, p, hw)

    def _feed_forward(self, t, W, p, hw=1):
        def geglu(out):
            if p + "ff.geglu.cs" in W:   # norm3 folded into the GEGLU projection
                return ops.linear(t, W[p + "ff.geglu.w"], bias=W[p + "ff.geglu.b"], geglu=True, bn=W[p + "ff.geglu.bn"],
                                  ln=(ops.row_stats(t), W[p + "ff.geglu.cs"]), out=out)
            xn = ops.layer_norm(t, W[p + "norm3.g"], W[p + "norm3.b"])
            return ops.linear(xn, W[p + "ff.geglu.w"], bias=W[p + "ff.geglu.b"], geglu=True, bn=W[p + "ff.geglu.bn"], out=out)
        return self._sublayer_out(t, W, p, "ff_adapter", "ff.net.2.", W[p + "ff.geglu.w"].shape[0] // 2, hw, geglu)

    def _spatial_transformer(self, x, ctx_tokens, L, W, f):
        """SpatialTransformer.forward, use_linear=True (util.py:354-373)."""
        p = L.prefix
        n, h, w, c = x.shape
        g = ops.group_norm(x, W[p + "norm.g"], W[p + "norm.b"], 1e-6, False)
        t = ops.linear(g.view(-1, c), W[p + "proj_in.w"], bias=W[p + "proj_in.b"])
        t = self._basic_block_spatial(t, ctx_tokens, W, p + "transformer_blocks.0.", L.heads, n, h * w, L.inner, f)
        out = ops.linear(t, W[p + "proj_out.w"], bias=W[p + "proj_out.b"], residual=x.view(-1, c))
        return out.view(n, h, w, c)

    def _temporal_attn(self, t, W, p, nrm, heads, b, f, hw, inner, out=None):
        qkv = self._ln_linear(t, W, p + "qkv", nrm).view(b, f, hw, 3 * inner)
        # all videos of the batch in one launch
        return ops.attention_temporal(qkv[..., :inner], qkv[..., inner:2 * inner], qkv[..., 2 * inner:], heads, 64,
                                      out=None if out is None else out.view(b, f, hw, inner))

    def _temporal_transformer(self, x, L, W, b, f):
        """TemporalTransformer.forward, only_self_att=True (util.py:1240-1286): both attentions are
        self-attention over the f frames of a pixel; GroupNorm statistics span all frames."""
        if self.WOIMG and f == 1:
            return x  # TemporalTransformerWoImg: 0.0 * branch + x_in (unet_higen.py:146-149)
        p = L.prefix
        n, h, w, c = x.shape
        hw, inner = h * w, L.inner
        g = ops.group_norm(x, W[p + "norm.g"], W[p + "norm.b"], 1e-6, False, n=b)
        t = ops.linear(g.view(-1, c), W[p + "proj_in.w"], bias=W[p + "proj_in.b"])
        q = p + "transformer_blocks.0."
        for att, nrm, mod in (("attn1.", "norm1.", "attn_adapter"), ("attn2.", "norm2.", "cross_attn_adapter")):
            t = self._sublayer_out(t, W, q, mod, att + "to_out.0.", inner, hw, lambda o, t=t, att=att, nrm=nrm: self._temporal_attn(
                t, W, q + att, q + nrm, L.heads, b, f, hw, inner, out=o))
        t = self._feed_forward(t, W, q, hw)
        out = ops.linear(t, W[p + "proj_out.w"], bias=W[p + "proj_out.b"], residual=x.view(-1, c))
        return out.view(n, h, w, c)

    def _run_layer(self, x, L, W, emb, ctx_tokens, b, f, conv_in_residual=None):
        if L.kind == "res":
            return self._res_block(x, emb, L, W, b, f)
        if L.kind == "spatial":
            return self._spatial_transformer(x, ctx_tokens, L, W, f)
        if L.kind == "temporal":
            return self._temporal_transformer(x, L, W, b, f)
        if L.kind == "down":
            # UNetSD_SR600 pads the height by 2 (unet_sr600.py:151-153)
            return self._conv3x3_s2(x, W, L.prefix + "op.", pad_h=2 if self.SR600 else 1)
        if L.kind == "up":
            if self.SR600:   # UpsampleSR600 drops the first and last upsampled row (util.py:799-801)
                up = ops.upsample_nearest2x_rows(x, 1, 2 * x.shape[1] - 2)
            else:
                up = ops.upsample_nearest2x(x)
            return ops.conv2d_3x3(up, W[L.prefix + "conv.w"], bias=W[L.prefix + "conv.b"])
        if L.kind == "conv_in":
            if conv_in_residual is not None:
                return self._conv3x3_any(x, W, L.prefix, residual=conv_in_residual)
            return self._conv3x3_any(x, W, L.prefix)
        raise ValueError(L.kind)

    def _merge_skip(self, x, skip, n):
        """torch.cat([x, xs.pop()], dim=1) of the decoder (unet_t2v.py:269); SR600 overrides it."""
        return ops.concat_channels(x, skip)

    def _trunk(self, x, emb, ctx_tokens, W, b, f, conv_in_residual=None):
        """encoder / middle / decoder with skip concatenation + head (unet_t2v.py:257-277)."""
        skips = []
        for blk in self.plan.input_blocks:
            for L in blk:
                x = self._run_layer(x, L, W, emb, ctx_tokens, b, f, conv_in_residual)
            skips.append(x)
        for L in self.plan.middle:
            x = self._run_layer(x, L, W, emb, ctx_tokens, b, f)
        for n, blk in enumerate(self.plan.output_blocks):
            x = self._merge_skip(x, skips.pop(), n)
            for L in blk:
                x = self._run_layer(x, L, W, emb, ctx_tokens, b, f)
        g = ops.group_norm(x, W["out.0.g"], W["out.0.b"], 1e-5, True)
        return ops.conv2d_3x3(g, W["out.2.w"], bias=W["out.2.b"])

    def _frame_transformer(self, x, W, p, b, f):
        """Transformer_v2 / TransformerV2(heads=2, dim=cd, dim_head=cd) over the f frames of each pixel (util.py:1396-1452,
        unet_videolcm.py:121-141) on x [(b f), h, w, cd] -> tokens [(b f h w), cd]."""
        n, h, w, cd = x.shape
        e = p + "layers.0."
        tok = x.view(-1, cd)
        xn = ops.layer_norm(tok, W[e + "0.norm.g"], W[e + "0.norm.b"])
        qkv = ops.linear_small(xn, W[e + "0.fn.to_qkv.w"]).view(b, f, h * w, 6 * cd)
        att = ops.attention_temporal(qkv[..., :2 * cd], qkv[..., 2 * cd:4 * cd], qkv[..., 4 * cd:], 2, cd)
        tok = ops.linear_small(att.view(-1, 2 * cd), W[e + "0.fn.to_out.0.w"], W[e + "0.fn.to_out.0.b"], residual=tok)
        hid = ops.linear_small(tok, W[e + "1.net.0.0.w"], W[e + "1.net.0.0.b"], gelu_out=True)
        return ops.linear_small(hid, W[e + "1.net.2.w"], W[e + "1.net.2.b"], residual=tok)

    def _context(self, parts, b):
        """torch.cat(parts, dim=1) of [b, L_i, context_dim] fp16 token blocks: one strided copy per part (rows = videos)."""
        if len(parts) == 1:
            return parts[0]
        ltot = sum(p.shape[1] for p in parts)
        ctx = torch.empty(b, ltot, self.context_dim, device=parts[0].device, dtype=torch.float16)
        off, cdim = 0, self.context_dim
        ctx_rows = ctx.view(b, ltot * cdim)
        for part in parts:
            lp = part.shape[1]
            ops.copy2d(part.reshape(b, lp * cdim), ctx_rows[:, off * cdim:(off + lp) * cdim])
            off += lp
        return ctx

    def _mlp(self, x, W, p):
        h = ops.linear_small(x, W[p + "0.w"], W[p + "0.b"])
        return ops.linear_small(h, W[p + "2.w"], W[p + "2.b"], silu_in=True)

    def _time_embedding(self, t, fps, W):
        emb = self._mlp(ops.sinusoidal_embedding(t, self.dim), W, "time_embed.")
        if self.plan.use_fps_condition and fps is not None:
            emb = ops.eltwise("add", emb, self._mlp(ops.sinusoidal_embedding(fps, self.dim), W, "fps_embedding."))
        return emb

    @staticmethod
    def _to_f16_rows(t):
        """[b, L, C] (fp32 or fp16) -> contiguous fp16 [b, L, C] through the cast kernel."""
        b, L, c = t.shape
        if t.dtype == torch.float16 and t.is_contiguous():
            return t
        return ops.cp_to_pc(t.contiguous().view(b * L, c, 1).float(), b * L, c, 1).view(b, L, c)

    def _check_x(self, x, t):
        if not x.is_cuda:
            raise ops._l.VgenError("vgen_b200 UNet: inputs must be CUDA tensors (no CPU path exists)")
        if x.dim() != 5:
            raise ValueError("x must be [b, c, f, h, w]")
        if t.numel() != x.shape[0]:
            raise ValueError("t must have one entry per batch element")


class UNetSD_T2VBase(_UNetBase):
    """Drop-in for tools/modules/unet/unet_t2v.py:19-20 (registered as MODEL 'UNetSD_T2VBase')."""
    KIND = "t2v"

    @graphed
    @torch.no_grad()
    def forward(self, x, t, y=None, fps=None, masked=None, video_mask=None, focus_present_mask=None,
                prob_focus_present=0., mask_last_frame_num=0, **kwargs):
        self._check_x(x, t)
        W = self._packed or self._pack()
        b, c, f, h, w = x.shape
        emb = self._time_embedding(t, fps, W)
        if y is None:
            if self.zero_y is None:
                raise ValueError("y is None and no zero_y was given")
            y = self.zero_y.to(x.device).repeat(b, 1, 1)[:, :1, :]
        ctx = self._to_f16_rows(y)
        xin = ops.cp_to_pc(x.contiguous(), b, c, f * h * w, c_pad=8).view(b * f, h, w, 8)
        out = self._trunk(xin, emb, ctx, W, b, f)                     # [(b f), h, w, out_dim]
        return ops.pc_to_cp(out.view(b, f * h * w, self.out_dim), b, self.out_dim, f * h * w).view(b, self.out_dim, f, h, w)


class UNetSD_I2VGen(_UNetBase):
    """Drop-in for tools/modules/unet/unet_i2vgen.py:19-20 (registered as MODEL 'UNetSD_I2VGen')."""
    KIND = "i2vgen"

    def _small_conv(self, x, W, p, stride=1, act_silu=False):
        n, h, w, c = x.shape
        if stride == 2:
            return self._conv3x3_s2(x, W, p, act_silu=act_silu)
        wt = W[p + "w"]
        col = ops.im2col(x, 3, 3, 1, 1, 1, h, w, wt.shape[1], act_silu=act_silu)
        return ops.linear(col, wt, bias=W[p + "b"]).view(n, h, w, wt.shape[0])

    def _local_concat(self, local_first, W, b, f, h, w):
        """[Concat] branch, unet_i2vgen.py:281-295.  local_first: [b, 4, 1, h, w] (first-frame latent)."""
        dev = local_first.device
        if f > 1:
            pos = (torch.arange(1, f, device=dev, dtype=torch.float32) / (f - 1)).view(1, 1, f - 1, 1, 1)
            ximg = torch.cat([local_first.float(), pos.expand(b, local_first.shape[1], f - 1, h, w)], dim=2)
        else:
            ximg = local_first.float()
        ximg = ops.cp_to_pc(ximg.contiguous(), b, ximg.shape[1], f * h * w, c_pad=8).view(b * f, h, w, 8)
        ximg = self._small_conv(ximg, W, "local_image_concat.0.")
        ximg = self._small_conv(ximg, W, "local_image_concat.2.", act_silu=True)
        ximg = self._small_conv(ximg, W, "local_image_concat.4.", act_silu=True)      # [(b f), h, w, cd]
        # TransformerV2(heads=2, dim=cd, dim_head=cd): tokens are the f frames of one pixel
        tok = self._frame_transformer(ximg, W, "local_temporal_encoder.", b, f)
        return ops.eltwise("scale", tok, s=2.0)   # "concat += _ximg" twice (:294-295), exact in fp16

    def _local_tokens(self, local_first, W, b, h, w):
        """local_image_embedding, unet_i2vgen.py:126-132,312-316 -> [b, 64, 1024] context tokens."""
        x = ops.cp_to_pc(local_first.float().contiguous(), b, local_first.shape[1], h * w, c_pad=8).view(b, h, w, 8)
        x = self._small_conv(x, W, "local_image_embedding.0.")
        x = ops.adaptive_avgpool(x, 32, 32, silu_in=True)
        x = self._small_conv(x, W, "local_image_embedding.3.", stride=2)
        x = self._small_conv(x, W, "local_image_embedding.5.", stride=2, act_silu=True)
        return x.view(b, -1, x.shape[-1])

    @graphed
    @torch.no_grad()
    def forward(self, x, t, y=None, image=None, local_image=None, masked=None, fps=None, video_mask=None,
                focus_present_mask=None, prob_focus_present=0., mask_last_frame_num=0, **kwargs):
        self._check_x(x, t)
        if local_image is None or fps is None:
            raise ValueError("UNetSD_I2VGen.forward needs local_image and fps")
        W = self._packed or self._pack()
        b, c, f, h, w = x.shape
        if local_image.ndim == 5 and local_image.size(2) > 1:
            local_image = local_image[:, :, :1]
        elif local_image.ndim != 5:
            local_image = local_image.unsqueeze(2)
        cd = self.plan.concat_dim
        concat = self._local_concat(local_image, W, b, f, h, w)                    # [(b f h w), cd]
        emb = self._time_embedding(t, fps, W)
        if y is None:
            if self.zero_y is None:
                raise ValueError("y is None and no zero_y was given")
            y = self.zero_y.to(x.device).repeat(b, 1, 1)[:, :1, :]
        y16 = self._to_f16_rows(y)
        loc = self._local_tokens(local_image[:, :, 0], W, b, h, w)               # [b, 64, 1024]
        parts = [y16, loc]
        if image is not None:
            img = self._to_f16_rows(image).view(-1, image.shape[-1])
            ce = self._mlp(img, W, "context_embedding.")
            parts.append(ce.view(b, self.num_tokens, self.context_dim))
        ctx = self._context(parts, b)
        xin = ops.cp_to_pc(x.contiguous(), b, c, f * h * w, c_pad=c + cd).view(-1, c + cd)
        ops.copy2d(concat, xin[:, c:])
        out = self._trunk(xin.view(b * f, h, w, c + cd), emb, ctx, W, b, f)
        return ops.pc_to_cp(out.view(b, f * h * w, self.out_dim), b, self.out_dim, f * h * w).view(b, self.out_dim, f, h, w)


def _cfg_get(config, key, default=None):
    """config.key for the reference's EasyDict / attribute configs and for plain dicts."""
    if config is None:
        return default
    if isinstance(config, dict):
        return config.get(key, default)
    return getattr(config, key, default)


class UNetSD_VideoLCM(_UNetBase):
    """Drop-in for tools/modules/unet/unet_videolcm.py:188-189 (MODEL 'UNetSD_VideoLCM'), text-to-video
    (configs/videolcm_t2v_infer.yaml) and VideoComposer (videolcm_vcomposer_infer.yaml) alike.

    config.video_compositions selects the condition encoders (:283-372): each spatial condition of the forward
    ([b, cin, f, H, W] in pixel space) goes through ops.cond_stem (Conv2d + SiLU + AdaptiveAvgPool2d to
    config.resolution / 2 in one kernel), two stride-2 convs and a Transformer_v2 over the frames; the encodings are summed
    in the reference's order into the concat_dim channels next to x (:598-703).  'image' adds num_tokens context tokens
    after the text tokens (pre_image_condition, :743-745).  A listed condition passed as None contributes nothing, as in
    the reference.  'histogram' (per-frame context tokens, no released config) and config.use_text_clip_vip_model raise."""
    KIND = "videolcm"

    def __init__(self, config=None, *args, **kwargs):
        comps = list(_cfg_get(config, "video_compositions", None) or ["text"])
        unknown = sorted(set(comps) - arch.VCOMP_NAMES)
        if unknown:
            raise ValueError(f"vgen_b200 {type(self).__name__}: unknown video_compositions {unknown}")
        if "histogram" in comps:
            raise NotImplementedError(f"vgen_b200 {type(self).__name__}: the 'histogram' composition (per-frame context "
                                      "tokens) is not supported")
        if _cfg_get(config, "use_text_clip_vip_model", False):
            raise NotImplementedError(f"vgen_b200 {type(self).__name__}: config.use_text_clip_vip_model is not supported")
        if "mask" in comps and not kwargs.get("inpainting", True):
            raise NotImplementedError(f"vgen_b200 {type(self).__name__}: 'mask' with inpainting=False is not supported")
        self._spatial = {kw: (enc, after, cin) for name, kw, enc, after, cin in arch.VCOMP_SPATIAL if name in comps}
        res = _cfg_get(config, "resolution", None)
        if self._spatial and (res is None or len(res) != 2):
            raise ValueError(f"vgen_b200 {type(self).__name__}: spatial compositions need config.resolution = [W, H]")
        self._comps, self._res = comps, tuple(res) if res is not None else ()
        super().__init__(config, *args, **kwargs)
        self.video_compositions = comps
        self.resolution = self._res
        self.concat_dim = self.plan.concat_dim

    def _plan_kwargs(self, config):
        return dict(video_compositions=tuple(self._comps), resolution=self._res)

    def _encode_condition(self, v, kw, W, b, f, h, w):
        """<kw>_embedding + <kw>_embedding_after (unet_videolcm.py:599-699) -> tokens [(b f h w), concat_dim] fp16."""
        enc, after, cin = self._spatial[kw]
        if v.dim() != 5 or v.shape[0] != b or v.shape[1] != cin or v.shape[2] != f:
            raise ValueError(f"condition '{kw}' must be [{b}, {cin}, {f}, H, W], got {list(v.shape)}")
        if v.dtype not in (torch.float32, torch.float16):
            v = v.float()
        res = self.plan.resolution
        s = ops.cond_stem(v.contiguous(), W[enc + "0.w"], W[enc + "0.b"], res[1] // 2, res[0] // 2)
        s = self._conv3x3_s2(s, W, enc + "3.")
        s = self._conv3x3_s2(s, W, enc + "5.", act_silu=True)                  # [(b f), h', w', cd]
        if s.shape[1:3] != (h, w):
            raise ValueError(f"condition '{kw}' encodes to {tuple(s.shape[1:3])} latent pixels, x has {(h, w)}: "
                             f"config.resolution {list(res)} does not match the latent")
        return self._frame_transformer(s, W, after, b, f)

    @graphed
    @torch.no_grad()
    def forward(self, x, t, y=None, depth=None, image=None, motion=None, local_image=None, single_sketch=None,
                masked=None, canny=None, sketch=None, histogram=None, fps=None, video_mask=None,
                focus_present_mask=None, prob_focus_present=0., mask_last_frame_num=0, **kwargs):
        self._check_x(x, t)
        name = type(self).__name__
        if histogram is not None:
            raise NotImplementedError(f"vgen_b200 {name}: the 'histogram' condition is not supported")
        conds = dict(depth=depth, local_image=local_image, motion=motion, canny=canny, sketch=sketch,
                     single_sketch=single_sketch, masked=masked)
        for kw, v in conds.items():
            if v is not None and kw not in self._spatial:
                raise ValueError(f"vgen_b200 {name}: condition '{kw}' was passed but its composition is not in "
                                 f"video_compositions {self.video_compositions}")
        if image is not None and "image" not in self.video_compositions:
            raise ValueError(f"vgen_b200 {name}: 'image' was passed but is not in video_compositions {self.video_compositions}")
        W = self._packed or self._pack()
        b, c, f, h, w = x.shape
        concat = None
        for kw in arch.VCOMP_SUM_ORDER:
            if conds[kw] is not None:
                e = self._encode_condition(conds[kw], kw, W, b, f, h, w)
                concat = e if concat is None else ops.eltwise("add", concat, e)
        emb = self._time_embedding(t, fps, W)
        if y is None:
            if self.zero_y is None:
                raise ValueError("y is None and no zero_y was given")
            y = self.zero_y.to(x.device).repeat(b, 1, 1)            # all tokens (:740), unlike T2VBase
        parts = [self._to_f16_rows(y)]
        if image is not None:                                       # pre_image_condition(image) -> num_tokens tokens (:743-745)
            img = self._to_f16_rows(image.reshape(b, -1, image.shape[-1]))
            parts.append(self._mlp(img.view(-1, img.shape[-1]), W, "pre_image_condition.").view(b, self.num_tokens, self.context_dim))
        ctx = self._context(parts, b)
        cin = self.plan.input_blocks[0][0].cin                      # in_dim + concat_dim; the concat channels are 0 without conditions
        cpad = ((cin + 7) // 8) * 8
        xin = ops.cp_to_pc(x.contiguous(), b, c, f * h * w, c_pad=cpad).view(b * f, h, w, cpad)
        if concat is not None:
            ops.copy2d(concat, xin.view(-1, cpad)[:, c:c + self.concat_dim])
        out = self._trunk(xin, emb, ctx, W, b, f)
        return ops.pc_to_cp(out.view(b, f * h * w, self.out_dim), b, self.out_dim, f * h * w).view(b, self.out_dim, f, h, w)


class UNetSD_TFT2V(UNetSD_VideoLCM):
    """Drop-in for tools/modules/unet/unet_tf2tv.py:188-189 (MODEL 'UNetSD_TFT2V'): the VideoLCM class under TF-T2V's name.
    The two differ only in the use_lcm / t_w arguments (unused upstream) and in y passing through misc_dropout
    (unet_tf2tv.py:727), which is the identity in eval() (DropPath.forward :151-153); the state_dict layout is the same."""


class UNetSD_DreamVideo(_UNetBase):
    """Drop-in for tools/modules/unet/unet_dreamvideo.py:19-20 (MODEL 'UNetSD_DreamVideo', every configs/dreamvideo UNet):
    the T2V trunk with DreamVideo's adapters (Adapter, util.py:499-519) in the transformer blocks.

      * spatial_adapter_list: identity adapters of the SpatialTransformers, without condition (util.py:385-442);
      * temporal_adapter_list: motion adapters of the TemporalTransformers, conditioned on y_image (the CLIP image embedding,
        [b, 1, C] repeated over the frames or [b, f, C]) scaled by ag_strength when temporal_adapter_condition_dim is set.

    Each adapted sublayer costs one extra launch (the down projection with GELU and the condition term, ops.linear_gelu_rowbias);
    the up projection is fused into the sublayer's output projection.  The condition terms of all adapters come from one
    launch per forward (ops.adapter_condition).  ag_strength may be a float or a [b] tensor; the CFG sampler merges the
    engine's two floats into one tensor (cfg_per_sample) so the pair runs as one batch-2b forward.  With no adapters the
    state_dict and the forward are UNetSD_T2VBase's."""
    KIND = "t2v"
    cfg_per_sample = ("ag_strength",)

    def __init__(self, config=None, *args, spatial_adapter_list=[], spatial_adapter_position_list=["", "parallel", ""],
                 spatial_adapter_hidden_dim=None, temporal_adapter_list=[],
                 temporal_adapter_position_list=["parallel", "parallel", "parallel"], temporal_adapter_condition_dim=None,
                 temporal_adapter_hidden_dim=None, **kwargs):
        name = type(self).__name__
        for kind, names, positions in (("spatial", spatial_adapter_list, spatial_adapter_position_list),
                                       ("temporal", temporal_adapter_list, temporal_adapter_position_list)):
            unknown = sorted(set(names) - arch.ADAPTER_NAMES)
            if unknown:
                raise ValueError(f"vgen_b200 {name}: unknown {kind} adapters {unknown} (known: {sorted(arch.ADAPTER_NAMES)})")
            for site, _mod, idx, _out in arch.ADAPTER_SITES:
                if site in names and (idx >= len(positions) or positions[idx] not in ("parallel", "serial")):
                    # the reference skips the whole sublayer then (util.py:649-670): a graph change, not swallowed
                    raise NotImplementedError(f"vgen_b200 {name}: {kind} adapter '{site}' at position "
                                              f"{positions[idx] if idx < len(positions) else None!r}: only 'parallel' and "
                                              "'serial' are supported")
        self._adapter_kwargs = dict(
            spatial_adapters=tuple(spatial_adapter_list), temporal_adapters=tuple(temporal_adapter_list),
            spatial_adapter_hidden=int(spatial_adapter_hidden_dim or 0), temporal_adapter_hidden=int(temporal_adapter_hidden_dim or 0),
            adapter_condition_dim=int(temporal_adapter_condition_dim or 0) if temporal_adapter_list else 0,
            spatial_adapter_positions=tuple(spatial_adapter_position_list), temporal_adapter_positions=tuple(temporal_adapter_position_list))
        super().__init__(config, *args, **kwargs)
        self.spatial_adapter_list, self.temporal_adapter_list = list(spatial_adapter_list), list(temporal_adapter_list)
        self.temporal_adapter_condition_dim = temporal_adapter_condition_dim

    def _plan_kwargs(self, config):
        return dict(self._adapter_kwargs)

    def _condition_rows(self, y_image, ag_strength, b, f):
        """Shape checks of y_image / ag_strength (before any device work).  -> (y_image as [b * fi, C], fi) or None when the
        motion adapters take no condition (no condition dim, or y_image is None: then y_image is ignored, as upstream)."""
        cdim = self.plan.adapter_condition_dim
        if not cdim or y_image is None:
            return None
        if y_image.dim() != 3 or y_image.shape[0] != b or y_image.shape[1] not in (1, f) or y_image.shape[2] != cdim:
            raise ValueError(f"y_image must be [{b}, 1, {cdim}] or [{b}, {f}, {cdim}], got {list(y_image.shape)}")
        if torch.is_tensor(ag_strength) and ag_strength.numel() not in (1, b):
            raise ValueError(f"ag_strength must be a number or have one entry per batch element ({b}), got "
                             f"{list(ag_strength.shape)}")
        return y_image, y_image.shape[1]

    @graphed
    @torch.no_grad()
    def forward(self, x, t, y=None, y_image=None, fps=None, masked=None, video_mask=None, focus_present_mask=None,
                prob_focus_present=0., mask_last_frame_num=0, ag_strength=1, **kwargs):
        self._check_x(x, t)
        b, c, f, h, w = x.shape
        cond = self._condition_rows(y_image, ag_strength, b, f)
        W = self._packed or self._pack()
        emb = self._time_embedding(t, fps, W)
        if y is None:
            if self.zero_y is None:
                raise ValueError("y is None and no zero_y was given")
            y = self.zero_y.to(x.device).repeat(b, 1, 1)[:, :1, :]
        ctx = self._to_f16_rows(y)
        rows = None
        if cond is not None and "adapter.cond.w" in W:
            yi, fi = cond
            c16 = self._to_f16_rows(yi).view(b * fi, yi.shape[-1])
            if torch.is_tensor(ag_strength):
                lam = ag_strength.to(device=x.device, dtype=torch.float32).reshape(-1).contiguous()
                g = ops.adapter_condition(c16, W["adapter.cond.w"], W["adapter.cond.v"], lam=lam,
                                          groups_per_lam=fi if lam.numel() == b else b * fi)
            else:
                g = ops.adapter_condition(c16, W["adapter.cond.w"], W["adapter.cond.v"], lam_scalar=float(ag_strength))
            rows = (g, f // fi)                                 # one row per video (fi = 1) or per frame
        xin = ops.cp_to_pc(x.contiguous(), b, c, f * h * w, c_pad=8).view(b * f, h, w, 8)
        self._adapter_rows = rows
        try:
            out = self._trunk(xin, emb, ctx, W, b, f)                 # [(b f), h, w, out_dim]
        finally:
            self._adapter_rows = None
        return ops.pc_to_cp(out.view(b, f * h * w, self.out_dim), b, self.out_dim, f * h * w).view(b, self.out_dim, f, h, w)


class UNetSD_LoRA(_UNetBase):
    """Drop-in for tools/modules/unet/unet_lora.py:1091-1409 (MODEL 'UNetSD_LoRA', every configs/instructvideo UNet): the
    T2V trunk whose attentions carry InstructVideo's LoRA pairs, q = to_q(x) + up(down(x)) and the same for k, v and out
    (:161-195).  The state_dict keeps the LoRA pairs (2 008 tensors at the released rank 4, 1 480 without LoRA), so strict
    loading and get_lora_merged_model (inference_instructvideo_entrance.py:301-353) work unchanged.

    The forward never runs the pairs: the pack folds each one into the projection it adapts, W + s * up @ down with
    s = lora_alpha / lora_rank (1 when lora_alpha is None), the merge the reference's inference performs, computed in fp64
    on the host and rounded to the masters' dtype (merged_state_dict).  The packed weights are then exactly
    UNetSD_T2VBase's for the merged dict, and the LoRA costs nothing per step.  fps is ignored and y is required, as in the
    reference (:1315-1316)."""
    KIND = "t2v"

    def __init__(self, in_dim=7, dim=512, y_dim=512, context_dim=512, out_dim=6, dim_mult=[1, 2, 3, 4], num_heads=None,
                 head_dim=64, num_res_blocks=3, attn_scales=[1 / 2, 1 / 4, 1 / 8], use_scale_shift_norm=True, dropout=0.1,
                 temporal_attn_times=1, temporal_attention=True, use_checkpoint=False, use_image_dataset=False,
                 use_fps_condition=False, use_sim_mask=False, training=True, inpainting=True, use_lora=False, lora_rank=None,
                 lora_alpha=None):
        if use_lora and (lora_rank is None or int(lora_rank) < 1):
            raise ValueError(f"vgen_b200 UNetSD_LoRA: use_lora=True needs lora_rank >= 1, got {lora_rank!r}")
        self._lora_rank = int(lora_rank) if use_lora else 0
        super().__init__(None, in_dim=in_dim, dim=dim, y_dim=y_dim, context_dim=context_dim, out_dim=out_dim,
                         dim_mult=dim_mult, num_heads=num_heads, head_dim=head_dim, num_res_blocks=num_res_blocks,
                         attn_scales=attn_scales, use_scale_shift_norm=use_scale_shift_norm, dropout=dropout,
                         temporal_attn_times=temporal_attn_times, temporal_attention=temporal_attention,
                         use_checkpoint=use_checkpoint, use_image_dataset=use_image_dataset,
                         use_fps_condition=use_fps_condition, use_sim_mask=use_sim_mask, training=training,
                         inpainting=inpainting)
        self.use_lora, self.lora_rank, self.lora_alpha = use_lora, lora_rank, lora_alpha
        # get_lora_merged_model's alpha (inference_instructvideo_entrance.py:315)
        self.lora_scale = lora_alpha / lora_rank if (lora_alpha is not None and self._lora_rank) else 1.0

    def _plan_kwargs(self, config):
        return dict(lora_rank=self._lora_rank)

    def merged_state_dict(self):
        """state_dict() with every LoRA pair folded into its projection (W + lora_scale * up @ down in fp64, rounded to W's
        dtype) and the LoRA keys dropped: the UNetSD_T2VBase / use_lora=False layout.  Without LoRA it is state_dict()."""
        sd = self.state_dict()
        if not self.plan.lora_rank:
            return dict(sd)
        targets = dict(arch.LORA_SITES)
        out = {k: v for k, v in sd.items() if "_lora." not in k}
        for k, down in sd.items():
            if not k.endswith("_lora.down_linear.weight"):
                continue
            att, mod = k[:-len(".down_linear.weight")].rsplit(".", 1)
            w, up = sd[f"{att}.{targets[mod]}"], sd[k.replace(".down_linear.", ".up_linear.")]
            delta = up.detach().double().cpu() @ down.detach().double().cpu()
            out[f"{att}.{targets[mod]}"] = (w.detach().double().cpu() + self.lora_scale * delta).to(device=w.device, dtype=w.dtype)
        return out

    def _pack_state_dict(self):
        return self.merged_state_dict()

    @graphed
    @torch.no_grad()
    def forward(self, x, t, y, fps=None, video_mask=None, focus_present_mask=None, prob_focus_present=0., mask_last_frame_num=0):
        self._check_x(x, t)
        if y is None:
            raise ValueError("UNetSD_LoRA.forward needs y (the reference has no zero_y fallback)")
        W = self._packed or self._pack()
        b, c, f, h, w = x.shape
        emb = self._time_embedding(t, None, W)                        # fps is ignored (unet_lora.py:1315)
        ctx = self._to_f16_rows(y)
        xin = ops.cp_to_pc(x.contiguous(), b, c, f * h * w, c_pad=8).view(b * f, h, w, 8)
        out = self._trunk(xin, emb, ctx, W, b, f)                     # [(b f), h, w, out_dim]
        return ops.pc_to_cp(out.view(b, f * h * w, self.out_dim), b, self.out_dim, f * h * w).view(b, self.out_dim, f, h, w)


class UNetSD_SR600(_UNetBase):
    """Drop-in for tools/modules/unet/unet_sr600.py:52-53 (MODEL 'UNetSD_SR600'): the T2V trunk with
    (2,1)-padded downsampling, row-cropped upsampling, and -- on the first two decoder blocks -- the
    backbone half scaled by 1.1 / 1.2 and the skip passed through Fourier_filter(threshold=1, 0.6 / 0.4)
    (:269-285).  The filter and the scaling are fused into the channel concat."""
    KIND = "sr600"
    SR600 = True
    _BACKBONE_SCALE = (1.1, 1.2)
    _SKIP_SCALE = (0.6, 0.4)

    def _merge_skip(self, x, skip, n):
        if n >= 2:
            return ops.concat_channels(x, skip)
        cx, cs = x.shape[-1], skip.shape[-1]
        out = torch.empty(*x.shape[:-1], cx + cs, device=x.device, dtype=torch.float16)
        o2, x2 = out.view(-1, cx + cs), x.view(-1, cx)
        half = cx // 2
        ops.scale_copy2d(x2[:, :half], o2[:, :half], self._BACKBONE_SCALE[n])
        ops.copy2d(x2[:, half:], o2[:, half:cx])
        ops.fourier_lowfreq_filter(skip, self._SKIP_SCALE[n], out=o2[:, cx:])
        return out

    @graphed
    @torch.no_grad()
    def forward(self, x, t, y, x_lr=None, fps=None, video_mask=None, focus_present_mask=None, prob_focus_present=0.,
                mask_last_frame_num=0, **kwargs):
        self._check_x(x, t)
        W = self._packed or self._pack()
        b, c, f, h, w = x.shape
        if h % 2:
            raise ValueError("UNetSD_SR600: latent height must be even (UpsampleSR600 restores 2*h'-2 rows)")
        emb = self._time_embedding(t, None, W)
        ctx = self._to_f16_rows(y)
        xin = ops.cp_to_pc(x.contiguous(), b, c, f * h * w, c_pad=8).view(b * f, h, w, 8)
        out = self._trunk(xin, emb, ctx, W, b, f)
        return ops.pc_to_cp(out.view(b, f * h * w, self.out_dim), b, self.out_dim, f * h * w).view(b, self.out_dim, f, h, w)


class UNetSD_HiGen(_UNetBase):
    """Drop-in for tools/modules/unet/unet_higen.py:175-176 (MODEL 'UNetSD_HiGen'), both stages of
    inference_higen_entrance.py (:198-203 one-frame spatial stage, :221-229 32-frame temporal stage):
      * per-frame embeddings = time + motion-similarity + appearance-similarity (:436-443,:387-399);
      * context = 16 learned tokens cross-attending to the projected text (:154-172);
      * the spatial prior enters through img_embedding right after the first conv (:544-547);
      * every temporal branch is multiplied by 0 when f == 1 (:80-83,:146-149) -- skipped here."""
    KIND = "higen"
    WOIMG = True

    def _context_tokens(self, y16, W, b):
        """TextContextCrossTransformerMultiLayer.forward (unet_higen.py:167-172) -> [b, num_tokens, context_dim]."""
        p = "context_embedding."
        E, T = self.embed_dim, self.num_tokens
        yy = ops.linear(y16.view(-1, y16.shape[-1]), W[p + "input_mapping.w"], bias=W[p + "input_mapping.b"]).view(b, -1, E)
        tok = torch.empty(b, T * E, device=y16.device, dtype=torch.float16)
        ops.copy2d(W[p + "tokens"].view(1, T * E).expand(b, T * E), tok)          # broadcast over the batch (row stride 0)
        tok = tok.view(b * T, E)
        heads = 8
        for d in range(self.plan.context_embedding_depth):
            q = f"{p}context_transformer.{d}."
            for att, nrm in (("attn1.", "norm1."), ("attn2.", "norm2.")):
                xn = ops.layer_norm(tok, W[q + nrm + "g"], W[q + nrm + "b"])
                qq = ops.linear(xn, W[q + att + "q"]).view(b, T, E)
                kv = ops.linear(yy.view(-1, E), W[q + att + "kv"]).view(b, -1, 2 * E)
                a = ops.attention_cross_small(qq, kv[:, :, :E], kv[:, :, E:], heads)
                tok = ops.linear(a.view(-1, E), W[q + att + "to_out.0.w"], bias=W[q + att + "to_out.0.b"], residual=tok)
            tok = self._feed_forward(tok, W, q)
        out = ops.linear(tok, W[p + "output_mapping.w"], bias=W[p + "output_mapping.b"])
        return out.view(b, T, self.context_dim)

    def _frame_embeddings(self, t, fps, motion_cond, appearance_cond, W, b, f):
        """[b*f, embed_dim]: time (+fps) embedding of the video repeated per frame + motion + appearance."""
        tt = t.reshape(-1).repeat_interleave(f)                   # index plumbing; the MLP is row-wise
        emb = self._time_embedding(tt, None if fps is None else fps.reshape(-1).repeat_interleave(f), W)
        if f > 1:
            if motion_cond.size(1) != f:
                me = ops.sinusoidal_embedding(motion_cond.reshape(-1), self.dim).view(b, f - 1, self.dim)
                me = ops.interp_linear_rows(me, f)
            else:
                me = ops.sinusoidal_embedding(motion_cond.reshape(-1), self.dim)
            me = self._mlp(me.view(b * f, self.dim), W, "msim_embedding.")
        else:
            me = self._mlp(ops.sinusoidal_embedding(motion_cond.reshape(-1), self.dim), W, "msim_embedding.")
        emb = ops.eltwise("add", emb, me)
        ac = self._to_f16_rows(appearance_cond.reshape(b, f, -1))
        return ops.eltwise("add", emb, self._mlp(ac.view(b * f, -1), W, "asim_embedding."))

    @graphed
    @torch.no_grad()
    def forward(self, x, t, y=None, fps=None, masked=None, video_mask=None, spat_prior=None, motion_cond=None,
                appearance_cond=None, focus_present_mask=None, prob_focus_present=0., mask_last_frame_num=0, **kwargs):
        self._check_x(x, t)
        if y is None or spat_prior is None or motion_cond is None or appearance_cond is None:
            raise ValueError("UNetSD_HiGen.forward needs y, spat_prior, motion_cond and appearance_cond")
        W = self._packed or self._pack()
        b, c, f, h, w = x.shape
        emb = self._frame_embeddings(t, fps, motion_cond, appearance_cond, W, b, f)
        ctx = self._context_tokens(self._to_f16_rows(y), W, b)
        # img_embedding(spat_prior) repeated over the frames, added to the first conv (residual epilogue)
        sp = ops.cp_to_pc(spat_prior.contiguous().float(), b, spat_prior.shape[1], h * w, c_pad=8).view(b, h, w, 8)
        img = self._conv3x3_any(sp, W, "img_embedding.").view(b, h * w, self.dim)
        img_rep = torch.empty(b, f, h * w, self.dim, device=x.device, dtype=torch.float16)
        for bi in range(b):                     # broadcast over the frames of a video (row stride 0): b launches, not b*f
            ops.copy2d(img[bi].reshape(1, -1).expand(f, -1), img_rep[bi].view(f, -1))
        xin = ops.cp_to_pc(x.contiguous(), b, c, f * h * w, c_pad=8).view(b * f, h, w, 8)
        out = self._trunk(xin, emb, ctx, W, b, f, conv_in_residual=img_rep.view(-1, self.dim))
        return ops.pc_to_cp(out.view(b, f * h * w, self.out_dim), b, self.out_dim, f * h * w).view(b, self.out_dim, f, h, w)
