"""TEST INFRASTRUCTURE ONLY -- CPU / plain-PyTorch restatements of DreamVideo's text path and DDIM inversion:

  * tools/modules/embedding_manager.py:27-116 (EmbeddingManager: placeholder -> learned vectors, replacement / insertion)
    and clip_embedder.py:348-358 (FrozenOpenCLIPCustomEmbedder.encode_with_transformer) on the CLIP blocks of
    oracle/clip_oracle.py;
  * diffusion_ddim.py:256-287 (DiffusionDDIM.ddim_reverse_sample / ddim_reverse_sample_loop) on the tables of
    oracle/vgen_oracle.py.

Pinned against the reference classes themselves by tools/make_golden_dreamvideo_text.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .clip_oracle import _block, _n_layers
from .vgen_oracle import ddim_tables


# ------------------------------------------------------------------ textual inversion
class EmbeddingManagerOracle:
    """Placeholder string -> (token id, learned vectors [k, W]); __call__(tokens, embedded) rewrites both in place exactly
    like EmbeddingManager.forward and returns embedded."""

    def __init__(self, string_to_token, string_to_param, num_vectors_per_token):
        self.string_to_token = dict(string_to_token)
        self.string_to_param = dict(string_to_param)
        self.max_vectors = num_vectors_per_token

    @staticmethod
    def initial_vectors(sd, token, num_vectors_per_token):
        """The initializer word's token-embedding row, repeated (embedding_manager.py:60-66)."""
        return sd["token_embedding.weight"][int(token)].unsqueeze(0).repeat(num_vectors_per_token, 1)

    def __call__(self, tokens, embedded):
        n = tokens.shape[1]
        for s, tok in self.string_to_token.items():
            vec = self.string_to_param[s].to(embedded)
            tok = int(tok)
            if self.max_vectors == 1:
                embedded[tokens == tok] = vec
                continue
            k = min(vec.shape[0], self.max_vectors)
            rows, cols = torch.where(tokens == tok)
            for c, r in sorted(zip(cols.tolist(), rows.tolist()), reverse=True):
                tokens[r] = torch.cat([tokens[r, :c], tokens.new_full((k,), tok), tokens[r, c + 1:]])[:n]
                embedded[r] = torch.cat([embedded[r, :c], vec[:k], embedded[r, c + 1:]])[:n]
        return embedded


def encode_text_with_manager(sd, tokens, heads, layer, manager):
    """clip_embedder.py:348-358: token embedding, the manager's substitution (which also rewrites the ids), + positional
    embedding, the blocks, ln_final, pooled at the rewritten ids' argmax.  -> (xt, x, rewritten ids)."""
    layer_idx = {"last": 0, "penultimate": 1}[layer]
    tokens = tokens.clone()
    x = sd["token_embedding.weight"][tokens]
    if manager is not None:
        x = manager(tokens, x)
    x = x + sd["positional_embedding"]
    n = _n_layers(sd, "transformer.resblocks.")
    for i in range(n - layer_idx):
        x = _block(x, sd, f"transformer.resblocks.{i}.", heads, True)
    x = F.layer_norm(x, (x.shape[-1],), sd["ln_final.weight"], sd["ln_final.bias"], 1e-5)
    xt = x[torch.arange(x.shape[0]), tokens.argmax(dim=-1)] @ sd["text_projection"]
    return xt, x, tokens


# ------------------------------------------------------------------ DDIM inversion
def ddim_reverse_sample_loop(x0, model, model_kwargs, betas, ddim_timesteps, mean_type="eps"):
    """diffusion_ddim.py:256-287 for guide_scale None, var_type fixed_small, clamp / percentile None: x0 / eps as in the
    forward step, then x_{t+stride} = sqrt(a_next) x0 + sqrt(1 - a_next) eps with
    a_next = cat([alphas_cumprod, 0])[clamp(t + stride, 0, T)]."""
    T = len(betas)
    tab = ddim_tables(betas)
    stride = T // ddim_timesteps
    ab_next = torch.cat([tab["alphas_cumprod"], tab["alphas_cumprod"].new_zeros([1])])
    xt = x0
    b = x0.size(0)

    def pick(table, t):
        return table.to(xt.device)[t].view(b, *([1] * (xt.ndim - 1))).to(xt)

    for step in torch.arange(0, T, stride):
        t = torch.full((b,), int(step), dtype=torch.long, device=xt.device)
        out = model(xt, t, **model_kwargs)
        if mean_type == "v":
            x0_ = pick(tab["sqrt_alphas_cumprod"], t) * xt - pick(tab["sqrt_one_minus_alphas_cumprod"], t) * out
        elif mean_type == "eps":
            x0_ = pick(tab["sqrt_recip_alphas_cumprod"], t) * xt - pick(tab["sqrt_recipm1_alphas_cumprod"], t) * out
        else:
            raise ValueError(mean_type)
        eps = (pick(tab["sqrt_recip_alphas_cumprod"], t) * xt - x0_) / pick(tab["sqrt_recipm1_alphas_cumprod"], t)
        a_next = pick(ab_next, (t + stride).clamp(0, T))
        xt = torch.sqrt(a_next) * x0_ + torch.sqrt(1 - a_next) * eps
    return xt
