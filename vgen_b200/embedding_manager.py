"""DreamVideo's textual inversion (tools/modules/embedding_manager.py:27-170, registry EMBEDMANAGER): learned vectors that
stand in for a placeholder token such as `*` in "a * running on the road".

Same constructor, attributes (`string_to_token_dict`, `string_to_param_dict`, `initial_embeddings`), `save` / `load` and
`forward(tokenized_text, embedded_text)` as the reference.  The native text embedder (`clip.FrozenOpenCLIPCustomEmbedder`)
does not call `forward`: it asks for `plan(tokens, vocab)` instead, which replays the reference's substitution on the host
over the int64 ids only (at most b x 77 of them, once per prompt) and returns

  ids      the rewritten token ids (multi-vector insertion shifts the row, so the pooled end-of-text position moves),
  gather   per position, the vocabulary id or vocab + row of `extra` to embed there,
  extra    fp32 [n_extra, W]: every placeholder's vectors, in dict order,

so the embedding itself is built once, on the device, by the token-gather kernel (`ops.embed_tokens_extra`).
Training-only pieces (`progressive_words`, `forward_with_text*`, the regularisers) raise NotImplementedError.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .clip_tokenizer import tokenize

DEFAULT_PLACEHOLDER_TOKEN = ["*"]
PER_IMG_TOKEN_LIST = ["א", "ב", "ג", "ד", "ה", "ו", "ז", "ח", "ט", "י", "כ", "ל", "מ", "נ", "ס", "ע", "פ", "צ", "ק",
                      "ר", "ש", "ת"]


def get_clip_token_for_string(string):
    """The first BPE piece of `string` (embedding_manager.py:18-21): tokenize(s)[0, 1]."""
    return tokenize(string)[0, 1]


def _token_embedding_row(embedder, token):
    """Row `token` of the text tower's token embedding, as a CPU fp32 copy (the model is not moved)."""
    w = embedder.model.get_parameter("token_embedding.weight")
    return w.detach()[int(token)].to(device="cpu", dtype=torch.float32).clone()


class EmbeddingManager(nn.Module):
    def __init__(self, embedder, placeholder_strings=None, initializer_words=None, per_image_tokens=False,
                 num_vectors_per_token=1, progressive_words=False, temporal_prompt_length=1, token_dim=1024, **kwargs):
        super().__init__()
        if progressive_words:
            self._training_only("progressive_words")
        self.string_to_token_dict = {}
        self.string_to_param_dict = nn.ParameterDict()
        self.initial_embeddings = nn.ParameterDict()     # not optimised
        self.progressive_words = progressive_words
        self.progressive_counter = 0
        self.max_vectors_per_token = num_vectors_per_token
        placeholder_strings = list(DEFAULT_PLACEHOLDER_TOKEN if placeholder_strings is None else placeholder_strings)
        if per_image_tokens:
            placeholder_strings.extend(PER_IMG_TOKEN_LIST)
        for idx, s in enumerate(placeholder_strings):
            token = get_clip_token_for_string(s)
            if initializer_words and idx < len(initializer_words):
                init = _token_embedding_row(embedder, get_clip_token_for_string(initializer_words[idx]))
                params = nn.Parameter(init.unsqueeze(0).repeat(num_vectors_per_token, 1), requires_grad=True)
                self.initial_embeddings[s] = nn.Parameter(init.unsqueeze(0).repeat(num_vectors_per_token, 1),
                                                          requires_grad=False)
            else:
                params = nn.Parameter(torch.rand(size=(num_vectors_per_token, token_dim), requires_grad=True))
            self.string_to_token_dict[s] = token
            self.string_to_param_dict[s] = params

    # ---- the substitution (embedding_manager.py:76-116) on ids --------------------------------------------------
    def _substitute(self, tokens):
        """-> (ids, src, extra): the rewritten ids, and per position the source of its embedding -- a column of the
        original row (0 <= src < n) or row src - n of extra.  Replays the reference step by step: placeholders in dict
        order; one vector per token replaces every occurrence; more vectors are inserted occurrence by occurrence in
        descending column order and each row is cut back to n."""
        ids = tokens.detach().to("cpu", torch.int64).clone()
        b, n = ids.shape
        src = torch.arange(n, dtype=torch.int64).repeat(b, 1)
        base, extra = n, []
        for s, tok in self.string_to_token_dict.items():
            param = self.string_to_param_dict[s].detach().to("cpu", torch.float32)
            tok = int(tok)
            rows_here = param.shape[0]
            if self.max_vectors_per_token == 1:
                rows, cols = torch.where(ids == tok)
                if rows_here == 1:
                    src[rows, cols] = base
                elif rows_here == rows.numel():           # the reference's assignment broadcasts row i to occurrence i
                    src[rows, cols] = base + torch.arange(rows_here)
                else:
                    raise ValueError(f"EmbeddingManager: {rows_here} vectors for '{s}' cannot replace its "
                                     f"{rows.numel()} occurrences")
            else:
                k = min(rows_here, self.max_vectors_per_token)
                rows, cols = torch.where(ids == tok)
                order = torch.sort(cols, descending=True).indices
                for r, c in zip(rows[order].tolist(), cols[order].tolist()):
                    ids[r] = torch.cat([ids[r, :c], torch.full((k,), tok, dtype=torch.int64), ids[r, c + 1:]])[:n]
                    src[r] = torch.cat([src[r, :c], base + torch.arange(k), src[r, c + 1:]])[:n]
            extra.append(param)
            base += rows_here
        return ids, src, (torch.cat(extra) if extra else None)

    def plan(self, tokens, vocab):
        """tokens int64 [b, n] -> (ids, gather, extra) on the CPU (module docstring); gather < vocab + len(extra)."""
        orig = tokens.detach().to("cpu", torch.int64)
        ids, src, extra = self._substitute(orig)
        n = ids.shape[1]
        from_row = src < n
        gather = torch.where(from_row, torch.gather(orig, 1, src.clamp(max=n - 1)), vocab + src - n)
        return ids, gather, extra

    def forward(self, tokenized_text, embedded_text):
        """embedding_manager.py:76-116, in place on both arguments like the reference (API parity; the native embedder
        uses plan())."""
        ids, src, extra = self._substitute(tokenized_text)
        if extra is None:
            return embedded_text
        n = ids.shape[1]
        from_row = (src < n).to(embedded_text.device)
        srcd = src.to(embedded_text.device)
        rows = torch.gather(embedded_text, 1, srcd.clamp(max=n - 1).unsqueeze(-1).expand_as(embedded_text))
        learned = extra.to(embedded_text)[(srcd - n).clamp(min=0)]
        embedded_text.copy_(torch.where(from_row.unsqueeze(-1), rows, learned))
        tokenized_text.copy_(ids.to(tokenized_text))
        return embedded_text

    # ---- checkpoints ------------------------------------------------------------------------------------------------
    def save(self, ckpt_path):
        torch.save({"string_to_token": self.string_to_token_dict, "string_to_param": self.string_to_param_dict}, ckpt_path)

    def load(self, ckpt_path):
        """Merge a checkpoint written by save() (the reference's format: {"string_to_token": {str: 0-d tensor},
        "string_to_param": nn.ParameterDict}).  It is read with torch.load's safe (weights_only) unpickler; the one
        class beyond plain tensors and containers that the format needs, nn.ParameterDict, is allowed for this call
        only, so a file that pickles anything else is still refused."""
        with torch.serialization.safe_globals([nn.ParameterDict]):
            ckpt = torch.load(ckpt_path, map_location="cpu", weights_only=True)
        for string, token in ckpt["string_to_token"].items():
            self.string_to_token_dict[string] = token
        for string, param in ckpt["string_to_param"].items():
            self.string_to_param_dict[string] = param

    def embedding_parameters(self):
        return self.string_to_param_dict.parameters()

    # ---- training only ----------------------------------------------------------------------------------------------
    @staticmethod
    def _training_only(name):
        raise NotImplementedError(f"vgen_b200 EmbeddingManager.{name}: textual-inversion training is not supported (the "
                                  "native path only applies learned embeddings); use the reference class to train")

    def forward_with_text(self, *args, **kwargs):
        self._training_only("forward_with_text")

    def forward_with_text_img(self, *args, **kwargs):
        self._training_only("forward_with_text_img")

    def embedding_to_coarse_loss(self, *args, **kwargs):
        self._training_only("embedding_to_coarse_loss")

    def get_embedding_norms_squared(self, *args, **kwargs):
        self._training_only("get_embedding_norms_squared")
