"""Freeze the reference's DreamVideo text path and DDIM inversion into tests/golden/ (cases: tests/_dreamvideo_text.py).

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it, see oracle/refload.py):
    python tools/make_golden_dreamvideo_text.py

  * The reference's tools/modules/embedding_manager.py (EmbeddingManager) and tools/modules/clip_embedder.py
    (FrozenOpenCLIPCustomEmbedder) are imported with the vendored utils/reward/open_clip standing in for the pip
    `open_clip` package and `ftfy` stubbed (as oracle/make_golden_clip.py does).  The embedder is made without its
    constructor (which would load pretrained ViT-H/14 weights): its `.model` is the vendored CLIP of tests/golden/clip_tiny.*.
  * Per case: the input ids, the ids the manager rewrote, the gather plan the manager's embedding substitution amounts to
    (probed by running its forward on position / row codes), the initial vectors, and encode_with_transformer's (xt, x),
    checked against oracle/dreamvideo_text_oracle.py before anything is written.
  * A checkpoint written by the reference's EmbeddingManager.save, and the vendored eval transform of a white image.
  * DiffusionDDIM.ddim_reverse_sample_loop on the t2v_tiny UNet at 4 and 20 steps, checked against the same oracle module.
"""
from __future__ import annotations

import copy
import importlib
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from oracle import dreamvideo_text_oracle as dto, refload, synth, vgen_oracle as vo  # noqa: E402
from oracle.cases import CASES, make_inputs  # noqa: E402
from oracle.make_golden_clip import TINY, clip_state_dict, load_reference_open_clip  # noqa: E402
import _dreamvideo_text as dt  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _maxrel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _reference_text_modules():
    model_mod, tok_mod = load_reference_open_clip()
    oc = types.ModuleType("open_clip")                     # the vendored package under the pip package's name
    oc.tokenize = tok_mod.tokenize
    sys.modules["open_clip"] = oc
    ref = refload.load()                                   # stubs tools / tools.modules parents, utils.registry_class
    em = importlib.import_module("tools.modules.embedding_manager")
    ce = importlib.import_module("tools.modules.clip_embedder")
    tr = importlib.import_module("utils.reward.open_clip.transform")
    return model_mod, tok_mod, em, ce, tr, ref


def _reference_embedder(ce, m, layer):
    e = ce.FrozenOpenCLIPCustomEmbedder.__new__(ce.FrozenOpenCLIPCustomEmbedder)
    nn.Module.__init__(e)
    e.model, e.device, e.max_length, e.layer = m, "cpu", 77, layer
    e.layer_idx = {"last": 0, "penultimate": 1}[layer]
    return e


def _gather_probe(mgr, tokens, vocab):
    """The reference manager's substitution as gather ids: embed every position with its own id and every learned row
    with vocab + its row number, run forward, read the codes back (exact in fp32 below 2**24)."""
    probe = copy.deepcopy(mgr)
    base = vocab
    for s in probe.string_to_token_dict:
        p = probe.string_to_param_dict[s]
        probe.string_to_param_dict[s] = nn.Parameter(
            (base + torch.arange(p.shape[0], dtype=torch.float32)).unsqueeze(1).expand(-1, p.shape[1]).clone())
        base += p.shape[0]
    toks = tokens.clone()
    emb = toks.float().unsqueeze(-1).expand(-1, -1, dt.WIDTH).clone()
    out = probe(toks, emb)
    assert torch.equal(out, out[..., :1].expand_as(out))
    return out[..., 0].to(torch.int64), toks


def main():
    torch.set_grad_enabled(False)
    model_mod, tok_mod, em, ce, tr, ref = _reference_text_modules()
    m, sd, spec = clip_state_dict(model_mod, TINY, seed=31)
    assert all(torch.equal(sd[k], v) for k, v in dt.tiny_clip_state_dict(GOLD).items()), "tiny CLIP recipe drifted"
    vocab = TINY["text_cfg"]["vocab_size"]
    heads = TINY["text_cfg"]["heads"]
    out, rep = {}, {}
    for name, case in dt.TEXT_CASES.items():
        e = _reference_embedder(ce, m, case["layer"])
        torch.manual_seed(0)                                  # placeholders without an initializer draw torch.rand
        mgr = em.EmbeddingManager(embedder=e, placeholder_strings=list(case["placeholders"]),
                                  initializer_words=list(case["init"]), per_image_tokens=case["per_image"],
                                  num_vectors_per_token=case["nv"], progressive_words=False, token_dim=dt.WIDTH)
        assert list(mgr.string_to_token_dict) == dt.placeholder_list(case)
        init = torch.stack([mgr.initial_embeddings[s].detach() for s in case["placeholders"][:len(case["init"])]])
        vecs = dt.learned_vectors(name, case)
        for i, s in enumerate(mgr.string_to_param_dict):
            mgr.string_to_param_dict[s] = nn.Parameter(vecs[i].clone(), requires_grad=False)
        tokens = tok_mod.tokenize(case["prompts"])
        gather, ids_probe = _gather_probe(mgr, tokens, vocab)
        toks = tokens.clone()
        xt, x = e.encode_with_transformer(toks, embedding_manager=mgr)      # rewrites toks in place
        assert torch.equal(toks, ids_probe)
        # the oracle against the reference
        omgr = dto.EmbeddingManagerOracle(mgr.string_to_token_dict, {k: v.detach() for k, v in mgr.string_to_param_dict.items()},
                                         case["nv"])
        oxt, ox, oids = dto.encode_text_with_manager(sd, tokens, heads, case["layer"], omgr)
        assert torch.equal(oids, toks)
        for i, s in enumerate(case["placeholders"][:len(case["init"])]):
            tok = tok_mod.tokenize(case["init"][i])[0, 1]
            assert torch.equal(dto.EmbeddingManagerOracle.initial_vectors(sd, tok, case["nv"]), init[i])
        rep[name] = {"xt": _maxrel(oxt, xt), "x": _maxrel(ox, x)}
        assert rep[name]["xt"] < 1e-5 and rep[name]["x"] < 1e-5, (name, rep[name])
        out.update({f"{name}_tokens": tokens.numpy(), f"{name}_ids": toks.numpy(), f"{name}_gather": gather.numpy(),
                    f"{name}_init": init.numpy(), f"{name}_xt": xt.numpy(), f"{name}_x": x.numpy()})
        if name == dt.CKPT_CASE:
            mgr.save(os.path.join(GOLD, dt.CKPT))
    # the vendored eval transform of a white image (clip_embedder.py:323-324)
    import torchvision.transforms as T
    pre = tr.image_transform(224, is_train=False)                                       # ViT-H/14's input size
    out["white_image_224"] = pre(T.ToPILImage()(np.ones((224, 224, 3), dtype=np.uint8) * 255)).unsqueeze(0).numpy()
    # DDIM inversion on the reference
    case = CASES[dt.REVERSE_CASE]
    spec_u = [(k, tuple(s)) for k, s in json.load(open(os.path.join(GOLD, f"{dt.REVERSE_CASE}.spec.json")))]
    sdu = synth.state_dict(spec_u, seed=case["seed"])
    unet = ref.UNetSD_T2VBase(**case["ctor"]).eval()
    unet.load_state_dict(sdu, strict=True)
    inp = make_inputs(case)
    diff = ref.DiffusionDDIM(**dt.REVERSE_DIFFUSION)
    sp = dict(dt.REVERSE_DIFFUSION["schedule_param"])
    betas = vo.make_betas(dt.REVERSE_DIFFUSION["schedule"], sp.pop("num_timesteps"), sp.pop("zero_terminal_snr"), **sp)
    assert torch.equal(betas, diff.betas)
    for S in dt.REVERSE_STEPS:
        state = torch.get_rng_state()
        lat = diff.ddim_reverse_sample_loop(x0=inp["x"].clone(), model=unet, model_kwargs={"y": inp["y_neg"]},
                                            guide_scale=None, ddim_timesteps=S)
        assert torch.equal(state, torch.get_rng_state()), "the reference's inversion draws no random numbers"
        mine = dto.ddim_reverse_sample_loop(inp["x"].clone(), lambda xt, t, **k: vo.unet_t2v_forward(sdu, xt, t, **k),
                                           {"y": inp["y_neg"]}, betas, S, mean_type=dt.REVERSE_DIFFUSION["mean_type"])
        rep[f"reverse_{S}"] = _maxrel(mine, lat)
        assert rep[f"reverse_{S}"] < 1e-4, rep
        out[f"reverse_{S}"] = lat.numpy()
    np.savez_compressed(os.path.join(GOLD, dt.GOLDEN), **out)
    print("oracle vs reference (max-rel):", json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
