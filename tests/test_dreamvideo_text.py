"""DreamVideo's textual-inversion text path and DDIM inversion, host side (no GPU): the oracle and the native manager's
substitution plan against outputs frozen from the reference's EmbeddingManager / FrozenOpenCLIPCustomEmbedder /
DiffusionDDIM (tools/make_golden_dreamvideo_text.py), its checkpoint format, the registry and the refusals."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import vgen_b200
from oracle import dreamvideo_text_oracle as dto, synth, vgen_oracle as vo
from oracle.cases import CASES, make_inputs
from oracle.make_golden_clip import TINY
from _dreamvideo_text import (CKPT, CKPT_CASE, GOLDEN, RELEASED_EMBEDDER, RELEASED_EMBEDMANAGER, REVERSE_CASE,
                              REVERSE_DIFFUSION, REVERSE_STEPS, TEXT_CASES, learned_vectors, placeholder_list,
                              tiny_clip_state_dict, use_golden_tokenizer)

VOCAB = TINY["text_cfg"]["vocab_size"]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, GOLDEN))


@pytest.fixture
def tiny_embedder(golden_dir, monkeypatch):
    """A native FrozenOpenCLIPCustomEmbedder holding the tiny CLIP (CPU: enough for the manager's host work)."""
    from vgen_b200 import clip
    use_golden_tokenizer(golden_dir, monkeypatch)
    e = clip.FrozenOpenCLIPCustomEmbedder(None, arch=TINY, layer="penultimate")
    e.model.load_state_dict(tiny_clip_state_dict(golden_dir), strict=True)
    return e


def _manager(embedder, name, case, set_vectors=True):
    from vgen_b200.embedding_manager import EmbeddingManager
    m = EmbeddingManager(embedder, placeholder_strings=list(case["placeholders"]), initializer_words=list(case["init"]),
                         per_image_tokens=case["per_image"], num_vectors_per_token=case["nv"], progressive_words=False,
                         token_dim=TINY["text_cfg"]["width"])
    if set_vectors:
        for i, s in enumerate(m.string_to_param_dict):
            m.string_to_param_dict[s] = nn.Parameter(learned_vectors(name, case)[i].clone(), requires_grad=False)
    return m


@pytest.mark.parametrize("name", sorted(TEXT_CASES))
def test_oracle_matches_reference(golden_dir, gold, name):
    case = TEXT_CASES[name]
    sd = tiny_clip_state_dict(golden_dir)
    vecs = learned_vectors(name, case)
    tokens = torch.from_numpy(gold[f"{name}_tokens"])
    # the tokens of the placeholders: the first BPE piece of each, fixed by the frozen prompts' ids
    from vgen_b200 import clip_tokenizer as ct
    tok = ct.ClipTokenizer(os.path.join(golden_dir, "clip_bpe_merges_head.txt.gz"))
    s2t = {s: tok(s)[0, 1] for s in placeholder_list(case)}
    mgr = dto.EmbeddingManagerOracle(s2t, {s: vecs[i] for i, s in enumerate(s2t)}, case["nv"])
    xt, x, ids = dto.encode_text_with_manager(sd, tokens, TINY["text_cfg"]["heads"], case["layer"], mgr)
    assert np.array_equal(ids.numpy(), gold[f"{name}_ids"])
    for got, key in ((xt, "xt"), (x, "x")):
        want = gold[f"{name}_{key}"]
        assert float(np.abs(got.numpy() - want).max()) < 1e-5 * float(np.abs(want).max())
    for i, w in enumerate(case["init"]):
        assert torch.equal(dto.EmbeddingManagerOracle.initial_vectors(sd, tok(w)[0, 1], case["nv"]),
                           torch.from_numpy(gold[f"{name}_init"][i]))


@pytest.mark.parametrize("name", sorted(TEXT_CASES))
def test_substitution_plan_matches_reference_manager(tiny_embedder, gold, name):
    """The host plan: rewritten ids (pooling) and gather ids (vocabulary row or learned row) equal to what the reference
    manager did to the ids and the embedding rows; the tokenizer reproduces the frozen input ids; the initial vectors are
    the initializer words' token-embedding rows."""
    from vgen_b200.clip_tokenizer import tokenize
    case = TEXT_CASES[name]
    m = _manager(tiny_embedder, name, case, set_vectors=False)
    assert list(m.string_to_token_dict) == placeholder_list(case)
    for i, s in enumerate(case["placeholders"][:len(case["init"])]):
        assert torch.equal(m.initial_embeddings[s], torch.from_numpy(gold[f"{name}_init"][i]))
        assert torch.equal(m.string_to_param_dict[s], m.initial_embeddings[s])
        assert not m.initial_embeddings[s].requires_grad and m.string_to_param_dict[s].requires_grad
    m = _manager(tiny_embedder, name, case)
    tokens = tokenize(case["prompts"])
    assert np.array_equal(tokens.numpy(), gold[f"{name}_tokens"])
    ids, gather, extra = m.plan(tokens, VOCAB)
    assert np.array_equal(ids.numpy(), gold[f"{name}_ids"])
    assert np.array_equal(gather.numpy(), gold[f"{name}_gather"])
    assert torch.equal(tokens, torch.from_numpy(gold[f"{name}_tokens"])), "plan() must not touch its input"
    vecs = learned_vectors(name, case)
    assert torch.equal(extra, vecs.reshape(-1, vecs.shape[-1]))
    assert int(gather.min()) >= 0 and int(gather.max()) < VOCAB + extra.shape[0]
    # forward(): the reference's in-place semantics on (ids, embeddings), through the same plan
    sd = tiny_clip_state_dict(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    toks = tokens.clone()
    emb = sd["token_embedding.weight"][toks]
    out = m(toks, emb)
    assert out is emb and torch.equal(toks, ids)
    table = torch.cat([sd["token_embedding.weight"], extra])
    assert torch.equal(emb, table[gather])


def test_reference_checkpoint_loads(tiny_embedder, golden_dir):
    """A file written by the reference's EmbeddingManager.save loads through torch's safe unpickler (nn.ParameterDict
    allowed for that call only) and merges into the existing dicts."""
    case = TEXT_CASES[CKPT_CASE]
    m = _manager(tiny_embedder, "single", TEXT_CASES["single"], set_vectors=False)
    m.string_to_param_dict["*"] = nn.Parameter(torch.zeros(1, 128))
    m.load(os.path.join(golden_dir, CKPT))
    assert list(m.string_to_token_dict) == ["*", "@"]
    vecs = learned_vectors(CKPT_CASE, case)
    for i, s in enumerate(placeholder_list(case)):
        assert torch.equal(m.string_to_param_dict[s].detach(), vecs[i])
        assert int(m.string_to_token_dict[s]) == int(_manager(tiny_embedder, CKPT_CASE, case).string_to_token_dict[s])


def test_save_load_round_trip(tiny_embedder, tmp_path):
    a = _manager(tiny_embedder, CKPT_CASE, TEXT_CASES[CKPT_CASE])
    a.save(tmp_path / "e.pt")
    b = _manager(tiny_embedder, "single", TEXT_CASES["single"], set_vectors=False)
    b.load(tmp_path / "e.pt")
    for s in a.string_to_param_dict:
        assert torch.equal(a.string_to_param_dict[s], b.string_to_param_dict[s])


def test_checkpoint_with_other_objects_is_refused(tiny_embedder, tmp_path):
    """Only nn.ParameterDict is allowed beyond tensors and containers: any other pickled object is still refused."""
    m = _manager(tiny_embedder, "single", TEXT_CASES["single"])
    torch.save({"string_to_token": {}, "string_to_param": nn.ParameterDict(), "x": nn.Linear(2, 2)}, tmp_path / "bad.pt")
    with pytest.raises(Exception, match="(?i)weights.only|unsupported|global"):
        m.load(tmp_path / "bad.pt")


def test_registry_builds_released_step2_sections(golden_dir, monkeypatch):
    """register() + EMBEDDER / EMBEDMANAGER.build of the released subject step-2 config's sections give the native
    classes (the embedder with pretrained=None here: the released weight file is not part of the suite)."""
    import sys
    from vgen_b200 import clip, registry
    from vgen_b200.embedding_manager import EmbeddingManager
    use_golden_tokenizer(golden_dir, monkeypatch)
    had_open_clip = "open_clip" in sys.modules
    vgen_b200.register(force_local=True)
    assert registry.EMBEDDER.get("FrozenOpenCLIPCustomEmbedder") is clip.FrozenOpenCLIPCustomEmbedder
    assert registry.EMBEDMANAGER.get("EmbeddingManager") is EmbeddingManager
    cfg = dict(RELEASED_EMBEDDER, pretrained=None, arch=TINY)
    e = registry.EMBEDDER.build(cfg)
    assert isinstance(e, clip.FrozenOpenCLIPCustomEmbedder) and e.layer_idx == 1 and e.vit_resolution == (224, 224)
    assert e.model.has_text and e.model.has_visual
    m = registry.EMBEDMANAGER.build(dict(RELEASED_EMBEDMANAGER, embedder=e, token_dim=TINY["text_cfg"]["width"]))
    assert isinstance(m, EmbeddingManager) and list(m.string_to_token_dict) == ["*"]
    for _, p in m.named_parameters():                # the engine's loop (inference_dreamvideo_entrance.py:148-149)
        p.requires_grad = False
    assert ("open_clip" in sys.modules) == had_open_clip, "the native text path must not import open_clip"
    assert hasattr(vgen_b200.DiffusionDDIM, "ddim_reverse_sample_loop")


def test_refusals(tiny_embedder):
    from vgen_b200 import lib
    from vgen_b200.embedding_manager import EmbeddingManager
    with pytest.raises(NotImplementedError):
        EmbeddingManager(tiny_embedder, ["*"], ["dog"], progressive_words=True, token_dim=128)
    m = _manager(tiny_embedder, "single", TEXT_CASES["single"])
    for fn in ("forward_with_text", "forward_with_text_img", "embedding_to_coarse_loss", "get_embedding_norms_squared"):
        with pytest.raises(NotImplementedError):
            getattr(m, fn)()
    with pytest.raises(TypeError, match="EmbeddingManager"):
        tiny_embedder.encode_with_transformer(torch.zeros(1, 77, dtype=torch.long), embedding_manager=object())
    # the model is on the CPU: no fallback path
    with pytest.raises(lib.VgenError):
        tiny_embedder.encode_with_transformer(torch.zeros(1, 77, dtype=torch.long), embedding_manager=m)


def test_white_image_matches_open_clip_transform(gold):
    from vgen_b200 import clip
    assert torch.equal(clip.white_image(224), torch.from_numpy(gold["white_image_224"]))


def test_reverse_coefficients_bit_exact():
    """reverse_step_coefficients against diffusion_ddim.py:265-273 evaluated like the reference (fp64 tables indexed,
    cast to fp32 by _i(), fp32 square roots)."""
    d = vgen_b200.DiffusionDDIM(**REVERSE_DIFFUSION)
    dz = vgen_b200.DiffusionDDIM(schedule="cosine", schedule_param=dict(num_timesteps=1000, cosine_s=0.008,
                                                                        zero_terminal_snr=True),
                                 mean_type="v", var_type="fixed_small")
    x = torch.zeros(1, 1)
    for diff in (d, dz):
        T = diff.num_timesteps
        for S in (4, 20, 50):
            steps = diff.ddim_reverse_steps(S)
            assert torch.equal(steps, torch.arange(0, T, T // S))
            for step in steps.tolist():
                t = torch.tensor([step])
                nxt = torch.cat([diff.alphas_cumprod, diff.alphas_cumprod.new_zeros([1])])[(t + T // S).clamp(0, T)].view(1, 1).to(x)
                want = [diff.sqrt_alphas_cumprod[t].view(1, 1).to(x), diff.sqrt_one_minus_alphas_cumprod[t].view(1, 1).to(x),
                        diff.sqrt_recip_alphas_cumprod[t].view(1, 1).to(x), diff.sqrt_recipm1_alphas_cumprod[t].view(1, 1).to(x),
                        torch.sqrt(nxt), torch.sqrt(1 - nxt)]
                got = diff.reverse_step_coefficients(step, S)
                assert got[:6] == [float(w) for w in want] and got[6] == 0.0, (step, S)
    assert d.reverse_step_coefficients(950, 20)[4:6] == [0.0, 1.0]          # t + stride == T: a_next = 0


def test_reverse_refusals():
    d = vgen_b200.DiffusionDDIM(**REVERSE_DIFFUSION)
    with pytest.raises(NotImplementedError):
        d.ddim_reverse_sample_loop(torch.zeros(1, 4, 1, 2, 2), lambda *a, **k: None, {}, clamp=1.0)
    with pytest.raises(NotImplementedError):
        d.ddim_reverse_sample(torch.zeros(1, 4, 1, 2, 2), torch.tensor([0]), lambda *a, **k: None, {}, percentile=0.9)
    for kw in (dict(mean_type="x0"), dict(var_type="learned_range")):
        dd = vgen_b200.DiffusionDDIM(**dict(REVERSE_DIFFUSION, **kw))
        with pytest.raises(NotImplementedError):
            dd.ddim_reverse_sample_loop(torch.zeros(1, 4, 1, 2, 2), lambda x, t, **k: x, {})


@pytest.mark.parametrize("steps", REVERSE_STEPS)
def test_reverse_oracle_matches_reference(golden_dir, gold, steps):
    import json
    case = CASES[REVERSE_CASE]
    spec = [(k, tuple(s)) for k, s in json.load(open(os.path.join(golden_dir, f"{REVERSE_CASE}.spec.json")))]
    sd = synth.state_dict(spec, seed=case["seed"])
    inp = make_inputs(case)
    sp = dict(REVERSE_DIFFUSION["schedule_param"])
    betas = vo.make_betas(REVERSE_DIFFUSION["schedule"], sp.pop("num_timesteps"), sp.pop("zero_terminal_snr"), **sp)
    with torch.no_grad():
        got = dto.ddim_reverse_sample_loop(inp["x"], lambda xt, t, **k: vo.unet_t2v_forward(sd, xt, t, **k),
                                          {"y": inp["y_neg"]}, betas, steps, mean_type=REVERSE_DIFFUSION["mean_type"])
    want = gold[f"reverse_{steps}"]
    assert float(np.abs(got.numpy() - want).max()) < 1e-4 * float(np.abs(want).max())
