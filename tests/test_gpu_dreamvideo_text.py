"""DreamVideo's textual-inversion text path and DDIM inversion on the H100: the token gather with learned rows, the native
FrozenOpenCLIPCustomEmbedder + EmbeddingManager against the reference's frozen outputs (tests/_dreamvideo_text.py), CUDA
graph replay with new vectors, DiffusionDDIM.ddim_reverse_sample_loop against the reference, and one subject chain
(placeholder prompt -> embedder -> UNetSD_DreamVideo with an identity adapter -> 4-step CFG DDIM) against the oracle chain."""
import gc
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import vgen_b200
from oracle import clip_oracle as co, dreamvideo_text_oracle as dto, synth, vgen_oracle as vo
from oracle.cases import CASES, make_inputs
from oracle.make_golden_clip import TINY
from _dreamvideo import DV_CASES, build_product, load_spec, make_inputs as dv_inputs
from _dreamvideo_text import (GOLDEN, REVERSE_CASE, REVERSE_DIFFUSION, REVERSE_STEPS, TEXT_CASES, learned_vectors,
                              tiny_clip_state_dict, use_golden_tokenizer)
from _helpers import build_product as build_t2v

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, GOLDEN))


def _embedder(golden_dir, layer, arch=TINY, sd=None):
    from vgen_b200 import clip
    e = clip.FrozenOpenCLIPCustomEmbedder(None, arch=arch, layer=layer)
    e.model.load_state_dict(sd if sd is not None else tiny_clip_state_dict(golden_dir), strict=True)
    e.model.cuda()
    return e


def _manager(e, name, case, vectors=None):
    from vgen_b200.embedding_manager import EmbeddingManager
    m = EmbeddingManager(e, placeholder_strings=list(case["placeholders"]), initializer_words=list(case["init"]),
                         per_image_tokens=case["per_image"], num_vectors_per_token=case["nv"], progressive_words=False,
                         token_dim=e.model.cfg["text_cfg"]["width"])
    vecs = learned_vectors(name, case) if vectors is None else vectors
    for i, s in enumerate(m.string_to_param_dict):
        m.string_to_param_dict[s] = nn.Parameter(vecs[i].clone(), requires_grad=False)
    m.cuda()                                           # the engine's .cuda() (inference_dreamvideo_entrance.py:147)
    return m


@pytest.mark.parametrize("n_extra", [1, 23 * 3])
def test_gather_with_learned_rows_bit_exact(n_extra):
    """fp16(table[id] + pos) for vocabulary ids, fp16(extra[id - vocab] + pos) for the learned ones: one fp32 add, one
    rounding, bit for bit."""
    from vgen_b200 import ops
    g = torch.Generator().manual_seed(5)
    vocab, L, W, b = 49408, 77, 1024, 3
    table = torch.randn(vocab, W, generator=g).cuda()
    extra = torch.randn(n_extra, W, generator=g).cuda()
    pos = torch.randn(L, W, generator=g).cuda()
    ids = torch.randint(0, vocab + n_extra, (b, L), generator=g)
    ids[:, 5] = vocab + n_extra - 1
    ids[:, 6] = vocab
    ids[:, 7] = vocab - 1
    ids = ids.cuda()
    out = ops.embed_tokens_extra(ids, table, extra, pos)
    want = (torch.cat([table, extra])[ids] + pos).half()
    assert torch.equal(out, want)
    # without learned rows it is the vocabulary gather
    vid = ids.clamp(max=vocab - 1)
    assert torch.equal(ops.embed_tokens_extra(vid, table, None, pos), ops.embed_tokens(vid, table, pos))


def test_gather_refuses_out_of_range_ids():
    from vgen_b200 import lib, ops
    table = torch.zeros(100, 8, device="cuda")
    extra = torch.zeros(2, 8, device="cuda")
    pos = torch.zeros(4, 8, device="cuda")
    for bad in (102, -1):
        ids = torch.tensor([[1, 2, 101, bad]], device="cuda")
        with pytest.raises(lib.VgenError, match="outside"):
            ops.embed_tokens_extra(ids, table, extra, pos)
    with pytest.raises(lib.VgenError, match="outside"):
        ops.embed_tokens_extra(torch.tensor([[1, 2, 3, 100]], device="cuda"), table, None, pos)


@pytest.mark.parametrize("name", sorted(TEXT_CASES))
def test_embedder_matches_reference(golden_dir, gold, monkeypatch, name):
    """encode_with_transformer / forward with the manager against the reference's frozen (xt, x); fp16 activations
    against the fp32 reference: relative L2 within 3e-3, as for the other CLIP embedders."""
    use_golden_tokenizer(golden_dir, monkeypatch)
    case = TEXT_CASES[name]
    e = _embedder(golden_dir, case["layer"])
    m = _manager(e, name, case)
    tokens = torch.from_numpy(gold[f"{name}_tokens"])
    xt, x = e.encode_with_transformer(tokens.clone(), embedding_manager=m)
    assert x.dtype == torch.float32 and x.shape == (len(case["prompts"]), 77, 128) and xt.shape == (len(case["prompts"]), 64)
    e_x, e_xt = _rel_l2(x, torch.from_numpy(gold[f"{name}_x"]).cuda()), _rel_l2(xt, torch.from_numpy(gold[f"{name}_xt"]).cuda())
    print(f"{name}: tokens {e_x:.3e}, pooled {e_xt:.3e}")
    assert e_x < 3e-3 and e_xt < 3e-3
    xi, xt2, x2 = e(image=e.white_image, text=case["prompts"], embedding_manager=m)
    assert torch.equal(x2, x) and torch.equal(xt2, xt) and xi.shape == (1, 64)


def test_graph_replay_and_new_embedding(golden_dir, gold, monkeypatch, tmp_path):
    """The second call with one signature replays a CUDA graph: equal to eager; the learned rows are a tensor input, so
    a replay after load() of a different embedding gives the new result, equal to its eager run."""
    from vgen_b200 import graph
    use_golden_tokenizer(golden_dir, monkeypatch)
    name, case = "two_placeholders", TEXT_CASES["two_placeholders"]
    e = _embedder(golden_dir, case["layer"])
    m = _manager(e, name, case)
    prompts = case["prompts"]
    monkeypatch.setenv("VGEN_CUDA_GRAPH", "0")
    eager = e(text=prompts, embedding_manager=m)[2]
    monkeypatch.setenv("VGEN_CUDA_GRAPH", "1")
    outs = [e(text=prompts, embedding_manager=m)[2] for _ in range(3)]
    assert graph.stats(e.model)["_text_tokens"] == (1, 2)
    for o in outs:
        assert torch.equal(o, eager)
    other = _manager(e, name, case, vectors=learned_vectors(name, case) * -2.0 + 0.01)
    other.save(tmp_path / "other.pt")
    m.load(tmp_path / "other.pt")
    replayed = e(text=prompts, embedding_manager=m)[2]
    assert graph.stats(e.model)["_text_tokens"] == (1, 3)
    monkeypatch.setenv("VGEN_CUDA_GRAPH", "0")
    eager2 = e(text=prompts, embedding_manager=m)[2]
    assert torch.equal(replayed, eager2) and not torch.equal(replayed, eager)


@pytest.mark.parametrize("steps", REVERSE_STEPS)
def test_ddim_reverse_sample_loop_matches_reference(golden_dir, gold, steps):
    """DDIM inversion of the t2v_tiny UNet (DreamVideo's Diffusion section) against the reference's frozen result; the
    same gate as the forward DDIM loop's parity (1.5e-2 relative L2).  No random numbers are drawn."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    case = CASES[REVERSE_CASE]
    spec = [(k, tuple(s)) for k, s in json.load(open(os.path.join(golden_dir, f"{REVERSE_CASE}.spec.json")))]
    unet = build_t2v(case)
    unet.load_state_dict(synth.state_dict(spec, seed=case["seed"]), strict=True)
    unet = unet.cuda().eval()
    inp = {k: v.cuda() for k, v in make_inputs(case).items()}
    diff = vgen_b200.DiffusionDDIM(**REVERSE_DIFFUSION)
    state = torch.cuda.get_rng_state()
    got = diff.ddim_reverse_sample_loop(x0=inp["x"], model=unet, model_kwargs={"y": inp["y_neg"]}, guide_scale=None,
                                        ddim_timesteps=steps)
    assert torch.equal(state, torch.cuda.get_rng_state())
    err = _rel_l2(got, torch.from_numpy(gold[f"reverse_{steps}"]).cuda())
    print(f"ddim_reverse_sample_loop {steps} steps: {err:.3e}")
    assert got.dtype == torch.float32 and err < 1.5e-2
    mu, x0 = diff.ddim_reverse_sample(inp["x"], torch.zeros(1, dtype=torch.long, device="cuda"), unet, {"y": inp["y_neg"]},
                                      ddim_timesteps=steps)
    assert mu.shape == x0.shape == inp["x"].shape and not torch.equal(mu, inp["x"])


def test_subject_chain_matches_oracle(golden_dir, monkeypatch):
    """A placeholder prompt through the native embedder (a small CLIP with 1024-wide text tokens, as the UNet's context
    expects) into UNetSD_DreamVideo with an identity adapter, through a 4-step CFG(9.0) DDIM loop on DreamVideo's
    Diffusion section; against the same chain on the fp32 oracles.  Gate: the forward DDIM loop's 1.5e-2."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    gc.collect()
    torch.cuda.empty_cache()
    use_golden_tokenizer(golden_dir, monkeypatch)
    from vgen_b200 import clip
    arch = dict(embed_dim=1024, vision_cfg=dict(image_size=28, layers=1, width=160, head_width=80, patch_size=14),
                text_cfg=dict(context_length=77, vocab_size=49408, width=1024, heads=16, layers=2))
    spec = clip.clip_spec(arch)
    csd = synth.state_dict([s for s in spec if len(s[1]) > 0], seed=51)
    for k in ("positional_embedding", "visual.positional_embedding", "visual.class_embedding", "token_embedding.weight"):
        csd[k] = synth.tensor(k, dict(spec)[k], 0.02, 51)
    csd["logit_scale"] = torch.tensor(2.6592)
    e = _embedder(golden_dir, "penultimate", arch, csd)
    case = dict(placeholders=["*"], init=["dog"], per_image=False, nv=1)
    mgr = _manager(e, "chain", case, vectors=synth.tensor("chain_vec", (1, 1, 1024), 0.05, 52))
    prompt, negative = "a * running on the road", "blurry"
    y = e(text=prompt, embedding_manager=mgr)[2]
    y_neg = e(text=negative)[2]

    dv = DV_CASES["dv_subject_tiny"]
    usd = synth.state_dict(load_spec(golden_dir, "dv_subject_tiny"), seed=dv["seed"])
    unet = build_product(dv)
    unet.load_state_dict(usd, strict=True)
    unet = unet.cuda().eval()
    noise = dv_inputs(dv)["x"].cuda()
    diff = vgen_b200.DiffusionDDIM(**REVERSE_DIFFUSION)
    mine = diff.ddim_sample_loop(noise, unet, [{"y": y}, {"y": y_neg}], guide_scale=9.0, ddim_timesteps=4, eta=0.0)

    csdg = {k: v.cuda() for k, v in csd.items()}
    from vgen_b200.clip_tokenizer import tokenize
    omgr = dto.EmbeddingManagerOracle(mgr.string_to_token_dict, {k: v.detach() for k, v in mgr.string_to_param_dict.items()}, 1)
    with torch.no_grad():
        oy = dto.encode_text_with_manager(csdg, tokenize(prompt).cuda(), 16, "penultimate", omgr)[1]
        oyn = co.encode_text(csdg, tokenize(negative).cuda(), 16, "penultimate")[1]
        assert _rel_l2(y, oy) < 3e-3 and _rel_l2(y_neg, oyn) < 3e-3
        usdg = {k: v.cuda() for k, v in usd.items()}
        fn = lambda xt, t, **k: vo.unet_dreamvideo_forward(usdg, dv["ctor"], xt, t, k["y"])  # noqa: E731
        sp = dict(REVERSE_DIFFUSION["schedule_param"])
        betas = vo.make_betas(REVERSE_DIFFUSION["schedule"], sp.pop("num_timesteps"), sp.pop("zero_terminal_snr"), **sp)
        want = vo.ddim_sample_loop(noise, fn, [{"y": oy}, {"y": oyn}], betas, 9.0, 4, mean_type="eps")
    err = _rel_l2(mine, want)
    print(f"subject chain: {err:.3e}")
    assert torch.isfinite(mine).all() and err < 1.5e-2
