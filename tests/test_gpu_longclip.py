"""Long clips on the H100: temporal attention at any frame count against fp32 SDPA, the kernel each frame count takes,
and forward parity of the long-clip cases (tests/_longclip.py) with the gates of tests/test_gpu_parity.py and
tests/test_gpu_fullsize.py, plus a CFG DDIM loop, CFG batching, CUDA-graph replay and determinism at 80 frames."""
import gc
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vgen_b200
from oracle import synth, vgen_oracle as vo
from oracle.cases import FULL_CASES, make_inputs as full_inputs
from vgen_b200 import ops
from _helpers import build_product as build_full, oracle_call as full_oracle, product_call as full_call
from _longclip import LONG_CASES, build_product, make_inputs, oracle_call, product_call, state_dict

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _rel_max(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _sdpa(q, k, v, heads):
    """fp32 SDPA on permuted copies of [b, f, npix, heads*d] views: the reference's '(b h w) f c' route."""
    b, f, npix, inner = q.shape
    d = inner // heads
    t = lambda x: x.float().permute(0, 2, 1, 3).reshape(b * npix, f, heads, d).transpose(1, 2)  # noqa: E731
    o = F.scaled_dot_product_attention(t(q), t(k), t(v))
    return o.transpose(1, 2).reshape(b, npix, f, inner).permute(0, 2, 1, 3)


def _qkv(b, f, npix, heads, d, scale=1.0, seed=0):
    """q/k/v as the column slices of one [b, f, npix, 3*inner] buffer, as unet._temporal_attn passes them."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    inner = heads * d
    qkv = (torch.randn(b, f, npix, 3 * inner, device="cuda", generator=g) * scale).half()
    return qkv[..., :inner], qkv[..., inner:2 * inner], qkv[..., 2 * inner:]


@pytest.mark.parametrize("heads", [1, 5, 8])
@pytest.mark.parametrize("L", [33, 47, 48, 63, 64, 65, 80, 96, 128, 129, 256, 1024])
def test_attention_temporal_any_length(L, heads):
    b, npix = 2, (37 if L <= 256 else 9)
    q, k, v = _qkv(b, L, npix, heads, 64, seed=L * 10 + heads)
    inner = heads * 64
    wide = torch.full((b, L, npix, inner + 64), 7.0, device="cuda", dtype=torch.float16)
    out = wide[..., 32:32 + inner]                       # a column slice of a wider buffer, 16-byte aligned
    got = ops.attention_temporal(q, k, v, heads, 64, out=out)
    ref = _sdpa(q, k, v, heads)
    assert got.data_ptr() == out.data_ptr()
    assert _rel_max(got, ref) < 3e-3
    assert bool((wide[..., :32] == 7).all()) and bool((wide[..., 32 + inner:] == 7).all()), "wrote outside the slice"
    fresh = ops.attention_temporal(q, k, v, heads, 64)   # default output buffer
    assert torch.equal(fresh, got)


def test_attention_temporal_single_video_views():
    """The [f, npix, c] form (one video) at 80 frames."""
    q, k, v = _qkv(1, 80, 50, 2, 64, seed=3)
    got = ops.attention_temporal(q[0], k[0], v[0], 2, 64)
    assert got.shape == (80, 50, 128)
    assert _rel_max(got, _sdpa(q, k, v, 2)[0]) < 3e-3


def test_attention_temporal_large_values():
    """x8 inputs: scores in the hundreds; the running max must keep every exponent finite."""
    q, k, v = _qkv(2, 129, 40, 5, 64, scale=8.0, seed=4)
    got = ops.attention_temporal(q, k, v, 5, 64)
    assert torch.isfinite(got.float()).all()
    assert _rel_max(got, _sdpa(q, k, v, 5)) < 3e-3


@pytest.mark.parametrize("L", [80, 200])
@pytest.mark.parametrize("d", [4, 8])
def test_attention_temporal_small_heads_past_64(L, d):
    """The frame transformers' 4- and 8-channel heads (heads 2) on the scalar kernel, past its former 64-frame limit."""
    q, k, v = _qkv(2, L, 30, 2, d, seed=L + d)
    got = ops.attention_temporal(q, k, v, 2, d)
    assert _rel_max(got, _sdpa(q, k, v, 2)) < 3e-3


def test_frame_count_selects_kernel():
    """Up to 32 frames the register-resident kernel runs unchanged; from 33 the flash-style kernel."""
    from torch.profiler import ProfilerActivity, profile
    args = {L: _qkv(1, L, 64, 5, 64, seed=L) for L in (16, 32, 33)}
    names = {}
    for L, (q, k, v) in args.items():
        ops.attention_temporal(q, k, v, 5, 64)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ops.attention_temporal(q, k, v, 5, 64)
            torch.cuda.synchronize()
        names[L] = [e.name for e in prof.events() if "attn" in e.name]
    assert names[16] and all("attn_temporal_kernel<16>" in n for n in names[16]), names
    assert names[32] and all("attn_temporal_kernel<32>" in n for n in names[32]), names
    assert names[33] and all("attn_temporal_flash_kernel" in n for n in names[33]), names


# ---- model level ---------------------------------------------------------------------------------------------------

def _setup(golden_dir, name):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    case = LONG_CASES[name]
    sd = state_dict(golden_dir, name)
    m = build_product(case)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    inp = {k: v.cuda() for k, v in make_inputs(case).items()}
    sdg = {k: v.cuda() for k, v in sd.items()}
    gold = np.load(os.path.join(golden_dir, f"longclip_{name}.npz"))
    return case, m, inp, sdg, gold


@pytest.mark.parametrize("name", sorted(LONG_CASES))
def test_forward_parity(golden_dir, name):
    case, m, inp, sdg, gold = _setup(golden_dir, name)
    with torch.no_grad():
        mine = product_call(case, m, inp)
        mine2 = product_call(case, m, inp)
        o32 = oracle_call(case, sdg, inp)
        with torch.autocast("cuda", dtype=torch.float16):
            o16 = oracle_call(case, sdg, inp)
    truth = torch.from_numpy(gold["out"]).cuda()
    assert mine.shape == truth.shape and mine.dtype == torch.float16 and torch.isfinite(mine.float()).all()
    assert torch.equal(mine, mine2), "forward must be deterministic"
    assert _rel_l2(o32, truth) < 1e-4, "GPU fp32 oracle must reproduce the reference's CPU fp32 result"
    e_mine, e_ref16 = _rel_l2(mine, truth), _rel_l2(o16, truth)
    print(f"{name}: ours vs fp32 truth {e_mine:.3e}; reference-autocast vs truth {e_ref16:.3e}")
    assert e_mine < 5e-3
    assert e_mine < 1.25 * e_ref16 + 2e-4


def _ddim():
    return vgen_b200.DiffusionDDIM(schedule="cosine", schedule_param=dict(num_timesteps=1000, cosine_s=0.008, zero_terminal_snr=True),
                                   mean_type="v", var_type="fixed_small")


def test_ddim_loop_parity_80_frames(golden_dir):
    case, m, inp, sdg, gold = _setup(golden_dir, "t2v_b2_f80")
    dd = case["ddim"]
    kw = [{"y": inp["y"]}, {"y": inp["y_neg"]}]
    lat = _ddim().ddim_sample_loop(inp["x"], m, kw, guide_scale=dd["guide_scale"], ddim_timesteps=dd["steps"], eta=0.0)
    fn = lambda xt, t, **k: vo.unet_t2v_forward(sdg, xt, t, **k)  # noqa: E731
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        lat16 = vo.ddim_sample_loop(inp["x"].clone(), fn, kw, vo.make_betas("cosine", 1000, True, cosine_s=0.008),
                                    dd["guide_scale"], dd["steps"], autocast_cfg=True)
    truth = torch.from_numpy(gold["ddim_latent"]).cuda()
    e_mine, e_ref16 = _rel_l2(lat, truth), _rel_l2(lat16, truth)
    print(f"t2v_b2_f80 ddim: ours {e_mine:.3e}; reference-autocast {e_ref16:.3e}")
    assert lat.dtype == torch.float32 and torch.isfinite(lat).all()
    assert e_mine < 2.5e-2 and e_mine < 1.25 * e_ref16 + 5e-4


def test_cfg_batching_matches_two_forwards(golden_dir, monkeypatch):
    case, m, inp, sdg, gold = _setup(golden_dir, "t2v_b2_f80")
    kw = [{"y": inp["y"]}, {"y": inp["y_neg"]}]
    calls = []
    orig = type(m).forward

    def spy(self, x, *a, **k):
        calls.append(x.shape[0])
        return orig(self, x, *a, **k)
    monkeypatch.setattr(type(m), "forward", spy)
    monkeypatch.setenv("VGEN_CFG_BATCH", "1")
    a = _ddim().ddim_sample_loop(inp["x"], m, kw, guide_scale=9.0, ddim_timesteps=4, eta=0.0)
    assert calls == [4] * 4
    calls.clear()
    monkeypatch.setenv("VGEN_CFG_BATCH", "0")
    b = _ddim().ddim_sample_loop(inp["x"], m, kw, guide_scale=9.0, ddim_timesteps=4, eta=0.0)
    assert calls == [2] * 8
    assert _rel_l2(a, b) < 2e-3


@pytest.mark.parametrize("name", ["t2v_b2_f80", "i2vgen_f72", "vcomp_f70"])
def test_cuda_graph_replay_matches_eager(golden_dir, name, monkeypatch):
    from vgen_b200 import graph
    case, m, inp, sdg, gold = _setup(golden_dir, name)
    monkeypatch.setenv("VGEN_CUDA_GRAPH", "0")
    eager = product_call(case, m, inp)
    monkeypatch.setenv("VGEN_CUDA_GRAPH", "1")
    outs = [product_call(case, m, inp) for _ in range(4)]   # eager (first sighting), capture + replay, replay, replay
    st = graph.stats(m)
    assert st["forward"][0] == 1 and st["forward"][1] == 3, st
    for o in outs:
        assert torch.equal(o, eager)
    inp2 = dict(inp, x=inp["x"] * 0.5 + 0.1)
    replayed = product_call(case, m, inp2)
    monkeypatch.setenv("VGEN_CUDA_GRAPH", "0")
    eager2 = product_call(case, m, inp2)
    assert torch.equal(replayed, eager2) and not torch.equal(replayed, eager)


def test_fullsize_t2v_64_frames(golden_dir):
    """The full_t2v architecture (1.4 B parameters) at 64 frames of a 32 x 32 latent against the fp32 oracle on this
    GPU, with the autocast yardstick and the gate of tests/test_gpu_fullsize.py."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    gc.collect()
    torch.cuda.empty_cache()
    case = dict(FULL_CASES["full_t2v"], f=64)
    spec = [(k, tuple(s)) for k, s in json.load(open(os.path.join(golden_dir, "full_t2v.spec.json")))]
    sd = synth.state_dict(spec, seed=case["seed"])
    m = build_full(case)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    sdg = {k: v.cuda() for k, v in sd.items()}
    del sd
    inp = {k: v.cuda() for k, v in full_inputs(case).items()}
    with torch.no_grad():
        mine = full_call(case, m, inp)
        truth = full_oracle(case, sdg, inp)
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = full_oracle(case, sdg, inp)
    assert mine.shape == truth.shape == (1, 4, 64, 32, 32) and torch.isfinite(mine.float()).all()
    e_mine, e_ref16 = _rel_l2(mine, truth), _rel_l2(ref16, truth)
    mx = float((mine.float() - truth).abs().max() / truth.abs().max())
    print(f"full_t2v f64: ours vs fp32 {e_mine:.3e} (max-abs/max-mag {mx:.3e}); reference-autocast vs fp32 {e_ref16:.3e}")
    assert e_mine < 6e-3
    assert e_mine < 1.25 * e_ref16 + 2e-4
    assert mx < 4 * 6e-3
