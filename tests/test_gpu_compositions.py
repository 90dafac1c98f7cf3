"""VideoComposer compositions on the H100: the fused condition stem against PyTorch, forward parity of UNetSD_VideoLCM /
UNetSD_TFT2V with conditions (same gates as tests/test_gpu_parity.py and tests/test_gpu_fullsize.py), CFG batching, CUDA
graph replay and determinism."""
import gc
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vgen_b200
from oracle import synth
from vgen_b200 import ops
from vgen_b200.diffusion import cfg_forward
from _vcomp import FULL_VCOMP_CASES, VCOMP_CASES, build_product, call_kwargs, load_spec, make_inputs, oracle_call

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _stem_reference(x, w, b, oh, ow):
    bb, cin, f, H, W = x.shape
    z = x.float().permute(0, 2, 1, 3, 4).reshape(bb * f, cin, H, W)
    z = F.adaptive_avg_pool2d(F.silu(F.conv2d(z, w, b, padding=1)), (oh, ow))
    return z.permute(0, 2, 3, 1)                                    # [(b f), oh, ow, cout]


@pytest.mark.parametrize("cin,dtype,b,f,H,W,oh,ow,cout", [
    (1, torch.float32, 1, 4, 64, 96, 32, 48, 32),     # exact 2 x 2 windows
    (2, torch.float16, 2, 3, 70, 100, 32, 48, 32),    # uneven, overlapping windows
    (3, torch.float32, 4, 16, 33, 47, 16, 24, 16),    # odd H / W, b*f = 64
    (4, torch.float16, 1, 5, 256, 448, 128, 224, 32),  # the released shape
    (4, torch.float32, 2, 2, 41, 29, 9, 7, 16),       # windows of up to 6 rows / 5 columns
    (1, torch.float16, 8, 8, 17, 23, 17, 23, 32),     # 1 x 1 windows: conv + SiLU alone
])
def test_cond_stem_matches_pytorch(cin, dtype, b, f, H, W, oh, ow, cout):
    g = torch.Generator(device="cuda").manual_seed(cin * 1000 + H)
    x = torch.randn(b, cin, f, H, W, device="cuda", generator=g).to(dtype)
    w = torch.randn(cout, cin, 3, 3, device="cuda", generator=g) / 3.0
    bias = torch.randn(cout, device="cuda", generator=g) * 0.1
    got = ops.cond_stem(x, w, bias, oh, ow)
    torch.backends.cudnn.allow_tf32 = False
    ref = _stem_reference(x, w, bias, oh, ow)
    assert got.shape == (b * f, oh, ow, cout) and got.dtype == torch.float16
    assert _rel_l2(got, ref) < 1e-3
    assert float((got.float() - ref).abs().max()) < 2e-3 * float(ref.abs().max())


def test_cond_stem_refusals():
    x = torch.randn(1, 5, 2, 16, 16, device="cuda")
    w, b = torch.randn(32, 5, 3, 3, device="cuda"), torch.randn(32, device="cuda")
    with pytest.raises(vgen_b200.lib.VgenError, match="cin"):
        ops.cond_stem(x, w, b, 8, 8)
    x = torch.randn(1, 1, 2, 16, 16, device="cuda")
    with pytest.raises(vgen_b200.lib.VgenError, match="cout"):
        ops.cond_stem(x, torch.randn(12, 1, 3, 3, device="cuda"), torch.randn(12, device="cuda"), 8, 8)
    with pytest.raises(vgen_b200.lib.VgenError, match="cout"):
        ops.cond_stem(x, torch.randn(72, 1, 3, 3, device="cuda"), torch.randn(72, device="cuda"), 8, 8)


def _setup(golden_dir, name, cases=VCOMP_CASES):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    gc.collect()
    torch.cuda.empty_cache()
    case = cases[name]
    spec = load_spec(golden_dir, name, cases)
    sd = synth.state_dict(spec, seed=case["seed"])
    m = build_product(case)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    sdg = {k: v.cuda() for k, v in sd.items()}
    del sd
    inp = {k: v.cuda() for k, v in make_inputs(case).items()}
    return case, m, inp, sdg


@pytest.mark.parametrize("name", sorted(VCOMP_CASES))
def test_forward_parity(golden_dir, name):
    case, m, inp, sdg = _setup(golden_dir, name)
    with torch.no_grad():
        mine = m(inp["x"], inp["t"], **call_kwargs(case, inp))
        o32 = oracle_call(case, sdg, inp)
        with torch.autocast("cuda", dtype=torch.float16):
            o16 = oracle_call(case, sdg, inp)
    truth = torch.from_numpy(np.load(os.path.join(golden_dir, name + ".npz"))["out"]).cuda()
    assert mine.shape == truth.shape and mine.dtype == torch.float16 and torch.isfinite(mine.float()).all()
    assert _rel_l2(o32, truth) < 1e-4, "GPU fp32 oracle must reproduce the reference's CPU fp32 result"
    e_mine, e_ref16 = _rel_l2(mine, truth), _rel_l2(o16, truth)
    print(f"{name}: ours vs fp32 truth {e_mine:.3e}; reference-autocast vs truth {e_ref16:.3e}")
    assert e_mine < 5e-3
    assert e_mine < 1.25 * e_ref16 + 2e-4


def test_conditions_change_the_output_and_none_contributes_nothing(golden_dir):
    case, m, inp, _ = _setup(golden_dir, "vcomp_tft2v_tiny_b2")
    kw = call_kwargs(case, inp)
    with torch.no_grad():
        full = m(inp["x"], inp["t"], **kw)
        no_depth = m(inp["x"], inp["t"], **dict(kw, depth=None))
        none = m(inp["x"], inp["t"], y=kw["y"], depth=None, motion=None, image=None)
        bare = m(inp["x"], inp["t"], y=kw["y"])
    assert not torch.equal(full, no_depth)
    assert torch.equal(none, bare)


def test_cfg_batch_equals_two_forwards(golden_dir):
    """The vcomposer engines' CFG pair: same spatial conditions, zeros_like(image) as the uncond image
    (inference_tft2v_vcomposer_entrance.py:457-480), evaluated as one batch-2b forward."""
    case, m, inp, _ = _setup(golden_dir, "vcomp_lcm_tiny")
    kc = call_kwargs(case, inp)
    ku = dict(kc, y=inp["y_neg"], image=torch.zeros_like(inp["image"]))
    with torch.no_grad():
        yc, yu = cfg_forward(m, inp["x"], inp["t"], [kc, ku])
        ac = m(inp["x"], inp["t"], **kc)
        au = m(inp["x"], inp["t"], **ku)
    assert _rel_l2(yc, ac) < 1e-3 and _rel_l2(yu, au) < 1e-3
    assert not torch.equal(yc, yu)


def test_cuda_graph_replay_equals_eager(golden_dir):
    from vgen_b200 import graph
    case, m, inp, _ = _setup(golden_dir, "vcomp_tft2v_tiny_b2")
    kw = call_kwargs(case, inp)
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        ref = eager(m, inp["x"], inp["t"], **kw)
        outs = [m(inp["x"], inp["t"], **kw) for _ in range(3)]          # eager, capture, replay
        assert graph.stats(m).get("forward", (0, 0))[0] == 1
        for o in outs:
            assert torch.equal(o, ref)
        # new condition tensors are copied into the graph's static inputs
        kw2 = dict(kw, depth=kw["depth"].flip(-1).contiguous(), motion=kw["motion"] * 0.5)
        ref2 = eager(m, inp["x"], inp["t"], **kw2)
        got2 = m(inp["x"], inp["t"], **kw2)
        assert graph.stats(m)["forward"][1] >= 2
    assert torch.equal(got2, ref2) and not torch.equal(got2, ref)


def test_forward_is_deterministic(golden_dir):
    case, m, inp, _ = _setup(golden_dir, "vcomp_lcm_tiny")
    kw = call_kwargs(case, inp)
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        a = eager(m, inp["x"], inp["t"], **kw)
        b = eager(m, inp["x"], inp["t"], **kw)
    assert torch.equal(a, b)


def test_fullsize_vcomposer_forward(golden_dir):
    """configs/tft2v_vcomposer_infer.yaml at 16 x 256 x 448 with six spatial conditions and the image tokens; truth = the
    oracle in fp32 on this GPU, yardstick = the oracle under autocast (tests/test_gpu_fullsize.py's gate)."""
    case, m, inp, sdg = _setup(golden_dir, "full_vcomposer", FULL_VCOMP_CASES)
    kw = call_kwargs(case, inp)
    with torch.no_grad():
        mine = m(inp["x"], inp["t"], **kw)
        truth = oracle_call(case, sdg, inp)
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = oracle_call(case, sdg, inp)
    assert mine.shape == truth.shape and torch.isfinite(mine.float()).all()
    ours, yard = _rel_l2(mine, truth), _rel_l2(ref16, truth)
    mx = float((mine.float() - truth).abs().max() / truth.abs().max())
    print(f"[fullsize] full_vcomposer: ours rel_l2 {ours:.3e} max {mx:.3e}; reference-autocast rel_l2 {yard:.3e}")
    assert ours < 6e-3
    assert ours < 1.25 * yard + 2e-4
    assert mx < 4 * 6e-3
