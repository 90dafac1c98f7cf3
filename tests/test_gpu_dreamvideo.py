"""DreamVideo on the H100: the adapter down projection against PyTorch on both tap-GEMM implementations, the condition
kernel, forward parity of UNetSD_DreamVideo (same gates as tests/test_gpu_parity.py and tests/test_gpu_fullsize.py), the
base flavour against UNetSD_T2VBase, the condition and its strength, CFG batching, CUDA graph replay and determinism."""
import gc
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vgen_b200
from oracle import synth
from vgen_b200 import graph, ops
from vgen_b200.diffusion import cfg_forward
from _dreamvideo import DV_CASES, FULL_DV_CASES, build_product, call_kwargs, load_spec, make_inputs, oracle_call

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("m,k,n,rpg,with_g", [
    (1000, 320, 192, 100, True),     # hidden 160 padded to 192, M not a multiple of 128
    (777, 512, 256, 7, True),
    (1536, 640, 320, 1536, True),    # one group
    (2100, 1280, 640, 30, False),
    (300, 320, 192, 1, True),        # a bias row per token
    (130, 128, 64, 13, False),
])
def test_linear_gelu_rowbias_matches_pytorch(impl, m, k, n, rpg, with_g):
    gen = torch.Generator(device="cuda").manual_seed(m + n)
    width = k + 64                                      # a is a column slice of a wider buffer, so is out
    abuf = torch.randn(m, width, device="cuda", generator=gen).half()
    a = abuf[:, 64:]
    w = (torch.randn(n, k, device="cuda", generator=gen) / k ** 0.5).half()
    bias = torch.randn(n, device="cuda", generator=gen) * 0.1
    groups = (m + rpg - 1) // rpg
    gbuf = torch.randn(groups, n + 8, device="cuda", generator=gen) * 0.5
    g = gbuf[:, 4:n + 4] if with_g else None
    obuf = torch.full((m, n + 192), 7.0, device="cuda", dtype=torch.float16)
    ops.set_tapgemm_impl(impl)
    try:
        out = ops.linear_gelu_rowbias(a, w, bias=bias, row_bias=g, rows_per_group=rpg, out=obuf[:, 192:])
    finally:
        ops.set_tapgemm_impl("auto")
    ref = a.float() @ w.float().t() + bias
    if with_g:
        ref = ref + g.repeat_interleave(rpg, dim=0)[:m]
    ref = F.gelu(ref)
    assert out.data_ptr() == obuf[:, 192:].data_ptr()
    assert torch.equal(obuf[:, :192], torch.full_like(obuf[:, :192], 7.0)), "wrote outside the output view"
    assert _rel_l2(out, ref) < 1e-3
    assert float((out.float() - ref).abs().max()) < 4e-3 * float(ref.abs().max())


@pytest.mark.parametrize("rows,groups_per_lam,per_sample", [(2, 1, True), (64, 32, True), (5, 5, False)])
def test_adapter_condition_matches_pytorch(rows, groups_per_lam, per_sample):
    gen = torch.Generator(device="cuda").manual_seed(rows)
    k, n = 1024, 1000
    c = torch.randn(rows, k, device="cuda", generator=gen).half()
    w = (torch.randn(n, k, device="cuda", generator=gen) / 32).half()
    v = torch.randn(n, device="cuda", generator=gen)
    lam = torch.rand((rows + groups_per_lam - 1) // groups_per_lam, device="cuda", generator=gen)
    g = ops.adapter_condition(c, w, v, lam=lam if per_sample else None, lam_scalar=0.3, groups_per_lam=groups_per_lam)
    scale = lam.repeat_interleave(groups_per_lam)[:rows, None] if per_sample else 0.3
    ref = scale * (c.float() @ w.float().t() + v)
    assert g.dtype == torch.float32 and _rel_l2(g, ref) < 1e-5


def _setup(golden_dir, name, cases=DV_CASES):
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


@pytest.mark.parametrize("name", sorted(DV_CASES))
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


def test_without_adapters_equals_t2vbase(golden_dir):
    case = DV_CASES["dv_motion_tiny"]
    ctor = {k: v for k, v in case["ctor"].items() if "adapter" not in k}
    spec = [(k, tuple(v.shape)) for k, v in vgen_b200.UNetSD_T2VBase(**ctor).state_dict().items()]
    sd = synth.state_dict(spec, seed=case["seed"])
    a, b = vgen_b200.UNetSD_DreamVideo(**ctor), vgen_b200.UNetSD_T2VBase(**ctor)
    a.load_state_dict(sd, strict=True), b.load_state_dict(sd, strict=True)
    a, b = a.cuda().eval(), b.cuda().eval()
    inp = {k: v.cuda() for k, v in make_inputs(case).items()}
    with torch.no_grad():
        out_a = a(inp["x"], inp["t"], y=inp["y"], y_image=inp["y_image"], ag_strength=1.0)   # no condition dim: ignored
        out_b = b(inp["x"], inp["t"], y=inp["y"])
    assert torch.equal(out_a, out_b)


def test_condition_and_strength(golden_dir):
    case, m, inp, _ = _setup(golden_dir, "dv_motion_tiny")
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        full = eager(m, inp["x"], inp["t"], y=inp["y"], y_image=inp["y_image"], ag_strength=1.0)
        other = eager(m, inp["x"], inp["t"], y=inp["y"], y_image=inp["y_image"] * -1.0, ag_strength=1.0)
        zero = eager(m, inp["x"], inp["t"], y=inp["y"], y_image=inp["y_image"], ag_strength=0.0)
        zero_t = eager(m, inp["x"], inp["t"], y=inp["y"], y_image=inp["y_image"], ag_strength=torch.zeros(1, device="cuda"))
        none = eager(m, inp["x"], inp["t"], y=inp["y"])
    assert not torch.equal(full, other)
    assert _rel_l2(zero, none) < 1e-3 and _rel_l2(zero_t, none) < 1e-3
    assert _rel_l2(full, none) > 1e-2


def test_cfg_pair_is_one_batched_forward(golden_dir, monkeypatch):
    """The engine's CFG pair (inference_dreamvideo_entrance.py:259-267): y_visual / ag 1 against zero feature / ag 0."""
    case, m, inp, _ = _setup(golden_dir, "dv_joint_tiny_b2")
    kc = {"y": inp["y"], "y_image": inp["y_image"], "ag_strength": 1}
    ku = {"y": inp["y_neg"], "y_image": torch.zeros_like(inp["y_image"]), "ag_strength": 0}
    calls = []
    fwd = type(m).forward
    monkeypatch.setattr(type(m), "forward", lambda self, x, t, **kw: calls.append(x.shape[0]) or fwd(self, x, t, **kw))
    with torch.no_grad():
        yc, yu = cfg_forward(m, inp["x"], inp["t"], [kc, ku])
        assert calls == [2 * case["b"]]
        ac = m(inp["x"], inp["t"], **kc)
        au = m(inp["x"], inp["t"], **ku)
    assert _rel_l2(yc, ac) < 1e-3 and _rel_l2(yu, au) < 1e-3
    assert not torch.equal(yc, yu)


def test_cuda_graph_replay_equals_eager(golden_dir):
    case, m, inp, _ = _setup(golden_dir, "dv_joint_tiny_b2")
    kw = call_kwargs(case, inp)                       # ag_strength is a [2] tensor here
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        ref = eager(m, inp["x"], inp["t"], **kw)
        outs = [m(inp["x"], inp["t"], **kw) for _ in range(3)]          # eager, capture, replay
        assert graph.stats(m).get("forward", (0, 0))[0] == 1
        for o in outs:
            assert torch.equal(o, ref)
        # new y_image / ag_strength values are copied into the graph's static inputs: no new capture
        kw2 = dict(kw, y_image=kw["y_image"].flip(-1).contiguous(), ag_strength=torch.tensor([0.25, 2.0], device="cuda"))
        ref2 = eager(m, inp["x"], inp["t"], **kw2)
        got2 = m(inp["x"], inp["t"], **kw2)
        assert graph.stats(m)["forward"] == (1, 3)
    assert torch.equal(got2, ref2) and not torch.equal(got2, ref)


def test_forward_is_deterministic(golden_dir):
    case, m, inp, _ = _setup(golden_dir, "dv_serial_tiny")
    kw = call_kwargs(case, inp)
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        a = eager(m, inp["x"], inp["t"], **kw)
        b = eager(m, inp["x"], inp["t"], **kw)
    assert torch.equal(a, b)


def test_fullsize_joint_forward(golden_dir):
    """The joint flavour at the released shape (32 frames, 32 x 32 latent, 77 tokens, y_image [1, 1, 1024]); truth = the
    oracle in fp32 on this GPU, yardstick = the oracle under autocast (tests/test_gpu_fullsize.py's gate)."""
    case, m, inp, sdg = _setup(golden_dir, "full_dv_joint", FULL_DV_CASES)
    kw = call_kwargs(case, inp)
    with torch.no_grad():
        mine = m(inp["x"], inp["t"], **kw)
        truth = oracle_call(case, sdg, inp)
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = oracle_call(case, sdg, inp)
    assert mine.shape == truth.shape and torch.isfinite(mine.float()).all()
    ours, yard = _rel_l2(mine, truth), _rel_l2(ref16, truth)
    mx = float((mine.float() - truth).abs().max() / truth.abs().max())
    print(f"[fullsize] full_dv_joint: ours rel_l2 {ours:.3e} max {mx:.3e}; reference-autocast rel_l2 {yard:.3e}")
    assert ours < 6e-3
    assert ours < 1.25 * yard + 2e-4
    assert mx < 4 * 6e-3
