"""UNetSD_LoRA's runtime LoRA on the H100.

Kernels: vgen_linear_lora (the projection GEMM with the LoRA up projection as a K tail) for every N tile, with and without
bias / residual, rows not a multiple of 128, a row-strided A, tail ranks 4 to 64 over 1 to 3 sets, the block-diagonal q/k/v
tail, and the SIMT kernel with the same tail, against tests/_tapgemm_ref.py's float64 reference; vgen_lora_down against
float64.  Model: strength 1 against the oracle's unmerged forward, mixed strengths in one batch, two sets, strength 0
against the use_lora=False model, batch invariance, the CFG pair as one forward, graph replay across strength changes,
runtime against merged, and the DDIM sampler with per-branch strengths."""
import gc
import zlib

import pytest
import torch

import _tapgemm_ref as R
import vgen_b200
from oracle import vgen_oracle as vo
from vgen_b200 import graph, ops
from vgen_b200.diffusion import cfg_forward
from _instructvideo import IV_CASES, RELEASED_DIFFUSION, build_product, load_spec, lora_scale, make_inputs, unet_lora_forward, weights
from _lora_runtime import lora_pairs, oracle_multi

pytestmark = pytest.mark.gpu

ALL_BN = (32, 64, 96, 128, 160, 192, 224, 256)


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


@pytest.fixture
def forced(request):
    impl, bn = request.param
    ops.set_tapgemm_impl(impl)
    ops.set_tapgemm_bn(bn)
    yield bn
    ops.set_tapgemm_bn(0)
    ops.set_tapgemm_impl("auto")


def _down_ref(x, d, col_set, col_scale, strength, rps):
    acc = x.double() @ d.double().t()
    rows = torch.arange(x.shape[0], device=x.device) // rps
    return acc * strength.double()[rows][:, col_set.long()] * col_scale.double()[None, :]


def _tail_case(bn, m, k, n_mod, ranks, blocks, bias, residual, lda_pad, key):
    """One projection with a LoRA tail built as the model builds it: `blocks` row blocks of n_mod outputs (3 = fused q/k/v,
    block-diagonal U), sets of the given ranks, per-sample strengths over 2 samples; lora_down then linear_lora."""
    g = _gen(key)
    n = n_mod * blocks
    full = torch.randn(m, k + lda_pad, generator=g, device="cuda").half()
    a = full[:, :k]
    w = (torch.randn(n, k, generator=g, device="cuda") * k ** -0.5).half()
    rtot = blocks * sum(ranks)
    rpad = -(-rtot // 64) * 64
    d = (torch.randn(rtot, k, generator=g, device="cuda") * k ** -0.5).half()
    u = torch.zeros(n, rpad, device="cuda", dtype=torch.float16)
    cset, cscale, col = [], [], 0
    for bi in range(blocks):
        for j, r in enumerate(ranks):
            u[bi * n_mod:(bi + 1) * n_mod, col:col + r] = (torch.randn(n_mod, r, generator=g, device="cuda") * r ** -0.5).half()
            cset += [j] * r
            cscale += [2.0 / r] * r
            col += r
    col_set = torch.tensor(cset, dtype=torch.int32, device="cuda")
    col_scale = torch.tensor(cscale, dtype=torch.float32, device="cuda")
    rps = -(-m // 2)
    strength = torch.tensor([[0.5 + j for j in range(len(ranks))], [-1.0 + 0.25 * j for j in range(len(ranks))]],
                            device="cuda")
    h = ops.lora_down(a, d, col_set, col_scale, strength, rps, rpad)
    href = _down_ref(a, d, col_set, col_scale, strength, rps)
    assert bool((h[:, rtot:] == 0).all()), "the padding columns of h must be exact zeros"
    mult = (href / (a.double() @ d.double().t())).nan_to_num(0.0).abs()
    hb = R.Bounded(href, R.ACC_C * k * R.U32 * mult * (a.double().abs() @ d.double().abs().t()) + R.EPI_C * R.U32 * href.abs())
    R.check(h[:, :rtot], hb, f"lora_down {key}")
    b = torch.randn(n, generator=g, device="cuda") if bias else None
    res = torch.randn(m, n, generator=g, device="cuda").half() if residual else None
    out = ops.linear_lora(a, w, h, u, bias=b, residual=res)
    acc, S = R.gemm(a, w)
    acc2, S2 = R.gemm(h, u)
    ref = R.epilogue(acc + acc2, S + S2, k + rpad, bias=b, residual=res)
    torch.cuda.synchronize()
    return R.check(out, ref, f"linear_lora {key}")


@pytest.mark.parametrize("forced", [("auto", bn) for bn in ALL_BN] + [("simt", 0)], indirect=True,
                         ids=[f"bn{bn}" for bn in ALL_BN] + ["simt"])
def test_linear_lora_kernel(forced):
    bn = forced
    cases = [  # m, k, n_mod, ranks, blocks, bias, residual, lda_pad
        (200, 320, 320, (4,), 1, True, True, 0),          # to_out: bias + residual, m not a multiple of 128
        (257, 320, 320, (4,), 3, False, False, 64),       # fused q/k/v, block-diagonal tail, row-strided A
        (129, 640, 160, (8, 4), 3, False, False, 0),      # two sets on q/k/v: R = 36
        (131, 1024, 192, (12, 8, 4), 2, False, False, 0),  # cross-attention k/v of the context, three sets
        (64, 128, 96, (64,), 1, True, False, 8),          # the largest rank: a 64-wide tail of one set
        (300, 256, 128, (64, 64, 12), 1, False, True, 0),  # three sets, R = 140: three tail k-iterations
    ]
    worst = 0.0
    for i, c in enumerate(cases):
        worst = max(worst, _tail_case(bn, *c, key=(bn, i)))
    print(f"BN {bn}: worst error / bound {worst:.3f}")


def test_linear_lora_refusals():
    a = torch.zeros(128, 64, device="cuda", dtype=torch.float16)
    w = torch.zeros(64, 64, device="cuda", dtype=torch.float16)
    with pytest.raises(vgen_b200.lib.VgenError):   # r not a multiple of 64
        ops.linear_lora(a, w, torch.zeros(128, 32, device="cuda", dtype=torch.float16),
                        torch.zeros(64, 32, device="cuda", dtype=torch.float16))


# ------------------------------------------------------------------------------------------------------------ model
def _setup(golden_dir, name):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    gc.collect()
    torch.cuda.empty_cache()
    case = IV_CASES[name]
    sd = weights(load_spec(golden_dir, name), case["seed"])
    m = build_product(case)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    sdg = {k: v.cuda() for k, v in sd.items()}
    inp = {k: v.cuda() for k, v in make_inputs(case).items()}
    return case, m, inp, sdg


def _gates(mine, truth, ref16, what):
    e_mine, e_ref16 = _rel_l2(mine, truth), _rel_l2(ref16, truth)
    print(f"{what}: ours {e_mine:.3e}; reference-autocast {e_ref16:.3e}")
    assert torch.isfinite(mine.float()).all()
    assert e_mine < 5e-3 and e_mine < 1.25 * e_ref16 + 2e-4, what


@pytest.mark.parametrize("name", ["iv_lora_tiny", "iv_lora_alpha_tiny_b2"])
def test_strength_one_against_oracle_and_merged(golden_dir, name):
    case, m, inp, sdg = _setup(golden_dir, name)
    with torch.no_grad():
        merged = m(inp["x"], inp["t"], inp["y"])
        assert m.lora_signature is None
        mine = m(inp["x"], inp["t"], inp["y"], lora_strength=1.0)
        assert m.lora_signature == (("default", 4),)
        truth = unet_lora_forward(sdg, inp["x"], inp["t"], inp["y"], lora_scale(case["ctor"]))
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = unet_lora_forward(sdg, inp["x"], inp["t"], inp["y"], lora_scale(case["ctor"]))
        again = m(inp["x"], inp["t"], inp["y"])   # runtime mode without lora_strength: every set at 1
    _gates(mine, truth, ref16, f"{name} runtime, strength 1")
    _gates(merged, truth, ref16, f"{name} merged")
    assert _rel_l2(mine, merged) < 1e-2   # both within 5e-3 of the truth
    assert torch.equal(again, mine)


def test_added_set_on_base_model(golden_dir):
    case, m, inp, sdg = _setup(golden_dir, "iv_nolora_tiny")
    pairs = lora_pairs(case["ctor"], seed=71)
    m.add_lora("tuned", pairs, alpha=8)
    assert m.lora_names == ["tuned"]
    with torch.no_grad():
        mine = m(inp["x"], inp["t"], inp["y"])
        base = {k: v for k, v in sdg.items() if "_lora." not in k}
        sd = dict(base, **{k: v.cuda() for k, v in pairs.items()})
        truth = unet_lora_forward(sd, inp["x"], inp["t"], inp["y"], 2.0)
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = unet_lora_forward(sd, inp["x"], inp["t"], inp["y"], 2.0)
    _gates(mine, truth, ref16, "iv_nolora_tiny + add_lora, alpha 8")


def test_mixed_strengths_in_one_batch_and_batch_invariance(golden_dir):
    case, m, inp, sdg = _setup(golden_dir, "iv_lora_tiny")
    strengths = [0.0, 0.5, 1.0, 2.0]
    b = len(strengths)
    x, t, y = inp["x"].repeat(b, 1, 1, 1, 1), inp["t"].repeat(b), inp["y"].repeat(b, 1, 1)
    s = lora_scale(case["ctor"])
    with torch.no_grad():
        mine = m(x, t, y, lora_strength=torch.tensor(strengths, device="cuda"))
        for i, si in enumerate(strengths):
            truth = unet_lora_forward(sdg, inp["x"], inp["t"], inp["y"], si * s)
            with torch.autocast("cuda", dtype=torch.float16):
                ref16 = unet_lora_forward(sdg, inp["x"], inp["t"], inp["y"], si * s)
            _gates(mine[i:i + 1], truth, ref16, f"sample {i} at strength {si}")
            alone = m(inp["x"], inp["t"], inp["y"], lora_strength=si)
            assert torch.equal(mine[i:i + 1], alone), f"sample {i} of the batch differs from the same sample run alone"


def test_two_sets(golden_dir):
    case, m, inp, sdg = _setup(golden_dir, "iv_lora_tiny")
    extra = lora_pairs(case["ctor"], seed=72, rank=8)
    m.add_lora("second", extra, alpha=4)
    assert m.lora_names == ["default", "second"] and m.lora_signature == (("default", 4), ("second", 8))
    strength = torch.tensor([[1.0, 0.5], [0.25, -1.0]], device="cuda")
    x, t, y = torch.cat([inp["x"], inp["x"].flip(-1)]), inp["t"].repeat(2), torch.cat([inp["y"], inp["y_neg"]])
    own = {k: v for k, v in sdg.items() if "_lora." in k}
    base = {k: v for k, v in sdg.items() if "_lora." not in k}
    sets = [(own, lora_scale(case["ctor"])), ({k: v.cuda() for k, v in extra.items()}, 4 / 8)]
    with torch.no_grad():
        mine = m(x, t, y, lora_strength=strength)
        truth = oracle_multi(base, sets, x, t, y, strength.cpu())
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = oracle_multi(base, sets, x, t, y, strength.cpu())
    for i in range(2):
        _gates(mine[i:i + 1], truth[i:i + 1], ref16[i:i + 1], f"two sets, sample {i}")
    m.remove_lora("second")
    assert m.lora_names == ["default"]
    with torch.no_grad():
        one = m(inp["x"], inp["t"], inp["y"], lora_strength=1.0)
        truth1 = unet_lora_forward(sdg, inp["x"], inp["t"], inp["y"], lora_scale(case["ctor"]))
    assert _rel_l2(one, truth1) < 5e-3


def test_strength_zero_is_the_base_model_bit_for_bit(golden_dir):
    case, m, inp, sdg = _setup(golden_dir, "iv_lora_tiny")
    plain = vgen_b200.UNetSD_LoRA(**dict(case["ctor"], use_lora=False))
    plain.load_state_dict({k: v.cpu() for k, v in sdg.items() if "_lora." not in k}, strict=True)
    plain = plain.cuda().eval()
    with torch.no_grad():
        zero = m(inp["x"], inp["t"], inp["y"], lora_strength=0.0)
        ref = plain(inp["x"], inp["t"], inp["y"])
    assert torch.equal(zero, ref)


def test_cfg_pair_with_per_branch_strengths_is_one_forward(golden_dir, monkeypatch):
    case, m, inp, _ = _setup(golden_dir, "iv_lora_alpha_tiny_b2")
    b = case["b"]
    kc = {"y": inp["y"], "lora_strength": 1.0}
    ku = {"y": inp["y_neg"], "lora_strength": torch.zeros(b, 1)}
    calls = []
    impl = type(m)._forward_graphed
    monkeypatch.setattr(type(m), "_forward_graphed", lambda self, x, *a, **k: calls.append(x.shape[0]) or impl(self, x, *a, **k))
    with torch.no_grad():
        yc, yu = cfg_forward(m, inp["x"], inp["t"], [kc, ku])
        assert calls == [2 * b]
        ac = m(inp["x"], inp["t"], **kc)
        au = m(inp["x"], inp["t"], **ku)
    assert torch.equal(yc, ac) and torch.equal(yu, au)


def test_graph_replays_across_strength_changes(golden_dir):
    case, m, inp, _ = _setup(golden_dir, "iv_lora_alpha_tiny_b2")
    eager = type(m).forward.__wrapped_eager__
    s1 = torch.tensor([1.0, 0.0], device="cuda")
    s2 = torch.tensor([[0.5], [2.0]], device="cuda")
    with torch.no_grad():
        outs = [m(inp["x"], inp["t"], inp["y"], lora_strength=s1) for _ in range(3)]   # eager, capture, replay
        assert graph.stats(m)["forward"] == (1, 2)     # the capturing call replays too
        got2 = m(inp["x"], inp["t"], inp["y"], lora_strength=s2)
        assert graph.stats(m)["forward"] == (1, 3), "a new strength value must replay the captured graph"
        ref1 = eager(m, inp["x"], inp["t"], inp["y"], lora_strength=s1)
        ref2 = eager(m, inp["x"], inp["t"], inp["y"], lora_strength=s2)
    assert all(torch.equal(o, ref1) for o in outs)
    assert torch.equal(got2, ref2) and not torch.equal(got2, ref1)


def test_ddim_loop_with_per_branch_strengths(golden_dir):
    """4 CFG DDIM steps through DiffusionDDIMReward with lora_strength in model_kwargs (tuned conditional branch, base
    unconditional branch) against the oracle loop, with test_gpu_instructvideo.py's sampler gates."""
    case, m, inp, sdg = _setup(golden_dir, "iv_lora_tiny")
    diff = vgen_b200.DiffusionDDIMReward(**{k: v for k, v in RELEASED_DIFFUSION.items() if k != "type"})
    kw = [{"y": inp["y"], "lora_strength": 1.0}, {"y": inp["y_neg"], "lora_strength": 0.0}]
    s = lora_scale(case["ctor"])
    fn = lambda xt, t, **k: unet_lora_forward(sdg, xt, t, k["y"], k["lora_strength"] * s)  # noqa: E731
    lat = diff.ddim_sample_loop(inp["x"], m, kw, guide_scale=9.0, ddim_timesteps=4, eta=0.0)
    betas = vo.make_betas("linear_sd", 1000, False, init_beta=0.00085, last_beta=0.0120)
    with torch.no_grad():
        truth = vo.ddim_sample_loop(inp["x"].clone(), fn, kw, betas, 9.0, 4, mean_type="eps")
        with torch.autocast("cuda", dtype=torch.float16):
            lat16 = vo.ddim_sample_loop(inp["x"].clone(), fn, kw, betas, 9.0, 4, mean_type="eps", autocast_cfg=True)
    e_mine, e_ref16 = _rel_l2(lat, truth), _rel_l2(lat16, truth)
    print(f"runtime LoRA ddim: ours {e_mine:.3e}; reference-autocast {e_ref16:.3e}")
    assert lat.dtype == torch.float32 and torch.isfinite(lat).all()
    assert e_mine < 2.5e-2 and e_mine < 1.25 * e_ref16 + 5e-4
