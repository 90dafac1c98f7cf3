"""UNetSD_LoRA's runtime LoRA without a GPU: add_lora / remove_lora / lora_strength validation, the modes and the graph
signature, refusals (fp8_linear, other classes), cfg_forward's merge of [b] and [b, n] per-sample values, and the
linearity of the several-set oracle restatement."""
import pytest
import torch
import torch.nn.functional as F

import vgen_b200
from vgen_b200 import graph
from vgen_b200.diffusion import _per_sample, cfg_forward
from _instructvideo import IV_CASES
from _lora_runtime import combined_pairs, lora_pairs, sites

CTOR = IV_CASES["iv_nolora_tiny"]["ctor"]


@pytest.fixture(scope="module")
def pairs():
    return lora_pairs(CTOR, seed=3)


def _base():
    return vgen_b200.UNetSD_LoRA(**CTOR)


def _x(b=1):
    return torch.zeros(b, 4, 2, 8, 8)


def test_add_and_remove(pairs):
    m = _base()
    assert m.lora_names == [] and m.lora_signature is None
    m.add_lora("a", pairs, alpha=8)
    m.add_lora("b", {**pairs, "unrelated.weight": torch.zeros(1)})   # a full checkpoint: only the LoRA keys are read
    assert m.lora_names == ["a", "b"] and m.lora_signature == (("a", 4), ("b", 4))
    assert m._lora_added["a"][2] == 2.0 and m._lora_added["b"][2] == 1.0
    m.remove_lora("a")
    assert m.lora_names == ["b"]
    own = vgen_b200.UNetSD_LoRA(**dict(CTOR, use_lora=True))
    assert own.lora_names == ["default"] and own.lora_signature is None


def test_add_lora_validation(pairs):
    m = _base()
    down = sorted(k for k in pairs if k.endswith("down_linear.weight"))
    k0, u0 = down[0], down[0].replace("down_linear", "up_linear")
    with pytest.raises(ValueError, match="lacks 1 of"):
        m.add_lora("x", {k: v for k, v in pairs.items() if k != k0})
    with pytest.raises(ValueError, match="no site for, first nowhere.attn1.to_q_lora"):
        m.add_lora("x", {**pairs, "nowhere.attn1.to_q_lora.down_linear.weight": pairs[k0]})
    with pytest.raises(ValueError, match="the site .* needs"):
        m.add_lora("x", {**pairs, k0: pairs[k0][:, :-1]})
    with pytest.raises(ValueError, match="rank 65, supported 1 to 64"):
        big = {k: (torch.zeros(65, v.shape[1]) if "down" in k else torch.zeros(v.shape[0], 65)) for k, v in pairs.items()}
        m.add_lora("x", big)
    with pytest.raises(ValueError, match="one rank"):
        m.add_lora("x", {**pairs, k0: torch.zeros(2, pairs[k0].shape[1]), u0: torch.zeros(pairs[u0].shape[0], 2)})
    with pytest.raises(ValueError, match="not finite"):
        bad = pairs[u0].clone()
        bad[0, 0] = float("nan")
        m.add_lora("x", {**pairs, u0: bad})
    with pytest.raises(ValueError, match="not finite"):
        m.add_lora("x", {**pairs, k0: pairs[k0] * 1e6})     # overflows fp16
    with pytest.raises(ValueError, match="alpha"):
        m.add_lora("x", pairs, alpha=float("inf"))
    with pytest.raises(ValueError, match="non-empty string"):
        m.add_lora("", pairs)
    assert m.lora_names == [] and not m._lora_rt, "a refused set changes nothing"
    m.add_lora("x", pairs)
    with pytest.raises(ValueError, match="exists already"):
        m.add_lora("x", pairs)
    with pytest.raises(ValueError, match="no added LoRA set named 'y'"):
        m.remove_lora("y")
    own = vgen_b200.UNetSD_LoRA(**dict(CTOR, use_lora=True))
    with pytest.raises(ValueError, match="exists already"):
        own.add_lora("default", pairs)
    with pytest.raises(ValueError, match="no added LoRA set named 'default'"):
        own.remove_lora("default")


def test_lora_strength_validation(pairs):
    m = _base()
    with pytest.raises(ValueError, match="no LoRA set"):
        m(_x(), torch.zeros(1), torch.zeros(1, 5, 1024), lora_strength=1.0)
    m.add_lora("a", pairs)
    m.add_lora("b", pairs)
    for bad in (torch.ones(3), torch.ones(2, 3), torch.ones(2, 2, 1), "1"):
        with pytest.raises(ValueError, match="lora_strength must be"):
            m(_x(2), torch.zeros(2), torch.zeros(2, 5, 1024), lora_strength=bad)
    for bad in (float("nan"), torch.tensor([1.0, float("inf")])):
        with pytest.raises(ValueError, match="finite"):
            m(_x(2), torch.zeros(2), torch.zeros(2, 5, 1024), lora_strength=bad)
    # valid strengths get as far as the device check (there is no CPU path)
    for good in (0.5, torch.ones(2), torch.ones(2, 2), torch.tensor(2.0)):
        with pytest.raises(vgen_b200.lib.VgenError, match="CUDA"):
            m(_x(2), torch.zeros(2), torch.zeros(2, 5, 1024), lora_strength=good)


def test_strength_rows_and_modes(pairs):
    own = vgen_b200.UNetSD_LoRA(**dict(CTOR, use_lora=True, lora_alpha=8))
    x = _x(2)
    assert own._strength_rows(None, x) is None and not own._lora_rt       # merged mode
    s = own._strength_rows(torch.tensor([0.0, 2.0]), x)
    assert own._lora_rt and s.shape == (2, 1) and s[:, 0].tolist() == [0.0, 2.0]
    assert torch.equal(own._strength_rows(None, x), torch.ones(2, 1))     # runtime mode, no lora_strength: 1 for every set
    own.add_lora("b", pairs)
    assert own._strength_rows(3.0, x).tolist() == [[3.0, 3.0]] * 2
    assert own.lora_signature == (("default", 4), ("b", 4))
    assert ("lora", own.lora_signature) in graph._mode(own)
    sd = own._pack_state_dict()
    assert not any("_lora." in k for k in sd)
    assert all(torch.equal(sd[k], v) for k, v in own.state_dict().items() if "_lora." not in k), "runtime mode packs unmerged"


def test_fp8_and_other_classes_refuse(pairs):
    m = _base()
    m.fp8_linear = True
    with pytest.raises(NotImplementedError, match="fp8_linear"):
        m.add_lora("a", pairs)
    m.fp8_linear = False
    m.add_lora("a", pairs)
    with pytest.raises(NotImplementedError, match="fp8_linear"):
        m.fp8_linear = True
    assert m.fp8_linear is False
    t2v = vgen_b200.UNetSD_T2VBase(**{k: v for k, v in CTOR.items() if "lora" not in k})
    with pytest.raises(NotImplementedError, match="UNetSD_LoRA"):
        t2v.add_lora("a", pairs)
    with pytest.raises(NotImplementedError, match="UNetSD_LoRA"):
        t2v(_x(), torch.zeros(1), y=torch.zeros(1, 5, 1024), lora_strength=1.0)


class _Stub:
    cfg_batch = True
    cfg_per_sample = ("lora_strength",)

    def __init__(self):
        self.calls = []

    def __call__(self, x, t, **kw):
        self.calls.append(kw)
        return x


def test_cfg_forward_merges_1d_and_2d_per_sample_values():
    xt, ts = torch.zeros(2, 4, 1, 2, 2), torch.zeros(2, dtype=torch.long)
    m = _Stub()
    cfg_forward(m, xt, ts, [{"lora_strength": torch.tensor([[1.0, 0.5], [2.0, 0.0]])}, {"lora_strength": 0.25}])
    assert len(m.calls) == 1
    assert m.calls[0]["lora_strength"].tolist() == [[1.0, 0.5], [2.0, 0.0], [0.25, 0.25], [0.25, 0.25]]
    m = _Stub()
    cfg_forward(m, xt, ts, [{"lora_strength": torch.tensor([1.0, 2.0])}, {"lora_strength": torch.ones(1, 3)}])
    assert m.calls[0]["lora_strength"].tolist() == [[1.0] * 3, [2.0] * 3, [1.0] * 3, [1.0] * 3]
    m = _Stub()
    cfg_forward(m, xt, ts, [{"lora_strength": 1.0}, {"lora_strength": 0.0}])
    assert m.calls[0]["lora_strength"].tolist() == [1.0, 1.0, 0.0, 0.0]       # 1-D stays 1-D, as before
    assert _per_sample(torch.ones(1, 2), xt).shape == (2, 2)
    with pytest.raises(ValueError):
        _per_sample(torch.ones(3, 2), xt)


def test_several_set_oracle_is_the_sum_of_single_set_deltas(pairs):
    """The concatenated pair at (s1, s2) adds, at every projection, the sum of the two sets' single-set terms."""
    other = lora_pairs(CTOR, seed=4, rank=8)
    sets = [(pairs, 2.0), (other, 0.5)]
    g = torch.Generator().manual_seed(0)
    for site in sites(pairs)[:8]:
        x = torch.randn(5, pairs[site + ".down_linear.weight"].shape[1], generator=g, dtype=torch.float64)

        def delta(s1, s2):
            c = combined_pairs(sets, [s1, s2])
            return F.linear(F.linear(x, c[site + ".down_linear.weight"]), c[site + ".up_linear.weight"])
        torch.testing.assert_close(delta(0.7, -1.5), delta(0.7, 0.0) + delta(0.0, -1.5), rtol=1e-12, atol=1e-12)
        one = F.linear(F.linear(x, pairs[site + ".down_linear.weight"].double()), pairs[site + ".up_linear.weight"].double())
        torch.testing.assert_close(delta(0.7, 0.0), 0.7 * 2.0 * one, rtol=1e-12, atol=1e-12)
