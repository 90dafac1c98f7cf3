"""The MiDaS v3 depth annotator on the host: parameter lists against the reference's, strict and pretrained loading, the
oracle against the reference's frozen outputs, the refusals, and the engine's module chain."""
import os

import numpy as np
import pytest
import torch

import vgen_b200
from oracle import depth_oracle
from vgen_b200 import lib
from vgen_b200.depth import MiDaS, midas_v3
from _depth import DEPTH_CASES, FULL, TINY, load_spec, make_input, oracle_kw, product_spec, state_dict


def test_specs_match_reference_digests(golden_dir):
    tiny, full = load_spec(golden_dir, "tiny"), load_spec(golden_dir, "full")
    assert len(full) == 364 and round(sum(torch.Size(s).numel() for _, s in full) / 1e6, 2) == 343.03
    assert len(tiny) == 124
    with torch.device("meta"):
        m = midas_v3()
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == full == product_spec(FULL)


def test_strict_loading(golden_dir):
    spec = load_spec(golden_dir, "tiny")
    m = vgen_b200.MiDaS(**TINY)
    sd = state_dict(spec, 1)
    m.load_state_dict(sd, strict=True)
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    with pytest.raises(RuntimeError):
        m.load_state_dict({k: v for k, v in sd.items() if k != "head.4.bias"}, strict=True)
    with torch.device("meta"):
        big = vgen_b200.midas_v3()
        big.load_state_dict({k: torch.empty(s) for k, s in load_spec(golden_dir, "full")}, strict=True)


def test_pretrained_loads_from_working_directory(golden_dir, tmp_path, monkeypatch):
    sd = state_dict(load_spec(golden_dir, "tiny"), 7)
    os.makedirs(tmp_path / "models")
    torch.save(sd, tmp_path / "models" / "midas_v3_dpt_large.pth")
    monkeypatch.chdir(tmp_path)
    m = midas_v3(pretrained=True, **TINY)
    assert isinstance(m, MiDaS)
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())


@pytest.mark.parametrize("name", sorted(DEPTH_CASES))
def test_oracle_against_reference_outputs(golden_dir, name):
    torch.set_grad_enabled(False)
    case = DEPTH_CASES[name]
    sd = state_dict(load_spec(golden_dir, "tiny"), case["seed"])
    out = depth_oracle.midas_forward(sd, make_input(case["n"], case["H"], case["W"], case["seed"]), **oracle_kw(case["ctor"]))
    ref = torch.from_numpy(np.load(os.path.join(golden_dir, f"depth_{name}.npz"))["out"])
    assert out.shape == ref.shape == (case["n"], 1, case["H"], case["W"])
    assert float((out - ref).abs().max() / ref.abs().max()) <= 1e-5
    assert float((ref > 0).float().mean()) > 0.3


@pytest.mark.parametrize("hw", [(48, 64), (64, 80), (64, 65)])
def test_sizes_off_multiples_of_32_are_refused(hw):
    m = MiDaS(**TINY)
    with pytest.raises(ValueError, match="multiples of 32"):
        m(torch.zeros(1, 3, *hw))


def test_cpu_forward_raises():
    m = MiDaS(**TINY)
    with pytest.raises(lib.VgenError, match="CUDA"):
        m(torch.zeros(1, 3, 64, 64))


def test_head_dim_other_than_64_is_refused():
    m = MiDaS(**dict(TINY, num_heads=4))
    with pytest.raises(NotImplementedError, match="head_dim 32"):
        m(torch.zeros(1, 3, 64, 64))


@pytest.mark.parametrize("kw", [dict(neck_dims=[64, 64, 128, 96]), dict(neck_dims=[32, 64, 128, 128]), dict(fusion_dim=64),
                                dict(fusion_dim=192)])
def test_neck_and_fusion_widths_are_refused_at_construction(kw):
    with pytest.raises(NotImplementedError):
        MiDaS(**dict(TINY, **kw))


def test_engine_chain_keeps_names_and_dtype_and_drops_packed_weights():
    m = MiDaS(**TINY)
    names = [k for k, _ in m.state_dict().items()]
    m._packed = {"stale": torch.zeros(1)}
    m = m.eval().requires_grad_(False).to(memory_format=torch.channels_last).half()
    assert m._packed is None
    assert [k for k, _ in m.state_dict().items()] == names
    assert all(v.dtype == torch.float16 for v in m.state_dict().values())
    assert m.patch_embedding.weight.is_contiguous(memory_format=torch.channels_last)
