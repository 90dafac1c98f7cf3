"""The sketch annotators (PiDiNet, sketch-simplification GAN) on the host: parameter lists against the reference's, strict
and pretrained loading (with the PDC -> vanilla conversion), the oracle against the reference's frozen outputs, the
refusals, and the engine's module chain."""
import json
import os

import numpy as np
import pytest
import torch

import vgen_b200
from oracle import sketch_oracle
from vgen_b200 import lib
from vgen_b200.sketch import PiDiNet, SketchSimplification, convert_pidinet, pidinet_bsd, sketch_simplification_gan
from _sketch import (CARV4, GAN_MEAN, GAN_STD, SKETCH_CASES, TINY_PIDINET, load_spec, make_input, non_vacuous,
                     pdc_state_dict, state_dict, tensor_digest)


def test_specs_match_reference_digests(golden_dir):
    full, tiny, gan = (load_spec(golden_dir, w) for w in ("pidinet_full", "pidinet_tiny", "cleaner"))
    assert len(full) == 83 and sum(torch.Size(s).numel() for _, s in full) == 720709
    assert len(gan) == 46 and sum(torch.Size(s).numel() for _, s in gan) == 44387249
    assert len(tiny) == 83
    with torch.device("meta"):
        assert [(k, tuple(v.shape)) for k, v in pidinet_bsd().state_dict().items()] == full
        assert [(k, tuple(v.shape)) for k, v in sketch_simplification_gan().state_dict().items()] == gan


@pytest.mark.parametrize("which", ["pidinet_tiny", "cleaner"])
def test_strict_loading(golden_dir, which):
    spec = load_spec(golden_dir, which)
    m = PiDiNet(**TINY_PIDINET) if which == "pidinet_tiny" else SketchSimplification(GAN_MEAN, GAN_STD)
    sd = state_dict(spec, 1, "pidinet" if which == "pidinet_tiny" else "cleaner")
    m.load_state_dict(sd, strict=True)
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    with pytest.raises(RuntimeError):
        m.load_state_dict({k: v for k, v in sd.items() if k != spec[-1][0]}, strict=True)


def test_pidinet_pretrained_converts_pdc_weights(golden_dir, tmp_path, monkeypatch):
    pdc = pdc_state_dict(load_spec(golden_dir, "pidinet_full"))
    os.makedirs(tmp_path / "models")
    torch.save({"state_dict": pdc, "epoch": 1}, tmp_path / "models" / "table5_pidinet.pth")
    monkeypatch.chdir(tmp_path)
    m = vgen_b200.pidinet_bsd(pretrained=True)
    assert isinstance(m, PiDiNet)
    want = json.load(open(os.path.join(golden_dir, "sketch_specs.json")))["pidinet_converted"]
    assert tensor_digest(m.state_dict()) == want
    conv = convert_pidinet(pdc, CARV4)
    assert tensor_digest({k[len("module."):]: v for k, v in conv.items()}) == want
    assert all(torch.equal(v, pdc[k]) for k, v in pdc_state_dict(load_spec(golden_dir, "pidinet_full")).items())


def test_cleaner_pretrained_loads_from_working_directory(golden_dir, tmp_path, monkeypatch):
    sd = state_dict(load_spec(golden_dir, "cleaner"), 7, "cleaner")
    os.makedirs(tmp_path / "models")
    torch.save(sd, tmp_path / "models" / "sketch_simplification_gan.pth")
    monkeypatch.chdir(tmp_path)
    m = vgen_b200.sketch_simplification_gan(pretrained=True)
    assert isinstance(m, SketchSimplification) and (m.mean, m.std) == (GAN_MEAN, GAN_STD)
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())


@pytest.mark.parametrize("name", sorted(SKETCH_CASES))
def test_oracle_against_reference_outputs(golden_dir, name):
    torch.set_grad_enabled(False)
    case = SKETCH_CASES[name]
    x = make_input(case["net"], case["n"], case["H"], case["W"], case["seed"])
    if case["net"] == "pidinet":
        out = sketch_oracle.pidinet_forward(state_dict(load_spec(golden_dir, "pidinet_tiny"), case["seed"], "pidinet"), x)
    else:
        out = sketch_oracle.cleaner_forward(state_dict(load_spec(golden_dir, "cleaner"), case["seed"], "cleaner"), x, GAN_MEAN,
                                            GAN_STD)
    ref = torch.from_numpy(np.load(os.path.join(golden_dir, f"sketch_{name}.npz"))["out"])
    assert out.shape == ref.shape == (case["n"], 1, case["H"], case["W"])
    assert float((out - ref).abs().max()) <= 1e-6
    std, sat = non_vacuous(ref)
    assert std > 0.05 and sat < 0.5


@pytest.mark.parametrize("kw", [dict(convert=False), dict(sa=False), dict(dil=None)])
def test_unsupported_pidinet_forms_are_refused(kw):
    with pytest.raises(NotImplementedError):
        PiDiNet(**dict(TINY_PIDINET, **kw))


def test_pdc_networks_are_refused():
    with pytest.raises(NotImplementedError):
        pidinet_bsd(vanilla_cnn=False)


@pytest.mark.parametrize("hw", [(7, 64), (64, 4)])
def test_pidinet_sizes_below_8_are_refused(hw):
    with pytest.raises(ValueError, match="at least 8"):
        PiDiNet(**TINY_PIDINET)(torch.zeros(1, 3, *hw))


@pytest.mark.parametrize("hw", [(60, 64), (64, 100), (36, 44)])
def test_cleaner_sizes_off_multiples_of_8_are_refused(hw):
    with pytest.raises(ValueError, match="multiples of 8"):
        sketch_simplification_gan()(torch.zeros(1, 1, *hw))


@pytest.mark.parametrize("net", ["pidinet", "cleaner"])
def test_cpu_forward_raises(net):
    m, c = (PiDiNet(**TINY_PIDINET), 3) if net == "pidinet" else (sketch_simplification_gan(), 1)
    with pytest.raises(lib.VgenError, match="CUDA"):
        m(torch.zeros(1, c, 64, 64))


def test_engine_chain_keeps_names_and_drops_packed_weights():
    for m in (pidinet_bsd(), sketch_simplification_gan()):
        names = [k for k, _ in m.state_dict().items()]
        m._packed = {"stale": torch.zeros(1)}
        m = m.eval().requires_grad_(False)
        m._packed = {"stale": torch.zeros(1)}
        m = m.to("cpu")
        assert m._packed is None
        m._packed = {"stale": torch.zeros(1)}
        m = m.half()
        assert m._packed is None and not any(p.requires_grad for p in m.parameters())
        assert [k for k, _ in m.state_dict().items()] == names
        assert all(v.dtype == torch.float16 for v in m.state_dict().values())
