"""DreamVideo (UNetSD_DreamVideo) on the host: parameter specs against the reference's, strict loading of a merged base +
adapter checkpoint, registry builds of the released UNet dicts, refusals, the oracle against the reference's frozen
outputs, cfg_forward's per-sample merge, and the new entry points in the binding."""
import os

import numpy as np
import pytest
import torch

import vgen_b200
from oracle import synth
from vgen_b200 import arch, lib
from vgen_b200.diffusion import cfg_forward
from _dreamvideo import (DV_CASES, RELEASED_ADAPTERS, RELEASED_COUNTS, RELEASED_UNET, build_product, load_spec, make_inputs,
                         oracle_call, product_spec, reference_digest, spec_digest)


@pytest.mark.parametrize("name", sorted(RELEASED_ADAPTERS))
def test_released_spec_equals_reference(golden_dir, name):
    spec = product_spec(dict(RELEASED_UNET, **RELEASED_ADAPTERS[name]))
    d = spec_digest(spec)
    assert (d["tensors"], d["parameters"]) == RELEASED_COUNTS[name]
    assert d == reference_digest(golden_dir, name)


def test_base_flavour_is_t2vbase():
    """Without adapters the parameter list is UNetSD_T2VBase's."""
    with torch.device("meta"):
        base = vgen_b200.UNetSD_T2VBase(**RELEASED_UNET)
    assert product_spec(RELEASED_UNET) == [(k, tuple(v.shape)) for k, v in base.state_dict().items()]


@pytest.mark.parametrize("name", sorted(DV_CASES))
def test_tiny_spec_equals_reference_and_loads_strictly(golden_dir, name):
    ref = load_spec(golden_dir, name)          # checks the digest
    m = build_product(DV_CASES[name])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == ref
    m.load_state_dict(synth.state_dict(ref, seed=1), strict=True)


def test_merged_base_and_adapter_checkpoints_load_strictly():
    """inference_dreamvideo_entrance.py:158-192: the base checkpoint updated with the identity and motion adapter
    checkpoints, loaded with strict=True."""
    ctor = DV_CASES["dv_joint_tiny_b2"]["ctor"]
    base_spec = product_spec({k: v for k, v in ctor.items() if "adapter" not in k})
    full_spec = product_spec(ctor)
    base = synth.state_dict(base_spec, seed=3)
    adapters = synth.state_dict([(k, s) for k, s in full_spec if "_adapter." in k], seed=4)
    m = build_product(DV_CASES["dv_joint_tiny_b2"])
    spatial = tuple(L.prefix for blk in m.plan.input_blocks + [m.plan.middle] + m.plan.output_blocks for L in blk
                    if L.kind == "spatial")
    merged = dict(base)
    merged.update({k: v for k, v in adapters.items() if k.startswith(spatial)})          # identity adapter checkpoint
    merged.update({k: v for k, v in adapters.items() if not k.startswith(spatial)})      # motion adapter checkpoint
    m.load_state_dict(merged, strict=True)
    assert torch.equal(m.state_dict()[next(k for k in adapters if "condition_linear" in k)],
                       adapters[next(k for k in adapters if "condition_linear" in k)])
    with pytest.raises(RuntimeError, match="Missing"):
        build_product(DV_CASES["dv_joint_tiny_b2"]).load_state_dict(base, strict=True)


class _AttrConfig(dict):
    __getattr__ = dict.__getitem__


@pytest.mark.parametrize("name", ["released_subject", "released_motion", "released_joint"])
def test_registry_builds_released_unet_dicts(golden_dir, name):
    MODEL, _, _ = vgen_b200.register(force_local=True)
    assert MODEL.get("UNetSD_DreamVideo") is vgen_b200.UNetSD_DreamVideo
    d = dict(RELEASED_UNET, **RELEASED_ADAPTERS[name], type="UNetSD_DreamVideo", config=_AttrConfig())
    with torch.device("meta"):
        m = MODEL.build(d)
    assert type(m) is vgen_b200.UNetSD_DreamVideo
    assert spec_digest([(k, tuple(v.shape)) for k, v in m.state_dict().items()]) == reference_digest(golden_dir, name)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == arch.unet_spec(m.plan)


def test_refusals():
    ctor = DV_CASES["dv_motion_tiny"]["ctor"]
    with pytest.raises(ValueError, match="unknown temporal adapters"):
        vgen_b200.UNetSD_DreamVideo(**dict(ctor, temporal_adapter_list=["self_attention", "ff"]))
    with pytest.raises(ValueError, match="unknown spatial adapters"):
        vgen_b200.UNetSD_DreamVideo(**dict(ctor, spatial_adapter_list=["cross"]))
    with pytest.raises(NotImplementedError, match="'parallel' and 'serial'"):
        vgen_b200.UNetSD_DreamVideo(**dict(ctor, temporal_adapter_position_list=["parallel", "", "parallel"]))
    with pytest.raises(NotImplementedError, match="'parallel' and 'serial'"):
        vgen_b200.UNetSD_DreamVideo(**dict(ctor, spatial_adapter_list=["self_attention"]))   # default positions ['', 'parallel', '']
    # shapes are checked before any device work (so this runs without a GPU)
    m = vgen_b200.UNetSD_DreamVideo(**ctor)
    m._check_x = lambda x, t: None
    x, t = torch.zeros(1, 4, 3, 8, 12), torch.zeros(1, dtype=torch.long)
    fwd = type(m).forward.__wrapped_eager__
    y = torch.zeros(1, 5, 1024)
    with pytest.raises(ValueError, match="y_image must be"):
        fwd(m, x, t, y=y, y_image=torch.zeros(1, 2, 1024))
    with pytest.raises(ValueError, match="y_image must be"):
        fwd(m, x, t, y=y, y_image=torch.zeros(1, 1, 512))
    with pytest.raises(ValueError, match="ag_strength"):
        fwd(m, x, t, y=y, y_image=torch.zeros(1, 1, 1024), ag_strength=torch.ones(2))


def test_training_kwargs_are_swallowed():
    m = vgen_b200.UNetSD_DreamVideo(**DV_CASES["dv_subject_tiny"]["ctor"], upper_len=128, default_fps=8, misc_dropout=0.4)
    assert m.spatial_adapter_list == ["cross_attention"] and m.temporal_adapter_list == []


@pytest.mark.parametrize("name", sorted(DV_CASES))
def test_oracle_against_reference_outputs(golden_dir, name):
    """The oracle restatement against the reference class's outputs frozen under two weight seeds."""
    torch.set_grad_enabled(False)
    case = DV_CASES[name]
    spec = load_spec(golden_dir, name)
    inp = make_inputs(case)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["out"]
    pin = np.load(os.path.join(golden_dir, "dreamvideo_pin.npz"))[f"{name}_seed82"]
    for seed, ref in ((case["seed"], gold), (82, pin)):
        out = oracle_call(case, synth.state_dict(spec, seed=seed), inp)
        ref = torch.from_numpy(ref)
        assert float((out - ref).abs().max() / ref.abs().max()) < 2e-5, seed


class _StandIn:
    """A CPU model with the attributes cfg_forward reads; records what it was called with."""
    cfg_batch = True

    def __init__(self, per_sample=None):
        if per_sample is not None:
            self.cfg_per_sample = per_sample
        self.calls = []

    def __call__(self, x, t, **kw):
        self.calls.append((x, t, kw))
        return x * (1.0 + torch.arange(x.shape[0], dtype=x.dtype).view(-1, 1, 1, 1, 1))


def test_cfg_forward_merges_per_sample_keys():
    xt, ts = torch.randn(2, 4, 3, 2, 2), torch.tensor([5, 5])
    y, yi = torch.randn(2, 3, 8), torch.randn(2, 1, 8)
    kc = {"y": y, "y_image": yi, "ag_strength": 1}
    ku = {"y": torch.zeros_like(y), "y_image": torch.zeros_like(yi), "ag_strength": 0.0}
    m = _StandIn(("ag_strength",))
    yc, yu = cfg_forward(m, xt, ts, [kc, ku])
    assert len(m.calls) == 1
    x, t, kw = m.calls[0]
    assert x.shape[0] == 4 and torch.equal(t, torch.tensor([5, 5, 5, 5]))
    assert kw["ag_strength"].dtype == torch.float32 and kw["ag_strength"].tolist() == [1.0, 1.0, 0.0, 0.0]
    assert kw["y_image"].shape == (4, 1, 8)
    assert yc.shape == xt.shape and yu.shape == xt.shape
    # a [b] tensor per branch
    m = _StandIn(("ag_strength",))
    cfg_forward(m, xt, ts, [dict(kc, ag_strength=torch.tensor([0.5, 1.0])), dict(ku, ag_strength=torch.tensor([0.0, 0.25]))])
    assert m.calls[0][2]["ag_strength"].tolist() == [0.5, 1.0, 0.0, 0.25]


def test_cfg_forward_unchanged_without_per_sample_keys():
    """A model that names no per-sample keys keeps today's behaviour: differing floats mean two calls."""
    xt, ts = torch.randn(1, 4, 2, 2, 2), torch.tensor([7])
    kc, ku = {"y": torch.randn(1, 3, 8), "ag_strength": 1}, {"y": torch.randn(1, 3, 8), "ag_strength": 0}
    m = _StandIn()
    cfg_forward(m, xt, ts, [kc, ku])
    assert len(m.calls) == 2 and m.calls[0][2]["ag_strength"] == 1 and m.calls[1][2]["ag_strength"] == 0
    m = _StandIn()
    cfg_forward(m, xt, ts, [{"y": kc["y"]}, {"y": ku["y"]}])
    assert len(m.calls) == 1 and m.calls[0][0].shape[0] == 2


def test_adapter_entry_points_are_part_of_the_abi():
    """Declared in the binding, hence (tests/test_host_logic.py) in the header and the library."""
    assert {"vgen_linear_gelu_rowbias", "vgen_adapter_condition"} <= set(lib.declared_symbols())
