"""VideoComposer compositions of UNetSD_VideoLCM / UNetSD_TFT2V on the host: parameter specs against the reference's,
strict checkpoint loading, registry builds of the released UNet dicts, refusals, the oracle against the reference's
frozen outputs, and the cond_stem entry point in the binding."""
import json
import os

import numpy as np
import pytest
import torch

import vgen_b200
from oracle import synth
from vgen_b200 import arch, lib
from _vcomp import (FULL_SPECS, RELEASED_UNET, VCOMP_CASES, build_product, load_spec, make_inputs, oracle_call,
                    product_spec, reference_digest, spec_digest)


def _plan(ctor, comps, resolution=(448, 256)):
    kk = dict(ctor, dim_mult=tuple(ctor["dim_mult"]), attn_scales=tuple(ctor.get("attn_scales", (1 / 2, 1 / 4, 1 / 8))))
    return arch.unet_plan("videolcm", video_compositions=tuple(comps), resolution=resolution, **kk)


@pytest.mark.parametrize("name,count", [("full_vcomposer", 1574), ("full_tft2v", 1484), ("released_vcomposer", 1574),
                                        ("released_tft2v", 1484)])
def test_full_spec_equals_reference(golden_dir, name, count):
    """The parameter list (names, shapes, order) equals the reference class's, through its frozen digest."""
    comps, ctor = FULL_SPECS[name]
    mine = arch.unet_spec(_plan(ctor, comps))
    assert len(mine) == count and spec_digest(mine) == reference_digest(golden_dir, name)


@pytest.mark.parametrize("name", sorted(VCOMP_CASES))
def test_tiny_spec_equals_reference_and_loads_strictly(golden_dir, name):
    case = VCOMP_CASES[name]
    ref = load_spec(golden_dir, name)          # checks the digest
    m = build_product(case)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == ref
    m.load_state_dict(synth.state_dict(ref, seed=1), strict=True)
    assert m.video_compositions == case["comps"]


def test_text_only_videolcm_spec_unchanged(golden_dir):
    """No composition but 'text': the layout of configs/videolcm_t2v_infer.yaml (1 480 tensors at full size)."""
    ref = [(k, tuple(s)) for k, s in json.load(open(os.path.join(golden_dir, "full_videolcm.spec.json")))]
    assert arch.unet_spec(_plan(FULL_SPECS["full_vcomposer"][1], ["text"])) == ref
    m = vgen_b200.UNetSD_VideoLCM(config={"video_compositions": ["text"]}, **VCOMP_CASES["tft2v_tiny"]["ctor"])
    assert not any("embedding_after" in k or "pre_image_condition" in k for k in m.state_dict())


def _released_unet_dict(cls):
    """The UNet section of configs/tft2v_vcomposer_infer.yaml / videolcm_vcomposer_infer.yaml (tft2v_t2v_infer.yaml has
    the same keys), with "config" filled in as the inference entrances do."""
    return dict(RELEASED_UNET, type=cls, config=None)


class _AttrConfig(dict):
    """The reference's EasyDict: keys readable as attributes."""
    __getattr__ = dict.__getitem__


@pytest.mark.parametrize("cls,spec", [("UNetSD_TFT2V", "released_vcomposer"), ("UNetSD_TFT2V", "released_tft2v"),
                                      ("UNetSD_VideoLCM", "released_vcomposer")])
def test_registry_builds_released_unet_dicts(golden_dir, cls, spec):
    MODEL, _, _ = vgen_b200.register(force_local=True)
    assert MODEL.get("UNetSD_TFT2V") is vgen_b200.UNetSD_TFT2V
    d = _released_unet_dict(cls)
    d["config"] = _AttrConfig(video_compositions=FULL_SPECS[spec][0], resolution=[448, 256])
    with torch.device("meta"):
        m = MODEL.build(d)
    assert type(m) is getattr(vgen_b200, cls)
    assert m.resolution == (448, 256)
    assert spec_digest([(k, tuple(v.shape)) for k, v in m.state_dict().items()]) == reference_digest(golden_dir, spec)
    assert product_spec(cls, FULL_SPECS[spec][0], (448, 256), RELEASED_UNET) == arch.unet_spec(m.plan)


def test_refusals():
    ctor = VCOMP_CASES["tft2v_tiny"]["ctor"]
    with pytest.raises(NotImplementedError, match="histogram"):
        vgen_b200.UNetSD_TFT2V(config={"video_compositions": ["text", "histogram"], "resolution": [96, 64]}, **ctor)
    with pytest.raises(NotImplementedError, match="use_text_clip_vip_model"):
        vgen_b200.UNetSD_TFT2V(config={"video_compositions": ["text"], "use_text_clip_vip_model": True}, **ctor)
    with pytest.raises(ValueError, match="unknown"):
        vgen_b200.UNetSD_VideoLCM(config={"video_compositions": ["text", "depth"], "resolution": [96, 64]}, **ctor)
    with pytest.raises(ValueError, match="resolution"):
        vgen_b200.UNetSD_VideoLCM(config={"video_compositions": ["text", "sketch"]}, **ctor)
    # a condition passed but not listed is rejected before any device work (so this runs without a GPU)
    m = vgen_b200.UNetSD_TFT2V(config={"video_compositions": ["text", "depthmap"], "resolution": [96, 64]}, **ctor)
    m._check_x = lambda x, t: None
    x, t = torch.zeros(1, 4, 2, 8, 12), torch.zeros(1, dtype=torch.long)
    fwd = type(m).forward.__wrapped_eager__
    with pytest.raises(ValueError, match="'sketch' was passed"):
        fwd(m, x, t, y=torch.zeros(1, 5, 1024), sketch=torch.zeros(1, 1, 2, 64, 96))
    with pytest.raises(ValueError, match="'image' was passed"):
        fwd(m, x, t, y=torch.zeros(1, 5, 1024), image=torch.zeros(1, 1, 1024))
    with pytest.raises(NotImplementedError, match="histogram"):
        fwd(m, x, t, y=torch.zeros(1, 5, 1024), histogram=torch.zeros(1, 2, 156))


@pytest.mark.parametrize("name", sorted(VCOMP_CASES))
def test_oracle_against_reference_outputs(golden_dir, name):
    """The oracle restatement against the reference classes' outputs frozen under two weight seeds."""
    torch.set_grad_enabled(False)
    case = VCOMP_CASES[name]
    spec = load_spec(golden_dir, name)
    inp = make_inputs(case)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["out"]
    pin = np.load(os.path.join(golden_dir, "vcomp_pin.npz"))[f"{name}_seed81"]
    for seed, ref in ((case["seed"], gold), (81, pin)):
        out = oracle_call(case, synth.state_dict(spec, seed=seed), inp)
        ref = torch.from_numpy(ref)
        assert float((out - ref).abs().max() / ref.abs().max()) < 2e-5, seed


def test_cond_stem_is_part_of_the_abi():
    """Declared in the binding, hence (tests/test_host_logic.py) in the header and the library."""
    assert "vgen_cond_stem" in lib.declared_symbols()
