"""Host side of the opt-in FP8 transformer projections (no GPU): the constructor keyword and its refusals, the weight
quantiser, the GEGLU tile choice, the C entry points and the graph signature."""
import os
import re

import pytest
import torch

import vgen_b200
from oracle.cases import CASES
from vgen_b200 import graph, lib, ops, unet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _meta(cls, **kw):
    with torch.device("meta"):
        return cls(**kw)


def test_constructor_keyword_and_property():
    ctor = CASES["t2v_tiny"]["ctor"]
    assert _meta(vgen_b200.UNetSD_T2VBase, **ctor).fp8_linear is False
    assert _meta(vgen_b200.UNetSD_T2VBase, **ctor, fp8_linear=False).fp8_linear is False
    assert _meta(vgen_b200.UNetSD_T2VBase, **ctor, fp8_linear=True).fp8_linear is True
    for cls, extra in ((vgen_b200.UNetSD_I2VGen, {}), (vgen_b200.UNetSD_SR600, {}), (vgen_b200.UNetSD_HiGen, {}),
                       (vgen_b200.UNetSD_DreamVideo, {"temporal_adapter_list": ["feedforward"]})):
        assert _meta(cls, **ctor, **extra, fp8_linear=True).fp8_linear is True, cls
    # UNetSD_LoRA keeps the reference's exact signature (no **kwargs): the mode is set on the model
    lora = _meta(vgen_b200.UNetSD_LoRA, **ctor, use_lora=True, lora_rank=4)
    assert lora.fp8_linear is False
    lora.fp8_linear = True
    assert lora.fp8_linear is True
    lcm = _meta(vgen_b200.UNetSD_VideoLCM, config=dict(video_compositions=["text"], resolution=[448, 256]), **ctor,
                fp8_linear=True)
    assert lcm.fp8_linear is True


@pytest.mark.parametrize("bad", ["e4m3", 1, 0, None, "true"])
def test_unknown_value_raises(bad):
    with pytest.raises(ValueError):
        _meta(vgen_b200.UNetSD_T2VBase, **CASES["t2v_tiny"]["ctor"], fp8_linear=bad)
    m = _meta(vgen_b200.UNetSD_T2VBase, **CASES["t2v_tiny"]["ctor"])
    with pytest.raises(ValueError):
        m.fp8_linear = bad
    assert m.fp8_linear is False


def test_yaml_dict_reaches_the_keyword():
    """A config's UNet dict is splatted into the constructor: the keyword needs no engine change."""
    cfg = dict(CASES["t2v_tiny"]["ctor"], fp8_linear=True, some_training_key=0.3)
    assert _meta(vgen_b200.UNetSD_T2VBase, **cfg).fp8_linear is True


def test_toggling_drops_the_packed_arena():
    m = _meta(vgen_b200.UNetSD_T2VBase, **CASES["t2v_tiny"]["ctor"])
    m._packed = {"sentinel": 1}
    m.fp8_linear = False              # unchanged: nothing to re-pack
    assert m._packed == {"sentinel": 1}
    m.fp8_linear = True
    assert m._packed is None and m.fp8_linear


def test_weight_quantiser_per_channel():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(40, 64, generator=g, dtype=torch.float64) * torch.logspace(-3, 2, 40, dtype=torch.float64)[:, None]
    w[3] = 0
    q, s = ops.quantize_weight_e4m3(w)
    assert q.dtype == torch.uint8 and q.shape == w.shape and s.dtype == torch.float32 and s.shape == (40,)
    amax = w.float().abs().amax(1)
    assert s[3] == 1.0 and not q[3].any()
    keep = amax > 0
    assert torch.equal(s[keep], (amax[keep].double() / 448.0).float())
    deq = q.view(torch.float8_e4m3fn).float() * s[:, None]
    # every row's largest element is exactly representable (code 448), the rest within half an e4m3 step (2^-4 relative
    # for normals, plus the subnormal floor of 2^-10 * scale)
    assert torch.equal(deq.abs().amax(1)[keep], (448.0 * s)[keep])
    err = (deq - w.float()).abs()
    assert torch.all(err <= w.float().abs() * 2.0 ** -4 + s[:, None] * 2.0 ** -10)


def test_geglu_tile_choice():
    assert unet._geglu_bn_fp8(2560) == 128 and unet._geglu_bn_fp8(5120) == 128 and unet._geglu_bn_fp8(64 * 5) == 64
    with pytest.raises(ValueError):
        unet._geglu_bn_fp8(96)


def test_entry_points_declared():
    hdr = open(os.path.join(ROOT, "include", "vgen_b200.h")).read()
    for sym in ("vgen_quantize_rows_e4m3", "vgen_linear_fp8"):
        assert sym in lib.declared_symbols() and re.search(rf"\bint {sym}\(", hdr)
    assert "#define VGEN_B200_ABI_VERSION 2" in hdr


def test_graph_signature_carries_the_mode():
    class Owner:
        fp8_linear = False
    a = graph._mode(Owner())
    Owner.fp8_linear = True
    assert graph._mode(Owner()) != a
    assert graph._mode(object()) == a    # modules without the option key as fp16
