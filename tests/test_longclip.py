"""Long clips on the host: the oracle against the reference's frozen outputs at frame counts past 32 and 64, the parameter
lists against the reference's, and the CPU refusal at a long clip."""
import os

import numpy as np
import pytest
import torch

from oracle import synth, vgen_oracle as vo
from vgen_b200 import lib
from _longclip import LONG_CASES, build_product, load_spec, make_inputs, oracle_call, product_call, state_dict


@pytest.mark.parametrize("name", sorted(LONG_CASES))
def test_oracle_against_reference_outputs(golden_dir, name):
    torch.set_grad_enabled(False)
    case = LONG_CASES[name]
    inp = make_inputs(case)
    out = oracle_call(case, state_dict(golden_dir, name), inp)
    ref = torch.from_numpy(np.load(os.path.join(golden_dir, f"longclip_{name}.npz"))["out"])
    assert out.shape == ref.shape and out.shape[2] == case["f"]
    assert float((out - ref).abs().max() / ref.abs().max()) < 2e-5


def test_oracle_ddim_loop_against_reference(golden_dir):
    """The 4-step CFG DDIM loop at 80 frames, restated by the oracle, against the reference's DiffusionDDIM."""
    torch.set_grad_enabled(False)
    name = "t2v_b2_f80"
    case = LONG_CASES[name]
    inp = make_inputs(case)
    sd = state_dict(golden_dir, name)
    fn = lambda xt, t, **k: vo.unet_t2v_forward(sd, xt, t, **k)  # noqa: E731
    lat = vo.ddim_sample_loop(inp["x"].clone(), fn, [{"y": inp["y"]}, {"y": inp["y_neg"]}],
                              vo.make_betas("cosine", 1000, True, cosine_s=0.008), case["ddim"]["guide_scale"], case["ddim"]["steps"])
    ref = torch.from_numpy(np.load(os.path.join(golden_dir, f"longclip_{name}.npz"))["ddim_latent"])
    assert float((lat - ref).abs().max() / ref.abs().max()) < 1e-4


@pytest.mark.parametrize("name", sorted(LONG_CASES))
def test_spec_equals_reference_and_loads_strictly(golden_dir, name):
    spec = load_spec(golden_dir, name)             # checks the digest
    m = build_product(LONG_CASES[name])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == spec
    m.load_state_dict(synth.state_dict(spec, seed=1), strict=True)


def test_cpu_forward_at_80_frames_raises(golden_dir):
    """No CPU path exists at any frame count: a long clip on the host is refused like a short one."""
    case = LONG_CASES["t2v_b2_f80"]
    m = build_product(case)
    with pytest.raises(lib.VgenError, match="CUDA"):
        product_call(case, m, make_inputs(case))
