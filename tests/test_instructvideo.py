"""InstructVideo (UNetSD_LoRA, DiffusionDDIMReward, FrozenOpenCLIPEmbedderZero) on the host: parameter specs against the
reference's, strict loading of LoRA and base checkpoints, registry builds of the released eval dicts, refusals, the
unmerged state and the merge, the sampler's step list, the training-only methods, and the oracle against the reference's
frozen outputs."""
import inspect
import os

import numpy as np
import pytest
import torch

import vgen_b200
from vgen_b200 import arch, registry
from _instructvideo import (DDIM20_STEPS, IV_CASES, RELEASED, RELEASED_COUNTS, RELEASED_DIFFUSION, build_product, load_spec,
                            make_inputs, oracle_call, product_spec, reference_digest, spec_digest, weights)


@pytest.mark.parametrize("name", sorted(RELEASED))
def test_released_spec_equals_reference(golden_dir, name):
    d = spec_digest(product_spec(RELEASED[name]))
    assert (d["tensors"], d["parameters"]) == RELEASED_COUNTS[name]
    assert d == reference_digest(golden_dir, name)


def test_without_lora_spec_is_t2vbase():
    ctor = {k: v for k, v in RELEASED["released_base"].items() if "lora" not in k}
    with torch.device("meta"):
        base = vgen_b200.UNetSD_T2VBase(**ctor)
    assert product_spec(RELEASED["released_base"]) == [(k, tuple(v.shape)) for k, v in base.state_dict().items()]


def test_lora_pairs_sit_after_each_attention():
    """66 attentions x {q, k, v, out} x {down, up}, each group right after its attention's to_out.0.bias."""
    spec = product_spec(RELEASED["released_lora"])
    names = [k for k, _ in spec]
    lora = [k for k in names if "_lora." in k]
    assert len(lora) == 528 and sum(int(np.prod(s)) for k, s in spec if "_lora." in k) == 1661440
    for i, k in enumerate(names):
        if k.endswith("to_out.0.bias"):
            att = k[:-len("to_out.0.bias")]
            assert names[i + 1:i + 9] == [f"{att}{m}.{p}_linear.weight" for m, _ in arch.LORA_SITES for p in ("down", "up")]
    shapes = dict(spec)
    # the init block's temporal transformer: 512 wide (8 heads of 64) inside a 320-channel block; attn2 is a self-attention
    p = "input_blocks.0.1.transformer_blocks.0.attn2."
    assert shapes[p + "to_k_lora.down_linear.weight"] == (4, 512) and shapes[p + "to_out_lora.up_linear.weight"] == (512, 4)
    # a decoder cross-attention reads the 1024-wide context
    assert shapes["output_blocks.3.1.transformer_blocks.0.attn2.to_k_lora.down_linear.weight"] == (4, 1024)


@pytest.mark.parametrize("name", sorted(IV_CASES))
def test_tiny_spec_equals_reference_and_loads_strictly(golden_dir, name):
    ref = load_spec(golden_dir, name)          # checks the digest
    m = build_product(IV_CASES[name])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == ref
    m.load_state_dict(weights(ref, 1), strict=True)


def test_strict_loading_tells_the_checkpoint_shapes_apart():
    lora_case, base_case = IV_CASES["iv_lora_tiny"], IV_CASES["iv_nolora_tiny"]
    lora_sd = weights(product_spec(lora_case["ctor"]), 3)
    base_sd = {k: v for k, v in lora_sd.items() if "_lora." not in k}
    build_product(lora_case).load_state_dict(lora_sd, strict=True)
    build_product(base_case).load_state_dict(base_sd, strict=True)
    with pytest.raises(RuntimeError, match="Missing"):
        build_product(lora_case).load_state_dict(base_sd, strict=True)
    with pytest.raises(RuntimeError, match="Unexpected"):
        build_product(base_case).load_state_dict(lora_sd, strict=True)


@pytest.mark.parametrize("name", sorted(RELEASED))
def test_registry_builds_released_eval_dicts(golden_dir, name):
    """All seven configs/instructvideo/eval configs: four with use_lora True, three with False, otherwise the same dicts."""
    MODEL, DIFFUSION, _ = vgen_b200.register(force_local=True)
    assert MODEL.get("UNetSD_LoRA") is vgen_b200.UNetSD_LoRA
    with torch.device("meta"):
        m = MODEL.build(dict(RELEASED[name], type="UNetSD_LoRA"))
    assert type(m) is vgen_b200.UNetSD_LoRA and m.use_lora == RELEASED[name]["use_lora"] and m.cfg_batch
    assert spec_digest([(k, tuple(v.shape)) for k, v in m.state_dict().items()]) == reference_digest(golden_dir, name)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == arch.unet_spec(m.plan)


def test_refusals():
    ctor = IV_CASES["iv_lora_tiny"]["ctor"]
    for rank in (None, 0, -1):
        with pytest.raises(ValueError, match="lora_rank"):
            vgen_b200.UNetSD_LoRA(**dict(ctor, lora_rank=rank))
    vgen_b200.UNetSD_LoRA(**dict(ctor, use_lora=False, lora_rank=None))      # no LoRA: the rank is not read
    with pytest.raises(NotImplementedError, match="head_dim"):
        vgen_b200.UNetSD_LoRA(**dict(ctor, head_dim=32))
    with pytest.raises(NotImplementedError, match="temporal_attn_times"):
        vgen_b200.UNetSD_LoRA(**dict(ctor, temporal_attn_times=2))
    with pytest.raises(TypeError):
        vgen_b200.UNetSD_LoRA(**dict(ctor, zero_y=torch.zeros(1, 1, 1024)))  # the reference takes no **kwargs
    m = vgen_b200.UNetSD_LoRA(**ctor)
    m._check_x = lambda x, t: None
    with pytest.raises(ValueError, match="needs y"):
        type(m).forward.__wrapped_eager__(m, torch.zeros(1, 4, 3, 8, 12), torch.zeros(1, dtype=torch.long), None)


def test_constructor_matches_the_reference():
    sig = inspect.signature(vgen_b200.UNetSD_LoRA.__init__)
    assert list(sig.parameters)[-3:] == ["use_lora", "lora_rank", "lora_alpha"]
    assert sig.parameters["in_dim"].default == 7 and sig.parameters["out_dim"].default == 6
    assert not any(p.kind is inspect.Parameter.VAR_KEYWORD for p in sig.parameters.values())
    fwd = list(inspect.signature(vgen_b200.UNetSD_LoRA.forward).parameters)
    assert fwd == ["self", "x", "t", "y", "fps", "video_mask", "focus_present_mask", "prob_focus_present", "mask_last_frame_num"]


@pytest.mark.parametrize("alpha", [None, 8])
def test_state_dict_stays_unmerged_and_the_merge_is_exact(alpha):
    case = IV_CASES["iv_lora_tiny"]
    m = vgen_b200.UNetSD_LoRA(**dict(case["ctor"], lora_alpha=alpha))
    sd = weights(product_spec(case["ctor"]), 5)
    m.load_state_dict(sd, strict=True)
    merged = m.merged_state_dict()
    after = m.state_dict()
    assert list(after) == list(sd) and all(torch.equal(after[k], sd[k]) for k in sd)
    assert sum(p.numel() for p in m.parameters()) == sum(v.numel() for v in sd.values())
    s = 1.0 if alpha is None else alpha / 4
    assert m.lora_scale == s
    base_keys = [k for k in sd if "_lora." not in k]
    assert list(merged) == base_keys
    changed = 0
    for k in base_keys:
        att = k.rsplit(".", 2)[0] if k.endswith("to_out.0.weight") else k.rsplit(".", 1)[0]
        mod = {"to_q": "to_q_lora", "to_k": "to_k_lora", "to_v": "to_v_lora", "to_out": "to_out_lora"}.get(att.rsplit(".", 1)[-1])
        if mod is None or not k.endswith("weight"):
            assert torch.equal(merged[k], sd[k]), k
            continue
        a = att.rsplit(".", 1)[0]
        want = (sd[k].double() + s * sd[f"{a}.{mod}.up_linear.weight"].double() @ sd[f"{a}.{mod}.down_linear.weight"].double())
        assert merged[k].dtype == torch.float32 and torch.equal(merged[k], want.float()), k
        # get_lora_merged_model's own fp32 arithmetic (inference_instructvideo_entrance.py:340) agrees to an ulp or two
        fp32 = sd[k] + s * torch.mm(sd[f"{a}.{mod}.up_linear.weight"], sd[f"{a}.{mod}.down_linear.weight"])
        torch.testing.assert_close(merged[k], fp32, rtol=3e-7, atol=3e-7)
        changed += 1
    assert changed == 4 * 2 * sum(1 for k in sd if k.endswith("attn1.to_q.weight"))


def test_released_diffusion_builds_the_native_sampler():
    _, DIFFUSION, _ = vgen_b200.register(force_local=True)
    d = DIFFUSION.build(RELEASED_DIFFUSION)
    assert type(d) is vgen_b200.DiffusionDDIMReward and isinstance(d, vgen_b200.DiffusionDDIM)
    assert d.ddim_steps(20).tolist() == DDIM20_STEPS
    assert d.ddim_steps(50).tolist() == list(range(981, 0, -20))   # the ddim50 config's list


@pytest.mark.parametrize("method", ["ddim_sample_loop_partial", "ddim_sample_gradient", "ddim_sample_with_logprob",
                                    "ddim_sample_loop_with_logprob", "loss"])
def test_reward_training_methods_raise(method):
    d = vgen_b200.DiffusionDDIMReward(**{k: v for k, v in RELEASED_DIFFUSION.items() if k != "type"})
    with pytest.raises(NotImplementedError, match="reward fine-tuning is not supported"):
        getattr(d, method)(None, None)


def test_embedder_zero_is_the_text_tower():
    vgen_b200.register(force_local=True)
    cls = registry.EMBEDDER.get("FrozenOpenCLIPEmbedderZero")
    assert cls is vgen_b200.FrozenOpenCLIPEmbedderZero and issubclass(cls, vgen_b200.FrozenOpenCLIPEmbedder)
    assert cls.forward is vgen_b200.FrozenOpenCLIPEmbedder.forward and not cls.VISUAL
    sig = inspect.signature(cls.__init__).parameters
    assert list(sig) == ["self", "pretrained", "vit_resolution", "arch", "device", "max_length", "freeze", "layer"]
    assert sig["pretrained"].default is inspect.Parameter.empty and sig["layer"].default == "last"
    for name in ("white_image", "zero_feature"):
        with pytest.raises(NotImplementedError, match="not provided"):
            getattr(cls, name).fget(cls)
    with pytest.raises(NotImplementedError, match="not provided"):
        cls.forward_image(cls, None)


@pytest.mark.parametrize("name", sorted(IV_CASES))
def test_oracle_against_reference_outputs(golden_dir, name):
    """The unmerged oracle against the reference class's outputs (merged by get_lora_merged_model for lora_alpha 8),
    frozen under two weight seeds."""
    torch.set_grad_enabled(False)
    case = IV_CASES[name]
    spec = load_spec(golden_dir, name)
    inp = make_inputs(case)
    gold = np.load(os.path.join(golden_dir, name + ".npz"))["out"]
    pin = np.load(os.path.join(golden_dir, "instructvideo_pin.npz"))[f"{name}_seed83"]
    for seed, ref in ((case["seed"], gold), (83, pin)):
        out = oracle_call(case, weights(spec, seed), inp)
        ref = torch.from_numpy(ref)
        assert float((out - ref).abs().max() / ref.abs().max()) < 2e-5, seed
