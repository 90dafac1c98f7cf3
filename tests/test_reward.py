"""InstructVideo's segmental HPSv2 reward on the CPU: the oracle against the reference's frozen values, the TSN draw, the
resize taps against F.interpolate, the size rule, the refusals, checkpoint loading and the C ABI surface."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vgen_b200
from oracle import reward_oracle as ro
from vgen_b200 import lib, reward
from vgen_b200.clip import ClipModel
from vgen_b200.reward import BilinearPlan, SegmentalReward, bilinear_taps, load_hps, segment_indices
from _reward import REWARD_CASES, SUB, TINY_HPS, hps_state_dict, load_case, load_spec, make_latents, vae_product

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


@pytest.mark.parametrize("name", sorted(REWARD_CASES))
def test_oracle_against_reference(golden_dir, name):
    torch.set_grad_enabled(False)
    case, z = REWARD_CASES[name], load_case(golden_dir, name)
    idx = torch.from_numpy(z["idx"])
    b, s = idx.shape
    assert (b, s) == (case["b"], case["segments"])
    video = ro.decode(vae_product()[2], make_latents(name))
    assert video.shape[-2:] == (8 * case["h"], 8 * case["w"])
    pre = ro.preprocess(video, case["antialias"])
    sel = pre[torch.arange(b)[:, None], idx].reshape(b * s, *pre.shape[2:])
    assert _rel(sel[:, :, ::SUB, ::SUB], torch.from_numpy(z["pre_sub"])) < 1e-5
    assert np.allclose(sel.double().sum((1, 2, 3)).numpy(), z["pre_sum"], rtol=1e-5, atol=1e-2)
    sd = hps_state_dict(load_spec(golden_dir, "hps_tiny"))
    img, txt = ro.features(sd, sel, torch.from_numpy(z["tokens"]).long(), TINY_HPS["vision_cfg"]["head_width"],
                           TINY_HPS["text_cfg"]["heads"])
    assert _rel(img, torch.from_numpy(z["image_features"])) < 1e-5
    assert _rel(txt, torch.from_numpy(z["text_features"])) < 1e-5
    got = ro.reward_scores(img, txt, idx, case["f"], case["tar"])
    assert float((got - torch.from_numpy(z["reward_scores"])).abs().max()) < 1e-6


def test_specs_match_reference_digests(golden_dir):
    for which in ("hps_tiny", "hps_full", "vae_tiny"):
        load_spec(golden_dir, which)


@pytest.mark.parametrize("name", sorted(n for n, c in REWARD_CASES.items() if c["selection"] == "TSN"))
def test_segment_indices_reproduce_the_reference_draw(golden_dir, name):
    case, z = REWARD_CASES[name], load_case(golden_dir, name)
    torch.manual_seed(case["seed"])
    got = segment_indices(case["b"], case["f"], case["segments"], "TSN")
    assert torch.equal(got, torch.from_numpy(z["idx"]))
    g = torch.Generator().manual_seed(case["seed"])
    assert torch.equal(segment_indices(case["b"], case["f"], case["segments"], "TSN", g), got)


def test_fixed_first_indices(golden_dir):
    z = load_case(golden_dir, "fixed_first")
    assert torch.equal(segment_indices(2, 16, 8, "fixed_first"), torch.from_numpy(z["idx"]))
    assert segment_indices(3, 16, 4, "fixed_first").tolist() == [[0, 4, 8, 12]] * 3


def test_tsn_indices_stay_in_their_segments():
    idx = segment_indices(64, 17, 4, "TSN", torch.Generator().manual_seed(3))
    span = 17 // 4
    assert ((idx // span) == torch.arange(4)[None]).all() and idx.max() < 16


@pytest.mark.parametrize("antialias", [False, True])
@pytest.mark.parametrize("n_in,n_out", [(256, 224), (224, 224), (96, 224), (448, 392), (1024, 224), (300, 224), (7, 224),
                                        (640, 373)])
def test_bilinear_taps_match_interpolate(n_in, n_out, antialias):
    x = torch.rand(2, 3, n_in, 5, generator=torch.Generator().manual_seed(n_in))         # fp32: the weights are fp32 math
    want = F.interpolate(x, size=(n_out, 5), mode="bilinear", align_corners=False, antialias=antialias).double()
    x = x.double()
    bounds, w = bilinear_taps(n_in, n_out, antialias)
    got = torch.zeros_like(want)
    for o in range(n_out):
        for t in range(int(bounds[o, 1])):
            got[:, :, o] += float(w[o, t]) * x[:, :, min(int(bounds[o, 0]) + t, n_in - 1)]
    assert float((got - want).abs().max()) < 2e-7


def test_plan_tile_rows_cover_the_windows():
    for h, aa in ((256, False), (1024, True), (96, True), (300, False)):
        p = BilinearPlan(h, h, 224, 224, aa)
        for r in range(0, 224, 16):
            last = min(r + 16, 224) - 1
            assert p.vb[last].sum() - p.vb[r, 0] <= p.tile_rows


@pytest.mark.parametrize("hw,ok", [((256, 256), True), ((96, 96), True), ((512, 512), True), ((256, 448), False),
                                   ((448, 256), False), ((225, 224), False)])
def test_size_rule(hw, ok):
    assert ro.resized_size(*hw, 224) == reward.resized_size(*hw, 224)
    scorer = SegmentalReward(ClipModel(TINY_HPS))
    if ok:
        assert (scorer.plan(*hw).oh, scorer.plan(*hw).ow) == (224, 224)
    else:
        with pytest.raises(ValueError, match="224x224"):
            scorer.plan(*hw)


def test_refusals():
    with pytest.raises(ValueError, match="cannot be split"):
        segment_indices(1, 3, 4, "TSN")
    with pytest.raises(ValueError, match="selects 6 frames, not 5"):
        segment_indices(1, 16, 5, "fixed_first")
    with pytest.raises(ValueError, match="needs selection_method='TSN'"):
        segment_indices(1, 16, 4, "fixed_first", exponential_TSN=True)
    with pytest.raises(ValueError, match="selection_method must be"):
        segment_indices(1, 16, 4, "uniform")
    hps = ClipModel(TINY_HPS)
    with pytest.raises(ValueError, match="needs selection_method='TSN'"):
        SegmentalReward(hps, selection_method="fixed_first")
    with pytest.raises(ValueError, match="selection_method must be"):
        SegmentalReward(hps, selection_method="uniform")
    SegmentalReward(hps, selection_method="fixed_first", exponential_TSN=False)
    with pytest.raises(ValueError, match="needs the autoencoder"):
        SegmentalReward(hps).score_latents(["a"], torch.zeros(1, 4, 4, 2, 2))
    with pytest.raises(lib.VgenError, match="CUDA"):
        SegmentalReward(hps).score_rgb8(["a"], torch.zeros(1, 4, 8, 8, 3, dtype=torch.uint8))


def test_defaults_are_the_training_config():
    s = SegmentalReward(ClipModel(TINY_HPS))
    assert (s.segments, s.selection_method, s.exponential_TSN, s.lambda_TAR, s.scale_factor, s.antialias) == \
        (4, "TSN", True, 1.0, 0.18215, False)


@pytest.mark.parametrize("fmt", ["wrapped", "plain"])
def test_load_hps_is_strict_in_both_formats(golden_dir, tmp_path, monkeypatch, fmt):
    monkeypatch.setitem(reward.ARCHS, "ViT-H-14", TINY_HPS)
    sd = hps_state_dict(load_spec(golden_dir, "hps_tiny"))
    path = tmp_path / "HPS_v2.pt"
    torch.save({"state_dict": sd} if fmt == "wrapped" else sd, path)
    m = load_hps(str(path), device="cpu")
    assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())
    torch.save({k: v for k, v in sd.items() if k != "visual.proj"}, path)
    with pytest.raises(RuntimeError, match="visual.proj"):
        load_hps(str(path), device="cpu")


def test_lazy_exports():
    assert vgen_b200.SegmentalReward is SegmentalReward and vgen_b200.load_hps is load_hps
    assert vgen_b200.segment_indices is segment_indices


def test_new_symbols_are_declared():
    hdr = open(os.path.join(ROOT, "include", "vgen_b200.h")).read()
    for sym in ("vgen_reward_frames", "vgen_segment_reward"):
        assert sym in lib.declared_symbols() and re.search(rf"\bint {sym}\(", hdr)


def test_product_never_imports_the_oracle():
    src = open(os.path.join(ROOT, "vgen_b200", "reward.py")).read()
    assert not re.search(r"^\s*(from|import)\s+(oracle|_reward)\b", src, re.M)
