"""DreamVideo's evaluation metric on the host: the Pillow restatement against the installed Pillow, the product's
coefficient tables, the oracle against the reference's frozen transforms / features / scores, the parameter lists,
strict checkpoint loading in both formats, and the refusals."""
import os
import re

import numpy as np
import pytest
import torch
import torchvision.transforms as T
from PIL import Image

import vgen_b200
from oracle import metric_oracle as mo
from vgen_b200 import lib
from vgen_b200.clip import OpenAIClipModel, clip_spec, openai_cfg
from vgen_b200.clip_tokenizer import tokenize
from vgen_b200.dino import DINOHead, VisionTransformer, vit_small
from vgen_b200.metric import (ImageTransform, ResizePlan, calculate_metric, clip_transform, dino_transform, load_clip,
                              pillow_bicubic_coeffs, score_video)
from _metric import (FULL_CLIP, FULL_DINO, METRIC_CASES, TINY_CLIP, TINY_DINO, clip_state_dict, dino_state_dict,
                     load_case, load_spec, make_frames, make_targets, tensor_sha)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _merge_list(golden_dir, monkeypatch):
    monkeypatch.setenv("VGEN_CLIP_BPE", os.path.join(golden_dir, "clip_bpe_merges_head.txt.gz"))


# (in h, in w) -> (out h, out w): downscale, upscale, odd, non-square, an unchanged axis, and the metric's real chains
RESIZE_GRID = [((256, 256), (224, 224)), ((256, 256), (256, 256)), ((512, 512), (256, 256)), ((256, 256), (37, 301)),
               ((37, 53), (19, 71)), ((100, 80), (100, 33)), ((64, 48), (200, 48)), ((13, 7), (13, 29)),
               ((31, 1000), (13, 400)), ((480, 640), (224, 298)), ((7, 5), (224, 160))]
CHAIN_SIZES = [(256, 256), (512, 512), (240, 320), (300, 200), (180, 320), (1080, 1920), (225, 224), (97, 131)]


def _image(h, w, seed):
    r = np.random.default_rng(seed)
    a = r.integers(0, 256, (h, w, 3), dtype=np.uint8)
    a[: h // 2] = (a[: h // 2] // 85) * 85                     # flat areas and hard edges next to noise
    return a


@pytest.mark.parametrize("src,dst", RESIZE_GRID)
def test_pillow_restatement_is_bit_exact(src, dst):
    a = _image(*src, seed=sum(src) + sum(dst))
    want = np.asarray(Image.fromarray(a).resize((dst[1], dst[0]), Image.BICUBIC))
    assert np.array_equal(mo.pillow_resize(a, dst[1], dst[0]), want)


@pytest.mark.parametrize("n_in,n_out", [(256, 224), (512, 256), (37, 19), (13, 29), (1000, 400), (7, 224), (298, 224)])
def test_product_coefficients_match_the_restatement(n_in, n_out):
    b, k = pillow_bicubic_coeffs(n_in, n_out)
    b2, k2 = mo.coeffs(n_in, n_out)
    assert np.array_equal(b, b2) and np.array_equal(k, k2) and b.dtype == k.dtype == np.int32
    assert (k.sum(1) >= (1 << 22) - k.shape[1]).all() and (k.sum(1) <= (1 << 22) + k.shape[1]).all()


@pytest.mark.parametrize("hw", CHAIN_SIZES)
def test_transform_chains_match_torchvision(hw):
    """256 -> 224, 256 -> 256 -> 224, 512 -> 256 -> 224 and others, through PIL exactly as the script runs them."""
    a = _image(*hw, seed=hw[0] * 7 + hw[1])
    clip_tv = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(),
                         T.Normalize(mo.OPENAI_MEAN, mo.OPENAI_STD)])
    dino_tv = T.Compose([T.Resize(256, interpolation=3), T.CenterCrop(224), T.ToTensor(),
                         T.Normalize(mo.IMAGENET_MEAN, mo.IMAGENET_STD)])
    pil = T.ToPILImage()(torch.from_numpy(a).permute(2, 0, 1))
    assert torch.equal(clip_tv(pil), torch.from_numpy(mo.clip_transform(a)))
    assert torch.equal(dino_tv(pil), torch.from_numpy(mo.dino_transform(a)))


def test_resize_plan_tables():
    p = ResizePlan(256, 256, 256, 224, mo.IMAGENET_MEAN, mo.IMAGENET_STD)     # no resample: identity taps, crop offset 16
    assert (p.hb[:, 0] == np.arange(16, 240)).all() and (p.hb[:, 1] == 1).all() and (p.hk == 1 << 22).all()
    assert p.tile_rows == 16
    p = ResizePlan(512, 384, 256, 224, mo.IMAGENET_MEAN, mo.IMAGENET_STD)     # 512x384 -> 341x256 -> crop (58, 16)
    b, k = pillow_bicubic_coeffs(512, 341)
    assert np.array_equal(p.vb, b[58:282]) and np.array_equal(p.vk, k[58:282])
    assert p.tile_rows == max(int(p.vb[min(r + 15, 223), 0] + p.vb[min(r + 15, 223), 1] - p.vb[r, 0]) for r in range(0, 224, 16))
    with pytest.raises(ValueError, match="smaller than"):
        ResizePlan(100, 100, 64, 224, mo.OPENAI_MEAN, mo.OPENAI_STD)


# ---- the oracle against the reference's frozen calculate_metric -----------------------------------------------------------
@pytest.mark.parametrize("name", sorted(METRIC_CASES))
def test_oracle_against_reference(golden_dir, name):
    torch.set_grad_enabled(False)
    z = load_case(golden_dir, name)
    case = METRIC_CASES[name]
    assert np.array_equal(z["frames"], make_frames(name))
    rgb = [np.asarray(Image.fromarray(a, mode).convert("RGB")) for a, mode in make_targets(name)]
    assert len(rgb) == len(z["targets"]) and all(np.array_equal(a, b) for a, b in zip(rgb, z["targets"]))
    images = list(z["frames"]) + z["targets"]
    x_clip = torch.stack([torch.from_numpy(mo.clip_transform(a)) for a in images])
    x_dino = torch.stack([torch.from_numpy(mo.dino_transform(a)) for a in images])
    assert [tensor_sha(x) for x in x_clip] == list(z["clip_sha"])
    assert [tensor_sha(x) for x in x_dino] == list(z["dino_sha"])
    assert torch.equal(tokenize([case["prompt"]], truncate=False), torch.from_numpy(z["tokens"]).long())
    csd = clip_state_dict(load_spec(golden_dir, "clip_tiny"), 61)
    dsd = dino_state_dict(load_spec(golden_dir, "dino_tiny"), 62)
    f = len(z["frames"])
    img, txt = mo.clip_encode_image(csd, x_clip), mo.clip_encode_text(csd, torch.from_numpy(z["tokens"]).long())[0]
    dino = mo.dino_forward(dsd, x_dino, TINY_DINO["num_heads"])
    for mine, ref in ((img[:f], z["clip_frames"]), (img[f:], z["clip_targets"]), (txt, z["text"]), (dino[:f], z["dino_frames"]),
                      (dino[f:], z["dino_targets"])):
        assert mine.shape == ref.shape
        if ref.size:
            assert float((mine - torch.from_numpy(ref)).abs().max()) <= 1e-5 * float(np.abs(ref).max())
    s = mo.scores(img[:f], txt, img[f:], dino[:f], dino[f:])
    assert np.allclose(s, z["scores"], rtol=0, atol=1e-6)
    # non-vacuous: temporal consistency clearly below 1, and the cases' CLIP-T differ
    assert z["scores"][3] < 0.9
    other = load_case(golden_dir, [n for n in METRIC_CASES if n != name][0])["scores"]
    assert abs(other[0] - z["scores"][0]) > 0.02
    if not case["targets"]:
        assert z["scores"][1] == 0 and z["scores"][2] == 0


def test_scores_edge_cases():
    g = torch.randn(1, 8, dtype=torch.float64)
    s = mo.scores(g, torch.randn(8, dtype=torch.float64), None, torch.randn(1, 4, dtype=torch.float64), None)
    assert np.isnan(s[3]) and s[1] == 0 and s[2] == 0


# ---- parameter lists and loading ----------------------------------------------------------------------------------------
def test_specs_match_reference_digests(golden_dir):
    cf, ct, df, dt = (load_spec(golden_dir, w) for w in ("clip_full", "clip_tiny", "dino_full", "dino_tiny"))
    assert len(cf) == 302 and sum(torch.Size(s).numel() for _, s in cf) == 151277313
    assert len(df) == 150 and sum(torch.Size(s).numel() for _, s in df) == 21665664
    assert len(ct) == 62 and len(dt) == 30
    with torch.device("meta"):
        assert [(k, tuple(v.shape)) for k, v in vit_small().state_dict().items()] == df


def _openai_sd(spec, seed):
    return dict(clip_state_dict(spec, seed), input_resolution=torch.tensor(224), context_length=torch.tensor(77),
                vocab_size=torch.tensor(49408))


def test_openai_cfg_is_derived_from_shapes(golden_dir):
    for which, cfg in (("clip_tiny", TINY_CLIP), ("clip_full", FULL_CLIP)):
        spec = load_spec(golden_dir, which)
        with torch.device("meta"):
            sd = {k: torch.empty(s) for k, s in spec}
        assert openai_cfg(sd) == cfg
    sd = {"visual.layer1.0.conv1.weight": torch.zeros(1), "visual.attnpool.positional_embedding": torch.zeros(50, 1)}
    with pytest.raises(NotImplementedError, match="ModifiedResNet"):
        openai_cfg(sd)


class _Holder(torch.nn.Module):
    """A module tree carrying a state dict's names, scripted like OpenAI's released TorchScript checkpoints."""

    def __init__(self, sd):
        super().__init__()
        for k, v in sd.items():
            node = self
            *path, leaf = k.split(".")
            for comp in path:
                if not hasattr(node, comp):
                    node.add_module(comp, torch.nn.Module())
                node = getattr(node, comp)
            if v.dim() == 0 and k in ("input_resolution", "context_length", "vocab_size"):
                node.register_buffer(leaf, v.clone())
            else:
                node.register_parameter(leaf, torch.nn.Parameter(v.clone(), requires_grad=False))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x


@pytest.mark.parametrize("fmt", ["state_dict", "torchscript"])
def test_load_clip_strict_in_both_formats(golden_dir, tmp_path, fmt):
    sd = _openai_sd(load_spec(golden_dir, "clip_tiny"), 61)
    path = str(tmp_path / "ViT-tiny.pt")
    if fmt == "torchscript":
        torch.jit.save(torch.jit.script(_Holder({k: v.half() if v.is_floating_point() else v for k, v in sd.items()})), path)
        assert {"input_resolution", "context_length", "vocab_size"} <= set(torch.jit.load(path).state_dict())
    else:
        torch.save(sd, path)
    model, tf = load_clip(path, device="cpu")
    assert isinstance(model, OpenAIClipModel) and isinstance(tf, ImageTransform) and model.act == "quick_gelu"
    assert (tf.resize, tf.crop, tf.mean, tf.std) == (224, 224, mo.OPENAI_MEAN, mo.OPENAI_STD)
    assert model.cfg == TINY_CLIP
    got = model.state_dict()
    assert list(got) == [k for k, _ in clip_spec(TINY_CLIP)]
    assert all(torch.equal(got[k], sd[k]) for k in got)
    with pytest.raises(RuntimeError):
        model.load_state_dict({k: v for k, v in sd.items() if k != "ln_final.bias"}, strict=True)


def test_load_clip_by_name_reads_the_cache_and_never_downloads(golden_dir, tmp_path, monkeypatch):
    monkeypatch.setenv("HOME", str(tmp_path))
    with pytest.raises(FileNotFoundError, match=re.escape(os.path.join(str(tmp_path), ".cache", "clip", "ViT-B-32.pt"))):
        load_clip("ViT-B/32", device="cpu")
    os.makedirs(tmp_path / ".cache" / "clip")
    torch.save(_openai_sd(load_spec(golden_dir, "clip_tiny"), 3), tmp_path / ".cache" / "clip" / "ViT-B-32.pt")
    model, _ = load_clip("ViT-B/32", device="cpu")
    assert model.cfg == TINY_CLIP
    with pytest.raises(FileNotFoundError):
        load_clip(str(tmp_path / "missing.pt"), device="cpu")


def test_resnet_checkpoints_are_refused(tmp_path):
    with pytest.raises(NotImplementedError):
        load_clip("RN50", device="cpu")
    torch.save({"visual.layer1.0.conv1.weight": torch.zeros(64, 64, 1, 1), "text_projection": torch.zeros(512, 1024)},
               tmp_path / "rn.pt")
    with pytest.raises(NotImplementedError, match="ModifiedResNet"):
        load_clip(str(tmp_path / "rn.pt"), device="cpu")


def test_dino_strict_loading(golden_dir):
    spec = load_spec(golden_dir, "dino_tiny")
    m = VisionTransformer(**TINY_DINO, norm_layer=__import__("functools").partial(torch.nn.LayerNorm, eps=1e-6))
    sd = dino_state_dict(spec, 5)
    m.load_state_dict(sd, strict=True)
    assert m.eps == 1e-6 and all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    with pytest.raises(RuntimeError):
        m.load_state_dict({k: v for k, v in sd.items() if k != "norm.bias"}, strict=True)
    assert VisionTransformer(embed_dim=128, depth=1, num_heads=2).eps == 1e-5
    assert [k for k, _ in VisionTransformer(embed_dim=128, depth=1, num_heads=2, num_classes=5).state_dict().items()][-2:] == \
        ["head.weight", "head.bias"]


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_overlong_prompt_is_refused():
    long = " ".join(["word"] * 80)
    with pytest.raises(RuntimeError, match="too long for context length 77"):
        tokenize([long], truncate=False)
    assert tokenize([long]).shape == (1, 77)                # the open_clip default still truncates
    assert tokenize([" ".join(["word"] * 75)], truncate=False)[0, 76] != 0


@pytest.mark.parametrize("hw", [(256, 256), (224, 240), (240, 224)])
def test_off_grid_dino_input_is_refused(hw):
    with pytest.raises(NotImplementedError, match="patch grid"):
        vit_small()(torch.zeros(1, 3, *hw))


def test_dino_training_pieces_are_refused():
    m = VisionTransformer(embed_dim=128, depth=1, num_heads=2)
    for fn in (lambda: m.get_last_selfattention(None), lambda: m.get_intermediate_layers(None), lambda: DINOHead(384, 65536)):
        with pytest.raises(NotImplementedError):
            fn()
    with pytest.raises(NotImplementedError, match="head_dim"):
        VisionTransformer(embed_dim=96, num_heads=3)


def test_foreign_preprocess_objects_are_refused(tmp_path):
    tv = T.Compose([T.Resize(224), T.CenterCrop(224), T.ToTensor()])
    with pytest.raises(TypeError, match="clip_preprocess"):
        calculate_metric(str(tmp_path / "v.mp4"), "a dog", [], None, tv, None, dino_transform("cpu"))
    with pytest.raises(TypeError, match="dino_preprocess"):
        calculate_metric(str(tmp_path / "v.mp4"), "a dog", [], None, clip_transform(224, "cpu"), None, tv)
    with pytest.raises(TypeError):
        score_video(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), "a dog", [], None, tv, None, tv)


def test_cpu_tensors_are_refused():
    with pytest.raises(lib.VgenError, match="CUDA"):
        score_video(torch.zeros(2, 64, 64, 3, dtype=torch.uint8), "a dog", [], None, clip_transform(224, "cpu"), None,
                    dino_transform("cpu"))
    with pytest.raises(lib.VgenError, match="CUDA"):
        vit_small()(torch.zeros(1, 3, 224, 224))
    with pytest.raises(lib.VgenError, match="CUDA"):
        OpenAIClipModel(TINY_CLIP).encode_image_nhwc(torch.zeros(1, 224, 224, 3, dtype=torch.float16))


def test_lazy_exports():
    assert vgen_b200.calculate_metric is calculate_metric and vgen_b200.load_clip is load_clip
    assert vgen_b200.vit_small is vit_small and vgen_b200.dino_transform is dino_transform
    assert vgen_b200.score_video is score_video


def test_new_symbols_are_declared():
    hdr = open(os.path.join(ROOT, "include", "vgen_b200.h")).read()
    for sym in ("vgen_resize_bicubic_crop_normalize", "vgen_video_scores"):
        assert sym in lib.declared_symbols() and re.search(rf"\bint {sym}\(", hdr)
    assert "#define VGEN_B200_ABI_VERSION 2" in hdr


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "vgen_b200")
    for fn in ("metric.py", "dino.py", "clip.py", "clip_tokenizer.py", "ops.py"):
        src = open(os.path.join(pkg, fn)).read()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), fn
        assert "_metric" not in re.findall(r"^\s*(?:from|import)\s+(\S+)", src, re.M), fn
