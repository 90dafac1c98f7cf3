"""DreamVideo's evaluation metric on the H100: the resize kernel bit-identical to torchvision + Pillow, QuickGELU and the
score kernel against PyTorch, the tiny models against the reference's frozen features, full-size ViT-B/32 and ViT-S/16
against the fp32 oracle, calculate_metric against the reference's scores, CUDA-graph replay, and the kernels a scoring
launches.

Model gates are the project's existing ones (tests/test_gpu_sketch.py): ours must be no further from the fp32 truth than
1.25x the yardstick's error + 2e-4, under a relative-L2 cap.  The CLIP yardstick is the oracle with fp16 weights and
activations, which is what clip.load runs on a GPU; the DINO yardstick is the oracle under fp16 autocast."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torchvision.transforms as T
from PIL import Image

from oracle import metric_oracle as mo
from vgen_b200 import graph, ops
from vgen_b200.clip import OpenAIClipModel
from vgen_b200.dino import VisionTransformer, vit_small
from vgen_b200.metric import calculate_metric, clip_transform, dino_transform, load_clip, score_video
from _metric import (FULL_CLIP, FULL_DINO, METRIC_CASES, QK_GAIN, TINY_CLIP, TINY_DINO, clip_state_dict, dino_state_dict,
                     load_case, load_spec, make_frames, tensor_sha)
from test_metric import CHAIN_SIZES, RESIZE_GRID, _image  # noqa: F401

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _merge_list(golden_dir, monkeypatch):
    monkeypatch.setenv("VGEN_CLIP_BPE", os.path.join(golden_dir, "clip_bpe_merges_head.txt.gz"))
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def _tv(kind):
    if kind == "clip":
        return T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(),
                          T.Normalize(mo.OPENAI_MEAN, mo.OPENAI_STD)])
    return T.Compose([T.Resize(256, interpolation=3), T.CenterCrop(224), T.ToTensor(), T.Normalize(mo.IMAGENET_MEAN, mo.IMAGENET_STD)])


# ---- kernels -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["clip", "dino"])
@pytest.mark.parametrize("hw", CHAIN_SIZES + [src for src, _ in RESIZE_GRID if min(src) >= 5])
def test_resize_kernel_is_bit_identical_to_torchvision(kind, hw):
    imgs = np.stack([_image(*hw, seed=s) for s in range(3)])
    tf = clip_transform() if kind == "clip" else dino_transform()
    got = tf.batch(torch.from_numpy(imgs).cuda(), out_f32=True).cpu()
    want = torch.stack([_tv(kind)(Image.fromarray(a)) for a in imgs])
    assert got.shape == want.shape and torch.equal(got, want)
    half = tf.batch(torch.from_numpy(imgs).cuda()).cpu()
    assert torch.equal(half, want.half().permute(0, 2, 3, 1))
    assert torch.equal(tf(imgs[0]).cpu(), want[0]) and torch.equal(tf(Image.fromarray(imgs[1])).cpu(), want[1])


@pytest.mark.parametrize("name", sorted(METRIC_CASES))
def test_resize_kernel_reproduces_the_frozen_tensors(golden_dir, name):
    z = load_case(golden_dir, name)
    for kind, tf in (("clip", clip_transform()), ("dino", dino_transform())):
        got = list(tf.batch(torch.from_numpy(z["frames"]).cuda(), out_f32=True))
        got += list(tf.images(z["targets"], "cuda", out_f32=True)) if z["targets"] else []
        assert [tensor_sha(x) for x in got] == list(z[f"{kind}_sha"])


def test_quick_gelu_matches_torch():
    x = (torch.randn(1 << 20, generator=torch.Generator().manual_seed(0)) * 4).half().cuda()
    y = ops.eltwise("quick_gelu", x)
    xf = x.float()
    want = xf * torch.sigmoid(1.702 * xf)
    assert float((y.float() - want).abs().max()) <= float((want.half().float() - want).abs().max()) * 2 + 1e-7


@pytest.mark.parametrize("f,t,e,d", [(32, 6, 512, 384), (16, 0, 512, 384), (1, 3, 64, 128), (1, 0, 768, 768), (2, 1, 8, 8),
                                     (64, 12, 1024, 384)])
def test_score_kernel_matches_fp64(f, t, e, d):
    g = torch.Generator().manual_seed(f * 100 + t)
    mk = lambda *s: (torch.randn(*s, generator=g) + 0.5).cuda()  # noqa: E731
    cf, tx, df = mk(f, e), mk(e), mk(f, d)
    ct, dt = (mk(t, e), mk(t, d)) if t else (None, None)
    got = ops.video_scores(cf, tx, ct, df, dt).cpu().double()
    want = torch.tensor(mo.scores(cf.double().cpu(), tx.double().cpu(), None if ct is None else ct.double().cpu(),
                                  df.double().cpu(), None if dt is None else dt.double().cpu()), dtype=torch.float64)
    if f == 1:
        assert torch.isnan(got[3]) and torch.isnan(want[3])
        got, want = got[:3], want[:3]
    assert float((got - want).abs().max()) < 1e-5
    if t == 0:
        assert got[1] == 0 and got[2] == 0


# ---- tiny models against the reference ----------------------------------------------------------------------------------
def _clip(spec_which, seed, tmp_path):
    sd = clip_state_dict(load_spec(os.path.join(ROOT, "tests", "golden"), spec_which), seed,
                         qk_gain=1.0 if spec_which == "clip_full" else QK_GAIN)
    path = tmp_path / f"clip_{spec_which}_{seed}.pt"
    torch.save(dict(sd, input_resolution=torch.tensor(224), context_length=torch.tensor(77), vocab_size=torch.tensor(49408)), path)
    model, tf = load_clip(str(path))
    return model, tf, {k: v.cuda() for k, v in sd.items()}


def _dino(kw, spec_which, seed):
    import functools
    sd = dino_state_dict(load_spec(os.path.join(ROOT, "tests", "golden"), spec_which), seed,
                         qk_gain=1.0 if spec_which == "dino_full" else QK_GAIN)
    m = VisionTransformer(**kw, norm_layer=functools.partial(torch.nn.LayerNorm, eps=1e-6))
    m.load_state_dict(sd, strict=True)
    return m.eval().cuda(), {k: v.cuda() for k, v in sd.items()}


def _gate(tag, mine, truth, yard, cap):
    e_mine, e_yard = _rel_l2(mine, truth), _rel_l2(yard, truth)
    print(f"{tag}: ours vs fp32 truth {e_mine:.3e}; yardstick {e_yard:.3e}")
    assert e_mine < cap
    assert e_mine < 1.25 * e_yard + 2e-4


def _clip_yard(csd, fn, x):
    return fn({k: v.half() for k, v in csd.items()}, x.half() if x.is_floating_point() else x).float()


def _dino_yard(dsd, x, heads):
    with torch.autocast("cuda", dtype=torch.float16):
        return mo.dino_forward(dsd, x, heads).float()


@pytest.mark.parametrize("name", sorted(METRIC_CASES))
def test_tiny_models_against_reference_features(golden_dir, name, tmp_path):
    torch.set_grad_enabled(False)
    z = load_case(golden_dir, name)
    clip_m, ctf, csd = _clip("clip_tiny", 61, tmp_path)
    dino_m, dsd = _dino(TINY_DINO, "dino_tiny", 62)
    dtf = dino_transform()
    frames = torch.from_numpy(z["frames"]).cuda()
    f = frames.shape[0]
    cx = ctf.batch(frames, out_f32=True)
    dx = dtf.batch(frames, out_f32=True)
    if z["targets"]:
        cx = torch.cat([cx, ctf.images(z["targets"], "cuda", out_f32=True)])
        dx = torch.cat([dx, dtf.images(z["targets"], "cuda", out_f32=True)])
    tokens = torch.from_numpy(z["tokens"]).long()
    truth = {"img": torch.from_numpy(np.concatenate([z["clip_frames"], z["clip_targets"]])).cuda(),
             "txt": torch.from_numpy(z["text"]).cuda(),
             "dino": torch.from_numpy(np.concatenate([z["dino_frames"], z["dino_targets"]])).cuda()}
    mine = {"img": clip_m.encode_image(cx), "txt": clip_m.encode_text(tokens)[0], "dino": dino_m(dx)}
    nhwc = {"img": clip_m.encode_image_nhwc(torch.cat([ctf.batch(frames)] + ([ctf.images(z["targets"], "cuda")] if z["targets"] else []))),
            "dino": dino_m.forward_nhwc(torch.cat([dtf.batch(frames)] + ([dtf.images(z["targets"], "cuda")] if z["targets"] else [])))}
    assert torch.equal(nhwc["img"], mine["img"]) and torch.equal(nhwc["dino"], mine["dino"])
    yard = {"img": _clip_yard(csd, mo.clip_encode_image, cx), "txt": _clip_yard(csd, mo.clip_encode_text, tokens.cuda())[0],
            "dino": _dino_yard(dsd, dx, TINY_DINO["num_heads"])}
    assert _rel_l2(mo.clip_encode_image(csd, cx), truth["img"]) < 1e-5
    for k in truth:
        assert mine[k].dtype == torch.float32 and mine[k].shape == truth[k].shape
        _gate(f"{name} {k}", mine[k], truth[k], yard[k], 5e-3)
    assert f == len(z["clip_frames"])


# ---- full size ----------------------------------------------------------------------------------------------------------
def test_fullsize_against_fp32_oracle(golden_dir, tmp_path):
    torch.set_grad_enabled(False)
    clip_m, ctf, csd = _clip("clip_full", 71, tmp_path)
    dino_m, dsd = _dino(FULL_DINO, "dino_full", 72)
    assert clip_m.cfg == FULL_CLIP
    frames = torch.from_numpy(np.concatenate([make_frames(n) for n in ("square_targets",)] * 4)).cuda()     # 16 frames
    cx, dx = ctf.batch(frames, out_f32=True), dino_transform().batch(frames, out_f32=True)
    tokens = torch.from_numpy(np.concatenate([load_case(golden_dir, n)["tokens"] for n in sorted(METRIC_CASES)])).long()
    _gate("ViT-B/32 image", clip_m.encode_image_nhwc(ctf.batch(frames)), mo.clip_encode_image(csd, cx),
          _clip_yard(csd, mo.clip_encode_image, cx), 6e-3)
    _gate("ViT-B/32 text", clip_m.encode_text(tokens), mo.clip_encode_text(csd, tokens.cuda()),
          _clip_yard(csd, mo.clip_encode_text, tokens.cuda()), 6e-3)
    _gate("ViT-S/16", dino_m.forward_nhwc(dino_transform().batch(frames)), mo.dino_forward(dsd, dx, FULL_DINO["num_heads"]),
          _dino_yard(dsd, dx, FULL_DINO["num_heads"]), 6e-3)


# ---- the metric end to end ----------------------------------------------------------------------------------------------
class _Capture:
    frames = {}

    def __init__(self, path):
        self._it = iter(self.frames[path])

    def read(self):
        f = next(self._it, None)
        return (f is not None), (None if f is None else np.ascontiguousarray(f[..., ::-1]))


@pytest.mark.parametrize("name", sorted(METRIC_CASES))
def test_calculate_metric_matches_reference_scores(golden_dir, name, tmp_path, monkeypatch, capsys):
    import cv2
    z = load_case(golden_dir, name)
    _Capture.frames = {name: list(z["frames"])}
    monkeypatch.setattr(cv2, "VideoCapture", _Capture)
    files = []
    for j, a in enumerate(z["targets"]):
        files.append(str(tmp_path / f"target{j}.png"))
        Image.fromarray(a).save(files[-1])
    clip_m, ctf, _ = _clip("clip_tiny", 61, tmp_path)
    dino_m, _ = _dino(TINY_DINO, "dino_tiny", 62)
    got = calculate_metric(name, METRIC_CASES[name]["prompt"], files, clip_m, ctf, dino_m, dino_transform())
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert line.startswith("CLIP-T: ") and "TemporalConsistency: " in line
    print(name, got, z["scores"].tolist())
    assert len(got) == 4 and float(np.max(np.abs(np.asarray(got, np.float64) - z["scores"]))) < 2e-3
    if not files:
        assert got[1] == 0 and got[2] == 0


def test_one_frame_video_has_nan_temporal_consistency(tmp_path):
    clip_m, ctf, _ = _clip("clip_tiny", 61, tmp_path)
    dino_m, _ = _dino(TINY_DINO, "dino_tiny", 62)
    s = score_video(torch.from_numpy(make_frames("wide_no_targets")[:1]).cuda(), "a dog", [], clip_m, ctf, dino_m,
                    dino_transform()).cpu()
    assert torch.isnan(s[3]) and s[1] == 0 and s[2] == 0 and torch.isfinite(s[0])


def test_graph_replay_equals_eager(tmp_path):
    clip_m, ctf, _ = _clip("clip_tiny", 61, tmp_path)
    dino_m, _ = _dino(TINY_DINO, "dino_tiny", 62)
    dtf = dino_transform()
    clips = [torch.from_numpy(make_frames(n)[:3]).cuda() for n in ("square_targets",)] * 1
    xs = [clips[0].roll(s, dims=2) for s in range(5)]
    outs = [(clip_m.encode_image_nhwc(ctf.batch(x)), dino_m.forward_nhwc(dtf.batch(x))) for x in xs]
    assert graph.stats(clip_m)["encode_image_nhwc"] == (1, 4) and graph.stats(dino_m)["_forward_nhwc"] == (1, 4)
    clip_m.use_cuda_graph = dino_m.use_cuda_graph = False
    eager = [(clip_m.encode_image_nhwc(ctf.batch(x)), dino_m.forward_nhwc(dtf.batch(x))) for x in xs]
    for (a, b), (c, d) in zip(outs, eager):
        assert torch.equal(a, c) and torch.equal(b, d)
    assert not torch.equal(outs[0][0], outs[1][0])


def test_cpu_resident_models_are_refused():
    from vgen_b200 import lib
    with pytest.raises(lib.VgenError, match="CUDA device"):
        vit_small()(torch.zeros(1, 3, 224, 224, device="cuda"))
    with pytest.raises(lib.VgenError, match="CUDA device"):
        OpenAIClipModel(TINY_CLIP).encode_image_nhwc(torch.zeros(1, 224, 224, 3, device="cuda", dtype=torch.float16))


# a child process, so the profiling session leaves no profiler state in the suite's process
_PROFILE_CHILD = r"""
import json, os, sys
root = sys.argv[1]
sys.path[:0] = [root, root + "/tests"]
os.environ["VGEN_CLIP_BPE"] = root + "/tests/golden/clip_bpe_merges_head.txt.gz"
import functools, torch
from torch.profiler import ProfilerActivity, profile
from _metric import TINY_CLIP, TINY_DINO, clip_state_dict, dino_state_dict, load_case, product_spec
from vgen_b200.clip import OpenAIClipModel
from vgen_b200.dino import VisionTransformer
from vgen_b200.metric import clip_transform, dino_transform, score_video
c = OpenAIClipModel(TINY_CLIP)
c.load_state_dict(clip_state_dict(product_spec("clip_tiny"), 61), strict=True)
d = VisionTransformer(**TINY_DINO, norm_layer=functools.partial(torch.nn.LayerNorm, eps=1e-6))
d.load_state_dict(dino_state_dict(product_spec("dino_tiny"), 62), strict=True)
c, d = c.eval().cuda(), d.eval().cuda()
z = load_case(root + "/tests/golden", "square_targets")
frames = torch.from_numpy(z["frames"]).cuda()
ctf, dtf = clip_transform(), dino_transform()
out = {}
for graphed in (False, True):
    c.use_cuda_graph = d.use_cuda_graph = graphed
    for _ in range(3):
        score_video(frames, "a dog", z["targets"], c, ctf, d, dtf)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        score_video(frames, "a dog", z["targets"], c, ctf, d, dtf).tolist()
        torch.cuda.synchronize()
    out["graphed" if graphed else "eager"] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
print(json.dumps(out))
"""


def test_scoring_launches_only_library_kernels():
    from test_gpu_sketch import _kernel_name, _library_kernels
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, ROOT], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    ours = _library_kernels()
    for mode, nms in names.items():
        foreign = {nm for nm in nms if _kernel_name(nm) not in ours and "memcpy" not in nm.lower() and "memset" not in nm.lower()}
        assert not foreign, (mode, foreign)
    for k in ("resize_crop_norm_kernel", "video_scores_kernel", "quick_gelu_kernel", "tapgemm_sm90_kernel"):
        assert any(k in nm for nm in names["eager"]), (k, names["eager"])
