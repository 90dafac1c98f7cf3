"""Freeze the reference's DreamVideo metric (metric/cal_metric_DreamVideo.py calculate_metric, run unmodified) for the
cases of tests/_metric.py into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it):
    python tools/make_golden_metric.py
The script's imports are provided on the CPU as follows:
  * `clip`: a stub built from the reference's vendored open_clip -- `build_model_from_openai_state_dict` for the model
    (then `.float()`, which is what clip.load does on the CPU), its tokenizer with OpenAI's truncate=False rule, and
    OpenAI's `_transform(224)` (Resize(BICUBIC), CenterCrop, RGB, ToTensor, Normalize);
  * `cv2.VideoCapture`: a capture yielding the case's synthetic frames as BGR images;
  * `Tensor.cuda`: the identity, as in oracle/refload.py;
  * `dino.vision_transformer`: the reference's own module.
Target images are written as PNG files (lossless, so the decoded arrays are the frozen ones) and opened by the script
with PIL.  The transforms' outputs, the models' features and the scores are recorded around the calls the script makes;
the oracle (oracle/metric_oracle.py) is checked against every one of them.  Only new files are written.
"""
from __future__ import annotations

import functools
import importlib.util
import json
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import _metric as mt  # noqa: E402
from oracle import metric_oracle as mo, refload, synth  # noqa: E402
from oracle.make_golden_clip import load_reference_open_clip  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _clip_stub(model_mod, tok_mod):
    import torchvision.transforms as T

    def tokenize(texts, context_length=77, truncate=False):
        if isinstance(texts, str):
            texts = [texts]
        enc = tok_mod._tokenizer
        sot, eot = enc.encoder["<start_of_text>"], enc.encoder["<end_of_text>"]
        result = torch.zeros(len(texts), context_length, dtype=torch.int)
        for i, t in enumerate(texts):
            ids = [sot] + enc.encode(t) + [eot]
            if len(ids) > context_length:
                if not truncate:
                    raise RuntimeError(f"Input {t} is too long for context length {context_length}")
                ids = ids[:context_length]
                ids[-1] = eot
            result[i, :len(ids)] = torch.tensor(ids)
        return result

    def _transform(n_px):
        return T.Compose([T.Resize(n_px, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(n_px),
                          lambda im: im.convert("RGB"), T.ToTensor(), T.Normalize(mo.OPENAI_MEAN, mo.OPENAI_STD)])

    def load_state_dict(sd, device="cpu"):
        model = model_mod.build_model_from_openai_state_dict(dict(sd))
        if str(device) == "cpu":
            model = model.float()
        return model, _transform(model.visual.image_size[0] if isinstance(model.visual.image_size, tuple)
                                 else model.visual.image_size)

    return types.SimpleNamespace(tokenize=tokenize, _transform=_transform, load_state_dict=load_state_dict)


def _reference_script(clip_stub):
    metric_dir = os.path.join(refload.require_root(), "metric")
    if metric_dir not in sys.path:
        sys.path.insert(0, metric_dir)
    sys.modules["clip"] = types.ModuleType("clip")
    sys.modules["clip"].__dict__.update(vars(clip_stub))
    spec = importlib.util.spec_from_file_location("vgen_reference_cal_metric", os.path.join(metric_dir, "cal_metric_DreamVideo.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _Capture:
    frames = {}

    def __init__(self, path):
        self._it = iter(self.frames[path])

    def read(self):
        f = next(self._it, None)
        return (f is not None), (None if f is None else np.ascontiguousarray(f[..., ::-1]))   # RGB -> BGR


def _recorder(fn, sink):
    @functools.wraps(fn)
    def run(*a, **k):
        out = fn(*a, **k)
        sink.append(out.detach().clone())
        return out
    return run


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-30))


def main():
    torch.set_grad_enabled(False)
    torch.Tensor.cuda = lambda self, *a, **k: self
    model_mod, tok_mod = load_reference_open_clip()
    stub = _clip_stub(model_mod, tok_mod)
    ref = _reference_script(stub)
    ref.cv2.VideoCapture = _Capture
    from dino import vision_transformer as ref_dino

    # parameter lists: full-size ViT-B/32 (the open_clip model build_model_from_openai_state_dict makes) and ViT-S/16
    with torch.device("meta"):
        full_clip = model_mod.CLIP(512, model_mod.CLIPVisionCfg(layers=12, width=768, patch_size=32, image_size=224),
                                   model_mod.CLIPTextCfg(context_length=77, vocab_size=49408, width=512, heads=8, layers=12),
                                   quick_gelu=True)
        tiny_clip = model_mod.CLIP(64, model_mod.CLIPVisionCfg(layers=2, width=128, patch_size=32, image_size=224),
                                   model_mod.CLIPTextCfg(context_length=77, vocab_size=49408, width=128, heads=2, layers=2),
                                   quick_gelu=True)
    full_dino = ref_dino.vit_small()                    # (its constructor reads values: not on the meta device)
    tiny_dino = ref_dino.VisionTransformer(**mt.TINY_DINO, norm_layer=functools.partial(nn.LayerNorm, eps=1e-6))
    specs = {"clip_full": synth.spec_of(full_clip), "clip_tiny": synth.spec_of(tiny_clip),
             "dino_full": synth.spec_of(full_dino), "dino_tiny": synth.spec_of(tiny_dino)}
    digests = {k: mt.spec_digest(v) for k, v in specs.items()}

    csd = mt.clip_state_dict(specs["clip_tiny"], seed=61)
    ckpt = dict(csd, input_resolution=torch.tensor(224), context_length=torch.tensor(77), vocab_size=torch.tensor(49408))
    clip_model, clip_preprocess = stub.load_state_dict(ckpt)
    assert all(torch.equal(v.float(), csd[k]) for k, v in clip_model.state_dict().items() if k in csd)
    dsd = mt.dino_state_dict(specs["dino_tiny"], seed=62)
    dino_model = ref_dino.VisionTransformer(**mt.TINY_DINO, norm_layer=functools.partial(nn.LayerNorm, eps=1e-6))
    dino_model.load_state_dict(dsd, strict=True)
    dino_model.eval()
    import torchvision.transforms as T
    dino_preprocess = T.Compose([T.Resize(256, interpolation=3), T.CenterCrop(224), T.ToTensor(),
                                 T.Normalize((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))])

    rec = {k: [] for k in ("clip_pre", "dino_pre", "clip_img", "clip_txt", "dino")}
    clip_model.encode_image = _recorder(clip_model.encode_image, rec["clip_img"])
    clip_model.encode_text = _recorder(clip_model.encode_text, rec["clip_txt"])
    dino_rec = _recorder(dino_model.forward, rec["dino"])
    dino_model.forward = dino_rec
    clip_pre = _recorder(clip_preprocess, rec["clip_pre"])
    dino_pre = _recorder(dino_preprocess, rec["dino_pre"])

    from PIL import Image
    report = {}
    for name, case in mt.METRIC_CASES.items():
        for v in rec.values():
            v.clear()
        frames = mt.make_frames(name)
        _Capture.frames = {name: list(frames)}
        with tempfile.TemporaryDirectory() as td:
            files = []
            for j, (a, mode) in enumerate(mt.make_targets(name)):
                files.append(os.path.join(td, f"target{j}.png"))
                Image.fromarray(a, mode).save(files[-1])
            targets = [np.asarray(Image.open(f).convert("RGB")) for f in files]
            scores = ref.calculate_metric(name, case["prompt"], files, clip_model, clip_pre, dino_model, dino_pre)
        f, t = len(frames), len(targets)
        images = list(frames) + targets
        out = {"frames_delta": mt.delta_encode(frames), "scores": np.asarray(scores, np.float64),
               "tokens": stub.tokenize([case["prompt"]]).numpy()}
        for j, a in enumerate(targets):
            out[f"target{j}_delta"] = mt.delta_encode(a)
        # transforms: the reference's tensors (frozen as digests) and the oracle's, bit for bit
        pre = {}
        for key, fn in (("clip", mo.clip_transform), ("dino", mo.dino_transform)):
            got = pre[key] = torch.stack(rec[f"{key}_pre"])
            assert got.shape == (f + t, 3, 224, 224)
            mine = torch.stack([torch.from_numpy(fn(a)) for a in images])
            assert torch.equal(mine, got), f"{name}: the {key} transform restatement is not bit-exact"
            out[f"{key}_sha"] = np.array([mt.tensor_sha(x) for x in got])
        clip_img = torch.cat(rec["clip_img"])          # frames, then targets (the script's call order)
        dino = torch.cat(rec["dino"])
        out.update(clip_frames=clip_img[:f].numpy(), clip_targets=clip_img[f:].numpy(), text=rec["clip_txt"][0][0].numpy(),
                   dino_frames=dino[:f].numpy(), dino_targets=dino[f:].numpy())
        # the oracle against every recorded value
        x_clip, x_dino = pre["clip"], pre["dino"]
        o_img, o_txt = mo.clip_encode_image(csd, x_clip), mo.clip_encode_text(csd, torch.from_numpy(out["tokens"]).long())
        o_dino = mo.dino_forward(dsd, x_dino, mt.TINY_DINO["num_heads"])
        o_scores = mo.scores(o_img[:f], o_txt[0], o_img[f:], o_dino[:f], o_dino[f:])
        rep = {"clip_img": _rel(o_img, clip_img), "clip_txt": _rel(o_txt[0], rec["clip_txt"][0][0]), "dino": _rel(o_dino, dino),
               "scores": float(np.max(np.abs(np.asarray(o_scores) - out["scores"])))}
        assert max(rep.values()) < 1e-5, (name, rep)
        tc = out["scores"][3]
        print(f"{name}: scores {np.round(out['scores'], 4).tolist()}, oracle vs reference {rep}", flush=True)
        assert tc < 0.9, f"{name}: temporal consistency {tc:.3f}: the synthetic weights make consecutive frames look alike"
        report[name] = out["scores"].tolist()
        np.savez_compressed(os.path.join(GOLD, f"metric_{name}.npz"), **out)
    a, b = report.values()
    assert abs(a[0] - b[0]) > 0.02, "CLIP-T does not tell the cases apart"
    with open(os.path.join(GOLD, "metric_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)
    for k in ("clip_full", "dino_full"):
        print(f"{k}: {digests[k]['parameters']} parameters in {digests[k]['tensors']} tensors")


if __name__ == "__main__":
    main()
