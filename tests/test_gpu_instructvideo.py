"""InstructVideo on the H100: forward parity of UNetSD_LoRA (same gates as tests/test_gpu_parity.py and
tests/test_gpu_fullsize.py), bit-exact packing against UNetSD_T2VBase loaded with the merged weights, the LoRA's effect and
re-packing, CFG batching, CUDA graph replay, determinism, the DiffusionDDIMReward loop and the video write-out."""
import gc
import os
import shutil

import numpy as np
import pytest
import torch

import vgen_b200
from oracle import vgen_oracle as vo
from vgen_b200 import graph, video_io
from vgen_b200.diffusion import cfg_forward
from _instructvideo import (FULL_IV_CASES, IV_CASES, RELEASED_DIFFUSION, build_product, load_spec, lora_scale, make_inputs,
                            make_video, oracle_call, unet_lora_forward, weights)

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _setup(golden_dir, name, cases=IV_CASES):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    gc.collect()
    torch.cuda.empty_cache()
    case = cases[name]
    spec = load_spec(golden_dir, name, cases)
    sd = weights(spec, case["seed"])
    m = build_product(case)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    sdg = {k: v.cuda() for k, v in sd.items()}
    del sd
    inp = {k: v.cuda() for k, v in make_inputs(case).items()}
    return case, m, inp, sdg


def _t2vbase(ctor, sd):
    m = vgen_b200.UNetSD_T2VBase(**{k: v for k, v in ctor.items() if "lora" not in k})
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("name", sorted(IV_CASES))
def test_forward_parity(golden_dir, name):
    case, m, inp, sdg = _setup(golden_dir, name)
    with torch.no_grad():
        mine = m(inp["x"], inp["t"], inp["y"])
        o32 = oracle_call(case, sdg, inp)
        with torch.autocast("cuda", dtype=torch.float16):
            o16 = oracle_call(case, sdg, inp)
    truth = torch.from_numpy(np.load(os.path.join(golden_dir, name + ".npz"))["out"]).cuda()
    assert mine.shape == truth.shape and mine.dtype == torch.float16 and torch.isfinite(mine.float()).all()
    assert _rel_l2(o32, truth) < 1e-4, "GPU fp32 oracle must reproduce the reference's CPU fp32 result"
    e_mine, e_ref16 = _rel_l2(mine, truth), _rel_l2(o16, truth)
    print(f"{name}: ours vs fp32 truth {e_mine:.3e}; reference-autocast vs truth {e_ref16:.3e}")
    assert e_mine < 5e-3
    assert e_mine < 1.25 * e_ref16 + 2e-4


@pytest.mark.parametrize("name", ["iv_lora_tiny", "iv_lora_alpha_tiny_b2"])
def test_packing_equals_t2vbase_with_merged_weights(golden_dir, name):
    """The LoRA model's packed arena is UNetSD_T2VBase's for the merged state dict, tensor for tensor and bit for bit."""
    case, m, inp, _ = _setup(golden_dir, name)
    b = _t2vbase(case["ctor"], m.merged_state_dict())
    pa, pb = m.packed_tensors(), b.packed_tensors()
    assert [k for k, _ in pa] == [k for k, _ in pb]
    for (k, ta), (_, tb) in zip(pa, pb):
        assert ta.dtype == tb.dtype and torch.equal(ta, tb), k
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        assert torch.equal(eager(m, inp["x"], inp["t"], inp["y"]), type(b).forward.__wrapped_eager__(b, inp["x"], inp["t"], y=inp["y"]))


def test_get_lora_merged_model_on_native_classes(golden_dir):
    """inference_instructvideo_entrance.py:301-353 restated on the native classes: a use_lora=False base built through the
    registry, the pairs merged through state_dict() in fp32, load_state_dict re-packs; the result runs T2VBase's arena."""
    case, m, inp, sdg = _setup(golden_dir, "iv_lora_alpha_tiny_b2")
    MODEL, _, _ = vgen_b200.register(force_local=True)
    cfg = dict(case["ctor"], type="UNetSD_LoRA")
    base = MODEL.build(dict(cfg, use_lora=False)).cuda().eval()
    bd, md = base.state_dict(), m.state_dict()
    for k, v in md.items():
        if "lora" not in k:
            bd[k] = v.clone()
    alpha = lora_scale(case["ctor"])
    for k, v in md.items():
        if "lora" in k and "up_linear" not in k:
            att = k.replace("_lora", ".0" if "to_out" in k else "").replace("down_linear.", "")
            bd[att] += alpha * torch.mm(md[k.replace("down_linear", "up_linear")], v)
    base.load_state_dict(bd)
    ref = _t2vbase(case["ctor"], bd)
    assert all(torch.equal(ta, tb) for (_, ta), (_, tb) in zip(base.packed_tensors(), ref.packed_tensors()))
    # the fp32 torch.mm merge differs from the pack's fp64 one by an fp32 ulp in many weights; the fp16 cast absorbs
    # almost all of it
    pb, pm = dict(base.packed_tensors()), dict(m.packed_tensors())
    assert pb.keys() == pm.keys()
    n = sum(t.numel() for t in pm.values())
    flips = sum(int((pb[k] != pm[k]).sum()) for k in pm)
    print(f"fp16 packed weights that differ between the fp32 and the fp64 merge: {flips} of {n}")
    assert flips < 1e-3 * n
    # the merged native model against the frozen output of the reference's merged model, with the parity gates
    with torch.no_grad():
        merged_out = base(inp["x"], inp["t"], inp["y"])
        with torch.autocast("cuda", dtype=torch.float16):
            o16 = oracle_call(case, sdg, inp)
    truth = torch.from_numpy(np.load(os.path.join(golden_dir, "iv_lora_alpha_tiny_b2.npz"))["out"]).cuda()
    e_mine, e_ref16 = _rel_l2(merged_out, truth), _rel_l2(o16, truth)
    print(f"get_lora_merged_model on native classes: {e_mine:.3e}; reference-autocast {e_ref16:.3e}")
    assert e_mine < 5e-3 and e_mine < 1.25 * e_ref16 + 2e-4


def test_without_lora_equals_t2vbase(golden_dir):
    case, m, inp, sdg = _setup(golden_dir, "iv_nolora_tiny")
    b = _t2vbase(case["ctor"], {k: v.cpu() for k, v in sdg.items()})
    assert all(torch.equal(ta, tb) for (_, ta), (_, tb) in zip(m.packed_tensors(), b.packed_tensors()))
    with torch.no_grad():
        assert torch.equal(m(inp["x"], inp["t"], inp["y"], fps=torch.full((1,), 8, device="cuda")), b(inp["x"], inp["t"], y=inp["y"]))


def test_lora_effect_and_repack(golden_dir):
    case, m, inp, sdg = _setup(golden_dir, "iv_lora_tiny")
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        with_lora = eager(m, inp["x"], inp["t"], inp["y"])
        plain = _t2vbase(case["ctor"], {k: v.cpu() for k, v in sdg.items() if "_lora." not in k})(inp["x"], inp["t"], y=inp["y"])
        assert _rel_l2(with_lora, plain) > 0.1, "the LoRA must move the output far above the parity tolerance"
        # new LoRA weights: load_state_dict re-packs, and the output follows them
        sd2 = {k: (-v if k.endswith("up_linear.weight") else v).cpu() for k, v in sdg.items()}
        m.load_state_dict(sd2, strict=True)
        flipped = eager(m, inp["x"], inp["t"], inp["y"])
        fresh = build_product(case)
        fresh.load_state_dict(sd2, strict=True)
        fresh = fresh.cuda().eval()
        assert torch.equal(flipped, eager(fresh, inp["x"], inp["t"], inp["y"]))
        truth = unet_lora_forward({k: v.cuda() for k, v in sd2.items()}, inp["x"], inp["t"], inp["y"])
    assert _rel_l2(flipped, with_lora) > 0.1 and _rel_l2(flipped, truth) < 5e-3


def test_cfg_pair_is_one_batched_forward(golden_dir, monkeypatch):
    """The engine's CFG pair (inference_instructvideo_entrance.py:234-237): y against the empty prompt's tokens."""
    case, m, inp, _ = _setup(golden_dir, "iv_lora_alpha_tiny_b2")
    kc, ku = {"y": inp["y"]}, {"y": inp["y_neg"]}
    calls = []
    fwd = type(m).forward
    monkeypatch.setattr(type(m), "forward", lambda self, x, t, **kw: calls.append(x.shape[0]) or fwd(self, x, t, **kw))
    with torch.no_grad():
        yc, yu = cfg_forward(m, inp["x"], inp["t"], [kc, ku])
        assert calls == [2 * case["b"]]
        ac = m(inp["x"], inp["t"], **kc)
        au = m(inp["x"], inp["t"], **ku)
    assert _rel_l2(yc, ac) < 1e-3 and _rel_l2(yu, au) < 1e-3
    assert not torch.equal(yc, yu)


def test_cuda_graph_replay_equals_eager_and_is_deterministic(golden_dir):
    case, m, inp, _ = _setup(golden_dir, "iv_lora_alpha_tiny_b2")
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        ref = eager(m, inp["x"], inp["t"], inp["y"])
        assert torch.equal(eager(m, inp["x"], inp["t"], inp["y"]), ref)
        outs = [m(inp["x"], inp["t"], inp["y"]) for _ in range(3)]          # eager, capture, replay
        assert graph.stats(m).get("forward", (0, 0))[0] == 1
        for o in outs:
            assert torch.equal(o, ref)
        x2, y2 = inp["x"].flip(-1).contiguous(), inp["y_neg"]
        ref2 = eager(m, x2, inp["t"], y2)
        got2 = m(x2, inp["t"], y2)
        assert graph.stats(m)["forward"] == (1, 3)
    assert torch.equal(got2, ref2) and not torch.equal(got2, ref)


def test_ddim_loop_through_reward_sampler(golden_dir):
    """4 CFG DDIM steps of the released sampler (linear_sd, eps) through DiffusionDDIMReward against the oracle loop:
    truth = the unmerged oracle in fp32, yardstick = the same under autocast (tests/test_gpu_parity.py's gate)."""
    case, m, inp, sdg = _setup(golden_dir, "iv_lora_tiny")
    diff = vgen_b200.DiffusionDDIMReward(**{k: v for k, v in RELEASED_DIFFUSION.items() if k != "type"})
    kw = [{"y": inp["y"]}, {"y": inp["y_neg"]}]
    s = lora_scale(case["ctor"])
    fn = lambda xt, t, **k: unet_lora_forward(sdg, xt, t, k["y"], s)  # noqa: E731
    lat = diff.ddim_sample_loop(inp["x"], m, kw, guide_scale=9.0, ddim_timesteps=4, eta=0.0)
    betas = vo.make_betas("linear_sd", 1000, False, init_beta=0.00085, last_beta=0.0120)
    with torch.no_grad():
        truth = vo.ddim_sample_loop(inp["x"].clone(), fn, kw, betas, 9.0, 4, mean_type="eps")
        with torch.autocast("cuda", dtype=torch.float16):
            lat16 = vo.ddim_sample_loop(inp["x"].clone(), fn, kw, betas, 9.0, 4, mean_type="eps", autocast_cfg=True)
    e_mine, e_ref16 = _rel_l2(lat, truth), _rel_l2(lat16, truth)
    print(f"instructvideo ddim: ours {e_mine:.3e}; reference-autocast {e_ref16:.3e}")
    assert lat.dtype == torch.float32 and torch.isfinite(lat).all()
    assert e_mine < 2.5e-2 and e_mine < 1.25 * e_ref16 + 5e-4


def test_fullsize_forward(golden_dir):
    """The released LoRA UNet at the eval shape: CFG pair as one batch of 2, 16 frames, 32 x 32 latent, 77 tokens; truth =
    the unmerged oracle in fp32 on this GPU, yardstick = the oracle under autocast (tests/test_gpu_fullsize.py's gate)."""
    case, m, inp, sdg = _setup(golden_dir, "full_iv_lora", FULL_IV_CASES)
    x, t, y = torch.cat([inp["x"]] * 2), torch.cat([inp["t"]] * 2), torch.cat([inp["y"], inp["y_neg"]])
    with torch.no_grad():
        mine = m(x, t, y)
        truth = unet_lora_forward(sdg, x, t, y, lora_scale(case["ctor"]))
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = unet_lora_forward(sdg, x, t, y, lora_scale(case["ctor"]))
    assert mine.shape == truth.shape and torch.isfinite(mine.float()).all()
    ours, yard = _rel_l2(mine, truth), _rel_l2(ref16, truth)
    mx = float((mine.float() - truth).abs().max() / truth.abs().max())
    print(f"[fullsize] full_iv_lora: ours rel_l2 {ours:.3e} max {mx:.3e}; reference-autocast rel_l2 {yard:.3e}")
    assert ours < 6e-3
    assert ours < 1.25 * yard + 2e-4
    assert mx < 4 * 6e-3


def _have_encoder():
    try:
        import cv2  # noqa: F401
        return True
    except ImportError:
        return bool(shutil.which("ffmpeg"))


def _count_frames(path):
    import cv2
    cap = cv2.VideoCapture(path)
    n = 0
    while cap.read()[0]:
        n += 1
    cap.release()
    return n


@pytest.mark.parametrize("name", ["iv_video", "iv_video_single"])
def test_save_video_local_matches_reference_frames(golden_dir, tmp_path, name):
    if not _have_encoder():
        pytest.skip("no encoder (ffmpeg / OpenCV) on this box")
    v, mean, std = make_video(name)
    gold = np.load(os.path.join(golden_dir, "instructvideo_video.npz"))[name]
    for src in (v.cuda(), v):                      # the entrance hands over a host tensor (gen_videos.cpu())
        keep = src.clone()
        path = str(tmp_path / f"{name}_{src.device.type}.mp4")
        frames = video_io.save_video_local(path, src, mean, std)
        assert torch.equal(src.cpu(), keep.cpu()), "the caller's video must not be modified"
        assert len(frames) == v.shape[2] and all(fr.dtype == np.uint8 for fr in frames)
        assert np.array_equal(np.stack(frames), gold)
        assert os.path.getsize(path) > 0 and _count_frames(path) == v.shape[2]
