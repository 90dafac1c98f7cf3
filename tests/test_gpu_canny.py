"""The canny annotator on the H100: every golden case bit-exact through both entry points, canny_video against per-frame
calls and the oracle at full size, no host synchronisation, and a TF-T2V UNet fed the native map."""
import numpy as np
import pytest
import torch

import _canny as cg
from oracle import canny_oracle as co, synth
from vgen_b200 import canny, ops
from _vcomp import VCOMP_CASES, build_product, call_kwargs, make_inputs, oracle_call, product_spec

pytestmark = pytest.mark.gpu


def _stream_state():
    """numpy's global stream position: the Mersenne Twister keys and the index into them."""
    _, keys, pos = np.random.get_state()[:3]
    return keys.tobytes(), pos


def _call(det, spec, frame):
    np.random.seed(spec["seed"])
    if spec["src"] == "u8":
        return det(frame, **cg.call_kwargs(spec))
    return det(torch.from_numpy(frame).cuda(), **cg.call_kwargs(spec))


@pytest.mark.parametrize("name", sorted(cg.specs()))
def test_golden_bit_exact(name):
    spec, frame, edge, z = cg.load(name)
    want = torch.from_numpy(edge.astype(np.float32))[:, :, None].cuda()
    got = _call(canny.CannyDetector(), spec, frame)
    assert got.shape == (spec["h"], spec["w"], 1) and got.dtype == torch.float32 and got.is_cuda
    assert int((got != want).sum()) == 0
    after = _stream_state()                # the reference draws once in random mode, else never
    np.random.seed(spec["seed"])
    if "r" in z:
        assert np.random.uniform(0.1, 0.4) == float(z["r"])
    assert _stream_state() == after
    # canny_video on the same frame as a 1 x 1 video; the device thresholds through ops.canny
    x = torch.from_numpy(frame).cuda()
    if spec["src"] == "u8":
        frames = x.permute(2, 0, 1)[None]
        mode, r, low, high = canny.threshold_plan(1, **cg.call_kwargs(spec))
        vid, thr = ops.canny(frames, mode, None, low, high, thresholds=True)
    else:
        np.random.seed(spec["seed"])
        vid = canny.canny_video(x.permute(2, 0, 1)[None, None], **cg.call_kwargs(spec))
        assert vid.shape == (1, 1, 1, spec["h"], spec["w"])
        np.random.seed(spec["seed"])
        mode, r, low, high = canny.threshold_plan(1, **cg.call_kwargs(spec))
        rand = torch.tensor(r, dtype=torch.float64, device="cuda") if r is not None else None
        _, thr = ops.canny(x.permute(2, 0, 1)[None], mode, rand, low, high, thresholds=True)
    assert int((vid.reshape(want.shape) != want).sum()) == 0
    assert thr.cpu().tolist() == [z["thr"].tolist()]


def _video(b, f, h, w, seed):
    """[b, f, 3, h, w] fp32 frames in [0, 1]: smooth fields with flat shapes, a different one per frame."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(b * f, 3, h // 8, w // 8, device="cuda", generator=g)
    x = torch.nn.functional.interpolate(x, size=(h, w), mode="bicubic", align_corners=False).clamp_(0, 1)
    yy, xx = torch.meshgrid(torch.arange(h, device="cuda"), torch.arange(w, device="cuda"), indexing="ij")
    for i in range(b * f):
        cy, cx, r = h * (0.2 + 0.06 * (i % 10)), w * (0.3 + 0.04 * (i % 7)), min(h, w) / 5
        x[i, :, (yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = torch.rand(3, 1, device="cuda", generator=g)
    return x.reshape(b, f, 3, h, w)


def _oracle_video(frames, r=None, **kw):
    b, f = frames.shape[:2]
    host = frames.permute(0, 1, 3, 4, 2).cpu().numpy()
    out = np.zeros((b, 1, f) + frames.shape[3:], np.float32)
    for i in range(b):
        for j in range(f):
            out[i, 0, j] = co.detect(host[i, j], r=None if r is None else r[i * f + j], **kw)[:, :, 0]
    return torch.from_numpy(out).cuda()


@pytest.mark.parametrize("kw", [{}, {"random_threshold": False}, {"low_threshold": 60, "high_threshold": 30.5}])
def test_video_equals_per_frame_calls(kw):
    frames = _video(2, 3, 64, 96, seed=11)
    np.random.seed(3)
    vid = canny.canny_video(frames, **kw)
    after_video = _stream_state()
    det = canny.CannyDetector()
    np.random.seed(3)
    per = torch.stack([torch.stack([det(frames[i, j].permute(1, 2, 0), **kw) for j in range(3)]) for i in range(2)])
    assert _stream_state() == after_video
    assert vid.shape == (2, 1, 3, 64, 96)
    assert torch.equal(vid, per[..., 0].unsqueeze(1))
    assert 0 < float(vid.mean()) < 0.5


@pytest.mark.parametrize("b, f, h, w", [(1, 16, 256, 448), (1, 1, 704, 1280)])
def test_matches_oracle_at_full_size(b, f, h, w):
    frames = _video(b, f, h, w, seed=12)
    np.random.seed(21)
    vid = canny.canny_video(frames)
    np.random.seed(21)
    r = [np.random.uniform(0.1, 0.4) for _ in range(b * f)]
    want = _oracle_video(frames, r)
    diff = int((vid != want).sum())
    print(f"canny {b}x{f}x{h}x{w}: {int(want.sum())} edge pixels, {diff} differ")
    assert diff == 0 and float(want.sum()) > 100 * b * f


def test_no_host_synchronisation():
    frames = _video(1, 4, 64, 96, seed=13)
    det = canny.CannyDetector()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        np.random.seed(4)
        vid = canny.canny_video(frames)
        one = det(frames[0, 0].permute(1, 2, 0), random_threshold=False)
        two = canny.canny_video(frames, 20, 80)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    np.random.seed(4)
    assert torch.equal(vid, _oracle_video(frames, [np.random.uniform(0.1, 0.4) for _ in range(4)]))
    assert torch.equal(one[:, :, 0], _oracle_video(frames[:1, :1], random_threshold=False)[0, 0, 0])
    assert torch.equal(two, _oracle_video(frames, low_threshold=20, high_threshold=80))


def test_refusals_on_the_device():
    det = canny.CannyDetector()
    x = torch.rand(8, 8, 3, device="cuda")
    with pytest.raises(ValueError, match="both thresholds"):
        det(x, low_threshold=10)
    with pytest.raises(ValueError, match="c = 1 or 3"):
        det(torch.rand(8, 8, 2, device="cuda"))
    with pytest.raises(Exception, match="CUDA fp32"):
        det(x.half())
    with pytest.raises(ValueError, match="both thresholds"):
        canny.canny_video(x.permute(2, 0, 1)[None, None], high_threshold=10)
    with pytest.raises(ValueError, match=r"\[b, f, c, h, w\]"):
        canny.canny_video(x.permute(2, 0, 1)[None])
    with pytest.raises(Exception, match="CUDA fp32"):
        canny.canny_video(x.permute(2, 0, 1)[None, None].double())


def test_tft2v_unet_with_native_canny_condition():
    """A tiny UNetSD_TFT2V with 'canny' in its compositions: the native map and the oracle's map give the same forward,
    and that forward matches the fp32 oracle UNet."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    base = VCOMP_CASES["vcomp_tft2v_tiny_b2"]
    case = dict(base, comps=base["comps"] + ["canny"], conds=base["conds"] + ["canny"])
    sd = synth.state_dict(product_spec(case["cls"], case["comps"], case["resolution"], case["ctor"]), seed=case["seed"])
    m = build_product(case)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    sdg = {k: v.cuda() for k, v in sd.items()}
    inp = {k: v.cuda() for k, v in make_inputs(dict(case, conds=base["conds"])).items()}
    frames = _video(case["b"], case["f"], case["H"], case["W"], seed=14)
    np.random.seed(7)
    native = canny.canny_video(frames)
    np.random.seed(7)
    oracle_map = _oracle_video(frames, [np.random.uniform(0.1, 0.4) for _ in range(case["b"] * case["f"])])
    assert torch.equal(native, oracle_map) and float(native.sum()) > 0
    with torch.no_grad():
        a = m(inp["x"], inp["t"], **call_kwargs(case, dict(inp, canny=native)))
        b = m(inp["x"], inp["t"], **call_kwargs(case, dict(inp, canny=oracle_map)))
        none = m(inp["x"], inp["t"], **call_kwargs(case, dict(inp, canny=torch.zeros_like(native))))
        o32 = oracle_call(case, sdg, dict(inp, canny=oracle_map))
    assert torch.equal(a, b)
    assert not torch.equal(a, none)
    rel = float((a.float() - o32.float()).norm() / o32.float().norm())
    print(f"tft2v with canny: ours vs fp32 oracle rel_l2 {rel:.3e}")
    assert rel < 5e-3
