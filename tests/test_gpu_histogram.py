"""The 'histogram' composition and the colour-palette annotator on the H100: the nearest-colour pass over every uint8
colour, histograms and quantize_image against the oracle and the reference's frozen outputs, UNet parity of the two
histogram cases, CFG batching, graph replay, fp8_linear, the unchanged no-histogram path, and the device-only chain from
frames to the forward."""
import gc
import os

import numpy as np
import pytest
import torch

from oracle import palette_oracle as po, synth
from vgen_b200 import ops, palette
from vgen_b200.diffusion import cfg_forward
from _histogram import (FRAMES, HIST_CASES, NEAREST_BOUND, SIGMAS, build_product, call_kwargs, load_palette_golden,
                        load_spec, make_inputs, oracle_call)

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _device_indices(pal, frames):
    """Each pixel's nearest palette index from the device pass (quantize with a table whose colour is the index)."""
    t = pal._tables(frames.device)
    idx_tab = torch.arange(t["lab4"].shape[0], device=frames.device, dtype=torch.float64)[:, None].repeat(1, 3)
    return ops.palette_quantize(frames, t["lab4"], idx_tab.contiguous(), t["lin"])[..., 0].long()


def test_nearest_index_every_uint8_colour():
    """All 2^24 uint8 colours as one 4096 x 4096 image against the oracle (skimage's rgb2lab restated, sklearn's
    distances).  The indices must be equal except where the oracle's distance to the device's choice is within
    NEAREST_BOUND (1e-9; squared Lab distances reach ~4e4, so that is ~25 ulps) of its minimum: a near tie that
    a last-bit difference in the cube root or the summation order may resolve either way."""
    pal, ora = palette.Palette(), po.PaletteOracle()
    v = torch.arange(1 << 24, dtype=torch.int64, device="cuda")
    img = torch.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], dim=-1).to(torch.uint8).view(4096, 4096, 3)
    got = _device_indices(pal, img.permute(2, 0, 1).unsqueeze(0))[0].view(-1).cpu().numpy()
    cube = img.view(-1, 3).cpu().numpy()
    exceptions, chunk = 0, 1 << 18
    for s in range(0, 1 << 24, chunk):
        want, d = ora.nearest(cube[s:s + chunk])
        g = got[s:s + chunk]
        bad = np.nonzero(g != want)[0]
        if bad.size:
            gap = d[bad, g[bad]] - d[bad, want[bad]]
            assert (gap <= NEAREST_BOUND).all(), (s + bad[gap > NEAREST_BOUND][:5], gap.max())
            exceptions += bad.size
    print(f"[palette] nearest index over 2^24 colours: {exceptions} near-tie exceptions (bound {NEAREST_BOUND})")
    assert exceptions <= 64


@pytest.mark.parametrize("name", list(FRAMES))
def test_fixture_histograms_and_quantize_match_reference(name):
    g, pal = load_palette_golden(), palette.Palette()
    img = g[f"frame_{name}"]
    for sigma in SIGMAS:
        got = pal.histogram(img, sigma=sigma)
        want = g[f"hist_{name}_s{sigma}"]
        assert got.dtype == np.float64 and got.shape == (156,)
        assert np.abs(got - want).max() <= 1e-12, (sigma, np.abs(got - want).max())
        assert np.array_equal(got == 0, want == 0)
    if name == "u8_61x97":
        q = pal.quantize_image(img)
        assert q.dtype == np.float64 and np.array_equal(q, g["quantize_u8_61x97"])
    # the same frame as a CUDA tensor
    t = torch.from_numpy(img).cuda()
    got = pal.histogram(t if img.dtype == np.uint8 else t.double(), sigma=20)
    assert np.abs(got - g[f"hist_{name}_s20"]).max() <= 1e-12


@pytest.mark.parametrize("h,w,b,f", [(61, 97, 4, 8), (256, 448, 2, 4), (704, 1280, 1, 2)])
@pytest.mark.parametrize("u8", [True, False])
def test_histogram_video_matches_oracle(h, w, b, f, u8):
    gen = torch.Generator(device="cuda").manual_seed(h * 7 + w + int(u8))
    if u8:
        frames = torch.randint(0, 256, (b, f, h, w, 3), device="cuda", generator=gen, dtype=torch.uint8)
        per_frame = frames.flatten(0, 1).cpu().numpy()
    else:
        frames = torch.rand(b, f, 3, h, w, device="cuda", generator=gen)
        frames[..., : h // 3, : w // 4] = 0.25                 # a flat block: some bins far above, others far below 1e-5
        per_frame = frames.flatten(0, 1).permute(0, 2, 3, 1).double().cpu().numpy()
    pal, ora = palette.Palette(), po.PaletteOracle()
    v = frames if not u8 else frames.permute(0, 1, 4, 2, 3)
    idx = [ora.nearest(x)[0] for x in per_frame]
    for sigma in SIGMAS:
        got64 = pal.device_histogram(v.flatten(0, 1), sigma, torch.float64).cpu().numpy()
        want = np.stack([ora.histogram_of(i, sigma=sigma) for i in idx])
        err = np.abs(got64 - want).max()
        assert err <= 1e-12, (sigma, err)
        assert np.array_equal(got64 == 0, want == 0)
        vid = palette.histogram_video(frames, sigma=sigma)
        assert vid.shape == (b, f, 156) and vid.dtype == torch.float32
        assert torch.equal(vid.view(b * f, -1).cpu(), torch.from_numpy(got64).float())
    if h == 61:
        q = palette.Palette().quantize_image(per_frame[0])
        assert np.array_equal(q, ora.quantize_image(per_frame[0]))


def test_smaller_palette_and_refusals():
    pal, ora = palette.Palette(num_hues=8), po.PaletteOracle(num_hues=8)
    img = np.random.default_rng(5).integers(0, 256, size=(33, 65, 3), dtype=np.uint8)
    got = pal.histogram(img, sigma=20)
    assert got.shape == (117,) and np.abs(got - ora.histogram(img, sigma=20)).max() <= 1e-12
    with pytest.raises(ops._l.VgenError, match="156"):
        palette.Palette(num_hues=12).histogram(img)
    with pytest.raises(ValueError):
        palette.histogram_video(torch.zeros(1, 2, 4, 8, 8, device="cuda"))
    one = palette.histogram_video(torch.rand(1, 1, 3, 1, 1, device="cuda"), sigma=0)   # a single pixel
    assert float(one.max()) == 1.0 and int((one > 0).sum()) == 1


# ------------------------------------------------------------------------------------------------ the UNet
def _setup(name, **ctor):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    gc.collect()
    torch.cuda.empty_cache()
    case = HIST_CASES[name]
    sd = synth.state_dict(load_spec(name), seed=case["seed"])
    m = build_product(case, **ctor)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    inp = {k: v.cuda() for k, v in make_inputs(case).items()}
    return case, m, inp, {k: v.cuda() for k, v in sd.items()}


@pytest.mark.parametrize("name", sorted(HIST_CASES))
def test_forward_parity(golden_dir, name):
    case, m, inp, sdg = _setup(name)
    with torch.no_grad():
        mine = m(inp["x"], inp["t"], **call_kwargs(case, inp))
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
    with torch.no_grad():
        other = m(inp["x"], inp["t"], **dict(call_kwargs(case, inp), histogram=inp["histogram"].flip(-1).contiguous()))
    assert not torch.equal(other, mine)


def test_cfg_batch_equals_two_forwards():
    case, m, inp, _ = _setup("histogram_lcm_tiny")
    kc = call_kwargs(case, inp)
    ku = dict(kc, y=inp["y_neg"], image=torch.zeros_like(inp["image"]), histogram=torch.zeros_like(inp["histogram"]))
    with torch.no_grad():
        yc, yu = cfg_forward(m, inp["x"], inp["t"], [kc, ku])
        ac = m(inp["x"], inp["t"], **kc)
        au = m(inp["x"], inp["t"], **ku)
    assert _rel_l2(yc, ac) < 1e-3 and _rel_l2(yu, au) < 1e-3
    assert not torch.equal(yc, yu)


def test_cuda_graph_replay_with_a_new_histogram_equals_eager():
    from vgen_b200 import graph
    case, m, inp, _ = _setup("histogram_tft2v_tiny_b2")
    kw = call_kwargs(case, inp)
    eager = type(m).forward.__wrapped_eager__
    with torch.no_grad():
        ref = eager(m, inp["x"], inp["t"], **kw)
        outs = [m(inp["x"], inp["t"], **kw) for _ in range(3)]          # eager, capture, replay
        assert graph.stats(m)["forward"][0] == 1
        for o in outs:
            assert torch.equal(o, ref)
        kw2 = dict(kw, histogram=kw["histogram"] * 0.5 + 0.1)
        ref2 = eager(m, inp["x"], inp["t"], **kw2)
        got2 = m(inp["x"], inp["t"], **kw2)
        assert graph.stats(m)["forward"][1] >= 2
        # without the histogram the signature differs: a separate graph, the shared-context path
        bare = m(inp["x"], inp["t"], y=kw["y"])
        assert torch.equal(bare, eager(m, inp["x"], inp["t"], y=kw["y"]))
    assert torch.equal(got2, ref2) and not torch.equal(got2, ref)


def test_fp8_linear_runs_with_the_histogram(golden_dir):
    case, m, inp, _ = _setup("histogram_lcm_tiny", fp8_linear=True)
    with torch.no_grad():
        mine = m(inp["x"], inp["t"], **call_kwargs(case, inp))
    truth = torch.from_numpy(np.load(os.path.join(golden_dir, "histogram_lcm_tiny.npz"))["out"]).cuda()
    assert torch.isfinite(mine.float()).all()
    assert m._packed["hist_context_embedding.0.w"].dtype == torch.float16
    err = _rel_l2(mine, truth)
    print(f"histogram_lcm_tiny fp8_linear: rel_l2 vs fp32 truth {err:.3e}")
    assert err < 0.25


def test_without_histogram_the_forward_is_bit_identical():
    """The same weights in a model built without 'histogram': the forward without a histogram is the same bits."""
    case, m, inp, _ = _setup("histogram_lcm_tiny")
    comps = [c for c in case["comps"] if c != "histogram"]
    plain = build_product(dict(case, comps=comps))
    plain.load_state_dict({k: v for k, v in m.state_dict().items() if not k.startswith("hist_context_embedding.")},
                          strict=True)
    plain = plain.cuda().eval()
    kw = call_kwargs(case, inp)
    kw.pop("histogram")
    with torch.no_grad():
        a = m(inp["x"], inp["t"], **kw)
        b = plain(inp["x"], inp["t"], **kw)
    assert torch.equal(a, b)
    assert set(plain._packed) | {k for k in m._packed if k.startswith("hist_context_embedding.")} == set(m._packed)


def test_histogram_video_feeds_the_forward_without_a_host_round_trip():
    case, m, inp, sdg = _setup("histogram_tft2v_tiny_b2")
    b, f = case["b"], case["f"]
    frames = torch.rand(b, f, 3, 64, 96, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    kw = dict(y=inp["y"], histogram=palette.histogram_video(frames))    # warm-up: packs weights, uploads the tables,
    with torch.no_grad():                                                # captures the graph the timed call replays
        m(inp["x"], inp["t"], **kw)
        m(inp["x"], inp["t"], **kw)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            hist = palette.histogram_video(frames)
            out = m(inp["x"], inp["t"], y=inp["y"], histogram=hist)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    ora = po.PaletteOracle()
    want = np.stack([ora.histogram(x, sigma=20) for x in frames.flatten(0, 1).permute(0, 2, 3, 1).double().cpu().numpy()])
    assert np.abs(hist.view(b * f, -1).double().cpu().numpy() - want).max() < 1e-7
    with torch.no_grad():
        ref = oracle_call(case, sdg, dict(inp, histogram=hist))
    assert _rel_l2(out, ref) < 5e-3
