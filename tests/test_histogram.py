"""The 'histogram' composition and the colour-palette annotator on the CPU: the oracles against the reference's frozen
outputs, the native Palette's host tables, the parameter lists, and the import boundary."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import palette_oracle as po, synth
from vgen_b200 import arch, lib, palette
from _histogram import (FRAMES, HIST_CASES, HIST_SPECS, SIGMAS, load_palette_golden, load_spec, make_frame, make_inputs,
                        oracle_call, product_spec, reference_digest)
from _vcomp import spec_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_palette_oracle_tables_equal_reference():
    g, o = load_palette_golden(), po.PaletteOracle()
    for k in ("rgb", "lab", "lab_dists", "thumbnail"):
        assert np.array_equal(getattr(o, k), g[k]), k


def test_native_palette_tables_equal_reference():
    g, p = load_palette_golden(), palette.Palette()
    for k in ("rgb", "lab", "lab_dists", "thumbnail"):
        assert getattr(p, k).dtype == np.float64 and np.array_equal(getattr(p, k), g[k]), k
    assert p.rgb.shape == (156, 3) and p.hex == reference_digest("palette_hex")


@pytest.mark.parametrize("num_hues", [8, 9, 10, 11, 12, 5])
def test_native_palette_tables_equal_oracle(num_hues):
    p, o = palette.Palette(num_hues=num_hues), po.PaletteOracle(num_hues=num_hues)
    for k in ("rgb", "lab", "lab_dists", "thumbnail"):
        assert np.array_equal(getattr(p, k), getattr(o, k)), k
    assert np.array_equal(palette.lab2rgb(p.lab), po.lab2rgb(o.lab))


def test_uint8_linearisation_table():
    """The 256-entry table the device uses for uint8 frames is rgb2xyz's transfer function of v * (1 / 255)."""
    lin = palette._linearise(palette._as_float(np.arange(256, dtype=np.uint8)))
    a = np.multiply(np.arange(256, dtype=np.uint8), 1.0 / 255, dtype=np.float64)
    ref = np.where(a > 0.04045, ((a + 0.055) / 1.055) ** 2.4, a / 12.92)
    assert np.array_equal(lin, ref)


@pytest.mark.parametrize("name", list(FRAMES))
@pytest.mark.parametrize("sigma", SIGMAS)
def test_palette_oracle_histograms_match_reference(name, sigma):
    g = load_palette_golden()
    img = g[f"frame_{name}"]
    assert np.array_equal(img, make_frame(name))
    x = img if img.dtype == np.uint8 else img.astype(np.float64)
    got = po.PaletteOracle().histogram(x, sigma=sigma)
    want = g[f"hist_{name}_s{sigma}"]
    assert np.abs(got - want).max() <= 1e-12
    assert (got == 0).sum() == (want == 0).sum()
    if sigma == 0:
        assert got.sum() == pytest.approx(1.0)


def test_palette_oracle_quantize_matches_reference():
    g = load_palette_golden()
    assert np.array_equal(po.PaletteOracle().quantize_image(g["frame_u8_61x97"]), g["quantize_u8_61x97"])


def test_smoothing_weights_and_palette_image():
    p = palette.Palette()
    assert p.smoothing_weights(0) is None and p.smoothing_weights(-1) is None
    w = p.smoothing_weights(20)
    assert w.shape == (156, 156) and np.allclose(w.sum(1), 1.0)
    hist = load_palette_golden()["hist_u8_32x48_flat_s0"]
    img = p.get_palette_image(hist)
    assert img.shape == (50, 200, 3) and img.dtype == np.float64
    # the strip starts with the most frequent entry
    assert np.array_equal(img[0, 0], p.rgb[np.argmax(hist)])
    with pytest.raises(NotImplementedError):
        p.export("/nonexistent")


@pytest.mark.parametrize("name", list(HIST_CASES))
def test_unet_oracle_matches_reference(name, golden_dir):
    case = HIST_CASES[name]
    spec = load_spec(name)
    sd = synth.state_dict(spec, seed=case["seed"])
    inp = make_inputs(case)
    got = oracle_call(case, sd, inp)
    want = torch.from_numpy(np.load(os.path.join(golden_dir, name + ".npz"))["out"])
    assert float((got - want).abs().max() / want.abs().max()) < 2e-5


@pytest.mark.parametrize("name", list(HIST_SPECS))
def test_full_size_spec_equals_reference(name):
    cls, comps, ctor = HIST_SPECS[name]
    spec = product_spec(cls, comps, [448, 256], ctor)
    assert spec_digest(spec) == reference_digest(name)
    names = [k for k, _ in spec]
    i = names.index("hist_context_embedding.0.weight")
    assert names[i:i + 4] == ["hist_context_embedding.0.weight", "hist_context_embedding.0.bias",
                              "hist_context_embedding.2.weight", "hist_context_embedding.2.bias"]
    assert dict(spec)["hist_context_embedding.0.weight"] == (1280, 156)


def test_without_histogram_the_spec_is_unchanged():
    cls, comps, ctor = HIST_SPECS["full_vcomposer_histogram"]
    with_h = product_spec(cls, comps, [448, 256], ctor)
    without = product_spec(cls, [c for c in comps if c != "histogram"], [448, 256], ctor)
    assert [s for s in with_h if not s[0].startswith("hist_context_embedding.")] == without


def test_load_state_dict_strict_with_histogram():
    import vgen_b200
    case = HIST_CASES["histogram_tft2v_tiny_b2"]
    spec = load_spec("histogram_tft2v_tiny_b2")
    m = vgen_b200.UNetSD_TFT2V(config=dict(video_compositions=case["comps"], resolution=case["resolution"]), **case["ctor"],
                               enable_histogram=True)
    m.load_state_dict(synth.state_dict(spec, seed=1), strict=True)
    assert m.plan.hist_dim == 156


def test_histogram_refusals_before_any_launch():
    import vgen_b200
    case = HIST_CASES["histogram_tft2v_tiny_b2"]
    m = vgen_b200.UNetSD_TFT2V(config=dict(video_compositions=["text"], resolution=case["resolution"]), **case["ctor"])
    assert "hist_context_embedding.0.weight" not in m.state_dict()
    with pytest.raises(lib.VgenError):   # no CUDA path for CPU inputs
        m(torch.zeros(1, 4, 2, 8, 12), torch.tensor([1]), y=torch.zeros(1, 5, 1024), histogram=torch.zeros(1, 2, 156))


def test_palette_device_path_refuses_cpu_tensors():
    with pytest.raises(lib.VgenError):
        palette.histogram_video(torch.zeros(1, 2, 3, 4, 4))
    t = torch.zeros(1, 3, 1, 4, dtype=torch.float64)
    with pytest.raises(lib.VgenError):
        palette.ops.palette_histogram(torch.zeros(1, 3, 4, 4), t)


def test_abi_declares_the_palette_entries():
    hdr = open(os.path.join(ROOT, "include", "vgen_b200.h")).read()
    for sym in ("vgen_palette_histogram", "vgen_palette_quantize"):
        assert sym in lib.declared_symbols() and f"int {sym}(" in hdr


def test_product_never_imports_the_oracle_or_the_stub():
    code = ("import sys, vgen_b200, vgen_b200.palette, vgen_b200.unet; vgen_b200.palette.Palette(); "
            "bad = [m for m in sys.modules if m.split('.')[0] in ('oracle', 'skimage', 'sklearn')]; "
            "assert not bad, bad")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for fn in ("palette.py", "unet.py", "arch.py", "ops.py"):
        src = open(os.path.join(ROOT, "vgen_b200", fn)).read()
        for mod in ("oracle", "skimage"):
            assert f"import {mod}" not in src and f"from {mod}" not in src, (fn, mod)


def test_histogram_is_a_known_composition():
    assert "histogram" in arch.VCOMP_NAMES


def test_histogram_is_opt_in():
    """Listing 'histogram' builds the composition only with enable_histogram=True; without it the model refuses it as
    before, and a histogram passed to a model built without the composition is refused before any device work (so this
    runs without a GPU).  A histogram of the wrong shape is refused too."""
    import vgen_b200
    ctor = HIST_CASES["histogram_tft2v_tiny_b2"]["ctor"]
    cfg = {"video_compositions": ["text", "histogram"], "resolution": [96, 64]}
    for cls in (vgen_b200.UNetSD_TFT2V, vgen_b200.UNetSD_VideoLCM):
        with pytest.raises(NotImplementedError, match="enable_histogram=True"):
            cls(config=cfg, **ctor)
        with pytest.raises(ValueError, match="enable_histogram"):
            cls(config=cfg, enable_histogram=1, **ctor)
    h = vgen_b200.UNetSD_TFT2V(config=cfg, enable_histogram=True, **ctor)
    assert h.video_compositions == ["text", "histogram"]
    assert "hist_context_embedding.0.weight" in h.state_dict()
    # the flag alone changes nothing: without 'histogram' listed the parameters are the plain model's
    a = vgen_b200.UNetSD_TFT2V(config={"video_compositions": ["text"]}, enable_histogram=True, **ctor)
    b = vgen_b200.UNetSD_TFT2V(config={"video_compositions": ["text"]}, **ctor)
    assert [(k, v.shape) for k, v in a.state_dict().items()] == [(k, v.shape) for k, v in b.state_dict().items()]
    m = vgen_b200.UNetSD_TFT2V(config={"video_compositions": ["text", "depthmap"], "resolution": [96, 64]}, **ctor)
    x, t = torch.zeros(1, 4, 2, 8, 12), torch.zeros(1, dtype=torch.long)
    for model in (m, h):
        model._check_x = lambda x, t: None
    with pytest.raises(NotImplementedError, match="enable_histogram=True"):
        type(m).forward.__wrapped_eager__(m, x, t, y=torch.zeros(1, 5, 1024), histogram=torch.zeros(1, 2, 156))
    with pytest.raises(ValueError, match="histogram must be"):
        type(h).forward.__wrapped_eager__(h, x, t, y=torch.zeros(1, 5, 1024), histogram=torch.zeros(1, 2, 155))
