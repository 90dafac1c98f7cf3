"""Freeze the reference's outputs for the 'histogram' composition and its colour-palette annotator into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it, see oracle/refload.py):
    python tools/make_golden_histogram.py
  * UNet: for each case of tests/_histogram.py it builds the reference class (UNetSD_VideoLCM or UNetSD_TFT2V) on CPU,
    loads synthetic weights (oracle/synth.py), runs the reference forward in fp32, checks the oracle against it and
    writes histogram_<case>.npz.  histogram_specs.json holds the digests of the reference's parameter lists (the cases
    and full-size models built on the meta device).
  * Palette: it runs the reference's tools/annotator/histogram/palette.py unmodified, with a `skimage.color` stub that
    holds oracle/palette_oracle.py's restatement of scikit-image 0.22.0 (skimage is not installed) and the real sklearn.
    histogram_palette.npz holds its tables (rgb, lab, lab_dists, thumbnail; hex in histogram_specs.json), the fixture
    frames of tests/_histogram.py, their histograms at every sigma in SIGMAS (float32 frames are widened to float64, as
    vgen_b200.palette does), and a quantize_image.  Each is checked against the oracle first.
Zip entries carry a fixed timestamp, so a rerun writes the same bytes.
"""
from __future__ import annotations

import importlib
import importlib.util
import io
import json
import os
import sys
import types
import zipfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import palette_oracle as po, refload, synth  # noqa: E402
import _histogram as hi  # noqa: E402
from _vcomp import spec_digest  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _maxrel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def savez_fixed(path, **arrays):
    """np.savez_compressed with a fixed zip timestamp."""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            b = io.BytesIO()
            np.lib.format.write_array(b, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, b.getvalue())
    with open(path, "wb") as fh:
        fh.write(buf.getvalue())


def reference_palette_module():
    """The reference's palette.py on the skimage stub."""
    root = refload.require_root()
    color = types.ModuleType("skimage.color")
    color.hsv2rgb, color.rgb2lab, color.lab2rgb = po.hsv2rgb, po.rgb2lab, po.lab2rgb
    sio = types.ModuleType("skimage.io")

    def imsave(*a, **k):
        raise NotImplementedError("skimage.io stub")
    sio.imsave = imsave
    sk = types.ModuleType("skimage")
    sk.color, sk.io = color, sio
    sys.modules.update({"skimage": sk, "skimage.color": color, "skimage.io": sio})
    spec = importlib.util.spec_from_file_location("ref_palette", os.path.join(root, "tools", "annotator", "histogram",
                                                                             "palette.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def palette_golden(specs):
    ref = reference_palette_module().Palette()
    ora = po.PaletteOracle()
    for k in ("rgb", "lab", "lab_dists", "thumbnail"):
        assert np.array_equal(getattr(ref, k), getattr(ora, k)), k
    for nh in (8, 9, 10, 12):
        r, o = reference_palette_module().Palette(num_hues=nh), po.PaletteOracle(num_hues=nh)
        assert np.array_equal(r.lab, o.lab) and np.array_equal(r.lab_dists, o.lab_dists), nh
    out = {"rgb": ref.rgb, "lab": ref.lab, "lab_dists": ref.lab_dists, "thumbnail": ref.thumbnail}
    specs["palette_hex"] = list(ref.hex)
    for name in hi.FRAMES:
        img = hi.make_frame(name)
        out[f"frame_{name}"] = img
        x = img if img.dtype == np.uint8 else img.astype(np.float64)
        for sigma in hi.SIGMAS:
            h = ref.histogram(x, sigma=sigma)
            err = float(np.abs(h - ora.histogram(x, sigma=sigma)).max())
            assert err <= 1e-12, (name, sigma, err)
            out[f"hist_{name}_s{sigma}"] = h
            print(f"palette {name} sigma {sigma}: oracle vs reference max abs {err:.1e}")
    q = ref.quantize_image(hi.make_frame("u8_61x97"))
    assert np.array_equal(q, ora.quantize_image(hi.make_frame("u8_61x97")))
    out["quantize_u8_61x97"] = q
    savez_fixed(os.path.join(GOLD, "histogram_palette.npz"), **out)


def unet_golden(specs):
    refload.load()
    from easydict import EasyDict
    classes = {"UNetSD_VideoLCM": importlib.import_module("tools.modules.unet.unet_videolcm").UNetSD_VideoLCM,
               "UNetSD_TFT2V": importlib.import_module("tools.modules.unet.unet_tf2tv").UNetSD_TFT2V}
    for name, case in hi.HIST_CASES.items():
        m = classes[case["cls"]](config=EasyDict(**hi.config_of(case)), **case["ctor"]).eval()
        spec = synth.spec_of(m)
        sd = synth.state_dict(spec, seed=case["seed"])
        m.load_state_dict(sd, strict=True)
        inp = hi.make_inputs(case)
        out = m(inp["x"], inp["t"], **hi.call_kwargs(case, inp))
        err = _maxrel(hi.oracle_call(case, sd, inp), out)
        assert err < 2e-5, (name, err)
        print(f"{name}: oracle vs reference maxrel {err:.2e}")
        savez_fixed(os.path.join(GOLD, name + ".npz"), out=out.numpy())
        specs[name] = spec_digest(spec)
    for name, (cls, comps, ctor) in hi.HIST_SPECS.items():
        with torch.device("meta"):
            m = classes[cls](config=EasyDict(video_compositions=list(comps), resolution=[448, 256]), **ctor)
        specs[name] = spec_digest(synth.spec_of(m))
        print(f"{name}: {specs[name]}")


def main():
    torch.set_grad_enabled(False)
    specs = {}
    palette_golden(specs)
    unet_golden(specs)
    with open(os.path.join(GOLD, "histogram_specs.json"), "w") as fh:
        json.dump(specs, fh, indent=1)


if __name__ == "__main__":
    main()
