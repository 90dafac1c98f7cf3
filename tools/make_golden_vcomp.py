"""Freeze the reference's outputs for the VideoComposer composition cases (tests/_vcomp.py) into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it, see oracle/refload.py):
    python tools/make_golden_vcomp.py
For each case it builds the reference class (UNetSD_VideoLCM or UNetSD_TFT2V) on CPU with the case's config, loads
synthetic weights (oracle/synth.py), runs the reference forward in fp32, checks the oracle restatement against it and
writes <case>.npz.  vcomp_pin.npz holds the reference outputs under a second weight seed.  vcomp_specs.json holds, for
every case and for the full-size models (built on the meta device; released_* with the UNet section of the released
configs), the digest of the reference's parameter list: tensor count, parameter count and the sha256 of the list.
Only new files are written; no other golden file is touched.
"""
from __future__ import annotations

import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import refload, synth  # noqa: E402
import _vcomp as vc  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
PIN_SEED = 81


def _maxrel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _classes():
    refload.load()
    from easydict import EasyDict
    lcm = importlib.import_module("tools.modules.unet.unet_videolcm")
    tft = importlib.import_module("tools.modules.unet.unet_tf2tv")
    return {"UNetSD_VideoLCM": lcm.UNetSD_VideoLCM, "UNetSD_TFT2V": tft.UNetSD_TFT2V}, EasyDict


def main():
    torch.set_grad_enabled(False)
    classes, EasyDict = _classes()
    pin, digests = {}, {}
    for name, case in vc.VCOMP_CASES.items():
        m = classes[case["cls"]](config=EasyDict(**vc.config_of(case)), **case["ctor"]).eval()
        spec = synth.spec_of(m)
        inp = vc.make_inputs(case)
        for seed in (case["seed"], PIN_SEED):
            sd = synth.state_dict(spec, seed=seed)
            m.load_state_dict(sd, strict=True)
            kw = vc.call_kwargs(case, inp)
            out = m(inp["x"], inp["t"], **kw)
            err = _maxrel(vc.oracle_call(case, sd, inp), out)
            assert err < 2e-5, (name, seed, err)
            print(f"{name} seed {seed}: oracle vs reference maxrel {err:.2e}")
            if seed == case["seed"]:
                np.savez_compressed(os.path.join(GOLD, name + ".npz"), out=out.numpy())
            else:
                pin[f"{name}_seed{seed}"] = out.numpy()
        digests[name] = vc.spec_digest(spec)
    np.savez_compressed(os.path.join(GOLD, "vcomp_pin.npz"), **pin)
    for name, (comps, ctor) in vc.FULL_SPECS.items():
        with torch.device("meta"):
            m = classes["UNetSD_TFT2V"](config=EasyDict(video_compositions=list(comps), resolution=[448, 256]), **ctor)
        digests[name] = vc.spec_digest(synth.spec_of(m))
        print(f"{name}: {digests[name]}")
    with open(os.path.join(GOLD, "vcomp_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)


if __name__ == "__main__":
    main()
