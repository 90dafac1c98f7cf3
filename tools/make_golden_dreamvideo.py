"""Freeze the reference's outputs for the DreamVideo cases (tests/_dreamvideo.py) into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it, see oracle/refload.py):
    python tools/make_golden_dreamvideo.py
For each case it builds the reference UNetSD_DreamVideo on CPU, loads synthetic weights (oracle/synth.py), runs the
reference forward in fp32 and checks the oracle restatement against it before anything is written: <case>.npz holds the
output under the case's weight seed, dreamvideo_pin.npz the outputs under a second seed.  The reference takes one
ag_strength per call, so a batch with per-video values is run one video at a time (videos never interact).
dreamvideo_specs.json holds the digests of the reference's parameter lists (tensor count, parameter count, sha256) for the
cases and for the released base / subject / motion / joint UNets, built on the meta device.
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
import _dreamvideo as dv  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
PIN_SEED = 82


def _maxrel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _reference_call(m, case, inp):
    kw = {"y": inp["y"]}
    if "y_image" not in inp:
        return m(inp["x"], inp["t"], **kw)
    outs = []
    for i in range(case["b"]):   # one video per call: the reference's ag_strength is one number
        outs.append(m(inp["x"][i:i + 1], inp["t"][i:i + 1], y=inp["y"][i:i + 1], y_image=inp["y_image"][i:i + 1],
                      ag_strength=float(inp["ag_strength"][i])))
    return torch.cat(outs)


def main():
    torch.set_grad_enabled(False)
    refload.load()
    ref_cls = importlib.import_module("tools.modules.unet.unet_dreamvideo").UNetSD_DreamVideo
    pin, digests = {}, {}
    for name, case in dv.DV_CASES.items():
        m = ref_cls(**case["ctor"]).eval()
        spec = synth.spec_of(m)
        assert spec == dv.product_spec(case["ctor"]), f"{name}: the product's parameter list differs from the reference's"
        inp = dv.make_inputs(case)
        for seed in (case["seed"], PIN_SEED):
            sd = synth.state_dict(spec, seed=seed)
            m.load_state_dict(sd, strict=True)
            out = _reference_call(m, case, inp)
            err = _maxrel(dv.oracle_call(case, sd, inp), out)
            assert err < 2e-5, (name, seed, err)
            print(f"{name} seed {seed}: oracle vs reference maxrel {err:.2e}")
            if seed == case["seed"]:
                np.savez_compressed(os.path.join(GOLD, name + ".npz"), out=out.numpy())
            else:
                pin[f"{name}_seed{seed}"] = out.numpy()
        digests[name] = dv.spec_digest(spec)
    np.savez_compressed(os.path.join(GOLD, "dreamvideo_pin.npz"), **pin)
    for name, adapters in dv.RELEASED_ADAPTERS.items():
        with torch.device("meta"):
            m = ref_cls(**dv.RELEASED_UNET, **adapters)
        digests[name] = dv.spec_digest(synth.spec_of(m))
        assert (digests[name]["tensors"], digests[name]["parameters"]) == dv.RELEASED_COUNTS[name], (name, digests[name])
        print(f"{name}: {digests[name]}")
    with open(os.path.join(GOLD, "dreamvideo_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)


if __name__ == "__main__":
    main()
