"""Freeze the reference's outputs for the long-clip cases (tests/_longclip.py) into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it, see oracle/refload.py):
    python tools/make_golden_longclip.py
For each case it builds the reference class on CPU, loads synthetic weights (oracle/synth.py), runs the reference
forward in fp32, checks the oracle restatement against it and writes longclip_<case>.npz ("out"; for cases with a
"ddim" recipe also "ddim_latent", the reference's DiffusionDDIM.ddim_sample_loop with CFG).  longclip_specs.json holds
the digest of each reference parameter list: tensor count, parameter count and the sha256 of the list.
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

from oracle import refload, synth, vgen_oracle as vo  # noqa: E402
import _longclip as lc  # noqa: E402
import _vcomp as vc  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _maxrel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _reference_model(ref, case):
    if case["kind"] == "t2v":
        return ref.UNetSD_T2VBase(**case["ctor"])
    if case["kind"] == "i2vgen":
        return ref.UNetSD_I2VGen(**case["ctor"])
    from easydict import EasyDict
    lcm = importlib.import_module("tools.modules.unet.unet_videolcm")
    return lcm.UNetSD_VideoLCM(config=EasyDict(**vc.config_of(case)), **case["ctor"])


def _reference_call(case, m, inp):
    if case["kind"] == "t2v":
        return m(inp["x"], inp["t"], y=inp["y"])
    if case["kind"] == "i2vgen":
        return m(inp["x"], inp["t"], y=inp["y"], image=inp["image"], local_image=inp["local_image"], fps=inp["fps"])
    return m(inp["x"], inp["t"], **vc.call_kwargs(case, inp))


def main():
    torch.set_grad_enabled(False)
    ref = refload.load()
    digests = {}
    for name, case in lc.LONG_CASES.items():
        m = _reference_model(ref, case).eval()
        spec = synth.spec_of(m)
        sd = synth.state_dict(spec, seed=case["seed"])
        m.load_state_dict(sd, strict=True)
        inp = lc.make_inputs(case)
        out = _reference_call(case, m, inp)
        err = _maxrel(lc.oracle_call(case, sd, inp), out)
        assert err < 2e-5, (name, err)
        print(f"{name}: out {tuple(out.shape)}, oracle vs reference maxrel {err:.2e}", flush=True)
        arrays = {"out": out.numpy()}
        if case.get("ddim"):
            dd = case["ddim"]
            sp = dict(num_timesteps=1000, cosine_s=0.008, zero_terminal_snr=True)
            diff = ref.DiffusionDDIM(schedule="cosine", schedule_param=sp, mean_type="v", var_type="fixed_small")
            kw = [{"y": inp["y"]}, {"y": inp["y_neg"]}]
            lat = diff.ddim_sample_loop(inp["x"].clone(), m, kw, guide_scale=dd["guide_scale"], ddim_timesteps=dd["steps"], eta=0.0)
            fn = lambda xt, t, **k: vo.unet_t2v_forward(sd, xt, t, **k)  # noqa: E731
            mine = vo.ddim_sample_loop(inp["x"].clone(), fn, kw, vo.make_betas("cosine", 1000, True, cosine_s=0.008),
                                       dd["guide_scale"], dd["steps"])
            e2 = _maxrel(mine, lat)
            assert e2 < 1e-4, (name, "ddim", e2)
            print(f"{name}: ddim oracle vs reference maxrel {e2:.2e}", flush=True)
            arrays["ddim_latent"] = lat.numpy()
        np.savez_compressed(os.path.join(GOLD, f"longclip_{name}.npz"), **arrays)
        digests[name] = vc.spec_digest(spec)
    with open(os.path.join(GOLD, "longclip_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)


if __name__ == "__main__":
    main()
