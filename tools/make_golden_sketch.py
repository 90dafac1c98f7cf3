"""Freeze the reference sketch annotators' outputs for the cases of tests/_sketch.py into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it):
    python tools/make_golden_sketch.py
tools/annotator/sketch/pidinet.py and sketch_simplification.py import only torch, so they are loaded from their files with
no stubs.  For each case the reference network is built on CPU with synthetic weights (tests/_sketch.state_dict), run in
fp32, and the oracle (oracle/sketch_oracle.py) is checked against it.  sketch_<case>.npz holds "out"; sketch_specs.json
the digests of the tiny and full-size parameter lists and of the reference's convert_pidinet() applied to a synthetic
PDC-format checkpoint of pidinet_bsd().  Only new files are written.
"""
from __future__ import annotations

import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _sketch as sk  # noqa: E402
from oracle import refload, sketch_oracle, synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _reference_module(name):
    path = os.path.join(refload.REF_ROOT, "tools", "annotator", "sketch", f"{name}.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"set VGEN_REFERENCE_ROOT to a checkout of ali-vilab/VGen (no {path})")
    spec = importlib.util.spec_from_file_location(f"vgen_reference_{name}", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    torch.set_grad_enabled(False)
    pid, gan = _reference_module("pidinet"), _reference_module("sketch_simplification")
    tiny = dict(sk.TINY_PIDINET, pdcs=pid.config_model_converted("carv4"))
    assert tiny["pdcs"] == sk.CARV4
    digests = {"pidinet_full": sk.spec_digest(synth.spec_of(pid.pidinet_bsd())),
               "pidinet_tiny": sk.spec_digest(synth.spec_of(pid.PiDiNet(**tiny))),
               "cleaner": sk.spec_digest(synth.spec_of(gan.sketch_simplification_gan()))}
    pdc = sk.pdc_state_dict(synth.spec_of(pid.pidinet_bsd()))
    conv = pid.convert_pidinet({k: v.clone() for k, v in pdc.items()}, "carv4")
    digests["pidinet_converted"] = sk.tensor_digest({k[len("module."):]: v for k, v in conv.items()})
    for name, case in sk.SKETCH_CASES.items():
        if case["net"] == "pidinet":
            m = pid.PiDiNet(**tiny).eval()
        else:
            m = gan.sketch_simplification_gan().eval()
        sd = sk.state_dict(synth.spec_of(m), case["seed"], case["net"])
        m.load_state_dict(sd, strict=True)
        x = sk.make_input(case["net"], case["n"], case["H"], case["W"], case["seed"])
        out = m(x)
        if case["net"] == "pidinet":
            mine = sketch_oracle.pidinet_forward(sd, x)
        else:
            mine = sketch_oracle.cleaner_forward(sd, x, m.mean, m.std)
        err = float((mine - out).abs().max() / out.abs().max())
        std, sat = sk.non_vacuous(out)
        assert err < 1e-6, (name, err)
        assert std > 0.05 and sat < 0.5, f"{name}: std {std:.3f}, saturated {sat:.0%}: the case would test little"
        print(f"{name}: out {tuple(out.shape)}, std {std:.3f}, saturated {sat:.1%}, oracle vs reference maxrel {err:.2e}",
              flush=True)
        np.savez_compressed(os.path.join(GOLD, f"sketch_{name}.npz"), out=out.numpy())
    for k in ("pidinet_full", "cleaner"):
        print(f"{k}: {digests[k]['parameters']} parameters in {digests[k]['tensors']} tensors")
    with open(os.path.join(GOLD, "sketch_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)


if __name__ == "__main__":
    main()
