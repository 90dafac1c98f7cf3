"""Freeze the reference depth annotator's outputs for the cases of tests/_depth.py into tests/golden/.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it):
    python tools/make_golden_depth.py
tools/annotator/depth/__init__.py imports only torch, so it is loaded from its file with no stubs.  For each case the
reference MiDaS is built on CPU with synthetic weights (tests/_depth.state_dict: oracle/synth.py, all-zero tensors such
as the reference's cls_embedding initialisation drawn again), run in fp32, and the oracle (oracle/depth_oracle.py) is
checked against it.  depth_<case>.npz holds "out"; depth_specs.json the digests of the tiny and the full-size midas_v3()
parameter lists.  Only new files are written.
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

import _depth as dp  # noqa: E402
from oracle import depth_oracle, refload, synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _reference_module():
    path = os.path.join(refload.REF_ROOT, "tools", "annotator", "depth", "__init__.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"set VGEN_REFERENCE_ROOT to a checkout of ali-vilab/VGen (no {path})")
    spec = importlib.util.spec_from_file_location("vgen_reference_depth", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    torch.set_grad_enabled(False)
    ref = _reference_module()
    with torch.device("meta"):
        full = ref.midas_v3()
    digests = {"full": dp.spec_digest(synth.spec_of(full))}
    for name, case in dp.DEPTH_CASES.items():
        m = ref.MiDaS(**case["ctor"]).eval()
        spec = synth.spec_of(m)
        digests["tiny"] = dp.spec_digest(spec)
        sd = dp.state_dict(spec, case["seed"])
        assert all(v.abs().max() > 0 for v in sd.values())
        m.load_state_dict(sd, strict=True)
        x = dp.make_input(case["n"], case["H"], case["W"], case["seed"])
        out = m(x)
        mine = depth_oracle.midas_forward(sd, x, **dp.oracle_kw(case["ctor"]))
        err = float((mine - out).abs().max() / out.abs().max())
        pos = float((out > 0).float().mean())
        assert err < 1e-5, (name, err)
        assert pos > 0.3, f"{name}: only {pos:.0%} of the output pixels are positive: the case would test little"
        print(f"{name}: out {tuple(out.shape)}, positive {pos:.0%}, oracle vs reference maxrel {err:.2e}", flush=True)
        np.savez_compressed(os.path.join(GOLD, f"depth_{name}.npz"), out=out.numpy())
    print(f"midas_v3(): {digests['full']['parameters'] / 1e6:.2f} M parameters in {digests['full']['tensors']} tensors")
    with open(os.path.join(GOLD, "depth_specs.json"), "w") as fh:
        json.dump(digests, fh, indent=1)


if __name__ == "__main__":
    main()
