"""The canny annotator's golden cases (tools/make_golden_canny.py freezes them into tests/golden/canny_*.npz and
canny_specs.json): loading, and the decoding of their frozen inputs.

An fp32 frame is code / 1020 in fp32 for integer codes 0..1020, so x * 255 lands on quarter steps (and on either side
of the .5 rounding boundary).  It is stored as the int16 differences of its codes along each channel plane, (c, h, w)
in C order, which compress well.  A uint8 frame is stored as it is.  The edge map is np.packbits of the h * w booleans.
"""
from __future__ import annotations

import json
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CODE_SCALE = 1020


def specs():
    with open(os.path.join(GOLD, "canny_specs.json")) as fh:
        return json.load(fh)


def load(name):
    """(spec, frame (h, w, c) fp32 or uint8, edge (h, w) bool, npz dict)."""
    spec = specs()[name]
    z = dict(np.load(os.path.join(GOLD, f"canny_{name}.npz")))
    frame = decode(z["frame"])
    h, w = frame.shape[:2]
    edge = np.unpackbits(z["edge"], count=h * w).reshape(h, w).astype(bool)
    return spec, frame, edge, z


def decode(stored):
    if stored.dtype == np.int16:
        codes = np.cumsum(stored.reshape(-1), dtype=np.int64).reshape(stored.shape)      # (c, h, w)
        return np.ascontiguousarray(codes.transpose(1, 2, 0)).astype(np.float32) / np.float32(CODE_SCALE)
    return stored


def encode(codes):
    """The stored form of an fp32 frame's codes (h, w, c) (see decode)."""
    planes = codes.transpose(2, 0, 1).astype(np.int64)
    return np.diff(planes.reshape(-1), prepend=0).astype(np.int16).reshape(planes.shape)


def call_kwargs(spec):
    """The CannyDetector keyword arguments of a case."""
    kw = {}
    if spec["mode"] == "fixed":
        kw["random_threshold"] = False
    elif spec["mode"] == "explicit":
        kw["low_threshold"], kw["high_threshold"] = spec["low"], spec["high"]
    return kw
