"""Freeze the reference canny annotator's edge maps for the cases below into tests/golden/canny_*.npz and canny_specs.json.

Run where a checkout of the reference is available (VGEN_REFERENCE_ROOT names it) and OpenCV is installed:
    python tools/make_golden_canny.py
tools/annotator/canny/__init__.py is loaded from its file, unmodified (its `tools.annotator.util` import resolves to the
reference's own util.py without running tools/__init__.py), and runs on the CPU with torch.Tensor.cuda as the identity.
cv2.Canny is wrapped only to record the thresholds the detector passes.  Each case checks oracle/canny_oracle.py against
the reference (edge map and thresholds), and the reference's map against cv2.Canny on the oracle's bytes.  The archives
are written with fixed zip timestamps, so a rerun reproduces them byte for byte.
"""
from __future__ import annotations

import importlib.util
import io
import json
import os
import sys
import types
import zipfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy import ndimage  # noqa: E402

import _canny as cg  # noqa: E402
from oracle import canny_oracle, refload  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

# name -> shape, source dtype, threshold mode, content; explicit thresholds as the detector receives them
CASES = {
    "rand_61x97_c3": dict(h=61, w=97, c=3, src="f32", mode="random", seed=1, content="field"),
    "rand_256x448_c1": dict(h=256, w=448, c=1, src="f32", mode="random", seed=2, content="field"),
    "fixed_64x96_c1": dict(h=64, w=96, c=1, src="f32", mode="fixed", seed=3, content="field"),
    "int_256x448_c3": dict(h=256, w=448, c=3, src="f32", mode="explicit", seed=4, content="field", low=40, high=100),
    "float_64x96_c3": dict(h=64, w=96, c=3, src="f32", mode="explicit", seed=5, content="field", low=35.7, high=90.2),
    "swapped_61x97_c1_u8": dict(h=61, w=97, c=1, src="u8", mode="explicit", seed=6, content="field", low=150, high=40),
    "black_64x96_c3": dict(h=64, w=96, c=3, src="f32", mode="random", seed=7, content="black"),
    "even_median_64x96_c1": dict(h=64, w=96, c=1, src="f32", mode="fixed", seed=8, content="split"),
    "serpentine_256x448_c1": dict(h=256, w=448, c=1, src="f32", mode="explicit", seed=9, content="serpentine", low=50,
                                  high=150),
}


def _shapes(rng, h, w, c, img):
    """A few flat rectangles and discs of random colour over img (h, w, c) in [0, 1]."""
    yy, xx = np.mgrid[:h, :w]
    for _ in range(6):
        col = rng.random(c)
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        if rng.random() < 0.5:
            r = rng.uniform(4, min(h, w) / 3)
            m = (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
        else:
            hh, hw = rng.uniform(3, h / 3), rng.uniform(3, w / 3)
            m = (abs(yy - cy) < hh) & (abs(xx - cx) < hw)
        img[m] = col
    return img


def _field(rng, h, w, c):
    sigma = max(2.0, min(h, w) / 16)                        # the same smoothness relative to the frame at every size
    f = ndimage.gaussian_filter(rng.random((h, w, c)), (sigma, sigma, 0))
    f = (f - f.min()) / (f.max() - f.min())
    return _shapes(rng, h, w, c, f)


def _serpentine(h, w):
    """Two serpentine bands (flat steps of 20 / 255 over black, so |dx| + |dy| = 80 on their straight edges: weak with
    thresholds 50 / 150) crossing many 32 x 16 tiles; the first ends in a bright square (strong edges), the second
    touches nothing strong."""
    img = np.zeros((h, w), np.float64)
    for band, (y0, y1) in enumerate(((4, 124), (132, 252))):
        level = 20 / 255
        rows = range(y0, y1 - 6, 20)
        for k, y in enumerate(rows):
            img[y:y + 6, 8:w - 8] = level
            if k + 1 < len(rows):
                x = w - 14 if k % 2 == 0 else 8
                img[y:y + 26, x:x + 6] = level
        if band == 0:
            img[y0:y0 + 10, 2:14] = 1.0
    return img[:, :, None]


def make_frame(spec):
    """The case's frame as stored (the encoded codes of an fp32 frame, or uint8) and as the detector receives it."""
    rng = np.random.default_rng(1000 + spec["seed"])
    h, w, c = spec["h"], spec["w"], spec["c"]
    if spec["content"] == "field":
        x = _field(rng, h, w, c)
    elif spec["content"] == "black":
        x = _shapes(rng, h, w, c, np.zeros((h, w, c)))
        x[h // 4:, :] = 0                                   # keep the median at 0
    elif spec["content"] == "split":
        # half the pixels at most 80 / 255, half at least 83 / 255: the median is (80 + 83) / 2 = 81.5
        x = _field(rng, h, w, c)
        order = np.argsort(x, axis=None, kind="stable")
        lo, hi = order[:x.size // 2], order[x.size // 2:]
        flat = x.reshape(-1).copy()
        flat[lo] = 80 / 255 * (flat[lo] - flat[lo].min()) / (flat[lo].max() - flat[lo].min())
        flat[hi] = 83 / 255 + (1 - 83 / 255) * (flat[hi] - flat[hi].min()) / (flat[hi].max() - flat[hi].min())
        x = flat.reshape(h, w, c)
    else:
        x = _serpentine(h, w)
    if spec["src"] == "u8":
        stored = np.rint(x * 255).astype(np.uint8)
    else:
        stored = cg.encode(np.rint(x * cg.CODE_SCALE))
    return stored, cg.decode(stored)


def _reference_detector():
    root = refload.REF_ROOT
    path = os.path.join(root, "tools", "annotator", "canny", "__init__.py")
    if not os.path.isfile(path):
        raise RuntimeError(f"set VGEN_REFERENCE_ROOT to a checkout of ali-vilab/VGen (no {path})")
    for pkg, sub in (("tools", "tools"), ("tools.annotator", os.path.join("tools", "annotator"))):
        if pkg not in sys.modules:                          # namespace parents: tools/__init__.py imports every engine
            m = types.ModuleType(pkg)
            m.__path__ = [os.path.join(root, sub)]
            sys.modules[pkg] = m
    spec = importlib.util.spec_from_file_location("vgen_reference_canny", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    calls = []

    class _Cv2Spy:
        def __getattr__(self, k):
            return getattr(cv2, k)

        @staticmethod
        def Canny(img, low, high):
            calls.append((img.copy(), low, high))
            return cv2.Canny(img, low, high)

    mod.cv2 = _Cv2Spy()
    return mod.CannyDetector(), calls


def _write_npz(path, arrays):
    """np.savez_compressed with fixed member timestamps."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(f"{k}.npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    torch.Tensor.cuda = lambda self, *a, **k: self
    det, calls = _reference_detector()
    out_specs = {}
    total = 0
    for name, spec in CASES.items():
        stored, frame = make_frame(spec)
        kw = cg.call_kwargs(spec)
        calls.clear()
        np.random.seed(spec["seed"])
        if spec["src"] == "u8":
            ref = det(frame, **kw)
        else:
            ref = det(torch.from_numpy(frame), **kw)
        (img_np, low, high), = calls
        r = None
        if spec["mode"] == "random":
            np.random.seed(spec["seed"])
            r = np.random.uniform(0.1, 0.4)
        ref = ref.numpy()
        assert ref.shape == (spec["h"], spec["w"], 1) and ref.dtype == np.float32
        assert set(np.unique(ref)) <= {0.0, 1.0}
        # the oracle against the reference: bytes, thresholds, edge map
        mine_bytes = frame if spec["src"] == "u8" else canny_oracle.quantise(frame)
        assert np.array_equal(mine_bytes.reshape(img_np.shape), img_np), name
        assert canny_oracle.thresholds(mine_bytes, kw.get("low_threshold"), kw.get("high_threshold"),
                                       kw.get("random_threshold", True), r) == (low, high), name
        mine = canny_oracle.detect(frame, r=r, **kw)
        assert np.array_equal(mine, ref), (name, int((mine != ref).sum()))
        assert np.array_equal(cv2.Canny(img_np, low, high), canny_oracle.canny(img_np, low, high)), name
        edge = ref[:, :, 0] > 0.5
        median = float(np.median(img_np))
        thr = canny_oracle.cv_thresholds(low, high)
        cls = canny_oracle.classify(img_np, *thr)
        n_edge, n_cand, n_strong = int(edge.sum()), int((cls > 0).sum()), int((cls == 2).sum())
        assert spec["content"] == "black" or n_edge > 0, name
        if spec["content"] == "black":
            assert median == 0.0 and (low, high) == (0, 0) and n_edge > 0, name
        if spec["content"] == "split":
            assert median == 81.5, median
        if spec["content"] == "serpentine":
            # the first band's weak edges are kept through one strong square, the second band's are dropped
            assert n_strong < n_edge // 20 and n_cand > 2 * n_edge - n_edge // 4 and n_edge > 2000, (n_strong, n_cand, n_edge)
            assert edge[:128, 300:].sum() > 500 and edge[128:].sum() == 0, name
        arrays = {"frame": stored, "edge": np.packbits(edge.reshape(-1)), "thr": np.array(thr, np.int32),
                  "median": np.float64(median)}
        if r is not None:
            arrays["r"] = np.float64(r)
        path = os.path.join(GOLD, f"canny_{name}.npz")
        _write_npz(path, arrays)
        total += os.path.getsize(path)
        out_specs[name] = dict(spec, ref_low=low, ref_high=high)
        print(f"{name}: median {median}, thresholds {low!r} / {high!r} -> {thr}, {n_cand} candidates, {n_strong} strong, "
              f"{n_edge} edge pixels; oracle == reference", flush=True)
    with open(os.path.join(GOLD, "canny_specs.json"), "w") as fh:
        json.dump(out_specs, fh, indent=1)
        fh.write("\n")
    print(f"{len(CASES)} cases, {total} bytes of archives")


if __name__ == "__main__":
    main()
