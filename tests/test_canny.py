"""The canny annotator without a GPU: the oracle against the reference's frozen edge maps, the threshold arithmetic and
numpy draw order of vgen_b200/canny.py, and its refusals."""
import math

import numpy as np
import pytest
import torch

import _canny as cg
from oracle import canny_oracle as co
from vgen_b200 import canny, lib, ops


def _stream_state():
    """numpy's global stream position: the Mersenne Twister keys and the index into them."""
    _, keys, pos = np.random.get_state()[:3]
    return keys.tobytes(), pos


@pytest.mark.parametrize("name", sorted(cg.specs()))
def test_oracle_matches_reference(name):
    spec, frame, edge, z = cg.load(name)
    assert frame.shape == (spec["h"], spec["w"], spec["c"])
    assert frame.dtype == (np.uint8 if spec["src"] == "u8" else np.float32)
    kw = cg.call_kwargs(spec)
    r = float(z["r"]) if "r" in z else None
    got = co.detect(frame, r=r, **kw)
    assert got.shape == (spec["h"], spec["w"], 1) and got.dtype == np.float32
    assert np.array_equal(got[:, :, 0] > 0.5, edge)
    assert set(np.unique(got)) <= {0.0, 1.0}
    img = frame if spec["src"] == "u8" else co.quantise(frame)
    assert float(np.median(img)) == float(z["median"])
    low, high = co.thresholds(img, kw.get("low_threshold"), kw.get("high_threshold"), kw.get("random_threshold", True), r)
    assert (low, high) == (spec["ref_low"], spec["ref_high"])
    assert co.cv_thresholds(low, high) == tuple(z["thr"])


def test_goldens_cover_the_required_cases():
    specs = cg.specs()
    assert {(v["h"], v["w"]) for v in specs.values()} == {(61, 97), (64, 96), (256, 448)}
    assert {v["c"] for v in specs.values()} == {1, 3}
    assert {v["mode"] for v in specs.values()} == {"random", "fixed", "explicit"}
    explicit = [(v["low"], v["high"]) for v in specs.values() if v["mode"] == "explicit"]
    assert any(isinstance(a, float) for a, _ in explicit) and any(a > b for a, b in explicit)
    assert specs["black_64x96_c3"]["ref_low"] == specs["black_64x96_c3"]["ref_high"] == 0
    assert float(cg.load("even_median_64x96_c1")[3]["median"]) == 81.5


def test_quantise_is_convert_scale_abs():
    x = np.array([0.0, -0.0, 1.0, 1.5, -0.2, 0.5 / 255, 1.5 / 255, 2.5 / 255, 254.5 / 255, np.nan], np.float32)
    want = []
    for v in x:
        p = np.float32(v) * np.float32(255.0)
        want.append(0 if np.isnan(p) else min(255, int(np.rint(abs(p)))))
    assert co.quantise(x).tolist() == want
    assert co.quantise(np.float32([2.5 / 255]))[0] == np.rint(np.float32(2.5 / 255) * np.float32(255))


def test_threshold_plan_modes_and_draw_order():
    np.random.seed(5)
    want = [np.random.uniform(0.1, 0.4) for _ in range(7)]
    np.random.seed(5)
    mode, r, low, high = canny.threshold_plan(7)
    assert mode == 2 and r == want
    assert np.random.uniform(0.1, 0.4) == np.random.RandomState(5).uniform(0.1, 0.4, 8)[-1]
    # the reference draws only with both thresholds None and random_threshold not the False object
    state = _stream_state()
    assert canny.threshold_plan(3, random_threshold=False) == (1, None, 0.0, 0.0)
    assert canny.threshold_plan(3, 10, 20.5) == (0, None, 10.0, 20.5)
    assert canny.threshold_plan(3, 10, 20, random_threshold=False)[0] == 0
    assert _stream_state() == state
    assert canny.threshold_plan(2, random_threshold=0)[0] == 2                # 0 is not False
    assert canny.threshold_plan(2, random_threshold=None)[0] == 2


@pytest.mark.parametrize("m", [0.0, 0.5, 1.0, 81.5, 100.0, 127.5, 191.0, 200.0, 255.0])
def test_threshold_arithmetic(m):
    """The reference's expressions in float64, as the device computes them: the median of a uint8 array with an even
    count is the mean of the two middle values."""
    a, b = int(math.floor(m)), int(math.ceil(m))
    img = np.array([0, a, b, 255], np.uint8) if a != b else np.array([0, a, 255], np.uint8)
    assert np.median(img) == m
    low, high = co.thresholds(img, random_threshold=False)
    assert (low, high) == (int(max(0, (1 - 0.33) * m)), int(min(255, (1 + 0.33) * m)))
    for r in (0.1, 0.25, 0.4, 0.39999999999999997, 0.1234567):
        low, high = co.thresholds(img, r=r)
        assert low == int(max(0, (1 - r) * m)) and high == 2 * low


def test_cv_thresholds_swap_and_floor():
    assert co.cv_thresholds(150, 40) == (40, 150)
    assert co.cv_thresholds(35.7, 90.2) == (35, 90)
    assert co.cv_thresholds(90.2, 35.7) == (35, 90)
    assert co.cv_thresholds(-0.5, 3) == (-1, 3)


def test_oracle_hysteresis_joins_chains_of_any_length():
    """A weak staircase touching a strong pixel at one end is kept whole; the same chain without it is dropped."""
    cls = np.zeros((40, 300), np.uint8)
    ys = (np.arange(300) // 10) % 40
    cls[ys, np.arange(300)] = 1
    assert co.hysteresis(cls).sum() == 0
    cls[ys[0], 0] = 2
    assert co.hysteresis(cls).sum() == 300


def test_refusals():
    with pytest.raises(ValueError, match="both thresholds"):
        canny.threshold_plan(1, 10, None)
    with pytest.raises(ValueError, match="both thresholds"):
        canny.threshold_plan(1, None, 10)
    for bad in (float("nan"), "10", True):
        with pytest.raises(ValueError, match="real numbers"):
            canny.threshold_plan(1, bad, 20)
    det = canny.CannyDetector()
    with pytest.raises(lib.VgenError, match="CUDA fp32"):
        det(torch.rand(8, 8, 3))                           # CPU tensor: no fallback
    with pytest.raises(lib.VgenError, match="CUDA fp32"):
        det(torch.rand(8, 8, 3, dtype=torch.float64))
    with pytest.raises(ValueError, match="uint8"):
        det(np.zeros((8, 8, 3), np.float32))
    with pytest.raises(ValueError, match="uint8"):
        det(np.zeros((8, 8, 4), np.uint8))
    with pytest.raises(ValueError, match="Tensor or np.ndarray"):
        det([[0, 1]])
    with pytest.raises(lib.VgenError, match="CUDA fp32"):
        canny.canny_video(torch.rand(1, 2, 3, 8, 8))
    with pytest.raises(lib.VgenError, match="CUDA fp32"):
        canny.canny_video(np.zeros((1, 2, 3, 8, 8), np.float32))
    with pytest.raises(lib.VgenError, match="CUDA fp32 or uint8"):
        ops.canny(torch.rand(1, 3, 8, 8), 1)


def test_package_exports():
    import vgen_b200
    assert vgen_b200.CannyDetector is canny.CannyDetector and vgen_b200.canny_video is canny.canny_video
    assert "vgen_canny" in lib.declared_symbols()
