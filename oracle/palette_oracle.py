"""numpy restatement of the VideoComposer colour-palette annotator (tools/annotator/histogram/palette.py `Palette`) and of
the scikit-image 0.22.0 colour conversions it calls (skimage is not a dependency here, so this part is restated from
skimage's documented algorithms, not pinned against it): rgb2xyz / xyz2lab / lab2xyz / xyz2rgb with the D65 2-degree
white, hsv2rgb, and img_as_float's uint8 scaling.  The distances are sklearn's euclidean_distances(squared=True), which
is installed, so the histogram path is the reference's own host procedure.  tools/make_golden_histogram.py runs the
reference's palette.py on top of these conversions (as a `skimage.color` stub) and checks this restatement against it.
"""
from __future__ import annotations

import numpy as np
from scipy import linalg
from sklearn.metrics import euclidean_distances

xyz_from_rgb = np.array([[0.412453, 0.357580, 0.180423],
                         [0.212671, 0.715160, 0.072169],
                         [0.019334, 0.119193, 0.950227]])
rgb_from_xyz = linalg.inv(xyz_from_rgb)
WHITE_D65_2 = np.array((0.95047, 1., 1.08883))


def img_as_float(a):
    a = np.asanyarray(a)
    if a.dtype == np.uint8:
        return np.multiply(a, 1. / 255, dtype=np.float64)
    if a.dtype == np.float16:
        return a.astype(np.float32)
    return a


def rgb2xyz(rgb):
    arr = img_as_float(rgb).copy()
    mask = arr > 0.04045
    arr[mask] = np.power((arr[mask] + 0.055) / 1.055, 2.4)
    arr[~mask] /= 12.92
    return arr @ xyz_from_rgb.T.astype(arr.dtype)


def xyz2lab(xyz):
    arr = img_as_float(xyz)
    arr = arr / WHITE_D65_2.astype(arr.dtype)
    mask = arr > 0.008856
    arr[mask] = np.cbrt(arr[mask])
    arr[~mask] = 7.787 * arr[~mask] + 16. / 116.
    x, y, z = arr[..., 0], arr[..., 1], arr[..., 2]
    return np.concatenate([c[..., np.newaxis] for c in (116. * y - 16., 500.0 * (x - y), 200.0 * (y - z))], axis=-1)


def rgb2lab(rgb):
    return xyz2lab(rgb2xyz(rgb))


def lab2xyz(lab):
    arr = img_as_float(lab).copy()
    L, a, b = arr[..., 0], arr[..., 1], arr[..., 2]
    y = (L + 16.) / 116.
    x = a / 500. + y
    z = y - b / 200.
    z[z < 0] = 0
    out = np.stack([x, y, z], axis=-1)
    mask = out > 0.2068966
    out[mask] = np.power(out[mask], 3.)
    out[~mask] = (out[~mask] - 16.0 / 116.) / 7.787
    return out * WHITE_D65_2


def xyz2rgb(xyz):
    arr = img_as_float(xyz) @ rgb_from_xyz.T.astype(np.float64)
    mask = arr > 0.0031308
    arr[mask] = 1.055 * np.power(arr[mask], 1 / 2.4) - 0.055
    arr[~mask] *= 12.92
    np.clip(arr, 0, 1, out=arr)
    return arr


def lab2rgb(lab):
    return xyz2rgb(lab2xyz(lab))


def hsv2rgb(hsv):
    arr = img_as_float(hsv)
    sector = np.floor(arr[..., 0] * 6)
    f = arr[..., 0] * 6 - sector
    v = arr[..., 2]
    p = v * (1 - arr[..., 1])
    q = v * (1 - f * arr[..., 1])
    t = v * (1 - (1 - f) * arr[..., 1])
    sel = np.stack([sector] * 3, axis=-1).astype(np.uint8) % 6
    return np.choose(sel, np.stack([np.stack(c, axis=-1) for c in
                                    ((v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q))]))


HUE_TABLES = {8: (0., 0.10, 0.15, 0.28, 0.51, 0.58, 0.77, 0.85),
              9: (0., 0.10, 0.15, 0.28, 0.49, 0.54, 0.60, 0.7, 0.87),
              10: (0., 0.10, 0.15, 0.28, 0.49, 0.54, 0.60, 0.66, 0.76, 0.87),
              11: (0.0, 0.0833, 0.166, 0.25, 0.333, 0.5, 0.56333, 0.666, 0.73, 0.803, 0.916)}


class PaletteOracle:
    """The palette tables and the per-frame host procedure of the reference's Palette."""

    def __init__(self, num_hues=11, num_sat=5, num_light=4):
        rows = num_sat + 2 * num_light
        hues = np.array(HUE_TABLES[num_hues]) if num_hues in HUE_TABLES else np.linspace(0, 1, num_hues + 1)[:-1]
        sats = np.array(list(np.linspace(0, 1, num_sat + 2)[1:-1]) + [1.0] * (num_light + 1) + [0.4] * (num_light - 1))
        lsteps = np.linspace(1, 0.2, num_light + 2)
        lights = np.array([1.0] * (num_sat + 1) + list(lsteps[1:-1]) + list(lsteps[1:-2]))
        hsv = np.stack(np.broadcast_arrays(hues[np.newaxis, :], sats[:, np.newaxis], lights[:, np.newaxis]), axis=-1)
        grid = hsv2rgb(hsv.astype(np.float64))                      # [rows, hues, 3]
        grey = np.linspace(1, 0, rows)[:, np.newaxis, np.newaxis] * np.ones((1, 1, 3))
        self.thumbnail = np.concatenate([grid, grey], axis=1)
        self.rgb = np.concatenate([np.swapaxes(grid, 0, 1).reshape(-1, 3), grey[:, 0, :]])
        self.lab = rgb2lab(self.rgb[np.newaxis]).squeeze()
        self.lab_dists = euclidean_distances(self.lab, squared=True)

    def nearest(self, rgb_img):
        """Each pixel's palette index: argmin of euclidean_distances(lab, palette lab, squared=True) -> (indices, distances)."""
        lab = rgb2lab(rgb_img).reshape(-1, 3)
        d = euclidean_distances(lab, self.lab, squared=True)
        return np.argmin(d, axis=1), d

    def histogram(self, rgb_img, sigma=20):
        return self.histogram_of(self.nearest(rgb_img)[0], sigma)

    def histogram_of(self, idx, sigma=20):
        """The (smoothed) histogram of a frame's nearest-entry indices."""
        hist = np.bincount(idx, minlength=self.lab.shape[0]) / float(idx.shape[0])
        if sigma > 0:
            w = np.exp(-self.lab_dists / (2.0 * sigma ** 2))
            w /= w.sum(1, keepdims=True)
            hist = (w * hist).sum(1)
            hist[hist < 1e-5] = 0
        return hist

    def quantize_image(self, rgb_img):
        idx, _ = self.nearest(rgb_img)
        return lab2rgb(self.lab[idx].reshape(np.shape(rgb_img)))
