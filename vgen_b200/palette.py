"""The VideoComposer colour-palette annotator on the device: a drop-in for tools/annotator/histogram/palette.py `Palette`,
and `histogram_video` for whole videos.

The reference computes the UNet's `histogram` condition per frame on the host: skimage's rgb2lab of every pixel in
float64, sklearn's euclidean_distances against the 156 palette colours (a pixels x 156 float64 matrix), argmin, bincount
and a 156 x 156 Gaussian smoothing.  Here the palette's tables are built once on the host in float64, and one call
(csrc/palette.cu, `vgen_palette_histogram`) reads the frames in place, computes each pixel's Lab in fp64, finds its
nearest entry, counts, normalises and smooths on the device.

The host tables restate scikit-image 0.22.0 (the version the reference pins): rgb2xyz (sRGB linearisation with the
0.04045 threshold and the 2.4 power, xyz_from_rgb), xyz2lab (D65, 2-degree observer, the 0.008856 threshold, cube root or
7.787 t + 16/116), lab2rgb and hsv2rgb, with its dtype rule that uint8 input is scaled by 1/255 (img_as_float).
`lab_dists` is sklearn's euclidean_distances(lab, squared=True): -2 X.X^T + |x|^2 + |y|^2, clipped at 0, zero diagonal.
There is no CPU fallback: without a CUDA device `histogram` and `quantize_image` raise `VgenError`.
"""
from __future__ import annotations

import numpy as np
import torch

from . import lib as _l
from . import ops

# skimage.color.colorconv (0.22.0): sRGB (D65) -> CIE XYZ, and the D65 / 2-degree reference white
XYZ_FROM_RGB = np.array([[0.412453, 0.357580, 0.180423],
                         [0.212671, 0.715160, 0.072169],
                         [0.019334, 0.119193, 0.950227]])
D65_2 = np.array([0.95047, 1.0, 1.08883])

_HUES = {8: [0., 0.10, 0.15, 0.28, 0.51, 0.58, 0.77, 0.85],
         9: [0., 0.10, 0.15, 0.28, 0.49, 0.54, 0.60, 0.7, 0.87],
         10: [0., 0.10, 0.15, 0.28, 0.49, 0.54, 0.60, 0.66, 0.76, 0.87],
         11: [0.0, 0.0833, 0.166, 0.25, 0.333, 0.5, 0.56333, 0.666, 0.73, 0.803, 0.916]}


def _as_float(a):
    """skimage's img_as_float as rgb2lab / hsv2rgb apply it: uint8 -> float64 a * (1 / 255); floats unchanged."""
    a = np.asarray(a)
    if a.dtype == np.uint8:
        return np.multiply(a, 1.0 / 255, dtype=np.float64)
    if a.dtype.kind != "f":
        raise ValueError(f"Palette: expected uint8 or floating-point colours, got {a.dtype}")
    return a


def _linearise(a):
    """The sRGB transfer function of rgb2xyz, on a float array (copied)."""
    a = np.array(a, copy=True)
    hi = a > 0.04045
    a[hi] = np.power((a[hi] + 0.055) / 1.055, 2.4)
    a[~hi] /= 12.92
    return a


def rgb2lab(rgb):
    """skimage.color.rgb2lab (D65, 2-degree observer) of [..., 3] colours."""
    xyz = _linearise(_as_float(rgb)) @ XYZ_FROM_RGB.T.astype(np.float64)
    t = xyz / D65_2
    hi = t > 0.008856
    t[hi] = np.cbrt(t[hi])
    t[~hi] = 7.787 * t[~hi] + 16. / 116.
    x, y, z = t[..., 0], t[..., 1], t[..., 2]
    return np.stack([116. * y - 16., 500.0 * (x - y), 200.0 * (y - z)], axis=-1)


def lab2rgb(lab):
    """skimage.color.lab2rgb (D65, 2-degree observer): lab2xyz (negative z clipped to 0), xyz2rgb, clipped to [0, 1]."""
    lab = np.asarray(lab, dtype=np.float64)
    y = (lab[..., 0] + 16.) / 116.
    x = lab[..., 1] / 500. + y
    z = y - lab[..., 2] / 200.
    z = np.where(z < 0, 0.0, z)
    xyz = np.stack([x, y, z], axis=-1)
    hi = xyz > 0.2068966
    xyz[hi] = np.power(xyz[hi], 3.)
    xyz[~hi] = (xyz[~hi] - 16.0 / 116.) / 7.787
    xyz *= D65_2
    import scipy.linalg   # skimage builds rgb_from_xyz with scipy.linalg.inv
    rgb = xyz @ scipy.linalg.inv(XYZ_FROM_RGB).T.astype(np.float64)
    hi = rgb > 0.0031308
    rgb[hi] = 1.055 * np.power(rgb[hi], 1 / 2.4) - 0.055
    rgb[~hi] *= 12.92
    return np.clip(rgb, 0, 1)


def hsv2rgb(hsv):
    """skimage.color.hsv2rgb of [..., 3] colours (sector floor(6 h) mod 6 picks (v, t, p), (q, v, p), ...)."""
    a = _as_float(hsv)
    h, s, v = a[..., 0], a[..., 1], a[..., 2]
    sector = np.floor(h * 6)
    frac = h * 6 - sector
    p, q, t = v * (1 - s), v * (1 - frac * s), v * (1 - (1 - frac) * s)
    table = np.stack([np.stack(c, axis=-1) for c in ((v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q))])
    idx = sector.astype(np.uint8) % 6
    return np.take_along_axis(table, idx[None, ..., None].repeat(3, axis=-1), axis=0)[0]


def squared_distances(x, y=None):
    """sklearn.metrics.euclidean_distances(x, y, squared=True) for float64 rows: -2 x.y^T + |x|^2 + |y|^2 in that order,
    clipped at 0; y None means y is x, whose diagonal is set to 0."""
    same = y is None
    y = x if same else y
    xx = np.einsum("ij,ij->i", x, x)[:, np.newaxis]
    yy = xx.reshape(1, -1) if same else np.einsum("ij,ij->i", y, y)[np.newaxis, :]
    d = -2 * (x @ y.T)
    d += xx
    d += yy
    np.maximum(d, 0, out=d)
    if same:
        np.fill_diagonal(d, 0)
    return d


def rgb2hex(rgb):
    return "#%02x%02x%02x" % tuple(int(round(255.0 * u)) for u in rgb)


class Palette:
    """`Palette(num_hues=11, num_sat=5, num_light=4)` as the reference: a (num_sat + 2 num_light) x (num_hues + 1) grid of
    colours whose last column is a grey ramp.  Attributes rgb / lab ([K, 3] float64, hue-major within the grid, then the
    greys), hex, lab_dists ([K, K]) and thumbnail ([rows, num_hues + 1, 3]).  The default has K = 156 = the UNet's
    hist_dim; the device path takes any K up to 156."""

    def __init__(self, num_hues=11, num_sat=5, num_light=4):
        rows = num_sat + 2 * num_light
        hue_row = _HUES.get(num_hues)
        if hue_row is None:
            hue_row = np.linspace(0, 1, num_hues + 1)[:-1]
        sat_col = np.concatenate([np.linspace(0, 1, num_sat + 2)[1:-1], [1], [1] * num_light, [0.4] * (num_light - 1)])
        ramp = np.linspace(1, 0.2, num_light + 2)
        light_col = np.concatenate([[1] * num_sat, [1], ramp[1:-1], ramp[1:-2]])
        hsv = np.empty((rows, num_hues, 3))
        hsv[..., 0] = np.asarray(hue_row, dtype=np.float64)[np.newaxis, :]
        hsv[..., 1] = sat_col[:, np.newaxis]
        hsv[..., 2] = light_col[:, np.newaxis]
        grid = hsv2rgb(hsv)
        grey = np.repeat(np.linspace(1, 0, rows)[:, np.newaxis, np.newaxis], 3, axis=2)
        self.thumbnail = np.concatenate([grid, grey], axis=1)
        # column-major flattening of the grid (rgb.T.reshape(3, -1).T): hue by hue, top row first; then the greys
        self.rgb = np.concatenate([grid.transpose(1, 0, 2).reshape(-1, 3), grey.reshape(-1, 3)])
        self.lab = rgb2lab(self.rgb[np.newaxis]).squeeze()
        self.hex = [rgb2hex(u) for u in self.rgb]
        self.lab_dists = squared_distances(self.lab)
        self._device = {}

    # ------------------------------------------------------------------------------------------ device tables
    def smoothing_weights(self, sigma):
        """The row-normalised exp(-lab_dists / 2 sigma^2) of Palette.histogram, or None for sigma <= 0 (no smoothing)."""
        if not sigma > 0:
            return None
        w = np.exp(-self.lab_dists / (2.0 * sigma ** 2))
        return w / w.sum(1)[:, np.newaxis]

    def _tables(self, device, sigma=None):
        t = self._device.get(device)
        if t is None:
            lab4 = np.concatenate([self.lab, np.einsum("ij,ij->i", self.lab, self.lab)[:, np.newaxis]], axis=1)
            lin = _linearise(_as_float(np.arange(256, dtype=np.uint8)))
            f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(device)  # noqa: E731
            t = self._device[device] = {"lab4": f64(lab4), "lin": f64(lin), "qrgb": f64(lab2rgb(self.lab)), "w": {}}
        if sigma is not None and sigma > 0 and float(sigma) not in t["w"]:
            t["w"][float(sigma)] = torch.from_numpy(self.smoothing_weights(float(sigma))).to(device)
        return t

    def device_histogram(self, frames, sigma=20, out_dtype=torch.float32):
        """Histograms of frames [n, 3, h, w] (CUDA fp32 / fp64 in [0, 1] or uint8, any strides) -> [n, K] on the device."""
        t = self._tables(frames.device, sigma)
        w = t["w"][float(sigma)] if sigma > 0 else None
        return ops.palette_histogram(frames, t["lab4"], t["lin"], w, out_dtype)

    @staticmethod
    def _frames_of(rgb_img, what):
        """An (..., 3) image (np.ndarray or CUDA tensor) -> a [1, 3, 1, pixels] CUDA view of it."""
        if isinstance(rgb_img, np.ndarray):
            a = rgb_img
            if a.dtype == np.float16:
                a = a.astype(np.float32)
            if a.dtype not in (np.uint8, np.float32, np.float64):
                raise ValueError(f"Palette.{what}: expected uint8 or floating-point pixels, got {a.dtype}")
            t = torch.from_numpy(np.ascontiguousarray(a))
            if not torch.cuda.is_available():
                raise _l.VgenError(f"Palette.{what} runs on the device and no CUDA device is available")
            t = t.cuda()
        elif isinstance(rgb_img, torch.Tensor):
            t = rgb_img if rgb_img.dtype != torch.float16 else rgb_img.float()
        else:
            raise ValueError(f"Palette.{what}: expected an np.ndarray or torch.Tensor, got {type(rgb_img).__name__}")
        if t.dim() < 2 or t.shape[-1] != 3:
            raise ValueError(f"Palette.{what}: expected (..., 3) RGB pixels, got {tuple(t.shape)}")
        return t.reshape(1, -1, 3).permute(0, 2, 1).unsqueeze(2)

    # ------------------------------------------------------------------------------------------ the reference's calls
    def histogram(self, rgb_img, sigma=20):
        """Palette.histogram: the [K] float64 np.ndarray of an (h, w, 3) image (uint8, or floats in [0, 1]), computed on
        the device.  Float32 pixels are widened to float64 before the conversion (skimage would convert them in float32)."""
        frames = self._frames_of(rgb_img, "histogram")
        return self.device_histogram(frames, sigma, torch.float64)[0].cpu().numpy()

    def quantize_image(self, rgb_img):
        """Palette.quantize_image: every pixel replaced by lab2rgb of its nearest palette entry, float64 np.ndarray of the
        image's shape."""
        frames = self._frames_of(rgb_img, "quantize_image")
        t = self._tables(frames.device)
        out = ops.palette_quantize(frames, t["lab4"], t["qrgb"], t["lin"])
        return out.cpu().numpy().reshape(tuple(rgb_img.shape))

    def get_palette_image(self, hist, percentile=90, width=200, height=50):
        """A height x width strip of the entries above the histogram's percentile, largest first, each as wide as its
        share of them (float64 [height, width, 3], zero-padded on the right)."""
        hist = hist.detach().cpu().numpy() if isinstance(hist, torch.Tensor) else np.asarray(hist)
        order = np.argsort(-hist)
        keep = order[hist[order] > np.percentile(hist, percentile)]
        if keep.size == 0:
            raise ValueError("get_palette_image: no histogram entry lies above the percentile")
        share = hist[keep] / hist[keep].sum()
        strip = np.repeat(self.rgb[keep], np.array(share * width, dtype=int), axis=0)
        out = np.zeros((height, max(width, strip.shape[0]), 3))
        out[:, :strip.shape[0]] = strip[np.newaxis]
        return out

    def export(self, dirname):
        raise NotImplementedError("vgen_b200 Palette.export writes image files through skimage.io, which is not a "
                                  "dependency here")


_DEFAULT = None


def histogram_video(frames, sigma=20, palette=None):
    """The UNet's `histogram` condition of videos on the device: frames CUDA fp32 [b, f, 3, H, W] in [0, 1] (the
    VideoComposer engines' misc_data layout) or uint8 [b, f, H, W, 3] -> fp32 [b, f, K] (K = 156 for the default
    palette), equal to Palette.histogram of every frame in (b, f) order.  Nothing is read back to the host."""
    global _DEFAULT
    if palette is None:
        if _DEFAULT is None:
            _DEFAULT = Palette()
        palette = _DEFAULT
    if not isinstance(frames, torch.Tensor) or not frames.is_cuda:
        what = f"{frames.dtype} on {frames.device}" if isinstance(frames, torch.Tensor) else type(frames).__name__
        raise _l.VgenError(f"histogram_video: expected a CUDA tensor, got {what}")
    if frames.dtype == torch.float32 and frames.dim() == 5 and frames.shape[2] == 3:
        v = frames
    elif frames.dtype == torch.uint8 and frames.dim() == 5 and frames.shape[4] == 3:
        v = frames.permute(0, 1, 4, 2, 3)
    else:
        raise ValueError(f"histogram_video: expected fp32 [b, f, 3, H, W] or uint8 [b, f, H, W, 3], got {frames.dtype} "
                         f"{tuple(frames.shape)}")
    b, f = v.shape[:2]
    return palette.device_histogram(v.flatten(0, 1), sigma, torch.float32).view(b, f, -1)
