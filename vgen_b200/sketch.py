"""H100-native sketch annotators of the VideoComposer engines: drop-ins for `PiDiNet` / `pidinet_bsd` of
tools/annotator/sketch/pidinet.py:527-746 and `SketchSimplification` / `sketch_simplification_gan` of
tools/annotator/sketch/sketch_simplification.py:14-90 (inference_{tft2v,videolcm}_vcomposer_entrance.py build the pair for
every config that lists 'sketch' or 'single_sketch' and run `1 - cleaner(1 - pidinet((x - mean) / std))` per chunk).

  PiDiNet (converted vanilla-CNN form, sa=True, int dil): init conv (im2col + GEMM) -> 16 blocks
  [maxpool2 ->] depthwise kxk -> ReLU -> 1x1 -> + x | shortcut(x) -> per stage CDCM (ReLU, 1x1, the four dilated 3x3
  convs as ONE 33-tap conv) -> CSAM + MapReduce -> bilinear resize of the four side maps, 4 -> 1 classifier, sigmoid.
  SketchSimplification: (x - mean) / std -> 22 convs with ReLU (stride-2 ones by im2col + GEMM, ConvTranspose2d(4, 2, 1)
  as four 2x2-tap output phases written in place) -> 3x3 conv to one channel + sigmoid.

Same constructors, parameter names, shapes and order as the reference, so reference checkpoints load with `strict=True`.
The forward takes [n, C, H, W] on the GPU (NCHW-contiguous or channels_last; C = 3 for PiDiNet, 1 for the cleaner) in
the module's parameter dtype and returns [n, 1, H, W] in that dtype.  Every op is a kernel of libvgen_b200.so;
activations are fp16 channels-last with fp32 accumulation.  Channel counts are zero-padded to multiples of 64 by the
pack (zero weights and zero bias, so the pad channels stay exactly zero).  No CPU path: a CPU input raises VgenError.
"""
from __future__ import annotations

import torch

from . import ops
from .graph import graphed
from .params import SpecModule

__all__ = ["PiDiNet", "pidinet_bsd", "SketchSimplification", "sketch_simplification_gan"]

CARV4 = ["cd", "ad", "rd", "cv"] * 4   # pidinet.py CONFIGS['carv4'], layer0 .. layer15
_CDCM_DILATIONS = (5, 7, 9, 11)


def _pad64(c):
    return (c + 63) // 64 * 64


def _padded(t, shape):
    """t zero-padded at the end of every dimension to `shape` (fp32)."""
    out = torch.zeros(shape, dtype=torch.float32, device=t.device)
    out[tuple(slice(0, s) for s in t.shape)] = t.detach().float()
    return out


# ---- PDC -> vanilla conversion (pretrained PiDiNet checkpoints store the pixel-difference form) ----------------------------
_RING = [0, 1, 2, 5, 8, 7, 6, 3]   # the eight off-centre taps of a 3x3 kernel (flat index), clockwise from the top left


def convert_pdc(op, w):
    """The vanilla conv weight equivalent to pixel-difference conv `op` with weight w [co, ci, 3, 3]:
      cv: w itself;
      cd: the centre tap minus the sum of all taps (y = conv(x, w) - x_centre * sum(w));
      ad: w minus its clockwise permutation (each ring tap minus the ring tap before it clockwise; the centre cancels);
      rd: a 5x5 kernel whose outer ring (stride 2) holds taps 1..8 of w in raster order, the inner ring their negatives, and
          a zero centre."""
    w = w.detach().clone()
    co, ci = w.shape[:2]
    if op == "cv":
        return w
    flat = w.reshape(co, ci, 9)
    if op == "cd":
        flat[:, :, 4] = flat[:, :, 4] - w.sum(dim=(2, 3))
        return flat.reshape(co, ci, 3, 3)
    if op == "ad":
        prev = list(range(9))
        for i, pos in enumerate(_RING):
            prev[pos] = _RING[i - 1]
        return (flat - flat[:, :, prev]).reshape(co, ci, 3, 3)
    if op == "rd":
        outer = [5 * y + x for y in (0, 2, 4) for x in (0, 2, 4) if (y, x) != (2, 2)]
        inner = [5 * y + x for y in (1, 2, 3) for x in (1, 2, 3) if (y, x) != (2, 2)]
        buf = torch.zeros(co, ci, 25, dtype=w.dtype, device=w.device)
        buf[:, :, outer] = flat[:, :, 1:]
        buf[:, :, inner] = -flat[:, :, 1:]
        return buf.reshape(co, ci, 5, 5)
    raise ValueError(f"unknown pixel-difference op {op!r}")


def convert_pidinet(state_dict, pdcs=CARV4):
    """A PDC-format PiDiNet state dict -> the converted vanilla form (init_block and every blockX_Y.conv1)."""
    names = ["init_block.weight"] + [f"block{s}_{b}.conv1.weight" for s, nb in ((1, 3), (2, 4), (3, 4), (4, 4))
                                     for b in range(1, nb + 1)]
    layer = {nm: i for i, nm in enumerate(names)}
    out = {}
    for k, v in state_dict.items():
        hit = [nm for nm in names if nm in k]
        out[k] = convert_pdc(pdcs[layer[hit[0]]], v) if hit else v
    return out


# ---- PiDiNet ---------------------------------------------------------------------------------------------------------------
def _blocks(inplane):
    """(name, cin, cout, pdc index, stride 2) of the 15 PDC blocks."""
    c1, c2, c4 = inplane, 2 * inplane, 4 * inplane
    out = [(f"block1_{i}", c1, c1, i, False) for i in (1, 2, 3)]
    for s, cin, c in ((2, c1, c2), (3, c2, c4), (4, c4, c4)):
        out += [(f"block{s}_1", cin, c, 4 * (s - 1), True)]
        out += [(f"block{s}_{i}", c, c, 4 * (s - 1) + i - 1, False) for i in (2, 3, 4)]
    return out


def pidinet_spec(inplane, pdcs, dil):
    """(name, shape) in the order of the reference PiDiNet(convert=True, sa=True, dil=int).state_dict()."""
    k0 = 5 if pdcs[0] == "rd" else 3
    spec = [("init_block.weight", (inplane, 3, k0, k0))]
    for nm, cin, cout, li, s2 in _blocks(inplane):
        k = 5 if pdcs[li] == "rd" else 3
        if s2:
            spec += [(nm + ".shortcut.weight", (cout, cin, 1, 1)), (nm + ".shortcut.bias", (cout,))]
        spec += [(nm + ".conv1.weight", (cin, 1, k, k)), (nm + ".conv2.weight", (cout, cin, 1, 1))]
    fuse = [inplane, 2 * inplane, 4 * inplane, 4 * inplane]
    spec += [s for i in range(4) for s in ((f"conv_reduces.{i}.conv.weight", (1, dil, 1, 1)), (f"conv_reduces.{i}.conv.bias", (1,)))]
    spec += [s for i in range(4) for s in ((f"attentions.{i}.conv1.weight", (4, dil, 1, 1)), (f"attentions.{i}.conv1.bias", (4,)),
                                           (f"attentions.{i}.conv2.weight", (1, 4, 3, 3)))]
    for i in range(4):
        spec += [(f"dilations.{i}.conv1.weight", (dil, fuse[i], 1, 1)), (f"dilations.{i}.conv1.bias", (dil,))]
        spec += [(f"dilations.{i}.conv2_{j}.weight", (dil, dil, 3, 3)) for j in (1, 2, 3, 4)]
    return spec + [("classifier.weight", (1, 4, 1, 1)), ("classifier.bias", (1,))]


def _cdcm_taps():
    """The 33 distinct (dy, dx) offsets of conv2_1 + conv2_2 + conv2_3 + conv2_4 (dilations 5, 7, 9, 11): the shared
    centre first, then each conv's eight off-centre taps in raster order."""
    taps = [(0, 0)]
    for d in _CDCM_DILATIONS:
        taps += [((ky - 1) * d, (kx - 1) * d) for ky in range(3) for kx in range(3) if (ky, kx) != (1, 1)]
    return taps


def _nhwc16(x, c):
    """[n, c, H, W] fp32 / fp16, NCHW-contiguous or channels_last -> fp16 [n, H, W, c]."""
    n, _, H, W = x.shape
    if x.is_contiguous():
        return ops.cp_to_pc(x, n, c, H * W).view(n, H, W, c)
    if x.is_contiguous(memory_format=torch.channels_last):
        nhwc = x.permute(0, 2, 3, 1)
        return nhwc if x.dtype == torch.float16 else ops.cp_to_pc(nhwc, n * H * W, c, 1).view(n, H, W, c)
    raise ValueError("x must be NCHW-contiguous or channels_last")


def _check_input(name, x, c, dt):
    if x.dim() != 4 or x.shape[1] != c:
        raise ValueError(f"{name}: expected [n, {c}, H, W], got {tuple(x.shape)}")
    if not x.is_cuda:
        raise ops._l.VgenError(f"vgen_b200 {name}: x must be a CUDA tensor (no CPU path exists)")
    if x.dtype not in (torch.float16, torch.float32) or x.dtype != dt:
        raise TypeError(f"{name}: x is {x.dtype}, the module's parameters are {dt}")


class PiDiNet(SpecModule):
    r"""PiDiNet in its converted vanilla-CNN form (pidinet.py:557-704) on the native path."""

    def __init__(self, inplane, pdcs, dil=None, sa=False, convert=False):
        super().__init__()
        if not convert or not sa or not isinstance(dil, int):
            raise NotImplementedError("vgen_b200 PiDiNet: only the converted vanilla-CNN form with sa=True and an int dil "
                                      f"(what pidinet_bsd() builds) runs natively; got convert={convert}, sa={sa}, dil={dil!r}")
        pdcs = list(pdcs)
        if len(pdcs) != 16 or any(p not in ("cv", "cd", "ad", "rd") for p in pdcs):
            raise ValueError(f"PiDiNet: pdcs must be 16 of 'cv' | 'cd' | 'ad' | 'rd', got {pdcs}")
        self.inplane, self.pdcs, self.dil, self.sa, self.convert = inplane, pdcs, dil, sa, convert
        self.fuseplanes = [inplane, 2 * inplane, 4 * inplane, 4 * inplane]
        self._build_params(pidinet_spec(inplane, pdcs, dil))

    def _k(self, i):
        return 5 if self.pdcs[i] == "rd" else 3

    def _pack(self):
        dev = self.device
        if dev.type != "cuda":
            raise ops._l.VgenError("vgen_b200 PiDiNet forward needs the model on a CUDA device (no CPU path exists)")
        sd = {k: v.detach().to(device=dev, dtype=torch.float32) for k, v in self.state_dict().items()}
        f16 = lambda t: t.to(torch.float16).contiguous()  # noqa: E731
        W = {}
        k0, c = self._k(0), self.inplane
        w0 = sd["init_block.weight"].permute(0, 2, 3, 1).reshape(c, k0 * k0 * 3)
        W["init.w"] = f16(_padded(w0, (_pad64(c), _pad64(k0 * k0 * 3))))
        for nm, cin, cout, li, s2 in _blocks(self.inplane):
            k = self._k(li)
            W[nm + ".dw"] = _padded(sd[nm + ".conv1.weight"].reshape(cin, k * k).t(), (k * k, _pad64(cin))).contiguous()
            W[nm + ".pw"] = f16(_padded(sd[nm + ".conv2.weight"].flatten(1), (_pad64(cout), _pad64(cin))))
            if s2:
                W[nm + ".sc.w"] = f16(_padded(sd[nm + ".shortcut.weight"].flatten(1), (_pad64(cout), _pad64(cin))))
                W[nm + ".sc.b"] = _padded(sd[nm + ".shortcut.bias"], (_pad64(cout),))
        d, dp = self.dil, _pad64(self.dil)
        for i, cin in enumerate(self.fuseplanes):
            q = f"dilations.{i}."
            W[q + "c1.w"] = f16(_padded(sd[q + "conv1.weight"].flatten(1), (dp, _pad64(cin))))
            W[q + "c1.b"] = _padded(sd[q + "conv1.bias"], (dp,))
            # one 33-tap conv: the four centre taps are added in fp32 and rounded once
            ws = [sd[q + f"conv2_{j}.weight"] for j in (1, 2, 3, 4)]
            taps = [ws[0][:, :, 1, 1] + ws[1][:, :, 1, 1] + ws[2][:, :, 1, 1] + ws[3][:, :, 1, 1]]
            for wj in ws:
                taps += [wj[:, :, ky, kx] for ky in range(3) for kx in range(3) if (ky, kx) != (1, 1)]
            W[q + "c2.w"] = f16(torch.cat([_padded(t, (dp, dp)) for t in taps], dim=1))
            a = f"attentions.{i}."
            W[a + "w1"] = _padded(sd[a + "conv1.weight"].flatten(1), (4, dp)).contiguous()
            W[a + "b1"] = sd[a + "conv1.bias"].contiguous()
            W[a + "w2"] = sd[a + "conv2.weight"].reshape(-1).contiguous()
            r = f"conv_reduces.{i}.conv."
            W[r + "w"] = _padded(sd[r + "weight"].reshape(-1), (dp,))
            W[r + "b"] = sd[r + "bias"].contiguous()
        W["cls"] = torch.cat([sd["classifier.weight"].reshape(-1), sd["classifier.bias"]]).contiguous()
        W["taps"] = _cdcm_taps()
        self._packed = W
        return W

    def forward(self, x):
        """x [n, 3, H, W] CUDA (the engines' normalised frames), NCHW-contiguous or channels_last, in the parameter dtype,
        H, W >= 8 -> edge map [n, 1, H, W] in x's dtype."""
        if x.dim() == 4 and (x.shape[2] < 8 or x.shape[3] < 8):
            raise ValueError(f"PiDiNet: H and W must be at least 8 (three 2x2 max-pools), got {tuple(x.shape[2:])}")
        _check_input("PiDiNet", x, 3, next(self.parameters()).dtype)
        img = _nhwc16(x, 3)
        if self._packed is None:
            self._pack()
        return self._forward_nhwc(img, x.dtype == torch.float32)

    @graphed
    @torch.no_grad()
    def _forward_nhwc(self, img, out_f32):
        W = self._packed
        n, H, Wd, _ = img.shape
        k0 = self._k(0)
        col = ops.im2col(img, k0, k0, 1, k0 // 2, k0 // 2, H, Wd, W["init.w"].shape[1])
        x = ops.linear(col, W["init.w"]).view(n, H, Wd, -1)
        feats = []
        for nm, _cin, _cout, li, s2 in _blocks(self.inplane):
            if s2:
                feats.append(x)
                y, pooled = ops.dwconv_relu(x, W[nm + ".dw"], self._k(li), pool=True)
                c = pooled.shape[-1]
                res = ops.linear(pooled.view(-1, c), W[nm + ".sc.w"], bias=W[nm + ".sc.b"])
            else:
                y, _ = ops.dwconv_relu(x, W[nm + ".dw"], self._k(li))
                res = x.view(-1, x.shape[-1])
            x = ops.linear(y.view(-1, y.shape[-1]), W[nm + ".pw"], residual=res).view(*y.shape[:3], -1)
        feats.append(x)
        es = []
        for i, f in enumerate(feats):
            q, a, r = f"dilations.{i}.", f"attentions.{i}.", f"conv_reduces.{i}.conv."
            nf, h, w, c = f.shape
            t = ops.linear(ops.eltwise("relu", f).view(-1, c), W[q + "c1.w"], bias=W[q + "c1.b"]).view(nf, h, w, -1)
            t = ops.conv2d_taps(t, W[q + "c2.w"], W["taps"])
            es.append(ops.csam_mapreduce(t, W[a + "w1"], W[a + "b1"], W[a + "w2"], W[r + "w"], W[r + "b"]))
        return ops.pidinet_fuse(es, W["cls"], H, Wd, torch.float32 if out_f32 else torch.float16)


def pidinet_bsd(pretrained=False, vanilla_cnn=True):
    """pidinet.py:732-746: PiDiNet(60, carv4, dil=24, sa=True, convert=True); pretrained=True loads
    models/table5_pidinet.pth relative to the working directory, converts its PDC weights and strips 'module.'."""
    if not vanilla_cnn:
        raise NotImplementedError("vgen_b200 pidinet_bsd: only vanilla_cnn=True (the converted form) runs natively")
    model = PiDiNet(60, CARV4, dil=24, sa=True, convert=True)
    if pretrained:
        state = convert_pidinet(torch.load("models/table5_pidinet.pth", map_location="cpu")["state_dict"], CARV4)
        model.load_state_dict({k[len("module."):] if k.startswith("module.") else k: v for k, v in state.items()})
    return model


# ---- sketch simplification --------------------------------------------------------------------------------------------------
# (cin, cout, kernel, stride, transposed) of the 23 convolutions, nn.Sequential indices 0, 2, .., 44
CLEANER_LAYERS = [(1, 48, 5, 2, False), (48, 128, 3, 1, False), (128, 128, 3, 1, False), (128, 128, 3, 2, False),
                  (128, 256, 3, 1, False), (256, 256, 3, 1, False), (256, 256, 3, 2, False), (256, 512, 3, 1, False),
                  (512, 1024, 3, 1, False), (1024, 1024, 3, 1, False), (1024, 1024, 3, 1, False),
                  (1024, 1024, 3, 1, False), (1024, 512, 3, 1, False), (512, 256, 3, 1, False), (256, 256, 4, 2, True),
                  (256, 256, 3, 1, False), (256, 128, 3, 1, False), (128, 128, 4, 2, True), (128, 128, 3, 1, False),
                  (128, 48, 3, 1, False), (48, 48, 4, 2, True), (48, 24, 3, 1, False), (24, 1, 3, 1, False)]

# ConvTranspose2d(k=4, s=2, p=1): output row 2m + p reads input rows m + dy with kernel row ky, per phase p
_TCONV_PHASE = {0: ((0, 1), (-1, 3)), 1: ((0, 2), (1, 0))}
_TAPS3 = [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)]


def cleaner_spec():
    spec = []
    for i, (cin, cout, k, _s, tr) in enumerate(CLEANER_LAYERS):
        spec += [(f"layers.{2 * i}.weight", (cin, cout, k, k) if tr else (cout, cin, k, k)), (f"layers.{2 * i}.bias", (cout,))]
    return spec


class SketchSimplification(SpecModule):
    r"""The sketch-simplification GAN (sketch_simplification.py:14-79) on the native path."""

    def __init__(self, mean, std):
        if not isinstance(mean, float) or not isinstance(std, float):
            raise TypeError("SketchSimplification: mean and std must be floats")
        super().__init__()
        self.mean, self.std = mean, std
        self._build_params(cleaner_spec())

    def _pack(self):
        dev = self.device
        if dev.type != "cuda":
            raise ops._l.VgenError("vgen_b200 SketchSimplification forward needs the model on a CUDA device (no CPU path exists)")
        sd = {k: v.detach().to(device=dev, dtype=torch.float32) for k, v in self.state_dict().items()}
        f16 = lambda t: t.to(torch.float16).contiguous()  # noqa: E731
        W = {}
        last = len(CLEANER_LAYERS) - 1
        for i, (cin, cout, k, s, tr) in enumerate(CLEANER_LAYERS):
            w, b = sd[f"layers.{2 * i}.weight"], sd[f"layers.{2 * i}.bias"]
            ci, co = _pad64(cin), _pad64(cout)
            if i == last:
                W[f"{i}.w"] = _padded(w[0].permute(1, 2, 0).reshape(9, cin), (9, ci)).contiguous()
                W[f"{i}.b"] = b.contiguous()
                continue
            W[f"{i}.b"] = _padded(b, (co,))
            if tr:      # one [co, 4 * ci] matrix per output phase (py, px), taps in _phase_taps order
                for py in (0, 1):
                    for px in (0, 1):
                        W[f"{i}.w{py}{px}"] = f16(torch.cat([_padded(w[:, :, ky, kx].t(), (co, ci))
                                                             for _dy, ky in _TCONV_PHASE[py] for _dx, kx in _TCONV_PHASE[px]], 1))
            elif i == 0:   # im2col columns (ky, kx) of the single input channel, padded to 64
                W["0.w"] = f16(_padded(w.reshape(cout, k * k), (co, 64)))
            else:
                W[f"{i}.w"] = f16(_padded(w.permute(0, 2, 3, 1), (co, k, k, ci)).reshape(co, k * k * ci))
        self._packed = W
        return W

    def forward(self, x):
        """x [n, 1, H, W] CUDA in [0, 1] (sketch pixels dark), H and W multiples of 8, in the parameter dtype -> the
        simplified sketch [n, 1, H, W] in x's dtype."""
        if x.dim() == 4 and (x.shape[2] % 8 or x.shape[3] % 8):
            raise ValueError(f"SketchSimplification: H and W must be multiples of 8, got {tuple(x.shape[2:])}")
        _check_input("SketchSimplification", x, 1, next(self.parameters()).dtype)
        if not (x.is_contiguous() or x.is_contiguous(memory_format=torch.channels_last)):
            raise ValueError("SketchSimplification: x must be NCHW-contiguous or channels_last")
        n, _, H, Wd = x.shape
        # one channel: NCHW and NHWC are the same memory; the normalisation precedes the first conv's zero padding
        img = ops.sketch_normalize(x.reshape(n, H, Wd, 1) if x.is_contiguous() else x.permute(0, 2, 3, 1).contiguous(),
                                   self.mean, self.std)
        if self._packed is None:
            self._pack()
        return self._forward_nhwc(img, x.dtype == torch.float32)

    @graphed
    @torch.no_grad()
    def _forward_nhwc(self, img, out_f32):
        W = self._packed
        n, H, Wd, _ = img.shape
        col = ops.im2col(img, 5, 5, 2, 2, 2, H // 2, Wd // 2, 64)
        x = ops.conv2d_taps(col.view(1, 1, -1, 64), W["0.w"], [(0, 0)], bias=W["0.b"], relu=True).view(n, H // 2, Wd // 2, -1)
        last = len(CLEANER_LAYERS) - 1
        for i in range(1, last):
            _cin, _cout, k, s, tr = CLEANER_LAYERS[i]
            nb, h, w, c = x.shape
            if tr:
                co = W[f"{i}.b"].shape[0]
                out = torch.empty(nb, 2 * h, 2 * w, co, device=x.device, dtype=torch.float16)
                for py in (0, 1):
                    for px in (0, 1):
                        taps = [(dy, dx) for dy, _ky in _TCONV_PHASE[py] for dx, _kx in _TCONV_PHASE[px]]
                        ops.conv2d_taps(x, W[f"{i}.w{py}{px}"], taps, bias=W[f"{i}.b"], relu=True,
                                        out=out[:, py:, px:], out_stride_y=2 * 2 * w * co, out_stride_x=2 * co)
                x = out
            elif s == 2:
                col = ops.im2col(x, 3, 3, 2, 1, 1, h // 2, w // 2, 9 * c)
                x = ops.conv2d_taps(col.view(1, 1, -1, 9 * c), W[f"{i}.w"], [(0, 0)], bias=W[f"{i}.b"], relu=True)
                x = x.view(nb, h // 2, w // 2, -1)
            else:
                x = ops.conv2d_taps(x, W[f"{i}.w"], _TAPS3, bias=W[f"{i}.b"], relu=True)
        return ops.conv3x3_to1_sigmoid(x, W[f"{last}.w"], W[f"{last}.b"], torch.float32 if out_f32 else torch.float16)


def sketch_simplification_gan(pretrained=False):
    """sketch_simplification.py:81-90; pretrained=True loads models/sketch_simplification_gan.pth relative to the working
    directory, as the reference does."""
    model = SketchSimplification(mean=0.9664114577640158, std=0.0858381272736797)
    if pretrained:
        model.load_state_dict(torch.load("models/sketch_simplification_gan.pth", map_location="cpu"))
    return model
