"""Plain-PyTorch restatement of the VideoComposer sketch annotators, driven by reference-format state dicts:
  * PiDiNet in its converted vanilla-CNN form with sa=True and an int dil (tools/annotator/sketch/pidinet.py:527-704);
  * the sketch-simplification GAN (tools/annotator/sketch/sketch_simplification.py:14-79).
Every op is a torch.nn.functional call in the reference's order, in fp32.  The engines run both networks in fp32 with
cuDNN's default TF32 convolutions; callers choose that arithmetic with torch.backends.cudnn.allow_tf32.  Runs on CPU or
GPU.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

_PIDINET_STAGES = ((1, 3), (2, 4), (3, 4), (4, 4))     # (stage, blocks); block s_1 of stages 2-4 has stride 2


def _f32(sd, device):
    return {k: v.detach().to(device=device, dtype=torch.float32) for k, v in sd.items()}


def pidinet_forward(sd, x):
    """edge map [n, 1, H, W] of x [n, 3, H, W] (fp32) with a PiDiNet(convert=True, sa=True, dil=int) state dict."""
    P = _f32(sd, x.device)
    x = x.float()
    H, W = x.shape[2:]
    w0 = P["init_block.weight"]
    x = F.conv2d(x, w0, padding=w0.shape[-1] // 2)
    feats = []
    for s, nb in _PIDINET_STAGES:
        for b in range(1, nb + 1):
            q = f"block{s}_{b}."
            stride2 = s > 1 and b == 1
            if stride2:
                x = F.max_pool2d(x, kernel_size=2, stride=2)
            w1 = P[q + "conv1.weight"]
            y = F.conv2d(x, w1, padding=w1.shape[-1] // 2, groups=w1.shape[0])
            y = F.conv2d(F.relu(y), P[q + "conv2.weight"])
            if stride2:
                x = F.conv2d(x, P[q + "shortcut.weight"], P[q + "shortcut.bias"])
            x = y + x
        feats.append(x)
    outs = []
    for i, xi in enumerate(feats):
        d, a, r = f"dilations.{i}.", f"attentions.{i}.", f"conv_reduces.{i}.conv."
        t = F.conv2d(F.relu(xi), P[d + "conv1.weight"], P[d + "conv1.bias"])
        t = sum(F.conv2d(t, P[d + f"conv2_{j}.weight"], dilation=dl, padding=dl) for j, dl in ((1, 5), (2, 7), (3, 9), (4, 11)))
        y = F.conv2d(F.conv2d(F.relu(t), P[a + "conv1.weight"], P[a + "conv1.bias"]), P[a + "conv2.weight"], padding=1)
        e = F.conv2d(t * torch.sigmoid(y), P[r + "weight"], P[r + "bias"])
        outs.append(F.interpolate(e, (H, W), mode="bilinear", align_corners=False))
    return torch.sigmoid(F.conv2d(torch.cat(outs, dim=1), P["classifier.weight"], P["classifier.bias"]))


def cleaner_forward(sd, x, mean, std):
    """simplified sketch [n, 1, H, W] of x [n, 1, H, W] in [0, 1] (fp32) with a SketchSimplification state dict."""
    P = _f32(sd, x.device)
    x = (x.float() - mean) / std
    i = 0
    while f"layers.{i}.weight" in P:
        w, b = P[f"layers.{i}.weight"], P[f"layers.{i}.bias"]
        last = f"layers.{i + 2}.weight" not in P
        if i in (28, 34, 40):                                  # the three ConvTranspose2d(c, c, 4, 2, 1)
            x = F.conv_transpose2d(x, w, b, stride=2, padding=1)
        else:
            x = F.conv2d(x, w, b, stride=2 if i in (0, 6, 12) else 1, padding=w.shape[-1] // 2)
        x = torch.sigmoid(x) if last else F.relu(x)
        i += 2
    return x
