"""The sketch annotators on the H100: the new kernels and tap-GEMM paths against PyTorch fp32, the tiny cases against the
reference's frozen outputs, full-size forwards against the fp32 oracle, CUDA-graph replay, and the kernels a forward
launches.

Gates are the project's existing ones (tests/test_gpu_depth.py): ours must be no further from the fp32 truth than 1.25x the
yardstick's error + 2e-4, with a relative-L2 cap of 5e-3 for the tiny cases and 6e-3 at full size, where max-abs over
max-magnitude must also stay below 4x the cap.  The yardstick is the oracle in fp32 with cuDNN's TF32 convolutions, what
the engines compute; the truth is the oracle with TF32 off."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sketch_oracle
from vgen_b200 import graph, ops
from vgen_b200.sketch import PiDiNet, SketchSimplification, _cdcm_taps, pidinet_bsd, sketch_simplification_gan
from _sketch import (GAN_MEAN, GAN_STD, SKETCH_CASES, TINY_PIDINET, full_state_dict, load_spec, make_input, non_vacuous,
                     state_dict)

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def _max_rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    ops.set_tapgemm_impl("auto")


def _g(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _h(*shape, seed=0, scale=1.0):
    return _g(*shape, seed=seed, scale=scale).half().cuda()


def _nchw(x):
    return x.float().permute(0, 3, 1, 2)


# ---- kernels ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pool", [False, True])
@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("n,h,w,c", [(2, 256, 448, 64), (2, 128, 224, 128), (1, 33, 51, 256), (2, 15, 9, 64), (1, 2, 3, 64)])
def test_dwconv_relu_matches_torch(n, h, w, c, k, pool):
    if pool and (h < 2 or w < 2):
        pytest.skip("nothing to pool")
    x = _h(n, h, w, c, seed=1)
    wt = _g(c, 1, k, k, seed=2, scale=1.0 / k)
    y, pooled = ops.dwconv_relu(x, wt.reshape(c, k * k).t().contiguous().cuda(), k, pool=pool)
    xin = _nchw(x)
    if pool:
        xin = F.max_pool2d(xin, 2)
        assert torch.equal(pooled.float(), xin.permute(0, 2, 3, 1))
    want = F.relu(F.conv2d(xin, wt.cuda(), padding=k // 2, groups=c)).permute(0, 2, 3, 1)
    assert y.shape == want.shape
    assert float((y.float() - want).abs().max()) <= float(want.abs().max()) * 2 ** -10 + 1e-5


def _phase_weights(wt, ci, co):
    """ConvTranspose2d(4, 2, 1) weight [ci, co, 4, 4] -> {(py, px): ([co, 4 ci] fp16, taps)}."""
    rows = {0: ((0, 1), (-1, 3)), 1: ((0, 2), (1, 0))}
    out = {}
    for py in (0, 1):
        for px in (0, 1):
            w = torch.cat([wt[:, :, ky, kx].t() for _dy, ky in rows[py] for _dx, kx in rows[px]], 1)
            out[py, px] = (w.half().cuda().contiguous(), [(dy, dx) for dy, _ in rows[py] for dx, _ in rows[px]])
    return out


@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("n,h,w,ci,co", [(2, 32, 56, 256, 256), (2, 64, 112, 128, 128), (1, 5, 7, 64, 64), (2, 3, 1, 64, 128)])
def test_conv_transpose_phases_match_torch(impl, n, h, w, ci, co):
    ops.set_tapgemm_impl(impl)
    x = _h(n, h, w, ci, seed=3)
    wt = _g(ci, co, 4, 4, seed=4, scale=ci ** -0.5)
    b = _g(co, seed=5, scale=0.1).cuda()
    out = torch.empty(n, 2 * h, 2 * w, co, device="cuda", dtype=torch.float16)
    for (py, px), (wp, taps) in _phase_weights(wt, ci, co).items():
        ops.conv2d_taps(x, wp, taps, bias=b, relu=True, out=out[:, py:, px:], out_stride_y=4 * w * co, out_stride_x=2 * co)
    want = F.relu(F.conv_transpose2d(_nchw(x), wt.half().float().cuda(), b, stride=2, padding=1)).permute(0, 2, 3, 1)
    assert _max_rel(out, want) < 2e-3


@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("n,h,w,c", [(2, 256, 448, 64), (1, 32, 56, 64), (2, 7, 12, 64)])
def test_cdcm_33_tap_conv_matches_four_dilated_convs(impl, n, h, w, c):
    ops.set_tapgemm_impl(impl)
    x = _h(n, h, w, c, seed=6)
    ws = [_g(c, c, 3, 3, seed=7 + j, scale=(9 * c) ** -0.5) for j in range(4)]
    taps = [ws[0][:, :, 1, 1] + ws[1][:, :, 1, 1] + ws[2][:, :, 1, 1] + ws[3][:, :, 1, 1]]
    for wj in ws:
        taps += [wj[:, :, ky, kx] for ky in range(3) for kx in range(3) if (ky, kx) != (1, 1)]
    y = ops.conv2d_taps(x, torch.cat(taps, 1).half().cuda().contiguous(), _cdcm_taps())
    xin = _nchw(x)
    want = sum(F.conv2d(xin, wj.cuda(), dilation=d, padding=d) for wj, d in zip(ws, (5, 7, 9, 11))).permute(0, 2, 3, 1)
    assert len(_cdcm_taps()) == 33
    assert _max_rel(y, want) < 3e-3


@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("n,h,w,ci,co", [(2, 64, 112, 256, 512), (1, 13, 17, 64, 64), (2, 32, 56, 128, 64)])
def test_conv3x3_relu_taps_match_torch(impl, n, h, w, ci, co):
    ops.set_tapgemm_impl(impl)
    x = _h(n, h, w, ci, seed=11)
    wt = _g(co, ci, 3, 3, seed=12, scale=(9 * ci) ** -0.5)
    b = _g(co, seed=13, scale=0.1).cuda()
    y = ops.conv2d_taps(x, wt.permute(0, 2, 3, 1).reshape(co, 9 * ci).half().cuda().contiguous(),
                        [(dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)], bias=b, relu=True)
    want = F.relu(F.conv2d(_nchw(x), wt.half().float().cuda(), b, padding=1)).permute(0, 2, 3, 1)
    assert _max_rel(y, want) < 2e-3
    assert float((want == 0).float().mean()) > 0.2


@pytest.mark.parametrize("n,h,w,c", [(2, 256, 448, 64), (2, 32, 56, 64), (1, 3, 5, 64), (2, 1, 1, 8)])
def test_csam_mapreduce_matches_torch(n, h, w, c):
    x = _h(n, h, w, c, seed=14)
    w1, b1, w2 = _g(4, c, seed=15, scale=c ** -0.5), _g(4, seed=16, scale=0.1), _g(1, 4, 3, 3, seed=17, scale=0.5)
    wm, bm = _g(c, seed=18, scale=c ** -0.5), _g(1, seed=19, scale=0.1)
    e = ops.csam_mapreduce(x, w1.cuda(), b1.cuda(), w2.reshape(-1).cuda(), wm.cuda(), bm.cuda())
    xin = _nchw(x)
    y = torch.sigmoid(F.conv2d(F.conv2d(F.relu(xin), w1.view(4, c, 1, 1).cuda(), b1.cuda()), w2.cuda(), padding=1))
    want = F.conv2d(xin * y, wm.view(1, c, 1, 1).cuda(), bm.cuda())[:, 0]
    assert float((e - want).abs().max()) <= float(want.abs().max()) * 1e-5 + 1e-5


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("n,H,W", [(2, 256, 448), (1, 512, 896), (2, 60, 100), (1, 9, 13)])
def test_pidinet_fuse_matches_torch(n, H, W, out_dtype):
    sizes = [(H, W), (H // 2, W // 2), (H // 4, W // 4), (H // 8, W // 8)]
    es = [_g(n, h, w, seed=20 + i).cuda() for i, (h, w) in enumerate(sizes)]
    cw = _g(5, seed=25, scale=0.5).cuda()
    out = ops.pidinet_fuse(es, cw, H, W, out_dtype)
    up = torch.cat([F.interpolate(e[:, None], (H, W), mode="bilinear", align_corners=False) for e in es], 1)
    want = torch.sigmoid(F.conv2d(up, cw[:4].view(1, 4, 1, 1), cw[4:]))
    assert out.dtype == out_dtype and out.shape == want.shape
    tol = 2 ** -11 if out_dtype == torch.float16 else 1e-6
    assert float((out.float() - want).abs().max()) <= tol + 1e-6


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("n,h,w,c", [(2, 256, 448, 64), (1, 512, 896, 64), (2, 7, 9, 64), (1, 1, 1, 8)])
def test_conv3x3_to1_sigmoid_matches_torch(n, h, w, c, out_dtype):
    x = _h(n, h, w, c, seed=26)
    wt, b = _g(1, c, 3, 3, seed=27, scale=(9 * c) ** -0.5), _g(1, seed=28, scale=0.1)
    y = ops.conv3x3_to1_sigmoid(x, wt[0].permute(1, 2, 0).reshape(9, c).contiguous().cuda(), b.cuda(), out_dtype)
    want = torch.sigmoid(F.conv2d(_nchw(x), wt.cuda(), b.cuda(), padding=1))
    assert y.dtype == out_dtype and y.shape == want.shape
    tol = 2 ** -11 if out_dtype == torch.float16 else 1e-6
    assert float((y.float() - want).abs().max()) <= tol + 1e-6


# ---- tiny cases against the reference ----------------------------------------------------------------------------------
def _model(net, sd):
    m = PiDiNet(**TINY_PIDINET) if net == "pidinet" else SketchSimplification(GAN_MEAN, GAN_STD)
    m.load_state_dict(sd, strict=True)
    return m.eval().requires_grad_(False).cuda()


def _oracle(net, sd, x, tf32=False):
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        if net == "pidinet":
            return sketch_oracle.pidinet_forward(sd, x)
        return sketch_oracle.cleaner_forward(sd, x, GAN_MEAN, GAN_STD)
    finally:
        torch.backends.cudnn.allow_tf32 = False


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
@pytest.mark.parametrize("name", sorted(SKETCH_CASES))
def test_tiny_parity(golden_dir, name, layout):
    case = SKETCH_CASES[name]
    net = case["net"]
    sd = state_dict(load_spec(golden_dir, "pidinet_tiny" if net == "pidinet" else "cleaner"), case["seed"], net)
    m = _model(net, sd)
    x = make_input(net, case["n"], case["H"], case["W"], case["seed"]).cuda()
    xin = x.contiguous(memory_format=torch.channels_last) if layout == "channels_last" else x
    sdg = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        mine = m(xin)
        o32, yard = _oracle(net, sdg, x), _oracle(net, sdg, x, tf32=True)
    torch.cuda.synchronize()
    truth = torch.from_numpy(np.load(os.path.join(golden_dir, f"sketch_{name}.npz"))["out"]).cuda()
    assert mine.shape == truth.shape and mine.dtype == torch.float32 and torch.isfinite(mine).all()
    assert _rel_l2(o32, truth) < 1e-4, "GPU fp32 oracle must reproduce the reference's CPU fp32 result"
    std, sat = non_vacuous(truth)
    assert std > 0.05 and sat < 0.5
    e_mine, e_yard = _rel_l2(mine, truth), _rel_l2(yard, truth)
    print(f"{name} {layout}: ours vs fp32 truth {e_mine:.3e}; TF32 oracle vs truth {e_yard:.3e}")
    assert e_mine < 5e-3
    assert e_mine < 1.25 * e_yard + 2e-4


# ---- full size -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full_models(golden_dir):
    sp, sc = full_state_dict(load_spec(golden_dir, "pidinet_full"), "pidinet"), full_state_dict(load_spec(golden_dir, "cleaner"), "cleaner")
    p, c = pidinet_bsd(), sketch_simplification_gan()
    p.load_state_dict(sp, strict=True)
    c.load_state_dict(sc, strict=True)
    p, c = (m.eval().requires_grad_(False).cuda() for m in (p, c))
    return p, c, {k: v.cuda() for k, v in sp.items()}, {k: v.cuda() for k, v in sc.items()}


def _check_full(tag, mine, truth, yard):
    d = lambda a: (_rel_l2(a, truth), _max_rel(a, truth))  # noqa: E731
    (e_mine, mx_mine), (e_yard, mx_yard) = d(mine), d(yard)
    std, sat = non_vacuous(truth)
    print(f"{tag}: truth std {std:.3f}, saturated {sat:.1%}; ours rel-L2 {e_mine:.3e} max {mx_mine:.3e}; "
          f"TF32 oracle rel-L2 {e_yard:.3e} max {mx_yard:.3e}")
    assert std > 0.05 and sat < 0.5, "the synthetic full-size output is vacuous"
    cap = 6e-3
    assert e_mine < cap and mx_mine < 4 * cap
    assert e_mine < 1.25 * e_yard + 2e-4


@pytest.mark.parametrize("n,H,W", [(2, 256, 448), (1, 512, 896)])
def test_fullsize_against_fp32_oracle(full_models, n, H, W):
    p, c, sp, sc = full_models
    x = make_input("pidinet", n, H, W, 65).cuda()
    xc = make_input("cleaner", n, H, W, 66).cuda()
    mean = torch.tensor([0.485, 0.456, 0.406], device="cuda").view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], device="cuda").view(1, 3, 1, 1)
    frames = (x * std + mean).clamp(0, 1)      # the engines' misc_imgs; pidinet sees (frames - mean) / std
    with torch.no_grad():
        _check_full(f"pidinet {n}x{H}x{W}", p(x), _oracle("pidinet", sp, x), _oracle("pidinet", sp, x, True))
        _check_full(f"cleaner {n}x{H}x{W}", c(xc), _oracle("cleaner", sc, xc), _oracle("cleaner", sc, xc, True))

        def chain(pf, cf):
            return 1.0 - cf(1.0 - pf(frames.sub(mean).div_(std)))
        mine = chain(p, c)
        truth = chain(lambda t: _oracle("pidinet", sp, t), lambda t: _oracle("cleaner", sc, t))
        yard = chain(lambda t: _oracle("pidinet", sp, t, True), lambda t: _oracle("cleaner", sc, t, True))
    _check_full(f"chain {n}x{H}x{W}", mine, truth, yard)


# ---- graphs, kernels -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", ["pidinet", "cleaner"])
def test_graph_replay_is_bit_equal_to_eager_and_repacks(golden_dir, net):
    which = "pidinet_tiny" if net == "pidinet" else "cleaner"
    m = _model(net, state_dict(load_spec(golden_dir, which), 3, net))
    xs = [make_input(net, 2, 64, 96, s).cuda() for s in range(8)]
    outs = [m(x) for x in xs]
    assert graph.stats(m)["_forward_nhwc"] == (1, 7)
    m.use_cuda_graph = False
    eager = [m(x) for x in xs]
    m.use_cuda_graph = True
    for a, b in zip(outs, eager):
        assert torch.equal(a, b)
    assert not torch.equal(outs[0], outs[1])
    sd2 = state_dict(load_spec(golden_dir, which), 99, net)
    m.load_state_dict(sd2, strict=True)
    assert m._packed is None and graph.stats(m) == {}
    new = m(xs[0])
    assert graph.stats(m)["_forward_nhwc"] == (0, 0)
    assert _rel_l2(new, _oracle(net, {k: v.cuda() for k, v in sd2.items()}, xs[0])) < 5e-3


def test_half_model_runs_in_half():
    m = pidinet_bsd().eval().requires_grad_(False).half().cuda()
    y = m(make_input("pidinet", 1, 64, 96, 1).cuda().half())
    assert y.dtype == torch.float16 and y.shape == (1, 1, 64, 96) and torch.isfinite(y).all()


def _library_kernels():
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vgen_b200", "csrc")
    pat = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\((?:[^()]|\([^()]*\))*\)\s*)?(\w+)\s*\(")
    names = set()
    for fn in os.listdir(src):
        if fn.endswith((".cu", ".cuh")):
            names |= set(pat.findall(open(os.path.join(src, fn)).read()))
    return names


def _kernel_name(demangled):
    head = demangled.split("(")[0].split("<")[0].strip()
    return head.split()[-1].split("::")[-1] if head else head


# a child process, so the profiling sessions leave no profiler state in the suite's process
_PROFILE_CHILD = r"""
import json, sys
root = sys.argv[1]
sys.path[:0] = [root, root + "/tests"]
import torch
from torch.profiler import ProfilerActivity, profile
from _sketch import TINY_PIDINET, load_spec, make_input, state_dict
from vgen_b200.sketch import PiDiNet, sketch_simplification_gan
p = PiDiNet(**TINY_PIDINET)
p.load_state_dict(state_dict(load_spec(root + "/tests/golden", "pidinet_tiny"), 1, "pidinet"), strict=True)
c = sketch_simplification_gan()
c.load_state_dict(state_dict(load_spec(root + "/tests/golden", "cleaner"), 1, "cleaner"), strict=True)
p, c = p.eval().cuda(), c.eval().cuda()
x = make_input("pidinet", 2, 64, 96, 1).cuda()
out = {}
for graphed in (False, True):
    p.use_cuda_graph = c.use_cuda_graph = graphed
    for _ in range(3):
        c(1 - p(x))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        c(p(x))
        torch.cuda.synchronize()
    out["graphed" if graphed else "eager"] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
print(json.dumps(out))
"""


def test_forward_launches_only_library_kernels():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, root], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    ours = _library_kernels()
    for mode, nms in names.items():
        foreign = {nm for nm in nms if _kernel_name(nm) not in ours and "memcpy" not in nm.lower() and "memset" not in nm.lower()}
        assert not foreign, (mode, foreign)
    for k in ("dwconv_relu_kernel", "csam_pre_kernel", "csam_out_kernel", "pidinet_fuse_kernel", "conv3x3_to1_sigmoid_kernel",
              "sketch_normalize_kernel", "tapgemm_sm90_kernel"):
        assert any(k in nm for nm in names["eager"]), (k, names["eager"])
