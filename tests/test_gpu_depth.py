"""The MiDaS v3 depth annotator on the H100: the new kernels against PyTorch fp32, the tiny cases against the reference's
frozen outputs, full-size forwards against the fp32 oracle, CUDA-graph replay, and the kernels a forward launches.

Gates are the existing ones: tiny cases as tests/test_gpu_parity.py (ours vs the fp32 truth within 1.25x the reference's
own fp16 path + 2e-4, cap 5e-3 relative L2); full size as tests/test_gpu_fullsize.py (the same ratio, cap 6e-3, max-abs
over max-magnitude below 4x the cap).  The yardstick is the oracle in fp16 channels_last, what the engines run."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import depth_oracle
from vgen_b200 import graph, ops
from vgen_b200.depth import MiDaS
from _depth import DEPTH_CASES, FULL, TINY, full_state_dict, load_spec, make_input, oracle_kw, state_dict

pytestmark = pytest.mark.gpu

DEPTH_STD, DEPTH_CLAMP = 20.0, 10.0     # the engines' post-processing, cfg.depth_std / cfg.depth_clamp


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


def _h(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


# ---- kernels ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nimg,h,w,cin,cout,s", [(2, 16, 28, 256, 256, 4), (2, 16, 28, 512, 512, 2), (1, 32, 56, 256, 256, 4),
                                                 (3, 5, 7, 64, 72, 3), (1, 3, 1, 40, 8, 2), (2, 4, 6, 128, 64, 1)])
def test_conv_transpose_stride_matches_torch(nimg, h, w, cin, cout, s):
    x = _h(nimg, h, w, cin, seed=1)
    wt = torch.randn(cin, cout, s, s, generator=torch.Generator().manual_seed(2)) / cin ** 0.5
    b = torch.randn(cout, generator=torch.Generator().manual_seed(3)) * 0.1
    y = ops.conv_transpose_stride(x, ops.pack_conv_transpose_weight(wt).half().cuda().contiguous(), b.cuda(), s)
    want = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wt.half().float().cuda(), b.cuda(), stride=s).permute(0, 2, 3, 1)
    assert y.shape == want.shape == (nimg, s * h, s * w, cout)
    assert _max_rel(y, want) < 2e-3


@pytest.mark.parametrize("nimg,h,w,c", [(2, 8, 14, 256), (2, 64, 112, 256), (1, 128, 224, 128), (3, 13, 5, 40), (1, 1, 1, 8),
                                        (2, 1, 9, 16)])
def test_upsample_bilinear2x_matches_torch(nimg, h, w, c):
    x = _h(nimg, h, w, c, seed=4)
    y = ops.upsample_bilinear2x(x)
    want = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    assert y.shape == want.shape
    # fp32 weights and sums, one rounding to fp16: within half an fp16 ulp of the fp32 result, plus the sum's reordering
    assert float((y.float() - want).abs().max()) <= float(want.abs().max()) * 2 ** -11 + 1e-6


@pytest.mark.parametrize("n", [1, 7, 1 << 20, (1 << 20) + 3])
def test_relu_matches_torch(n):
    x = _h(n, seed=5)
    x[:3] = torch.tensor([float("nan"), -0.0, float("-inf")], device="cuda", dtype=torch.float16)[: min(3, n)]
    y = ops.eltwise("relu", x)
    want = torch.relu(x)
    assert torch.equal(y.isnan(), want.isnan()) and torch.equal(y.nan_to_num(), want.nan_to_num())


@pytest.mark.parametrize("rows,c,out_dtype", [(2 * 256 * 448, 32, torch.float16), (512 * 896, 32, torch.float32),
                                              (1, 32, torch.float32), (1001, 40, torch.float16), (77, 8, torch.float32)])
def test_head_out_matches_torch(rows, c, out_dtype):
    x = _h(rows, c, seed=6)
    w = (torch.randn(c, generator=torch.Generator().manual_seed(7)) / c ** 0.5).cuda()
    b = torch.tensor([0.05], device="cuda")
    y = ops.dpt_head_out(x, w, b, out_dtype)
    want = torch.relu(torch.relu(x.float()) @ w + b)
    assert y.dtype == out_dtype and y.shape == (rows,)
    tol = 2 ** -10 if out_dtype == torch.float16 else 1e-5
    assert float((y.float() - want).abs().max()) <= float(want.abs().max()) * tol + 1e-6
    if rows > 1000:
        assert float((want > 0).float().mean()) > 0.2


# ---- tiny cases against the reference ----------------------------------------------------------------------------------
def _tiny(golden_dir, name, half):
    case = DEPTH_CASES[name]
    sd = state_dict(load_spec(golden_dir, "tiny"), case["seed"])
    m = MiDaS(**case["ctor"])
    m.load_state_dict(sd, strict=True)
    m = m.eval().requires_grad_(False)
    if half:
        m = m.to(memory_format=torch.channels_last).half()
    m = m.cuda()
    x = make_input(case["n"], case["H"], case["W"], case["seed"]).cuda()
    return case, sd, m, x


@pytest.mark.parametrize("half", [True, False], ids=["fp16_channels_last", "fp32_contiguous"])
@pytest.mark.parametrize("name", sorted(DEPTH_CASES))
def test_tiny_parity(golden_dir, name, half):
    case, sd, m, x = _tiny(golden_dir, name, half)
    xin = x.half().contiguous(memory_format=torch.channels_last) if half else x
    sdg = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        mine = m(xin)
        o32 = depth_oracle.midas_forward(sdg, x, **oracle_kw(case["ctor"]))
        o16 = depth_oracle.midas_forward(sdg, x, half=True, **oracle_kw(case["ctor"]))
    torch.cuda.synchronize()
    truth = torch.from_numpy(np.load(os.path.join(golden_dir, f"depth_{name}.npz"))["out"]).cuda()
    assert mine.shape == truth.shape and mine.dtype == xin.dtype and torch.isfinite(mine.float()).all()
    assert _rel_l2(o32, truth) < 1e-4, "GPU fp32 oracle must reproduce the reference's CPU fp32 result"
    e_mine, e_ref16 = _rel_l2(mine, truth), _rel_l2(o16, truth)
    print(f"{name} {'fp16' if half else 'fp32'}: ours vs fp32 truth {e_mine:.3e}; fp16 oracle vs truth {e_ref16:.3e}")
    assert e_mine < 5e-3
    assert e_mine < 1.25 * e_ref16 + 2e-4


# ---- full size -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full_model_and_sd(golden_dir):
    sd = full_state_dict(load_spec(golden_dir, "full"))
    m = MiDaS(**FULL)
    m.load_state_dict(sd, strict=True)
    m = m.eval().requires_grad_(False).to(memory_format=torch.channels_last).half().cuda()
    return m, {k: v.cuda() for k, v in sd.items()}


def _metrics(a, truth):
    d = a.float() - truth
    return float(d.norm() / (truth.norm() + 1e-30)), float(d.abs().max() / (truth.abs().max() + 1e-30))


@pytest.mark.parametrize("n,H,W", [(2, 256, 448), (1, 512, 896)])
def test_fullsize_against_fp32_oracle(full_model_and_sd, n, H, W):
    m, sdg = full_model_and_sd
    x = make_input(n, H, W, 65).cuda()
    with torch.no_grad():
        mine = m(x.half().contiguous(memory_format=torch.channels_last))
        truth = depth_oracle.midas_forward(sdg, x).float()
        yard = depth_oracle.midas_forward(sdg, x, half=True)
    torch.cuda.synchronize()
    pos = float((truth > 0).float().mean())
    print(f"{n}x{H}x{W}: truth max {float(truth.max()):.3g}, mean {float(truth.mean()):.3g}, positive {pos:.1%}")
    assert pos > 0.2, "the synthetic full-size output is mostly clipped by the final ReLU"
    cap = 6e-3
    for tag, f in (("raw", lambda t: t.float()), ("post", lambda t: (t.float() / DEPTH_STD).clamp_(0, DEPTH_CLAMP))):
        t = f(truth)
        (e_mine, mx_mine), (e_yard, mx_yard) = _metrics(f(mine), t), _metrics(f(yard), t)
        print(f"{n}x{H}x{W} {tag}: ours rel-L2 {e_mine:.3e} max {mx_mine:.3e}; fp16 oracle rel-L2 {e_yard:.3e} max {mx_yard:.3e}")
        assert e_mine < cap and mx_mine < 4 * cap
        assert e_mine < 1.25 * e_yard + 2e-4


# ---- graphs, determinism, kernels ------------------------------------------------------------------------------------
def test_graph_replay_is_bit_equal_to_eager_and_repacks(golden_dir):
    case, sd, m, _ = _tiny(golden_dir, "tiny_64x96_b2", True)
    xs = [make_input(2, 64, 96, s).cuda().half().contiguous(memory_format=torch.channels_last) for s in range(8)]
    outs = [m(x) for x in xs]                        # eager, capture, then six replays of one graph
    assert graph.stats(m)["_forward_nhwc"] == (1, 7)
    m.use_cuda_graph = False
    eager = [m(x) for x in xs]
    m.use_cuda_graph = True
    for a, b in zip(outs, eager):
        assert torch.equal(a, b)
    assert not torch.equal(outs[0], outs[1])
    assert torch.equal(m(xs[3]), outs[3])            # deterministic replay
    sd2 = state_dict(load_spec(golden_dir, "tiny"), 99)
    m.load_state_dict({k: v.half() for k, v in sd2.items()}, strict=True)
    assert m._packed is None and graph.stats(m) == {}   # the old graphs went with the old packed weights
    new = m(xs[0])
    assert graph.stats(m)["_forward_nhwc"] == (0, 0)    # re-packed; this signature starts over with an eager call
    assert not torch.equal(new, outs[0])
    ref = depth_oracle.midas_forward({k: v.cuda() for k, v in sd2.items()}, make_input(2, 64, 96, 0).cuda(), **oracle_kw(TINY))
    assert _rel_l2(new, ref) < 5e-3


def _library_kernels():
    """Names of the __global__ functions defined in libvgen_b200.so's sources."""
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vgen_b200", "csrc")
    pat = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\((?:[^()]|\([^()]*\))*\)\s*)?(\w+)\s*\(")
    names = set()
    for fn in os.listdir(src):
        if fn.endswith((".cu", ".cuh")):
            names |= set(pat.findall(open(os.path.join(src, fn)).read()))
    return names


def _kernel_name(demangled):
    """'void vg::foo_kernel<32>(int, ...)' -> 'foo_kernel'."""
    head = demangled.split("(")[0].split("<")[0].strip()
    return head.split()[-1].split("::")[-1] if head else head


# Runs in a child process, so its profiling sessions leave no profiler state in the suite's process: run in-process, this
# test made test_gpu_longclip.py's profiler test, later in the same session, record no kernel events at all.
_PROFILE_CHILD = r"""
import json, sys
root, half = sys.argv[1], sys.argv[2] == "1"
sys.path[:0] = [root, root + "/tests"]
import torch
from torch.profiler import ProfilerActivity, profile
from _depth import DEPTH_CASES, load_spec, make_input, state_dict
from vgen_b200.depth import MiDaS
case = DEPTH_CASES["tiny_96x160_b2"]
m = MiDaS(**case["ctor"])
m.load_state_dict(state_dict(load_spec(root + "/tests/golden", "tiny"), case["seed"]), strict=True)
m = m.eval().requires_grad_(False)
x = make_input(case["n"], case["H"], case["W"], case["seed"]).cuda()
if half:
    m, x = m.to(memory_format=torch.channels_last).half(), x.half().contiguous(memory_format=torch.channels_last)
m = m.cuda()
out = {}
for graphed in (False, True):
    m.use_cuda_graph = graphed
    for _ in range(3):
        m(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m(x)
        torch.cuda.synchronize()
    out["graphed" if graphed else "eager"] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
print(json.dumps(out))
"""


@pytest.mark.parametrize("half", [True, False], ids=["fp16_channels_last", "fp32_contiguous"])
def test_forward_launches_only_library_kernels(half):
    """Every kernel of a forward, eager and graph-replayed, is one of libvgen_b200's (memcpy / memset aside)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, root, "1" if half else "0"], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    ours = _library_kernels()
    for mode, nms in names.items():
        foreign = {nm for nm in nms if _kernel_name(nm) not in ours and "memcpy" not in nm.lower() and "memset" not in nm.lower()}
        assert not foreign, (mode, foreign)
    for k in ("dpt_head_out_kernel", "dpt_tconv_scatter_kernel", "dpt_upsample_bilinear2x_kernel", "attn_sm90_kernel"):
        assert any(k in nm for nm in names["eager"]), (k, names["eager"])
