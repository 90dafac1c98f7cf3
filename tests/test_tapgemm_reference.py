"""The tap-GEMM reference and its per-element bound (tests/_tapgemm_ref.py), on the CPU: the reference agrees with
PyTorch's float64 conv / LayerNorm / linear / GELU, a correct fp32 computation passes the bound, and outputs with the
kinds of bugs a GEMM kernel has are rejected -- including ones the max-normalised metric of tools/gpu_check.py
(max |error| / max |ref| <= 2e-3) lets through."""
import pytest
import torch
import torch.nn.functional as F

import _tapgemm_ref as R


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _operands(m=200, k=256, n=96, seed=0):
    g = _gen(seed)
    a = torch.randn(m, k, generator=g)
    a[:16] *= 1e-3                                   # a small-magnitude region (rows 0..15)
    w = torch.randn(n, k, generator=g) * k ** -0.5
    return a.half(), w.half(), torch.randn(n, generator=g), torch.randn(m, n, generator=g).half()


def _out(ref):
    """What a kernel without fp32 error would store: the final value rounded once."""
    return R.rn16(ref.v).half()


def _max_normalised(out, ref):
    return float((out.double() - ref.v).abs().max() / ref.v.abs().max())


def _rejects(out, ref):
    with pytest.raises(AssertionError, match="outside the bound"):
        R.check(out, ref)


# ------------------------------------------------------------------------------------------------ rounding helpers
def test_rn16_and_ulp16_match_fp16():
    g = _gen(1)
    x = torch.cat([torch.randn(20000, generator=g) * 10 ** torch.randint(-8, 4, (20000,), generator=g).float(),
                   torch.tensor([0.0, 2.0 ** -24, 3 * 2.0 ** -25, 2.0 ** -14, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11,
                                 2048.0 + 1.0, 65504.0, -(2.0 ** -15) - 2.0 ** -25])])
    # float32 inputs: PyTorch's float32 -> fp16 conversion is a single correct rounding
    assert torch.equal(R.rn16(x.double()), x.half().double())
    h = x.half().double()
    nxt = torch.nextafter(x.half(), torch.tensor(float("inf")).half()).double()
    fin = (h > 0) & (h < 65504)
    assert torch.equal(R.ulp16(h)[fin], (nxt - h)[fin])


def test_gelu64_matches_torch():
    x = torch.linspace(-12, 12, 4001, dtype=torch.float64)
    assert torch.allclose(R.gelu64(x), F.gelu(x), rtol=1e-14, atol=1e-15)


# ------------------------------------------------------------------------------------------------ reference vs torch
@pytest.mark.parametrize("nimg,h,w", [(2, 5, 7), (3, 1, 1), (1, 1, 37), (2, 4, 3)])
def test_conv3x3_reference_matches_conv2d(nimg, h, w):
    g = _gen(h * 100 + w)
    x = torch.randn(nimg, h, w, 8, generator=g, dtype=torch.float64)
    wt = torch.randn(5, 8, 3, 3, generator=g, dtype=torch.float64)
    acc, _ = R.gemm(R.tap_rows(x, R.TAPS_3X3), wt.permute(0, 2, 3, 1).reshape(5, 72))
    want = F.conv2d(x.permute(0, 3, 1, 2), wt, padding=1).permute(0, 2, 3, 1).reshape(-1, 5)
    assert torch.allclose(acc, want, rtol=1e-12, atol=1e-12)


def test_tap_list_reference_matches_dilated_conv_and_far_taps_read_zeros():
    g = _gen(2)
    x = torch.randn(2, 6, 9, 4, generator=g, dtype=torch.float64)
    wt = torch.randn(3, 4, 3, 3, generator=g, dtype=torch.float64)
    taps = [(2 * (ky - 1), 2 * (kx - 1)) for ky in range(3) for kx in range(3)]
    acc, _ = R.gemm(R.tap_rows(x, taps), wt.permute(0, 2, 3, 1).reshape(3, 36))
    want = F.conv2d(x.permute(0, 3, 1, 2), wt, padding=2, dilation=2).permute(0, 2, 3, 1).reshape(-1, 3)
    assert torch.allclose(acc, want, rtol=1e-12, atol=1e-12)
    far = R.tap_rows(x, [(127, 0), (0, -127), (-127, 127)])
    assert not far.any()


def test_tconv3_reference_pads_each_video():
    g = _gen(3)
    x = torch.randn(3, 5, 6, 4, generator=g, dtype=torch.float64)       # [videos, f, hw, c]
    wt = torch.randn(7, 4, 3, generator=g, dtype=torch.float64)
    acc, _ = R.gemm(R.tap_rows(x, R.TAPS_T3), wt.permute(0, 2, 1).reshape(7, 12))
    want = torch.cat([F.conv3d(v.permute(2, 0, 1)[None, :, :, :, None], wt[..., None, None], padding=(1, 0, 0))[0]
                      .permute(1, 2, 3, 0).reshape(-1, 7) for v in x])
    assert torch.allclose(acc, want, rtol=1e-12, atol=1e-12)


def test_folded_layer_norm_reference_is_layer_norm_then_linear():
    g = _gen(4)
    x = torch.randn(33, 64, generator=g, dtype=torch.float64) * 2 + 40 * torch.randn(33, 1, generator=g, dtype=torch.float64)
    w = torch.randn(24, 64, generator=g, dtype=torch.float64)
    b, gam, bet = (torch.randn(24, generator=g, dtype=torch.float64), 1 + 0.3 * torch.randn(64, generator=g, dtype=torch.float64),
                   0.2 * torch.randn(64, generator=g, dtype=torch.float64))
    mean, var = x.mean(1), x.var(1, unbiased=False)
    rstd = (var + 1e-5).rsqrt()
    stats = torch.stack([rstd, -mean * rstd], 1)
    wf = w * gam[None, :]
    acc, _ = R.gemm(x, wf)
    got = R.ln_reference(stats, wf.sum(1), acc, b + w @ bet)
    want = F.linear(F.layer_norm(x, (64,), gam, bet, 1e-5), w, b)
    assert torch.allclose(got, want, rtol=1e-9, atol=1e-9)


# ------------------------------------------------------------------------------------------------ the bound has teeth
def test_fp32_computation_passes_the_bound():
    """An honest fp32 implementation of each epilogue (a CPU fp32 matmul, fp16 roundings where the kernel rounds) passes."""
    a, w, b, r = _operands(k=1024)
    acc, S = R.gemm(a, w)
    acc32 = a.float() @ w.float().t()
    r1 = R.check(((acc32 * 0.37 + b).half().float() + r.float()).half(), R.epilogue(acc, S, 1024, alpha=0.37, bias=b, residual=r))
    hb = 48
    v32, g32 = acc32[:, :hb] + b[:hb], acc32[:, hb:] + b[hb:]
    geglu32 = (v32.half().float() * F.gelu(g32.half().float()).half().float()).half()
    r2 = R.check(geglu32, R.epilogue(acc, S, 1024, bias=b, geglu=True))
    r3 = R.check(F.gelu(acc32 + b).half(), R.epilogue(acc, S, 1024, bias=b, gelu=True))
    r4 = R.check(torch.relu(acc32 + b).half(), R.epilogue(acc, S, 1024, bias=b, relu=True))
    assert max(r1, r2, r3, r4) <= 1.0


def test_rejects_four_ulp_in_a_small_region():
    a, w, b, _ = _operands()
    acc, S = R.gemm(a, w)
    ref = R.epilogue(acc, S, a.shape[1])
    out = _out(ref)
    R.check(out, ref)
    bad = out.clone()
    bad[3, 5] = (bad[3, 5].double() + 4 * R.ulp16(bad[3, 5].double())).half()
    assert _max_normalised(bad, ref) < 2e-3           # invisible to max |error| / max |ref|
    _rejects(bad, ref)


def test_rejects_two_rows_swapped_in_a_tile():
    a, w, b, _ = _operands()
    acc, S = R.gemm(a, w)
    ref = R.epilogue(acc, S, a.shape[1], bias=b)
    out = _out(ref)
    R.check(out, ref)
    _rejects(out[[*range(0, 40), 41, 40, *range(42, 200)]], ref)


def test_rejects_a_dropped_k_chunk():
    a, w, b, _ = _operands(k=512)
    acc, S = R.gemm(a, w)
    ref = R.epilogue(acc, S, 512, bias=b)
    a_drop = a.clone()
    a_drop[:, 192:256] = 0
    acc_drop, _ = R.gemm(a_drop, w)
    out = _out(R.epilogue(acc_drop, S, 512, bias=b))
    _rejects(out, ref)
    # confined to the small rows, the same bug stays under the max-normalised tolerance
    out_small = _out(ref).clone()
    out_small[:16] = out[:16]
    assert _max_normalised(out_small, ref) < 2e-3
    _rejects(out_small, ref)


def test_rejects_an_omitted_residual():
    a, w, b, r = _operands()
    acc, S = R.gemm(a, w)
    ref = R.epilogue(acc, S, a.shape[1], bias=b, residual=r)
    R.check(_out(ref), ref)
    _rejects(_out(R.epilogue(acc, S, a.shape[1], bias=b)), ref)


def test_rejects_bias_on_the_neighbouring_column_pair():
    a, w, b, _ = _operands()
    acc, S = R.gemm(a, w)
    ref = R.epilogue(acc, S, a.shape[1], bias=b)
    _rejects(_out(R.epilogue(acc, S, a.shape[1], bias=torch.roll(b, -2))), ref)


def test_rejects_geglu_gate_from_the_next_block():
    """A kernel reading the gate of value block j from block j + 1 of the per-tile interleave (BN = 64: 32 columns)."""
    a, w, b, _ = _operands(n=256)
    acc, S = R.gemm(a, w)
    ref = R.epilogue(acc, S, a.shape[1], bias=b, geglu=True)
    R.check(_out(ref), ref)
    y = acc + b.double()
    value, gate = y[:, :128], torch.roll(y[:, 128:], -32, dims=1)
    bad = R.rn16(R.rn16(value) * R.rn16(R.gelu64(R.rn16(gate)))).half()
    _rejects(bad, ref)


def test_rejects_non_finite_output():
    a, w, b, _ = _operands()
    acc, S = R.gemm(a, w)
    ref = R.epilogue(acc, S, a.shape[1])
    out = _out(ref).clone()
    out[7, 7] = float("nan")
    _rejects(out, ref)
