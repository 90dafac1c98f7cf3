"""Float64 reference of the tap-GEMM entry points and a per-element error bound to compare a kernel's output with.

Every conv and linear runs on one kernel family (`tapgemm_sm90_kernel<BN, kEpi>`).  The reference below computes what
that kernel is documented to compute, in float64 on the operands' device (so TF32 never enters), rounding to fp16
exactly where the kernel does and nowhere else:

    y = alpha * acc + bias                       (folded LayerNorm: alpha * (rstd * acc + (-mean rstd) * col_sum) + bias)
    per-frame bias / residual:  fp16(y) + g, then fp16(... ) + r
    GEGLU:                      fp16(fp16(value) * fp16(gelu(fp16(gate))))
    GELU / row bias:            fp16(gelu(acc + bias + row_bias))
    ReLU:                       fp16(max(alpha * acc + bias, 0))

with acc = sum over taps and channels of A[coord + tap offset] * W, the taps reading zeros outside the tensor.

Error bound.  Each quantity carries a value v (float64) and a bound d >= |kernel's fp32 value - v| (class `Bounded`):

* Accumulation.  The products of two fp16 numbers are exact in fp32; summing K of them in fp32 (the tensor core
  aligns and may truncate instead of round) errs by at most ~K * 2^-24 * S with S = (|A| @ |W|^T), the sum of the
  magnitudes.  The bound takes twice that: d_acc = 2 * K * 2^-24 * |scale| * S.
* Epilogue fp32 arithmetic (scale, bias, LayerNorm shift, row bias): a few roundings of 2^-24 relative to the
  magnitudes involved: 6 * 2^-24 * (|scale| S + |shift col_sum| + |bias| + |row_bias|).
* GELU is 1.13-Lipschitz (max of gelu'), so an input error d becomes 1.13 d, plus the kernel's own approximation
  (Abramowitz-Stegun erf, |error| < 1.5e-7, and approximate rcp / ex2), below 1e-6 * |x|.  ReLU passes d through.
* Intermediate fp16 rounding (before a per-frame bias or residual, and GEGLU's value, gate and gelu(gate)).  The
  reference rounds v itself; the kernel rounds some x in [v - d, v + d].  Rounding is monotone, so the kernel's
  result lies in [fp16(v - d), fp16(v + d)] and differs from fp16(v) by at most
      max(|fp16(v - d) - fp16(v)|, |fp16(v + d) - fp16(v)|),
  which is 0 unless a rounding boundary lies within d of v, and one ulp when one does (the "flip" of one ulp).
  That is the d carried forward: no ulp is added where no flip is possible.
* Products (GEGLU): |A' H' - A H| <= |A| dH + |H| dA + dA dH.
* Final fp16 rounding.  The output is fp16(x) with |x - v| <= d, so
      |out - v| <= 1/2 ulp16(|v| + d) + d.
  That is the per-element bound `check` enforces; the ratio |out - v| / bound is reported (a correctly rounded
  result sits at up to 1/2 ulp, i.e. a ratio near 1 for the worst element of a large tensor).

Unlike max|error| / max|ref|, the bound is relative to each element's own magnitude: an error confined to small
outputs (a dropped K chunk of a small row, a wrong bias on a column of small values) is caught.

The accumulation term is a worst case and grows with K.  For Gaussian data with unit-scale weights (the GPU matrix's
inputs), the median bound is 0.53 fp16 ulp of the output at K = 64, 0.58 at K = 128 and 0.83 at K = 320, so short-K
cases check the result to the last ulp.  At K = 5120 the median is 23 ulps (90th percentile 136), so long-K cases catch
gross faults such as a lost K chunk or a wrong ring wrap, but not a systematic error of a few ulps.
"""
from __future__ import annotations

import torch

U32 = 2.0 ** -24          # unit roundoff of fp32
ACC_C = 2.0               # fp32 accumulation: d_acc = ACC_C * K * U32 * S
EPI_C = 6.0               # epilogue fp32 roundings, relative to the magnitudes involved
GELU_L = 1.13             # max |gelu'(x)|
GELU_APPROX = 1e-6        # |kernel gelu - exact gelu| <= GELU_APPROX * |x|
FP16_MAX = 65504.0


def ulp16(x):
    """Spacing of fp16 numbers at |x| (subnormal spacing 2^-24 below 2^-14), float64."""
    ax = x.abs()
    e = torch.frexp(ax)[1].to(torch.float64) - 1.0           # floor(log2 |x|) for x != 0
    e = torch.where(ax == 0, torch.full_like(e, -14.0), e).clamp(min=-14.0)
    return torch.exp2(e - 10.0)


def rn16(x):
    """Round float64 to the nearest fp16 value, ties to even, exactly (x / ulp is exact: ulp is a power of two)."""
    q = ulp16(x)
    return torch.round(x / q) * q


class Bounded:
    """A float64 value v and a bound d on how far the kernel's fp32 value of the same quantity may be from it."""

    def __init__(self, v, d):
        self.v, self.d = v, d

    def round16(self):
        r = rn16(self.v)
        d = torch.maximum((rn16(self.v - self.d) - r).abs(), (rn16(self.v + self.d) - r).abs())
        return Bounded(r, d)

    def add(self, t):
        """self + t for an exact (fp16) addend t, summed in fp32."""
        return Bounded(self.v + t, self.d + U32 * (self.v.abs() + t.abs()))

    def gelu(self):
        v = gelu64(self.v)
        return Bounded(v, GELU_L * self.d + GELU_APPROX * (self.v.abs() + self.d) + 2 * U32 * v.abs())

    def relu(self):
        return Bounded(self.v.clamp(min=0), self.d)

    def mul(self, o):
        return Bounded(self.v * o.v, self.v.abs() * o.d + o.v.abs() * self.d + self.d * o.d)


def gelu64(x):
    """Exact-erf GELU (F.gelu's default) in float64."""
    return 0.5 * x * (1.0 + torch.erf(x * 0.5 ** 0.5))


def gemm(a, w):
    """acc = a @ w^T and S = |a| @ |w|^T in float64 on a's device (a [rows, K], w [n, K], any float dtype)."""
    a, w = a.double(), w.double()
    return a @ w.t(), a.abs() @ w.abs().t()


def tap_rows(x, taps):
    """x [d3, d2, d1, c] -> [d3 * d2 * d1, len(taps) * c] float64: row (i3, i2, i1) holds x[i3, i2 + o2, i1 + o1, :] for
    each tap (o2, o1) in turn, zero where that falls outside the d2 x d1 plane (the kernel's zero padding; the planes
    of different i3 -- images, videos -- never mix)."""
    d3, d2, d1, c = x.shape
    out = torch.zeros(d3, d2, d1, len(taps), c, dtype=torch.float64, device=x.device)
    xd = x.double()
    for t, (o2, o1) in enumerate(taps):
        a2, b2 = max(0, -o2), min(d2, d2 - o2)
        a1, b1 = max(0, -o1), min(d1, d1 - o1)
        if a2 < b2 and a1 < b1:
            out[:, a2:b2, a1:b1, t] = xd[:, a2 + o2:b2 + o2, a1 + o1:b1 + o1]
    return out.reshape(d3 * d2 * d1, len(taps) * c)


TAPS_3X3 = [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)]   # k = (ky * 3 + kx) * c + ci
TAPS_T3 = [(kt - 1, 0) for kt in range(3)]                              # x viewed as [videos, f, hw, c]


def epilogue(acc, S, k, alpha=1.0, bias=None, group_bias=None, residual=None, ln=None, geglu=False, gelu=False,
             row_bias=None, relu=False):
    """The kernel's epilogue on float64 accumulators acc [rows, n] (S = |A| @ |W|^T, k = the reduction length).

    bias [n]; group_bias / residual / row_bias already expanded to [rows, n]; ln = (row_stats [rows, 2] = {rstd,
    -mean rstd}, col_sum [n]).  GEGLU: columns in GEGLU.proj's order, the n / 2 values then their n / 2 gates (the
    reference never sees the kernel's per-tile interleave of the weight rows).
    Returns a `Bounded` output of n (GEGLU: n / 2) columns."""
    z = torch.zeros((), dtype=torch.float64, device=acc.device)
    f64 = lambda t: z if t is None else t.double()   # noqa: E731
    if ln is not None:
        stats, cs = ln[0].double(), ln[1].double()
        scale = alpha * stats[:, :1]
        shift = alpha * stats[:, 1:] * cs[None, :]
    else:
        scale, shift = torch.full((1, 1), float(alpha), dtype=torch.float64, device=acc.device), z
    b, rb = f64(bias), f64(row_bias)
    y = acc * scale + shift + b + rb
    mag = scale.abs() * S + shift.abs() + b.abs() + rb.abs()
    out = Bounded(y, ACC_C * k * U32 * scale.abs() * S + EPI_C * U32 * mag)
    if geglu:
        h = y.shape[1] // 2
        value = Bounded(out.v[:, :h], out.d[:, :h]).round16()
        gate = Bounded(out.v[:, h:], out.d[:, h:]).round16()
        return value.mul(gate.gelu().round16())
    if gelu:
        out = out.gelu()
    if relu:
        out = out.relu()
    if group_bias is not None:
        out = out.round16().add(group_bias.double())
    if residual is not None:
        out = out.round16().add(residual.double())
    return out


def ln_reference(stats, col_sum, acc, bias=None):
    """rstd * acc + (-mean rstd) * col_sum + bias: the folded LayerNorm -> Linear of the epilogue, in float64."""
    y = stats[:, :1].double() * acc + stats[:, 1:].double() * col_sum.double()[None, :]
    return y if bias is None else y + bias.double()


def check(out, ref: Bounded, what=""):
    """Assert |out - ref.v| <= 1/2 ulp16(|ref.v| + ref.d) + ref.d for every element; return the largest error / bound."""
    assert out.shape == ref.v.shape, (what, tuple(out.shape), tuple(ref.v.shape))
    top = float((ref.v.abs() + ref.d).max()) if ref.v.numel() else 0.0
    assert top < FP16_MAX, f"{what}: the reference leaves the fp16 range ({top}); the test data are too large"
    o = out.double()
    bound = 0.5 * ulp16(ref.v.abs() + ref.d) + ref.d
    err = (o - ref.v).abs()
    bad = ~(torch.isfinite(o) & (err <= bound))
    if bool(bad.any()):
        idx = bad.nonzero()[:5].tolist()
        det = [(i, float(o[tuple(i)]), float(ref.v[tuple(i)]), float(bound[tuple(i)])) for i in idx]
        raise AssertionError(f"{what}: {int(bad.sum())} of {o.numel()} elements outside the bound; "
                             f"first (index, out, ref, bound): {det}")
    return float((err / bound).max()) if err.numel() else 0.0

