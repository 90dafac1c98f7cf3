"""Tensor-level wrappers over the C ABI: they check shapes/dtypes, allocate outputs with torch
(device memory plumbing only) and pass raw pointers + the current CUDA stream to libvgen_b200.so.

Layout convention: activations fp16 channels-last ("rows x channels"); weights fp16 [out][taps*in];
bias / affine parameters fp32.
"""
from __future__ import annotations

import ctypes

import torch

from . import lib as _l
from .lib import Epilogue


class KernelProfile:
    """Optional per-kernel-family device timing (CUDA events on the launching stream) + algorithmic
    work counters.  Used by bench.py for the roofline line; off by default (PROF is None)."""

    def __init__(self):
        self.records = []  # (family, flops, bytes, start_event, stop_event)

    def run(self, family, flops, nbytes, fn, tag=None):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        rc = fn()
        e.record()
        self.records.append((family, float(flops), float(nbytes), s, e, tag))
        return rc

    def by_shape(self):
        torch.cuda.synchronize()
        out = {}
        for fam, fl, nb, s, e, tag in self.records:
            d = out.setdefault(f"{fam}:{tag}", {"launches": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            d["launches"] += 1
            d["ms"] += s.elapsed_time(e)
            d["flops"] += fl
            d["bytes"] += nb
        return out

    def summary(self):
        torch.cuda.synchronize()
        out = {}
        for fam, fl, nb, s, e, _tag in self.records:
            d = out.setdefault(fam, {"launches": 0, "ms": 0.0, "flops": 0.0, "bytes": 0.0})
            d["launches"] += 1
            d["ms"] += s.elapsed_time(e)
            d["flops"] += fl
            d["bytes"] += nb
        return out


PROF = None  # set to a KernelProfile() to instrument calls


def _run(family, flops, nbytes, fn, tag=None):
    if PROF is None:
        return fn()
    return PROF.run(family, flops, nbytes, fn, tag)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk16(t, name):
    if t.dtype != torch.float16 or not t.is_cuda:
        raise _l.VgenError(f"{name}: expected a CUDA fp16 tensor, got {t.dtype} on {t.device}")


def _rows_view(t, name):
    """(rows, ld) of a tensor whose last dim is contiguous and whose leading dims are row-dense."""
    if t.stride(-1) != 1:
        raise _l.VgenError(f"{name}: innermost dimension must be contiguous")
    t2 = t.reshape(-1, t.shape[-1]) if t.is_contiguous() else t
    if t2.dim() != 2:
        raise _l.VgenError(f"{name}: non-contiguous tensors must be 2-D row views")
    return t2, t2.stride(0)


def _epilogue(n_out, bias=None, group_bias=None, residual=None, alpha=1.0, geglu=False, bn=0, group_div=1, ln=None):
    e = Epilogue()
    e.alpha = float(alpha)
    keep = []
    if ln is not None:   # (row_stats [rows, 2] fp32, col_sum [n] fp32): LayerNorm folded into the GEMM
        stats, col_sum = ln
        if stats.dtype != torch.float32 or col_sum.dtype != torch.float32 or not stats.is_contiguous() or not col_sum.is_contiguous():
            raise _l.VgenError("ln: row_stats and col_sum must be contiguous fp32 tensors")
        if residual is not None or group_bias is not None:
            raise _l.VgenError("ln: a folded LayerNorm cannot be combined with residual / group_bias")
        e.row_stats = stats.data_ptr()
        e.col_sum = col_sum.data_ptr()
        keep += [stats, col_sum]
    if bias is not None:
        if bias.dtype != torch.float32:
            raise _l.VgenError("bias must be fp32")
        e.bias = bias.data_ptr()
        keep.append(bias)
    if group_bias is not None:
        _chk16(group_bias, "group_bias")
        e.group_bias = group_bias.data_ptr()
        e.group_bias_ld = group_bias.stride(0)
        e.group_bias_div = int(group_div)
        keep.append(group_bias)
    if residual is not None:
        _chk16(residual, "residual")
        r2, ldr = _rows_view(residual, "residual")
        if r2.shape[-1] != n_out:
            raise _l.VgenError(f"residual has {r2.shape[-1]} columns, expected {n_out}")
        e.residual = r2.data_ptr()
        e.residual_ld = ldr
        keep.append(r2)
    if geglu and residual is not None:
        raise _l.VgenError("the GEGLU epilogue takes no residual")
    e.geglu = 1 if geglu else 0
    e.bn = int(bn)
    return e, keep


def linear(a, w, bias=None, residual=None, alpha=1.0, geglu=False, out=None, bn=0, ln=None):
    """out[m, n] = epi(a[m, k] @ w[n, k]^T).  `a` may be a row-strided 2-D view.

    ln = (row_stats(a), col_sum): `a` is the INPUT of a LayerNorm whose affine part was folded into w / bias
    (fold_layer_norm); the epilogue applies the per-row statistics, so LN(a) is never materialised."""
    _chk16(a, "a"), _chk16(w, "w")
    lead = a.shape[:-1]
    a2, lda = _rows_view(a, "a")
    m, k = a2.shape
    n = w.shape[0]
    if w.shape[1] != k or not w.is_contiguous():
        raise _l.VgenError(f"linear: weight {tuple(w.shape)} does not match k={k}")
    n_out = n // 2 if geglu else n
    if out is None:
        out = torch.empty(*lead, n_out, device=a.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    if ln is not None and (ln[0].shape != (m, 2) or ln[1].numel() != n):
        raise _l.VgenError(f"linear: ln shapes {tuple(ln[0].shape)} / {tuple(ln[1].shape)} do not match m={m}, n={n}")
    e, keep = _epilogue(n_out, bias, None, residual, alpha, geglu, bn, ln=ln)
    rc = _run("tapgemm", 2.0 * m * n * k, 2.0 * (m * k + n * k + m * n_out),
              lambda: _l.load().vgen_linear(_p(a2), m, k, lda, _p(w), n, _p(o2), ldo, ctypes.byref(e), _stream()),
              tag=f"linear m{m} k{k} n{n}{' geglu' if geglu else ''}{' res' if residual is not None else ''}{' ln' if ln is not None else ''}")
    _l.check(rc, "vgen_linear")
    return out


def linear_lora(a, w, h, u, bias=None, residual=None, out=None, bn=0):
    """out[m, n] = epi(a[m, k] @ w[n, k]^T + h[m, r] @ u[n, r]^T): a projection with the LoRA up projection as a K tail of
    the same GEMM (one fp32 accumulator, one rounding).  h: lora_down's [m, r] output (r a multiple of 64), u: the up weights
    [n, r].  `a` and `h` may be row-strided 2-D views."""
    _chk16(a, "a"), _chk16(w, "w"), _chk16(h, "h"), _chk16(u, "u")
    lead = a.shape[:-1]
    a2, lda = _rows_view(a, "a")
    h2, ldh = _rows_view(h, "h")
    m, k = a2.shape
    n, r = w.shape[0], u.shape[1]
    if w.shape[1] != k or not w.is_contiguous():
        raise _l.VgenError(f"linear_lora: weight {tuple(w.shape)} does not match k={k}")
    if tuple(h2.shape) != (m, r) or u.shape[0] != n or not u.is_contiguous():
        raise _l.VgenError(f"linear_lora: h {tuple(h2.shape)} / u {tuple(u.shape)} do not match m={m}, n={n}")
    if out is None:
        out = torch.empty(*lead, n, device=a.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    e, keep = _epilogue(n, bias, None, residual, 1.0, False, bn)
    rc = _run("tapgemm", 2.0 * m * n * (k + r), 2.0 * (m * (k + r) + n * (k + r) + m * n),
              lambda: _l.load().vgen_linear_lora(_p(a2), m, k, lda, _p(w), n, _p(h2), r, ldh, _p(u), _p(o2), ldo,
                                                 ctypes.byref(e), _stream()),
              tag=f"linear_lora m{m} k{k} r{r} n{n}{' res' if residual is not None else ''}")
    _l.check(rc, "vgen_linear_lora")
    return out


def lora_down(x, d, col_set, col_scale, strength, rows_per_sample, r_pad, out=None):
    """h[m, r_pad] = fp16(strength[row // rows_per_sample, col_set[j]] * col_scale[j] * x[row] . d[j]), zero past d's rows:
    the LoRA down projection of every set and every projection reading x, with the per-sample strength [samples, sets]
    (fp32 on the device) folded in."""
    _chk16(x, "x"), _chk16(d, "d")
    x2, ldx = _rows_view(x, "x")
    m, k = x2.shape
    r = d.shape[0]
    if d.shape[1] != k or not d.is_contiguous():
        raise _l.VgenError(f"lora_down: d {tuple(d.shape)} does not match k={k}")
    if col_set.dtype != torch.int32 or col_scale.dtype != torch.float32 or col_set.numel() != r or col_scale.numel() != r:
        raise _l.VgenError(f"lora_down: col_set must be int32 [{r}] and col_scale fp32 [{r}]")
    if (strength.dtype != torch.float32 or strength.dim() != 2 or not strength.is_contiguous()
            or strength.shape[0] * rows_per_sample < m or strength.device != x.device):
        raise _l.VgenError(f"lora_down: strength must be contiguous fp32 [samples, sets] covering {m} rows")
    if out is None:
        out = torch.empty(m, r_pad, device=x.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    rc = _run("lora_down", 2.0 * m * r * k, 2.0 * (m * k + r * k + m * r_pad),
              lambda: _l.load().vgen_lora_down(_p(x2), m, k, ldx, _p(d), r, _p(col_set), _p(col_scale), _p(strength),
                                               strength.shape[1], int(rows_per_sample), _p(o2), ldo, int(r_pad), _stream()),
              tag=f"m{m} k{k} r{r}")
    _l.check(rc, "vgen_lora_down")
    return out


E4M3_MAX = 448.0


def quantize_weight_e4m3(w):
    """Per-output-channel e4m3 quantisation of a GEMM weight [n, k] (any float dtype; the amax is taken in fp32):
    -> (codes uint8 [n, k], scale fp32 [n]) with scale = amax / 448 (1 for an all-zero row) and
    codes = e4m3(w / scale), round to nearest even.  Runs on w's device (pack time, not the hot path)."""
    w = w.detach().float()
    amax = w.abs().amax(dim=1)
    scale = torch.where(amax > 0, (amax.double() / E4M3_MAX).float(), torch.ones_like(amax))   # correctly rounded
    codes = (w / scale[:, None]).to(torch.float8_e4m3fn).view(torch.uint8)
    return codes.contiguous(), scale.contiguous()


def quantize_rows_e4m3(x, out=None, scale=None):
    """x fp16 [m, k] (a row-strided 2-D view is fine) -> (codes uint8 [m, k], scale fp32 [m]): one launch of the row
    quantiser, scale = amax_row / 448 (1 for an all-zero row), codes = e4m3(x / scale) with saturation."""
    _chk16(x, "x")
    x2, ldx = _rows_view(x, "x")
    m, k = x2.shape
    if out is None:
        out = torch.empty(m, k, device=x.device, dtype=torch.uint8)
    if scale is None:
        scale = torch.empty(m, device=x.device, dtype=torch.float32)
    if out.dtype != torch.uint8 or tuple(out.shape) != (m, k) or out.stride(1) != 1:
        raise _l.VgenError(f"quantize_rows_e4m3: out must be uint8 [{m}, {k}] with contiguous rows")
    if scale.dtype != torch.float32 or scale.numel() != m or not scale.is_contiguous():
        raise _l.VgenError(f"quantize_rows_e4m3: scale must be contiguous fp32 [{m}]")
    rc = _run("quantize_e4m3", 0.0, 3.0 * m * k,
              lambda: _l.load().vgen_quantize_rows_e4m3(_p(x2), m, k, ldx, _p(out), out.stride(0), _p(scale), _stream()),
              tag=f"quantize m{m} k{k}")
    _l.check(rc, "vgen_quantize_rows_e4m3")
    return out, scale


def linear_e4m3(a8, a_scale, w8, w_scale, bias=None, residual=None, alpha=1.0, geglu=False, out=None, bn=0):
    """out[m, n] = epi(a_scale[m] * w_scale[n] * (a8[m, k] @ w8[n, k]^T)) on e4m3 codes (uint8 tensors) with fp32
    accumulation; the epilogue (bias / residual / GEGLU, fp16 output) is that of linear()."""
    if a8.dtype != torch.uint8 or w8.dtype != torch.uint8 or not a8.is_cuda:
        raise _l.VgenError("linear_e4m3: a8 and w8 must be CUDA uint8 tensors of e4m3 codes")
    a2, lda = _rows_view(a8, "a8")
    m, k = a2.shape
    n = w8.shape[0]
    if w8.dim() != 2 or w8.shape[1] != k or not w8.is_contiguous():
        raise _l.VgenError(f"linear_e4m3: weight {tuple(w8.shape)} does not match k={k}")
    for t, cnt, name in ((a_scale, m, "a_scale"), (w_scale, n, "w_scale")):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != cnt:
            raise _l.VgenError(f"linear_e4m3: {name} must be contiguous fp32 [{cnt}]")
    n_out = n // 2 if geglu else n
    if out is None:
        out = torch.empty(*a8.shape[:-1], n_out, device=a8.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    e, keep = _epilogue(n_out, bias, None, residual, alpha, geglu, bn)
    rc = _run("tapgemm_fp8", 2.0 * m * n * k, 1.0 * (m * k + n * k) + 2.0 * m * n_out,
              lambda: _l.load().vgen_linear_fp8(_p(a2), _p(a_scale), m, k, lda, _p(w8), _p(w_scale), n, _p(o2), ldo,
                                                ctypes.byref(e), _stream()),
              tag=f"linear_fp8 m{m} k{k} n{n}{' geglu' if geglu else ''}{' res' if residual is not None else ''}")
    _l.check(rc, "vgen_linear_fp8")
    return out


def linear_fp8(a, w8, w_scale, bias=None, residual=None, alpha=1.0, geglu=False, out=None, bn=0):
    """linear() with e4m3 operands: the fp16 activations `a` are quantised per row (quantize_rows_e4m3), then multiplied
    with the per-channel quantised weight (w8, w_scale from quantize_weight_e4m3) by the FP8 tap-GEMM."""
    lead = a.shape[:-1]
    n_out = w8.shape[0] // 2 if geglu else w8.shape[0]
    _epilogue(n_out, bias, None, residual, alpha, geglu, bn)   # refuse a bad epilogue before the quantiser launches
    a8, a_scale = quantize_rows_e4m3(a)
    if out is None:
        out = torch.empty(*lead, n_out, device=a.device, dtype=torch.float16)
    linear_e4m3(a8, a_scale, w8, w_scale, bias=bias, residual=residual, alpha=alpha, geglu=geglu, out=out, bn=bn)
    return out


def linear_gelu_rowbias(a, w, bias=None, row_bias=None, rows_per_group=1, out=None):
    """out[m, j] = fp16(gelu_erf(a[m] . w[j] + bias[j] + row_bias[m // rows_per_group, j])): the adapter down projection.
    The fp32 row bias [groups, n] (a row-strided 2-D view is fine) is added to the fp32 accumulator before the activation;
    `a` and `out` may be row-strided 2-D views (out e.g. the K tail of the buffer the fused up projection reads)."""
    _chk16(a, "a"), _chk16(w, "w")
    a2, lda = _rows_view(a, "a")
    m, k = a2.shape
    n = w.shape[0]
    if w.shape[1] != k or not w.is_contiguous():
        raise _l.VgenError(f"linear_gelu_rowbias: weight {tuple(w.shape)} does not match k={k}")
    if bias is not None and (bias.dtype != torch.float32 or not bias.is_contiguous() or bias.numel() != n):
        raise _l.VgenError(f"linear_gelu_rowbias: bias must be contiguous fp32 [{n}]")
    ldg = 0
    if row_bias is not None:
        if (row_bias.dtype != torch.float32 or row_bias.dim() != 2 or row_bias.shape[1] != n or row_bias.stride(1) != 1
                or row_bias.device != a.device):
            raise _l.VgenError(f"linear_gelu_rowbias: row_bias must be fp32 [groups, {n}] with contiguous rows on {a.device}")
        if rows_per_group < 1 or row_bias.shape[0] * rows_per_group < m:
            raise _l.VgenError(f"linear_gelu_rowbias: {row_bias.shape[0]} row-bias rows x {rows_per_group} do not cover {m} rows")
        ldg = row_bias.stride(0)
    if out is None:
        out = torch.empty(m, n, device=a.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    if tuple(o2.shape) != (m, n):
        raise _l.VgenError(f"linear_gelu_rowbias: out is {tuple(o2.shape)}, expected {(m, n)}")
    rc = _run("tapgemm", 2.0 * m * n * k, 2.0 * (m * k + n * k + m * n),
              lambda: _l.load().vgen_linear_gelu_rowbias(_p(a2), m, k, lda, _p(w), n, _p(bias), _p(row_bias), ldg,
                                                         int(rows_per_group), _p(o2), ldo, _stream()),
              tag=f"adapter down m{m} k{k} n{n}")
    _l.check(rc, "vgen_linear_gelu_rowbias")
    return out


def adapter_condition(c, w, v, lam=None, lam_scalar=1.0, groups_per_lam=1):
    """g[r, j] = lam[r // groups_per_lam] * (c[r] . w[j] + v[j]) as fp32 [rows, n]: the condition term of every conditioned
    adapter at once (w / v: the stacked down.W @ condition_linear.W / down.W @ condition_linear.b).  lam: fp32 [groups]
    on the device, or None for lam_scalar."""
    _chk16(c, "c"), _chk16(w, "w")
    c2, ldc = _rows_view(c, "c")
    rows, k = c2.shape
    n = w.shape[0]
    if w.shape[1] != k or not w.is_contiguous():
        raise _l.VgenError(f"adapter_condition: weight {tuple(w.shape)} does not match k={k}")
    if v.dtype != torch.float32 or not v.is_contiguous() or v.numel() != n:
        raise _l.VgenError(f"adapter_condition: v must be contiguous fp32 [{n}]")
    if lam is not None and (lam.dtype != torch.float32 or not lam.is_contiguous() or lam.device != c.device
                            or lam.numel() * groups_per_lam < rows):
        raise _l.VgenError("adapter_condition: lam must be a contiguous fp32 tensor on c's device with one entry per group")
    g = torch.empty(rows, n, device=c.device, dtype=torch.float32)
    rc = _run("adapter_condition", 2.0 * rows * n * k, 2.0 * (rows * k + n * k) + 4.0 * rows * n,
              lambda: _l.load().vgen_adapter_condition(_p(c2), rows, k, ldc, _p(w), _p(v), n, _p(lam), float(lam_scalar),
                                                       int(groups_per_lam), _p(g), n, _stream()))
    _l.check(rc, "vgen_adapter_condition")
    return g


def conv2d_3x3(x, w, bias=None, group_bias=None, residual=None, out=None, bn=0, group_div=1):
    """x [nimg, h, w, c] fp16 -> [nimg, h, w, n]; w [n, 9*c] with k = (ky*3+kx)*c + ci."""
    _chk16(x, "x"), _chk16(w, "w")
    if not x.is_contiguous() or x.dim() != 4:
        raise _l.VgenError("conv2d_3x3: x must be contiguous [nimg,h,w,c]")
    nimg, h, wd, c = x.shape
    n = w.shape[0]
    if w.shape[1] != 9 * c or not w.is_contiguous():
        raise _l.VgenError(f"conv2d_3x3: weight {tuple(w.shape)} does not match c={c}")
    if out is None:
        out = torch.empty(nimg, h, wd, n, device=x.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    e, keep = _epilogue(n, bias, group_bias, residual, 1.0, False, bn, group_div)
    rows = nimg * h * wd
    rc = _run("tapgemm", 2.0 * rows * n * 9 * c, 2.0 * (rows * c + 9 * c * n + rows * n),
              lambda: _l.load().vgen_conv2d_3x3(_p(x), nimg, h, wd, c, _p(w), n, _p(o2), ldo, ctypes.byref(e), _stream()),
              tag=f"conv3x3 {nimg}x{h}x{wd} c{c} n{n}")
    _l.check(rc, "vgen_conv2d_3x3")
    return out


def tconv3(x, w, bias=None, residual=None, out=None, bn=0):
    """x [f, hw, c] (one video) or [b, f, hw, c] (videos back to back) fp16 -> same with n channels; temporal 3-tap
    conv, zero padded at every video's first / last frame; w [n, 3*c], k = kt*c + ci."""
    _chk16(x, "x"), _chk16(w, "w")
    if not x.is_contiguous() or x.dim() not in (3, 4):
        raise _l.VgenError("tconv3: x must be contiguous [f,hw,c] or [b,f,hw,c]")
    b = 1 if x.dim() == 3 else x.shape[0]
    f, hw, c = x.shape[-3:]
    n = w.shape[0]
    if w.shape[1] != 3 * c or not w.is_contiguous():
        raise _l.VgenError(f"tconv3: weight {tuple(w.shape)} does not match c={c}")
    if out is None:
        out = torch.empty(*x.shape[:-1], n, device=x.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    e, keep = _epilogue(n, bias, None, residual, 1.0, False, bn)
    rc = _run("tapgemm", 2.0 * b * f * hw * n * 3 * c, 2.0 * (b * f * hw * c + 3 * c * n + b * f * hw * n),
              lambda: _l.load().vgen_tconv3_batch(_p(x), b, f, hw, c, _p(w), n, _p(o2), ldo, ctypes.byref(e), _stream()),
              tag=f"tconv3 b{b} f{f} hw{hw} c{c} n{n}")
    _l.check(rc, "vgen_tconv3")
    return out


def set_tapgemm_impl(impl: str):
    _l.check(_l.load().vgen_set_tapgemm_impl({"auto": 0, "simt": 1}[impl]), "vgen_set_tapgemm_impl")


def set_tapgemm_bn(bn: int):
    """Force the N tile of every fp16 tap-GEMM launch that does not pass its own bn (0 = the heuristic again).  A debug
    knob: the tests reach each kernel instantiation with it."""
    _l.check(_l.load().vgen_set_tapgemm_bn(int(bn)), "vgen_set_tapgemm_bn")


def pack_geglu_weight(w, bias, bn):
    """Interleave GEGLU.proj rows so every bn-block holds bn/2 value rows then their bn/2 gate rows.

    w: [2*inner, k] (first half = value, second half = gate, reference util.py:711-714).
    """
    two_inner, k = w.shape
    inner = two_inner // 2
    hb = bn // 2
    assert inner % hb == 0
    v = w[:inner].reshape(inner // hb, hb, k)
    g = w[inner:].reshape(inner // hb, hb, k)
    wp = torch.cat([v, g], dim=1).reshape(two_inner, k).contiguous()
    bp = None
    if bias is not None:
        bv = bias[:inner].reshape(inner // hb, hb)
        bg = bias[inner:].reshape(inner // hb, hb)
        bp = torch.cat([bv, bg], dim=1).reshape(two_inner).contiguous()
    return wp, bp


# ------------------------------------------------------------------------------------------------
# normalisation
_gn_ws = {}


def _gn_workspace(device, n):
    """Partial-statistics scratch of vgen_group_norm, one per (device, stream): two streams of one device must not
    share it (the stats -> finalize -> apply launches of different calls would interleave)."""
    need = int(_l.load().vgen_group_norm_workspace_bytes(n))
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    ws = _gn_ws.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, device=device, dtype=torch.uint8)
        _gn_ws[key] = ws
    return ws


def group_norm(x, gamma, beta, eps, silu, n=None, out=None):
    """x [..., c] fp16 channels-last; statistics per sample over everything but the leading `n` dim.
    x is viewed as [n, p, c]: pass n explicitly when the leading dims are not (n, ...)."""
    _chk16(x, "x")
    if not x.is_contiguous():
        raise _l.VgenError("group_norm: x must be contiguous")
    c = x.shape[-1]
    n = x.shape[0] if n is None else n
    p = x.numel() // (n * c)
    if out is None:
        out = torch.empty_like(x)
    ws = _gn_workspace(x.device, n)
    rc = _run("group_norm", 0.0, 4.0 * x.numel(),
              lambda: _l.load().vgen_group_norm(_p(x), _p(out), n, p, c, _p(gamma), _p(beta), float(eps), 1 if silu else 0,
                                                _p(ws), _stream()),
              tag=f"n{n} p{p} c{c}")
    _l.check(rc, "vgen_group_norm")
    return out


def layer_norm(x, gamma, beta, eps=1e-5, out=None):
    _chk16(x, "x")
    x2, ldx = _rows_view(x, "x")
    rows, c = x2.shape
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    rc = _run("layer_norm", 0.0, 4.0 * rows * c,
              lambda: _l.load().vgen_layer_norm(_p(x2), _p(o2), rows, c, ldx, ldo, _p(gamma), _p(beta), float(eps), _stream()),
              tag=f"rows{rows} c{c}")
    _l.check(rc, "vgen_layer_norm")
    return out


def row_stats(x, eps=1e-5):
    """LayerNorm statistics of the rows of x [rows, c] -> fp32 [rows, 2] = {rstd, -mean * rstd} (for linear(..., ln=...))."""
    _chk16(x, "x")
    x2, ldx = _rows_view(x, "x")
    rows, c = x2.shape
    out = torch.empty(rows, 2, device=x.device, dtype=torch.float32)
    rc = _run("layer_norm", 0.0, 2.0 * rows * c + 8.0 * rows,
              lambda: _l.load().vgen_row_stats(_p(x2), rows, c, ldx, float(eps), _p(out), _stream()), tag=f"stats rows{rows} c{c}")
    _l.check(rc, "vgen_row_stats")
    return out


def fold_layer_norm(w, bias, gamma, beta):
    """Fold a LayerNorm's affine part into the linear that follows it (host-side, once per weight load).

    w [n, k] / bias [n] or None (fp32 masters), gamma / beta [k].  Returns (w' fp16 [n, k] = w * gamma, col_sum fp32 [n] of the
    ROUNDED w', bias' fp32 [n] = bias + w @ beta):  LN(x) w^T + bias = rstd (x w'^T) - mean rstd col_sum + bias'."""
    w32, g, be = w.detach().float(), gamma.detach().float(), beta.detach().float()
    wf = (w32 * g[None, :]).to(torch.float16)
    lb = w32.double() @ be.double()
    if bias is not None:
        lb = lb + bias.detach().double()
    return wf, wf.double().sum(1).float(), lb.float()


# ------------------------------------------------------------------------------------------------
# attention
def attention_d64(q, k, v, heads, kv_batch_div=1, out=None, scale=None):
    """q [b, lq, heads*64] (last-dim-contiguous views allowed, e.g. slices of a fused qkv buffer),
    k/v [b // kv_batch_div, lk, heads*64] -> out [b, lq, heads*64].  scale: the softmax scale (None: 64 ** -0.5)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _chk16(t, nm)
        if t.dim() != 3 or t.stride(2) != 1 or t.stride(0) != t.shape[1] * t.stride(1):
            raise _l.VgenError(f"attention_d64: {nm} must be [b, l, h*64] with dense batch stride")
    b, lq, inner = q.shape
    lk = k.shape[1]
    if inner != heads * 64 or k.shape[2] != inner or v.shape != k.shape or k.shape[0] * kv_batch_div != b:
        raise _l.VgenError("attention_d64: shape mismatch")
    if out is None:
        out = torch.empty(b, lq, inner, device=q.device, dtype=torch.float16)
    rc = _run("attention_d64", 4.0 * b * heads * lq * lk * 64, 2.0 * (2 * b * lq * inner + 2 * k.shape[0] * lk * inner),
              lambda: _l.load().vgen_attention_d64(_p(q), _p(k), _p(v), _p(out), b, heads, lq, lk, q.stride(1), k.stride(1),
                                                   v.stride(1), out.stride(1), kv_batch_div,
                                                   64 ** -0.5 if scale is None else float(scale), _stream()),
              tag=f"b{b} h{heads} lq{lq} lk{lk}")
    _l.check(rc, "vgen_attention_d64")
    return out


def attention_d512(q, k, v, out=None):
    """Single-head flash attention, head_dim 512: q [b, lq, 512], k/v [b, lk, 512] (last-dim-contiguous views allowed,
    e.g. slices of a fused qkv buffer) -> [b, lq, 512]."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _chk16(t, nm)
        if t.dim() != 3 or t.shape[2] != 512 or t.stride(2) != 1 or t.stride(0) != t.shape[1] * t.stride(1):
            raise _l.VgenError(f"attention_d512: {nm} must be [b, l, 512] with dense batch stride")
    b, lq, _ = q.shape
    lk = k.shape[1]
    if k.shape[0] != b or v.shape != k.shape:
        raise _l.VgenError("attention_d512: shape mismatch")
    if out is None:
        out = torch.empty(b, lq, 512, device=q.device, dtype=torch.float16)
    rc = _run("attention_d512", 4.0 * b * lq * lk * 512, 2.0 * (2 * b * lq * 512 + 2 * b * lk * 512),
              lambda: _l.load().vgen_attention_d512(_p(q), _p(k), _p(v), _p(out), b, lq, lk, q.stride(1), k.stride(1), v.stride(1),
                                                    out.stride(1), 512 ** -0.5, _stream()),
              tag=f"b{b} lq{lq} lk{lk}")
    _l.check(rc, "vgen_attention_d512")
    return out


def attention_temporal(q, k, v, heads, head_dim, out=None):
    """q/k/v [f, npix, heads*head_dim] views (frame-major) of one video, or [b, f, npix, heads*head_dim] for b videos back
    to back (one launch): attention over the f tokens of each pixel, for any f and any head_dim <= 64."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _chk16(t, nm)
        if t.dim() not in (3, 4) or t.stride(-1) != 1:
            raise _l.VgenError(f"attention_temporal: {nm} must be [(b,) f, npix, c] with contiguous channels")
    if q.dim() == 3:
        q, k, v = q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0)
        out4 = None if out is None else out.unsqueeze(0)
        squeeze = True
    else:
        out4, squeeze = out, False
    b, f, npix, inner = q.shape
    if inner != heads * head_dim or k.shape != q.shape or v.shape != q.shape:
        raise _l.VgenError("attention_temporal: shape mismatch")
    if k.stride() != q.stride() or v.stride() != q.stride():
        raise _l.VgenError("attention_temporal: q/k/v must share strides")
    if out4 is None:
        out4 = torch.empty(b, f, npix, inner, device=q.device, dtype=torch.float16)
    elif out4.shape != q.shape or out4.stride(-1) != 1:
        raise _l.VgenError("attention_temporal: out must be shaped like q with contiguous channels")
    rc = _run("attention_temporal", 4.0 * b * npix * heads * f * f * head_dim, 2.0 * 4 * b * f * npix * inner,
              lambda: _l.load().vgen_attention_temporal(_p(q), _p(k), _p(v), _p(out4), b * npix, heads, f, head_dim, q.stride(1),
                                                        q.stride(2), out4.stride(1), out4.stride(2), npix, q.stride(0),
                                                        out4.stride(0), head_dim ** -0.5, _stream()))
    _l.check(rc, "vgen_attention_temporal")
    return out4[0] if squeeze else out4


def attention_cross_small(q, k, v, heads, kv_batch_div=1, out=None, causal=False):
    """q [b, lq, heads*d], k/v [b // kv_batch_div, lk, heads*d] for any d <= 256 (tiny problems only); causal: query i
    attends keys 0 .. i + (lk - lq) (the CLIP text tower's mask)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        _chk16(t, nm)
        if t.dim() != 3 or t.stride(2) != 1 or t.stride(0) != t.shape[1] * t.stride(1):
            raise _l.VgenError(f"attention_cross_small: {nm} must be [b, l, h*d] with dense batch stride")
    b, lq, inner = q.shape
    lk = k.shape[1]
    d = inner // heads
    if inner != heads * d or k.shape[2] != inner or v.shape != k.shape or k.shape[0] * kv_batch_div != b:
        raise _l.VgenError("attention_cross_small: shape mismatch")
    if out is None:
        out = torch.empty(b, lq, inner, device=q.device, dtype=torch.float16)
    rc = _l.load().vgen_attention_cross_small(_p(q), _p(k), _p(v), _p(out), b, heads, lq, lk, d, q.stride(1), k.stride(1),
                                              v.stride(1), out.stride(1), kv_batch_div, 1 if causal else 0, d ** -0.5, _stream())
    _l.check(rc, "vgen_attention_cross_small")
    return out


def interp_linear_rows(x, lout):
    """x [nseq, lin, c] fp16 -> [nseq, lout, c] (F.interpolate mode='linear' over the middle axis)."""
    _chk16(x, "x")
    if x.dim() != 3 or not x.is_contiguous():
        raise _l.VgenError("interp_linear_rows: x must be contiguous [nseq, lin, c]")
    nseq, lin, c = x.shape
    y = torch.empty(nseq, lout, c, device=x.device, dtype=torch.float16)
    rc = _l.load().vgen_interp_linear_rows(_p(x), _p(y), nseq, lin, lout, c, _stream())
    _l.check(rc, "vgen_interp_linear_rows")
    return y


def fourier_lowfreq_filter(x, scale, out=None):
    """Fourier_filter(threshold=1) on channels-last x [nimg, h, w, c]; `out` may be a channel slice of a
    wider channels-last buffer."""
    _chk16(x, "x")
    nimg, h, w, c = x.shape
    x2, ldx = _rows_view(x, "x")
    if out is None:
        out = torch.empty(nimg, h, w, c, device=x.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    if o2.shape != x2.shape:
        raise _l.VgenError("fourier_lowfreq_filter: shape mismatch")
    rc = _l.load().vgen_fourier_lowfreq_filter(_p(x2), ldx, _p(o2), ldo, nimg, h, w, c, float(scale), _stream())
    _l.check(rc, "vgen_fourier_lowfreq_filter")
    return out


def scale_copy2d(src, dst, s):
    s2, lds = _rows_view(src, "src")
    d2, ldd = _rows_view(dst, "dst")
    if s2.shape != d2.shape:
        raise _l.VgenError("scale_copy2d: shape mismatch")
    rc = _l.load().vgen_scale_copy2d(_p(s2), lds, _p(d2), ldd, s2.shape[0], s2.shape[1], float(s), _stream())
    _l.check(rc, "vgen_scale_copy2d")
    return dst


def softmax_rows_(x, scale=1.0):
    _chk16(x, "x")
    x2, ld = _rows_view(x, "x")
    rc = _l.load().vgen_softmax_rows(_p(x2), x2.shape[0], x2.shape[1], ld, float(scale), _stream())
    _l.check(rc, "vgen_softmax_rows")
    return x


# ------------------------------------------------------------------------------------------------
# data movement / pointwise
def cp_to_pc(x, n, c, p, c_pad=None):
    """x viewed as [n, c, p] (fp32 or fp16, contiguous) -> [n, p, c_pad] fp16."""
    c_pad = c if c_pad is None else c_pad
    if not x.is_contiguous() or x.dtype not in (torch.float32, torch.float16):
        raise _l.VgenError("cp_to_pc: x must be contiguous fp32/fp16")
    y = torch.empty(n, p, c_pad, device=x.device, dtype=torch.float16)
    rc = _l.load().vgen_cp_to_pc(_p(x), 1 if x.dtype == torch.float32 else 0, _p(y), n, c, p, c_pad, _stream())
    _l.check(rc, "vgen_cp_to_pc")
    return y


def pc_to_cp(x, n, c, p, out_dtype=torch.float16):
    """x [n, p, ld>=c] fp16 -> [n, c, p]."""
    _chk16(x, "x")
    ldx = x.shape[-1]
    y = torch.empty(n, c, p, device=x.device, dtype=out_dtype)
    rc = _l.load().vgen_pc_to_cp(_p(x), ldx, _p(y), 1 if out_dtype == torch.float32 else 0, n, c, p, _stream())
    _l.check(rc, "vgen_pc_to_cp")
    return y


def im2col(x, kh, kw, stride, pad_t, pad_l, ho, wo, kpad, act_silu=False):
    _chk16(x, "x")
    nimg, h, w, c = x.shape
    out = torch.empty(nimg * ho * wo, kpad, device=x.device, dtype=torch.float16)
    rc = _l.load().vgen_im2col(_p(x), _p(out), nimg, h, w, c, kh, kw, stride, pad_t, pad_l, ho, wo, kpad,
                               1 if act_silu else 0, _stream())
    _l.check(rc, "vgen_im2col")
    return out


def upsample_nearest2x(x):
    _chk16(x, "x")
    nimg, h, w, c = x.shape
    y = torch.empty(nimg, 2 * h, 2 * w, c, device=x.device, dtype=torch.float16)
    rc = _l.load().vgen_upsample_nearest2x(_p(x), _p(y), nimg, h, w, c, _stream())
    _l.check(rc, "vgen_upsample_nearest2x")
    return y


def upsample_nearest2x_rows(x, row0, rows_out):
    """nearest x2 upsampling keeping rows [row0, row0+rows_out) (UpsampleSR600 crops one row each side)."""
    _chk16(x, "x")
    nimg, h, w, c = x.shape
    y = torch.empty(nimg, rows_out, 2 * w, c, device=x.device, dtype=torch.float16)
    rc = _l.load().vgen_upsample_nearest2x_rows(_p(x), _p(y), nimg, h, w, c, row0, rows_out, _stream())
    _l.check(rc, "vgen_upsample_nearest2x_rows")
    return y


def copy2d(src, dst):
    """dst[r, :cols] = src[r, :cols] for 2-D row views."""
    s2, lds = _rows_view(src, "src")
    d2, ldd = _rows_view(dst, "dst")
    if s2.shape != d2.shape:
        raise _l.VgenError("copy2d: shape mismatch")
    rc = _l.load().vgen_copy2d(_p(s2), lds, _p(d2), ldd, s2.shape[0], s2.shape[1], _stream())
    _l.check(rc, "vgen_copy2d")
    return dst


def broadcast_row(src, dst):
    """dst[r, :] = src for every row r of the 2-D row view dst (src: a contiguous 1-D tensor of dst's width)."""
    d2, ldd = _rows_view(dst, "dst")
    if src.dim() != 1 or not src.is_contiguous() or src.shape[0] != d2.shape[1] or src.dtype != d2.dtype:
        raise _l.VgenError("broadcast_row: src must be a contiguous row of dst's width and dtype")
    rc = _l.load().vgen_copy2d(_p(src), 0, _p(d2), ldd, d2.shape[0], d2.shape[1], _stream())
    _l.check(rc, "vgen_copy2d")
    return dst


def concat_channels(a, b):
    """torch.cat([a, b], dim=-1) for channels-last tensors with equal leading dims."""
    ca, cb = a.shape[-1], b.shape[-1]
    out = torch.empty(*a.shape[:-1], ca + cb, device=a.device, dtype=torch.float16)
    o2 = out.reshape(-1, ca + cb)
    copy2d(a.reshape(-1, ca), o2[:, :ca])
    copy2d(b.reshape(-1, cb), o2[:, ca:])
    return out


_ELT = {"silu": 0, "add": 1, "gelu": 2, "scale": 3, "axpy": 4, "relu": 5, "quick_gelu": 6}


def eltwise(op, a, b=None, s=1.0, out=None):
    _chk16(a, "a")
    if out is None:
        out = torch.empty_like(a)
    rc = _l.load().vgen_eltwise(_ELT[op], _p(a), _p(b), _p(out), a.numel(), float(s), _stream())
    _l.check(rc, "vgen_eltwise")
    return out



def conv_transpose_stride(x, w, bias, s):
    """nn.ConvTranspose2d(cin, cout, s, stride=s) on channels-last x [nimg, h, w, cin] fp16 -> [nimg, s*h, s*w, cout]:
    one tap-GEMM against w [s*s*cout, cin] (rows (ky, kx, co), pack_conv_transpose_weight) and a scatter that adds the
    fp32 bias [cout]."""
    _chk16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise _l.VgenError("conv_transpose_stride: x must be contiguous [nimg, h, w, cin]")
    nimg, h, wd, cin = x.shape
    cout = w.shape[0] // (s * s)
    if w.shape[0] != s * s * cout or w.shape[1] != cin:
        raise _l.VgenError(f"conv_transpose_stride: weight {tuple(w.shape)} does not match cin={cin}, stride {s}")
    if bias.dtype != torch.float32 or not bias.is_contiguous() or bias.numel() != cout:
        raise _l.VgenError(f"conv_transpose_stride: bias must be contiguous fp32 [{cout}]")
    g = linear(x.view(nimg * h * wd, cin), w)
    out = torch.empty(nimg, s * h, s * wd, cout, device=x.device, dtype=torch.float16)
    rc = _run("dpt_tconv_scatter", 0.0, 4.0 * out.numel(),
              lambda: _l.load().vgen_dpt_tconv_scatter(_p(g), g.stride(0), _p(bias), _p(out), nimg, h, wd, s, cout, _stream()))
    _l.check(rc, "vgen_dpt_tconv_scatter")
    return out


def pack_conv_transpose_weight(w):
    """ConvTranspose2d weight [cin, cout, s, s] -> [s*s*cout, cin] with row (ky*s + kx)*cout + co."""
    cin, cout, kh, kw = w.shape
    return w.detach().permute(2, 3, 1, 0).reshape(kh * kw * cout, cin)


def upsample_bilinear2x(x):
    """F.interpolate(scale_factor=2, mode='bilinear', align_corners=True) on channels-last x [nimg, h, w, c] fp16."""
    _chk16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise _l.VgenError("upsample_bilinear2x: x must be contiguous [nimg, h, w, c]")
    nimg, h, w, c = x.shape
    y = torch.empty(nimg, 2 * h, 2 * w, c, device=x.device, dtype=torch.float16)
    rc = _run("upsample_bilinear", 0.0, 2.0 * (x.numel() + y.numel()),
              lambda: _l.load().vgen_upsample_bilinear2x_ac(_p(x), _p(y), nimg, h, w, c, _stream()))
    _l.check(rc, "vgen_upsample_bilinear2x_ac")
    return y


def dpt_head_out(x, w, bias, out_dtype=torch.float16):
    """relu(relu(x) @ w + bias) per pixel of x [..., c] fp16 (c % 8 == 0), w fp32 [c], bias fp32 [1] -> x.shape[:-1] in
    out_dtype (fp16 or fp32)."""
    _chk16(x, "x")
    x2, ldx = _rows_view(x, "x")
    rows, c = x2.shape
    for t, nm, n in ((w, "w", c), (bias, "bias", 1)):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n or t.device != x.device:
            raise _l.VgenError(f"dpt_head_out: {nm} must be contiguous fp32 [{n}] on {x.device}")
    if out_dtype not in (torch.float16, torch.float32):
        raise _l.VgenError("dpt_head_out: out_dtype must be fp16 or fp32")
    out = torch.empty(x.shape[:-1], device=x.device, dtype=out_dtype)
    rc = _run("dpt_head_out", 2.0 * rows * c, 2.0 * rows * c + out.numel() * out.element_size(),
              lambda: _l.load().vgen_dpt_head_out(_p(x2), ldx, rows, c, _p(w), _p(bias), _p(out),
                                                  1 if out_dtype == torch.float32 else 0, _stream()))
    _l.check(rc, "vgen_dpt_head_out")
    return out

def linear_small(a, w, bias=None, residual=None, silu_in=False, gelu_out=False, out=None):
    _chk16(a, "a"), _chk16(w, "w")
    lead = a.shape[:-1]
    a2, lda = _rows_view(a, "a")
    m, k = a2.shape
    n = w.shape[0]
    if out is None:
        out = torch.empty(*lead, n, device=a.device, dtype=torch.float16)
    o2, ldo = _rows_view(out, "out")
    r2, ldr = (None, 0) if residual is None else _rows_view(residual, "residual")
    rc = _l.load().vgen_linear_small(_p(a2), m, k, lda, _p(w), _p(bias), n, _p(r2), ldr, _p(o2), ldo,
                                     1 if silu_in else 0, 1 if gelu_out else 0, _stream())
    _l.check(rc, "vgen_linear_small")
    return out


def sinusoidal_embedding(t, dim):
    t32 = t.to(torch.float32).contiguous()
    out = torch.empty(t32.numel(), dim, device=t.device, dtype=torch.float16)
    rc = _l.load().vgen_sinusoidal_embedding(_p(t32), _p(out), t32.numel(), dim, _stream())
    _l.check(rc, "vgen_sinusoidal_embedding")
    return out


def adaptive_avgpool(x, oh, ow, silu_in=False):
    _chk16(x, "x")
    nimg, h, w, c = x.shape
    y = torch.empty(nimg, oh, ow, c, device=x.device, dtype=torch.float16)
    rc = _l.load().vgen_adaptive_avgpool(_p(x), _p(y), nimg, h, w, c, oh, ow, 1 if silu_in else 0, _stream())
    _l.check(rc, "vgen_adaptive_avgpool")
    return y


def cond_stem(x, weight, bias, oh, ow):
    """AdaptiveAvgPool_{oh x ow}(SiLU(conv3x3_pad1(x) + bias)) of a pixel-space condition x [b, cin, f, h, w] (fp32 or
    fp16) -> fp16 channels-last [(b f), oh, ow, cout].  weight [cout, cin, 3, 3] and bias [cout] fp32 on x's device."""
    if not x.is_cuda or x.dim() != 5 or not x.is_contiguous() or x.dtype not in (torch.float32, torch.float16):
        raise _l.VgenError("cond_stem: x must be a contiguous CUDA fp32/fp16 tensor [b, cin, f, h, w]")
    b, cin, f, h, w = x.shape
    cout = weight.shape[0]
    if (weight.dtype != torch.float32 or not weight.is_contiguous() or weight.device != x.device
            or tuple(weight.shape) != (cout, cin, 3, 3)):
        raise _l.VgenError(f"cond_stem: weight must be contiguous fp32 [cout, {cin}, 3, 3] on {x.device}")
    if bias.dtype != torch.float32 or not bias.is_contiguous() or bias.device != x.device or tuple(bias.shape) != (cout,):
        raise _l.VgenError(f"cond_stem: bias must be contiguous fp32 [{cout}] on {x.device}")
    y = torch.empty(b * f, oh, ow, cout, device=x.device, dtype=torch.float16)
    rc = _run("cond_stem", 2.0 * b * f * h * w * cout * cin * 9, x.numel() * x.element_size() + y.numel() * 2,
              lambda: _l.load().vgen_cond_stem(_p(x), 1 if x.dtype == torch.float32 else 0, b, cin, f, h, w, _p(weight),
                                               _p(bias), cout, _p(y), oh, ow, _stream()))
    _l.check(rc, "vgen_cond_stem")
    return y


def ddim_step_(xt, y, u, coef7, guide_scale, mean_type_v=True, noise=None, x0_out=None):
    """In-place fused CFG + DDIM update of the fp32 latent xt; y/u fp16 model outputs (same layout).
    x0_out (optional, fp32 like xt) receives the predicted x0 (diffusion_ddim.py:241 returns it)."""
    if xt.dtype != torch.float32 or not xt.is_contiguous() or not xt.is_cuda:
        raise _l.VgenError("ddim_step_: xt must be a contiguous CUDA fp32 tensor")
    _chk16(y, "y")
    if not y.is_contiguous() or y.numel() != xt.numel():
        raise _l.VgenError("ddim_step_: y must be contiguous with xt's element count")
    if u is not None:
        _chk16(u, "u")
        if not u.is_contiguous() or u.numel() != xt.numel():
            raise _l.VgenError("ddim_step_: u must be contiguous with xt's element count")
    if noise is not None and (noise.dtype != torch.float32 or not noise.is_contiguous() or not noise.is_cuda
                              or noise.numel() != xt.numel()):
        raise _l.VgenError("ddim_step_: noise must be a contiguous CUDA fp32 tensor with xt's element count")
    if x0_out is not None and (x0_out.dtype != torch.float32 or not x0_out.is_contiguous() or x0_out.numel() != xt.numel()):
        raise _l.VgenError("ddim_step_: x0_out must be a contiguous fp32 tensor with xt's element count")
    c = (ctypes.c_float * 7)(*[float(v) for v in coef7])
    rc = _l.load().vgen_ddim_step(_p(xt), _p(y), _p(u), _p(noise), xt.numel(), float(guide_scale or 0.0), c,
                                  1 if mean_type_v else 0, _p(x0_out), _stream())
    _l.check(rc, "vgen_ddim_step")
    return xt


def cfg_combine(y, u, guide_scale):
    """out = u + g*(y-u) (fp16) and the fp64 per-sample sums needed by the std-ratio guidance rescale."""
    _chk16(y, "y"), _chk16(u, "u")
    if y.shape != u.shape or not y.is_contiguous() or not u.is_contiguous():
        raise _l.VgenError("cfg_combine: y/u must be contiguous and equally shaped")
    b = y.shape[0]
    out = torch.empty_like(y)
    stats = torch.empty(b, 4, device=y.device, dtype=torch.float64)
    rc = _l.load().vgen_cfg_combine(_p(y), _p(u), _p(out), b, y.numel() // b, float(guide_scale), _p(stats), _stream())
    _l.check(rc, "vgen_cfg_combine")
    return out, stats


def gauss_x0(xt, out, alpha, sigma, prediction_type, stats=None, guide_rescale=0.0):
    """x0 prediction of GaussianDiffusion.denoise from the fp32 latent and the fp16 model output."""
    _chk16(out, "out")
    if xt.dtype != torch.float32 or not xt.is_contiguous() or not out.is_contiguous() or xt.shape != out.shape:
        raise _l.VgenError("gauss_x0: xt must be contiguous fp32 and shaped like out")
    b = xt.shape[0]
    x0 = torch.empty_like(xt)
    rc = _l.load().vgen_gauss_x0(_p(xt), _p(out), _p(stats), float(guide_rescale), float(alpha), float(sigma),
                                 {"x0": 0, "eps": 1, "v": 2}[prediction_type], _p(x0), b, xt.numel() // b, _stream())
    _l.check(rc, "vgen_gauss_x0")
    return x0


def lincomb_f32(terms, out=None):
    """out = sum_i a_i * x_i over up to four (a_i, x_i) fp32 terms."""
    if not 1 <= len(terms) <= 4:
        raise _l.VgenError("lincomb_f32: 1..4 terms")
    x0 = terms[0][1]
    for a, x in terms:
        if x.dtype != torch.float32 or not x.is_contiguous() or x.shape != x0.shape or not x.is_cuda:
            raise _l.VgenError("lincomb_f32: terms must be contiguous CUDA fp32 tensors of one shape")
    if out is None:
        out = torch.empty_like(x0)
    args = []
    for i in range(4):
        a, x = terms[i] if i < len(terms) else (0.0, None)
        args += [_p(x), float(a)]
    rc = _l.load().vgen_lincomb_f32(_p(out), x0.numel(), *args, _stream())
    _l.check(rc, "vgen_lincomb_f32")
    return out


def vae_sample(moments, noise, scale):
    """moments fp16 [n, p, 2*zc] (mean | logvar), noise fp32 [n, zc, p] -> fp32 z [n, zc, p]."""
    _chk16(moments, "moments")
    n, p, c2 = moments.shape
    zc = c2 // 2
    if noise.dtype != torch.float32 or not noise.is_contiguous() or noise.numel() != n * zc * p:
        raise _l.VgenError("vae_sample: noise must be contiguous fp32 [n, zc, p]")
    z = torch.empty(n, zc, p, device=moments.device, dtype=torch.float32)
    rc = _l.load().vgen_vae_sample(_p(moments), _p(noise), _p(z), n, zc, p, float(scale), _stream())
    _l.check(rc, "vgen_vae_sample")
    return z


def video_to_rgb8(video, mean, std, want_band=True):
    """video fp32 [3, f, h, w] (one batch entry, contiguous, CUDA) -> (uint8 [f, h, w, 3], per-frame count of bytes in
    [117, 137] or None).  mean / std: 3 floats each (cfg.mean / cfg.std)."""
    if video.dtype != torch.float32 or not video.is_cuda or not video.is_contiguous() or video.dim() != 4 or video.shape[0] != 3:
        raise _l.VgenError("video_to_rgb8: video must be a contiguous CUDA fp32 tensor [3, f, h, w]")
    c, f, h, w = video.shape
    out = torch.empty(f, h, w, 3, device=video.device, dtype=torch.uint8)
    band = torch.empty(f, device=video.device, dtype=torch.int64) if want_band else None
    m3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in std])
    rc = _run("video_out", 0.0, 5.0 * video.numel(),
              lambda: _l.load().vgen_video_to_rgb8(_p(video), c, f, h, w, m3, s3, _p(out), _p(band), _stream()))
    _l.check(rc, "vgen_video_to_rgb8")
    return out, band


def embed_tokens(ids, table, pos):
    """ids int64 [b, L] (CUDA), table fp32 [vocab, W], pos fp32 [L, W] -> fp16 [b, L, W] = table[ids] + pos."""
    if ids.dtype != torch.int64 or not ids.is_cuda or not ids.is_contiguous() or ids.dim() != 2:
        raise _l.VgenError("embed_tokens: ids must be a contiguous CUDA int64 tensor [b, L]")
    for t, nm in ((table, "table"), (pos, "pos")):
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
            raise _l.VgenError(f"embed_tokens: {nm} must be a contiguous CUDA fp32 tensor")
    b, L = ids.shape
    vocab, W = table.shape
    if pos.shape != (L, W):
        raise _l.VgenError("embed_tokens: pos must be [L, W]")
    out = torch.empty(b, L, W, device=ids.device, dtype=torch.float16)
    rc = _l.load().vgen_embed_tokens(_p(ids), _p(table), _p(pos), _p(out), b * L, L, W, vocab, _stream())
    _l.check(rc, "vgen_embed_tokens")
    return out


def check_token_ids(ids, n_rows):
    """Raise unless every id is in [0, n_rows): one small device-to-host read of (min, max)."""
    if ids.numel():
        lo, hi = (int(v) for v in torch.aminmax(ids))
        if lo < 0 or hi >= n_rows:
            raise _l.VgenError(f"embed_tokens: token ids span [{lo}, {hi}], outside the {n_rows} rows of the vocabulary "
                               "plus the learned embeddings")


def embed_tokens_extra(ids, table, extra, pos, check=True):
    """embed_tokens with learned rows: an id >= vocab reads extra[id - vocab] (fp32 [n_extra, W]; None = no extra rows).
    An id outside [0, vocab + n_extra) is an error, not a clamp: the ids are checked on the host before the launch.
    check=False is for a caller that has already checked them (CUDA-graph capture cannot read them back)."""
    if ids.dtype != torch.int64 or not ids.is_cuda or not ids.is_contiguous() or ids.dim() != 2:
        raise _l.VgenError("embed_tokens: ids must be a contiguous CUDA int64 tensor [b, L]")
    for t, nm in ((table, "table"), (pos, "pos")) + (() if extra is None else ((extra, "extra"),)):
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
            raise _l.VgenError(f"embed_tokens: {nm} must be a contiguous CUDA fp32 tensor")
    b, L = ids.shape
    vocab, W = table.shape
    n_extra = 0 if extra is None else extra.shape[0]
    if pos.shape != (L, W) or (extra is not None and (extra.dim() != 2 or extra.shape[1] != W)):
        raise _l.VgenError("embed_tokens: pos must be [L, W] and extra [n_extra, W]")
    if check:
        check_token_ids(ids, vocab + n_extra)
    out = torch.empty(b, L, W, device=ids.device, dtype=torch.float16)
    rc = _l.load().vgen_embed_tokens_extra(_p(ids), _p(table), vocab, _p(extra), n_extra, _p(pos), _p(out), b * L, L, W,
                                           _stream())
    _l.check(rc, "vgen_embed_tokens_extra")
    return out


def add_rows_f32_(x, add):
    """x fp16 [b, ...] += add fp32 [...] broadcast over the leading dim, in place."""
    _chk16(x, "x")
    if not x.is_contiguous() or add.dtype != torch.float32 or not add.is_contiguous() or add.numel() * x.shape[0] != x.numel():
        raise _l.VgenError("add_rows_f32_: x must be contiguous fp16 [b, n...] and add contiguous fp32 [n...]")
    rc = _l.load().vgen_add_rows_f32(_p(x), _p(add), x.shape[0], add.numel(), _stream())
    _l.check(rc, "vgen_add_rows_f32")
    return x


# ------------------------------------------------------------------------------------------------
# sketch annotators (sketch.cu, and the tap-GEMM's arbitrary-tap entry)
def conv2d_taps(x, w, taps, bias=None, relu=False, out=None, out_stride_y=None, out_stride_x=None):
    """out[b, y, x, :] = epi(sum_t x[b, y + dy_t, x + dx_t, :] @ w[:, t*c:(t+1)*c]^T) with zero padding, for channels-last
    x [nimg, h, w, c] fp16 and taps [(dy, dx), ...] (1..33).  relu: relu(acc + bias) in fp32.  With out given, output
    pixel (b, y, x) lands at element b*h*out_stride_y + y*out_stride_y + x*out_stride_x of out (a strided sub-grid, which
    goes with relu=True)."""
    _chk16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise _l.VgenError("conv2d_taps: x must be contiguous [nimg, h, w, c]")
    nimg, h, wd, c = x.shape
    nt, n = len(taps), w.shape[0]
    if w.shape[1] != nt * c:
        raise _l.VgenError(f"conv2d_taps: weight {tuple(w.shape)} does not match {nt} taps x c={c}")
    if out is None:
        out = torch.empty(nimg, h, wd, n, device=x.device, dtype=torch.float16)
        out_stride_y, out_stride_x = wd * n, n
    e, keep = _epilogue(n, bias=bias)
    dy = (ctypes.c_int32 * nt)(*[int(t[0]) for t in taps])
    dx = (ctypes.c_int32 * nt)(*[int(t[1]) for t in taps])
    rc = _run("conv_taps", 2.0 * nimg * h * wd * n * nt * c, 2.0 * (x.numel() + w.numel() + nimg * h * wd * n),
              lambda: _l.load().vgen_conv2d_taps(_p(x), nimg, h, wd, c, nt, dy, dx, _p(w), n, _p(out), int(out_stride_y),
                                                 int(out_stride_x), ctypes.byref(e), 1 if relu else 0, _stream()),
              tag=f"taps{nt} c{c} n{n}")
    _l.check(rc, "vgen_conv2d_taps")
    return out


def _chk32(t, name, n, dev):
    if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n or t.device != dev:
        raise _l.VgenError(f"{name} must be contiguous fp32 [{n}] on {dev}")


def dwconv_relu(x, w, k, pool=False):
    """relu(depthwise k x k conv) of channels-last x [nimg, h, w, c] fp16 (c % 64 == 0), w fp32 [k*k, c]; with pool the
    conv runs on the floored 2x2 max-pool of x.  -> (out, pooled or None)."""
    _chk16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise _l.VgenError("dwconv_relu: x must be contiguous [nimg, h, w, c]")
    nimg, h, wd, c = x.shape
    _chk32(w, "dwconv_relu: w", k * k * c, x.device)
    ho, wo = (h // 2, wd // 2) if pool else (h, wd)
    out = torch.empty(nimg, ho, wo, c, device=x.device, dtype=torch.float16)
    pooled = torch.empty_like(out) if pool else None
    rc = _run("dwconv", 2.0 * out.numel() * k * k, 2.0 * (x.numel() + out.numel() * (2 if pool else 1)),
              lambda: _l.load().vgen_dwconv_relu(_p(x), nimg, h, wd, c, k, _p(w), 1 if pool else 0, _p(pooled), _p(out),
                                                 _stream()))
    _l.check(rc, "vgen_dwconv_relu")
    return out, pooled


def csam_mapreduce(x, w1, b1, w2, wm, bm):
    """MapReduce(CSAM(x)) of channels-last x [nimg, h, w, c] fp16: w1 fp32 [4, c], b1 [4], w2 [4, 3, 3], wm [c], bm [1]
    -> fp32 [nimg, h, w]."""
    _chk16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise _l.VgenError("csam_mapreduce: x must be contiguous [nimg, h, w, c]")
    nimg, h, wd, c = x.shape
    for t, nm, n in ((w1, "w1", 4 * c), (b1, "b1", 4), (w2, "w2", 36), (wm, "wm", c), (bm, "bm", 1)):
        _chk32(t, f"csam_mapreduce: {nm}", n, x.device)
    t_ws = torch.empty(nimg * h * wd, 4, device=x.device, dtype=torch.float32)
    s_ws = torch.empty(nimg * h * wd, device=x.device, dtype=torch.float32)
    e = torch.empty(nimg, h, wd, device=x.device, dtype=torch.float32)
    rc = _run("csam", 12.0 * x.numel(), 2.0 * x.numel() + 40.0 * e.numel(),
              lambda: _l.load().vgen_csam_mapreduce(_p(x), nimg, h, wd, c, _p(w1), _p(b1), _p(w2), _p(wm), _p(bm), _p(t_ws),
                                                    _p(s_ws), _p(e), _stream()))
    _l.check(rc, "vgen_csam_mapreduce")
    return e


def pidinet_fuse(es, cw, H, W, out_dtype=torch.float16):
    """sigmoid(cw[:4] . bilinear_resize(es, (H, W)) + cw[4]) for four fp32 side maps [nimg, h_i, w_i] -> [nimg, 1, H, W]."""
    nimg = es[0].shape[0]
    for e in es:
        if e.dtype != torch.float32 or e.dim() != 3 or not e.is_contiguous() or e.shape[0] != nimg or e.device != es[0].device:
            raise _l.VgenError("pidinet_fuse: side maps must be contiguous fp32 [nimg, h, w] on one device")
    _chk32(cw, "pidinet_fuse: cw", 5, es[0].device)
    if out_dtype not in (torch.float16, torch.float32):
        raise _l.VgenError("pidinet_fuse: out_dtype must be fp16 or fp32")
    out = torch.empty(nimg, 1, H, W, device=es[0].device, dtype=out_dtype)
    hw = (ctypes.c_int64 * 8)(*[int(d) for e in es for d in e.shape[1:]])
    rc = _run("pidinet_fuse", 40.0 * out.numel(), 16.0 * out.numel() + out.numel() * out.element_size(),
              lambda: _l.load().vgen_pidinet_fuse(_p(es[0]), _p(es[1]), _p(es[2]), _p(es[3]), hw, nimg, H, W, _p(cw), _p(out),
                                                  1 if out_dtype == torch.float32 else 0, _stream()))
    _l.check(rc, "vgen_pidinet_fuse")
    return out


def conv3x3_to1_sigmoid(x, w, bias, out_dtype=torch.float16):
    """sigmoid(3x3 conv to one channel + bias) of channels-last x [nimg, h, w, c] fp16; w fp32 [9, c], bias fp32 [1]
    -> [nimg, 1, h, w] in out_dtype."""
    _chk16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise _l.VgenError("conv3x3_to1_sigmoid: x must be contiguous [nimg, h, w, c]")
    nimg, h, wd, c = x.shape
    _chk32(w, "conv3x3_to1_sigmoid: w", 9 * c, x.device)
    _chk32(bias, "conv3x3_to1_sigmoid: bias", 1, x.device)
    if out_dtype not in (torch.float16, torch.float32):
        raise _l.VgenError("conv3x3_to1_sigmoid: out_dtype must be fp16 or fp32")
    out = torch.empty(nimg, 1, h, wd, device=x.device, dtype=out_dtype)
    rc = _run("conv3x3_to1", 18.0 * x.numel(), 2.0 * x.numel() + out.numel() * out.element_size(),
              lambda: _l.load().vgen_conv3x3_to1_sigmoid(_p(x), nimg, h, wd, c, _p(w), _p(bias), _p(out),
                                                         1 if out_dtype == torch.float32 else 0, _stream()))
    _l.check(rc, "vgen_conv3x3_to1_sigmoid")
    return out


def sketch_normalize(x, mean, std):
    """fp16((x - mean) / std) of a contiguous fp32 / fp16 CUDA tensor, same shape."""
    if not x.is_cuda or not x.is_contiguous() or x.dtype not in (torch.float32, torch.float16):
        raise _l.VgenError("sketch_normalize: x must be a contiguous fp32 / fp16 CUDA tensor")
    y = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    rc = _l.load().vgen_sketch_normalize(_p(x), 1 if x.dtype == torch.float32 else 0, x.numel(), float(mean), float(std),
                                         _p(y), _stream())
    _l.check(rc, "vgen_sketch_normalize")
    return y


# ------------------------------------------------------------------------------------------------
# DreamVideo's evaluation metric (metric.cu)
def resize_crop_normalize(images, plan, out_f32=False, out=None):
    """Pillow-exact bicubic resize + centre crop + normalisation of uint8 images [n, h, w, 3] (contiguous, CUDA) with the
    fixed-point tables of `plan` (metric.ResizePlan, moved to the images' device) -> fp16 [n, crop_h, crop_w, 3] or, with
    out_f32, fp32 [n, 3, crop_h, crop_w]; `out` (contiguous, that shape and dtype) receives it if given."""
    if images.dtype != torch.uint8 or not images.is_cuda or not images.is_contiguous() or images.dim() != 4 or images.shape[3] != 3:
        raise _l.VgenError("resize_crop_normalize: images must be a contiguous CUDA uint8 tensor [n, h, w, 3]")
    n, h, w, _ = images.shape
    if (h, w) != (plan.h, plan.w):
        raise _l.VgenError(f"resize_crop_normalize: the plan is for {plan.h}x{plan.w} images, got {h}x{w}")
    hb, hk, vb, vk = plan.tables(images.device)
    ch, cw = plan.crop_h, plan.crop_w
    shape, dtype = ((n, 3, ch, cw), torch.float32) if out_f32 else ((n, ch, cw, 3), torch.float16)
    if out is None:
        out = torch.empty(shape, device=images.device, dtype=dtype)
    elif tuple(out.shape) != shape or out.dtype != dtype or not out.is_contiguous() or out.device != images.device:
        raise _l.VgenError(f"resize_crop_normalize: out must be a contiguous {dtype} tensor {list(shape)} on {images.device}")
    m3 = (ctypes.c_float * 3)(*[float(v) for v in plan.mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in plan.std])
    rc = _run("resize_crop_norm", 0.0, images.numel() + out.numel() * out.element_size(),
              lambda: _l.load().vgen_resize_bicubic_crop_normalize(_p(images), n, h, w, _p(hb), _p(hk), hk.shape[1], _p(vb),
                                                                   _p(vk), vk.shape[1], ch, cw, plan.tile_rows, m3, s3,
                                                                   _p(out), 1 if out_f32 else 0, _stream()))
    _l.check(rc, "vgen_resize_bicubic_crop_normalize")
    return out


def video_scores(clip_frames, text, clip_targets, dino_frames, dino_targets):
    """(CLIP-T, CLIP-I, DINO-I, temporal consistency) of one video as a CUDA fp32 [4] tensor, from fp32 features
    clip_frames [f, e], text [e], dino_frames [f, d] and the targets' [t, e] / [t, d] (None or t = 0: no targets)."""
    f, e = clip_frames.shape
    d = dino_frames.shape[1]
    t = 0 if clip_targets is None else clip_targets.shape[0]
    ts = [(clip_frames, "clip_frames", (f, e)), (text, "text", (e,)), (dino_frames, "dino_frames", (f, d))]
    if t:
        ts += [(clip_targets, "clip_targets", (t, e)), (dino_targets, "dino_targets", (t, d))]
    for x, nm, shape in ts:
        if x.dtype != torch.float32 or not x.is_cuda or not x.is_contiguous() or tuple(x.shape) != shape:
            raise _l.VgenError(f"video_scores: {nm} must be a contiguous CUDA fp32 tensor {list(shape)}")
    out = torch.empty(4, device=clip_frames.device, dtype=torch.float32)
    rc = _l.load().vgen_video_scores(_p(clip_frames), f, e, _p(text), _p(clip_targets) if t else None, t, _p(dino_frames),
                                     _p(dino_targets) if t else None, d, _p(out), _stream())
    _l.check(rc, "vgen_video_scores")
    return out


# ------------------------------------------------------------------------------------------------
# InstructVideo's segmental video reward (reward.cu)
def reward_frames(src, frame_idx, plan, out_f32=False, out=None):
    """The reward's image-tower input of the frames frame_idx (int32 CUDA [n], flat frame numbers v * f + t) of src:
    fp32 decoder output [b, 3, f, H, W] or [n, 3, H, W] (any element strides; x * 0.5 + 0.5) or uint8 RGB [n, H, W, 3]
    (x / 255); clamp(0, 1), the bilinear resize of `plan` (reward.BilinearPlan) and its normalisation -> fp16
    [n, oh, ow, 3] or, with out_f32, fp32 [n, 3, oh, ow] (into `out` if given)."""
    if not src.is_cuda or src.dtype not in (torch.float32, torch.uint8):
        raise _l.VgenError("reward_frames: src must be a CUDA fp32 or uint8 tensor")
    if src.dtype == torch.uint8:
        if src.dim() != 4 or src.shape[3] != 3:
            raise _l.VgenError(f"reward_frames: uint8 frames must be [n, H, W, 3], got {tuple(src.shape)}")
        nsrc, fp, (h, w) = src.shape[0], 1, src.shape[1:3]
        sv, sf, sc, sy, sx = src.stride(0), 0, src.stride(3), src.stride(1), src.stride(2)
    elif src.dim() == 5 and src.shape[1] == 3:
        nsrc, fp, (h, w) = src.shape[0] * src.shape[2], src.shape[2], src.shape[3:]
        sv, sc, sf, sy, sx = src.stride()
    elif src.dim() == 4 and src.shape[1] == 3:
        nsrc, fp, (h, w) = src.shape[0], 1, src.shape[2:]
        sv, sc, sy, sx = src.stride()
        sf = 0
    else:
        raise _l.VgenError(f"reward_frames: fp32 frames must be [b, 3, f, H, W] or [n, 3, H, W], got {tuple(src.shape)}")
    if (h, w) != (plan.h, plan.w):
        raise _l.VgenError(f"reward_frames: the plan is for {plan.h}x{plan.w} frames, got {h}x{w}")
    if (frame_idx.dtype != torch.int32 or not frame_idx.is_contiguous() or frame_idx.dim() != 1
            or frame_idx.device != src.device):
        raise _l.VgenError(f"reward_frames: frame_idx must be a contiguous int32 [n] tensor on {src.device}")
    n = frame_idx.shape[0]
    hb, hk, vb, vk = plan.tables(src.device)
    oh, ow = plan.oh, plan.ow
    shape, dtype = ((n, 3, oh, ow), torch.float32) if out_f32 else ((n, oh, ow, 3), torch.float16)
    if out is None:
        out = torch.empty(shape, device=src.device, dtype=dtype)
    elif tuple(out.shape) != shape or out.dtype != dtype or not out.is_contiguous() or out.device != src.device:
        raise _l.VgenError(f"reward_frames: out must be a contiguous {dtype} tensor {list(shape)} on {src.device}")
    m3 = (ctypes.c_float * 3)(*[float(v) for v in plan.mean])
    s3 = (ctypes.c_float * 3)(*[float(v) for v in plan.std])
    rc = _run("reward_frames", 0.0, n * 3 * h * w * src.element_size() + out.numel() * out.element_size(),
              lambda: _l.load().vgen_reward_frames(_p(src), 1 if src.dtype == torch.uint8 else 0, _p(frame_idx), n, fp, sv,
                                                   sf, sc, sy, sx, h, w, _p(hb), _p(hk), hk.shape[1], _p(vb), _p(vk),
                                                   vk.shape[1], oh, ow, plan.tile_rows, m3, s3, _p(out),
                                                   1 if out_f32 else 0, _stream()))
    _l.check(rc, "vgen_reward_frames")
    return out


def segment_reward(image_features, text_features, frame_idx, f, tar, lambda_tar):
    """reward_scores fp32 [b] from fp32 image_features [b * s, e] (video-major), text_features [b, e] and the segments'
    frame indices frame_idx (int32 [b, s] on the device; read only with tar) of f-frame videos."""
    b, e = text_features.shape
    s = image_features.shape[0] // max(b, 1)
    for x, nm, shape in ((image_features, "image_features", (b * s, e)), (text_features, "text_features", (b, e))):
        if x.dtype != torch.float32 or not x.is_cuda or not x.is_contiguous() or tuple(x.shape) != shape:
            raise _l.VgenError(f"segment_reward: {nm} must be a contiguous CUDA fp32 tensor {list(shape)}")
    if (frame_idx.dtype != torch.int32 or not frame_idx.is_contiguous() or tuple(frame_idx.shape) != (b, s)
            or frame_idx.device != text_features.device):
        raise _l.VgenError(f"segment_reward: frame_idx must be a contiguous int32 tensor [{b}, {s}] on {text_features.device}")
    out = torch.empty(b, device=text_features.device, dtype=torch.float32)
    rc = _run("segment_reward", 6.0 * b * s * e, 4.0 * (b * s * e + b * e),
              lambda: _l.load().vgen_segment_reward(_p(image_features), _p(text_features), _p(frame_idx), b, s, e, int(f),
                                                    1 if tar else 0, float(lambda_tar), _p(out), _stream()))
    _l.check(rc, "vgen_segment_reward")
    return out


# ------------------------------------------------------------------------------------------------
# the VideoComposer canny annotator (canny.cu)
def canny(frames, mode, rand=None, low=0.0, high=0.0, out=None, thresholds=False):
    """cv2.Canny edge maps (aperture 3, L1 gradient) of frames [n, c, h, w] (any element strides, c = 1 or 3): CUDA fp32
    in [0, 1], quantised as convertScaleAbs(x * 255), or uint8.  Thresholds from each frame's median: mode 0 (low,
    high) as given, mode 1 (1 -/+ 0.33) * median, mode 2 (1 - rand[i]) * median and twice that (rand: CUDA fp64 [n]).
    Returns fp32 [n, h, w] of 0.0 / 1.0 (into `out`, any contiguous tensor of n * h * w fp32, if given) and, with
    thresholds, also the int32 [n, 2] (low, high) the magnitudes were compared with."""
    if not frames.is_cuda or frames.dtype not in (torch.float32, torch.uint8):
        raise _l.VgenError(f"canny: frames must be a CUDA fp32 or uint8 tensor, got {frames.dtype} on {frames.device}")
    if frames.dim() != 4 or frames.shape[1] not in (1, 3) or frames.shape[2] == 0 or frames.shape[3] == 0:
        raise _l.VgenError(f"canny: frames must be [n, c, h, w] with c = 1 or 3, got {tuple(frames.shape)}")
    n, c, h, w = frames.shape
    dev = frames.device
    if mode == 2:
        if (rand is None or rand.dtype != torch.float64 or rand.device != dev or not rand.is_contiguous()
                or tuple(rand.shape) != (n,)):
            raise _l.VgenError(f"canny: rand must be a contiguous fp64 tensor [{n}] on {dev}")
    elif mode not in (0, 1):
        raise _l.VgenError(f"canny: mode must be 0, 1 or 2, got {mode}")
    if out is None:
        out = torch.empty(n, h, w, device=dev, dtype=torch.float32)
    elif out.numel() != n * h * w or out.dtype != torch.float32 or not out.is_contiguous() or out.device != dev:
        raise _l.VgenError(f"canny: out must be a contiguous fp32 tensor of {n * h * w} elements on {dev}")
    u8 = lambda *s: torch.empty(s, device=dev, dtype=torch.uint8)  # noqa: E731
    i32 = lambda *s: torch.empty(s, device=dev, dtype=torch.int32)  # noqa: E731
    bytes_, hist, thr, cls, label, keep = u8(n, c, h, w), i32(n, 256), i32(n, 2), u8(n, h, w), i32(n, h, w), u8(n, h, w)
    s_n, s_c, s_y, s_x = frames.stride()
    px = n * h * w
    rc = _run("canny", 0.0, n * c * h * w * (frames.element_size() + 2) + px * 16,
              lambda: _l.load().vgen_canny(_p(frames), 1 if frames.dtype == torch.uint8 else 0, n, c, h, w, s_n, s_c, s_y,
                                           s_x, mode, _p(rand) if mode == 2 else None, float(low), float(high),
                                           _p(bytes_), _p(hist), _p(thr), _p(cls), _p(label), _p(keep), _p(out),
                                           _stream()))
    _l.check(rc, "vgen_canny")
    return (out, thr) if thresholds else out


# ------------------------------------------------------------------------------------------------
# the VideoComposer colour-palette annotator (palette.cu)
_PAL_KIND = {torch.float32: 0, torch.uint8: 1, torch.float64: 2}


def _palette_src(frames, name, lab4, lin):
    if not frames.is_cuda or frames.dtype not in _PAL_KIND:
        raise _l.VgenError(f"{name}: frames must be a CUDA fp32, fp64 or uint8 tensor, got {frames.dtype} on {frames.device}")
    if frames.dim() != 4 or frames.shape[1] != 3 or frames.shape[2] == 0 or frames.shape[3] == 0:
        raise _l.VgenError(f"{name}: frames must be [n, 3, h, w] (any strides), got {tuple(frames.shape)}")
    dev = frames.device
    npal = lab4.shape[0] if lab4.dim() == 2 else -1
    if lab4.dtype != torch.float64 or lab4.device != dev or not lab4.is_contiguous() or lab4.shape[-1] != 4 \
            or not 1 <= npal <= 156:
        raise _l.VgenError(f"{name}: the palette table must be a contiguous fp64 [npal, 4] tensor on {dev} with 1 to 156 "
                           f"entries (the UNet's hist_dim), got {tuple(lab4.shape)}")
    if frames.dtype == torch.uint8 and (lin is None or lin.dtype != torch.float64 or lin.device != dev
                                        or tuple(lin.shape) != (256,) or not lin.is_contiguous()):
        raise _l.VgenError(f"{name}: uint8 frames need the contiguous fp64 [256] linearisation table on {dev}")
    return _PAL_KIND[frames.dtype], npal


def palette_histogram(frames, lab4, lin=None, weight=None, out_dtype=torch.float32):
    """Palette.histogram of frames [n, 3, h, w] (any element strides; CUDA fp32 / fp64 in [0, 1], or uint8) against the
    palette lab4 (fp64 [npal, 4]: L, a, b, |Lab|^2; npal <= 156) -> [n, npal] of out_dtype (fp32 or fp64).  lin: the
    uint8 linearisation table (fp64 [256]); weight: the row-normalised smoothing matrix (fp64 [npal, npal]) or None
    (sigma <= 0: the plain normalised counts, no zeroing)."""
    kind, npal = _palette_src(frames, "palette_histogram", lab4, lin)
    dev = frames.device
    if weight is not None and (weight.dtype != torch.float64 or weight.device != dev or not weight.is_contiguous()
                               or tuple(weight.shape) != (npal, npal)):
        raise _l.VgenError(f"palette_histogram: weight must be a contiguous fp64 [{npal}, {npal}] tensor on {dev}")
    if out_dtype not in (torch.float32, torch.float64):
        raise _l.VgenError(f"palette_histogram: out_dtype must be fp32 or fp64, got {out_dtype}")
    n, _, h, w = frames.shape
    counts = torch.empty(n, npal, device=dev, dtype=torch.int32)
    out = torch.empty(n, npal, device=dev, dtype=out_dtype)
    s_n, s_c, s_y, s_x = frames.stride()
    rc = _run("palette", 1250.0 * n * h * w, n * h * w * 3 * frames.element_size(),
              lambda: _l.load().vgen_palette_histogram(_p(frames), kind, n, h, w, s_n, s_c, s_y, s_x, _p(lab4), npal,
                                                       _p(lin) if kind == 1 else None, _p(weight), _p(counts), _p(out),
                                                       1 if out_dtype == torch.float64 else 0, _stream()))
    _l.check(rc, "vgen_palette_histogram")
    return out


def palette_quantize(frames, lab4, qrgb, lin=None):
    """Palette.quantize_image of frames [n, 3, h, w] (as palette_histogram) -> fp64 [n, h, w, 3]: qrgb[k] (fp64 [npal, 3],
    lab2rgb of each palette entry) of each pixel's nearest entry k."""
    kind, npal = _palette_src(frames, "palette_quantize", lab4, lin)
    dev = frames.device
    if qrgb.dtype != torch.float64 or qrgb.device != dev or not qrgb.is_contiguous() or tuple(qrgb.shape) != (npal, 3):
        raise _l.VgenError(f"palette_quantize: qrgb must be a contiguous fp64 [{npal}, 3] tensor on {dev}")
    n, _, h, w = frames.shape
    out = torch.empty(n, h, w, 3, device=dev, dtype=torch.float64)
    s_n, s_c, s_y, s_x = frames.stride()
    rc = _run("palette", 1250.0 * n * h * w, n * h * w * (3 * frames.element_size() + 24),
              lambda: _l.load().vgen_palette_quantize(_p(frames), kind, n, h, w, s_n, s_c, s_y, s_x, _p(lab4), npal,
                                                      _p(lin) if kind == 1 else None, _p(qrgb), _p(out), _stream()))
    _l.check(rc, "vgen_palette_quantize")
    return out
