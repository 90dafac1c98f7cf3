"""Every instantiation of the tap-GEMM kernel (`tapgemm_sm90_kernel<BN, kEpi>`, tapgemm_sm90.cu), with its N tile forced
(ops.set_tapgemm_bn), against the float64 reference of tests/_tapgemm_ref.py under its per-element bound.

Per (BN, kind): the epilogue's store paths (TMA tile stores; direct scalar stores for an unaligned output or bias, a
partial chunk or out_n < 32; direct vector stores, which only a strided kind-8 output reaches: see _padded_rows_case),
tiles whose N block ends early, rows m = 1 ... 129, more
than three tiles per persistent CTA (the staging-slot parity carries across tiles), K from one k-iteration to 5120,
a row-strided A; for the conv kinds (0, 8) the box geometries pick_box chooses, 33 taps, taps that only read padding,
the temporal conv over several videos and the strided output of a transposed-conv phase; the epilogue fields (per-frame
bias shared by a video's frames, strided residual / bias / row bias, alpha).  Outputs written as a slice of a wider
buffer leave the other columns bit-identical.  Host-side refusals launch nothing."""
import ctypes
import math
import zlib

import pytest
import torch

import _tapgemm_ref as R
from vgen_b200 import lib, ops
from vgen_b200.lib import VgenError

pytestmark = pytest.mark.gpu

ALL_BN = (32, 64, 96, 128, 160, 192, 224, 256)
# kEpi -> the N tiles launch_bn instantiates it for (tapgemm_sm90.cu)
KERNELS = {
    0: ALL_BN,                  # plain / bias / per-frame bias / residual
    1: (64, 128, 192, 256),     # GEGLU
    2: ALL_BN,                  # folded LayerNorm
    3: (64, 128, 192, 256),     # folded LayerNorm + GEGLU
    4: ALL_BN[:-1],             # GELU + fp32 row bias (adapter down projection)
    8: ALL_BN,                  # ReLU, optional strided output
}
PAIRS = [(bn, kind) for kind, bns in KERNELS.items() for bn in bns]
SENTINEL = -777.0
WORST = {}   # kind -> largest error / bound seen


def test_matrix_lists_every_instantiation():
    assert len(PAIRS) == 39 and len(set(PAIRS)) == 39


@pytest.fixture
def forced_bn(request):
    bn = request.param if hasattr(request, "param") else 0
    ops.set_tapgemm_impl("auto")
    ops.set_tapgemm_bn(bn)
    yield bn
    ops.set_tapgemm_bn(0)
    ops.set_tapgemm_impl("auto")


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, device="cuda")


def _activations(g, rows, k, lda_pad=0, shift=0.0):
    """fp16 [rows, k] (a row view of [rows, k + lda_pad]) with row magnitudes spread over 2^-4 .. 2^1."""
    scale = torch.exp2(torch.rand(rows, 1, generator=g, device="cuda") * 5 - 4)
    full = _randn(g, rows, k + lda_pad) * scale + shift * _randn(g, rows, 1)
    return full.half()[:, :k]


def _out_buffer(rows, n_out, odd):
    """(buffer filled with a sentinel, out view): out is the whole buffer, or a column slice at offset 1 with odd ldo."""
    if not odd:
        buf = torch.full((rows, n_out), SENTINEL, device="cuda", dtype=torch.float16)
        return buf, buf
    ldo = n_out + 1 if n_out % 2 == 0 else n_out + 2
    buf = torch.full((rows, ldo), SENTINEL, device="cuda", dtype=torch.float16)
    return buf, buf[:, 1:1 + n_out]


def _untouched(buf, out, what):
    mask = torch.ones_like(buf, dtype=torch.bool)
    off = (out.data_ptr() - buf.data_ptr()) // 2
    mask.view(-1)[torch.as_strided(torch.arange(buf.numel(), device="cuda"), out.shape, out.stride(), off).reshape(-1)] = False
    assert bool((buf[mask] == SENTINEL).all()), f"{what}: a kernel wrote outside its output"


def _record(kind, what, ratio, log):
    WORST[kind] = max(WORST.get(kind, 0.0), ratio)
    log.append((ratio, what))


def _linear_case(kind, bn, m, k, n, log, lda_pad=0, odd_out=False, bias="aligned", alpha=1.0, residual=False,
                 shift=4.0, row_bias=True):
    """One GEMM through the entry point of `kind` (kind 8: a one-tap conv2d_taps over a 1 x m image)."""
    what = f"BN{bn} kind{kind} m{m} k{k} n{n} pad{lda_pad} odd{int(odd_out)} bias={bias} alpha{alpha} res{int(residual)}"
    g = _gen(kind, bn, m, k, n, lda_pad, odd_out, bias, alpha, residual)
    geglu, ln = kind in (1, 3), kind in (2, 3)
    a = _activations(g, m, k, lda_pad, shift if ln else 0.0)
    w32 = _randn(g, n, k) * k ** -0.5
    b = None
    if bias is not None:
        b = _randn(g, n)
    n_out = n // 2 if geglu else n
    buf, out = _out_buffer(m, n_out, odd_out)
    ref_kw = dict(alpha=alpha, bias=b, geglu=geglu)
    if ln:
        gam, bet = 1 + 0.3 * _randn(g, k), 0.2 * _randn(g, k)
        w, cs, b = ops.fold_layer_norm(w32, b, gam, bet)
        stats = ops.row_stats(a)
        ref_kw.update(bias=b, ln=(stats, cs))
    else:
        w = w32.half()
    if bias == "odd":                                # 4 bytes past an aligned address: the scalar bias loads
        b = torch.cat([torch.zeros(1, device="cuda"), ref_kw["bias"]])[1:]
        ref_kw["bias"] = b
    acc, S = R.gemm(a, w)
    if kind in (0, 2) or geglu:
        r = None
        if residual:
            r = _randn(g, m, n + 8).half()[:, :n]
            ref_kw["residual"] = r
        if geglu:
            wk, bk = ops.pack_geglu_weight(w, ref_kw["bias"], bn)
            lnk = (stats, ops.pack_geglu_weight(w, cs, bn)[1]) if ln else None
        else:
            wk, bk, lnk = w, ref_kw["bias"], (ref_kw["ln"] if ln else None)
        ops.linear(a, wk, bias=bk, residual=r, alpha=alpha, geglu=geglu, out=out, ln=lnk)
    elif kind == 4:
        rb = None
        if row_bias:
            rb = _randn(g, (m + 3) // 4, n + 6)[:, :n]
            ref_kw["row_bias"] = rb.repeat_interleave(4, 0)[:m]
        ops.linear_gelu_rowbias(a, w, bias=b, row_bias=rb, rows_per_group=4, out=out)
        ref_kw.update(gelu=True)
    else:
        ops.conv2d_taps(a.contiguous().view(1, 1, m, k), w, [(0, 0)], bias=b, relu=True, out=out,
                        out_stride_y=m * out.stride(0), out_stride_x=out.stride(0))
        ref_kw.update(relu=True)
    torch.cuda.synchronize()
    _record(kind, what, R.check(out, R.epilogue(acc, S, k, **ref_kw), what), log)
    _untouched(buf, out, what)


def _conv_case(kind, bn, nimg, h, w_, c, n, taps, log, group=False, residual=False):
    """conv2d_3x3 (kind 0, the 3x3 taps) or conv2d_taps (kind 0 with other taps, kind 8 always) on [nimg, h, w, c]."""
    what = f"BN{bn} kind{kind} conv {nimg}x{h}x{w_} c{c} n{n} taps{len(taps)} group{int(group)} res{int(residual)}"
    g = _gen(kind, bn, nimg, h, w_, c, n, len(taps), group, residual)
    x = _activations(g, nimg * h * w_, c).reshape(nimg, h, w_, c)
    w = (_randn(g, n, len(taps) * c) * (len(taps) * c) ** -0.5).half()
    b = _randn(g, n)
    acc, S = R.gemm(R.tap_rows(x, taps), w)
    ref_kw = dict(bias=b, relu=kind == 8)
    rows = nimg * h * w_
    if group or residual:
        gb = _randn(g, (nimg + 2) // 3, n + 8).half()[:, :n] if group else None
        r = _randn(g, rows, n + 8).half()[:, :n] if residual else None
        out = ops.conv2d_3x3(x, w, bias=b, group_bias=gb, residual=r, group_div=3)
        if group:
            ref_kw["group_bias"] = gb.repeat_interleave(3, 0)[:nimg].repeat_interleave(h * w_, 0)
        ref_kw["residual"] = r
    elif kind == 0 and taps == R.TAPS_3X3:
        out = ops.conv2d_3x3(x, w, bias=b)
    else:
        out = ops.conv2d_taps(x, w, taps, bias=b, relu=kind == 8)
    torch.cuda.synchronize()
    _record(kind, what, R.check(out.reshape(rows, n), R.epilogue(acc, S, len(taps) * c, **ref_kw), what), log)


def _strided_phase_case(bn, nimg, h, w_, c, n, phase, log):
    """ReLU conv written into phase (py, px) of a 2x-upsampled [nimg, 2h, 2w, n] grid, as the transposed-conv phases do;
    the other three phases hold a sentinel that must survive."""
    py, px = phase
    what = f"BN{bn} kind8 strided phase{phase} {nimg}x{h}x{w_} n{n}"
    g = _gen(8, bn, nimg, h, w_, c, n, phase)
    x = _activations(g, nimg * h * w_, c).reshape(nimg, h, w_, c)
    taps = [(0, 0), (0, -1), (-1, 0), (-1, -1)]
    w = (_randn(g, n, 4 * c) * (4 * c) ** -0.5).half()
    b = _randn(g, n)
    buf = torch.full((nimg, 2 * h, 2 * w_, n), SENTINEL, device="cuda", dtype=torch.float16)
    ops.conv2d_taps(x, w, taps, bias=b, relu=True, out=buf.view(-1)[(py * 2 * w_ + px) * n:],
                    out_stride_y=4 * w_ * n, out_stride_x=2 * n)
    torch.cuda.synchronize()
    acc, S = R.gemm(R.tap_rows(x, taps), w)
    sub = buf[:, py::2, px::2]
    _record(8, what, R.check(sub.reshape(-1, n), R.epilogue(acc, S, 4 * c, bias=b, relu=True), what), log)
    _untouched(buf, sub, what)


def _padded_rows_case(bn, nimg, h, w_, c, n, log):
    """ReLU conv whose output rows of w * n elements are w * n + 4 apart (the gaps hold a sentinel).  An output stride
    that is not a multiple of 8 elements rules out the TMA map, while the base, ldo = n and the bias stay 16-byte aligned:
    the full chunks take the direct vector stores, the partial last chunk (n % 32 == 8) the scalar ones.  Only a strided
    output reaches the vector path: for a dense output (kinds 0-4, the FP8 entry) the alignment that enables vector
    stores also enables the TMA map, and without one (out_n < 32) no chunk is full."""
    what = f"BN{bn} kind8 padded rows {nimg}x{h}x{w_} n{n}"
    g = _gen(8, bn, nimg, h, w_, c, n, "padded")
    x = _activations(g, nimg * h * w_, c).reshape(nimg, h, w_, c)
    w = (_randn(g, n, 9 * c) * (9 * c) ** -0.5).half()
    b = _randn(g, n)
    buf = torch.full((nimg * h, w_ * n + 4), SENTINEL, device="cuda", dtype=torch.float16)
    ops.conv2d_taps(x, w, R.TAPS_3X3, bias=b, relu=True, out=buf, out_stride_y=w_ * n + 4, out_stride_x=n)
    torch.cuda.synchronize()
    acc, S = R.gemm(R.tap_rows(x, R.TAPS_3X3), w)
    sub = buf[:, :w_ * n].unflatten(1, (w_, n))
    _record(8, what, R.check(sub.reshape(-1, n), R.epilogue(acc, S, 9 * c, bias=b, relu=True), what), log)
    _untouched(buf, sub, what)


def _tconv_case(bn, batch, f, hw, c, n, log, residual=False):
    what = f"BN{bn} kind0 tconv3 b{batch} f{f} hw{hw} c{c} n{n} res{int(residual)}"
    g = _gen(0, bn, batch, f, hw, c, n, residual)
    x = _activations(g, batch * f * hw, c).reshape(batch, f, hw, c)
    w = (_randn(g, n, 3 * c) * (3 * c) ** -0.5).half()
    b = _randn(g, n)
    r = _randn(g, batch * f * hw, n + 8).half()[:, :n] if residual else None
    out = ops.tconv3(x, w, bias=b, residual=r)
    torch.cuda.synchronize()
    acc, S = R.gemm(R.tap_rows(x, R.TAPS_T3), w)
    _record(0, what, R.check(out.reshape(-1, n), R.epilogue(acc, S, 3 * c, bias=b, residual=r), what), log)


def _persistent_rows(n_blocks):
    """Rows (not a multiple of 128) giving at least 3 tiles per CTA of the persistent grid (one CTA per SM)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 128 * (math.ceil(3 * sms / n_blocks) + 1) - 37


@pytest.mark.parametrize("forced_bn,kind", PAIRS, indirect=["forced_bn"], ids=[f"bn{b}-kind{k}" for b, k in PAIRS])
def test_kernel(forced_bn, kind):
    bn, geglu, log = forced_bn, kind in (1, 3), []
    lin = lambda m, k, n, **kw: _linear_case(kind, bn, m, k, n, log, **kw)   # noqa: E731
    # rows around the 64-row warpgroup halves and the 128-row tile; two N blocks, every chunk TMA-staged
    for m in (1, 64, 65, 127, 129):
        kw = {}
        if kind == 0:
            kw = {1: dict(bias=None), 65: dict(alpha=0.37, residual=True), 129: dict(residual=True)}.get(m, {})
        if kind == 4 and m == 1:
            kw = dict(row_bias=False)
        lin(m, 128, 2 * bn, **kw)
    lin(129, 5120, bn)                                   # long K: the ring wraps many times
    lin(_persistent_rows(2), 64, 2 * bn)                 # >= 3 tiles per CTA, one k-iteration each
    lin(65, 64, 2 * bn, odd_out=True)                    # direct scalar stores: unaligned output, odd ldo
    if kind != 8:
        lin(65, 64, 2 * bn, lda_pad=64)                  # row-strided A
    if kind in (2, 3):
        lin(129, 320, 2 * bn, alpha=0.37, shift=30.0)    # folded LayerNorm, alpha != 1, a large common row offset
    if kind == 1:
        lin(129, 128, 2 * bn, alpha=0.37)
    if not geglu:
        lin(65, 128, 2 * bn, odd_out=True, bias="odd")   # scalar bias loads
        lin(65, 128, 2 * bn, bias="odd")                 # TMA map valid, but the bias forces direct scalar stores
        lin(129, 128, bn + 48)                           # staged chunks, then a direct partial chunk
        lin(129, 128, 24)                                # out_n < 32: no TMA map, direct scalar stores
        if bn >= 64:
            lin(129, 128, bn + 32)                       # the last N block ends after one chunk
    if kind in (0, 8):
        n = bn + 32
        for nimg, h, w_ in ((3, 1, 1), (2, 1, 37), (2, 3, 37), (1, 2, 129), (1, 2, 200), (6, 4, 5)):
            _conv_case(kind, bn, nimg, h, w_, 64, n, R.TAPS_3X3, log)
        g = torch.Generator().manual_seed(33)
        offs = torch.randperm(49, generator=g)[:33]
        _conv_case(kind, bn, 2, 9, 11, 64, n, [(int(o) // 7 - 3, int(o) % 7 - 3) for o in offs], log)
        _conv_case(kind, bn, 2, 5, 6, 64, n, [(127, 0), (-127, 5), (0, 127), (3, -127)], log)
    if kind == 0:
        _conv_case(0, bn, 6, 3, 5, 64, bn + 32, R.TAPS_3X3, log, group=True, residual=True)
        for f in (1, 2, 5):
            _tconv_case(bn, 3, f, 40, 64, bn + 32, log, residual=f == 5)
    if kind == 8:
        _strided_phase_case(bn, 2, 5, 7, 64, bn + 32, (1, 1), log)
        _strided_phase_case(bn, 2, 5, 7, 64, 36, (0, 1), log)
        _padded_rows_case(bn, 2, 3, 37, 64, bn + 40, log)
    worst = max(log)
    print(f"\nBN {bn} kind {kind}: {len(log)} cases, largest error / bound {worst[0]:.3f} ({worst[1]}); "
          f"so far per kind {dict(sorted(WORST.items()))}")


# ------------------------------------------------------------------------------------------------ refusals
def _epi(**kw):
    e = lib.Epilogue()
    e.alpha = 1.0
    for k, v in kw.items():
        setattr(e, k, v)
    return e


def test_refusals_launch_nothing(forced_bn):
    g = _gen("refusals")
    m, k, n = 129, 128, 256
    a = _activations(g, m, k)
    w = (_randn(g, n, k) * k ** -0.5).half()
    wp, bp = ops.pack_geglu_weight(w, _randn(g, n), 128)
    r = _randn(g, m, n // 2).half()
    w8, sw = ops.quantize_weight_e4m3(w.float())
    a8, sa = ops.quantize_rows_e4m3(a)
    out = torch.empty(m, n // 2, device="cuda", dtype=torch.float16)
    torch.cuda.synchronize()
    l = lib.load()
    l0 = lib.launch_count()
    # GEGLU drops a residual: refused by ops and, past ops, by both C entries
    with pytest.raises(VgenError, match="residual"):
        ops.linear(a, wp, bias=bp, residual=r, geglu=True)
    with pytest.raises(VgenError, match="residual"):
        ops.linear_e4m3(a8, sa, w8, sw, residual=r, geglu=True, bn=128)
    with pytest.raises(VgenError, match="residual"):
        ops.linear_fp8(a, w8, sw, residual=r, geglu=True, bn=128)
    e = _epi(residual=r.data_ptr(), residual_ld=n // 2, geglu=1, bn=128)
    assert l.vgen_linear(a.data_ptr(), m, k, k, wp.data_ptr(), n, out.data_ptr(), n // 2, ctypes.byref(e), None) != 0
    assert b"residual" in l.vgen_last_error()
    assert l.vgen_linear_fp8(a8.data_ptr(), sa.data_ptr(), m, k, k, w8.data_ptr(), sw.data_ptr(), n, out.data_ptr(), n // 2,
                             ctypes.byref(e), None) != 0
    assert b"residual" in l.vgen_last_error()
    # the conv entries too, on the SIMT kernel (c % 64 != 0) as on any other: with a residual or a per-frame bias
    x = _activations(g, 16, 8).reshape(1, 4, 4, 8)
    wc = (_randn(g, 64, 9 * 8) * 0.1).half()
    oc, rc = torch.empty(16, 32, device="cuda", dtype=torch.float16), _randn(g, 16, 32).half()
    gb = _randn(g, 1, 32).half()
    for e in (_epi(residual=rc.data_ptr(), residual_ld=32, geglu=1, bn=64),
              _epi(group_bias=gb.data_ptr(), group_bias_ld=32, geglu=1, bn=64)):
        assert l.vgen_conv2d_3x3(x.data_ptr(), 1, 4, 4, 8, wc.data_ptr(), 64, oc.data_ptr(), 32, ctypes.byref(e), None) != 0
        assert b"GEGLU epilogue takes no residual" in l.vgen_last_error()
    e = _epi(residual=rc.data_ptr(), residual_ld=32, geglu=1, bn=64)
    assert l.vgen_tconv3(x.data_ptr(), 4, 4, 8, wc[:, :24].contiguous().data_ptr(), 64, oc.data_ptr(), 32, ctypes.byref(e),
                         None) != 0
    assert b"GEGLU epilogue takes no residual" in l.vgen_last_error()
    # GEGLU loads its bias as float2 pairs of 16-byte aligned blocks
    bp_odd = torch.cat([torch.zeros(1, device="cuda"), bp])[1:]
    with pytest.raises(VgenError, match="16-byte aligned bias"):
        ops.linear(a, wp, bias=bp_odd, geglu=True, bn=128)
    # N tiles the knob or the launch cannot use
    for bad in (16, 48, 288):
        with pytest.raises(VgenError, match="bn must be"):
            ops.set_tapgemm_bn(bad)
    ops.set_tapgemm_bn(96)
    with pytest.raises(VgenError, match="GEGLU needs"):
        ops.linear(a, wp, bias=bp, geglu=True)              # GEGLU: BN % 64 != 0
    ops.set_tapgemm_bn(256)
    with pytest.raises(VgenError, match="BN <= 224"):
        ops.linear_gelu_rowbias(a, w)                       # the GELU epilogue spills at BN = 256
    with pytest.raises(VgenError, match="GEGLU needs"):
        ops.linear(a, wp[:192].contiguous(), geglu=True)    # n % BN != 0
    torch.cuda.synchronize()
    assert lib.launch_count() == l0, "a refused call launched a kernel"
    # with a tile the call can use, the same GEGLU call runs
    ops.set_tapgemm_bn(128)
    ops.linear(a, wp, bias=bp, geglu=True, out=out)
    assert lib.launch_count() == l0 + 1
