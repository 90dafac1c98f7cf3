"""GPU bring-up checks: run each op of libvgen_b200.so against a plain PyTorch fp32 reference and
print one line per case (never stops at the first failure, so one run yields a full picture).

  python tools/gpu_check.py --group tapgemm          # one group in-process
  python tools/gpu_check.py --all                    # every group, each in its own subprocess + timeout

This is a diagnostic tool; the pytest -m gpu suite is the gate.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import traceback

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

# the fp32 references (matmuls, cuDNN convs) must not run in TF32, whichever tests ran before in the same process
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

RESULTS = []


def rel_err(a, b):
    a = a.float()
    b = b.float()
    denom = b.abs().max().item() + 1e-12
    return (a - b).abs().max().item() / denom


def report(name, err, tol, extra=""):
    ok = err == err and err <= tol
    RESULTS.append({"name": name, "err": err, "tol": tol, "ok": bool(ok)})
    print(f"{'PASS' if ok else 'FAIL'}  {name:58s} err={err:.3e} tol={tol:.1e} {extra}", flush=True)


def run_case(name, fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        RESULTS.append({"name": name, "err": float("nan"), "ok": False, "exc": repr(e)})
        print(f"FAIL  {name:58s} EXC {e!r}", flush=True)
        traceback.print_exc()


# ----------------------------------------------------------------------------------------------
def group_tapgemm(impl="auto"):
    from vgen_b200 import ops
    ops.set_tapgemm_impl(impl)
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(1)

    def rnd(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).to(dev)

    def lin_case(m, k, n, bias=False, res=False, alpha=1.0, bn=0, lda_pad=0):
        def f():
            a_full = rnd(m, k + lda_pad).half()
            a = a_full[:, :k]
            w = rnd(n, k, scale=k ** -0.5).half()
            b = rnd(n) if bias else None
            r = rnd(m, n).half() if res else None
            out = ops.linear(a, w, bias=b, residual=r, alpha=alpha, bn=bn)
            torch.cuda.synchronize()
            ref = (a.float() @ w.float().t()) * alpha
            if b is not None:
                ref = ref + b
            if r is not None:
                ref = ref.half().float() + r.float()
            report(f"[{impl}] linear m{m} k{k} n{n} bias{int(bias)} res{int(res)} a{alpha} bn{bn} pad{lda_pad}",
                   rel_err(out, ref), 2e-3)
        run_case(f"linear m{m} k{k} n{n}", f)

    lin_case(128, 64, 32)
    lin_case(128, 64, 128)
    lin_case(128, 128, 128)
    lin_case(256, 256, 256, bn=256)
    lin_case(1000, 320, 320)
    lin_case(1000, 320, 320, bias=True, res=True, alpha=0.5)
    lin_case(77, 1024, 640, bias=True)
    lin_case(4096, 1280, 1280, bias=True, res=True)
    lin_case(300, 320, 4, bias=True)          # tiny N, scalar store path
    lin_case(513, 192, 960, lda_pad=64)        # row-strided A
    lin_case(20000, 640, 1920)                 # many tiles (persistent loop, accumulator ping-pong)

    def geglu_case(m, k, inner, bn):
        def f():
            a = rnd(m, k).half()
            w = rnd(2 * inner, k, scale=k ** -0.5).half()
            b = rnd(2 * inner)
            wp, bp = ops.pack_geglu_weight(w, b, bn)
            out = ops.linear(a, wp, bias=bp, geglu=True, bn=bn)
            torch.cuda.synchronize()
            proj = (a.float() @ w.float().t() + b).half().float()
            v, gate = proj[:, :inner], proj[:, inner:]
            ref = v * torch.nn.functional.gelu(gate).half().float()
            report(f"[{impl}] geglu m{m} k{k} inner{inner} bn{bn}", rel_err(out, ref), 2e-3)
        run_case(f"geglu m{m}", f)

    geglu_case(256, 320, 1280, 256)
    geglu_case(1000, 640, 2560, 128)

    # nn.LayerNorm folded into the projection (vgen_row_stats + vgen_epilogue.row_stats / col_sum) against LayerNorm -> Linear in
    # fp32; rows with a large common offset (|mean| = `shift` standard deviations) exercise the cancellation in the fold
    def ln_case(m, k, n, bias=False, geglu_bn=0, shift=0.0, lda_pad=0):
        def f():
            a_full = (rnd(m, k + lda_pad) * (1.0 + torch.rand(m, 1, generator=g).to(dev)) + shift * rnd(m, 1)).half()
            a = a_full[:, :k]
            w = rnd(n, k, scale=k ** -0.5)
            b = rnd(n) if bias else None
            gam, bet = 1.0 + 0.3 * rnd(k), 0.2 * rnd(k)
            ref = torch.nn.functional.layer_norm(a.float(), (k,), gam, bet, 1e-5) @ w.t()
            if b is not None:
                ref = ref + b
            if geglu_bn:
                inner = n // 2
                proj = ref.half().float()
                ref = proj[:, :inner] * torch.nn.functional.gelu(proj[:, inner:]).half().float()
                wb = w * gam[None, :]
                bb = (b if b is not None else torch.zeros(n, device=dev)) + w @ bet
                wp, bp = ops.pack_geglu_weight(wb, bb, geglu_bn)
                wp = wp.half()
                out = ops.linear(a, wp, bias=bp, geglu=True, bn=geglu_bn, ln=(ops.row_stats(a), wp.double().sum(1).float()))
            else:
                wf, cs, lb = ops.fold_layer_norm(w, b, gam, bet)
                out = ops.linear(a, wf, bias=lb, ln=(ops.row_stats(a), cs))
            torch.cuda.synchronize()
            report(f"[{impl}] ln-folded linear m{m} k{k} n{n} bias{int(bias)} geglu{geglu_bn} shift{shift} pad{lda_pad}",
                   rel_err(out, ref), 2e-3)
        run_case(f"ln linear m{m} k{k} n{n}", f)

    def stats_case(m, k):
        def f():
            a = (rnd(m, k) * 2.0 + 0.5).half()
            st = ops.row_stats(a)
            torch.cuda.synchronize()
            mean = a.float().mean(1)
            rstd = (a.float().var(1, unbiased=False) + 1e-5).rsqrt()
            report(f"row_stats m{m} k{k}", rel_err(st, torch.stack([rstd, -mean * rstd], 1)), 2e-5)
        run_case(f"row_stats m{m} k{k}", f)

    ln_case(1000, 320, 960)
    ln_case(513, 320, 320, shift=8.0)
    ln_case(2000, 640, 1920, bias=True, lda_pad=64)
    ln_case(300, 1280, 1280, shift=3.0)
    ln_case(1000, 320, 2560, bias=True, geglu_bn=256)
    ln_case(777, 640, 5120, bias=True, geglu_bn=128, shift=4.0)
    ln_case(100, 192, 40)                      # scalar epilogue path, LayerNorm width outside the vector kernels' set
    if impl == "auto":
        for (m, k) in [(1000, 320), (1001, 640), (64, 1280), (50, 2560), (33, 100), (7, 4096)]:
            stats_case(m, k)

    def conv_case(nimg, h, w_, c, n, bias=True, gb=False, res=False):
        def f():
            x = rnd(nimg, h, w_, c).half()
            wt = rnd(n, c, 3, 3, scale=(9 * c) ** -0.5).half()
            wp = wt.permute(0, 2, 3, 1).reshape(n, 9 * c).contiguous()
            b = rnd(n) if bias else None
            gbt = rnd(nimg, n).half() if gb else None
            r = rnd(nimg, h, w_, n).half() if res else None
            out = ops.conv2d_3x3(x, wp, bias=b, group_bias=gbt, residual=r)
            torch.cuda.synchronize()
            ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).float(), wt.float(), b, padding=1)
            ref = ref.permute(0, 2, 3, 1)
            if gbt is not None:
                ref = ref.half().float() + gbt.float()[:, None, None, :]
            if r is not None:
                ref = ref.half().float() + r.float()
            report(f"[{impl}] conv3x3 n{nimg} {h}x{w_} c{c}->{n} gb{int(gb)} res{int(res)}", rel_err(out, ref), 2e-3)
        run_case(f"conv n{nimg} {h}x{w_}", f)

    conv_case(1, 8, 16, 64, 64)
    conv_case(2, 8, 16, 64, 64, gb=True, res=True)
    conv_case(2, 32, 32, 128, 320)
    conv_case(2, 22, 40, 128, 320, gb=True)
    conv_case(3, 11, 20, 192, 128)
    conv_case(2, 44, 80, 320, 640, gb=True, res=True)
    conv_case(1, 88, 160, 320, 4)

    def tconv_case(f_, hw, c, n, res=False):
        def f():
            x = rnd(f_, hw, c).half()
            wt = rnd(n, c, 3, scale=(3 * c) ** -0.5).half()
            wp = wt.permute(0, 2, 1).reshape(n, 3 * c).contiguous()
            b = rnd(n)
            r = rnd(f_, hw, n).half() if res else None
            out = ops.tconv3(x, wp, bias=b, residual=r)
            torch.cuda.synchronize()
            xr = x.float().permute(2, 0, 1).unsqueeze(0)  # [1, c, f, hw]
            ref = torch.nn.functional.conv2d(xr, wt.float().unsqueeze(-1), b, padding=(1, 0))
            ref = ref[0].permute(1, 2, 0)
            if r is not None:
                ref = ref.half().float() + r.float()
            report(f"[{impl}] tconv3 f{f_} hw{hw} c{c}->{n} res{int(res)}", rel_err(out, ref), 2e-3)
        run_case(f"tconv f{f_} hw{hw}", f)

    def tconv_batch_case(b, f_, hw, c, n):
        def f():
            x = rnd(b, f_, hw, c).half()
            wt = rnd(n, c, 3, scale=(3 * c) ** -0.5).half()
            wp = wt.permute(0, 2, 1).reshape(n, 3 * c).contiguous()
            bias = rnd(n)
            r = rnd(b, f_, hw, n).half()
            out = ops.tconv3(x, wp, bias=bias, residual=r)
            per_video = torch.stack([ops.tconv3(x[i].contiguous(), wp, bias=bias, residual=r[i].contiguous()) for i in range(b)])
            torch.cuda.synchronize()
            report(f"[{impl}] tconv3 batched b{b} f{f_} hw{hw} c{c}->{n} == per video (frames of videos never mix)",
                   float((out.float() - per_video.float()).abs().max()), 0.0)
        run_case(f"tconv batch {b} {f_} {hw}", f)

    tconv_batch_case(2, 4, 220, 128, 128)
    tconv_batch_case(3, 16, 64, 64, 96)
    tconv_case(4, 256, 64, 64)
    tconv_case(8, 220, 128, 128, res=True)
    tconv_case(16, 32, 64, 96)
    tconv_case(16, 1024, 320, 320, res=True)
    tconv_case(1, 300, 64, 64)


def group_tapgemm_simt():
    group_tapgemm("simt")




def group_norm_checks():
    from vgen_b200 import ops
    F = torch.nn.functional
    g = torch.Generator(device="cpu").manual_seed(2)

    def rnd(*s, scale=1.0, shift=0.0):
        return (torch.randn(*s, generator=g) * scale + shift).cuda()

    for (n, p, c, eps, silu, shift) in [(2, 96, 64, 1e-5, True, 0.0), (16, 220, 1280, 1e-5, True, 0.5), (1, 16 * 880, 640, 1e-6, False, 3.0),
                                        (3, 3520, 320, 1e-5, True, 0.0), (2, 300, 2560, 1e-5, True, -1.0), (2, 1000, 1920, 1e-5, True, 0.0),
                                        (2, 5000, 32, 1e-6, True, 10.0), (1, 14080, 960, 1e-5, True, 0.0), (2, 4096, 128, 1e-6, True, 0.0)]:
        def f():
            x = rnd(n, p, c, scale=1.5, shift=shift).half()
            ga, be = rnd(c, scale=0.2, shift=1.0), rnd(c, scale=0.2)
            y = ops.group_norm(x, ga, be, eps, silu)
            torch.cuda.synchronize()
            ref = F.group_norm(x.float().permute(0, 2, 1), 32, ga, be, eps)
            if silu:
                ref = F.silu(ref)
            report(f"group_norm n{n} p{p} c{c} silu{int(silu)} shift{shift}", rel_err(y, ref.permute(0, 2, 1)), 2e-3)
        run_case(f"gn {n} {p} {c}", f)

    for (rows, c) in [(1000, 320), (1001, 320), (3, 320), (777, 640), (4096, 1280), (100, 512), (5000, 4), (33, 2560), (64, 64)]:
        def f():
            x = rnd(rows, c, scale=2.0, shift=0.3).half()
            ga, be = rnd(c, scale=0.2, shift=1.0), rnd(c, scale=0.2)
            y = ops.layer_norm(x, ga, be)
            torch.cuda.synchronize()
            report(f"layer_norm rows{rows} c{c}", rel_err(y, F.layer_norm(x.float(), (c,), ga, be, 1e-5)), 2e-3)
        run_case(f"ln {rows} {c}", f)


def group_attention():
    from vgen_b200 import ops
    F = torch.nn.functional
    g = torch.Generator(device="cpu").manual_seed(3)

    def rnd(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).cuda()

    def sdpa(q, k, v, heads):
        b, lq, inner = q.shape
        d = inner // heads
        sp = lambda t: t.float().reshape(t.shape[0], t.shape[1], heads, d).permute(0, 2, 1, 3)  # noqa: E731
        o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v))
        return o.permute(0, 2, 1, 3).reshape(b, lq, inner)

    for (b, heads, lq, lk, div, fused) in [(1, 1, 128, 128, 1, False), (1, 1, 256, 128, 1, False), (1, 1, 256, 256, 1, False),
                                           (2, 2, 300, 300, 1, True), (2, 5, 880, 880, 1, True), (4, 5, 220, 77, 4, False),
                                           (4, 10, 3520, 145, 2, False), (1, 5, 14080, 14080, 1, True), (3, 1, 96, 96, 1, True),
                                           (2, 2, 1000, 1, 1, False), (1, 2, 385, 64, 1, False), (1, 2, 400, 600, 1, False),
                                           (2, 1, 384, 65, 2, False)]:
        def f():
            inner = heads * 64
            if fused:
                qkv = rnd(b, lq, 3 * inner, scale=1.0).half()
                q, k, v = qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:]
            else:
                q = rnd(b, lq, inner).half()
                kv = rnd(b // div, lk, 2 * inner).half()
                k, v = kv[:, :, :inner], kv[:, :, inner:]
            out = ops.attention_d64(q, k, v, heads, kv_batch_div=div)
            torch.cuda.synchronize()
            kk = k.repeat_interleave(div, dim=0)
            vv = v.repeat_interleave(div, dim=0)
            report(f"attention_d64 b{b} h{heads} lq{lq} lk{lk} div{div} fused{int(fused)}", rel_err(out, sdpa(q, kk, vv, heads)), 3e-3)
        run_case(f"attn {b} {heads} {lq} {lk}", f)

    # head_dim 512 single-head flash attention (VAE AttnBlock): ragged lengths, fused qkv views, the 1280x704 size,
    # large-magnitude inputs (scores ~ +-60: fp32 statistics must hold where fp16 logits would not), batches of 3 videos
    # through the batched temporal entry
    for (b, lq, lk, fused, scale) in [(1, 128, 64, False, 1.0), (2, 200, 200, True, 1.0), (1, 96, 96, True, 1.0), (2, 130, 77, False, 1.0),
                                      (3, 1792, 1792, True, 1.0), (2, 14080, 14080, True, 1.0), (1, 640, 640, True, 4.0)]:
        def f():
            if fused:
                qkv = rnd(b, lq, 3 * 512, scale=scale).half()
                q, k, v = qkv[:, :, :512], qkv[:, :, 512:1024], qkv[:, :, 1024:]
            else:
                q = rnd(b, lq, 512, scale=scale).half()
                kv = rnd(b, lk, 1024, scale=scale).half()
                k, v = kv[:, :, :512], kv[:, :, 512:]
            out = ops.attention_d512(q, k, v)
            torch.cuda.synchronize()
            report(f"attention_d512 b{b} lq{lq} lk{lk} fused{int(fused)} x{scale}", rel_err(out, sdpa(q, k, v, 1)), 3e-3)
        run_case(f"attn512 {b} {lq} {lk}", f)

    def f():
        qkv = rnd(3, 8, 200, 3 * 128).half()
        q, k, v = qkv[..., :128], qkv[..., 128:256], qkv[..., 256:]
        out = ops.attention_temporal(q, k, v, 2, 64)
        torch.cuda.synchronize()
        tq = lambda t: t.permute(0, 2, 1, 3).reshape(3 * 200, 8, 128)  # noqa: E731  [(b npix), f, inner]
        ref = sdpa(tq(q), tq(k), tq(v), 2).reshape(3, 200, 8, 128).permute(0, 2, 1, 3)
        report("attention_temporal batched b3 f8 npix200 h2", rel_err(out, ref), 3e-3)
    run_case("tattn batched", f)

    for (f_, npix, heads, d) in [(16, 100, 1, 64), (16, 1000, 5, 64), (8, 333, 2, 64), (4, 96, 2, 64), (3, 60, 1, 64),
                                 (32, 500, 5, 64), (20, 64, 2, 64), (16, 14080, 8, 64), (16, 300, 2, 4), (4, 50, 2, 4)]:
        def f():
            inner = heads * d
            qkv = rnd(f_, npix, 3 * inner).half()
            q, k, v = qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:]
            out = ops.attention_temporal(q, k, v, heads, d)
            torch.cuda.synchronize()
            tq = lambda t: t.permute(1, 0, 2)  # noqa: E731  [npix, f, inner]
            ref = sdpa(tq(q), tq(k), tq(v), heads).permute(1, 0, 2)
            report(f"attention_temporal f{f_} npix{npix} h{heads} d{d}", rel_err(out, ref), 3e-3)
        run_case(f"tattn {f_} {npix}", f)

    for (b, heads, L, d) in [(3, 2, 77, 64), (1, 16, 77, 64), (2, 2, 17, 80)]:
        def f():
            inner = heads * d
            qkv = rnd(b, L, 3 * inner).half()
            q, k, v = qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:]
            out = ops.attention_cross_small(q, k, v, heads, causal=True)
            torch.cuda.synchronize()
            sp = lambda t: t.float().reshape(b, L, heads, d).permute(0, 2, 1, 3)  # noqa: E731
            ref = F.scaled_dot_product_attention(sp(q), sp(k), sp(v), is_causal=True).permute(0, 2, 1, 3).reshape(b, L, inner)
            report(f"attention_cross_small causal b{b} h{heads} L{L} d{d}", rel_err(out, ref), 3e-3)
        run_case(f"causal attn {b} {heads} {L}", f)

    def f():
        ids = torch.randint(0, 1000, (3, 77), generator=g).cuda()
        table, pos = rnd(1000, 128, scale=0.02), rnd(77, 128, scale=0.02)
        out = ops.embed_tokens(ids, table, pos)
        x = rnd(4, 17, 160).half()
        add = rnd(17, 160)
        ref2 = (x.float() + add).half()
        ops.add_rows_f32_(x, add)
        torch.cuda.synchronize()
        report("embed_tokens", rel_err(out, (table[ids] + pos).half()), 1e-6)
        report("add_rows_f32", rel_err(x, ref2), 1e-6)
    run_case("clip embeddings", f)

    def f():
        x = rnd(700, 1500, scale=3.0).half()
        ref = torch.softmax(x.float() * 0.25, dim=-1)
        ops.softmax_rows_(x, 0.25)
        torch.cuda.synchronize()
        report("softmax_rows 700x1500", rel_err(x, ref), 2e-3)
    run_case("softmax", f)


def group_elementwise():
    from vgen_b200 import ops
    F = torch.nn.functional
    g = torch.Generator(device="cpu").manual_seed(4)

    def rnd(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).cuda()

    def f():
        x = rnd(2, 4, 3, 8, 12)
        y = ops.cp_to_pc(x.reshape(2, 4, -1), 2, 4, 3 * 8 * 12, c_pad=8)
        torch.cuda.synchronize()
        ref = torch.zeros(2, 288, 8, device="cuda")
        ref[:, :, :4] = x.reshape(2, 4, 288).permute(0, 2, 1)
        report("cp_to_pc fp32 pad8", rel_err(y, ref.half()), 1e-6)
        z = ops.pc_to_cp(y, 2, 4, 288, torch.float32)
        torch.cuda.synchronize()
        report("pc_to_cp fp32", rel_err(z, x.reshape(2, 4, 288).half().float()), 1e-6)
    run_case("layout", f)

    for (nimg, h, w, c, n, stride, act) in [(2, 8, 12, 8, 64, 1, False), (2, 16, 20, 64, 128, 2, False), (1, 9, 13, 4, 16, 1, True),
                                            (3, 32, 32, 32, 64, 2, True), (2, 11, 21, 320, 320, 2, False)]:
        def f():
            x = rnd(nimg, h, w, c).half()
            wt = rnd(n, c, 3, 3, scale=(9 * c) ** -0.5).half()
            b = rnd(n)
            ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
            kpad = ((9 * c + 63) // 64) * 64
            col = ops.im2col(x, 3, 3, stride, 1, 1, ho, wo, kpad, act_silu=act)
            wp = torch.zeros(n, kpad, device="cuda", dtype=torch.float16)
            wp[:, :9 * c] = wt.permute(0, 2, 3, 1).reshape(n, 9 * c)
            out = ops.linear(col, wp, bias=b).reshape(nimg, ho, wo, n)
            torch.cuda.synchronize()
            xin = x.float().permute(0, 3, 1, 2)
            if act:
                xin = F.silu(xin).half().float()
            ref = F.conv2d(xin, wt.float(), b, stride=stride, padding=1).permute(0, 2, 3, 1)
            report(f"im2col+linear n{nimg} {h}x{w} c{c}->{n} s{stride} silu{int(act)}", rel_err(out, ref), 2e-3)
        run_case(f"im2col {h}x{w} c{c}", f)

    def f():
        x = rnd(2, 5, 7, 64).half()
        y = ops.upsample_nearest2x(x)
        torch.cuda.synchronize()
        ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
        report("upsample_nearest2x", rel_err(y, ref), 1e-6)
        a, b = rnd(100, 320).half(), rnd(100, 640).half()
        c = ops.concat_channels(a, b)
        torch.cuda.synchronize()
        report("concat_channels", rel_err(c, torch.cat([a, b], -1)), 1e-6)
        a2, b2 = rnd(33, 4).half(), rnd(33, 4).half()
        c2 = ops.concat_channels(a2, b2)
        torch.cuda.synchronize()
        report("concat_channels small", rel_err(c2, torch.cat([a2, b2], -1)), 1e-6)
        report("eltwise silu", rel_err(ops.eltwise("silu", a), F.silu(a.float())), 2e-3)
        report("eltwise gelu", rel_err(ops.eltwise("gelu", a), F.gelu(a.float())), 2e-3)
        report("eltwise axpy", rel_err(ops.eltwise("axpy", a, a, s=1.0), 2 * a.float()), 2e-3)
    run_case("misc", f)

    for (m, k, n, silu, gelu, res) in [(1, 320, 1280, False, False, False), (2, 1280, 1280, True, False, False), (3, 1024, 4096, True, False, False),
                                       (5000, 4, 24, False, False, False), (5000, 8, 4, False, False, True), (5000, 4, 16, False, True, False)]:
        def f():
            a = rnd(m, k).half()
            w = rnd(n, k, scale=k ** -0.5).half()
            b = rnd(n)
            r = rnd(m, n).half() if res else None
            out = ops.linear_small(a, w, b, residual=r, silu_in=silu, gelu_out=gelu)
            torch.cuda.synchronize()
            ain = F.silu(a.float()).half().float() if silu else a.float()
            ref = ain @ w.float().t() + b
            if gelu:
                ref = F.gelu(ref.half().float())
            if res:
                ref = ref.half().float() + r.float()
            report(f"linear_small m{m} k{k} n{n} silu{int(silu)} gelu{int(gelu)} res{int(res)}", rel_err(out, ref), 2e-3)
        run_case(f"linear_small {m} {k} {n}", f)

    def f():
        t = torch.tensor([981, 1, 500], device="cuda")
        e = ops.sinusoidal_embedding(t, 320)
        torch.cuda.synchronize()
        half = 160
        tf = t.float()
        sin = torch.outer(tf, torch.pow(10000, -torch.arange(half, device="cuda").to(tf).div(half)))
        ref = torch.cat([torch.cos(sin), torch.sin(sin)], dim=1)
        report("sinusoidal_embedding", (e.float() - ref).abs().max().item(), 2e-3)
        x = rnd(2, 11, 20, 32).half()
        y = ops.adaptive_avgpool(x, 32, 32, silu_in=True)
        torch.cuda.synchronize()
        ref = F.adaptive_avg_pool2d(F.silu(x.float()).half().float().permute(0, 3, 1, 2), (32, 32)).permute(0, 2, 3, 1)
        report("adaptive_avgpool 11x20->32x32", rel_err(y, ref), 2e-3)
        x = rnd(1, 88, 160, 32).half()
        y = ops.adaptive_avgpool(x, 32, 32)
        torch.cuda.synchronize()
        ref = F.adaptive_avg_pool2d(x.float().permute(0, 3, 1, 2), (32, 32)).permute(0, 2, 3, 1)
        report("adaptive_avgpool 88x160->32x32", rel_err(y, ref), 2e-3)
    run_case("embed/pool", f)

    def f():
        xt = rnd(1, 4, 4, 8, 12)
        y, u = rnd(1, 4, 4, 8, 12).half(), rnd(1, 4, 4, 8, 12).half()
        coef = [0.6, 0.8, 1.0 / 0.6, (1 / 0.36 - 1) ** 0.5, 0.7, (1 - 0.49) ** 0.5, 0.0]
        out = u + 9.0 * (y - u)           # fp16 tensor arithmetic, like the reference under autocast
        # _i() yields fp32 tensors of shape [b,1,1,1,1] (dimensioned, so they take part in type promotion)
        ct = [torch.tensor(v, device="cuda", dtype=torch.float32).view(1, 1, 1, 1, 1) for v in coef]
        x0 = ct[0] * xt - ct[1] * out
        eps = (ct[2] * xt - x0) / ct[3]
        ref = ct[4] * x0 + ct[5] * eps
        got = ops.ddim_step_(xt.clone(), y, u, coef, 9.0, True)
        torch.cuda.synchronize()
        report("ddim_step cfg v-pred", rel_err(got, ref), 1e-5)
    run_case("ddim", f)


def group_variants():
    """Kernels of the a21 model variants (variants.cu) against torch fp32 references of the reference ops."""
    from vgen_b200 import ops
    F = torch.nn.functional
    g = torch.Generator(device="cpu").manual_seed(5)

    def rnd(*s, scale=1.0):
        return (torch.randn(*s, generator=g) * scale).cuda()

    for (b, heads, lq, lk, d, div) in [(2, 8, 16, 77, 160, 1), (1, 8, 3, 5, 32, 1), (4, 2, 7, 9, 256, 2), (1, 1, 1, 1, 8, 1)]:
        def f():
            inner = heads * d
            q = rnd(b, lq, inner).half()
            kv = rnd(b // div, lk, 2 * inner).half()
            k, v = kv[:, :, :inner], kv[:, :, inner:]
            out = ops.attention_cross_small(q, k, v, heads, kv_batch_div=div)
            sp = lambda t: t.float().reshape(t.shape[0], t.shape[1], heads, d).permute(0, 2, 1, 3)  # noqa: E731
            kk, vv = k.repeat_interleave(div, 0), v.repeat_interleave(div, 0)
            ref = F.scaled_dot_product_attention(sp(q), sp(kk), sp(vv)).permute(0, 2, 1, 3).reshape(b, lq, inner)
            report(f"attention_cross_small b{b} h{heads} lq{lq} lk{lk} d{d} div{div}", rel_err(out, ref), 2e-3)
        run_case(f"attn_small {b} {heads} {lq} {lk} {d}", f)

    for (nseq, lin, lout, c) in [(2, 31, 32, 320), (1, 2, 3, 64), (3, 7, 16, 20), (1, 1, 4, 8)]:
        def f():
            x = rnd(nseq, lin, c).half()
            out = ops.interp_linear_rows(x, lout)
            ref = F.interpolate(x.float().transpose(1, 2), size=lout, mode="linear").transpose(1, 2)
            report(f"interp_linear_rows {nseq}x{lin}->{lout} c{c}", rel_err(out, ref), 1e-3)
        run_case(f"interp {nseq} {lin} {lout}", f)

    def fft_filter(x_nchw, scale):
        xf = torch.fft.fftshift(torch.fft.fftn(x_nchw.float(), dim=(-2, -1)), dim=(-2, -1))
        hh, ww = xf.shape[-2:]
        mask = torch.ones_like(xf.real)
        mask[..., hh // 2 - 1:hh // 2 + 1, ww // 2 - 1:ww // 2 + 1] = scale
        return torch.fft.ifftn(torch.fft.ifftshift(xf * mask, dim=(-2, -1)), dim=(-2, -1)).real

    for (n, h, w, c, scale) in [(3, 5, 6, 128, 0.6), (32, 12, 20, 1280, 0.4), (2, 7, 9, 100, 0.6), (1, 2, 2, 64, 0.4)]:
        def f():
            x = (rnd(n, h, w, c) + 0.7).half()
            wide = torch.zeros(n, h, w, c + 64, device="cuda", dtype=torch.float16)
            ops.fourier_lowfreq_filter(x, scale, out=wide.view(-1, c + 64)[:, 32:32 + c])
            ref = fft_filter(x.permute(0, 3, 1, 2), scale).permute(0, 2, 3, 1)
            report(f"fourier_lowfreq {n}x{h}x{w} c{c} s{scale}", rel_err(wide[..., 32:32 + c], ref), 1e-3)
            report(f"fourier_lowfreq {n}x{h}x{w} c{c} untouched columns", float(wide[..., :32].abs().max() + wide[..., 32 + c:].abs().max()), 0.0)
        run_case(f"fourier {n} {h} {w} {c}", f)

    def f():
        x = rnd(3, 5, 7, 64).half()
        out = ops.upsample_nearest2x_rows(x, 1, 8)
        ref = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest")[..., 1:-1, :].permute(0, 2, 3, 1)
        report("upsample_nearest2x_rows crop 1", rel_err(out, ref), 0.0)
        src = rnd(100, 96).half()
        dst = torch.zeros(100, 200, device="cuda", dtype=torch.float16)
        ops.scale_copy2d(src[:, :40], dst[:, 8:48], 1.1)
        report("scale_copy2d", rel_err(dst[:, 8:48], (src[:, :40] * 1.1)), 0.0)
        report("scale_copy2d untouched", float(dst[:, :8].abs().max() + dst[:, 48:].abs().max()), 0.0)
    run_case("upsample_rows/scale_copy", f)

    # GaussianDiffusion step kernels (sampler_gauss.cu) vs the reference expressions under fp16 autocast dtypes
    def f():
        b, n = 2, 4 * 3 * 10 * 12
        y, u = rnd(b, 4, 3, 10, 12).half(), rnd(b, 4, 3, 10, 12).half()
        xt = rnd(b, 4, 3, 10, 12)
        out, stats = ops.cfg_combine(y, u, 9.0)
        ref_out = u + 9.0 * (y - u)                                   # fp16 tensor ops, like upstream
        report("cfg_combine out (bit-exact fp16 op order)", float((out.float() - ref_out.float()).abs().max()), 0.0)
        s = stats.cpu()
        for i, (nm, t) in enumerate((("sum y", y), ("sum y^2", y.float() ** 2), ("sum out", ref_out), ("sum out^2", ref_out.float() ** 2))):
            want = t.double().flatten(1).sum(1).cpu()
            report(f"cfg_combine stats {nm}", float(((s[:, i] - want).abs() / (want.abs() + 1)).max()), 1e-9)
        ratio = (y.flatten(1).std(dim=1) / (ref_out.flatten(1).std(dim=1) + 1e-12)).view(-1, 1, 1, 1, 1)
        resc = ref_out * (0.3 * ratio + (1 - 0.3) * 1.0)
        al, sg = torch.full((b, 1, 1, 1, 1), 0.8, device="cuda"), torch.full((b, 1, 1, 1, 1), 0.6, device="cuda")  # fp32 tensors, like _i()
        for pred, want in (("v", al * xt - sg * resc), ("eps", (xt - sg * resc) / al), ("x0", resc.float())):
            got = ops.gauss_x0(xt, out, 0.8, 0.6, pred, stats, 0.3)
            report(f"gauss_x0 {pred} with guide_rescale", rel_err(got, want), 2e-3)
        got = ops.gauss_x0(xt, out, 0.8, 0.6, "v")
        report("gauss_x0 v no rescale", rel_err(got, al * xt - sg * ref_out), 1e-6)
        a, c, d = rnd(5, 77), rnd(5, 77), rnd(5, 77)
        report("lincomb_f32 4 terms", rel_err(ops.lincomb_f32([(0.5, a), (-2.0, c), (3.0, d), (0.25, a)]), 0.75 * a - 2 * c + 3 * d), 1e-6)
        report("lincomb_f32 1 term in place", rel_err(ops.lincomb_f32([(0.3, a)], out=a.clone()), 0.3 * a), 1e-7)
    run_case("gauss sampler kernels", f)


GROUPS = {
    "variants": group_variants,
    "tapgemm": group_tapgemm,
    "tapgemm_simt": group_tapgemm_simt,
    "norm": group_norm_checks,
    "attention": group_attention,
    "elementwise": group_elementwise,
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--group", default=None)
    ap.add_argument("--all", action="store_true")
    ap.add_argument("--only", default=None, help="comma-separated group names for --all")
    ap.add_argument("--timeout", type=int, default=240)
    ap.add_argument("--out", default="gpurun_out/gpu_check.json")
    args = ap.parse_args()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    if args.all:
        summary = {}
        names = args.only.split(",") if args.only else list(GROUPS)
        for name in names:
            out = args.out.replace(".json", f".{name}.json")
            t0 = time.time()
            try:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--group", name, "--out", out],
                                   timeout=args.timeout)
                summary[name] = {"rc": r.returncode, "s": round(time.time() - t0, 1)}
            except subprocess.TimeoutExpired:
                summary[name] = {"rc": "timeout", "s": round(time.time() - t0, 1)}
            print(f"== group {name}: {summary[name]}", flush=True)
        with open(args.out, "w") as fh:
            json.dump(summary, fh, indent=1)
        return 0
    print(f"device: {torch.cuda.get_device_name(0)}; torch {torch.__version__}", flush=True)
    GROUPS[args.group]()
    torch.cuda.synchronize()
    with open(args.out, "w") as fh:
        json.dump(RESULTS, fh, indent=1)
    nfail = sum(1 for r in RESULTS if not r["ok"])
    print(f"== {args.group}: {len(RESULTS) - nfail} pass, {nfail} fail", flush=True)
    return 1 if nfail else 0


if __name__ == "__main__":
    sys.exit(main())
