"""Numerics + timing report of every native kernel against fp32 PyTorch references.

Run on an H100:  python tests/gpu_kernel_check.py [--out output/kernel_check.json]
Never aborts on the first failure: every case is recorded (ok / max error / device time / achieved
TFLOP/s or GB/s) so one GPU call yields the full picture.
"""
import argparse
import json
import math
import os
import sys
import traceback

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from libai_b200 import ops  # noqa: E402

RESULTS = []


def timeit(fn, iters=20, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    times = []
    for _ in range(iters):
        flush.zero_()  # evict L2 (50 MB on H100)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    return times[len(times) // 2]


ONLY = None
OUT_PATH = None


def record(name, fn):
    if ONLY and not any(name.startswith(o) for o in ONLY):
        return
    try:
        info = fn() or {}
        info.setdefault("ok", True)
    except Exception as e:  # noqa
        info = {"ok": False, "error": f"{type(e).__name__}: {e}", "trace": traceback.format_exc()[-1500:]}
        try:
            torch.cuda.synchronize()
        except Exception as e2:  # a sticky CUDA error poisons the context: stop here
            info["fatal"] = str(e2)
            RESULTS.append({"name": name, **info})
            print(json.dumps(RESULTS[-1]), flush=True)
            raise SystemExit(3)
    RESULTS.append({"name": name, **info})
    print(json.dumps({k: v for k, v in RESULTS[-1].items() if k != "trace"}), flush=True)
    if OUT_PATH:
        os.makedirs(os.path.dirname(OUT_PATH) or ".", exist_ok=True)
        with open(OUT_PATH, "w") as f:
            json.dump(RESULTS, f, indent=1)


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def check_gemm(ext, layout, M, N, K, bn=0, splits=1, fp32_out=False, time_it=False):
    def run():
        g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K + layout)
        if layout == 0:
            a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
            b = torch.randn(N, K, device="cuda", generator=g).bfloat16()
            ref = a.float() @ b.float().t()
        elif layout == 1:
            a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
            b = torch.randn(K, N, device="cuda", generator=g).bfloat16()
            ref = a.float() @ b.float()
        else:
            a = torch.randn(K, M, device="cuda", generator=g).bfloat16()
            b = torch.randn(K, N, device="cuda", generator=g).bfloat16()
            ref = a.float().t() @ b.float()
        out = ext.gemm_tuned(a, b, layout, bn, splits, fp32_out)
        torch.cuda.synchronize()
        err = rel_err(out, ref)
        tol = 2e-2 if out.dtype == torch.bfloat16 else 2e-3
        info = {"ok": err < tol, "rel_err": err, "shape": [M, N, K], "layout": layout, "bn": bn, "splits": splits}
        if time_it:
            ms = timeit(lambda: ext.gemm_tuned(a, b, layout, bn, splits, fp32_out))
            lib = timeit(lambda: (a @ b.t()) if layout == 0 else ((a @ b) if layout == 1 else (a.t() @ b)))
            info.update(ms=ms, tflops=2.0 * M * N * K / ms / 1e9, cublas_ms=lib, cublas_tflops=2.0 * M * N * K / lib / 1e9)
        return info

    record(f"gemm L{layout} {M}x{N}x{K} bn{bn} s{splits}{' f32' if fp32_out else ''}", run)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="output/kernel_check.json")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--only", default="", help="comma separated name prefixes")
    args = ap.parse_args()
    global ONLY, OUT_PATH
    ONLY = [o for o in args.only.split(",") if o] or None
    OUT_PATH = args.out
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    ext = ops.load_ext()
    torch.manual_seed(0)
    print("device:", torch.cuda.get_device_name(0), flush=True)

    # ------------------------------------------------------------------ GEMM correctness
    for layout in (0, 1, 2):
        for bn in (64, 128, 192, 256):
            check_gemm(ext, layout, 256, 512, 256, bn=bn)
    check_gemm(ext, 0, 1000, 1304, 1032)          # ragged M, N, K tails
    check_gemm(ext, 1, 1000, 1304, 1032)
    check_gemm(ext, 2, 1000, 1304, 1032, splits=3)
    check_gemm(ext, 0, 384, 256, 4096, fp32_out=True)
    check_gemm(ext, 2, 1024, 1024, 8192, splits=0)  # heuristic split-K with atomics
    # ------------------------------------------------------------------ GEMM speed (GPT-2 / BERT shapes)
    if not args.quick:
        for (M, N, K) in [(8192, 3072, 1024), (8192, 1024, 1024), (8192, 4096, 1024), (8192, 1024, 4096),
                          (8192, 50304, 1024), (8192, 8192, 8192)]:
            check_gemm(ext, 0, M, N, K, time_it=True)
        check_gemm(ext, 1, 8192, 1024, 4096, time_it=True)   # dgrad
        check_gemm(ext, 1, 8192, 1024, 50304, time_it=True)  # LM-head dgrad
        check_gemm(ext, 2, 4096, 1024, 8192, splits=0, time_it=True)  # wgrad [f, h]
        check_gemm(ext, 2, 1024, 1024, 8192, splits=0, time_it=True)
        check_gemm(ext, 2, 50304, 1024, 8192, splits=0, time_it=True)

    # ------------------------------------------------------------------ fused linear fwd (bias + gelu, pre-activation)
    def lin():
        x = torch.randn(512, 1024, device="cuda").bfloat16()
        w = (torch.randn(4096, 1024, device="cuda") * 0.05).bfloat16()
        b = torch.randn(4096, device="cuda").bfloat16()
        y, pre = ext.linear_fwd(x, w, b, 1, True)
        ref_pre = x.float() @ w.float().t() + b.float()
        ref = torch.nn.functional.gelu(ref_pre)
        return {"ok": rel_err(y, ref) < 2e-2 and rel_err(pre, ref_pre) < 2e-2, "rel_err": rel_err(y, ref)}

    record("linear_fwd bias+gelu", lin)

    def lin_speed():
        # the h->4h projection of the benchmark model: bias + GELU + pre-activation copy in the GEMM epilogue
        x = torch.randn(8192, 1024, device="cuda").bfloat16()
        w = (torch.randn(4096, 1024, device="cuda") * 0.02).bfloat16()
        b = torch.randn(4096, device="cuda").bfloat16()
        ms = timeit(lambda: ext.linear_fwd(x, w, b, 1, True))
        ms_plain = timeit(lambda: ext.linear_fwd(x, w, None, 0, False))
        return {"ok": True, "ms_bias_gelu_pre": ms, "ms_plain": ms_plain,
                "tflops": 2 * 8192 * 4096 * 1024 / ms / 1e9}

    record("linear_fwd speed", lin_speed)

    def mlp_fn():
        from libai_b200.ops import functional as OF
        x = (torch.randn(1024, 512, device="cuda")).bfloat16().requires_grad_(True)
        w1 = (torch.randn(2048, 512, device="cuda") * 0.05).bfloat16().requires_grad_(True)
        b1 = (torch.randn(2048, device="cuda") * 0.1).bfloat16().requires_grad_(True)
        w2 = (torch.randn(512, 2048, device="cuda") * 0.05).bfloat16().requires_grad_(True)
        y = OF.mlp(x, w1, b1, w2, "gelu")
        gy = torch.randn_like(y)
        y.backward(gy)
        xf, w1f, b1f, w2f = [t.detach().float().requires_grad_(True) for t in (x, w1, b1, w2)]
        ref = torch.nn.functional.gelu(xf @ w1f.t() + b1f) @ w2f.t()
        ref.backward(gy.float())
        e = [rel_err(y, ref), rel_err(x.grad, xf.grad), rel_err(w1.grad, w1f.grad), rel_err(b1.grad, b1f.grad),
             rel_err(w2.grad, w2f.grad)]
        pre = (torch.randn(8192, 4096, device="cuda")).bfloat16()
        g = torch.randn(8192, 1024, device="cuda").bfloat16()
        w = (torch.randn(1024, 4096, device="cuda") * 0.02).bfloat16()
        ms = timeit(lambda: ext.dgrad_actgrad(g, w, pre, 1))
        ms_sep = timeit(lambda: ext.act_bwd(ext.gemm(g, w, 1, None, None, False, torch.bfloat16), pre, 1))
        return {"ok": max(e) < 3e-2, "errs": e, "dgrad_actgrad_ms": ms, "dgrad_then_actbwd_ms": ms_sep}

    record("mlp fused fwd/bwd", mlp_fn)

    def fused_bias_grad():
        """Bias gradient (column sums of dpre) accumulated by the dgrad+act' epilogue: raw op against a column sum of
        its own output (incl. ragged M / N and accumulation into a non-zero buffer), then through the MLP autograd node
        with main_grad parameters against the unfused path."""
        from libai_b200 import ops
        from libai_b200.ops import functional as OF

        e = {}
        for (M, N, K) in [(777, 520, 256), (8192, 4096, 1024)]:
            g = torch.randn(M, K, device="cuda").bfloat16()
            w = (torch.randn(K, N, device="cuda") * 0.05).bfloat16()
            pre = torch.randn(M, N, device="cuda").bfloat16()
            acc = torch.full((N,), 0.5, device="cuda")
            out = ext.dgrad_actgrad(g, w, pre, 1, acc)
            plain = ext.dgrad_actgrad(g, w, pre, 1, None)
            e[f"out_unchanged_{M}x{N}"] = rel_err(out, plain)
            e[f"colsum_{M}x{N}"] = rel_err(acc, out.float().sum(0) + 0.5)
        g = torch.randn(8192, 1024, device="cuda").bfloat16()
        w = (torch.randn(1024, 4096, device="cuda") * 0.02).bfloat16()
        pre = torch.randn(8192, 4096, device="cuda").bfloat16()
        acc = torch.zeros(4096, device="cuda")
        ms_fused = timeit(lambda: ext.dgrad_actgrad(g, w, pre, 1, acc))
        ms_plain = timeit(lambda: ext.dgrad_actgrad(g, w, pre, 1, None))
        out = ext.dgrad_actgrad(g, w, pre, 1, None)
        ms_colsum = timeit(lambda: ext.colsum(out, acc))

        def run(fused):
            ops.set_fused_bias_grad(fused)
            torch.manual_seed(0)
            x = torch.randn(1024, 512, device="cuda").bfloat16().requires_grad_(True)
            ps = [torch.nn.Parameter((torch.randn(2048, 512, device="cuda") * 0.05).bfloat16()),
                  torch.nn.Parameter((torch.randn(2048, device="cuda") * 0.1).bfloat16()),
                  torch.nn.Parameter((torch.randn(512, 2048, device="cuda") * 0.05).bfloat16())]
            for p_ in ps:
                p_.main_grad = torch.zeros(p_.shape, device="cuda")
            y = OF.mlp(x, ps[0], ps[1], ps[2], "gelu")
            y.backward(torch.ones_like(y))
            assert all(p_.grad is None for p_ in ps)
            return [x.grad] + [p_.main_grad for p_ in ps]

        try:
            a, b = run(False), run(True)
        finally:
            ops.set_fused_bias_grad(False)
        e["mlp_node"] = max(rel_err(u, v) for u, v in zip(b, a))
        return {"ok": max(e.values()) < 2e-3, "errs": e, "dgrad_fused_ms": ms_fused, "dgrad_plain_ms": ms_plain,
                "separate_colsum_ms": ms_colsum}

    record("fused bias grad", fused_bias_grad)

    def bias_residual_epilogue():
        """x·Wᵀ + bias + residual in the GEMM epilogue (raw op, autograd op, and inside the fused MLP node)."""
        from libai_b200.ops import functional as OFn

        M, K, N = 2048 + 64, 1024, 768
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.03).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        r = torch.randn(M, N, device="cuda").bfloat16()
        ref = x.float() @ w.float().t() + b.float() + r.float()
        e = [rel_err(ext.linear_bias_residual(x, w, b, r), ref), rel_err(ext.linear_bias_residual(x, w, None, r), ref - b.float())]
        xa, wa, ba, ra = (t.clone().requires_grad_(True) for t in (x, w, b, r))
        xb, wb, bb, rb = (t.clone().requires_grad_(True) for t in (x, w, b, r))
        gy = torch.randn(M, N, device="cuda").bfloat16()
        OFn.linear_bias_residual(xa, wa, ba, ra).backward(gy)
        (OFn.linear(xb, wb, bb) + rb).backward(gy)
        e += [rel_err(xa.grad, xb.grad), rel_err(wa.grad, wb.grad), rel_err(ba.grad, bb.grad), rel_err(ra.grad, rb.grad)]
        F1 = 512
        w1 = (torch.randn(F1, K, device="cuda") * 0.03).bfloat16().requires_grad_(True)
        b1 = torch.randn(F1, device="cuda").bfloat16().requires_grad_(True)
        w2 = (torch.randn(K, F1, device="cuda") * 0.03).bfloat16().requires_grad_(True)
        b2 = torch.randn(K, device="cuda").bfloat16().requires_grad_(True)
        res = torch.randn(M, K, device="cuda").bfloat16().requires_grad_(True)
        xin = x.clone().requires_grad_(True)
        y1 = OFn.mlp(xin, w1, b1, w2, "gelu", b2, res)
        g = torch.randn_like(y1)
        y1.backward(g)
        got = [t.grad.clone() for t in (xin, w1, b1, w2, b2, res)]
        for t in (xin, w1, b1, w2, b2, res):
            t.grad = None
        y0 = OFn.mlp(xin, w1, b1, w2, "gelu") + b2 + res
        y0.backward(g)
        e.append(rel_err(y1, y0))
        e += [rel_err(a, t.grad) for a, t in zip(got, (xin, w1, b1, w2, b2, res))]
        ms_fused = timeit(lambda: ext.linear_bias_residual(x, w, b, r))
        ms_sep = timeit(lambda: ext.bias_residual_fwd(ext.linear_fwd(x, w, None, 0, False)[0], b, r))
        return {"ok": max(e) < 2e-2, "errs": e, "fused_ms": ms_fused, "gemm_then_bias_residual_ms": ms_sep}

    record("bias+residual GEMM epilogue", bias_residual_epilogue)

    def embedding_native():
        """Native embedding gather + scatter-add backward into an fp32 main_grad (with a vocabulary-shard offset)."""
        from libai_b200.ops import functional as OFn

        V, H, start = 1000, 256, 300
        table = torch.nn.Parameter(torch.randn(V, H, device="cuda").bfloat16())
        ids = torch.randint(0, V + 2 * start, (4, 96), device="cuda")
        ids[0, :8] = ids[0, 0]                                   # duplicates: several tokens hit the same row
        out = OFn.embedding(ids, table, start)
        local = ids - start
        inside = (local >= 0) & (local < V)
        ref = torch.nn.functional.embedding(local.clamp(0, V - 1), table.detach().float()) * inside[..., None]
        e = [rel_err(out, ref)]
        gy = torch.randn_like(out)
        table.main_grad = torch.full((V, H), 0.25, device="cuda")
        out.backward(gy)
        want = torch.zeros(V, H, device="cuda").index_add_(0, local.clamp(0, V - 1).reshape(-1),
                                                            (gy.float() * inside[..., None]).reshape(-1, H)) + 0.25
        e.append(rel_err(table.main_grad, want))
        assert table.grad is None
        t2 = torch.nn.Parameter(table.detach().clone())          # no main_grad: gradient returned to autograd
        OFn.embedding(ids, t2, start).backward(gy)
        e.append(rel_err(t2.grad, want - 0.25))
        big = torch.nn.Parameter(torch.randn(50304, 1024, device="cuda").bfloat16())
        big.main_grad = torch.zeros(50304, 1024, device="cuda")
        tok = torch.randint(0, 50304, (8, 1024), device="cuda")
        g8 = torch.randn(8, 1024, 1024, device="cuda").bfloat16()
        ms_f = timeit(lambda: ext.embedding_fwd(tok.reshape(-1), big, 0))
        ms_b = timeit(lambda: ext.embedding_bwd(tok.reshape(-1), g8.view(-1, 1024), big.main_grad, 0))
        return {"ok": max(e) < 1e-2, "errs": e, "fwd_ms_8192x1024": ms_f, "bwd_ms_8192x1024": ms_b}

    record("embedding gather / scatter-add", embedding_native)

    def fp8_forward_gemm():
        """E4M3 forward GEMM (wgmma e4m3): close to an fp32 matmul of the *dequantised* operands (the errors left are
        the fp8 accumulator, which keeps about 12-13 bits rather than fp32's 24 (dev/measure_fp8_acc.py), and the bf16
        rounding of the output), close to the bf16 GEMM, plus quantiser checks and timing."""
        e = {}
        x = torch.randn(777, 1040, device="cuda").bfloat16() * 3
        xq, dx = ext.quantize_e4m3(x)
        amax = x.float().abs().max()
        e["deq_scale"] = abs(float(dx) * 448 / float(amax) - 1)
        e["quant_vs_torch"] = rel_err(xq.float() * dx, (x.float() * (448 / amax)).to(torch.float8_e4m3fn).float() * dx)
        e["quant_roundtrip"] = rel_err(xq.float() * dx, x)              # e4m3: 3 mantissa bits -> a few percent
        odd = torch.randn(1003, device="cuda").bfloat16()               # tail path (n % 8 != 0)
        oq, do = ext.quantize_e4m3(odd)
        e["quant_tail"] = rel_err(oq.float() * do, (odd.float() * (448 / odd.float().abs().max())).to(torch.float8_e4m3fn).float() * do)
        res = {}
        for (M, N, K) in [(777, 520, 1040), (8192, 3072, 1024), (8192, 4096, 1024), (8192, 1024, 4096)]:
            x = torch.randn(M, K, device="cuda").bfloat16()
            w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
            b = torch.randn(N, device="cuda").bfloat16()
            r = torch.randn(M, N, device="cuda").bfloat16()
            xq, dx = ext.quantize_e4m3(x)
            wq, dw = ext.quantize_e4m3(w)
            ref = (xq.float() * dx) @ (wq.float() * dw).t()
            y, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, False, None)
            e[f"{M}x{N}x{K}"] = rel_err(y, ref)
            yb, pre = ext.linear_fp8_fwd(xq, wq, dx, dw, b, 1, True, None)     # bias + GELU, pre-activation copy
            e[f"{M}x{N}x{K}_bias_gelu"] = max(rel_err(pre, ref + b.float()), rel_err(yb, torch.nn.functional.gelu(ref + b.float())))
            yr, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, b, 0, False, r)
            e[f"{M}x{N}x{K}_residual"] = rel_err(yr, ref + b.float() + r.float())
            e[f"{M}x{N}x{K}_vs_bf16_gemm"] = rel_err(y, x.float() @ w.float().t())
            if M >= 8192:
                flops = 2.0 * M * N * K
                ms8 = timeit(lambda: ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, False, None))
                ms16 = timeit(lambda: ext.linear_fwd(x, w, None, 0, False))
                msq = timeit(lambda: ext.quantize_e4m3(x))
                res[f"{M}x{N}x{K}"] = {"fp8_ms": ms8, "fp8_pflops": flops / ms8 / 1e12, "bf16_ms": ms16,
                                       "bf16_pflops": flops / ms16 / 1e12, "quantize_x_ms": msq}
        vs_dequant = [v for k, v in e.items() if "x" in k and "vs_bf16" not in k and not k.startswith("quant")]
        ok = (max(vs_dequant) < 1e-2 and e["deq_scale"] < 1e-5 and e["quant_vs_torch"] < 1e-6 and e["quant_tail"] < 1e-6
              and e["quant_roundtrip"] < 0.06 and all(v < 0.08 for k, v in e.items() if "vs_bf16" in k))
        return {"ok": ok, "errs": e, "timing": res}

    record("fp8 forward GEMM", fp8_forward_gemm)

    # ------------------------------------------------------------------ norms
    for rms in (False, True):
        for H in (1024, 768, 4096, 200):
            for wdt in (torch.bfloat16, torch.float32):
                def norm(rms=rms, H=H, wdt=wdt):
                    x = torch.randn(777, H, device="cuda").bfloat16()
                    g = (1 + 0.1 * torch.randn(H, device="cuda")).to(wdt)
                    b = None if rms else (0.1 * torch.randn(H, device="cuda")).to(wdt)
                    y, mean, rstd = ext.norm_fwd(x, g, b, 1e-5, rms)
                    xf = x.float().requires_grad_(True)
                    gf = g.float().requires_grad_(True)
                    bf = None if b is None else b.float().requires_grad_(True)
                    if rms:
                        ref = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * gf
                    else:
                        ref = torch.nn.functional.layer_norm(xf, (H,), gf, bf, 1e-5)
                    gy = torch.randn_like(ref)
                    ref.backward(gy)
                    gx, dg, db = ext.norm_bwd(gy.bfloat16(), x, g, mean, rstd, rms, b is not None)
                    e = [rel_err(y, ref), rel_err(gx, xf.grad), rel_err(dg, gf.grad)]
                    if b is not None:
                        e.append(rel_err(db, bf.grad))
                    return {"ok": max(e) < 3e-2, "errs": e}

                record(f"norm rms={rms} H={H} w={str(wdt)[6:]}", norm)

    def norm_speed():
        x = torch.randn(8192, 1024, device="cuda").bfloat16()
        g = torch.ones(1024, device="cuda").bfloat16()
        b = torch.zeros(1024, device="cuda").bfloat16()
        ms = timeit(lambda: ext.norm_fwd(x, g, b, 1e-5, False))
        y, mean, rstd = ext.norm_fwd(x, g, b, 1e-5, False)
        msb = timeit(lambda: ext.norm_bwd(x, x, g, mean, rstd, False, True))
        nbytes = x.numel() * 2
        return {"fwd_ms": ms, "fwd_GBs": 2 * nbytes / ms / 1e6, "bwd_ms": msb, "bwd_GBs": 3 * nbytes / msb / 1e6}

    record("layernorm speed 8192x1024", norm_speed)

    # ------------------------------------------------------------------ elementwise
    def ew():
        x = torch.randn(1000, 4096, device="cuda").bfloat16()
        b = torch.randn(4096, device="cuda").bfloat16()
        r = torch.randn(1000, 4096, device="cuda").bfloat16()
        errs = []
        for act, name in ((1, "gelu"), (2, "gelu_tanh"), (3, "relu"), (4, "silu"), (5, "quick")):
            y = ext.bias_act_fwd(x, b, act)
            xf = (x.float() + b.float()).requires_grad_(True)
            ref = {1: torch.nn.functional.gelu(xf), 2: torch.nn.functional.gelu(xf, approximate="tanh"),
                   3: torch.relu(xf), 4: torch.nn.functional.silu(xf), 5: xf * torch.sigmoid(1.702 * xf)}[act]
            gy = torch.randn_like(ref)
            ref.backward(gy)
            gx = ext.bias_act_bwd(gy.bfloat16(), x, b, act)
            errs += [rel_err(y, ref), rel_err(gx, xf.grad)]
        y = ext.bias_residual_fwd(x, b, r)
        errs.append(rel_err(y, x.float() + b.float() + r.float()))
        cs = ext.colsum(x)
        errs.append(rel_err(cs, x.float().sum(0)))
        g, u = x, r
        y = ext.swiglu_fwd(g, u)
        gf, uf = g.float().requires_grad_(True), u.float().requires_grad_(True)
        ref = torch.nn.functional.silu(gf) * uf
        gy = torch.randn_like(ref)
        ref.backward(gy)
        dg, du = ext.swiglu_bwd(gy.bfloat16(), g, u)
        errs += [rel_err(y, ref), rel_err(dg, gf.grad), rel_err(du, uf.grad)]
        return {"ok": max(errs) < 3e-2, "errs": errs}

    record("elementwise", ew)

    def accum_grads():
        # bias / LayerNorm gradients accumulated straight into fp32 main-grad slices
        x = torch.randn(4096, 1024, device="cuda").bfloat16()
        acc = torch.full((1024,), 0.5, device="cuda")
        ext.colsum(x, acc)
        e = [rel_err(acc, x.float().sum(0) + 0.5)]
        g = (1 + 0.1 * torch.randn(1024, device="cuda")).bfloat16()
        b = (0.1 * torch.randn(1024, device="cuda")).bfloat16()
        y, mean, rstd = ext.norm_fwd(x, g, b, 1e-5, False)
        gy = torch.randn_like(x)
        gx0, dg0, db0 = ext.norm_bwd(gy, x, g, mean, rstd, False, True, None, None)
        dga = torch.full((1024,), 1.0, device="cuda")
        dba = torch.full((1024,), -2.0, device="cuda")
        gx1, _, _ = ext.norm_bwd(gy, x, g, mean, rstd, False, True, dga, dba)
        e += [rel_err(dga, dg0 + 1.0), rel_err(dba, db0 - 2.0), rel_err(gx1, gx0)]
        # skip-connection gradient folded into the LayerNorm backward (fast path H=1024; fallback path H=320)
        gskip = torch.randn_like(x)
        gx2, _, _ = ext.norm_bwd(gy, x, g, mean, rstd, False, True, None, None, gskip)
        e.append(rel_err(gx2, gx0.float() + gskip.float()))
        xs = torch.randn(512, 320, device="cuda").bfloat16()
        gs, bs = g[:320].contiguous(), b[:320].contiguous()
        _, mean_s, rstd_s = ext.norm_fwd(xs, gs, bs, 1e-5, False)
        gys, gsk = torch.randn_like(xs), torch.randn_like(xs)
        a0, _, _ = ext.norm_bwd(gys, xs, gs, mean_s, rstd_s, False, True, None, None)
        a1, _, _ = ext.norm_bwd(gys, xs, gs, mean_s, rstd_s, False, True, None, None, gsk)
        e.append(rel_err(a1, a0.float() + gsk.float()))
        # autograd level: (norm(x), x) with both outputs used == norm(x) and x used separately
        from libai_b200.ops import functional as OFn

        xa = x[:1024].clone().requires_grad_(True)
        xb = x[:1024].clone().requires_grad_(True)
        w1, w2 = torch.randn_like(xa), torch.randn_like(xa)
        ln, skip = OFn.layer_norm_with_skip(xa, g, b)
        ((ln.float() * w1.float()).sum() + (skip.float() * w2.float()).sum()).backward()
        ((OFn.layer_norm(xb, g, b).float() * w1.float()).sum() + (xb.float() * w2.float()).sum()).backward()
        e.append(rel_err(xa.grad, xb.grad))
        ms = timeit(lambda: ext.colsum(x, acc))
        x2 = torch.randn(8192, 4096, device="cuda").bfloat16()
        acc2 = torch.zeros(4096, device="cuda")
        ms2 = timeit(lambda: ext.colsum(x2, acc2))
        return {"ok": max(e) < 1e-2, "errs": e, "colsum_4096x1024_ms": ms, "colsum_8192x4096_ms": ms2,
                "colsum_8192x4096_GBs": x2.numel() * 2 / ms2 / 1e6}

    record("accumulating colsum / norm_bwd", accum_grads)

    def rope_qkv():
        from libai_b200.ops.functional import rotate_half

        b, sq, a, d, off = 2, 96, 4, 64, 5
        qkv = torch.randn(b, sq, a, 3 * d, device="cuda").bfloat16()
        pos = torch.arange(sq + off, device="cuda").float()
        inv = 1.0 / (10000 ** (torch.arange(0, d, 2, device="cuda").float() / d))
        fr = torch.outer(pos, inv)
        emb = torch.cat([fr, fr], -1)
        cos, sin = emb.cos().contiguous(), emb.sin().contiguous()
        y = ext.rope_qkv(qkv, cos, sin, off, False, False)
        c, s_ = cos[off:off + sq, None, :], sin[off:off + sq, None, :]
        qf = qkv.float()
        q, k, v = qf[..., :d], qf[..., d:2 * d], qf[..., 2 * d:]
        ref = torch.cat([q * c + rotate_half(q) * s_, k * c + rotate_half(k) * s_, v], -1)
        back = ext.rope_qkv(y.clone(), cos, sin, off, True, True)  # inverse rotation in place
        e = [rel_err(y, ref), rel_err(back, qf)]
        return {"ok": max(e) < 2e-2, "errs": e}

    record("rope_qkv packed", rope_qkv)

    def rope_qkv_positions():
        from libai_b200.ops.functional import rotate_half

        b, sq, g, r, d = 2, 96, 2, 4, 128
        qkv = torch.randn(b, sq, g, r + 2, d, device="cuda").bfloat16()
        inv = 1.0 / (10000 ** (torch.arange(0, d, 2, device="cuda").float() / d))
        fr = torch.outer(torch.arange(sq, device="cuda").float(), inv)
        emb = torch.cat([fr, fr], -1)
        cos, sin = emb.cos().contiguous(), emb.sin().contiguous()
        pos = torch.randint(0, sq, (b, sq), device="cuda", dtype=torch.int32)
        y = ext.rope_qkv(qkv, cos, sin, 0, False, False, pos)
        c, s_ = cos[pos.long()][:, :, None, None], sin[pos.long()][:, :, None, None]
        qf = qkv.float().requires_grad_(True)
        qk = qf[..., :r + 1, :]
        ref = torch.cat([qk * c + rotate_half(qk) * s_, qf[..., r + 1:, :]], 3)
        gy = torch.randn_like(ref)
        ref.backward(gy)
        gx = ext.rope_qkv(gy.bfloat16(), cos, sin, 0, True, False, pos)
        e = [rel_err(y, ref.detach()), rel_err(gx, qf.grad)]
        return {"ok": max(e) < 2e-2, "errs": e}

    record("rope_qkv grouped, per-token positions (fwd + bwd)", rope_qkv_positions)

    # ------------------------------------------------------------------ cross entropy
    def ce():
        T, V = 513, 50304
        logits = (torch.randn(T, V, device="cuda") * 2).bfloat16()
        labels = torch.randint(0, V, (T,), device="cuda")
        mx, se, tgt = ext.ce_stats(logits, labels, 0)
        lf = logits.float().requires_grad_(True)
        ref = torch.nn.functional.cross_entropy(lf, labels, reduction="none")
        loss = mx + torch.log(se) - tgt
        gl = torch.rand(T, device="cuda")
        ref.backward(gl)
        d = ext.ce_bwd(logits.clone(), labels, mx + torch.log(se), gl, 0)
        e = [rel_err(loss, ref), rel_err(d, lf.grad)]
        ms = timeit(lambda: ext.ce_stats(logits, labels, 0))
        return {"ok": max(e) < 2e-2, "errs": e, "stats_ms": ms, "GBs": T * V * 2 / ms / 1e6}

    record("cross entropy", ce)

    # ------------------------------------------------------------------ adam
    def adam():
        n = 1 << 20
        p = torch.randn(n, device="cuda")
        g = torch.randn(n, device="cuda")
        m = torch.zeros(n, device="cuda")
        v = torch.zeros(n, device="cuda")
        lp = torch.empty(n, device="cuda", dtype=torch.bfloat16)
        pr = p.clone().requires_grad_(True)
        opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
        for step in (1, 2, 3):
            pr.grad = g.clone()
            opt.step()
            ext.fused_adamw(p, g, m, v, lp, torch.ones(1, device="cuda"), 1e-2, 0.9, 0.999, 1e-8, 0.01,
                            1 - 0.9 ** step, 1 - 0.999 ** step, True)
        e = [rel_err(p, pr.detach()), rel_err(lp, pr.detach())]
        sq = ext.sqnorm(g)
        e.append(abs(float(sq) - float((g * g).sum())) / float((g * g).sum()))
        ms = timeit(lambda: ext.fused_adamw(p, g, m, v, lp, torch.ones(1, device="cuda"), 1e-2, 0.9, 0.999, 1e-8, 0.01, 0.5, 0.5, True))
        return {"ok": e[0] < 1e-4 and e[1] < 1e-2 and e[2] < 1e-3, "errs": e, "ms": ms, "GBs": n * (4 * 7 + 2) / ms / 1e6}

    record("fused adamw + sqnorm", adam)

    # ------------------------------------------------------------------ attention
    from libai_b200.ops.functional import attention_ref

    for (B, A, S, D, causal) in [(2, 4, 256, 64, True), (2, 4, 256, 64, False), (1, 2, 384, 128, True),
                                 (2, 3, 200, 64, True), (1, 2, 1024, 64, True), (1, 2, 512, 128, False)]:
        def att(B=B, A=A, S=S, D=D, causal=causal):
            qkv = torch.randn(B, S, A, 3 * D, device="cuda").bfloat16()
            v4 = qkv.view(B, S, A, 3 * D).permute(0, 2, 1, 3)
            q, k, v = v4[..., :D], v4[..., D:2 * D], v4[..., 2 * D:]
            scale = 1.0 / math.sqrt(D)
            o, lse, _ = ext.attn_fwd(q, k, v, causal, scale, None)
            qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
            ref = attention_ref(qf, kf, vf, causal=causal, scale=scale, fill=-1e30)
            e = [rel_err(o, ref)]
            go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
            ref.backward(go.float())
            dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, causal, scale, None)
            e += [rel_err(dq, qf.grad), rel_err(dk, kf.grad), rel_err(dv, vf.grad)]
            return {"ok": max(e) < 3e-2, "errs": e}

        record(f"attention B{B} A{A} S{S} D{D} causal={causal}", att)

    def att_kvlens():
        B, A, S, D = 3, 2, 320, 64
        qkv = torch.randn(B, S, A, 3 * D, device="cuda").bfloat16()
        v4 = qkv.permute(0, 2, 1, 3)
        q, k, v = v4[..., :D], v4[..., D:2 * D], v4[..., 2 * D:]
        lens = torch.tensor([320, 200, 77], device="cuda", dtype=torch.int32)
        scale = 0.125
        o, lse, _ = ext.attn_fwd(q, k, v, False, scale, lens)
        qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
        mask = (torch.arange(S, device="cuda")[None, :] < lens[:, None])[:, None, None, :]
        ref = attention_ref(qf, kf, vf, causal=False, scale=scale, mask=mask, fill=-1e30)
        go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
        ref.backward(go.float())
        dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, False, scale, lens)
        e = [rel_err(o, ref), rel_err(dq, qf.grad), rel_err(dk, kf.grad), rel_err(dv, vf.grad)]
        return {"ok": max(e) < 3e-2, "errs": e}

    record("attention kv_lens (key padding)", att_kvlens)

    def att_bias():
        """Dense additive bias (T5 relative positions: [1, A, S, S] broadcast over the batch) fwd + bwd + dbias."""
        B, A, S, D = 2, 3, 256, 64
        qkv = torch.randn(B, S, A, 3 * D, device="cuda").bfloat16()
        v4 = qkv.permute(0, 2, 1, 3)
        q, k, v = v4[..., :D], v4[..., D:2 * D], v4[..., 2 * D:]
        bias = (torch.randn(1, A, S, S, device="cuda") * 2.0).bfloat16()
        o, lse, _ = ext.attn_fwd(q, k, v, False, 1.0, None, bias, None, 0.0, 0)
        qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
        bf = bias.float().detach().requires_grad_(True)
        ref = attention_ref(qf, kf, vf, causal=False, scale=1.0, bias=bf, fill=-1e30)
        go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
        ref.backward(go.float())
        dbias = torch.zeros(1, A, S, S, device="cuda")
        dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, False, 1.0, None, bias, None, dbias, 0.0, None)
        e = [rel_err(o, ref), rel_err(dq, qf.grad), rel_err(dk, kf.grad), rel_err(dv, vf.grad), rel_err(dbias, bf.grad)]
        # per-sample bias + causal through the autograd wrapper
        from libai_b200.ops import functional as OF
        bias2 = (torch.randn(B, A, S, S, device="cuda")).bfloat16().requires_grad_(True)
        q2, k2, v2 = (t.detach().contiguous().requires_grad_(True) for t in (q, k, v))
        o2 = OF.attention(q2, k2, v2, causal=True, scale=0.125, bias=bias2)
        o2.backward(go)
        q3, k3, v3, b3 = (t.detach().float().requires_grad_(True) for t in (q, k, v, bias2))
        r2 = attention_ref(q3, k3, v3, causal=True, scale=0.125, bias=b3, fill=-1e30)
        r2.backward(go.float())
        e += [rel_err(o2, r2), rel_err(q2.grad, q3.grad), rel_err(bias2.grad, b3.grad)]
        return {"ok": max(e) < 3e-2, "errs": e}

    record("attention dense bias (+dbias)", att_bias)

    def att_alibi():
        B, A, S, D = 2, 4, 384, 64
        qkv = torch.randn(B, S, A, 3 * D, device="cuda").bfloat16()
        v4 = qkv.permute(0, 2, 1, 3)
        q, k, v = v4[..., :D], v4[..., D:2 * D], v4[..., 2 * D:]
        slopes = torch.tensor([0.5, 0.25, 0.125, 0.0625], device="cuda")
        o, lse, _ = ext.attn_fwd(q, k, v, True, 0.125, None, None, slopes, 0.0, 0)
        rel = (torch.arange(S, device="cuda")[None, :] - torch.arange(S, device="cuda")[:, None]).float()
        bias = slopes[None, :, None, None] * rel[None, None]
        qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
        ref = attention_ref(qf, kf, vf, causal=True, scale=0.125, bias=bias, fill=-1e30)
        go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
        ref.backward(go.float())
        dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, True, 0.125, None, None, slopes, None, 0.0, None)
        e = [rel_err(o, ref), rel_err(dq, qf.grad), rel_err(dk, kf.grad), rel_err(dv, vf.grad)]
        return {"ok": max(e) < 3e-2, "errs": e}

    record("attention ALiBi slopes", att_alibi)

    def att_dropout():
        """Dropout inside the flash kernels: the mask is recovered exactly (q = k = 0 → uniform P, V = I) and the
        kernel's forward / backward are compared with the reference math using that very mask."""
        B, A, S, D, pdrop = 2, 2, 64, 64, 0.25
        eye = torch.eye(S, device="cuda").bfloat16()[None, None].expand(B, A, S, D).contiguous()
        zero = torch.zeros(B, A, S, D, device="cuda").bfloat16()
        torch.cuda.manual_seed(4321)
        om, _, st_m = ext.attn_fwd(zero, zero, eye, False, 1.0, None, None, None, pdrop, 3)
        keep = (om.float() > 0)
        inv_keep = 256.0 / (256.0 - round(pdrop * 256))
        frac = float(keep.float().mean())
        qkv = torch.randn(B, S, A, 3 * D, device="cuda").bfloat16()
        v4 = qkv.permute(0, 2, 1, 3)
        q, k, v = v4[..., :D], v4[..., D:2 * D], v4[..., 2 * D:]
        torch.cuda.manual_seed(4321)
        o, lse, st = ext.attn_fwd(q, k, v, False, 0.125, None, None, None, pdrop, 3)
        same_state = torch.equal(st, st_m)
        qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
        probs = torch.softmax(qf @ kf.transpose(-1, -2) * 0.125, dim=-1)
        ref = (probs * keep.float() * inv_keep) @ vf
        go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
        ref.backward(go.float())
        dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, False, 0.125, None, None, None, None, pdrop, st)
        e = [rel_err(o, ref), rel_err(dq, qf.grad), rel_err(dk, kf.grad), rel_err(dv, vf.grad)]
        # another TP salt → another mask; statistics on a long sequence (causal, ragged)
        torch.cuda.manual_seed(4321)
        om2, _, _ = ext.attn_fwd(zero, zero, eye, False, 1.0, None, None, None, pdrop, 4)
        differs = float(((om2.float() > 0) != keep).float().mean())
        return {"ok": max(e) < 3e-2 and abs(frac - (1 - round(pdrop * 256) / 256)) < 0.02 and same_state and differs > 0.2,
                "errs": e, "keep_fraction": frac, "mask_differs_across_salts": differs, "same_rng_state": same_state}

    record("attention dropout (exact mask)", att_dropout)

    def dropout_ew():
        """bias + dropout + residual kernel: exact mask recovery, backward with the stored state, salts, statistics."""
        M, N, pdrop = 512, 1024, 0.1
        ones = torch.ones(M, N, device="cuda").bfloat16()
        torch.cuda.manual_seed(99)
        ym, st_m = ext.bias_dropout_residual(ones, None, None, pdrop, 0, None)
        keep = ym.float() > 0
        scale = 65536.0 / (65536.0 - round(pdrop * 65536))
        x = torch.randn(M, N, device="cuda").bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        r = torch.randn(M, N, device="cuda").bfloat16()
        torch.cuda.manual_seed(99)
        y, st = ext.bias_dropout_residual(x, b, r, pdrop, 0, None)
        ref = r.float() + (x.float() + b.float()) * keep.float() * scale
        gy = torch.randn(M, N, device="cuda").bfloat16()
        gx, _ = ext.bias_dropout_residual(gy, None, None, pdrop, 0, st)
        e = [rel_err(y, ref), rel_err(gx, gy.float() * keep.float() * scale)]
        torch.cuda.manual_seed(99)
        y2, _ = ext.bias_dropout_residual(ones, None, None, pdrop, 2, None)
        differs = float(((y2.float() > 0) != keep).float().mean())
        frac = float(keep.float().mean())
        # consecutive calls advance the generator offset: different masks
        y3, _ = ext.bias_dropout_residual(ones, None, None, pdrop, 0, None)
        y4, _ = ext.bias_dropout_residual(ones, None, None, pdrop, 0, None)
        adv = float(((y3.float() > 0) != (y4.float() > 0)).float().mean())
        ms = timeit(lambda: ext.bias_dropout_residual(x, b, r, pdrop, 0, None))
        big = torch.randn(8192, 1024, device="cuda").bfloat16()
        ms_big = timeit(lambda: ext.bias_dropout_residual(big, b, big, pdrop, 0, None))
        ms_nodrop = timeit(lambda: ext.bias_residual_fwd(big, b, big))
        return {"ok": max(e) < 1e-2 and abs(frac - 0.9) < 0.01 and differs > 0.1 and adv > 0.1, "errs": e, "keep_fraction": frac,
                "mask_differs_across_salts": differs, "mask_differs_across_calls": adv, "ms_8192x1024": ms_big,
                "ms_8192x1024_without_dropout": ms_nodrop, "gbs": 3 * big.numel() * 2 / ms_big / 1e6}

    record("bias+dropout+residual (Philox)", dropout_ew)

    def dropout_graph():
        """Captured dropout draws a fresh mask on every replay (PyTorch refreshes the Philox offset of the graph)."""
        ones = torch.ones(256, 1024, device="cuda").bfloat16()
        for _ in range(2):
            ext.bias_dropout_residual(ones, None, None, 0.5, 0, None)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y, st = ext.bias_dropout_residual(ones, None, None, 0.5, 0, None)
            gx, _ = ext.bias_dropout_residual(ones, None, None, 0.5, 0, st)
        masks = []
        consistent = True
        for _ in range(3):
            g.replay()
            torch.cuda.synchronize()
            masks.append(y.float() > 0)
            consistent = consistent and torch.equal(y, gx)       # backward regenerates the forward's mask
        d01 = float((masks[0] != masks[1]).float().mean())
        d12 = float((masks[1] != masks[2]).float().mean())
        return {"ok": d01 > 0.3 and d12 > 0.3 and consistent, "replay_mask_diff": [d01, d12], "fwd_bwd_consistent": consistent}

    record("dropout inside a CUDA graph", dropout_graph)

    if not args.quick:
        def att_speed():
            B, A, S, D = 8, 16, 1024, 64
            qkv = torch.randn(B, S, A, 3 * D, device="cuda").bfloat16()
            v4 = qkv.permute(0, 2, 1, 3)
            q, k, v = v4[..., :D], v4[..., D:2 * D], v4[..., 2 * D:]
            scale = 0.125
            ms = timeit(lambda: ext.attn_fwd(q, k, v, True, scale, None))
            o, lse, _ = ext.attn_fwd(q, k, v, True, scale, None)
            go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
            msb = timeit(lambda: ext.attn_bwd(go, q, k, v, o, lse, True, scale, None))
            flops = 4.0 * B * A * S * S * D / 2
            qc, kc, vc = q.contiguous(), k.contiguous(), v.contiguous()
            sd = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qc, kc, vc, is_causal=True))
            qg, kg, vg = (t.detach().clone().requires_grad_(True) for t in (qc, kc, vc))
            og = torch.nn.functional.scaled_dot_product_attention(qg, kg, vg, is_causal=True)
            gog = torch.randn_like(og)
            sdb = timeit(lambda: torch.autograd.grad(og, (qg, kg, vg), gog, retain_graph=True))
            msd = timeit(lambda: ext.attn_fwd(q, k, v, True, scale, None, None, None, 0.1, 0))
            od, lsed, std = ext.attn_fwd(q, k, v, True, scale, None, None, None, 0.1, 0)
            msbd = timeit(lambda: ext.attn_bwd(go, q, k, v, od, lsed, True, scale, None, None, None, None, 0.1, std))
            return {"fwd_ms": ms, "fwd_tflops": flops / ms / 1e9, "bwd_ms": msb, "bwd_tflops": 2.5 * flops / msb / 1e9,
                    "sdpa_fwd_ms": sd, "sdpa_bwd_ms": sdb, "fwd_ms_dropout0.1": msd, "bwd_ms_dropout0.1": msbd}

        record("attention speed B8 A16 S1024 D64 causal", att_speed)

    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(RESULTS, f, indent=1)
    bad = [r["name"] for r in RESULTS if not r.get("ok", False)]
    print(f"SUMMARY: {len(RESULTS) - len(bad)}/{len(RESULTS)} ok; failed: {bad}")


if __name__ == "__main__":
    main()
