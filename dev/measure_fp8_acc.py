"""Measures how many bits the accumulator of the fp8 (E4M3) forward GEMM keeps.  The result backs FP8_ACC in
tests/train_ref.py.

Cancellation probe: ``linear_fp8_fwd`` with deq = 1 on operands where row i / column j hold three products, a large
+2^(i+j-16), the small 2^-18 and -2^(i+j-16), at positions ``(big, small, -big)`` along K.  The exact result is the
small product, a power of two that bf16 holds exactly; it survives only while the accumulator keeps log2(large / small)
bits below the large product's leading bit.  The three
positions put the products inside one 32-wide k-step (one wgmma), in different k-steps of one 128-wide k-block, and in
different k-blocks; "small first" adds the small product to an empty accumulator before the large pair arrives.

Model-K probe: random E4M3 operands at K 1024 and 4096 through the fp8 GEMM and, as bf16 values (exact: every E4M3
value is a bf16 value), through the bf16 GEMM, whose accumulator is fp32.  Both are compared with the correctly rounded
bf16 of the exact fp64 result.

Usage: python dev/measure_fp8_acc.py (needs a GPU and the built extension)."""
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = {           # (position of +big, of the small product, of -big) along K
    "one k-step": (0, 1, 2),
    "across k-steps of one k-block": (0, 32, 64),
    "across k-blocks": (0, 128, 256),
    "small first, across k-steps": (32, 0, 64),
    "small first, across k-blocks": (128, 0, 256),
}


def card():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return f"{name}, power limit {limit}"


def cancellation(ext, pos, K=512, rows=17, cols=24):
    """Row i, column j: products +2^(i+j-16), 2^-18 and -2^(i+j-16) at the K positions ``pos``; the exact result 2^-18
    lies 2^(i+j+2) below the large products."""
    big, small, neg = pos
    x = torch.zeros(rows, K, dtype=torch.float64)
    w = torch.zeros(cols, K, dtype=torch.float64)
    ei = torch.arange(rows, dtype=torch.float64)
    ej = torch.arange(cols, dtype=torch.float64).clamp(max=16)
    x[:, big] = x[:, neg] = 2.0 ** (ei - 8)
    w[:, big] = 2.0 ** (ej - 8)
    w[:, neg] = -(2.0 ** (ej - 8))
    x[:, small] = 2.0 ** -9                   # the smallest E4M3 value (subnormal)
    w[:, small] = 2.0 ** -9
    xq = x.to(torch.float8_e4m3fn).cuda()
    wq = w.to(torch.float8_e4m3fn).cuda()
    assert torch.equal(xq.double().cpu(), x) and torch.equal(wq.double().cpu(), w)
    one = torch.ones(1, device="cuda")
    y, _ = ext.linear_fp8_fwd(xq, wq, one, one, None, 0, False, None)
    want = x @ w.t()                          # 2^-18, exact in bf16
    got = y.double().cpu()
    ratio = ei[:, None] + ej[None, :] + 2     # log2(large / small)
    kept = ratio[got == want]
    lost = ratio[got != want]
    return (int(kept.max()) if kept.numel() else None, int(lost.min()) if lost.numel() else None,
            sorted({float(v) for v in (got[got != want] / want[got != want]).reshape(-1).tolist()}))


def model_k(ext, M, N, K, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = torch.randn(N, K, device="cuda", generator=g).bfloat16()
    xq, _ = ext.quantize_e4m3(x)
    wq, _ = ext.quantize_e4m3(w)
    one = torch.ones(1, device="cuda")
    y8, _ = ext.linear_fp8_fwd(xq, wq, one, one, None, 0, False, None)
    y16, _ = ext.linear_fwd(xq.bfloat16(), wq.bfloat16(), None, 0, False)
    a, b = xq.double(), wq.double()
    exact = a @ b.t()
    terms = a.abs() @ b.abs().t()
    rne = exact.bfloat16().double()
    out = {}
    for name, y in (("fp8 GEMM", y8), ("bf16 GEMM (fp32 accumulator)", y16)):
        err = (y.double() - exact).abs()
        out[name] = dict(differs_from_rne=float((y.double() != rne).double().mean()),
                         max_err_over_sum_abs_terms=float((err / terms).max()),
                         median_err_over_abs_result=float((err / exact.abs().clamp(min=1e-30)).median()))
    return out


def main():
    from libai_b200 import ops

    ext = ops.load_ext(required=True)
    print(card())
    for name, pos in CASES.items():
        kept, lost, ratios = cancellation(ext, pos)
        print(f"cancellation, {name}: small product survives up to 2^{kept} below the large ones, "
              f"first lost at 2^{lost}; lost values came out as {ratios} x the exact one")
    for K in (1024, 4096):
        for name, r in model_k(ext, 1024, 1024, K).items():
            print(f"random E4M3 operands, M = N = 1024, K = {K}, {name}: {r['differs_from_rne'] * 100:.2f} % of outputs "
                  f"differ from the correctly rounded bf16; max |err| / sum|terms| = "
                  f"2^{math.log2(max(r['max_err_over_sum_abs_terms'], 1e-300)):.2f}; median |err| / |result| = "
                  f"2^{math.log2(max(r['median_err_over_abs_result'], 1e-300)):.2f}")


if __name__ == "__main__":
    main()
