"""Attention kernel development loop: numerics against the fp32 reference on a few shapes, then CUDA-event timings of
the benchmark shape (B8 H16 S1024 D64 causal) next to PyTorch SDPA (cuDNN / flash); the backward is timed with its
delta and dQ-convert kernels, under an L2 flush, and reported in TFLOP/s of its MMA work too.  `python dev/attn_dev.py [--ncu]`
(--ncu: three launches of each kernel only, for `ncu -k regex:attn_`)."""
import json
import math
import sys

import torch

sys.path.insert(0, ".")
from libai_b200.ops import load_ext
from libai_b200.ops.functional import attention_ref

ext = load_ext()


def rel_err(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6))


def timeit(fn, iters=50, warmup=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    flush = torch.empty(160 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def inputs(B, A, S, D):
    qkv = torch.randn(B, S, A, 3 * D, device="cuda").bfloat16()
    v4 = qkv.permute(0, 2, 1, 3)
    return v4[..., :D], v4[..., D:2 * D], v4[..., 2 * D:]


def main():
    torch.manual_seed(0)
    if "--ncu" in sys.argv:
        q, k, v = inputs(8, 16, 1024, 64)
        go = torch.randn(8, 1024, 16, 64, device="cuda").bfloat16().permute(0, 2, 1, 3)
        for _ in range(3):
            o, lse, _ = ext.attn_fwd(q, k, v, True, 0.125, None)
            ext.attn_bwd(go, q, k, v, o, lse, True, 0.125, None)
        torch.cuda.synchronize()
        return
    out = {"numerics": []}
    for (B, A, S, D, causal) in [] if "--speed-only" in sys.argv else [(2, 4, 256, 64, True), (2, 4, 256, 64, False), (2, 3, 200, 64, True), (1, 2, 1024, 64, True),
                                 (1, 2, 384, 128, True), (2, 2, 1024, 64, False)]:
        q, k, v = inputs(B, A, S, D)
        scale = 1.0 / math.sqrt(D)
        o, lse, _ = ext.attn_fwd(q, k, v, causal, scale, None)
        qf, kf, vf = (t.float().detach().requires_grad_(True) for t in (q, k, v))
        ref = attention_ref(qf, kf, vf, causal=causal, scale=scale, fill=-1e30)
        go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
        ref.backward(go.float())
        dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, causal, scale, None)
        e = [rel_err(o, ref), rel_err(dq, qf.grad), rel_err(dk, kf.grad), rel_err(dv, vf.grad)]
        out["numerics"].append({"shape": [B, A, S, D, causal], "errs": [round(x, 5) for x in e], "ok": max(e) < 3e-2})
    B, A, S, D = 8, 16, 1024, 64
    q, k, v = inputs(B, A, S, D)
    go = torch.randn(B, S, A, D, device="cuda").bfloat16().permute(0, 2, 1, 3)
    o, lse, _ = ext.attn_fwd(q, k, v, True, 0.125, None)
    qc, kc, vc = (t.contiguous().detach().requires_grad_(True) for t in (q, k, v))
    og = torch.nn.functional.scaled_dot_product_attention(qc, kc, vc, is_causal=True)
    gog = torch.randn_like(og)
    out["speed"] = {
        "fwd_ms": timeit(lambda: ext.attn_fwd(q, k, v, True, 0.125, None)),
        "bwd_ms": timeit(lambda: ext.attn_bwd(go, q, k, v, o, lse, True, 0.125, None)),
        "sdpa_fwd_ms": timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qc, kc, vc, is_causal=True)),
        "sdpa_bwd_ms": timeit(lambda: torch.autograd.grad(og, (qc, kc, vc), gog, retain_graph=True)),
    }
    # the backward's tensor-core work: 5 MMAs of 64 x 64 x D per (64-key, 64-query) block pair the causal mask keeps
    nb = S // 64
    bwd_flop = B * A * nb * (nb + 1) // 2 * 5 * 2 * 64 * 64 * D
    out["speed"]["bwd_gflop"] = bwd_flop / 1e9
    out["speed"]["bwd_tflops"] = bwd_flop / (out["speed"]["bwd_ms"] * 1e-3) / 1e12
    props = torch.cuda.get_device_properties(0)
    out["device"] = props.name
    od, lsed, std = ext.attn_fwd(q, k, v, True, 0.125, None, None, None, 0.1, 0)
    out["speed"]["fwd_ms_dropout0.1"] = timeit(lambda: ext.attn_fwd(q, k, v, True, 0.125, None, None, None, 0.1, 0))
    out["speed"]["bwd_ms_dropout0.1"] = timeit(lambda: ext.attn_bwd(go, q, k, v, od, lsed, True, 0.125, None, None, None, None, 0.1, std))
    # Llama-like shape (head dim 128: the sequential backward kernel)
    q, k, v = inputs(2, 8, 2048, 128)
    go = torch.randn(2, 2048, 8, 128, device="cuda").bfloat16().permute(0, 2, 1, 3)
    sc = 1.0 / math.sqrt(128)
    o, lse, _ = ext.attn_fwd(q, k, v, True, sc, None)
    qc, kc, vc = (t.contiguous().detach().requires_grad_(True) for t in (q, k, v))
    og = torch.nn.functional.scaled_dot_product_attention(qc, kc, vc, is_causal=True)
    gog = torch.randn_like(og)
    out["speed_B2_H8_S2048_D128"] = {
        "fwd_ms": timeit(lambda: ext.attn_fwd(q, k, v, True, sc, None)),
        "bwd_ms": timeit(lambda: ext.attn_bwd(go, q, k, v, o, lse, True, sc, None)),
        "sdpa_fwd_ms": timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qc, kc, vc, is_causal=True)),
        "sdpa_bwd_ms": timeit(lambda: torch.autograd.grad(og, (qc, kc, vc), gog, retain_graph=True)),
    }
    out["ok"] = all(x["ok"] for x in out["numerics"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
