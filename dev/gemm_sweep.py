"""Tile-N sweep of every GEMM of the benchmark model's training step (GPT-2 medium, micro-batch 8 x 1024 tokens): does
the heuristic of gemm_sm90.cu (bn = 0) pick the fastest tile, and how far is each shape from cuBLAS?

For the NT and NN layouts `pingpong` is the ping-pong kernel (128 x 128 tiles, what the dispatch runs for bf16 outputs)
and `bn*` the 288-thread kernel at each width, forced with `gemm_schedule(1)`.  `epilogues` times the fused epilogues
the step runs at K = 1024 (fc1 forward with bias + GELU + pre-activation copy, attention-out and fc2 forward with bias
+ residual, the fc2 dgrad fused with GELU') with both kernels.

Shapes: forward NT and dgrad NN of the four transformer linears, their wgrad TN with the fp32 `red.add` epilogue into
a main_grad buffer, and the LM head's forward, dgrad and wgrad.  Prints one JSON line: per shape the median time (ms)
and TFLOP/s (2·M·N·K over time) of each tile width and of torch.matmul (cuBLAS) on the same operands.  The forced tile
widths of the wgrad go through `gemm_tuned`, which also zero-fills the fp32 output (M·N·4 bytes) inside the timed
region; `bn0` of the wgrad accumulates into an existing buffer, as the training step does.  cuBLAS writes bf16."""
import json
import sys

import torch

sys.path.insert(0, ".")
from libai_b200.ops import load_ext  # noqa: E402

T, H, FFN, VOCAB = 8192, 1024, 4096, 50304

# (name, layout, M, N, K); layout 0 = NT (A[M,K], B[N,K]), 1 = NN (A[M,K], B[K,N]), 2 = TN (A[K,M], B[K,N])
SHAPES = [
    ("fwd_qkv", 0, T, 3 * H, H), ("fwd_proj", 0, T, H, H), ("fwd_fc1", 0, T, FFN, H), ("fwd_fc2", 0, T, H, FFN),
    ("dgrad_qkv", 1, T, H, 3 * H), ("dgrad_proj", 1, T, H, H), ("dgrad_fc2", 1, T, FFN, H), ("dgrad_fc1", 1, T, H, FFN),
    ("wgrad_qkv", 2, 3 * H, H, T), ("wgrad_proj", 2, H, H, T), ("wgrad_fc1", 2, FFN, H, T), ("wgrad_fc2", 2, H, FFN, T),
    ("lmhead_fwd", 0, T, VOCAB, H), ("lmhead_dgrad", 1, T, H, VOCAB), ("lmhead_wgrad", 2, VOCAB, H, T),
]


def timeit(fn, iters=40, warmup=8):
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


def operands(layout, M, N, K):
    a = (torch.randn(K, M, device="cuda") if layout == 2 else torch.randn(M, K, device="cuda")).bfloat16()
    b = (torch.randn(N, K, device="cuda") if layout == 0 else torch.randn(K, N, device="cuda")).bfloat16()
    return a, b


def main():
    ext = load_ext()
    torch.manual_seed(0)
    out = {}
    for name, layout, M, N, K in SHAPES:
        a, b = operands(layout, M, N, K)
        flop = 2.0 * M * N * K
        res = {"shape": [M, N, K]}

        def record(key, ms):
            res[key] = {"ms": round(ms, 4), "tflops": round(flop / (ms * 1e-3) / 1e12, 1)}

        if layout == 2:
            main_grad = torch.zeros(M, N, device="cuda")
            record("bn0", timeit(lambda: ext.gemm(a, b, 2, None, main_grad, True, torch.float32)))
        if layout != 2:
            record("pingpong", timeit(lambda: ext.gemm_tuned(a, b, layout, 128, 1, False)))
        prev = ext.gemm_schedule(1)
        for bn in (0, 64, 128, 192, 256) if layout != 2 else (64, 128, 192, 256):
            try:
                record(f"bn{bn}", timeit(lambda: ext.gemm_tuned(a, b, layout, bn, 0 if layout == 2 else 1, False)))
            except Exception as e:  # noqa: BLE001
                res[f"bn{bn}"] = f"{type(e).__name__}"
        ext.gemm_schedule(prev)
        if layout == 0:
            record("cublas", timeit(lambda: torch.matmul(a, b.t())))
        elif layout == 1:
            record("cublas", timeit(lambda: torch.matmul(a, b)))
        else:
            record("cublas", timeit(lambda: torch.matmul(a.t(), b)))
        out[name] = res
        del a, b
        torch.cuda.empty_cache()
    out["epilogues"] = epilogues(ext)
    print(json.dumps(out))


def epilogues(ext):
    x, x4 = torch.randn(T, H, device="cuda").bfloat16(), torch.randn(T, FFN, device="cuda").bfloat16()
    w_fc1, w_proj = torch.randn(FFN, H, device="cuda").bfloat16(), torch.randn(H, H, device="cuda").bfloat16()
    w_fc2 = torch.randn(H, FFN, device="cuda").bfloat16()
    b_fc1, b_h = torch.randn(FFN, device="cuda").bfloat16(), torch.randn(H, device="cuda").bfloat16()
    res, gy = torch.randn(T, H, device="cuda").bfloat16(), torch.randn(T, H, device="cuda").bfloat16()
    cases = {
        "fwd_fc1_bias_gelu_pre": ([T, FFN, H], lambda: ext.linear_fwd(x, w_fc1, b_fc1, 1, True)),
        "fwd_proj_bias_residual": ([T, H, H], lambda: ext.linear_bias_residual(x, w_proj, b_h, res)),
        "fwd_fc2_bias_residual": ([T, H, FFN], lambda: ext.linear_bias_residual(x4, w_fc2, b_h, res)),
        "dgrad_fc2_gelu_grad": ([T, FFN, H], lambda: ext.dgrad_actgrad(gy, w_fc2, x4, 1, None)),
    }
    out = {}
    for name, ((M, N, K), fn) in cases.items():
        flop = 2.0 * M * N * K
        res_ = {"shape": [M, N, K]}
        for key, schedule in (("pingpong", 0), ("old", 1)):
            prev = ext.gemm_schedule(schedule)
            ms = timeit(fn)
            ext.gemm_schedule(prev)
            res_[key] = {"ms": round(ms, 4), "tflops": round(flop / (ms * 1e-3) / 1e12, 1)}
        out[name] = res_
    return out


if __name__ == "__main__":
    main()
