"""Tile-N sweep of the forward (NT) and dgrad (NN) GEMMs on the benchmark model's shapes: does the heuristic of
gemm_sm90.cu (bn = 0) pick the fastest tile?"""
import json
import sys

import torch

sys.path.insert(0, ".")
from libai_b200.ops import load_ext  # noqa: E402


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


def main():
    ext = load_ext()
    out = {}
    shapes = [("fwd_qkv", 0, 8192, 3072, 1024), ("fwd_proj", 0, 8192, 1024, 1024), ("fwd_fc1", 0, 8192, 4096, 1024),
              ("fwd_fc2", 0, 8192, 1024, 4096), ("dgrad_qkv", 1, 8192, 1024, 3072), ("dgrad_proj", 1, 8192, 1024, 1024),
              ("dgrad_fc2", 1, 8192, 4096, 1024), ("dgrad_fc1", 1, 8192, 1024, 4096)]
    for name, layout, M, N, K in shapes:
        a = torch.randn(M, K, device="cuda").bfloat16()
        b = (torch.randn(N, K, device="cuda") if layout == 0 else torch.randn(K, N, device="cuda")).bfloat16()
        res = {}
        for bn in (0, 128, 192, 256):
            try:
                res[f"bn{bn}"] = round(timeit(lambda: ext.gemm_tuned(a, b, layout, bn, 1, False)), 4)
            except Exception as e:  # noqa: BLE001
                res[f"bn{bn}"] = f"{type(e).__name__}"
        res["cublas"] = round(timeit(lambda: torch.matmul(a, b.t() if layout == 0 else b)), 4)
        out[name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
