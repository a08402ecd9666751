"""FP8 (E4M3) weights for generate(): the weight-streaming kernel and the end-to-end effect on a Llama-7B-shaped model.

    python dev/fp8_weights_bench.py [--quick] [--out output/fp8_weights_bench.json]

Kernel level: Llama-7B's projections (K, N) = (4096, 12288), (4096, 4096), (4096, 11008), (11008, 4096) and
GPT-2-medium's (1024, 3072 + bias), (1024, 4096 + bias + GELU), (4096, 1024), at M = 1, 4, 16, 32, 48, 64 rows.  Median
microseconds over CUDA events with the L2 flushed before every launch, for: the FP8 kernel (``ext.linear_fp8w``); the
prefill path over the same FP8 weight (``dequant_e4m3_rows`` + ``ext.linear_fwd``), whose comparison with the kernel
sets ``OF.FP8W_KERNEL_MAX_M``; and, over the bf16 weight, today's path (``ext.linear_fwd``) and cuBLAS
(``torch.nn.functional.linear``).  Bytes: weights + scales + x + y (+ bias), as GB/s and as a share of 3.35 TB/s.

End to end: ``generate()`` on a randomly initialised Llama-7B-shaped model (32 layers), a 512-token prompt and 256 new
tokens at batch 1 and 16, bf16 weights and FP8 weights (a second copy of the same model, quantized) alternated in one
launch.  New tokens/s, the prefill's time (one forward over the prompt), the weights' bytes and the peak memory
allocated during the call on top of what was allocated before it.  The card name, power limit and SM clock are printed
with the figures and stored in the JSON output.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "dev"))

from decode_bench import gpu_info, llama_7b, time_us  # noqa: E402
from libai_b200.inference import quantize_weights_fp8_  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = [("llama-7b qkv", 4096, 12288, False, None), ("llama-7b o_proj", 4096, 4096, False, None),
          ("llama-7b gate/up", 4096, 11008, False, None), ("llama-7b down", 11008, 4096, False, None),
          ("gpt2-medium qkv", 1024, 3072, True, None), ("gpt2-medium h_to_4h", 1024, 4096, True, "gelu"),
          ("gpt2-medium 4h_to_h", 4096, 1024, False, None)]
MS = (1, 4, 16, 32, 48, 64)


def kernel_level(ext, quick):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for name, K, N, has_bias, act in (SHAPES[:2] + SHAPES[4:5] if quick else SHAPES):
        g = torch.Generator(device="cuda").manual_seed(K + N)
        wb = (torch.randn(N, K, device="cuda", generator=g) * 0.02).bfloat16()
        e, s = OF.kv_cache_quantize_ref(wb)
        b = (torch.randn(N, device="cuda", generator=g) * 0.1).bfloat16() if has_bias else None
        a = OF._ACT_IDS[act]
        for M in ((1, 16, 32, 64) if quick else MS):
            x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
            deq = (e.float() * s[:, None]).to(torch.bfloat16)
            y8 = ext.linear_fp8w(x, e, s, b, a)
            ref = F.linear(x.float(), deq.float(), None if b is None else b.float())
            ref = OF._act_ref(ref, act)
            err = float((y8.float() - ref).abs().max() / ref.abs().max())
            t_fp8 = time_us(lambda: ext.linear_fp8w(x, e, s, b, a), 50, flush)
            t_deq = time_us(lambda: ext.linear_fwd(x, ext.dequant_e4m3_rows(e, s), b, a, False), 50, flush)
            t_bf16 = time_us(lambda: ext.linear_fwd(x, wb, b, a, False), 50, flush)
            t_cublas = time_us(lambda: F.linear(x, wb, b), 50, flush)
            io = M * K * 2 + M * N * 2 + (2 * N if has_bias else 0)
            b8, b16 = N * K + 4 * N + io, 2 * N * K + io
            r = dict(shape=name, K=K, N=N, bias=has_bias, act=act, M=M, fp8_us=t_fp8, dequant_gemm_us=t_deq,
                     bf16_linear_fwd_us=t_bf16, cublas_bf16_us=t_cublas, fp8_bytes=b8, bf16_bytes=b16,
                     fp8_GBps=b8 / t_fp8 / 1e3, fp8_hbm_share=b8 / (t_fp8 * 1e-6) / HBM_BYTES_PER_S,
                     bf16_linear_fwd_GBps=b16 / t_bf16 / 1e3, cublas_GBps=b16 / t_cublas / 1e3,
                     fp8_vs_bf16_linear_fwd=t_bf16 / t_fp8, fp8_vs_dequant_gemm=t_deq / t_fp8,
                     fp8_rel_err_vs_fp32=err)
            rows.append(r)
            print(json.dumps(r), flush=True)
        del wb, e, s, deq
        torch.cuda.empty_cache()
    return rows


def end_to_end(quick):
    layers = 4 if quick else 32
    prompt, new = (128, 32) if quick else (512, 256)
    models = {"bf16": llama_7b(layers), "fp8": quantize_weights_fp8_(llama_7b(layers))}
    weight_bytes = {k: sum(p.numel() * p.element_size() for p in m.parameters()) for k, m in models.items()}
    print(json.dumps(dict(weights_bytes=weight_bytes)), flush=True)
    rows = []
    for B in (1, 16):
        ids = torch.randint(3, 32000, (B, prompt), device="cuda", generator=torch.Generator("cuda").manual_seed(B))
        res = {}
        for rep in range(3):                     # alternate the two models; the first round is the warm-up
            for name, m in models.items():
                m.kv_cache = None
                torch.cuda.empty_cache()
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                with torch.no_grad():
                    m.allocate_kv_cache(B, prompt)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    m(ids, use_cache=True)
                    torch.cuda.synchronize()
                    t_prefill = time.perf_counter() - t0
                    m.set_cache(None)
                    t0 = time.perf_counter()
                    seqs = m.generate(ids, max_new_tokens=new, eos_token_id=None, pad_token_id=0)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                peak = torch.cuda.max_memory_allocated() - base
                if rep > 0:
                    res.setdefault(name, []).append(dict(seconds=dt, new_tokens_per_s=B * new / dt,
                                                         prefill_ms=t_prefill * 1e3, peak_extra_gb=peak / 1e9))
                res[name + "_seqs"] = seqs
        agree = float((res["bf16_seqs"][:, prompt:] == res["fp8_seqs"][:, prompt:]).float().mean())
        r = dict(layers=layers, B=B, prompt=prompt, new_tokens=new, bf16=res["bf16"], fp8=res["fp8"],
                 weights_bytes=weight_bytes, token_agreement=agree,
                 fp8_speedup=[b["seconds"] / f["seconds"] for b, f in zip(res["bf16"], res["fp8"])])
        rows.append(r)
        print(json.dumps(r), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "fp8_weights_bench.json"))
    ap.add_argument("--quick", action="store_true", help="a subset of the sizes (a rehearsal, not a measurement)")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--skip-kernel", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_weights_bench needs a CUDA device")
    from libai_b200 import ops
    from libai_b200.config import DictConfig
    from libai_b200.utils import distributed as dist

    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    ext = ops.load_ext(required=True)
    info = gpu_info()
    print(json.dumps(info), flush=True)
    result = dict(info, kernel_max_m=OF.FP8W_KERNEL_MAX_M, kernel=[] if a.skip_kernel else kernel_level(ext, a.quick))
    result["e2e"] = [] if a.skip_e2e else end_to_end(a.quick)
    result["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
