"""INT4 weights for generate(): the weight-streaming kernel, the end-to-end effect on a Llama-7B-shaped model, and the
logit error of quantized weights.

    python dev/int4_weights_bench.py [--quick] [--out output/int4_weights_bench.json]

Kernel level: the shapes of dev/fp8_weights_bench.py (Llama-7B's four projections and GPT-2 medium's three) at M = 1, 4,
16, 32, 48, 64 rows.  Median microseconds over CUDA events with the L2 flushed before every launch, for five paths on
the same random weight, in one launch: the INT4 kernel (``ext.linear_int4w``); the INT4 prefill path
(``dequant_int4_rows`` + ``ext.linear_fwd``), whose comparison with the kernel sets ``OF.INT4W_KERNEL_MAX_M``; the FP8
kernel (``ext.linear_fp8w``); and, over the bf16 weight, ``ext.linear_fwd`` and cuBLAS (``torch.nn.functional.linear``).
Bytes: weights + scales (+ zeros) + x + y (+ bias), as GB/s and as a share of 3.35 TB/s.

End to end: ``generate(decode_graphs=True)`` on randomly initialised Llama-7B-shaped models (32 layers), a 512-token
prompt and 256 new tokens at batch 1 and 16.  Four configurations, alternated round by round (the first round is the
warm-up): bf16 weights, FP8 weights with an FP8 cache, INT4 weights, and INT4 weights with an FP8 cache.  New tokens/s,
the device time per decode step ((generate − prefill) / (new − 1), CUDA events), the weights' bytes and the peak memory
allocated during the call on top of what was allocated before it.

Accuracy: teacher-forced logits of a 512-token prompt with FP8 and INT4 weights against the bf16 model, as the relative
Frobenius error.  The weights are random Gaussians, so these figures say nothing about quality on trained checkpoints.

The card name, power limit and SM clock are printed with the figures and stored in the JSON output.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "dev"))

from decode_bench import gpu_info, llama_7b, time_us  # noqa: E402
from fp8_weights_bench import HBM_BYTES_PER_S, MS, SHAPES  # noqa: E402
from libai_b200.inference import quantize_weights_fp8_, quantize_weights_int4_  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402


def kernel_level(ext, quick):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for name, K, N, has_bias, act in (SHAPES[:2] + SHAPES[4:5] if quick else SHAPES):
        g = torch.Generator(device="cuda").manual_seed(K + N)
        wb = (torch.randn(N, K, device="cuda", generator=g) * 0.02).bfloat16()
        q, s, z = OF.int4_quantize_ref(wb)
        e, s8 = OF.kv_cache_quantize_ref(wb)
        deq = OF.int4_dequant_ref(q, s, z)
        b = (torch.randn(N, device="cuda", generator=g) * 0.1).bfloat16() if has_bias else None
        a = OF._ACT_IDS[act]
        for M in ((1, 16, 64) if quick else MS):
            x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
            y4 = ext.linear_int4w(x, q, s, z, b, a)
            ref = OF._act_ref(F.linear(x.float(), deq.float(), None if b is None else b.float()), act)
            err = float((y4.float() - ref).abs().max() / ref.abs().max())
            t = {}
            for rep in range(2):   # the five paths alternate twice; each figure is the median of the two
                for k, fn in (("int4", lambda: ext.linear_int4w(x, q, s, z, b, a)),
                              ("int4_dequant_gemm", lambda: ext.linear_fwd(x, ext.dequant_int4_rows(q, s, z), b, a,
                                                                           False)),
                              ("fp8", lambda: ext.linear_fp8w(x, e, s8, b, a)),
                              ("bf16_linear_fwd", lambda: ext.linear_fwd(x, wb, b, a, False)),
                              ("cublas_bf16", lambda: F.linear(x, wb, b))):
                    t.setdefault(k, []).append(time_us(fn, 50, flush))
            t = {k: statistics.median(v) for k, v in t.items()}
            io = M * K * 2 + M * N * 2 + (2 * N if has_bias else 0)
            by = dict(int4=N * K // 2 + 3 * N * (K // 128) + io, fp8=N * K + 4 * N + io, bf16=2 * N * K + io)
            by.update(int4_dequant_gemm=by["int4"], bf16_linear_fwd=by["bf16"], cublas_bf16=by["bf16"])
            r = dict(shape=name, K=K, N=N, bias=has_bias, act=act, M=M, int4_rel_err_vs_fp32=err)
            for k, us in t.items():
                r[k + "_us"] = us
                r[k + "_GBps"] = by[k] / us / 1e3
                r[k + "_hbm_share"] = by[k] / (us * 1e-6) / HBM_BYTES_PER_S
            r["int4_vs_dequant_gemm"] = t["int4_dequant_gemm"] / t["int4"]
            r["int4_vs_fp8"] = t["fp8"] / t["int4"]
            rows.append(r)
            print(json.dumps(r), flush=True)
        del wb, q, s, z, e, s8, deq
        torch.cuda.empty_cache()
    return rows


def _weight_bytes(m):
    return sum(p.numel() * p.element_size() for p in m.parameters())


def end_to_end(models, quick):
    prompt, new = (128, 32) if quick else (512, 256)
    configs = {"bf16": ("bf16", None), "fp8_w_fp8_kv": ("fp8", "fp8"), "int4": ("int4", None),
               "int4_w_fp8_kv": ("int4", "fp8")}
    rows = []
    for B in (1, 16):
        ids = torch.randint(3, 32000, (B, prompt), device="cuda", generator=torch.Generator("cuda").manual_seed(B))
        res, seqs = {}, {}
        for rep in range(3):                     # alternate the configurations; the first round is the warm-up
            for name, (wname, kv) in configs.items():
                m = models[wname]
                m.kv_cache, m._decode_graph = None, None
                torch.cuda.empty_cache()
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                with torch.no_grad():
                    m.kv_cache_dtype = torch.float8_e4m3fn if kv else None
                    m.allocate_kv_cache(B, prompt)
                    ev[0].record()
                    m(ids, use_cache=True)
                    ev[1].record()
                    m.set_cache(None)
                    ev[2].record()
                    out = m.generate(ids, max_new_tokens=new, eos_token_id=None, pad_token_id=0, decode_graphs=True,
                                     kv_cache_dtype=kv)
                    ev[3].record()
                    torch.cuda.synchronize()
                prefill_ms, gen_ms = ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3])
                peak = torch.cuda.max_memory_allocated() - base
                m.kv_cache_dtype = None
                if rep > 0:
                    res.setdefault(name, []).append(dict(
                        seconds=gen_ms / 1e3, new_tokens_per_s=B * new / (gen_ms / 1e3), prefill_ms=prefill_ms,
                        ms_per_decode_step=(gen_ms - prefill_ms) / (new - 1), peak_extra_gb=peak / 1e9))
                seqs[name] = out[:, prompt:]
        r = dict(B=B, prompt=prompt, new_tokens=new, runs=res,
                 token_agreement_with_bf16={k: float((v == seqs["bf16"]).float().mean()) for k, v in seqs.items()})
        rows.append(r)
        print(json.dumps(r), flush=True)
    return rows


def accuracy(models, quick):
    prompt = 128 if quick else 512
    ids = torch.randint(3, 32000, (1, prompt), device="cuda", generator=torch.Generator("cuda").manual_seed(7))
    logits = {}
    for name, m in models.items():
        m.kv_cache = None
        with torch.no_grad():
            m.allocate_kv_cache(1, prompt)
            logits[name] = m(ids, use_cache=True)["logits"].float()
            m.set_cache(None)
    ref = logits["bf16"]
    r = {f"{k}_logit_rel_err": float((v - ref).norm() / ref.norm()) for k, v in logits.items() if k != "bf16"}
    r.update({f"{k}_top1_agreement": float((v.argmax(-1) == ref.argmax(-1)).float().mean())
              for k, v in logits.items() if k != "bf16"})
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "int4_weights_bench.json"))
    ap.add_argument("--quick", action="store_true", help="a subset of the sizes (a rehearsal, not a measurement)")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--skip-kernel", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("int4_weights_bench needs a CUDA device")
    from libai_b200 import ops
    from libai_b200.config import DictConfig
    from libai_b200.utils import distributed as dist

    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    ext = ops.load_ext(required=True)
    info = gpu_info()
    print(json.dumps(info), flush=True)
    result = dict(info, kernel_max_m=OF.INT4W_KERNEL_MAX_M,
                  kernel=[] if a.skip_kernel else kernel_level(ext, a.quick))
    if not a.skip_e2e:
        layers = 4 if a.quick else 32
        models = {"bf16": llama_7b(layers), "fp8": quantize_weights_fp8_(llama_7b(layers)),
                  "int4": quantize_weights_int4_(llama_7b(layers))}
        result["layers"] = layers
        result["weights_bytes"] = {k: _weight_bytes(m) for k, m in models.items()}
        print(json.dumps(dict(weights_bytes=result["weights_bytes"])), flush=True)
        result["accuracy"] = accuracy(models, a.quick)
        result["e2e"] = end_to_end(models, a.quick)
    result["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
