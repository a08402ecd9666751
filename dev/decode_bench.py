"""Decode-attention and cached-generation timings on one GPU.

    python dev/decode_bench.py [--out output/decode_bench.json] [--quick]

Kernel level: the split-KV decode attention (one new query per sample and head) over a KV cache holding L keys, for a
Llama-7B-shaped layer (32 heads of 128) and a GPT-2-medium-shaped layer (16 heads of 64), B in {1, 8, 32} and L in
{512, 2048, 8192}.  Median microseconds over CUDA events (L2 flushed before every launch), the bytes the attention must
move (K and V of the window, q and o) over that time, and its share of the H100 SXM's 3.35 TB/s.  Comparators on the
same data: torch SDPA over the cache slices, and the path the models took before the cache existed (``torch.cat`` of
the past keys and values with the new row, then ``attention_ref``).  The fp8 column runs the same attention over an
FP8 (E4M3) cache holding the same rows quantized (``kv_cache_quantize_ref``); its bytes count 1 per element plus the
4-byte scale of every row, and its error is against SDPA over the dequantized rows.

End to end: ``generate()`` on a randomly initialised Llama-7B-shaped model (32 layers, hidden 4096, 32 heads), a
512-token prompt and 256 new tokens, batch 1 and 16, with the native decode path against the same run with
``decode_attention`` and ``kv_cache_append`` replaced by their reference implementations.

FP8 cache, end to end (``--fp8-e2e``): ``generate()`` on the same Llama-7B-shaped model with a 2048-token prompt and 256
new tokens, with a bf16 and an FP8 cache alternated, at batch 16 and at the largest batch (of a few candidates) whose
bf16 run fits; and the largest batch at 8192 context per cache dtype, computed from the bytes of the weights and the
cache (labelled as computed).

The card name, power limit and SM clock are printed with the figures and stored in the JSON output.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from libai_b200.ops import functional as OF  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name() + ", unknown, unknown, unknown"
    name, power, sm, sm_max = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def time_us(fn, iters, flush):
    for _ in range(3):
        fn()
    times = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3)
    return statistics.median(times)


def kernel_level(quick):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    shapes = [("llama-7b", 32, 128), ("gpt2-medium", 16, 64)]
    for name, A, D in shapes:
        for B in ((1, 8) if quick else (1, 8, 32)):
            for L in ((512, 2048) if quick else (512, 2048, 8192)):
                C = L + 64
                g = torch.Generator(device="cuda").manual_seed(0)
                k = torch.randn(B, A, C, D, device="cuda", generator=g, dtype=torch.bfloat16)
                v = torch.randn(B, A, C, D, device="cuda", generator=g, dtype=torch.bfloat16)
                q = torch.randn(B, 1, A, D, device="cuda", generator=g, dtype=torch.bfloat16)
                lens = torch.full((B,), L - 1, dtype=torch.int32, device="cuda")   # + the new token = L keys
                start = torch.zeros(B, dtype=torch.int32, device="cuda")
                scale = D ** -0.5
                out = OF.decode_attention(q, k, v, lens, start, scale=scale)
                qh = q.transpose(1, 2)
                ks, vs = k[:, :, :L], v[:, :, :L]
                sdpa = torch.nn.functional.scaled_dot_product_attention(qh, ks, vs, scale=scale).transpose(1, 2)
                err = float((out.float() - sdpa.float()).abs().max() / sdpa.float().abs().max())
                t_kernel = time_us(lambda: OF.decode_attention(q, k, v, lens, start, scale=scale), 50, flush)
                t_sdpa = time_us(lambda: torch.nn.functional.scaled_dot_product_attention(qh, ks, vs, scale=scale),
                                 50, flush)
                past_k, past_v = ks[:, :, : L - 1].contiguous(), vs[:, :, : L - 1].contiguous()
                new_k, new_v = ks[:, :, L - 1 :].contiguous(), vs[:, :, L - 1 :].contiguous()

                def previous():
                    kk = torch.cat((past_k, new_k), dim=2)
                    vv = torch.cat((past_v, new_v), dim=2)
                    return OF.attention_ref(qh, kk, vv, causal=False, scale=scale)

                t_prev = time_us(previous, 10, flush)
                del past_k, past_v
                (k8, k_s), (v8, v_s) = OF.kv_cache_quantize_ref(k), OF.kv_cache_quantize_ref(v)
                fp8 = dict(k_scale=k_s, v_scale=v_s)
                out8 = OF.decode_attention(q, k8, v8, lens, start, scale=scale, **fp8)
                ks8, vs8 = OF.kv_cache_dequant(k8[:, :, :L], k_s[:, :, :L]), OF.kv_cache_dequant(v8[:, :, :L],
                                                                                                 v_s[:, :, :L])
                sdpa8 = torch.nn.functional.scaled_dot_product_attention(qh, ks8, vs8, scale=scale).transpose(1, 2)
                err8 = float((out8.float() - sdpa8.float()).abs().max() / sdpa8.float().abs().max())
                del ks8, vs8
                t_fp8 = time_us(lambda: OF.decode_attention(q, k8, v8, lens, start, scale=scale, **fp8), 50, flush)
                nbytes = 2 * B * A * L * D * 2 + 2 * B * A * D * 2
                nbytes8 = 2 * B * A * L * (D + 4) + 2 * B * A * D * 2
                r = dict(shape=name, A=A, D=D, B=B, L=L, kernel_us=t_kernel, sdpa_us=t_sdpa, previous_us=t_prev,
                         bytes=nbytes, kernel_GBps=nbytes / t_kernel / 1e3,
                         kernel_hbm_share=nbytes / (t_kernel * 1e-6) / HBM_BYTES_PER_S, rel_err_vs_sdpa=err,
                         fp8_us=t_fp8, fp8_bytes=nbytes8, fp8_GBps=nbytes8 / t_fp8 / 1e3,
                         fp8_hbm_share=nbytes8 / (t_fp8 * 1e-6) / HBM_BYTES_PER_S, fp8_speedup=t_kernel / t_fp8,
                         fp8_rel_err_vs_sdpa_dequant=err8)
                del k8, v8
                rows.append(r)
                print(json.dumps(r), flush=True)
                del k, v
                torch.cuda.empty_cache()
    return rows


def llama_7b(layers):
    from libai_b200.config import DictConfig
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=32000, hidden_size=4096, intermediate_size=11008,
                          num_attention_heads=32, max_position_embeddings=4096, rms_norm_eps=1e-6,
                          initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device="cuda:0", seed=1234):
        return LlamaForCausalLM(cfg).eval()


def end_to_end(quick):
    layers = 4 if quick else 32
    model = llama_7b(layers)
    prompt, new = (128, 32) if quick else (512, 256)
    real = {"decode_attention": OF.decode_attention, "kv_cache_append": OF.kv_cache_append}
    ref = {"decode_attention": OF.decode_attention_ref,
           "kv_cache_append": lambda qkv, k, v, lens, cos=None, sin=None, return_q=True:
               OF.kv_cache_append_ref(qkv, k, v, lens, cos, sin)}
    rows = []
    for B in (1, 16):
        ids = torch.randint(3, 32000, (B, prompt), device="cuda", generator=torch.Generator("cuda").manual_seed(B))
        res = {}
        for rep in range(2):                     # alternate the two paths; the first round is the warm-up
            for path, fns in (("native", real), ("reference", ref)):
                for k, fn in fns.items():
                    setattr(OF, k, fn)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                seqs = model.generate(ids, max_new_tokens=new, eos_token_id=None, pad_token_id=0)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if rep == 1:
                    res[path] = dict(seconds=dt, new_tokens_per_s=B * new / dt, seqs=seqs)
        for k, fn in real.items():
            setattr(OF, k, fn)
        same = bool(torch.equal(res["native"]["seqs"], res["reference"]["seqs"]))
        r = dict(layers=layers, B=B, prompt=prompt, new_tokens=new, same_tokens=same,
                 **{f"{p}_{k}": v for p, d in res.items() for k, v in d.items() if k != "seqs"})
        r["speedup"] = r["reference_seconds"] / r["native_seconds"]
        rows.append(r)
        print(json.dumps(r), flush=True)
    return rows


def fp8_end_to_end(quick):
    """bf16 against FP8 cache in generate(), alternated; the capacity at 8192 context computed from bytes."""
    layers = 4 if quick else 32
    model = llama_7b(layers)
    prompt, new = (128, 32) if quick else (2048, 256)
    weights = sum(p.numel() * p.element_size() for p in model.parameters())
    per_token = {"bf16": layers * 2 * 32 * 128 * 2, "fp8": layers * 2 * 32 * (128 + 4)}   # K and V of every layer
    card = 80e9
    capacity = {dt: int((card - weights) // (8192 * b)) for dt, b in per_token.items()}
    print(json.dumps(dict(computed_max_batch_at_8192=capacity, weights_bytes=weights, cache_bytes_per_token=per_token,
                          card_bytes=card, note="computed from bytes (weights + cache), not measured")), flush=True)
    rows = []

    def run(B, dtype):
        ids = torch.randint(3, 32000, (B, prompt), device="cuda", generator=torch.Generator("cuda").manual_seed(B))
        model.kv_cache = None
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seqs = model.generate(ids, max_new_tokens=new, eos_token_id=None, pad_token_id=0, kv_cache_dtype=dtype)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, seqs

    big = None
    for B in ((4,) if quick else (48, 40, 32, 24)):   # the largest of these whose bf16 run fits
        try:
            run(B, None)
            big = B
            break
        except torch.cuda.OutOfMemoryError:
            model.kv_cache = None
            torch.cuda.empty_cache()
    for B in sorted({16 if not quick else 2, big} - {None}):
        res = {}
        for rep in range(3):                     # alternate the two caches; the first round is the warm-up
            for name, dtype in (("bf16", None), ("fp8", "fp8")):
                dt, seqs = run(B, dtype)
                if rep > 0:
                    res.setdefault(name, []).append(dict(seconds=dt, new_tokens_per_s=B * new / dt))
                res[name + "_seqs"] = seqs
        agree = float((res["bf16_seqs"][:, prompt:] == res["fp8_seqs"][:, prompt:]).float().mean())
        r = dict(layers=layers, B=B, prompt=prompt, new_tokens=new, bf16=res["bf16"], fp8=res["fp8"],
                 token_agreement=agree, peak_gb=torch.cuda.max_memory_allocated() / 1e9)
        rows.append(r)
        print(json.dumps(r), flush=True)
    return dict(capacity_computed=capacity, runs=rows, largest_bf16_batch_tried=big)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "decode_bench.json"))
    ap.add_argument("--quick", action="store_true", help="a subset of the sizes (a rehearsal, not a measurement)")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--fp8-e2e", action="store_true", help="generate() with a bf16 against an FP8 cache")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("decode_bench needs a CUDA device")
    from libai_b200 import ops

    ops.load_ext(required=True)
    info = gpu_info()
    print(json.dumps(info), flush=True)
    result = dict(info, kernel=[] if a.skip_kernel else kernel_level(a.quick),
                  e2e=[] if a.skip_e2e else end_to_end(a.quick))
    if a.fp8_e2e:
        result["fp8_e2e"] = fp8_end_to_end(a.quick)
    result["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
