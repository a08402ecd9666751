"""Decode-attention and cached-generation timings on one GPU.

    python dev/decode_bench.py [--out output/decode_bench.json] [--quick]

Kernel level: the split-KV decode attention (one new query per sample and head) over a KV cache holding L keys, for a
Llama-7B-shaped layer (32 heads of 128) and a GPT-2-medium-shaped layer (16 heads of 64), B in {1, 8, 32} and L in
{512, 2048, 8192}.  Median microseconds over CUDA events (L2 flushed before every launch), the bytes the attention must
move (K and V of the window, q and o) over that time, and its share of the H100 SXM's 3.35 TB/s.  Comparators on the
same data: torch SDPA over the cache slices, and the path the models took before the cache existed (``torch.cat`` of
the past keys and values with the new row, then ``attention_ref``).

End to end: ``generate()`` on a randomly initialised Llama-7B-shaped model (32 layers, hidden 4096, 32 heads), a
512-token prompt and 256 new tokens, batch 1 and 16, with the native decode path against the same run with
``decode_attention`` and ``kv_cache_append`` replaced by their reference implementations.

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
                nbytes = 2 * B * A * L * D * 2 + 2 * B * A * D * 2
                r = dict(shape=name, A=A, D=D, B=B, L=L, kernel_us=t_kernel, sdpa_us=t_sdpa, previous_us=t_prev,
                         bytes=nbytes, kernel_GBps=nbytes / t_kernel / 1e3,
                         kernel_hbm_share=nbytes / (t_kernel * 1e-6) / HBM_BYTES_PER_S, rel_err_vs_sdpa=err)
                rows.append(r)
                print(json.dumps(r), flush=True)
                del k, v
                torch.cuda.empty_cache()
    return rows


def end_to_end(quick):
    from libai_b200.config import DictConfig
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    layers = 4 if quick else 32
    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=32000, hidden_size=4096, intermediate_size=11008,
                          num_attention_heads=32, max_position_embeddings=2048, rms_norm_eps=1e-6,
                          initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device="cuda:0", seed=1234):
        model = LlamaForCausalLM(cfg).eval()
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "decode_bench.json"))
    ap.add_argument("--quick", action="store_true", help="a subset of the sizes (a rehearsal, not a measurement)")
    ap.add_argument("--skip-e2e", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("decode_bench needs a CUDA device")
    from libai_b200 import ops

    ops.load_ext(required=True)
    info = gpu_info()
    print(json.dumps(info), flush=True)
    result = dict(info, kernel=kernel_level(a.quick), e2e=[] if a.skip_e2e else end_to_end(a.quick))
    result["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
