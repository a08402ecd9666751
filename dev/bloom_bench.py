"""BLOOM generation on the KV cache and the ALiBi decode kernel, timed on one GPU.

    python dev/bloom_bench.py --parent-model OLD/projects/BLOOM/modeling/bloom_model.py [--out output/bloom_bench.json]
                              [--quick]

- ``generate()``: randomly initialised bf16 models shaped like BLOOM-560m (24 layers × 1024, 16 heads of 64) and
  BLOOM-7b1 (30 × 4096, 32 heads of 128), vocab 250880; greedy, 128 new tokens, batch 1 and 16, prompts left-padded
  to 1024 tokens with lengths spread evenly from 128 to 1024 (batch 1: one 1024-token prompt).  New tokens per second
  (batch × 128 over the wall time of the call, after a short warm-up call), the time of the prompt's forward into an
  empty cache (median of 3) and the peak memory allocated during the call.  ``--parent-model`` is the
  ``bloom_model.py`` of another version, run on this tree's library with the same weights; the two versions alternate,
  ``--reps`` rounds each, and the fraction of equal generated tokens is recorded.
- The kernel alone: ``decode_attn`` with and without slopes, one new token, the two head shapes, caches of 1152 rows
  (1024 + 128) per sample, batch 1 and 16; median microseconds over 200 calls timed with CUDA events, and the K/V bytes
  the call must read over that time as a share of the H100 SXM's 3.35 TB/s.

The card name, power limit and SM clock are stored with the figures.
"""
import argparse
import importlib.util
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
VOCAB, PROMPT, NEW = 250880, 1024, 128
SHAPES = {"bloom-560m": (24, 1024, 16), "bloom-7b1": (30, 4096, 32)}   # layers, hidden, heads
HBM_BYTES_PER_S = 3.35e12


def load_module(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build(mod, shape):
    from libai_b200.config import LazyConfig
    from libai_b200.layers._param import param_defaults

    layers, hidden, heads = SHAPES[shape]
    cfg = LazyConfig.load(os.path.join(ROOT, "projects/BLOOM/configs/bloom_inference.py")).cfg
    cfg.update(dict(vocab_size=VOCAB, hidden_size=hidden, hidden_layers=layers, n_head=heads))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return mod.BloomForCausalLM(cfg).eval()


def prompts(batch):
    g = torch.Generator(device=DEV).manual_seed(batch)
    ids = torch.randint(4, VOCAB, (batch, PROMPT), device=DEV, generator=g)
    am = torch.ones_like(ids)
    lens = [PROMPT] if batch == 1 else [128 + (PROMPT - 128) * i // (batch - 1) for i in range(batch)]
    for i, n in enumerate(lens):
        ids[i, : PROMPT - n], am[i, : PROMPT - n] = 3, 0
    return ids, am


@torch.no_grad()
def run_generate(m, ids, am, new):
    gen = dict(attention_mask=am, eos_token_id=None, pad_token_id=3, do_sample=False, num_beams=1, use_cache=True)
    m.generate(ids, max_new_tokens=4, **gen)   # warm-up: kernels, cache allocation
    prefill = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m(ids, attention_mask=am, use_cache=True)
        torch.cuda.synchronize()
        prefill.append(time.perf_counter() - t0)
        m.set_cache(None)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = m.generate(ids, max_new_tokens=new, **gen)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    made = out.shape[1] - ids.shape[1]
    return out[:, ids.shape[1]:], dict(new_tokens=made, seconds=round(dt, 3),
                                       new_tokens_per_s=round(ids.shape[0] * made / dt, 1),
                                       prefill_ms=round(1e3 * statistics.median(prefill), 1),
                                       peak_gib=round(torch.cuda.max_memory_allocated() / 2**30, 2))


def generation(parent_path, reps, new):
    from projects.BLOOM.modeling import bloom_model as this

    versions = {"this": this}
    if parent_path:
        versions["parent"] = load_module(os.path.abspath(parent_path), "parent_bloom_model")
    rows = []
    for shape in SHAPES:
        models = {v: build(mod, shape) for v, mod in versions.items()}
        for batch in (1, 16):
            ids, am = prompts(batch)
            outs = {}
            for rep in range(reps):
                for v, m in models.items():
                    toks, row = run_generate(m, ids, am, new)
                    outs[v] = toks
                    rows.append(dict(case="generate", model=shape, version=v, batch=batch, rep=rep, **row))
                    print(json.dumps(rows[-1]), flush=True)
            if "parent" in outs:
                same = (outs["parent"] == outs["this"]).float().mean().item()
                rows.append(dict(case="generate_tokens_equal", model=shape, batch=batch, fraction=round(same, 4)))
                print(json.dumps(rows[-1]), flush=True)
        del models
        torch.cuda.empty_cache()
    return rows


def kernel(iters):
    from libai_b200 import ops

    ext = ops.load_ext(required=True)
    rows = []
    L = PROMPT + NEW
    for shape, (_, hidden, heads) in SHAPES.items():
        d = hidden // heads
        for batch in (1, 16):
            g = torch.Generator(device=DEV).manual_seed(heads + batch)
            q = torch.randn(batch, 1, heads, d, device=DEV, generator=g).bfloat16()
            kc = torch.randn(batch, heads, L, d, device=DEV, generator=g).bfloat16()
            vc = torch.randn_like(kc)
            lens = torch.full((batch,), L - 1, dtype=torch.int32, device=DEV)
            kv_start = torch.zeros(batch, dtype=torch.int32, device=DEV)
            slopes = torch.rand(heads, device=DEV, generator=g)
            nbytes = 2 * batch * heads * L * d * 2   # every visible K and V row once, bf16
            for alibi in (False, True):
                def call():
                    return ext.decode_attn(q, kc, vc, lens, kv_start, d ** -0.5, 0, slopes if alibi else None)
                for _ in range(10):
                    call()
                times = []
                for _ in range(iters):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    call()
                    b.record()
                    b.synchronize()
                    times.append(a.elapsed_time(b) * 1e3)
                us = statistics.median(times)
                rows.append(dict(case="decode_attn", heads=heads, head_dim=d, batch=batch, cache_rows=L, alibi=alibi,
                                 median_us=round(us, 2), kv_gbytes_per_s=round(nbytes / us / 1e3, 1),
                                 share_of_3_35_tb_s=round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)))
                print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-model", default="", help="bloom_model.py of the version to compare against")
    ap.add_argument("--out", default="output/bloom_bench.json")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--only", default="", choices=["", "generate", "kernel"])
    args = ap.parse_args()
    os.chdir(ROOT)
    from dev.decode_bench import gpu_info
    from libai_b200 import ops
    from libai_b200.config import DictConfig
    from libai_b200.utils import distributed as dutil

    ops.load_ext(required=True)
    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1)))
    info = gpu_info()
    print(json.dumps(info), flush=True)
    rows = []
    if args.only in ("", "kernel"):
        rows += kernel(20 if args.quick else 200)
    if args.only in ("", "generate"):
        rows += generation(args.parent_model, 1 if args.quick else args.reps, 8 if args.quick else NEW)
    out = args.out if os.path.isabs(args.out) else os.path.join(ROOT, args.out)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
