"""T5 / mT5 generation on the KV caches and the T5 decode-kernel instances, timed on one GPU.

    python dev/t5_decode_bench.py --parent-model OLD/projects/MT5/mt5_model.py [--out output/t5_decode_bench.json]
                                  [--quick]

- ``generate()``: randomly initialised bf16 models shaped like mT5-base (12 + 12 layers × 768, 12 heads of 64,
  gated-GELU d_ff 2048, vocab 250112) and T5-v1.1-large (24 + 24 × 1024, 16 heads of 64, d_ff 2816, vocab 32128), with
  weights at 0.02 and relative-bias tables of unit scale (larger random weights make T5's unscaled attention nearly
  hard, and bf16 then parts from fp32 from the first token); 128 new tokens, greedy at batch 1 (one 512-token encoder
  input) and batch 16 (right-padded encoder inputs of 128 to 512 tokens), and beam search with 4 beams at batch 4 (the
  first four of those inputs).  New tokens per second (batch × 128 over the wall time of the call, after a short
  warm-up call), the time of the first decoder step, which runs the encoder (median of 3), and the peak memory
  allocated during the call.  ``--parent-model`` is the ``mt5_model.py`` of another version, run on this tree's
  library with the same weights; the two versions alternate, ``--reps`` rounds each, and the fraction of equal
  generated tokens is recorded.
- The kernel alone, head dim 64, batch 1 and 16, at both models' head counts: the decoder self-attention step,
  ``decode_attn`` over caches of 640 rows (512 + 128) with and without ``rel_bias``; the cross-attention step,
  ``decode_attn(causal=False)`` over 512 encoder keys against the flash kernel at Sq = 1 over the same keys (with
  ``kv_lens``).  Median microseconds over 200 calls timed with CUDA events, L2 flushed before every call, in three
  rounds that alternate the variants, and the K/V bytes the call must read over that time as a share of the H100 SXM's
  3.35 TB/s.

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
ENC, NEW, CACHE = 512, 128, 640
SHAPES = {"mt5-base": (12, 768, 12, 2048, 250112), "t5-v1_1-large": (24, 1024, 16, 2816, 32128)}
HBM_BYTES_PER_S = 3.35e12


def load_module(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build(mod, shape):
    from libai_b200.config import DictConfig
    from libai_b200.layers._param import param_defaults

    layers, hidden, heads, ff, vocab = SHAPES[shape]
    cfg = DictConfig(dict(vocab_size=vocab, hidden_size=hidden, hidden_layers=layers, num_attention_heads=heads,
                          head_size=hidden // heads, intermediate_size=ff, embedding_dropout_prob=0.0,
                          hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                          relative_attention_num_buckets=32, initializer_range=0.02, layernorm_eps=1e-6,
                          amp_enabled=False, model_type="mt5", padding_idx=0, is_encoder_decoder=True,
                          tie_word_embeddings=False, eos_token_id=1, pad_token_id=0, decoder_start_token_id=0,
                          use_cache=True, max_length=NEW + 1))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        m = mod.MT5Model(cfg).eval()
    g = torch.Generator(device=DEV).manual_seed(5)
    with torch.no_grad():
        for stack in (m.encoder, m.decoder):
            table = stack.layers[0].self_attention.relative_attention_bias
            table.copy_(torch.randn(table.shape, device=DEV, generator=g))
    return m


def inputs(batch, vocab):
    g = torch.Generator(device=DEV).manual_seed(batch)
    ids = torch.randint(2, vocab, (batch, ENC), device=DEV, generator=g)
    am = torch.ones_like(ids)
    lens = [ENC] if batch == 1 else [128 + (ENC - 128) * i // 15 for i in range(16)][:batch]
    for i, n in enumerate(lens):
        ids[i, n:], am[i, n:] = 0, 0
    return ids, am


@torch.no_grad()
def run_generate(m, ids, am, new, beams):
    gen = dict(encoder_attn_mask=am, eos_token_id=None, do_sample=False, num_beams=beams, use_cache=True)
    m.generate(ids, max_length=5, **gen)   # warm-up: kernels, cache allocation
    first = []
    start = torch.zeros(ids.shape[0], 1, dtype=torch.long, device=DEV)
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m(ids, start, am, use_cache=True)
        torch.cuda.synchronize()
        first.append(time.perf_counter() - t0)
        m.set_cache(None, None)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = m.generate(ids, max_length=new + 1, **gen)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    made = out.shape[1] - 1
    return out, dict(new_tokens=made, seconds=round(dt, 3), new_tokens_per_s=round(ids.shape[0] * made / dt, 1),
                     first_step_ms=round(1e3 * statistics.median(first), 1),
                     peak_gib=round(torch.cuda.max_memory_allocated() / 2**30, 2))


def generation(parent_path, reps, new):
    from projects.MT5 import mt5_model as this

    versions = {"this": this}
    if parent_path:
        versions["parent"] = load_module(os.path.abspath(parent_path), "parent_mt5_model")
    rows = []
    for shape in SHAPES:
        models = {v: build(mod, shape) for v, mod in versions.items()}
        for batch, beams in ((1, 1), (16, 1), (4, 4)):
            ids, am = inputs(batch, SHAPES[shape][4])
            outs = {}
            for rep in range(reps):
                for v, m in models.items():
                    toks, row = run_generate(m, ids, am, new, beams)
                    outs[v] = toks
                    rows.append(dict(case="generate", model=shape, version=v, batch=batch, beams=beams, rep=rep, **row))
                    print(json.dumps(rows[-1]), flush=True)
            if "parent" in outs:
                same = (outs["parent"] == outs["this"]).float().mean().item()
                rows.append(dict(case="generate_tokens_equal", model=shape, batch=batch, beams=beams,
                                 fraction=round(same, 4)))
                print(json.dumps(rows[-1]), flush=True)
        del models
        torch.cuda.empty_cache()
    return rows


def kernel(iters):
    from dev.decode_bench import time_us
    from libai_b200 import ops
    from libai_b200.ops import functional as OF

    ext = ops.load_ext(required=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    rows = []
    d = 64
    for heads in sorted({s[2] for s in SHAPES.values()}):
        for batch in (1, 16):
            g = torch.Generator(device=DEV).manual_seed(heads + batch)
            q = torch.randn(batch, 1, heads, d, device=DEV, generator=g).bfloat16()
            kc = torch.randn(batch, heads, CACHE, d, device=DEV, generator=g).bfloat16()
            vc = torch.randn_like(kc)
            kv_start = torch.zeros(batch, dtype=torch.int32, device=DEV)
            # self-attention: one new token on a cache of CACHE rows
            lens = torch.full((batch,), CACHE - 1, dtype=torch.int32, device=DEV)
            rel = torch.randn(heads, 129, device=DEV, generator=g)
            nbytes = 2 * batch * heads * CACHE * d * 2   # every visible K and V row once, bf16
            for rnd, with_rel in [(r, w) for r in range(3) for w in (False, True)]:
                us = time_us(lambda: ext.decode_attn(q, kc, vc, lens, kv_start, 1.0, 0, None,
                                                     rel if with_rel else None, True), iters, flush)
                rows.append(dict(case="decode_attn_self", heads=heads, head_dim=d, batch=batch, cache_rows=CACHE,
                                 rel_bias=with_rel, round=rnd, median_us=round(us, 2),
                                 kv_gbytes_per_s=round(nbytes / us / 1e3, 1),
                                 share_of_3_35_tb_s=round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)))
                print(json.dumps(rows[-1]), flush=True)
            # cross-attention: one new token over ENC encoder keys
            enc_len = torch.full((batch,), ENC, dtype=torch.int32, device=DEV)
            kce, vce = kc[:, :, :ENC].contiguous(), vc[:, :, :ENC].contiguous()
            nbytes = 2 * batch * heads * ENC * d * 2
            calls = {"decode_attn_noncausal": lambda: ext.decode_attn(q, kce, vce, enc_len, kv_start, 1.0, 0, None,
                                                                      None, False),
                     "flash_sq1": lambda: OF.attention(q.transpose(1, 2), kce, vce, causal=False, scale=1.0,
                                                       kv_lens=enc_len)}
            for rnd, name in [(r, n) for r in range(3) for n in calls]:
                us = time_us(calls[name], iters, flush)
                rows.append(dict(case="cross_" + name, heads=heads, head_dim=d, batch=batch, enc_keys=ENC, round=rnd,
                                 median_us=round(us, 2), kv_gbytes_per_s=round(nbytes / us / 1e3, 1),
                                 share_of_3_35_tb_s=round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)))
                print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-model", default="", help="mt5_model.py of the version to compare against")
    ap.add_argument("--out", default="output/t5_decode_bench.json")
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
