"""Chat turns with and without prefix caching, at a Llama-7B shape.

    python dev/prefix_cache_bench.py [--out OUT.json] [--quick]

A Llama-7B shape (32 layers, 32 heads of 128, hidden 4096, FFN 11008, vocab 32000) with random bf16 weights, greedy,
no EOS, on a paged cache.  A turn's prompt is a shared prefix (1,024 or 4,096 tokens) followed by a new suffix (32 or
256 tokens), at batch 1 and 4.  ``off``: ``prefix_cache_tokens=0``; ``on``: ``prefix_cache_tokens`` = the prefix
length + 512, after one call that cached the prefix.  Each case runs both arms alternately after a warm-up of both and
reports the median over rounds of: time to first token (host clock around a synchronised call with
``max_new_tokens=1``: the prefill and its first token), call time (the same with 64 new tokens), the rows reused, and
whether the tokens of the two arms agree (else the largest difference of their first logits).  The card's name and
power limit are read in the same launch.  The paged flash prefill against the gather path it replaced is measured by
``dev/paged_prefill_bench.py``.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dev.paged_kv_bench import card  # noqa: E402
from libai_b200.config import DictConfig  # noqa: E402
from libai_b200.layers._param import param_defaults  # noqa: E402
from libai_b200.utils import distributed as dist  # noqa: E402

NEW = 64


def build(quick):
    from libai_b200.models import LlamaForCausalLM

    cfg = dict(hidden_layers=32, vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_attention_heads=32,
               max_position_embeddings=8192, rms_norm_eps=1e-5, initializer_range=0.02,
               use_scaled_init_for_output_weights=True, scale_mask_softmax_fusion=False, amp_enabled=False,
               bos_token_id=1, eos_token_id=2, pad_token_id=0, max_length=20)
    if quick:
        cfg.update(hidden_layers=2, hidden_size=256, intermediate_size=512, num_attention_heads=2, vocab_size=1000)
    with param_defaults(dtype=torch.bfloat16, device="cuda", seed=0):
        return LlamaForCausalLM(DictConfig(cfg)).eval()


def timed(m, ids, new, budget):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = m.generate(ids, max_new_tokens=new, eos_token_id=None, output_scores=True, prefix_cache_tokens=budget,
                     paged_kv_cache=True)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefix_cache_bench: needs a GPU")
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    m = build(a.quick)
    vocab = m.cfg.vocab_size
    gen = torch.Generator().manual_seed(0)
    grid = [(1, 128, 32)] if a.quick else [(b, p, s) for b in (1, 4) for p in (1024, 4096) for s in (32, 256)]
    results = {"card": card(), "cases": []}
    print(results["card"], flush=True)
    for b, prefix, suffix in grid:
        shared = torch.randint(3, vocab, (1, prefix), generator=gen).expand(b, prefix)
        budget = prefix + 512   # the prefix, and room for each turn's own pages
        m.clear_prefix_cache()
        timed(m, shared.cuda(), 1, budget)   # caches the prefix
        rows = {"off": [], "on": []}
        times = {k: {"ttft": [], "call": []} for k in rows}
        outs = {}
        for r in range(a.rounds + 1):   # round 0: warm-up
            ids = torch.cat([shared, torch.randint(3, vocab, (b, suffix), generator=gen)], dim=1).cuda()
            for arm, bud in (("off", 0), ("on", budget)):
                kept = m.kv_cache   # the off arm allocates a pool per call: keep the on arm's pool and index
                ttft, _ = timed(m, ids, 1, bud)
                reused = m.kv_cache.reused_rows
                call, out = timed(m, ids, NEW, bud)
                outs[arm] = out
                if arm == "off":
                    m.kv_cache, m._decode_graph = kept, None
                if r:
                    times[arm]["ttft"].append(ttft)
                    times[arm]["call"].append(call)
                    rows[arm].append(reused)
            same = torch.equal(outs["off"][0], outs["on"][0])
        diff = float((outs["off"][1][0] - outs["on"][1][0]).abs().max())
        row = {"batch": b, "prefix": prefix, "suffix": suffix, "tokens_equal_last_round": same,
               "first_logits_max_diff_last_round": diff, "reused_rows": rows["on"][-1],
               **{f"{arm}_{k}_ms": statistics.median(v) for arm, t in times.items() for k, v in t.items()}}
        results["cases"].append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
