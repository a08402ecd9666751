"""Beam search and multi-sample generation on the contiguous and the paged KV cache, at a Llama-7B shape.

    python dev/paged_kv_bench.py [--out OUT.json] [--quick]

A Llama-7B shape (32 layers, 32 heads of 128, hidden 4096, FFN 11008, vocab 32000) with random bf16 weights.  Every
case runs the contiguous and the paged cache alternately, after one warm-up round of both, and reports per run: new
tokens per second (host clock around the synchronised call), prefill ms and device ms per decode step (CUDA events
around each step), reorder ms (events around the cache reorder of each beam step), the peak of
``torch.cuda.max_memory_allocated`` and whether the paged sequences equal the contiguous ones.  The card's name and
power limit are read in the same launch.  Cases: 4-beam search at batch 1 and 4 with 512- and 2048-token prompts and
128 new tokens, with and without decode graphs; sampling with ``num_return_sequences = 8`` at batch 1 with a
1024-token prompt; and 4-beam search on an FP8 cache.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from libai_b200.config import DictConfig  # noqa: E402
from libai_b200.layers._param import param_defaults  # noqa: E402
from libai_b200.utils import distributed as dist  # noqa: E402

NEW = 128


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        out = torch.cuda.get_device_name()
    return out


def build(quick):
    from libai_b200.models import LlamaForCausalLM

    cfg = dict(hidden_layers=32, vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_attention_heads=32,
               max_position_embeddings=4096, rms_norm_eps=1e-5, initializer_range=0.02,
               use_scaled_init_for_output_weights=True, scale_mask_softmax_fusion=False, amp_enabled=False,
               bos_token_id=1, eos_token_id=2, pad_token_id=0, max_length=20)
    if quick:
        cfg.update(hidden_layers=2, hidden_size=256, intermediate_size=512, num_attention_heads=2, vocab_size=1000)
    with param_defaults(dtype=torch.bfloat16, device="cuda", seed=0):
        return LlamaForCausalLM(DictConfig(cfg)).eval()


class Timers:
    """CUDA events around every decode step (the first is the prefill) and every cache reorder of one call."""

    def __init__(self, m):
        self.m, self.steps, self.reorders = m, [], []
        cls = type(m)
        step, reorder = cls._decode_step, cls._reorder_cache

        def timed(store, fn):
            def run(*a, **k):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn(*a, **k)
                e1.record()
                store.append((e0, e1))
                return out
            return run

        m._decode_step = timed(self.steps, lambda *a, **k: step(m, *a, **k))
        m._reorder_cache = timed(self.reorders, lambda *a, **k: reorder(m, *a, **k))

    def result(self):
        ms = [a.elapsed_time(b) for a, b in self.steps]
        rs = [a.elapsed_time(b) for a, b in self.reorders]
        del self.m._decode_step, self.m._reorder_cache
        return dict(prefill_ms=round(ms[0], 3), decode_step_ms=round(sum(ms[1:]) / max(len(ms) - 1, 1), 4),
                    reorder_ms=round(sum(rs) / len(rs), 4) if rs else None)


def run(m, ids, paged, graphs, kv, **kw):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    timers = Timers(m)
    torch.manual_seed(0)
    t0 = time.perf_counter()
    with torch.no_grad():
        out = m.generate(ids, max_length=ids.shape[1] + NEW, eos_token_id=None, decode_graphs=graphs,
                         kv_cache_dtype=kv, paged_kv_cache=paged, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    res = timers.result()
    res.update(new_tokens_per_s=round(out.shape[0] * NEW / dt, 1),
               peak_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    m.kv_cache = m._decode_graph = None   # the next run allocates its own cache
    torch.cuda.empty_cache()
    return out, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="a tiny model and prompts: rehearse the script")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paged_kv_bench: no CUDA device")
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    m = build(a.quick)
    cases = [dict(name=f"beam4 b{b} prompt{p}{' graphs' if g else ''}", b=b, prompt=p, graphs=g, kv=None,
                  kw=dict(num_beams=4)) for b in (1, 4) for p in (512, 2048) for g in (False, True)]
    cases += [dict(name="sample n8 b1 prompt1024", b=1, prompt=1024, graphs=False, kv=None,
                   kw=dict(do_sample=True, num_return_sequences=8)),
              dict(name="beam4 b4 prompt2048 fp8", b=4, prompt=2048, graphs=False, kv="fp8", kw=dict(num_beams=4))]
    if a.quick:
        for c in cases:
            c["prompt"] //= 16
    rows = []
    gen = torch.Generator().manual_seed(0)
    for c in cases:
        ids = torch.randint(3, 1000, (c["b"], c["prompt"]), generator=gen).cuda()
        for paged in (False, True):   # warm-up round
            run(m, ids, paged, c["graphs"], c["kv"], **c["kw"])
        res = {}
        for paged in (False, True):
            out, r = run(m, ids, paged, c["graphs"], c["kv"], **c["kw"])
            res["paged" if paged else "contiguous"] = (out, r)
        same = torch.equal(res["contiguous"][0], res["paged"][0])
        for kind in ("contiguous", "paged"):
            row = dict(case=c["name"], cache=kind, **res[kind][1], same_sequences=same)
            rows.append(row)
            print(json.dumps(row), flush=True)
    result = dict(card=card(), rows=rows)
    print(json.dumps(dict(card=result["card"])))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
