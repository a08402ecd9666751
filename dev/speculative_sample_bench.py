"""Speculative sampling (``generate(do_sample=True, assistant_model=...)``) on one GPU.

    python dev/speculative_sample_bench.py [--out output/speculative_sample_bench.json] [--quick] [--skip-e2e]

In one launch (the card name, power limit and clocks are read in it):

1. Kernels: the device time (CUDA events, mean over repeated launches) of one acceptance call
   (``OF.spec_accept_sample``, b·(k + 1) rows) and of the k draft draws of an iteration (``OF.spec_sample``, k calls
   of b rows) for b = 1, 4, 16, k = 2, 4, 8, V = 32000, 151936, 250880 and each warp (temperature only, top-k 50,
   top-p 0.8, both), bf16 logits.  Beside them the eager PyTorch chain ``multinomial_sample`` runs on the same b·(k + 1)
   rows: the warpers, softmax and ``torch.multinomial``.
2. End to end: new tokens per second (host clock around ``generate()``, synchronised) of a Llama-7B-shape target with
   decode graphs, for ``multinomial_sample`` and for speculative sampling at k = 2, 4, 8 with the TinyLlama-shape draft
   and with an INT4 copy of the target as the draft, at batch 1 and 4, a 512-token prompt and 128 new tokens,
   temperature 0.8, top-k 50, top-p 0.8.  The measured acceptance (accepted proposals over proposals) is beside each
   row.  The weights are random: the TinyLlama-shape draft and the target agree on almost nothing, so its acceptance
   is near zero and its rows are a worst case, not what a trained pair does.
"""
import argparse
import json
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from dev.decode_bench import gpu_info  # noqa: E402
from dev.decode_graph_bench import llama_7b  # noqa: E402
from dev.speculative_bench import CTX, _events_ms, tiny_llama  # noqa: E402
from libai_b200.config import DictConfig  # noqa: E402
from libai_b200.inference import quantize_weights_int4_  # noqa: E402
from libai_b200.inference.generator.generation_logits_processor import (  # noqa: E402
    LogitsProcessorList,
    TemperatureLogitsWarper,
    TopKLogitsWarper,
    TopPLogitsWarper,
)
from libai_b200.ops import functional as OF  # noqa: E402
from libai_b200.utils import distributed as dist  # noqa: E402

DEV = "cuda:0"
WARPS = {"T": (0.8, 0, 1.0), "topk50": (1.0, 50, 1.0), "topp0.8": (1.0, 0, 0.8), "both": (0.8, 50, 0.8)}


def _eager_chain(warp):
    T, tk, tp = warp
    w = LogitsProcessorList()
    if T != 1.0:
        w.append(TemperatureLogitsWarper(T))
    if tk:
        w.append(TopKLogitsWarper(tk))
    if tp < 1.0:
        w.append(TopPLogitsWarper(tp))
    return lambda rows: torch.multinomial(torch.softmax(w(None, rows.float()), dim=-1), 1)


@torch.no_grad()
def kernels(quick):
    out = []
    iters = 5 if quick else 50
    for V in (32000, 151936, 250880):
        for b in (1, 4, 16):
            for k in (2, 4, 8):
                g = torch.Generator(device=DEV).manual_seed(V + b + k)
                logits = (torch.randn(b, k + 1, V, device=DEV, generator=g) * 3).to(torch.bfloat16)
                q = (logits[:, :k].float() + torch.randn(b, k, V, device=DEV, generator=g)).to(torch.bfloat16)
                u = torch.rand(b, k + 1, 2, device=DEV, generator=g)
                ud = torch.rand(b, k, device=DEV, generator=g)
                props = torch.empty(b, k, dtype=torch.long, device=DEV)
                unfinished = torch.ones(b, dtype=torch.long, device=DEV)
                draft_rows = [q[:, j].contiguous() for j in range(k)]
                qb = torch.empty_like(q)
                flat = logits.view(b * (k + 1), V)
                for name, warp in WARPS.items():
                    acc = _events_ms(lambda: OF.spec_accept_sample(logits, q, props, u, unfinished, *warp, None, None),
                                     iters)
                    draws = _events_ms(lambda: [OF.spec_sample(draft_rows[j], qb, j, ud, props, *warp)
                                                for j in range(k)], iters)
                    chain = _eager_chain(warp)
                    eager = _events_ms(lambda: chain(flat), iters)
                    row = dict(V=V, batch=b, k=k, warp=name, accept_us=round(acc * 1e3, 1),
                               draft_draws_us=round(draws * 1e3, 1), eager_chain_us=round(eager * 1e3, 1))
                    print(json.dumps(row), flush=True)
                    out.append(row)
    return out


def end_to_end(target, drafts, quick):
    new = 32 if quick else 128
    warp = dict(do_sample=True, temperature=0.8, top_k=50, top_p=0.8)
    configs = [("multinomial", None, 0)] + [(n, d, k) for n, d in drafts.items() for k in (2, 4, 8)]
    stats = {}
    accept = OF.spec_accept_sample

    def counted(*a, **kw):
        res = accept(*a, **kw)
        R = a[0].shape[1]
        stats["acc"] += int(res[:, 2 * R].sum())
        stats["props"] += res.shape[0] * (R - 1)
        return res

    OF.spec_accept_sample = counted
    results = []
    try:
        for rnd in range(2):   # round 0 is the warm-up
            for b in (1, 4):
                ids = torch.randint(3, 32000, (b, CTX), device=DEV, generator=torch.Generator(device=DEV).manual_seed(b))
                for name, draft, k in configs:
                    kw = dict(max_length=CTX + new, eos_token_id=None, decode_graphs=True, **warp)
                    if draft is not None:
                        kw.update(assistant_model=draft, num_assistant_tokens=k)
                    stats.update(acc=0, props=0)
                    torch.manual_seed(0)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    target.generate(ids, **kw)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    if rnd == 0:
                        continue
                    row = dict(batch=b, draft=name, k=k, tokens_per_s=round(b * new / dt, 2),
                               ms_per_token=round(dt * 1e3 / new, 3),
                               acceptance=round(stats["acc"] / stats["props"], 4) if stats["props"] else None)
                    print(json.dumps(row), flush=True)
                    results.append(row)
    finally:
        OF.spec_accept_sample = accept
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "speculative_sample_bench.json"))
    ap.add_argument("--quick", action="store_true", help="fewer layers, tokens and launches (a rehearsal)")
    ap.add_argument("--skip-e2e", action="store_true", help="the kernels only")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("speculative_sample_bench needs a CUDA device")
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    info = gpu_info()
    print(json.dumps(info), flush=True)
    result = dict(info)
    result["kernels"] = kernels(a.quick)
    if not a.skip_e2e:
        layers, draft_layers = (2, 2) if a.quick else (32, 22)
        target = llama_7b(layers)
        drafts = {"tinyllama": tiny_llama(draft_layers), "int4_copy": quantize_weights_int4_(llama_7b(layers))}
        result["e2e"] = end_to_end(target, drafts, a.quick)
    result["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
