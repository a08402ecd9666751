"""Speculative decoding (``generate(assistant_model=...)`` / ``generate(prompt_lookup_num_tokens=...)``) on one GPU.

    python dev/speculative_bench.py [--out output/speculative_bench.json] [--quick]

Randomly initialised models, decode graphs on, in one launch (the card name, power limit and clocks are read in it):
the target has the Llama-7B shape (32 layers, hidden 4096, 32 heads, FFN 11008, vocabulary 32000), the draft the
TinyLlama-1.1B shape (22 layers, hidden 2048, 32 query and 4 key/value heads of 64, FFN 5632, vocabulary 32000).

1. Verify-step cost: the device time (CUDA events) of one replayed target step of s = 1, 2, 4, 8, 16 new tokens over a
   512-row cache, at batch 1 and 4, with bf16, FP8 and INT4 weights; after each step the cache rolls back s rows, so
   every step sees the same context.  The rollback's kernel is inside the timed window.  The values of s alternate
   over three rounds, and the first round is discarded.
2. Draft cost: the draft's replayed single-token step, and the acceptance kernel (``OF.spec_accept``) alone.
3. End to end: new tokens per second (host clock around ``generate()``, synchronised) for plain greedy and for both
   proposers at k = 2, 4, 8, batch 1 and 4, a 512-token prompt and 256 new tokens, bf16 weights.  The configurations
   alternate, and a warm-up round of all of them is discarded.  With random weights the draft and the target agree on
   almost nothing and a random prompt has no repeats to look up, so the acceptance rate beside each row is measured
   but says nothing about trained checkpoints: these rows are a worst case.
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
from libai_b200.config import DictConfig  # noqa: E402
from libai_b200.inference import decode_graph, quantize_weights_fp8_, quantize_weights_int4_  # noqa: E402
from libai_b200.inference.generator.generation_utils import Generator  # noqa: E402
from libai_b200.layers._param import param_defaults  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402
from libai_b200.utils import distributed as dist  # noqa: E402

DEV = "cuda:0"
CTX = 512


def tiny_llama(layers):
    from libai_b200.models import LlamaForCausalLM

    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=32000, hidden_size=2048, intermediate_size=5632,
                          num_attention_heads=32, num_key_value_heads=4, max_position_embeddings=4096,
                          rms_norm_eps=1e-5, initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=4321):
        return LlamaForCausalLM(cfg).eval()


def _events_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


@torch.no_grad()
def step_ms(model, b, s, iters):
    """Device ms of one replayed cached step of s new tokens over a CTX-row cache (rolled back after each step)."""
    call = decode_graph.DecodeCall()
    model.allocate_kv_cache(b, CTX + 32)
    g = torch.Generator(device=DEV).manual_seed(0)
    model(torch.randint(3, 32000, (b, CTX), device=DEV, generator=g), use_cache=True)
    ids = torch.randint(3, 32000, (b, s), device=DEV, generator=g)
    cache = model.kv_cache

    def one():
        decode_graph.step(model, {"input_ids": ids, "use_cache": True}, call, tokens=s)
        cache.rollback(s)
        model.past_length = cache.length

    for _ in range(3):   # eager, capture, replay
        one()
    assert decode_graph.current_graph(model).graph is not None, "the step was not captured"
    ms = _events_ms(one, iters)
    model._decode_graph = None
    model._reset_cache()
    return ms


def verify_cost(models, quick):
    """Per batch and weights: the step sizes alternate over three rounds; round 0 is a warm-up, and each s reports
    the mean of rounds 1 and 2 with both values beside it."""
    rows = []
    sizes = (1, 2, 4, 8, 16)
    for b in (1, 4):
        for name, m in models.items():
            runs = {s: [] for s in sizes}
            for rnd in range(3):
                for s in sizes:
                    ms = step_ms(m, b, s, 10 if quick else 50)
                    if rnd:
                        runs[s].append(ms)
            t = {s: sum(v) / len(v) for s, v in runs.items()}
            row = dict(weights=name, batch=b, ms={str(s): round(v, 4) for s, v in t.items()},
                       rounds={str(s): [round(x, 4) for x in v] for s, v in runs.items()},
                       ratio={str(s): round(v / t[1], 3) for s, v in t.items()})
            print(json.dumps(row), flush=True)
            rows.append(row)
    return rows


@torch.no_grad()
def draft_cost(draft, quick):
    rows = []
    for b in (1, 4):
        ms = step_ms(draft, b, 1, 10 if quick else 100)
        for k in (2, 4, 8):
            logits = torch.randn(b, k + 1, 32000, device=DEV).to(torch.bfloat16)
            prop = logits[:, :k].argmax(-1)
            unfinished = torch.ones(b, dtype=torch.long, device=DEV)
            from libai_b200 import ops

            n0 = ops.launch_count()
            OF.spec_accept(logits, prop, unfinished, 2, 0)
            launches = ops.launch_count() - n0
            acc = _events_ms(lambda: OF.spec_accept(logits, prop, unfinished, 2, 0), 50 if quick else 500)
            row = dict(batch=b, k=k, draft_step_ms=round(ms, 4), accept_us=round(acc * 1e3, 2),
                       accept_launches=launches)
            print(json.dumps(row), flush=True)
            rows.append(row)
    return rows


def end_to_end(target, draft, quick):
    new = 32 if quick else 256
    configs = [("greedy", 0)] + [(p, k) for p in ("assistant", "prompt_lookup") for k in (2, 4, 8)]
    counter = {"n": 0}
    verify = Generator._verify_step

    def counted(model, block):
        counter["n"] += 1
        return verify(model, block)

    Generator._verify_step = counted
    results = {}
    try:
        for rnd in range(2):   # round 0 is the warm-up
            for b in (1, 4):
                ids = torch.randint(3, 32000, (b, CTX), device=DEV, generator=torch.Generator(device=DEV).manual_seed(b))
                for proposer, k in configs:
                    kw = dict(max_length=CTX + new, eos_token_id=None, decode_graphs=True)
                    if proposer == "assistant":
                        kw.update(assistant_model=draft, num_assistant_tokens=k)
                    elif proposer == "prompt_lookup":
                        kw.update(prompt_lookup_num_tokens=k)
                    counter["n"] = 0
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    out = target.generate(ids, **kw)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    if rnd == 0:
                        continue
                    it = counter["n"]
                    # each iteration emits n + 1 tokens; the prefill emits the first
                    accepted = (new - 1 - it) / it if it else None
                    row = dict(batch=b, proposer=proposer, k=k, tokens_per_s=round(b * new / dt, 2),
                               ms_per_token=round(dt * 1e3 / new, 3), iterations=it,
                               acceptance=None if accepted is None else round(accepted / k, 4))
                    results.setdefault((b, proposer, k), row)
                    key = (b, "greedy", 0)
                    if key in results and proposer != "greedy":
                        row["speedup_vs_greedy"] = round(results[key]["ms_per_token"] / row["ms_per_token"], 3)
                    print(json.dumps(row), flush=True)
                    del out
    finally:
        Generator._verify_step = verify
    return list(results.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "speculative_bench.json"))
    ap.add_argument("--quick", action="store_true", help="fewer layers and tokens (a rehearsal, not a measurement)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("speculative_bench needs a CUDA device")
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    info = gpu_info()
    print(json.dumps(info), flush=True)
    layers, draft_layers = (2, 2) if a.quick else (32, 22)
    result = dict(info, layers=layers, draft_layers=draft_layers, context=CTX)
    draft = tiny_llama(draft_layers)
    result["draft"] = draft_cost(draft, a.quick)
    target = llama_7b(layers)
    result["e2e"] = end_to_end(target, draft, a.quick)
    models = {"bf16": target}
    models["fp8"] = quantize_weights_fp8_(llama_7b(layers))
    result["verify"] = verify_cost(models, a.quick)
    del models["fp8"]
    models = {"int4": quantize_weights_int4_(llama_7b(layers))}
    result["verify"] += verify_cost(models, a.quick)
    result["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
