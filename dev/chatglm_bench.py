"""ChatGLM3-6B-shaped generation and training timings on one GPU.

    python dev/chatglm_bench.py [--out output/chatglm_bench.json] [--quick] [--tree DIR]

All models are randomly initialised in bf16 with the ChatGLM3-6B shape: hidden 4096, 32 query heads sharing 2 key/value
groups of 128, ffn 13696, vocab 65024, rotary over the first half of every head.

- ``generate()``: the full 28-layer model, greedy, 512-token prompts and 256 new tokens, batch 1 and 16, and a batch of
  16 left-padded by 0..127 tokens.  New tokens per second (batch × 256 over the wall time of the call, after one short
  warm-up call) and the peak memory allocated during the call.
- Training: 4 layers at full width (the optimizer state of all 28 does not fit one GPU), forward + backward of the
  loss, seq 256 (the SFT recipe's 128 + 128) and 2048, micro-batches 1 and 8.  Median milliseconds over timed steps.
- P-tuning v2: the full 28-layer model frozen, a 128-token prefix, seq 256, micro-batch 8, forward + backward.

``--tree`` measures the code of another checkout of the project (the default is this script's own), so two versions can
be alternated in one session.  The card name, power limit and SM clock are stored with the figures.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

DEV = "cuda:0"
HIDDEN, HEADS, GROUPS, HEAD_DIM, FFN, VOCAB, LAYERS = 4096, 32, 2, 128, 13696, 65024, 28


def build(layers, pre_seq_len=None):
    from libai_b200.config import LazyConfig, instantiate
    from libai_b200.layers._param import param_defaults

    c = LazyConfig.load("projects/ChatGLM/configs/chatglm_config.py")
    over = dict(num_layers=layers, hidden_size=HIDDEN, num_attention_heads=HEADS, multi_query_group_num=GROUPS,
                kv_channels=HEAD_DIM, ffn_hidden_size=FFN, padded_vocab_size=VOCAB, pad_token_id=0)
    if pre_seq_len:
        over.update(pre_seq_len=pre_seq_len, prefix_projection=False)
    c = LazyConfig.apply_overrides(c, [f"cfg.{k}={v}" for k, v in over.items()])
    c.model.cfg = c.cfg
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        m = instantiate(c.model)
    return m.to(DEV, torch.bfloat16)


def generation(quick):
    m = build(LAYERS).eval()
    g = torch.Generator(device=DEV).manual_seed(0)
    rows = []
    new = 32 if quick else 256
    for name, batch, padded in (("b1", 1, False), ("b16", 16, False), ("b16_left_padded", 16, True)):
        ids = torch.randint(3, VOCAB, (batch, 512), device=DEV, generator=g)
        kw = {}
        if padded:
            am = torch.ones_like(ids)
            for i in range(1, batch):
                n = int(torch.randint(0, 128, (1,), device=DEV, generator=g))
                ids[i, :n], am[i, :n] = 0, 0
            kw["attention_mask"] = am
        gen = dict(eos_token_id=None, pad_token_id=0, do_sample=False, num_beams=1, use_cache=True, **kw)
        m.generate(ids, max_new_tokens=4, **gen)   # warm-up: kernels, cache allocation
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = m.generate(ids, max_new_tokens=new, **gen)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        made = out.shape[1] - 512   # every sequence runs to max_new_tokens (no eos)
        rows.append(dict(case=name, batch=batch, prompt=512, new_tokens=made, seconds=round(dt, 3),
                         new_tokens_per_s=round(batch * made / dt, 1),
                         peak_gib=round(torch.cuda.max_memory_allocated() / 2**30, 2)))
        print(json.dumps(rows[-1]), flush=True)
    del m
    torch.cuda.empty_cache()
    return rows


def step_ms(m, ids, steps, warmup):
    times = []
    for i in range(warmup + steps):
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m(ids, labels=ids)["loss"].backward()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(times), 2), round(min(times), 2)


def training(quick):
    m = build(4).train()
    g = torch.Generator(device=DEV).manual_seed(1)
    rows = []
    for seq in (256, 2048):
        for batch in (1, 8):
            ids = torch.randint(3, VOCAB, (batch, seq), device=DEV, generator=g)
            med, best = step_ms(m, ids, 5 if quick else 20, 3)
            rows.append(dict(case="train_4_layers", seq=seq, batch=batch, median_ms=med, min_ms=best))
            print(json.dumps(rows[-1]), flush=True)
    del m
    torch.cuda.empty_cache()
    return rows


def ptuning(quick):
    m = build(LAYERS, pre_seq_len=128).train()
    ids = torch.randint(3, VOCAB, (8, 256), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    med, best = step_ms(m, ids, 3 if quick else 10, 2)
    row = dict(case="ptuning_28_layers", prefix=128, seq=256, batch=8, median_ms=med, min_ms=best)
    print(json.dumps(row), flush=True)
    del m
    torch.cuda.empty_cache()
    return [row]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="output/chatglm_bench.json")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="the checkout whose code is measured")
    ap.add_argument("--only", default="", choices=["", "generate", "train", "ptuning"])
    args = ap.parse_args()
    tree = os.path.abspath(args.tree)
    sys.path.insert(0, tree)
    os.chdir(tree)   # the model config is loaded by its path in the tree
    from dev.decode_bench import gpu_info
    from libai_b200 import ops

    ops.load_ext(required=True)
    info = dict(gpu_info(), tree=tree)
    print(json.dumps(info), flush=True)
    rows = []
    if args.only in ("", "generate"):
        rows += generation(args.quick)
    if args.only in ("", "train"):
        rows += training(args.quick)
    if args.only in ("", "ptuning"):
        rows += ptuning(args.quick)
    out = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", args.out)) \
        if not os.path.isabs(args.out) else args.out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
