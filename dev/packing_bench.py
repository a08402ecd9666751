"""Packed-sequence SFT on one GPU: what packing saves in attention and in a Llama-shaped training step.

    python dev/packing_bench.py [--out results.json]

(a) Attention forward + backward (bf16, causal, grouped heads) on rows of packed documents, with ``doc_start``,
    against the plain causal kernels on the same rows; several seeded document-length distributions.  Reports µs
    and the fraction of forward key tiles and backward (key block, query block) visits the packed kernels run,
    computed by the same arithmetic as the kernels (tests/test_packed_sft_cpu.py mirrors it).
(b) Forward + backward of a Llama-shaped model (bf16, no optimizer step) on one seeded synthetic SFT length
    distribution: every sample padded to the row length, one per row, against the same samples packed.  Reports
    non-padding tokens per second, since the padded run also processes padding.
Times are CUDA-event medians over repeated runs after a warm-up.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from libai_b200.ops import functional as OF  # noqa: E402

DEV = "cuda"


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def doc_lengths(kind, n_tokens, gen):
    """Seeded document lengths summing to at least n_tokens."""
    out, total = [], 0
    while total < n_tokens:
        if kind == "sft":        # log-normal around 250 tokens, Alpaca-like
            n = int(math.exp(5.5 + 0.7 * float(torch.randn((), generator=gen))))
        elif kind == "short":
            n = int(torch.randint(8, 128, (), generator=gen))
        elif kind == "long":
            n = int(torch.randint(512, 2048, (), generator=gen))
        else:
            n = n_tokens
        n = max(2, n)
        out.append(n)
        total += n
    return out


def pack_rows(lengths, L):
    """doc_start [rows, L] of lengths packed in order (a document longer than L is cut at L); tails are one document."""
    rows, cur, used = [], [], 0
    for n in lengths:
        n = min(n, L)
        if used + n > L:
            rows.append(cur)
            cur, used = [], 0
        cur.append(n)
        used += n
    if cur:
        rows.append(cur)
    ds = torch.empty(len(rows), L, dtype=torch.int32)
    for r, docs in enumerate(rows):
        at = 0
        for n in docs + [L - sum(docs)]:
            ds[r, at : at + n] = at
            at += n
    return ds, rows


def visited_fraction(ds):
    """(forward tiles, backward visits) run with doc_start over those of the plain causal kernels."""
    B, S = ds.shape
    i = torch.arange(S)
    beg = torch.minimum(ds.long().clamp(min=0), i[None])
    f_all = f_doc = 0
    for q0 in range(0, S, 128):
        end = (min(q0 + 128, S) + 127) // 128
        f_all += B * end
        f_doc += int((end - beg[:, q0 : q0 + 128].min(1).values // 128).sum())
    b_all = b_doc = 0
    for k0 in range(0, S, 64):
        for q0 in range(k0 // 64 * 64, S, 64):
            b_all += B
            b_doc += int((beg[:, q0 : q0 + 64].min(1).values < k0 + 64).sum())
    return f_doc / f_all, b_doc / b_all


def cuda_time(fn, reps):
    for _ in range(3):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def attention_bench(rows=8, S=4096, G=8, r=4, D=128):
    from libai_b200 import ops

    ext = ops.load_ext(required=True)
    out = []
    for kind in ("sft", "short", "long", "one"):
        gen = torch.Generator().manual_seed(1)
        ds, _ = pack_rows(doc_lengths(kind, rows * S, gen), S)
        ds = ds[:rows].to(DEV)
        B = ds.shape[0]
        qkv = torch.randn(B, S, G, r + 2, D, device=DEV).bfloat16()
        do = torch.randn(B, G * r, S, D, device=DEV).bfloat16()
        q, k, v = OF._packed_views(qkv)

        def step(doc):
            o, lse, _ = ext.attn_fwd(q, k, v, True, D ** -0.5, None, None, None, 0.0, 0, None, doc)
            ext.attn_bwd(do, q, k, v, o, lse, True, D ** -0.5, None, None, None, None, 0.0, None, None, doc)

        plain, packed = [], []
        for _ in range(3):   # alternated rounds
            plain.append(cuda_time(lambda: step(None), 10))
            packed.append(cuda_time(lambda: step(ds), 10))
        fwd_frac, bwd_frac = visited_fraction(ds.cpu())
        res = dict(dist=kind, rows=B, seq=S, heads=G * r, kv_heads=G, head_dim=D,
                   plain_us=round(1e3 * sorted(plain)[1], 1), packed_us=round(1e3 * sorted(packed)[1], 1),
                   fwd_tiles=round(fwd_frac, 3), bwd_visits=round(bwd_frac, 3))
        res["speedup"] = round(res["plain_us"] / res["packed_us"], 2)
        print(json.dumps(res), flush=True)
        out.append(res)
    return out


def step_bench(L=2048, n_samples=96, layers=4, hidden=2048, heads=16, kv_heads=4, inter=5632, vocab=32000):
    from libai_b200.layers._param import param_defaults
    from libai_b200.models.llama_model import LlamaForCausalLM

    gen = torch.Generator().manual_seed(2)
    lens = [min(L, n) for n in doc_lengths("sft", 1, gen)]
    while len(lens) < n_samples:
        lens += [min(L, n) for n in doc_lengths("sft", 1, gen)]
    real = sum(lens)
    ds, rows = pack_rows(lens, L)
    pos = (torch.arange(L)[None] - ds).long()
    ids = torch.randint(1, vocab, (len(rows), L))
    packed = dict(input_ids=ids.to(DEV), labels=ids.to(DEV), position_ids=pos.to(DEV))
    pad_ids = torch.randint(1, vocab, (len(lens), L))
    padded = dict(input_ids=pad_ids.to(DEV), labels=pad_ids.to(DEV))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=3):
        model = LlamaForCausalLM(hidden_layers=layers, vocab_size=vocab, hidden_size=hidden, intermediate_size=inter,
                                 num_attention_heads=heads, num_key_value_heads=kv_heads, max_position_embeddings=L,
                                 amp_enabled=True).to(DEV)

    def run(batch, mb):
        n = batch["input_ids"].shape[0]
        for s in range(0, n, mb):
            part = {k: v[s : s + mb] for k, v in batch.items()}
            model(**part)["lm_loss"].backward()
        model.zero_grad(set_to_none=True)

    mb = 8
    t_pad, t_pk = [], []
    for _ in range(3):
        t_pad.append(cuda_time(lambda: run(padded, mb), 3))
        t_pk.append(cuda_time(lambda: run(packed, mb), 3))
    tp, tk = sorted(t_pad)[1] / 1e3, sorted(t_pk)[1] / 1e3
    res = dict(samples=len(lens), real_tokens=real, row_len=L, padded_rows=len(lens), packed_rows=len(rows),
               fill_padded=round(real / (len(lens) * L), 3), fill_packed=round(real / (len(rows) * L), 3),
               padded_tok_s=round(real / tp), packed_tok_s=round(real / tk), speedup=round(tp / tk, 2),
               model=dict(layers=layers, hidden=hidden, heads=heads, kv_heads=kv_heads, inter=inter, vocab=vocab),
               micro_batch=mb)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="", help="also write the results as JSON to this path")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "packing_bench needs a GPU"
    info = gpu_info()
    print("gpu:", info, flush=True)
    res = dict(gpu=info, attention=attention_bench(), step=step_bench())
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
