"""The paged flash-attention prefill against the path it replaces, per attention layer, at a Llama-7B attention shape.

    python dev/paged_prefill_bench.py [--out OUT.json] [--quick]

Llama-7B attention: 32 query and 32 K/V heads of 128.  A paged cache holds ``past + s`` rows per sequence at shuffled
page ids; ``s`` new queries attend causally over them.  Two arms, per layer:

- ``gather``: what a paged step of more than 16 tokens ran before, ``OF.decode_attention_paged_ref`` with ``past``:
  the K and V rows ``[:past + s]`` gathered into contiguous tensors (``kv_pages_gather``, one host sync each), then
  the contiguous flash kernel;
- ``paged``: ``OF.attention_paged``, the flash kernel reading the pages in place.

Each case runs both arms alternately, after a warm-up of both, for ``--rounds`` rounds of ``--iters`` calls each, and
reports the median over rounds of the mean time per call (CUDA events around a round: the gather arm's host syncs are
part of its time), and whether the two outputs are equal bit for bit.  The card's name and power limit are read in
the same launch.  Cases: batch 1 and 4, ``past`` in {0, 1024, 4096}, ``s`` in {64, 512}.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from libai_b200.ops import functional as OF  # noqa: E402

HEADS, DIM = 32, 128


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        out = torch.cuda.get_device_name()
    return out


def case(b, past, s, gen):
    Sk = past + s
    M = -(-Sk // 64)
    P = b * M
    table = torch.randperm(P, generator=gen).to(torch.int32).view(b, M).cuda()
    k = torch.randn(P, HEADS, 64, DIM, generator=gen).to("cuda", torch.bfloat16)
    v = torch.randn(P, HEADS, 64, DIM, generator=gen).to("cuda", torch.bfloat16)
    q = torch.randn(b, s, HEADS, DIM, generator=gen).to("cuda", torch.bfloat16)
    seqlens = torch.full((b,), past, dtype=torch.int32, device="cuda")
    start = torch.zeros(b, dtype=torch.int32, device="cuda")
    scale = DIM ** -0.5
    arms = {
        "gather": lambda: OF.decode_attention_paged_ref(q, k, v, table, seqlens, start, scale=scale, past=past),
        "paged": lambda: OF.attention_paged(q, k, v, table, past, start, scale=scale),
    }
    return arms


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paged_prefill_bench: needs a GPU")
    gen = torch.Generator().manual_seed(0)
    grid = [(1, 0, 64)] if a.quick else [(b, p, s) for b in (1, 4) for p in (0, 1024, 4096) for s in (64, 512)]
    results = {"card": card(), "cases": []}
    print(results["card"], flush=True)
    for b, past, s in grid:
        arms = case(b, past, s, gen)
        outs = {name: fn() for name, fn in arms.items()}
        equal = torch.equal(outs["gather"], outs["paged"])
        for fn in arms.values():   # warm-up
            timed(fn, 3)
        times = {name: [] for name in arms}
        for _ in range(a.rounds):
            for name, fn in arms.items():
                times[name].append(timed(fn, a.iters))
        row = {"batch": b, "past": past, "s": s, "equal": equal,
               **{f"{name}_ms": statistics.median(t) for name, t in times.items()}}
        row["speedup"] = row["gather_ms"] / row["paged_ms"]
        results["cases"].append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
