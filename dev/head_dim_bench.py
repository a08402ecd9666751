"""Attention at the head dims of the shipped recipes on one GPU.

    python dev/head_dim_bench.py [--out output/head_dim_bench.json] [--iters 20]

Forward + backward milliseconds (median over CUDA events, arms alternated, every arm warmed up first) and the peak
memory allocated during one forward + backward, for three arms on the same bf16 tensors:
  * ``native``: ``OF.attention`` on the flash kernels;
  * ``attention_ref``: fp32 math with autograd over a materialised ``[b, a, sq, sk]`` score tensor, the path these head
    dims took before the kernels accepted them;
  * ``sdpa``: PyTorch ``scaled_dot_product_attention`` (the masks and the bias as an ``attn_mask``).
Shapes (batch chosen so that one call does a few GFLOP):
  * GPT-2 recipe: 16 heads of 24, s 1024, causal, batch 8;
  * T5 (384 / 12): 12 heads of 32, s 512, a learned dense bias [1, 12, s, s] (with its gradient), batch 16;
  * BERT-large recipe: 16 heads of 48, s 512, right padding through ``kv_lens`` (lengths spread over 256-512),
    batch 16;
  * ViT-H/14, ViT-g/14, ViT-G/14: 16 heads of 80, 88, 104, 257 tokens, full, batch 64.
Each shape is repeated at the tile width its head dim runs on (64 or 128), with the same number of heads: the native
time at d against the native time at the tile width is what the zero-filled columns cost.

The card name, power limit and SM clock are printed with the figures and stored in the JSON output.
"""
import argparse
import json
import os
import statistics
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from dev.decode_bench import gpu_info  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402

# name, batch, heads, seq, head dim, kind
RECIPES = [
    ("gpt2 recipe", 8, 16, 1024, 24, "causal"),
    ("t5 384/12", 16, 12, 512, 32, "bias"),
    ("bert-large recipe", 16, 16, 512, 48, "kv_lens"),
    ("vit-h/14", 64, 16, 257, 80, "full"),
    ("vit-g/14", 64, 16, 257, 88, "full"),
    ("vit-G/14", 64, 16, 257, 104, "full"),
]


def _tile(d):
    return 64 if d <= 64 else 128


def _arms(B, A, S, D, kind):
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(B, A, S, D, device="cuda", generator=g, dtype=torch.bfloat16).requires_grad_()
               for _ in range(3))
    go = torch.randn(B, A, S, D, device="cuda", generator=g, dtype=torch.bfloat16)
    scale = D ** -0.5
    causal = kind == "causal"
    bias = kv_lens = None
    vis = OF.visible_keys(S, S, causal=causal, device="cuda")
    if kind == "bias":
        bias = (torch.randn(1, A, S, S, device="cuda", generator=g) * 2).bfloat16().requires_grad_()
    if kind == "kv_lens":
        kv_lens = torch.tensor([S // 2 + i * (S - S // 2) // (B - 1) for i in range(B)], dtype=torch.int32,
                               device="cuda")
        vis = OF.visible_keys(S, S, causal=False, kv_lens=kv_lens, device="cuda")
    leaves = [t for t in (q, k, v, bias) if t is not None]

    def fwd_bwd(fn):
        def run():
            for t in leaves:
                t.grad = None
            fn().backward(go)
        return run

    mask = vis if kind == "kv_lens" else None
    sdpa_mask = bias if bias is not None else mask
    return {
        "native": fwd_bwd(lambda: OF.attention(q, k, v, causal=causal, scale=scale, bias=bias, kv_lens=kv_lens)),
        "attention_ref": fwd_bwd(lambda: OF.attention_ref(q, k, v, causal=causal, scale=scale, mask=mask, bias=bias)),
        "sdpa": fwd_bwd(lambda: torch.nn.functional.scaled_dot_product_attention(
            q, k, v, attn_mask=sdpa_mask, is_causal=causal, scale=scale)),
    }


def _peak_gib(run):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    run()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def _time_alternated(arms, iters):
    """Median ms per arm; the arms are launched in turn so that clock and neighbour drift hit all of them alike."""
    for run in arms.values():
        run()
    times = {name: [] for name in arms}
    for _ in range(iters):
        for name, run in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    return {name: statistics.median(t) for name, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "head_dim_bench.json"))
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("head_dim_bench needs a GPU")
    info = gpu_info()
    print(json.dumps(info), flush=True)
    rows = []
    for name, B, A, S, d, kind in RECIPES:
        for D in (d, _tile(d)):
            arms = _arms(B, A, S, D, kind)
            # the native arm must really run the kernels at this head dim
            assert OF.flash_head_dim_supported(D)
            ms = _time_alternated(arms, a.iters)
            peak = {arm: _peak_gib(run) for arm, run in arms.items()}
            row = dict(case=name, B=B, A=A, S=S, D=D, kind=kind, padded_from=None if D == d else d,
                       **{f"{arm}_ms": round(t, 3) for arm, t in ms.items()},
                       **{f"{arm}_peak_gib": round(p, 3) for arm, p in peak.items()},
                       native_speedup_vs_ref=round(ms["attention_ref"] / ms["native"], 2),
                       native_speedup_vs_sdpa=round(ms["sdpa"] / ms["native"], 2))
            rows.append(row)
            print(json.dumps(row), flush=True)
            del arms
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
