"""Rectangular flash-attention timings on one GPU.

    python dev/rect_attn_bench.py [--out output/rect_attn_bench.json] [--quick] [--skip-e2e]

Kernel level: forward + backward milliseconds (median over CUDA events, alternated arms) of ``OF.attention`` on the
native kernels, of ``attention_ref`` (fp32 math with autograd, the path these shapes took before) and of PyTorch SDPA
on the same bf16 tensors, for
  * MT5-base-shaped cross-attention: 12 heads of 64, decoder 128 against encoder 512, batch 16, full;
  * chunked prefill: 512 new queries against 4096 or 16384 keys, causal with bottom-right alignment, 32 heads of 128
    (MHA and 32 / 8 GQA), batch 1 and 8.  SDPA gets the bottom-right mask as a boolean tensor.
TFLOP/s count the non-masked score and context products (4·Sq·Sk·D per head forward, 2.5x that backward; causal
pairs exactly).  The grid of the forward is ceil(Sq / 128)·A·B CTAs, so batch 1 with Sq = 512 fills 128 of 132 SMs.

End to end: ``generate()`` on a randomly initialised Llama-7B-shaped model (32 layers, hidden 4096, 32 heads,
intermediate 11008), batch 16, left-padded prompts of lengths spread evenly over 128-2048.  The native arm prefills
with the flash kernel and ``kv_start``; the reference arm is the previous path: the dense ``CasualMask`` and
``attention_ref`` for the prefill (``OF.attention_supported`` forced to False; the decode steps stay native in both).
Reported: prefill seconds, peak allocated memory of the prefill, new tokens/s of ``generate()``.  An out-of-memory
error is reported as such.

The card name, power limit and SM clock are printed with the figures and stored in the JSON output.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from dev.decode_bench import gpu_info  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402


def _fwd_bwd(fn, q, k, v, go):
    def run():
        for t in (q, k, v):
            t.grad = None
        fn(q, k, v).backward(go)
    return run


def _time_alternated(arms, iters):
    """Median ms per arm; the arms are launched in turn so that clock and neighbour drift hit all of them alike."""
    for run in arms.values():
        if run is not None:
            run()
    times = {name: [] for name in arms}
    for _ in range(iters):
        for name, run in arms.items():
            if run is None:
                continue
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    return {name: (statistics.median(t) if t else None) for name, t in times.items()}


def _oom_safe(run):
    try:
        run()
        torch.cuda.synchronize()
        return run
    except torch.OutOfMemoryError:
        torch.cuda.empty_cache()
        return None


def kernel_level(quick):
    cases = [("mt5-base cross", 16, 12, 12, 64, 128, 512, False)]
    for B in (1, 8):
        for sk in ((4096,) if quick else (4096, 16384)):
            for G in (32, 8):
                cases.append((f"chunked prefill {32}/{G}", B, 32, G, 128, 512, sk, True))
    rows = []
    for name, B, A, G, D, sq, sk, causal in cases:
        g = torch.Generator(device="cuda").manual_seed(0)
        q = torch.randn(B, A, sq, D, device="cuda", generator=g, dtype=torch.bfloat16).requires_grad_()
        k = torch.randn(B, G, sk, D, device="cuda", generator=g, dtype=torch.bfloat16).requires_grad_()
        v = torch.randn(B, G, sk, D, device="cuda", generator=g, dtype=torch.bfloat16).requires_grad_()
        go = torch.randn(B, A, sq, D, device="cuda", generator=g, dtype=torch.bfloat16)
        scale = D ** -0.5
        vis = OF.visible_keys(sq, sk, causal=causal, device="cuda")
        native = _fwd_bwd(lambda q, k, v: OF.attention(q, k, v, causal=causal, scale=scale), q, k, v, go)
        ref = _fwd_bwd(lambda q, k, v: OF.attention_ref(q, k, v, causal=causal, scale=scale), q, k, v, go)
        sdpa = _fwd_bwd(lambda q, k, v: torch.nn.functional.scaled_dot_product_attention(
            q, k, v, attn_mask=vis if causal else None, scale=scale, enable_gqa=G != A), q, k, v, go)
        arms = {"native": native, "attention_ref": _oom_safe(ref), "sdpa": _oom_safe(sdpa)}
        ms = _time_alternated(arms, 5 if quick else 20)
        pairs = float(vis.sum()) * B * A
        flop = pairs * D * 4 * 3.5
        row = dict(case=name, B=B, A=A, G=G, D=D, Sq=sq, Sk=sk, causal=causal,
                   **{f"{k}_ms": (None if v is None else round(v, 3)) for k, v in ms.items()},
                   native_tflops=round(flop / (ms["native"] * 1e-3) / 1e12, 1))
        for other in ("attention_ref", "sdpa"):
            row[f"native_speedup_vs_{other}"] = None if ms[other] is None else round(ms[other] / ms["native"], 2)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del q, k, v, go
        torch.cuda.empty_cache()
    return rows


def end_to_end(quick):
    from libai_b200.config import DictConfig
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    layers = 4 if quick else 32
    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=32000, hidden_size=4096, intermediate_size=11008,
                          num_attention_heads=32, max_position_embeddings=4096, rms_norm_eps=1e-6,
                          initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device="cuda:0", seed=1234):
        model = LlamaForCausalLM(cfg).eval()
    B, S, new = 16, 2048, 64
    lens = [int(128 + i * (S - 128) / (B - 1)) for i in range(B)]
    g = torch.Generator(device="cuda").manual_seed(0)
    ids = torch.zeros(B, S, dtype=torch.long, device="cuda")
    am = torch.zeros_like(ids)
    for b, n in enumerate(lens):
        ids[b, S - n:] = torch.randint(3, 32000, (n,), device="cuda", generator=g)
        am[b, S - n:] = 1
    real_supported = OF.attention_supported

    def arm(name):
        OF.attention_supported = real_supported if name == "native" else (lambda *a, **k: False)
        try:
            with torch.no_grad():
                model.allocate_kv_cache(B, S + new)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                t0 = time.perf_counter()
                model(ids, attention_mask=am, use_cache=True)
                torch.cuda.synchronize()
                prefill = time.perf_counter() - t0
                peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
                model.set_cache(None)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.generate(ids, attention_mask=am, max_new_tokens=new, eos_token_id=None, pad_token_id=0)
                torch.cuda.synchronize()
                total = time.perf_counter() - t0
            return dict(prefill_s=prefill, prefill_peak_gib=peak, generate_s=total, new_tokens_per_s=B * new / total)
        except torch.OutOfMemoryError:
            model.set_cache(None)
            torch.cuda.empty_cache()
            return "OOM"
        finally:
            OF.attention_supported = real_supported

    for name in ("native", "reference"):   # warm-up of both paths
        arm(name)
    results = {"native": [], "reference": []}
    for _ in range(1 if quick else 3):
        for name in results:
            results[name].append(arm(name))
    rows = []
    for name, runs in results.items():
        if any(r == "OOM" for r in runs):
            row = dict(arm=name, result="OOM")
        else:
            row = dict(arm=name, **{k: round(statistics.median(r[k] for r in runs), 3) for k in runs[0]})
        row.update(layers=layers, B=B, prompt_lengths=f"{lens[0]}-{lens[-1]}", padded_to=S, new_tokens=new)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "rect_attn_bench.json"))
    ap.add_argument("--quick", action="store_true", help="a subset of the sizes (a rehearsal, not a measurement)")
    ap.add_argument("--skip-e2e", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rect_attn_bench needs a GPU")
    info = gpu_info()
    print(json.dumps(info), flush=True)
    res = dict(info, kernel=kernel_level(a.quick))
    if not a.skip_e2e:
        res["end_to_end"] = end_to_end(a.quick)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
