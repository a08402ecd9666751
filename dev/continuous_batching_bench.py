"""Continuous batching against static batching at a Llama-7B shape (32 layers, 32 heads of 128, hidden 4096, FFN 11008,
vocab 32000; random bf16 weights, no EOS), on one GPU.

Workload: ``--requests`` requests (default 256) with prompts uniform in [64, 2048] tokens and ``max_new_tokens``
uniform in [16, 512], from a fixed seed; a second workload prepends a shared 1,024-token system prompt to every
prompt.  Arms, alternated after a warm-up:

- ``static``: ``generate()`` in batches of ``max_batch`` requests in arrival order, left-padded, on the paged cache,
  each batch run to its largest ``max_new_tokens`` (what a user can do without the engine); useful tokens are each
  request's own ``max_new_tokens``;
- ``engine``: :class:`GenerationEngine` with every request queued at the start;
- each with and without decode graphs; and on the shared-prefix workload the engine with ``prefix_caching`` off and on.

Reported per arm: useful output tokens/s, total time, p50/p90 request latency and time to first token (from the
start of the run), peak memory, and the kernel launches of a decode-only engine step.  Kernel level: the ragged
prefill against one ``attention_paged`` launch per sequence on a ragged batch (8 sequences, q_len in [1, 512], past in
[0, 4096]), outputs checked bit for bit.  One JSON document goes to stdout (and ``--out``); the card's name and power
limit are read in the same launch.

``--kv-cache-dtype fp8`` runs the mixed workload on the engine only, eagerly, in three arms: the bf16 engine as above
(``max_batch`` 32, 1,300 pages), FP8 pools of the same bytes (``max_batch`` 64, 2,521 pages: a page of K and V over 32
layers is 33.55 MB in bf16 and 17.30 MB in E4M3 with its fp32 row scales), and FP8 at ``max_batch`` 32 with 1,300
pages, which isolates the decode kernels from admission.  Its kernel-level pair is the FP8 ragged prefill against the
bf16 ragged prefill on the same batch, the FP8 output checked bit for bit against the bf16 kernel over the dequantized
pools.
"""
import argparse
import json
import random
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from libai_b200 import ops  # noqa: E402
from libai_b200.config import DictConfig  # noqa: E402
from libai_b200.inference import GenerationEngine  # noqa: E402
from libai_b200.layers._param import param_defaults  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402
from libai_b200.utils import distributed as dist  # noqa: E402

DEV = "cuda:0"


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def _model(layers):
    from libai_b200.models import LlamaForCausalLM

    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=32000, hidden_size=4096, intermediate_size=11008,
                          num_attention_heads=32, max_position_embeddings=4096, rms_norm_eps=1e-5,
                          initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=False, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=0):
        return LlamaForCausalLM(cfg).eval()


def _workload(n, seed, system=0):
    rng = random.Random(seed)
    sys_prompt = [rng.randrange(3, 32000) for _ in range(system)]
    return [(sys_prompt + [rng.randrange(3, 32000) for _ in range(rng.randint(64, 2048))], rng.randint(16, 512))
            for _ in range(n)]


def _pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * len(xs)))]


def _static(model, work, max_batch, graphs):
    t0 = time.perf_counter()
    lat, ttft = [], []
    for i in range(0, len(work), max_batch):
        batch = work[i : i + max_batch]
        L = max(len(p) for p, _ in batch)
        ids = torch.zeros(len(batch), L, dtype=torch.long)
        mask = torch.zeros(len(batch), L, dtype=torch.long)
        for b, (p, _) in enumerate(batch):
            ids[b, L - len(p) :] = torch.tensor(p)
            mask[b, L - len(p) :] = 1
        new = max(m for _, m in batch)
        # min_length: no EOS before the batch's largest max_new_tokens (the random model has none of its own)
        model.generate(ids.to(DEV), attention_mask=mask.to(DEV), max_new_tokens=new, min_length=L + new,
                       do_sample=False, use_cache=True, paged_kv_cache=True, decode_graphs=graphs, pad_token_id=0)
        torch.cuda.synchronize()
        done = time.perf_counter() - t0
        lat += [done] * len(batch)
        ttft += [done] * len(batch)   # generate() returns the batch's tokens at its end
    total = time.perf_counter() - t0
    return total, lat, ttft


def _engine(model, work, max_batch, graphs, prefix=False, num_pages=1300, kv_cache_dtype=None):
    model.kv_cache = model._decode_graph = None   # the static arm's cache and graph
    torch.cuda.empty_cache()
    # by default 1,300 pages of 64 rows: 41.6 GB of bf16 K/V at this shape (22.5 GB in FP8), beside the 13.5 GB of
    # weights; 2,521 FP8 pages take the bytes of 1,300 bf16 ones
    e = GenerationEngine(model, max_batch=max_batch, max_tokens_per_step=2048, num_pages=num_pages,
                         prefix_caching=prefix, decode_graphs=graphs, kv_cache_dtype=kv_cache_dtype)
    t0 = time.perf_counter()
    ids = [e.add_request(p, m) for p, m in work]
    for r in e.requests.values():
        r.t_arrival = t0
    launches = None
    while e.has_unfinished():
        n0 = ops.launch_count()
        e.step()
        if launches is None and e.cache.chunks == 0 and e.steps > 2 and not e.waiting:
            launches = ops.launch_count() - n0
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    reqs = [e.requests[i] for i in ids]
    return (total, [r.t_done - t0 for r in reqs], [r.t_first - t0 for r in reqs], launches, e.reused_pages)


def _arm(name, fn, useful):
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    total, lat, ttft = out[:3]
    res = {"arm": name, "useful_tokens_per_s": useful / total, "total_s": total, "latency_p50_s": _pct(lat, 0.5),
           "latency_p90_s": _pct(lat, 0.9), "ttft_p50_s": _pct(ttft, 0.5), "ttft_p90_s": _pct(ttft, 0.9),
           "peak_gb": torch.cuda.max_memory_allocated() / 1e9}
    if len(out) > 3:
        res["launches_per_decode_step"], res["reused_pages"] = out[3], out[4]
    print(json.dumps(res), flush=True)
    return res


def _kernel(reps=20, fp8=False):
    rng = random.Random(0)
    q_lens = [rng.randint(1, 512) for _ in range(8)]
    past = [rng.randint(0, 4096) for _ in range(8)]
    G, A, D = 32, 32, 128
    need = [-(-(s + p) // 64) for s, p in zip(q_lens, past)]
    mp, P = max(need), sum(need)
    perm = torch.randperm(P).tolist()
    table = torch.full((8, mp), -1, dtype=torch.int32)
    for n in range(8):
        table[n, : need[n]] = torch.tensor([perm.pop() for _ in range(need[n])], dtype=torch.int32)
    table = table.to(DEV)
    k = torch.randn(P, G, 64, D, device=DEV).to(torch.bfloat16)
    v = torch.randn(P, G, 64, D, device=DEV).to(torch.bfloat16)
    q = torch.randn(sum(q_lens), A, D, device=DEV).to(torch.bfloat16)
    cu = torch.tensor([0] + torch.tensor(q_lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    pa = torch.tensor(past, dtype=torch.int32, device=DEV)
    tiles = OF.varlen_tiles(q_lens, past).to(DEV)
    c = cu.tolist()

    def ragged():
        return OF.attention_paged_varlen(q, k, v, table, cu, pa, tiles, scale=D ** -0.5)

    if fp8:
        (k8, ks), (v8, vs) = OF.kv_cache_quantize_ref(k), OF.kv_cache_quantize_ref(v)
        kd, vd = OF.kv_cache_dequant(k8, ks), OF.kv_cache_dequant(v8, vs)

        def ragged_fp8():
            return OF.attention_paged_varlen(q, k8, v8, table, cu, pa, tiles, scale=D ** -0.5, k_scale=ks,
                                             v_scale=vs)

        equal = torch.equal(ragged_fp8(), OF.attention_paged_varlen(q, kd, vd, table, cu, pa, tiles, scale=D ** -0.5))
        pair = (("fp8", ragged_fp8), ("bf16", ragged))
    else:
        def per_seq():
            return [OF.attention_paged(q[None, c[n] : c[n + 1]], k, v, table[n : n + 1], past[n], scale=D ** -0.5)
                    for n in range(8)]

        o, refs = ragged(), per_seq()
        equal = all(torch.equal(o[c[n] : c[n + 1]], refs[n][0]) for n in range(8))
        pair = (("ragged", ragged), ("per_sequence", per_seq))
    times = {}
    for name, fn in pair * 2:
        fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        times[name] = s.elapsed_time(e) / reps
    res = {"kernel": "ragged_prefill_fp8" if fp8 else "ragged_prefill", "q_lens": q_lens, "past": past,
           "bit_equal": equal, **{f"{name}_ms": t for name, t in times.items()}}
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--out", default=None)
    # the two workloads take minutes each at the default size: one launch can run either
    ap.add_argument("--workload", choices=("mixed", "shared", "both"), default="both")
    ap.add_argument("--kv-cache-dtype", choices=("bf16", "fp8"), default="bf16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("continuous_batching_bench needs a GPU")
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    ops.load_ext(required=True)
    doc = {"card": _card(), "requests": args.requests, "max_batch": args.max_batch, "layers": args.layers,
           "workload": args.workload, "kv_cache_dtype": args.kv_cache_dtype}
    if args.kv_cache_dtype == "fp8":
        doc["workload"] = "mixed"
        doc["kernel"] = _kernel(fp8=True)
        model = _model(args.layers)
        work = _workload(args.requests, 0)
        useful = sum(m for _, m in work)
        # (name, max_batch, num_pages, kv_cache_dtype)
        fp8_arms = (("engine_bf16", 32, 1300, None), ("engine_fp8_same_bytes", 64, 2521, "fp8"),
                    ("engine_fp8", 32, 1300, "fp8"))
        for _, mb, pages, kv in fp8_arms:   # warm-up
            _engine(model, work[:4], mb, False, num_pages=pages, kv_cache_dtype=kv)
        doc["arms"] = [_arm(name, lambda: _engine(model, work, mb, False, num_pages=pages, kv_cache_dtype=kv), useful)
                       for name, mb, pages, kv in fp8_arms]
        text = json.dumps(doc, indent=1)
        if args.out:
            Path(args.out).parent.mkdir(parents=True, exist_ok=True)
            Path(args.out).write_text(text)
        print(text)
        return
    if args.workload != "shared":
        doc["kernel"] = _kernel()
    model = _model(args.layers)
    work = _workload(args.requests, 0)
    shared = _workload(args.requests, 1, system=1024)
    useful = sum(m for _, m in work)
    # warm-up: every arm once on a few requests
    few = work[: min(len(work), 4)]
    if args.workload != "shared":
        _static(model, few, args.max_batch, False)
        _static(model, few, args.max_batch, True)
    _engine(model, few, args.max_batch, False)
    _engine(model, few, args.max_batch, True)
    _engine(model, shared[:4], args.max_batch, True, True)
    arms = []
    if args.workload != "shared":
        for graphs in (False, True):   # alternated: static, engine, static, engine
            g = "+graphs" if graphs else ""
            arms.append(_arm("static" + g, lambda: _static(model, work, args.max_batch, graphs), useful))
            arms.append(_arm("engine" + g, lambda: _engine(model, work, args.max_batch, graphs), useful))
    if args.workload != "mixed":
        useful_shared = sum(m for _, m in shared)
        for prefix in (False, True):
            arms.append(_arm("engine_shared_prefix" + ("+prefix_caching" if prefix else ""),
                             lambda: _engine(model, shared, args.max_batch, True, prefix), useful_shared))
    doc["arms"] = arms
    text = json.dumps(doc, indent=1)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)
    print(text)


if __name__ == "__main__":
    main()
