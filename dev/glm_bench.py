"""GLM generation on the KV cache and the prefix-LM flash kernels, timed on one GPU.

    python dev/glm_bench.py --parent-model OLD/projects/GLM/modeling_glm.py [--out output/glm_bench.json] [--new N]
                            [--shapes glm-large,glm-10b] [--only generate|kernel]

- ``generate()``: randomly initialised bf16 models shaped like GLM-large (24 layers × 1024, 16 heads of 64) and GLM-10B
  (48 × 4096, 64 heads of 64), vocab 30592; greedy, 128 new tokens, batch 1 and 16.  Contexts are laid out by the
  tokenizer's own code (``GLMTokenizerMixin.build_inputs_for_generation``), right-padded to 896 tokens with lengths
  spread evenly from 128 to 896 (batch 1: one 896-token context).  New tokens per second (batch × new tokens over the
  wall time of the call, after a short warm-up call), the time of the prefill (median of 3) and the peak memory
  allocated during the call.  ``--parent-model`` is the ``modeling_glm.py`` of another version (the hidden-state
  memory path before the KV cache), run on this tree's library with the same weights; the versions alternate,
  ``--reps`` rounds each (one model resident at a time), and the fraction of equal generated tokens is recorded.
- The kernel alone: ``attn_fwd`` and ``attn_bwd`` with ``prefix_lens`` at 0, S/4, S/2 and S next to the causal and
  non-causal kernels, S = 1024, head dim 64, 4 × 16 heads; median microseconds over CUDA events.

The card name, power limit and SM clock are stored with the figures.
"""
import argparse
import importlib.util
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = "cuda:0"
VOCAB, CONTEXT, NEW = 30592, 896, 128
SHAPES = {"glm-large": (24, 1024, 16), "glm-10b": (48, 4096, 64)}   # layers, hidden, heads
MASK, SOP, EOP, PAD = 30000, 30001, 30002, 0


def load_module(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build(mod, shape):
    from libai_b200.config import LazyConfig
    from libai_b200.layers._param import param_defaults

    layers, hidden, heads = SHAPES[shape]
    cfg = LazyConfig.load(os.path.join(ROOT, "projects/GLM/configs/glm_inference.py")).cfg
    cfg.update(dict(vocab_size=VOCAB, hidden_size=hidden, num_layers=layers, num_attention_heads=heads))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return mod.GLMForConditionalGeneration(cfg).eval()


def contexts(batch, new):
    from projects.GLM.tokenizer.glm_tokenizer import GLMTokenizerMixin

    class Host:
        mask_token_id, pad_token_id = MASK, PAD

        def convert_tokens_to_ids(self, t):
            return {"<|startofpiece|>": SOP, "<|endofpiece|>": EOP, "[gMASK]": MASK + 3, "[sMASK]": MASK + 4}[t]

    class Tok(GLMTokenizerMixin, Host):
        pass

    g = torch.Generator().manual_seed(batch)
    ids = torch.randint(100, 29000, (batch, CONTEXT), generator=g)
    am = torch.ones_like(ids)
    lens = [CONTEXT] if batch == 1 else [128 + (CONTEXT - 128) * i // (batch - 1) for i in range(batch)]
    for i, n in enumerate(lens):
        ids[i, n // 2] = MASK
        ids[i, n:], am[i, n:] = PAD, 0
    inp = Tok().build_inputs_for_generation({"input_ids": ids, "attention_mask": am}, max_gen_length=new)
    return {k: v.to(DEV) for k, v in inp.items()}


@torch.no_grad()
def run_generate(m, inp, new):
    ids = inp["input_ids"]
    s = ids.shape[1]
    gen = dict(position_ids=inp["position_ids"], generation_attention_mask=inp["generation_attention_mask"],
               eos_token_id=None, pad_token_id=PAD, do_sample=False, num_beams=1, use_cache=True)
    m.generate(ids, max_length=s + 2, **gen)   # warm-up: kernels, cache allocation
    prefill = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.generate(ids, max_length=s + 1, **gen)
        torch.cuda.synchronize()
        prefill.append(time.perf_counter() - t0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = m.generate(ids, max_length=s + new, **gen)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    made = out.shape[1] - s
    return out[:, s:], dict(new_tokens=made, seconds=round(dt, 3), new_tokens_per_s=round(ids.shape[0] * made / dt, 1),
                            prefill_ms=round(1e3 * statistics.median(prefill), 1),
                            peak_gib=round(torch.cuda.max_memory_allocated() / 2**30, 2))


def generation(parent_path, reps, new, shapes):
    """One model resident at a time (two GLM-10B copies and their caches do not fit 80 GB together): each round builds
    every version from the same seed, runs both batches, and frees it before the next version."""
    from projects.GLM import modeling_glm as this

    versions = {"this": this}
    if parent_path:
        versions["parent"] = load_module(os.path.abspath(parent_path), "parent_modeling_glm")
    rows = []
    for shape in shapes:
        outs = {}
        for rep in range(reps):
            for v, mod in versions.items():
                m = build(mod, shape)
                for batch in (1, 16):
                    toks, row = run_generate(m, contexts(batch, NEW), new)
                    outs[(v, batch)] = toks
                    rows.append(dict(case="generate", model=shape, version=v, batch=batch, rep=rep, **row))
                    print(json.dumps(rows[-1]), flush=True)
                del m
                torch.cuda.empty_cache()
        for batch in (1, 16):
            if ("parent", batch) in outs:
                same = (outs[("parent", batch)] == outs[("this", batch)]).float().mean().item()
                rows.append(dict(case="generate_tokens_equal", model=shape, batch=batch, fraction=round(same, 4)))
                print(json.dumps(rows[-1]), flush=True)
    return rows


def time_us(call, iters):
    for _ in range(5):
        call()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3)
    return statistics.median(times)


def kernel(iters):
    from libai_b200 import ops

    ext = ops.load_ext(required=True)
    B, A, S, d = 4, 16, 1024, 64
    g = torch.Generator(device=DEV).manual_seed(0)
    q, k, v, do = (torch.randn(B, A, S, d, device=DEV, generator=g).bfloat16() for _ in range(4))
    rows = []
    cases = [("causal", True, None), ("prefix_0", True, 0), ("prefix_S/4", True, S // 4), ("prefix_S/2", True, S // 2),
             ("prefix_S", True, S), ("non_causal", False, None)]
    for name, causal, pre in cases:
        extra = {} if pre is None else {"prefix_lens": torch.full((B,), pre, dtype=torch.int32, device=DEV)}
        o, lse, _ = ext.attn_fwd(q, k, v, causal, d ** -0.5, None, None, None, 0.0, 0, None, **extra)
        fwd = time_us(lambda: ext.attn_fwd(q, k, v, causal, d ** -0.5, None, None, None, 0.0, 0, None, **extra), iters)
        bwd = time_us(lambda: ext.attn_bwd(do, q, k, v, o, lse, causal, d ** -0.5, None, None, None, None, 0.0, None,
                                           None, **extra), iters)
        rows.append(dict(case="attn", kind=name, batch=B, heads=A, seq=S, head_dim=d, fwd_median_us=round(fwd, 1),
                         bwd_median_us=round(bwd, 1)))
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-model", default="", help="modeling_glm.py of the version to compare against")
    ap.add_argument("--out", default="output/glm_bench.json")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--new", type=int, default=NEW)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--only", default="", choices=["", "generate", "kernel"])
    args = ap.parse_args()
    os.chdir(ROOT)
    from dev.decode_bench import gpu_info
    from libai_b200 import ops
    from libai_b200.config import DictConfig
    from libai_b200.utils import distributed as dutil

    ops.load_ext(required=True)
    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1)))
    info = gpu_info()
    print(json.dumps(info), flush=True)
    rows = []
    if args.only in ("", "kernel"):
        rows += kernel(100)
    if args.only in ("", "generate"):
        rows += generation(args.parent_model, args.reps, args.new, args.shapes.split(","))
    out = args.out if os.path.isabs(args.out) else os.path.join(ROOT, args.out)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
