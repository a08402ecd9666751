"""Eager against CUDA-graph decoding (``generate(decode_graphs=True)``) on one GPU.

    python dev/decode_graph_bench.py [--out output/decode_graph_bench.json] [--quick]

``generate()`` on randomly initialised bf16 models, eager and graph runs alternated in one launch (a warm-up round of
both, then the measured round):

- Llama-7B shape (32 layers, hidden 4096, 32 heads), a 512-token prompt and 256 new tokens, at batch 1 and 16 on a bf16
  cache, and at batch 1 with an FP8 cache and FP8 weights;
- GPT-2 medium (24 layers, hidden 1024, 16 heads), a 512-token prompt and 256 new tokens, batch 1;
- mT5-base (12 + 12 layers, hidden 768, 12 heads, vocabulary 250112), a 512-token encoder input and 256 new tokens,
  greedy at batch 1 and 4-beam search at batch 4.

Per run: new tokens per second (host clock around ``generate()``, synchronised), device milliseconds per decode step
(CUDA events at the start of the third decode step and after the last one), the host time to enqueue a step (the
median host time of one ``model(**inputs)`` or graph replay), ``ops.launch_count()`` per decode step (median), the
capture time, the peak memory (``max_memory_allocated``, the graph's private pool included) and whether the tokens equal
the eager run's.  The card name, power limit and SM clock are read in the same launch.
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
from libai_b200 import ops  # noqa: E402
from libai_b200.config import DictConfig  # noqa: E402
from libai_b200.inference import decode_graph, quantize_weights_fp8_  # noqa: E402
from libai_b200.inference.generator.generation_utils import Generator  # noqa: E402
from libai_b200.layers._param import param_defaults  # noqa: E402
from libai_b200.utils import distributed as dist  # noqa: E402

DEV = "cuda:0"


def llama_7b(layers):
    from libai_b200.models import LlamaForCausalLM

    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=32000, hidden_size=4096, intermediate_size=11008,
                          num_attention_heads=32, max_position_embeddings=4096, rms_norm_eps=1e-6,
                          initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return LlamaForCausalLM(cfg).eval()


def gpt2_medium(layers):
    from projects.MagicPrompt.gpt2 import GPTModel

    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=50257, hidden_size=1024, ffn_hidden_size=4096,
                          num_attention_heads=16, max_seq_length=1024, embedding_dropout_prob=0.0,
                          attention_dropout_prob=0.0, output_dropout_prob=0.0, layernorm_epsilon=1e-5,
                          initializer_range=0.02, use_scaled_init_for_output_weights=True, bias_gelu_fusion=True,
                          bias_dropout_fusion=True, scale_mask_softmax_fusion=False, apply_query_key_layer_scaling=True,
                          apply_residual_post_layernorm=False, amp_enabled=False, eos_token_id=50256, pad_token_id=0,
                          bos_token_id=50256))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return GPTModel(cfg).eval()


def mt5_base(layers):
    from projects.MT5.mt5_model import MT5Model

    cfg = DictConfig(dict(vocab_size=250112, hidden_size=768, hidden_layers=layers, num_attention_heads=12, head_size=64,
                          intermediate_size=2048, embedding_dropout_prob=0.0, hidden_dropout_prob=0.0,
                          attention_probs_dropout_prob=0.0, relative_attention_num_buckets=32, initializer_range=0.02,
                          layernorm_eps=1e-6, amp_enabled=False, model_type="mt5", padding_idx=0,
                          is_encoder_decoder=True, tie_word_embeddings=False, eos_token_id=1, pad_token_id=0,
                          decoder_start_token_id=0, use_cache=True))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return MT5Model(cfg).eval()


class StepProbe:
    """Times every decode step of a ``generate()`` call: the host time of the model call (or replay), its launches,
    and CUDA events at the start of each step."""

    def __init__(self):
        self.host, self.launches, self.events = [], [], []
        self.step = Generator._decode_step

    def __enter__(self):
        probe = self

        def timed(model, input_ids, model_kwargs):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            probe.events.append(ev)
            inputs = model._model_inputs(input_ids, model_kwargs)
            n0, t0 = ops.launch_count(), time.perf_counter()
            if model._decode_graphs is not None:
                out = decode_graph.step(model, inputs, model._decode_graphs)
            else:
                out = model(**inputs)
            probe.host.append(time.perf_counter() - t0)
            probe.launches.append(ops.launch_count() - n0)
            return out

        Generator._decode_step = timed
        return self

    def __exit__(self, *exc):
        Generator._decode_step = self.step


def run(model, ids, new, graphs, **kw):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    with StepProbe() as probe, torch.no_grad():
        t0 = time.perf_counter()
        seqs = model.generate(ids, max_new_tokens=new, eos_token_id=None, pad_token_id=0, decode_graphs=graphs, **kw)
        end = torch.cuda.Event(enable_timing=True)
        end.record()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    # from the third decode step on (the prefill is step 0; a graph run's first decode step is eager, its second
    # captures)
    later = slice(3, None)
    graph = decode_graph.current_graph(model)
    return seqs, dict(
        new_tokens_per_s=round(ids.shape[0] * new / dt, 1),
        device_ms_per_step=round(probe.events[3].elapsed_time(end) / (len(probe.events) - 3), 3),
        host_enqueue_ms_per_step=round(1e3 * statistics.median(probe.host[later]), 3),
        launches_per_step=int(statistics.median(probe.launches[later])),
        capture_ms=round(graph.capture_ms, 1) if graphs and graph is not None else None,
        peak_gib=round(torch.cuda.max_memory_allocated() / 2**30, 2))


def case(name, model, ids, new, **kw):
    res = {}
    for rep in range(2):                    # alternate eager and graphs; the first round is the warm-up
        for graphs in (False, True):
            model._decode_graph = None      # every graph run captures (the capture time is reported)
            seqs, r = run(model, ids, new, graphs, **kw)
            if rep == 1:
                res["graphs" if graphs else "eager"] = (seqs, r)
    same = bool(torch.equal(res["eager"][0], res["graphs"][0]))
    row = dict(case=name, batch=ids.shape[0], prompt=ids.shape[1], new_tokens=new, same_tokens=same,
               **{f"{k}_{m}": v for k, (_, r) in res.items() for m, v in r.items()})
    row["speedup"] = round(row["graphs_new_tokens_per_s"] / row["eager_new_tokens_per_s"], 2)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="output/decode_graph_bench.json")
    ap.add_argument("--quick", action="store_true", help="4-layer models, 64-token prompts, 32 new tokens")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_graph_bench needs a GPU")
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    info = gpu_info()
    print(json.dumps(info), flush=True)
    layers, prompt, new = (4, 64, 32) if args.quick else (None, 512, 256)
    g = torch.Generator(device=DEV).manual_seed(0)
    rows = []

    m = llama_7b(layers or 32)
    for B in (1, 16):
        ids = torch.randint(3, 32000, (B, prompt), device=DEV, generator=g)
        rows.append(case("llama-7b bf16 cache", m, ids, new))
    quantize_weights_fp8_(m)
    ids = torch.randint(3, 32000, (1, prompt), device=DEV, generator=g)
    rows.append(case("llama-7b fp8 cache + fp8 weights", m, ids, new, kv_cache_dtype="fp8"))
    del m
    torch.cuda.empty_cache()

    m = gpt2_medium(layers or 24)
    ids = torch.randint(3, 50257, (1, prompt), device=DEV, generator=g)
    rows.append(case("gpt2-medium", m, ids, new))
    del m
    torch.cuda.empty_cache()

    m = mt5_base(layers or 12)
    for B, beams in ((1, 1), (4, 4)):
        ids = torch.randint(2, 250112, (B, prompt), device=DEV, generator=g)
        rows.append(case(f"mt5-base {'greedy' if beams == 1 else f'{beams}-beam'}", m, ids, new, num_beams=beams))
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
