"""Grouped-query attention timings on one GPU.

    python dev/gqa_bench.py [--out output/gqa_bench.json] [--quick] [--skip-e2e]

Kernel level, decode: one new query per sample and head over a KV cache holding L keys, for a Llama-3-8B-shaped layer
(32 query / 8 key-value heads of 128) and a Qwen2-7B-shaped layer (28 / 4), B in {1, 8, 32} and L in {1024, 4096,
16384}.  Median microseconds over CUDA events (L2 flushed before every launch) of the native grouped kernel, of the MHA
kernel on the cache expanded with ``repeat_interleave`` (expansion outside the timed region and with it), and of
PyTorch SDPA with ``enable_gqa=True`` on the same cache slices.  Bytes count K and V once per key/value head, plus q and
o; the share is of the H100 SXM's 3.35 TB/s.

Attention training cost: forward + backward of the grouped kernels on the grouped packed projection against the MHA
kernels on a projection whose K/V heads are repeated, at Llama-3-8B-like training shapes and for MQA at batch 1.

End to end: ``generate()`` on a randomly initialised Llama-3-8B-shaped model (32 layers, hidden 4096, 32 / 8 heads,
intermediate 14336), a 512-token prompt and 256 new tokens, batch 1 and 16.

The card name, power limit and SM clock are printed with the figures and stored in the JSON output.
"""
import argparse
import json
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from dev.decode_bench import HBM_BYTES_PER_S, gpu_info, time_us  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402


def decode_kernels(quick):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    sdpa = torch.nn.functional.scaled_dot_product_attention
    rows = []
    for name, A, G, D in (("llama3-8b", 32, 8, 128), ("qwen2-7b", 28, 4, 128)):
        r = A // G
        for B in ((1, 8) if quick else (1, 8, 32)):
            for L in ((1024, 4096) if quick else (1024, 4096, 16384)):
                C = L + 64
                g = torch.Generator(device="cuda").manual_seed(0)
                k = torch.randn(B, G, C, D, device="cuda", generator=g, dtype=torch.bfloat16)
                v = torch.randn(B, G, C, D, device="cuda", generator=g, dtype=torch.bfloat16)
                q = torch.randn(B, 1, A, D, device="cuda", generator=g, dtype=torch.bfloat16)
                lens = torch.full((B,), L - 1, dtype=torch.int32, device="cuda")
                start = torch.zeros(B, dtype=torch.int32, device="cuda")
                scale = D ** -0.5
                out = OF.decode_attention(q, k, v, lens, start, scale=scale)
                ke, ve = k.repeat_interleave(r, 1), v.repeat_interleave(r, 1)
                mha = OF.decode_attention(q, ke, ve, lens, start, scale=scale)
                qh, ks, vs = q.transpose(1, 2), k[:, :, :L], v[:, :, :L]
                ref = sdpa(qh, ks, vs, scale=scale, enable_gqa=True).transpose(1, 2)
                err = float((out.float() - ref.float()).abs().max() / ref.float().abs().max())
                t_gqa = time_us(lambda: OF.decode_attention(q, k, v, lens, start, scale=scale), 50, flush)
                t_mha = time_us(lambda: OF.decode_attention(q, ke, ve, lens, start, scale=scale), 50, flush)
                t_mha_expand = time_us(lambda: OF.decode_attention(q, k[:, :, :L].repeat_interleave(r, 1),
                                                                   v[:, :, :L].repeat_interleave(r, 1),
                                                                   lens, start, scale=scale), 10, flush)
                t_sdpa = time_us(lambda: sdpa(qh, ks, vs, scale=scale, enable_gqa=True), 50, flush)
                nbytes = 2 * B * G * L * D * 2 + 2 * B * A * D * 2
                row = dict(shape=name, A=A, G=G, D=D, B=B, L=L, gqa_us=t_gqa, mha_expanded_cache_us=t_mha,
                           repeat_interleave_plus_mha_us=t_mha_expand, sdpa_gqa_us=t_sdpa, bytes=nbytes,
                           gqa_GBps=nbytes / t_gqa / 1e3, gqa_hbm_share=nbytes / (t_gqa * 1e-6) / HBM_BYTES_PER_S,
                           bit_identical_to_mha_on_expanded=bool(torch.equal(out, mha)), rel_err_vs_sdpa=err)
                rows.append(row)
                print(json.dumps(row), flush=True)
                del k, v, ke, ve
                torch.cuda.empty_cache()
    return rows


def training_attention(quick):
    from libai_b200.ops import load_ext

    ext = load_ext()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    cases = [(1, 32, 8, 4096, 128), (2, 32, 8, 2048, 128), (1, 32, 1, 2048, 128), (4, 16, 4, 1024, 64)]
    for B, A, G, S, D in cases[:2] if quick else cases:
        r = A // G
        g = torch.Generator(device="cuda").manual_seed(0)
        qkv = torch.randn(B, S, G, r + 2, D, device="cuda", generator=g, dtype=torch.bfloat16)
        go = torch.randn(B, S, A, D, device="cuda", generator=g, dtype=torch.bfloat16).permute(0, 2, 1, 3)
        q5, k5, v5 = OF._packed_views(qkv)
        # MHA projection [B, S, A, 3D] with every K/V head repeated
        mq, mk, mv = qkv[:, :, :, :r].reshape(B, S, A, D), qkv[:, :, :, r], qkv[:, :, :, r + 1]
        mha = torch.cat([mq, mk.repeat_interleave(r, 2), mv.repeat_interleave(r, 2)], -1)
        q4, k4, v4 = OF._packed_views(mha)
        sc = D ** -0.5

        def step(q, k, v):
            o, lse, _ = ext.attn_fwd(q, k, v, True, sc, None)
            return ext.attn_bwd(go, q, k, v, o, lse, True, sc, None)

        o5, lse5, _ = ext.attn_fwd(q5, k5, v5, True, sc, None)
        o4, lse4, _ = ext.attn_fwd(q4, k4, v4, True, sc, None)
        row = dict(B=B, A=A, G=G, S=S, D=D, fwd_equal=bool(torch.equal(o5, o4)),
                   gqa_fwd_ms=time_us(lambda: ext.attn_fwd(q5, k5, v5, True, sc, None), 20, flush) / 1e3,
                   mha_fwd_ms=time_us(lambda: ext.attn_fwd(q4, k4, v4, True, sc, None), 20, flush) / 1e3,
                   gqa_bwd_ms=time_us(lambda: ext.attn_bwd(go, q5, k5, v5, o5, lse5, True, sc, None), 20, flush) / 1e3,
                   mha_bwd_ms=time_us(lambda: ext.attn_bwd(go, q4, k4, v4, o4, lse4, True, sc, None), 20, flush) / 1e3,
                   bwd_ctas_gqa=((S + 63) // 64) * G * B, bwd_ctas_mha=((S + 63) // 64) * A * B)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def end_to_end(quick):
    from libai_b200.config import DictConfig
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    layers = 4 if quick else 32
    cfg = DictConfig(dict(hidden_layers=layers, vocab_size=128256, hidden_size=4096, intermediate_size=14336,
                          num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=2048,
                          rms_norm_eps=1e-5, initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0, rope_base=500000.0))
    with param_defaults(dtype=torch.bfloat16, device="cuda:0", seed=1234):
        model = LlamaForCausalLM(cfg).eval()
    prompt, new = (128, 32) if quick else (512, 256)
    rows = []
    for B in (1, 16):
        ids = torch.randint(3, 32000, (B, prompt), device="cuda", generator=torch.Generator("cuda").manual_seed(B))
        for rep in range(2):                     # the first round is the warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.generate(ids, max_new_tokens=new, eos_token_id=None, pad_token_id=0)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
        row = dict(layers=layers, B=B, prompt=prompt, new_tokens=new, seconds=dt, new_tokens_per_s=B * new / dt,
                   kv_cache_heads=model.kv_cache.heads)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "gqa_bench.json"))
    ap.add_argument("--quick", action="store_true", help="a subset of the sizes (a rehearsal, not a measurement)")
    ap.add_argument("--skip-e2e", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gqa_bench needs a CUDA device")
    from libai_b200 import ops

    ops.load_ext(required=True)
    info = gpu_info()
    print(json.dumps(info), flush=True)
    result = dict(info, decode=decode_kernels(a.quick), training_attention=training_attention(a.quick))
    result["e2e"] = [] if a.skip_e2e else end_to_end(a.quick)
    result["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
