"""Continuous batching on FP8 (E4M3) pools, on the reference path: the FP8 ragged reference ops against per-sequence
appends and attention over dequantized rows, the FP8 cache's pools, scales and page accounting, the ``ValueError`` of a
bad ``kv_cache_dtype``, tiny fp32 Llama (MHA and GQA) and BLOOM models run end to end against ``generate()`` on an FP8
cache, and the argument checks of the two FP8 ragged bindings."""
import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference import GenerationEngine
from libai_b200.inference.kv_cache import RaggedPagedKVCache
from libai_b200.models.llama_model import rotary_tables
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests import op_args_cases as C
from tests.test_continuous_batching_cpu import _bloom, _error, _ids, _llama, _ragged, ext  # noqa: F401

FP8 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


def _fp8_ragged(q_lens, past, G=2, D=64, seed=0):
    table, k, v, cu, pa = _ragged(q_lens, past, G=G, D=D, seed=seed)
    (k8, ks), (v8, vs) = OF.kv_cache_quantize_ref(k), OF.kv_cache_quantize_ref(v)
    return table, k8, v8, ks, vs, cu, pa


@pytest.mark.parametrize("alibi", [False, True])
def test_fp8_ragged_attention_ref_is_attention_over_dequantized_rows(alibi):
    q_lens, past = [1, 70, 3, 130], [0, 64, 100, 5]
    table, k8, v8, ks, vs, cu, pa = _fp8_ragged(q_lens, past)
    A, D = 4, 64
    q = torch.randn(sum(q_lens), A, D, generator=torch.Generator().manual_seed(3))
    slopes = torch.tensor([0.5, 0.25, 0.125, 0.0625]) if alibi else None
    o = OF.attention_paged_varlen(q, k8, v8, table, cu, pa, scale=0.125, alibi_slopes=slopes, k_scale=ks, v_scale=vs)
    kd, vd = OF.kv_cache_dequant(k8, ks, q.dtype), OF.kv_cache_dequant(v8, vs, q.dtype)
    assert torch.equal(o, OF.attention_paged_varlen(q, kd, vd, table, cu, pa, scale=0.125, alibi_slopes=slopes))
    for n in range(len(q_lens)):
        qn = q[cu[n] : cu[n + 1]][None]
        ref = OF.decode_attention_paged_ref(qn, k8, v8, table[n : n + 1], pa[n : n + 1],
                                            torch.zeros(1, dtype=torch.int32), scale=0.125, alibi_slopes=slopes,
                                            k_scale=ks, v_scale=vs)
        torch.testing.assert_close(o[cu[n] : cu[n + 1]], ref[0], atol=1e-5, rtol=1e-5)


@pytest.mark.parametrize("grouped", [False, True])
def test_fp8_ragged_append_ref_matches_per_sequence_append(grouped):
    q_lens, past = [1, 70, 3], [0, 64, 100]
    table, k, v, ks, vs, cu, pa = _fp8_ragged(q_lens, past)
    T, G, D = sum(q_lens), 2, 64
    g = torch.Generator().manual_seed(4)
    qkv = torch.randn(1, T, G, 4, D, generator=g) if grouped else torch.randn(1, T, G, 3 * D, generator=g)
    cos, sin = rotary_tables(D, 256)
    k2, v2, ks2, vs2 = k.clone(), v.clone(), ks.clone(), vs.clone()
    q = OF.kv_cache_append_paged_varlen(qkv, k, v, table, cu, pa, cos, sin, k_scale=ks, v_scale=vs)
    for n in range(len(q_lens)):
        qn = OF.kv_cache_append(qkv[:, cu[n] : cu[n + 1]], k2, v2, pa[n : n + 1], cos, sin, k_scale=ks2, v_scale=vs2,
                                block_table=table[n : n + 1])
        assert torch.equal(q[:, cu[n] : cu[n + 1]], qn)
    for a, b in ((k, k2), (v, v2)):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    assert torch.equal(ks, ks2) and torch.equal(vs, vs2)


def test_fp8_ops_need_their_scales():
    table, k8, v8, ks, vs, cu, pa = _fp8_ragged([3], [0])
    q = torch.randn(3, 4, 64)
    with pytest.raises(ValueError, match="k_scale"):
        OF.attention_paged_varlen(q, k8, v8, table, cu, pa, scale=0.125)
    with pytest.raises(ValueError, match="FP8"):
        OF.attention_paged_varlen(q, k8.float(), v8.float(), table, cu, pa, scale=0.125, k_scale=ks, v_scale=vs)


# ---- the cache and the engine ------------------------------------------------------------------------------------------

def test_fp8_pools_scales_and_sink():
    c = RaggedPagedKVCache(3, 2, 4, 64, 6, 3, 40, torch.bfloat16, layers=[0, 2], kv_dtype=FP8)
    assert c.fp8 and c.kv_dtype == FP8 and c.dtype == torch.bfloat16 and c.sink == 6
    for i in (0, 2):
        for pool in (c.k[i], c.v[i]):
            assert pool.dtype == FP8 and pool.shape == (7, 4, 64, 64)
        for s in (c.k_scale[i], c.v_scale[i]):
            assert s.dtype == torch.float32 and s.shape == (7, 4, 64)
    assert c.k[1] is None and c.k_scale[1] is None
    bf = RaggedPagedKVCache(1, 2, 4, 64, 6, 3, 40, torch.bfloat16)
    assert not bf.fp8 and bf.k[0].dtype == torch.bfloat16 and bf.k_scale[0] is None
    with pytest.raises(ValueError, match="kv_dtype"):
        RaggedPagedKVCache(1, 2, 4, 64, 6, 3, 40, torch.bfloat16, kv_dtype=torch.float16)


def _generate_fp8(model, prompt, n):
    out = model.generate(torch.tensor([prompt]), max_length=len(prompt) + n, do_sample=False, use_cache=True,
                         kv_cache_dtype="fp8")
    return out[0, len(prompt) :].tolist()


@pytest.mark.parametrize("name", ["llama", "llama_gqa", "bloom"])
def test_fp8_engine_end_to_end_with_arrivals_and_chunks(name):
    model = {"llama": _llama, "llama_gqa": lambda: _llama(num_key_value_heads=1), "bloom": _bloom}[name]()
    e = GenerationEngine(model, max_batch=3, max_tokens_per_step=3 + 40, num_pages=12, kv_cache_dtype="fp8")
    assert e.cache.fp8 and e.cache.k[0].dtype == FP8
    prompts = [_ids(n, i) for i, n in enumerate([5, 90, 17, 33, 1, 64])]
    news = [6, 4, 9, 3, 5, 2]
    ids, pending = [], list(zip(prompts, news))
    ids.append(e.add_request(*pending.pop(0)))
    chunked = False
    while e.has_unfinished() or pending:
        if pending and e.steps % 2 == 1:   # requests arrive while others run
            ids.append(e.add_request(*pending.pop(0)))
        e.step()
        chunked |= any(r is not None and 0 < r.fed < r.prompt_len for r in e.slots)
    assert chunked
    for rid, p, n in zip(ids, prompts, news):
        assert e.requests[rid].generated == _generate_fp8(model, p, n), rid
    assert sorted(e.cache.free) == list(range(e.cache.num_pages)) and e.cache.refs == [0] * e.cache.num_pages


def test_fp8_engine_prefix_caching_reuses_pages():
    model = _llama(max_position_embeddings=1024)
    e = GenerationEngine(model, max_batch=2, max_tokens_per_step=300, num_pages=8, prefix_caching=True,
                         kv_cache_dtype=FP8)
    system = _ids(128, 9)
    first = e.generate([system + _ids(10, 1)], max_new_tokens=3)[0]
    again = e.generate([system + _ids(10, 1)], max_new_tokens=3)[0]
    assert e.reused_pages == 2 and again == first == _generate_fp8(model, system + _ids(10, 1), 3)


def test_bad_kv_cache_dtype_is_a_value_error():
    for bad in ("int8", torch.float16, "bf16"):
        with pytest.raises(ValueError, match="kv_cache_dtype"):
            GenerationEngine(_llama(), max_batch=2, max_tokens_per_step=100, num_pages=3, kv_cache_dtype=bad)
    m = _llama()
    m.kv_cache_dtype = FP8   # generate()'s per-call attribute is not how the engine is told
    with pytest.raises(ValueError, match="FP8"):
        GenerationEngine(m, max_batch=2, kv_cache_dtype="fp8")


# ---- the bindings' argument checks (tests/op_args_cases.py form) ----------------------------------------------------

def fp8_varlen_cases(dev):
    """Argument cases of the FP8 ragged ops, in the form of ``tests/op_args_cases.py``."""
    g = torch.Generator().manual_seed(0)

    def r(*shape, dtype=torch.bfloat16):
        return torch.randn(*shape, generator=g).to(dtype).to(dev)

    def i32(*rows):
        return torch.tensor(rows, dtype=torch.int32).to(dev)

    common = dict(block_table=i32([0, -1], [1, 2]), cu_q=i32(0, 3, 10), past=i32(0, 64))
    cos, sin = (t.to(dev) for t in rotary_tables(64, 256))
    pools = dict(k_pool=r(4, 2, 64, 64, dtype=FP8), v_pool=r(4, 2, 64, 64, dtype=FP8),
                 k_scale=r(4, 2, 64, dtype=torch.float32).abs(), v_scale=r(4, 2, 64, dtype=torch.float32).abs())
    return [
        C._c("attn_fwd_paged_varlen_fp8",
             dict(q=r(10, 4, 64), **pools, **common, tiles=i32([1, 0], [0, 0]), scale=0.125,
                  alibi_slopes=r(4, dtype=torch.float32)),
             ["q:dtype=float32", "q:misalign", "q:rank", "k_pool:dtype=bfloat16", "k_pool:narrow", "k_pool:device",
              "k_pool:misalign", "v_pool:short", "v_pool:noncontig", "k_scale:short", "k_scale:dtype=bfloat16",
              "k_scale:misalign", "v_scale:noncontig", "v_scale:device", "block_table:dtype=int64",
              "block_table:rank", "cu_q:short", "past:short", "tiles:narrow", "tiles:misalign",
              "alibi_slopes:short"], [(10, 4, 64)]),
        C._c("kv_append_fp8_paged_varlen",
             dict(qkv=r(1, 10, 2, 4, 64), **{n: t.clone() for n, t in pools.items()}, **common, cos=cos, sin=sin,
                  write_q=True),
             ["qkv:dtype=float32", ("qkv:rank", "kv_append_fp8_paged_varlen: packed projection"),
              ("k_pool:dtype=bfloat16", "kv_append_fp8_paged_varlen: k_cache"),
              ("k_pool:narrow", "kv_append_fp8_paged_varlen: k_cache"),
              ("v_pool:short", "kv_append_fp8_paged_varlen: v_cache"),
              ("v_pool:device", "kv_append_fp8_paged_varlen: v_cache must be on"), "k_scale:short",
              "k_scale:misalign", "v_scale:dtype=bfloat16", "v_scale:device", "block_table:dtype=int64",
              "cu_q:short", "past:dtype=int64", ("cos:narrow", "kv_append_fp8_paged_varlen: cos/sin"),
              ("sin:none", "kv_append_fp8_paged_varlen: cos and sin")], [(1, 10, 4, 64)]),
    ]


CASES = fp8_varlen_cases("cpu")
MUTATIONS = [(c, m) for c in CASES for m in c.mutations]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_valid_fp8_arguments_fail_only_for_not_being_on_a_cuda_device(ext, case):  # noqa: F811
    msg = _error(lambda: getattr(ext, case.op)(*case.values()))
    assert msg.startswith(f"{case.op}: ") and "must be a CUDA tensor" in msg, msg


@pytest.mark.parametrize("case,mutation", MUTATIONS, ids=[f"{c.id}-{n}-{k}" for c, (n, k, _) in MUTATIONS])
def test_each_fp8_mutation_is_rejected_by_its_own_rule(ext, case, mutation):  # noqa: F811
    name, kind, fragment = mutation
    msg = _error(lambda: getattr(ext, case.op)(*C.mutated(case, name, kind, "meta")))
    assert fragment in msg, msg
    assert "must be a CUDA tensor" not in msg, msg
