"""Continuous batching on the reference path: the ragged reference ops against per-sequence attention and appends, the
engine's scheduler (first-come-first-served admission under the slot and page limits, chunking under
``max_tokens_per_step``, pages reserved at admission and all returned, reference counts of shared prefix pages,
eviction of index-only pages on demand), the ``ValueError``s, and tiny fp32 Llama and BLOOM models run end to end with
requests arriving between steps."""
import os
from types import SimpleNamespace

import pytest
import torch

from libai_b200.config import DictConfig, LazyConfig
from libai_b200.inference import GenerationEngine
from libai_b200.inference.kv_cache import RaggedPagedKVCache
from libai_b200.layers._param import param_defaults
from libai_b200.models.llama_model import rotary_tables
from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests import op_args_cases as C
from tests.test_cached_attention_cpu import LLAMA, MODELS


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


def _llama(dtype=torch.float32, **kw):
    from libai_b200.models import LlamaForCausalLM

    with param_defaults(dtype=dtype, device="cpu", seed=0):
        return LlamaForCausalLM(DictConfig({**LLAMA, "max_position_embeddings": 256, **kw})).eval()


def _bloom(dtype=torch.float32):
    from projects.BLOOM.modeling.bloom_model import BloomForCausalLM

    cfg = LazyConfig.load("projects/BLOOM/configs/bloom_inference.py").cfg
    cfg.update(dict(vocab_size=100, hidden_size=128, hidden_layers=2, n_head=2))
    with param_defaults(dtype=dtype, device="cpu", seed=0):
        return BloomForCausalLM(cfg).eval()


def _ids(n, seed):
    return torch.randint(3, 100, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


# ---- the ragged reference ops ----------------------------------------------------------------------------------------

def _ragged(q_lens, past, G=2, r=2, D=64, pages=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(pages, generator=g).tolist()
    mp = 6
    table = torch.full((len(q_lens), mp), -1, dtype=torch.int32)
    for n, (s, p) in enumerate(zip(q_lens, past)):
        need = -(-(s + p) // 64)
        table[n, :need] = torch.tensor([perm.pop() for _ in range(need)], dtype=torch.int32)
    k = torch.randn(pages, G, 64, D, generator=g)
    v = torch.randn(pages, G, 64, D, generator=g)
    cu = torch.tensor([0] + torch.tensor(q_lens).cumsum(0).tolist(), dtype=torch.int32)
    return table, k, v, cu, torch.tensor(past, dtype=torch.int32)


@pytest.mark.parametrize("alibi", [False, True])
def test_ragged_attention_ref_matches_per_sequence_attention(alibi):
    q_lens, past = [1, 70, 3, 130], [0, 64, 100, 5]
    table, k, v, cu, pa = _ragged(q_lens, past)
    A, D = 4, 64
    q = torch.randn(sum(q_lens), A, D, generator=torch.Generator().manual_seed(3))
    slopes = torch.tensor([0.5, 0.25, 0.125, 0.0625]) if alibi else None
    o = OF.attention_paged_varlen(q, k, v, table, cu, pa, scale=0.125, alibi_slopes=slopes)
    for n in range(len(q_lens)):
        qn = q[cu[n] : cu[n + 1]][None]   # [1, s, a, d]
        ref = OF.decode_attention_paged_ref(qn, k, v, table[n : n + 1], pa[n : n + 1], torch.zeros(1, dtype=torch.int32),
                                            scale=0.125, alibi_slopes=slopes)
        torch.testing.assert_close(o[cu[n] : cu[n + 1]], ref[0], atol=1e-5, rtol=1e-5)


@pytest.mark.parametrize("grouped", [False, True])
def test_ragged_append_ref_matches_per_sequence_append(grouped):
    q_lens, past = [1, 70, 3], [0, 64, 100]
    table, k, v, cu, pa = _ragged(q_lens, past)
    T, G, D = sum(q_lens), 2, 64
    g = torch.Generator().manual_seed(4)
    qkv = torch.randn(1, T, G, 4, D, generator=g) if grouped else torch.randn(1, T, G, 3 * D, generator=g)
    cos, sin = rotary_tables(D, 256)
    k2, v2 = k.clone(), v.clone()
    q = OF.kv_cache_append_paged_varlen(qkv, k, v, table, cu, pa, cos, sin)
    for n in range(len(q_lens)):
        qn = OF.kv_cache_append(qkv[:, cu[n] : cu[n + 1]], k2, v2, pa[n : n + 1], cos, sin,
                                block_table=table[n : n + 1])
        assert torch.equal(q[:, cu[n] : cu[n + 1]], qn)
    assert torch.equal(k, k2) and torch.equal(v, v2)


def test_varlen_tiles_list_every_block_heaviest_first():
    q_lens = [1, 300, 128, 0]
    t = OF.varlen_tiles(q_lens).tolist()
    assert sorted(map(tuple, t)) == [(0, 0), (1, 0), (1, 1), (1, 2), (2, 0)]
    assert t[0] == [1, 2]
    sizes = [min(128 * (b + 1), q_lens[n]) for n, b in t]
    assert sizes == sorted(sizes, reverse=True)
    # the keys a block sees count the rows held before it: a short continuation of a long sequence goes first
    past = [4000, 0, 100, 0]
    t = OF.varlen_tiles(q_lens, past).tolist()
    assert t[0] == [0, 0]
    keys = [past[n] + min(128 * (b + 1), q_lens[n]) for n, b in t]
    assert keys == sorted(keys, reverse=True)


# ---- the engine ------------------------------------------------------------------------------------------------------

def _greedy_ref(model, tokens, n):
    """n greedy tokens of the uncached model."""
    out = list(tokens)
    with torch.no_grad():
        for _ in range(n):
            logits = model(torch.tensor([out]))["logits"][0, -1]
            out.append(int(logits.float().argmax()))
    return out[len(tokens) :]


def _books(e):
    c = e.cache
    refs = [0] * c.num_pages
    for p in c.prefix.keys:
        refs[p] += 1
    for req in e.slots:
        if req is not None:
            for p in req.pages:
                refs[p] += 1
    assert refs == c.refs
    assert sorted(c.free) == [p for p in range(c.num_pages) if refs[p] == 0]


@pytest.mark.parametrize("name", ["llama", "bloom"])
def test_engine_end_to_end_with_arrivals_and_chunks(name):
    model = _llama() if name == "llama" else _bloom()
    e = GenerationEngine(model, max_batch=3, max_tokens_per_step=3 + 40, num_pages=12)
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
        _books(e)
    assert chunked
    for rid, p, n in zip(ids, prompts, news):
        assert e.requests[rid].generated == _greedy_ref(model, p, n), rid
        assert e.requests[rid].finish_reason == "length"
    assert sorted(e.cache.free) == list(range(e.cache.num_pages))


def test_admission_is_first_come_first_served_under_slots_and_pages():
    e = GenerationEngine(_llama(), max_batch=2, max_tokens_per_step=200, num_pages=5)
    a = e.add_request(_ids(100, 0), max_new_tokens=10)    # 2 pages
    b = e.add_request(_ids(130, 1), max_new_tokens=10)    # 3 pages
    c = e.add_request(_ids(10, 2), max_new_tokens=10)     # 1 page: no slot left
    e.step()
    assert [r.id if r else None for r in e.slots] == [a, b] and [r.id for r in e.waiting] == [c]
    assert e.cache.free == [] and e.requests[a].pages == [0, 1] and e.requests[b].pages == [2, 3, 4]
    d = e.add_request(_ids(200, 3), max_new_tokens=50)    # 4 pages: waits for a and b
    while e.requests[a].finish_reason is None:
        e.step()
    e.step()
    assert e.requests[c].slot >= 0 and e.requests[d].slot == -1   # c first; d does not fit beside b and c
    e.generate([], max_new_tokens=1)
    assert e.requests[d].finish_reason == "length" and sorted(e.cache.free) == list(range(5))


def test_chunking_under_the_token_budget():
    e = GenerationEngine(_llama(), max_batch=2, max_tokens_per_step=2 + 50, num_pages=8)
    a = e.add_request(_ids(120, 0), max_new_tokens=2)
    b = e.add_request(_ids(30, 1), max_new_tokens=2)
    e.step()
    assert e.cache.T == 52 and e.cache.chunks == 1 and e.requests[a].fed == 50 and e.requests[b].fed == 0
    e.step()
    assert e.requests[a].fed == 100 and e.requests[b].fed == 0
    out = e.step()   # a's last 20 tokens and b's 30: both prompts end
    assert e.cache.chunks == 2 and [o.request_id for o in out] == [a, b]
    assert e.requests[b].fed == 30 and len(e.requests[b].tokens) == 31
    out = e.step()   # two decode rows
    assert e.cache.T == 2 and e.cache.chunks == 0 and {o.request_id for o in out} == {a, b}


def test_prefix_pages_are_shared_counted_and_evicted_on_demand():
    model = _llama(max_position_embeddings=1024)
    e = GenerationEngine(model, max_batch=2, max_tokens_per_step=300, num_pages=8, prefix_caching=True)
    system = _ids(128, 9)
    first = e.generate([system + _ids(10, 1)], max_new_tokens=3)[0]
    assert len(e.cache.prefix) == 2 and e.cache.index_only() == 2
    assert sorted(e.cache.free) == [p for p in range(8) if p not in e.cache.prefix.keys]
    r1 = e.add_request(system + _ids(10, 1), max_new_tokens=3)
    r2 = e.add_request(system + _ids(20, 2), max_new_tokens=3)
    e.step()
    assert e.reused_pages == 4
    shared = e.requests[r1].pages[:2]
    assert shared == e.requests[r2].pages[:2] and all(e.cache.refs[p] == 3 for p in shared)
    _books(e)
    while e.has_unfinished():
        e.step()
        _books(e)
    assert e.requests[r1].generated == first == _greedy_ref(model, system + _ids(10, 1), 3)
    assert e.requests[r2].generated == _greedy_ref(model, system + _ids(20, 2), 3)
    # a request that needs every page evicts the index-only ones
    big = e.add_request(_ids(8 * 64 - 5, 5), max_new_tokens=5)
    e.step()
    assert e.requests[big].slot >= 0 and len(e.cache.prefix) == 0 and e.cache.free == []
    e.generate([], max_new_tokens=1)
    assert sorted(e.cache.free) == [p for p in range(8) if p not in e.cache.prefix.keys]
    _books(e)


def test_prefix_index_cleared_when_the_weights_change():
    model = _llama()
    e = GenerationEngine(model, max_batch=1, max_tokens_per_step=200, num_pages=6, prefix_caching=True)
    e.generate([_ids(130, 0)], max_new_tokens=2)
    assert len(e.cache.prefix) == 2
    with torch.no_grad():
        model.lm_head.weight.mul_(1.0)   # an in-place update bumps _version
    e.generate([_ids(130, 0)], max_new_tokens=2)
    assert e.reused_pages == 0


def test_max_length_finishes_a_request():
    e = GenerationEngine(_llama(), max_batch=1, max_tokens_per_step=300, num_pages=4)
    out = e.generate([_ids(250, 0)], max_new_tokens=20)[0]
    assert len(out) == 6 and e.requests[0].finish_reason == "max_length"


def test_value_errors(monkeypatch):
    e = GenerationEngine(_llama(), max_batch=2, max_tokens_per_step=100, num_pages=3)
    with pytest.raises(ValueError):
        e.add_request(_ids(150, 0), max_new_tokens=50)   # 4 pages > 3
    with pytest.raises(ValueError):
        e.add_request(_ids(257, 0), max_new_tokens=1)    # past the rotary table
    with pytest.raises(ValueError):
        e.add_request([], max_new_tokens=1)
    with pytest.raises(ValueError):
        GenerationEngine(_llama(), max_batch=4, max_tokens_per_step=4)
    for name in ("gpt2", "chatglm", "t5"):
        with pytest.raises(ValueError, match="continuous batching"):
            GenerationEngine(MODELS[name](), max_batch=2)
    from projects.Llama.adapter.adapter_model import LlamaForCausalLM as Adapter

    with param_defaults(dtype=torch.float32, device="cpu", seed=0):
        adapter = Adapter(DictConfig({**LLAMA, "adapter_len": 4, "adapter_layer": 2})).eval()
    with pytest.raises(ValueError, match="continuous batching"):
        GenerationEngine(adapter, max_batch=2)
    from projects.GLM.modeling_glm import GLMForConditionalGeneration
    assert not GLMForConditionalGeneration.continuous_batching
    m = _llama()
    m.kv_cache_dtype = torch.float8_e4m3fn
    with pytest.raises(ValueError, match="FP8"):
        GenerationEngine(m, max_batch=2)
    m = _llama()
    for tp, pp in ((2, 1), (1, 2)):
        monkeypatch.setattr(dist, "get_dist_util", lambda: SimpleNamespace(tensor_parallel_size=tp,
                                                                           pipeline_parallel_size=pp))
        with pytest.raises(ValueError, match="parallel"):
            GenerationEngine(m, max_batch=2)


def test_generate_unchanged_around_an_engine():
    model = _llama()
    ids = torch.tensor([_ids(20, 0)])
    before = model.generate(ids, max_length=30, do_sample=False, use_cache=True)
    GenerationEngine(model, max_batch=2, max_tokens_per_step=64, num_pages=4).generate([_ids(20, 1)], 5)
    after = model.generate(ids, max_length=30, do_sample=False, use_cache=True)
    assert torch.equal(before, after)


def test_cache_descriptor_layout():
    c = RaggedPagedKVCache(1, 2, 2, 64, 6, 3, 40, torch.float32)
    ids, rows = c.write_step([None, (7, 65, [4, 2])], [([1, 2, 3], 0, [0]), ([5], 64, [1, 3])], [1, 5])
    assert ids.tolist() == [[0, 7, 1, 2, 3, 5]] and rows.tolist() == [1, 5]
    assert c.cu_q.tolist() == [0, 1, 2, 5, 6] and c.past.tolist() == [0, 65, 0, 64]
    assert c.table.tolist() == [[6, -1, -1], [4, 2, -1], [0, -1, -1], [1, 3, -1]]
    assert c.cu_c.tolist() == [0, 3, 4] and c.tiles.tolist() == [[1, 0], [0, 0]]   # 65 keys before 3


def test_steps_record_no_autograd_graph():
    model = _llama()
    seen = []
    forward = model.continuous_batching_logits

    def spy(ids, cache):
        out = forward(ids, cache)
        seen.append((torch.is_grad_enabled(), out.requires_grad))
        return out

    model.continuous_batching_logits = spy
    e = GenerationEngine(model, max_batch=2, max_tokens_per_step=40, num_pages=4)
    assert torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters())
    e.generate([_ids(50, 0), _ids(3, 1)], max_new_tokens=3)
    assert len(seen) >= 3 and not any(g or r for g, r in seen)


# ---- the bindings' argument checks (tests/op_args_cases.py form) ----------------------------------------------------

def varlen_cases(dev):
    """Argument cases of the ragged ops, in the form of ``tests/op_args_cases.py``."""
    g = torch.Generator().manual_seed(0)

    def r(*shape, dtype=torch.bfloat16):
        return torch.randn(*shape, generator=g).to(dtype).to(dev)

    def i32(*rows):
        return torch.tensor(rows, dtype=torch.int32).to(dev)

    # two sequences: 3 tokens after 0 rows in page 0, 7 tokens after 64 rows in pages 1, 2
    common = dict(block_table=i32([0, -1], [1, 2]), cu_q=i32(0, 3, 10), past=i32(0, 64))
    cos, sin = (t.to(dev) for t in rotary_tables(64, 256))
    return [
        C._c("attn_fwd_paged_varlen",
             dict(q=r(10, 4, 64), k_pool=r(4, 2, 64, 64), v_pool=r(4, 2, 64, 64), **common,
                  tiles=i32([1, 0], [0, 0]), scale=0.125, alibi_slopes=r(4, dtype=torch.float32)),
             ["q:dtype=float32", "q:misalign", "q:rank", "k_pool:dtype=float32", "k_pool:narrow", "k_pool:device",
              "v_pool:short", "v_pool:noncontig", "block_table:dtype=int64", "block_table:rank", "cu_q:short",
              "cu_q:dtype=int64", "past:short", "past:device", "tiles:narrow", "tiles:noncontig", "tiles:misalign",
              "tiles:dtype=int64", "alibi_slopes:short", "alibi_slopes:dtype=bfloat16"], [(10, 4, 64)]),
        C._c("kv_append_paged_varlen",
             dict(qkv=r(1, 10, 2, 4, 64), k_pool=r(4, 2, 64, 64), v_pool=r(4, 2, 64, 64), **common, cos=cos, sin=sin,
                  write_q=True),
             ["qkv:dtype=float32", ("qkv:rank", "kv_append_paged_varlen: packed projection"),
              ("k_pool:dtype=float32", "kv_append_paged_varlen: k_cache"),
              ("k_pool:narrow", "kv_append_paged_varlen: k_cache"),
              ("k_pool:misalign", "kv_append_paged_varlen: k_cache"),
              ("v_pool:short", "kv_append_paged_varlen: v_cache"),
              ("v_pool:device", "kv_append_paged_varlen: v_cache must be on"), "block_table:dtype=int64",
              "cu_q:short", "past:short", "past:dtype=int64", ("cos:narrow", "kv_append_paged_varlen: cos/sin"),
              ("cos:dtype=bfloat16", "kv_append_paged_varlen: cos/sin"),
              ("sin:none", "kv_append_paged_varlen: cos and sin")], [(1, 10, 4, 64)]),
    ]


CASES = varlen_cases("cpu")
MUTATIONS = [(c, m) for c in CASES for m in c.mutations]


@pytest.fixture(scope="module")
def ext():
    if not os.path.exists(ops_build.NVCC):
        pytest.skip("needs nvcc to build the extension")
    torch.ops.load_library(ops_build.build(force=False))
    return torch.ops.libai_b200


def _error(fn):
    with pytest.raises(RuntimeError) as e:
        fn()
    return str(e.value).splitlines()[0]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_valid_arguments_fail_only_for_not_being_on_a_cuda_device(ext, case):
    msg = _error(lambda: getattr(ext, case.op)(*case.values()))
    assert msg.startswith(f"{case.op}: ") and "must be a CUDA tensor" in msg, msg


@pytest.mark.parametrize("case,mutation", MUTATIONS, ids=[f"{c.id}-{n}-{k}" for c, (n, k, _) in MUTATIONS])
def test_each_mutation_is_rejected_by_its_own_rule(ext, case, mutation):
    name, kind, fragment = mutation
    msg = _error(lambda: getattr(ext, case.op)(*C.mutated(case, name, kind, "meta")))
    assert fragment in msg, msg
    assert "must be a CUDA tensor" not in msg, msg
