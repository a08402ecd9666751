"""Continuous batching on the H100: the ragged paged append and flash prefill bit for bit against the paged kernels run
per sequence (NaN in every pool row outside the windows), and the engine's tokens against an uncached fp32 forward,
with prefix caching, decode graphs and ``generate()`` around an engine run."""
import copy

import pytest
import torch

from libai_b200.config import DictConfig, LazyConfig
from libai_b200.inference import GenerationEngine
from libai_b200.layers._param import param_defaults
from libai_b200.models.llama_model import rotary_tables
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import LLAMA

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        torch.manual_seed(0)
        yield


# ---- kernels ---------------------------------------------------------------------------------------------------------

def _pools(q_lens, past, G, D, seed, share=True):
    """Pools of shuffled pages filled with NaN except each sequence's window rows; sequence 1 shares sequence 0's first
    page when both windows cover it; table entries past a window are -1."""
    g = torch.Generator().manual_seed(seed)
    need = [-(-(s + p) // 64) for s, p in zip(q_lens, past)]
    pages = sum(need) + 3
    perm = torch.randperm(pages, generator=g).tolist()
    mp = max(need) + 1
    table = torch.full((len(q_lens), mp), -1, dtype=torch.int32)
    for n in range(len(q_lens)):
        table[n, : need[n]] = torch.tensor([perm.pop() for _ in range(need[n])], dtype=torch.int32)
    if share and len(q_lens) > 1 and past[0] + q_lens[0] >= 64 and past[1] + q_lens[1] >= 64:
        table[1, 0] = table[0, 0]
    k = torch.full((pages, G, 64, D), float("nan"), dtype=torch.bfloat16)
    v = k.clone()
    for n, (s, p) in enumerate(zip(q_lens, past)):
        for j in range(p + s):
            page = int(table[n, j // 64])
            k[page, :, j % 64] = torch.randn(G, D, generator=g).to(torch.bfloat16)
            v[page, :, j % 64] = torch.randn(G, D, generator=g).to(torch.bfloat16)
    cu = torch.tensor([0] + torch.tensor(q_lens).cumsum(0).tolist(), dtype=torch.int32)
    return (table.to(DEV), k.to(DEV), v.to(DEV), cu.to(DEV), torch.tensor(past, dtype=torch.int32, device=DEV))


CASES = [([1, 70, 3, 130, 128, 257], [0, 64, 100, 5, 640, 63]), ([200, 1, 64], [129, 4095, 0])]


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G,A", [(4, 4), (2, 8)])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_ragged_prefill_bit_identical_to_per_sequence_paged(D, G, A, alibi, case):
    q_lens, past = CASES[case]
    table, k, v, cu, pa = _pools(q_lens, past, G, D, seed=case)
    q = torch.randn(sum(q_lens), A, D, device=DEV).to(torch.bfloat16)
    slopes = torch.linspace(0.5, 0.01, A, device=DEV) if alibi else None
    o = OF.attention_paged_varlen(q, k, v, table, cu, pa, scale=D ** -0.5, alibi_slopes=slopes)
    assert torch.isfinite(o).all()
    c = cu.tolist()
    for n, p in enumerate(past):
        ref = OF.attention_paged(q[None, c[n] : c[n + 1]], k, v, table[n : n + 1], p, scale=D ** -0.5,
                                 alibi_slopes=slopes)
        assert torch.equal(o[c[n] : c[n + 1]], ref[0]), n


@pytest.mark.parametrize("grouped", [False, True])
def test_ragged_append_bit_identical_to_per_sequence_paged(grouped):
    q_lens, past = [1, 70, 3, 130], [0, 64, 100, 5]
    G, D = 2, 128
    table, k, v, cu, pa = _pools(q_lens, past, G, D, seed=7, share=False)
    k.fill_(float("nan"))
    v.fill_(float("nan"))
    T = sum(q_lens)
    qkv = (torch.randn(1, T, G, 4, D, device=DEV) if grouped else torch.randn(1, T, G, 3 * D, device=DEV))
    qkv = qkv.to(torch.bfloat16)
    cos, sin = rotary_tables(D, 1024, device=DEV)
    k2, v2 = k.clone(), v.clone()
    q = OF.kv_cache_append_paged_varlen(qkv, k, v, table, cu, pa, cos, sin)
    c = cu.tolist()
    for n in range(len(q_lens)):
        qn = OF.kv_cache_append(qkv[:, c[n] : c[n + 1]].contiguous(), k2, v2, pa[n : n + 1], cos, sin,
                                block_table=table[n : n + 1])
        assert torch.equal(q[:, c[n] : c[n + 1]], qn)
    # every byte, NaN rows included: what no sequence writes stays as it was
    assert torch.equal(k.view(torch.int16), k2.view(torch.int16)) and torch.equal(v.view(torch.int16), v2.view(torch.int16))
    assert int(torch.isnan(k).any(dim=-1).logical_not().sum()) == T * G


# ---- the engine ------------------------------------------------------------------------------------------------------

def _llama(**kw):
    from libai_b200.models import LlamaForCausalLM

    cfg = {**LLAMA, "max_position_embeddings": 1024, "hidden_size": 256, "num_attention_heads": 4, **kw}
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=0):
        return LlamaForCausalLM(DictConfig(cfg)).eval()


def _bloom():
    from projects.BLOOM.modeling.bloom_model import BloomForCausalLM

    cfg = LazyConfig.load("projects/BLOOM/configs/bloom_inference.py").cfg
    cfg.update(dict(vocab_size=100, hidden_size=128, hidden_layers=2, n_head=2))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=0):
        return BloomForCausalLM(cfg).eval()


MODELS = {"llama": _llama, "llama_gqa": lambda: _llama(num_key_value_heads=2),
          "qwen2_bias": lambda: _llama(num_key_value_heads=2, qkv_bias=True), "bloom": _bloom}


def _ids(n, seed):
    return torch.randint(3, 100, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


def _run(e, work):
    """Add the requests of ``work`` (prompt, max_new) two at a time between steps; returns their ids."""
    ids, pending = [], list(work)
    while pending or e.has_unfinished():
        for _ in range(2):
            if pending:
                ids.append(e.add_request(*pending.pop(0)))
        e.step()
    return ids


def _near_argmax(model, e, ids):
    """Every emitted token is a near-argmax of the uncached fp32 forward over the request's tokens, and most are its
    exact argmax.  The bound is derived per request: a bf16 forward's logits are off the fp32 ones by at most ``err``
    (measured here on the uncached bf16 forward of the same tokens), so a token the bf16 model ranks first trails the
    fp32 maximum by at most ``2 err``; the engine's GEMMs see other row counts than that forward, whence a margin of
    1.5 over it: ``gap <= 3 err``."""
    ref_model = copy.deepcopy(model).float()
    exact = total = 0
    with torch.no_grad():
        for rid in ids:
            r = e.requests[rid]
            toks = torch.tensor([r.tokens[:-1]], device=DEV)
            logits = ref_model(toks)["logits"][0, r.prompt_len - 1 :].float()
            err = float((model(toks)["logits"][0, r.prompt_len - 1 :].float() - logits).abs().max())
            got = logits.gather(1, torch.tensor(r.generated, device=DEV)[:, None])[:, 0]
            gap = logits.max(dim=1).values - got
            assert float(gap.max()) <= 3 * err, (rid, float(gap.max()), err)
            exact += int((gap == 0).sum())
            total += gap.numel()
    assert exact >= 0.9 * total, (exact, total)


WORK = [(_ids(n, i), m) for i, (n, m) in enumerate([(5, 12), (300, 6), (17, 20), (130, 9), (1, 7), (64, 15),
                                                     (200, 4), (90, 11)])]


@pytest.mark.parametrize("name", list(MODELS))
def test_engine_greedy_is_near_argmax_of_fp32(name):
    model = MODELS[name]()
    e = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40)
    ids = _run(e, WORK)
    assert all(e.requests[i].finish_reason == "length" for i in ids)
    assert sorted(e.cache.free) == list(range(40))
    _near_argmax(model, e, ids)


def test_engine_prefix_caching_reuses_pages():
    model = _llama()
    e = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 256, num_pages=48, prefix_caching=True)
    system = _ids(200, 99)
    first = _run(e, [(system + _ids(10, i), 5) for i in range(3)])
    before = e.reused_pages
    second = _run(e, [(system + _ids(30, 10 + i), 8) for i in range(4)])
    assert e.reused_pages - before >= 4 * 3   # the system prompt's three full pages, per request
    _near_argmax(model, e, first + second)


def test_engine_decode_graphs_match_eager_with_one_capture():
    model = _llama(num_key_value_heads=2)
    outs = []
    for graphs in (False, True):
        e = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40, decode_graphs=graphs)
        ids = _run(e, WORK)
        outs.append([e.requests[i].generated for i in ids])
        if graphs:
            assert e.graph_captures == 1
    assert outs[0] == outs[1]
    # weights moved to new storage (same values): the graph is captured again and reads them, tokens unchanged
    with torch.no_grad():
        for p in model.parameters():
            p.data = p.data.clone()
    ids = _run(e, WORK)
    assert e.graph_captures == 2 and [e.requests[i].generated for i in ids] == outs[0]
    # and new values in the new storage are read too
    with torch.no_grad():
        model.lm_head.weight.data = torch.randn_like(model.lm_head.weight) * 0.02
    eager = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40)
    want = [eager.requests[i].generated for i in _run(eager, WORK)]
    ids = _run(e, WORK)
    assert e.graph_captures == 3 and [e.requests[i].generated for i in ids] == want


def test_engine_long_prompt_chunked_on_an_idle_engine():
    # 700 prompt tokens at 96 per step: seven steps of prompt chunks that sample nothing (no host sync), back to back
    model = _llama()
    e = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40)
    rid = e.add_request(_ids(700, 5), 12)
    quiet = 0
    while e.has_unfinished():
        quiet += int(not e.step())
    assert quiet >= 7
    _near_argmax(model, e, [rid])


def test_varlen_ops_argument_cases():
    from tests import op_args_cases as C
    from tests.test_continuous_batching_cpu import varlen_cases

    ext = __import__("libai_b200.ops", fromlist=["load_ext"]).load_ext(required=True)
    for case in varlen_cases(DEV):
        out = getattr(ext, case.op)(*case.values())
        torch.cuda.synchronize()
        assert tuple(out.shape) == case.outputs[0] and out.device == torch.device(DEV)
        for name, kind, fragment in case.mutations:
            with pytest.raises(RuntimeError, match=fragment):
                getattr(ext, case.op)(*C.mutated(case, name, kind, "cpu"))


@pytest.mark.parametrize("name", ["llama", "bloom"])
def test_generate_unchanged_around_an_engine(name):
    model = MODELS[name]()
    ids = torch.tensor([_ids(40, 0), _ids(40, 1)], device=DEV)
    kw = dict(max_length=60, do_sample=False, use_cache=True)
    before = model.generate(ids, **kw)
    GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40).generate(
        [w[0] for w in WORK[:3]], max_new_tokens=5)
    assert torch.equal(before, model.generate(ids, **kw))
