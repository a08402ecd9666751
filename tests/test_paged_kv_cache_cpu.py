"""The paged KV cache on the reference path: its logical rows, reference counts and free list through random appends,
forks, beam reorders and rollbacks against a contiguous cache; what a reorder copies; the pool size; and
``generate(paged_kv_cache=True)`` against the contiguous cache on every decoder-only model with a preallocated cache."""
import random

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference.kv_cache import PagedKVCache, StaticKVCache
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import LLAMA, MODELS, _prompt


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


G, D = 2, 64


def _qkv(b, s, gen):
    return torch.randn(b, s, G, 3, D, generator=gen).to(torch.bfloat16)   # grouped, r = 1


def _append(c, qkv):
    c.reserve(qkv.shape[1])
    for i in c.owned:
        c.layer(i).append(qkv)
    c.advance(qkv.shape[1])


def _logical(c, i):
    if isinstance(c, PagedKVCache):
        L = c.length
        return OF.kv_pages_gather(c.k[i], c.block_table, L), OF.kv_pages_gather(c.v[i], c.block_table, L)
    return c.k[i][:, :, : c.length], c.v[i][:, :, : c.length]


def _check_books(c):
    refs = [0] * c.num_pages
    for row in c.host_table[: c.batch]:
        assert all(p >= 0 for p in row[: c.mapped]) and all(p == -1 for p in row[c.mapped:])
        for p in row[: c.mapped]:
            refs[p] += 1
    assert refs == c.refs
    assert sorted(c.free) == [p for p in range(c.num_pages) if refs[p] == 0]
    assert torch.equal(c.block_table, torch.tensor(c.host_table[: c.batch], dtype=torch.int32))


@pytest.mark.parametrize("seed", range(6))
def test_random_operations_keep_the_logical_rows_of_a_contiguous_cache(seed):
    rnd, gen = random.Random(seed), torch.Generator().manual_seed(seed)
    b, n, cap, prompt = 2, 3, 300, rnd.choice([5, 64, 100])
    paged = PagedKVCache(2, b, G, D, cap, fork=n, prompt_len=prompt)
    qkv = _qkv(b, prompt, gen)
    ref = StaticKVCache(2, b * n, G, D, cap)
    _append(paged, qkv)
    _append(ref, qkv.repeat_interleave(n, 0))
    paged.fork(n)
    _check_books(paged)
    for _ in range(40):
        op = rnd.choice(["append", "append", "reorder", "rollback", "chunk"])
        if op == "reorder":
            idx = torch.tensor([p * n + rnd.randrange(n) for p in range(b) for _ in range(n)])
            paged.reorder_(idx)
            ref.reorder_(idx)
        elif op == "rollback":
            k = rnd.randrange(0, min(paged.length - prompt, 5) + 1)
            paged.rollback(k)
            ref.rollback(k)
        else:
            s = 1 if op == "append" else rnd.randrange(2, 20)
            if paged.length + s > cap:
                continue
            x = _qkv(b * n, s, gen)
            _append(paged, x)
            _append(ref, x)
        _check_books(paged)
        assert paged.length == ref.length and torch.equal(paged.seqlens, ref.seqlens)
        for i in paged.owned:
            for x, y in zip(_logical(paged, i), _logical(ref, i)):
                assert torch.equal(x, y)


def test_a_reorder_copies_at_most_the_last_page_of_each_sequence(monkeypatch):
    copied = []
    real = OF.kv_page_copy
    monkeypatch.setattr(OF, "kv_page_copy", lambda arrays, pairs: (copied.append(list(pairs)), real(arrays, pairs)))
    gen = torch.Generator().manual_seed(0)
    b, n, prompt = 2, 4, 150
    c = PagedKVCache(2, b, G, D, 400, fork=n, prompt_len=prompt)
    _append(c, _qkv(b, prompt, gen))
    c.fork(n)
    for step in range(120):
        c.reorder_(torch.tensor([p * n + (step * 7 + j) % n for p in range(b) for j in range(n)]))
        full = {p for row in c.host_table[: c.batch] for p in row[: c.length // 64]}
        copied.clear()
        _append(c, _qkv(b * n, 1, gen))
        pairs = [pair for call in copied for pair in call]
        assert len(pairs) <= b * n and not {src for src, _ in pairs} & full


def test_a_full_page_is_never_copied(monkeypatch):
    copied = []
    monkeypatch.setattr(OF, "kv_page_copy", lambda arrays, pairs: copied.extend(pairs))
    b, n = 1, 3
    c = PagedKVCache(1, b, G, D, 256, fork=n, prompt_len=128)   # two full prompt pages
    c.reserve(128)
    c.advance(128)
    c.fork(n)
    for _ in range(3):
        c.reorder_(torch.tensor([0, 0, 1]))
        c.reserve(1)
        c.advance(1)
    full = set(c.host_table[0][:2])
    assert copied and not {src for src, _ in copied} & full


@pytest.mark.parametrize("b,n,prompt,max_length", [(1, 4, 100, 228), (2, 3, 512, 640), (3, 8, 1024, 1152),
                                                   (2, 1, 70, 90), (1, 2, 10, 300)])
def test_pool_size_formula_and_bytes(b, n, prompt, max_length):
    c = PagedKVCache(2, b, G, D, max_length, fork=n, prompt_len=prompt)
    M, S = -(-max_length // 64), prompt // 64
    assert c.max_pages == M and c.capacity == M * 64
    assert c.num_pages == b * S + b * n * (M - S)
    contiguous = StaticKVCache(2, b * n, G, D, max_length)
    paged_bytes = sum(t.numel() * t.element_size() for t in c.arrays())
    flat_bytes = sum(t.numel() * t.element_size() for t in (*contiguous.k, *contiguous.v))
    if n >= 2 and prompt >= 64 and (n - 1) * S * 64 > n * (M * 64 - max_length):
        assert paged_bytes < flat_bytes


def _qwen():
    from libai_b200.models import LlamaForCausalLM

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return LlamaForCausalLM(DictConfig(dict(LLAMA, qkv_bias=True))).eval()


def _adapter():
    from projects.Llama.adapter.adapter_model import LlamaForCausalLM

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        m = LlamaForCausalLM(DictConfig(dict(LLAMA, hidden_size=256, num_attention_heads=4, adapter_len=4,
                                             adapter_layer=2))).eval()
    with torch.no_grad():
        for layer in m.model.layers:
            gate = layer.self_attn.gate
            gate.copy_(torch.linspace(0.5, 2.0, gate.numel()).view_as(gate))
    return m


BUILDERS = {**{k: v for k, v in MODELS.items() if k != "t5"}, "qwen": _qwen, "llama_adapter": _adapter}
# the models whose forward takes a padding mask (ChatGLM's P-tuning prefix takes no padded prompt)
PADDED = ("llama", "llama_gqa", "bloom", "chatglm", "qwen", "llama_adapter")


def _generate(m, name, paged, case, **kw):
    ids, am = _prompt(case)
    if am is not None:
        kw["attention_mask"] = am
    torch.manual_seed(0)
    with torch.no_grad():
        return m.generate(ids, max_length=ids.shape[1] + 6, eos_token_id=None, paged_kv_cache=paged, **kw)


MODES = {"greedy": dict(), "beams": dict(num_beams=3), "sample": dict(do_sample=True, num_return_sequences=3)}


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_generate_on_pages_gives_the_contiguous_tokens(name, mode):
    m = BUILDERS[name]()
    case = "left_padded" if name in PADDED else "plain"
    contiguous = _generate(m, name, False, case, **MODES[mode])
    assert type(m.kv_cache) is StaticKVCache
    paged = _generate(m, name, True, case, **MODES[mode])
    assert isinstance(m.kv_cache, PagedKVCache)
    assert torch.equal(contiguous, paged)


def test_the_prompt_is_prefilled_once(monkeypatch):
    m = BUILDERS["llama_gqa"]()
    seen = []
    forward = type(m).forward
    monkeypatch.setattr(type(m), "forward", lambda self, input_ids, *a, **k: (seen.append(tuple(input_ids.shape)),
                                                                            forward(self, input_ids, *a, **k))[1])
    _generate(m, "llama_gqa", True, "left_padded", num_beams=3)
    assert seen[0] == (3, 7) and all(s == (9, 1) for s in seen[1:])
    assert m.kv_cache.num_pages < 9 * m.kv_cache.max_pages or m.kv_cache.max_pages == 1


def test_invalid_requests_raise():
    m = BUILDERS["llama"]()
    ids, _ = _prompt("plain")
    with pytest.raises(ValueError, match="paged_kv_cache must be True or False"):
        m.generate(ids, max_length=10, paged_kv_cache="yes")
    with pytest.raises(ValueError, match="speculative decoding"):
        m.generate(ids[:1], max_length=10, paged_kv_cache=True, prompt_lookup_num_tokens=2)
    with pytest.raises(ValueError, match="speculative decoding"):
        m.generate(ids[:1], max_length=10, paged_kv_cache=True, assistant_model=BUILDERS["llama"]())
    with pytest.raises(ValueError, match="not a decoder-only model"):
        MODELS["t5"]().generate(ids, max_length=6, paged_kv_cache=True)

    class TwoWay:   # a tensor-parallel topology
        tensor_parallel_size, pipeline_parallel_size = 2, 1

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(dist, "get_dist_util", lambda: TwoWay())
        with pytest.raises(ValueError, match="tensor- and pipeline-parallel"):
            m.generate(ids, max_length=10, paged_kv_cache=True)


def test_the_reference_path_checks_page_ids():
    pool = torch.zeros(3, G, 64, D, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="outside"):
        OF.kv_pages_gather(pool, torch.tensor([[0, 5]], dtype=torch.int32), 100)
    with pytest.raises(ValueError, match="page ids"):
        OF.kv_page_copy([pool], [(0, 3)])
