"""Prefix caching on the reference path: the index's matching (left padding, a mismatch inside a page, the
``(s - 1) // 64`` cap), LRU leaf eviction at the budget, reference counts and the free list across calls, hits, forks,
beam reorders and ``reset()``; invalidation and ``clear_prefix_cache()``; the prompts that are not cached; the
``ValueError``s; and ``generate()`` with a hit against the same rows in a contiguous cache."""
import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference.kv_cache import PagedKVCache, StaticKVCache
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import LLAMA, MODELS


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


G, D = 2, 64


def _books(c):
    """The reference counts and free list recounted from the tables and the index."""
    refs = [0] * c.num_pages
    for page in c._entry:
        refs[page] += 1
    for row in c.host_table[: c.batch]:
        for p in row[: c.mapped]:
            refs[p] += 1
    assert refs == c.refs
    assert sorted(c.free) == [p for p in range(c.num_pages) if refs[p] == 0]
    assert len(c._entry) <= c.prefix_pages


def _prefill(c, ids, mask=None):
    """A call's prefill on cache ``c``: lookup, append the remaining rows, insert."""
    hit = c.lookup(ids, mask)
    n = ids.shape[1] - c.length
    c.reserve(n)
    c.layer(0).append(torch.randn(c.batch, n, G, 3, D).to(torch.bfloat16))
    c.advance(n)
    c.insert(ids, mask)
    return hit


def _cache(b=2, prefix=640, fork=1):
    return PagedKVCache(1, b, G, D, 400, fork=fork, prompt_len=200, prefix_tokens=prefix)


def _ids(b, s, seed=0):
    return torch.randint(3, 100, (b, s), generator=torch.Generator().manual_seed(seed))


def test_matching_left_padding_and_a_mismatch_inside_a_page():
    c = _cache()
    ids = _ids(2, 200)
    assert _prefill(c, ids) == 0 and c.cached_pages() == 6   # three full pages per prompt
    _books(c)
    c.reset()
    assert _prefill(c, ids) == 3 and c.reused_rows == 192
    _books(c)
    c.reset()
    other = ids.clone()
    other[1, 70] += 1   # row 1 differs inside its second page: the batch's hit is one page
    assert _prefill(c, other) == 1
    c.reset()
    mask = torch.ones_like(ids)
    mask[:, :3] = 0   # left padding: other keys
    assert _prefill(c, ids.masked_fill(mask == 0, 0), mask) == 0
    c.reset()
    assert _prefill(c, ids.masked_fill(mask == 0, 0), mask) == 3 and c.kv_start.tolist() == [3, 3]
    _books(c)


def test_the_hit_leaves_at_least_one_token_to_prefill():
    c = _cache()
    ids = _ids(2, 128)
    _prefill(c, ids)
    c.reset()
    assert _prefill(c, ids) == 1   # (128 - 1) // 64


def test_dense_mask_prompts_are_neither_looked_up_nor_inserted():
    c = _cache()
    ids, mask = _ids(2, 150), torch.ones(2, 150, dtype=torch.long)
    mask[1, 10] = 0   # a hole
    assert _prefill(c, ids, mask) == 0 and c.cached_pages() == 0 and not c.prefix_ok


def test_lru_leaves_are_evicted_at_the_budget():
    c = _cache(b=1, prefix=192)
    x, y = _ids(1, 140, 1), _ids(1, 140, 2)
    _prefill(c, x)   # x0 -> x1
    c.reset()
    _prefill(c, y)   # y0 -> y1: four pages, the least recently used leaf x1 goes
    assert c.cached_pages() == 3
    keys = {page: key for page, key in c._entry.items()}
    assert sum(1 for p, k in keys.items() if k[0] == -1) == 2   # both first pages stay
    _books(c)
    c.reset()
    assert _prefill(c, x) == 1   # x0 is still there, x1 is not
    _books(c)


def test_books_across_forks_reorders_and_reset():
    c = _cache(b=2, fork=3)
    ids = _ids(2, 150)
    for _ in range(2):
        _prefill(c, ids)
        c.fork(3)
        _books(c)
        for step in range(70):
            c.reserve(1)
            c.layer(0).append(torch.randn(c.batch, 1, G, 3, D).to(torch.bfloat16))
            c.advance(1)
            if step % 7 == 0:
                c.reorder_(torch.tensor([0, 0, 1, 5, 4, 4]))
            _books(c)
        c.reset()
        _books(c)
    assert c.reused_rows == 128


def test_clear_prefix_cache():
    c = _cache()
    _prefill(c, _ids(2, 200))
    c.reset()
    c.clear_prefix_index()
    assert c.cached_pages() == 0 and len(c.free) == c.num_pages
    _books(c)


def _llama():
    from libai_b200.models import LlamaForCausalLM

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return LlamaForCausalLM(DictConfig(dict(LLAMA, max_position_embeddings=512))).eval()


def _gen(m, ids, **kw):
    return m.generate(ids, max_new_tokens=6, eos_token_id=None, output_scores=True, prefix_cache_tokens=512, **kw)


def test_generate_hit_matches_the_same_rows_in_a_contiguous_cache():
    m = _llama()
    a = _ids(2, 150, 3)
    _gen(m, a)
    assert m.kv_cache.reused_rows == 0
    b = torch.cat([a[:, :140], _ids(2, 30, 4)], dim=1)
    ids, scores = _gen(m, b)
    c = m.kv_cache
    assert isinstance(c, PagedKVCache) and c.reused_rows == 128
    # the reference: the index pages' rows written into a contiguous cache, the suffix as one cached step, then greedy
    table = []
    for row in b.tolist():
        parent, pages = -1, []
        for key in c._page_keys(row, [1] * 170, 2):
            parent = c._index[(parent, key)]
            pages.append(parent)
        table.append(pages)
    table = torch.tensor(table, dtype=torch.int32)
    ref = StaticKVCache(2, 2, c.heads, c.head_dim, 200, torch.bfloat16)
    for i in range(2):
        ref.write_rows(i, OF.kv_pages_gather(c.k[i], table, 128), OF.kv_pages_gather(c.v[i], table, 128))
    ref.advance(128)
    m.kv_cache, m.kv_cache_paging = ref, None
    with torch.no_grad():
        seq, want = b, []
        out = m(seq[:, 128:], use_cache=True)
        for _ in range(6):
            logits = out["logits"][:, -1].float()
            want.append(logits)
            seq = torch.cat([seq, logits.argmax(-1, keepdim=True)], dim=1)
            out = m(seq[:, -1:], use_cache=True)
    del m.kv_cache_paging
    assert torch.equal(ids, seq)
    assert all(torch.equal(x, y) for x, y in zip(scores, want))


def test_invalidation_and_clear_prefix_cache():
    m = _llama()
    a = _ids(1, 150, 5)
    _gen(m, a)
    _gen(m, a)
    assert m.kv_cache.reused_rows == 128
    m.load_state_dict(m.state_dict())
    _gen(m, a)
    assert m.kv_cache.reused_rows == 0
    with torch.no_grad():
        next(m.parameters()).add_(0)
    _gen(m, a)
    assert m.kv_cache.reused_rows == 0
    _gen(m, a)
    assert m.kv_cache.reused_rows == 128
    _gen(m, a, kv_cache_dtype="fp8")   # another cache format: a new pool
    assert m.kv_cache.reused_rows == 0
    m.clear_prefix_cache()
    _gen(m, a, kv_cache_dtype="fp8")
    assert m.kv_cache.reused_rows == 0


def test_p_tuning_rows_are_not_cached():
    m = MODELS["chatglm_prefix"]()
    ids = _ids(1, 40, 6)
    for _ in range(2):
        m.generate(ids, max_new_tokens=2, eos_token_id=None, prefix_cache_tokens=256)
        assert m.kv_cache.reused_rows == 0 and m.kv_cache.cached_pages() == 0


def test_value_errors():
    m = _llama()
    ids = _ids(1, 10)
    with pytest.raises(ValueError, match="paged_kv_cache=False"):
        m.generate(ids, max_new_tokens=2, prefix_cache_tokens=64, paged_kv_cache=False)
    with pytest.raises(ValueError, match="prefix_cache_tokens must be"):
        m.generate(ids, max_new_tokens=2, prefix_cache_tokens=-1)
    with pytest.raises(ValueError, match="prefix_cache_tokens > 0: speculative"):
        m.generate(ids, max_new_tokens=2, prefix_cache_tokens=64, prompt_lookup_num_tokens=2)
    with pytest.raises(ValueError, match="prefix_cache_tokens > 0: MT5Model"):
        MODELS["t5"]().generate(ids, max_new_tokens=2, prefix_cache_tokens=64)
    m.prefix_caching = False   # as GLM's class marks itself
    with pytest.raises(ValueError, match="prefix_cache_tokens > 0: LlamaForCausalLM's cached rows"):
        m.generate(ids, max_new_tokens=2, prefix_cache_tokens=64)
