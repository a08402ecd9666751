"""The paged KV cache on the H100: the paged split-KV decode kernel is bit-identical to the contiguous one over the same
logical rows (bf16 and FP8, no bias and ALiBi, both head dims, shuffled and shared pages, NaN in every page the table
does not reference); the paged appends write the contiguous appends' bytes and scales; the page copy copies exactly
its pages; and ``generate(paged_kv_cache=True)`` returns the contiguous cache's tokens, with one decode-graph capture
through beam search."""
import pytest
import torch

from libai_b200.inference import decode_graph
from libai_b200.inference.kv_cache import PagedKVCache
from libai_b200.ops import functional as OF
from tests.test_decode_graphs_gpu import BUILDERS, PADDED, _Captures, _generate, _model, _same, _topo  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP8 = torch.float8_e4m3fn


def _paged_copy(k, v, ks, vs, gen, shared=True):
    """Pools holding the rows of contiguous caches ``[B, G, C, D]`` at shuffled page ids, samples 0 and 1 sharing
    their first page (whose rows are made equal first); every other page NaN."""
    B, G, C, D = k.shape
    M = C // 64
    if shared and B > 1:
        for t in (k, v) + ((ks, vs) if ks is not None else ()):
            t[1, :, :64] = t[0, :, :64]
    P = B * M + 5
    perm = torch.randperm(P, generator=gen).tolist()
    table = torch.tensor([[perm[b * M + j] for j in range(M)] for b in range(B)], dtype=torch.int32)
    if shared and B > 1:
        table[1, 0] = table[0, 0]
    pools = []
    for t in (k, v) + ((ks, vs) if ks is not None else ()):
        pool = torch.empty((P, G, 64) + tuple(t.shape[3:]), dtype=t.dtype, device=t.device)
        if t.dtype == FP8:
            pool.view(torch.uint8).fill_(0x7F)   # E4M3 NaN
        else:
            pool.fill_(float("nan"))
        for b in range(B):
            for j in range(M):
                pool[table[b, j]] = t[b, :, j * 64 : (j + 1) * 64]
        pools.append(pool)
    return table.to(t.device), pools


@pytest.mark.parametrize("Sq,r", [(1, 1), (4, 4), (16, 1), (1, 16), (4, 16)])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_paged_decode_is_bit_identical_to_contiguous(kv, alibi, D, Sq, r):
    gen = torch.Generator().manual_seed(D * 100 + Sq * 10 + r)
    B, G, C = 3, 2, 320
    A = G * r
    q = torch.randn(B, Sq, A, D, generator=gen).to(DEV, torch.bfloat16)
    k = torch.randn(B, G, C, D, generator=gen).to(DEV, torch.bfloat16)
    v = torch.randn(B, G, C, D, generator=gen).to(DEV, torch.bfloat16)
    ks = vs = None
    if kv == "fp8":
        (k, ks), (v, vs) = OF.kv_cache_quantize_ref(k), OF.kv_cache_quantize_ref(v)
    table, pools = _paged_copy(k, v, ks, vs, gen)
    slopes = torch.linspace(0.05, 0.5, A, device=DEV) if alibi else None
    for kv_start in (0, 37, 64, 100):
        for lens in ([kv_start + 1, 63, 130], [64, 127, 200], [129, 191, 256 - Sq]):
            seqlens = torch.tensor([max(x, kv_start) for x in lens], dtype=torch.int32, device=DEV)
            start = torch.full((B,), kv_start, dtype=torch.int32, device=DEV)
            for splits in (1, 0):
                scales = {} if ks is None else {"k_scale": ks, "v_scale": vs}
                want = OF.decode_attention(q, k, v, seqlens, start, scale=D ** -0.5, splits=splits,
                                           alibi_slopes=slopes, **scales)
                pscales = {} if ks is None else {"k_scale": pools[2], "v_scale": pools[3]}
                got = OF.decode_attention(q, pools[0], pools[1], seqlens, start, scale=D ** -0.5, splits=splits,
                                          alibi_slopes=slopes, block_table=table, **pscales)
                assert not got.isnan().any()
                assert torch.equal(got, want), (kv_start, lens, splits)


@pytest.mark.parametrize("case", ["bf16", "bf16_rotary", "gqa", "fp8"])
@pytest.mark.parametrize("D", [64, 128])
def test_paged_appends_write_the_contiguous_bytes(case, D):
    gen = torch.Generator().manual_seed(D)
    B, G, C, Sq = 3, 2, 256, 5
    r = 4 if case == "gqa" else 1
    qkv = torch.randn(B, Sq, G, r + 2, D, generator=gen).to(DEV, torch.bfloat16)
    seqlens = torch.tensor([0, 61, 130], dtype=torch.int32, device=DEV)
    cos = sin = None
    if case == "bf16_rotary":
        ang = torch.arange(C, dtype=torch.float32)[:, None] * torch.linspace(0.01, 1, D)[None]
        cos, sin = ang.cos().to(DEV), ang.sin().to(DEV)
    dtype = FP8 if case == "fp8" else torch.bfloat16
    k = torch.zeros(B, G, C, D, device=DEV).to(dtype)
    v = torch.zeros_like(k)
    ks = vs = None
    scales = {}
    if case == "fp8":
        ks, vs = torch.ones(B, G, C, device=DEV), torch.ones(B, G, C, device=DEV)
        scales = {"k_scale": ks, "v_scale": vs}
    table, pools = _paged_copy(k, v, ks, vs, gen, shared=False)
    q_want = OF.kv_cache_append(qkv, k, v, seqlens, cos, sin, **scales)
    pscales = {} if ks is None else {"k_scale": pools[2], "v_scale": pools[3]}
    q_got = OF.kv_cache_append(qkv, pools[0], pools[1], seqlens, cos, sin, block_table=table, **pscales)
    assert torch.equal(q_got, q_want)
    arrays = (k, v) + ((ks, vs) if ks is not None else ())
    for pool, full in zip(pools, arrays):
        got = OF.kv_pages_gather(pool, table, C)
        assert torch.equal(got.view(torch.uint8) if got.dtype == FP8 else got,
                           full.view(torch.uint8) if full.dtype == FP8 else full)


def test_page_copy_copies_exactly_the_listed_pages_of_every_array():
    gen = torch.Generator().manual_seed(0)
    arrays = [torch.randn(12, 2, 64, 64, generator=gen).to(DEV, torch.bfloat16) for _ in range(4)]
    arrays += [torch.randn(12, 2, 64, generator=gen).to(DEV) for _ in range(2)]
    before = [a.clone() for a in arrays]
    OF.kv_page_copy(arrays, [(1, 7), (3, 0), (11, 5)])
    for a, b in zip(arrays, before):
        want = b.clone()
        want[7], want[0], want[5] = b[1], b[3], b[11]
        assert torch.equal(a, want)


NAMES = sorted(n for n in BUILDERS if n != "t5")


@pytest.mark.parametrize("kv", [None, "fp8"])
@pytest.mark.parametrize("name", NAMES)
def test_generate_on_pages_matches_contiguous(name, kv):
    m = _model(name)
    case = "left_padded" if name in PADDED else "plain"
    _same(_generate(m, name, False, case, kv_cache_dtype=kv), _generate(m, name, False, case, kv_cache_dtype=kv,
                                                                          paged_kv_cache=True))
    assert isinstance(m.kv_cache, PagedKVCache)
    modes = [dict(num_beams=3)] + ([] if name == "glm" else [dict(do_sample=True, num_return_sequences=3)])
    for kw in modes:   # (GLM's test inputs are expanded per beam only)
        outs = []
        for paged in (False, True):
            torch.manual_seed(0)
            outs.append(_generate(m, name, False, case, kv_cache_dtype=kv, paged_kv_cache=paged, **kw)[0])
        assert torch.equal(*outs), kw


@pytest.mark.parametrize("name", NAMES)
def test_shared_prefill_logits_equal_the_expanded_prefill(name):
    m = _model(name)
    if name == "glm":
        pytest.skip("GLM's prompt inputs are built per beam by its tokenizer")
    from tests.test_cached_attention_cpu import _prompt

    ids, am = _prompt("left_padded" if name in PADDED else "plain")
    ids = ids.to(DEV)
    kw = {} if name not in PADDED else {"attention_mask": am.to(DEV)}
    with torch.no_grad():
        once = m(ids, **kw)
        many = m(ids.repeat_interleave(3, 0), **{k: x.repeat_interleave(3, 0) for k, x in kw.items()})
    key = "logits" if "logits" in once else "prediction_scores"
    assert torch.equal(once[key][:, -1].repeat_interleave(3, 0), many[key][:, -1])


@pytest.mark.parametrize("name", NAMES)
def test_paged_beam_search_keeps_one_capture(monkeypatch, name):
    m = _model(name)
    eager = _generate(m, name, False, paged_kv_cache=True, num_beams=3)
    captures = _Captures(monkeypatch)
    graphs = _generate(m, name, True, paged_kv_cache=True, num_beams=3)
    _same(eager, graphs)
    assert captures.n == 1 and decode_graph.current_graph(m).graph is not None
