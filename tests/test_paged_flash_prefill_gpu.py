"""The paged flash-attention prefill on the H100: ``OF.attention_paged`` reads a paged cache's pages in place and is
bit-identical to the contiguous flash kernel over the gathered rows (both head dims, grouped-query heads, ALiBi, left
padding, shuffled and shared pages, NaN in every page the table does not reference and in every row past the window);
a paged prefill, and a continuation of more than 16 tokens, gather nothing."""
import pytest
import torch

from libai_b200 import ops
from libai_b200.inference.kv_cache import PagedKVCache
from libai_b200.ops import functional as OF

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pools(B, G, D, Sk, gen):
    """K and V pools holding ``B`` sequences of ``Sk`` random rows at shuffled page ids, samples 0 and 1 sharing their
    first page; every unreferenced page, and every row of a referenced page at or past ``Sk``, NaN.  The table has one
    slot more than the rows need, left unmapped (-1)."""
    M = -(-Sk // 64)
    P = B * M + 5
    perm = torch.randperm(P, generator=gen).tolist()
    table = torch.full((B, M + 1), -1, dtype=torch.int32)
    for b in range(B):
        for j in range(M):
            table[b, j] = perm[b * M + j]
    table[1, 0] = table[0, 0]
    pools = []
    for _ in range(2):
        pool = torch.full((P, G, 64, D), float("nan"), dtype=torch.bfloat16)
        for b in range(B):
            for j in range(M):
                n = min(64, Sk - 64 * j)
                if not (b == 1 and j == 0):   # the shared page holds sample 0's rows
                    pool[table[b, j], :, :n] = torch.randn(G, n, D, generator=gen).to(torch.bfloat16)
        pools.append(pool.to(DEV))
    return table.to(DEV), pools


@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("r", [1, 4])
@pytest.mark.parametrize("D", [64, 128])
def test_paged_prefill_is_bit_identical_to_the_gathered_flash_kernel(D, r, alibi):
    gen = torch.Generator().manual_seed(D * 10 + r + alibi)
    B, G = 3, 2
    A = G * r
    start = torch.tensor([0, 37, 100], dtype=torch.int32, device=DEV)   # a different left padding per sample
    slopes = torch.linspace(0.05, 0.5, A, device=DEV) if alibi else None
    scale = D ** -0.5
    for past in (0, 64, 100, 192):
        for s in (17, 64, 129, 300):
            Sk = past + s
            table, (kp, vp) = _pools(B, G, D, Sk, gen)
            q = torch.randn(B, s, A, D, generator=gen).to(DEV, torch.bfloat16)
            k, v = OF.kv_pages_gather(kp, table, Sk), OF.kv_pages_gather(vp, table, Sk)
            want = OF.attention(q.transpose(1, 2), k, v, causal=True, scale=scale, kv_start=start,
                                alibi_slopes=slopes).transpose(1, 2)
            got = OF.attention_paged(q, kp, vp, table, past, start, scale=scale, alibi_slopes=slopes)
            assert not got.isnan().any(), (past, s)
            assert torch.equal(got, want), (past, s)


def test_paged_prefill_and_long_continuation_gather_nothing(monkeypatch):
    gen = torch.Generator().manual_seed(0)
    B, G, r, D = 2, 2, 2, 128
    c = PagedKVCache(1, B, G, D, 320, torch.bfloat16, DEV)
    c.kv_start.copy_(torch.tensor([0, 5], dtype=torch.int32))
    layer, scale = c.layer(0), D ** -0.5
    for s in (150, 40):   # the prefill, then a continuation past the decode kernel's 16 tokens
        qkv = torch.randn(B, s, G, r + 2, D, generator=gen).to(DEV, torch.bfloat16)
        c.reserve(s)
        q = layer.append(qkv)
        k, v = layer.window(c.length + s, torch.bfloat16)   # the gathered window, the reference's input
        want = OF.attention(q.transpose(1, 2), k, v, causal=True, scale=scale, kv_start=c.kv_start).transpose(1, 2)
        with monkeypatch.context() as mp:
            mp.setattr(OF, "kv_pages_gather", lambda *a, **k: pytest.fail("a paged prefill gathered its rows"))
            ops.reset_launch_count()
            got = layer.attend(q, scale=scale)
            assert ops.launch_count() == 1
        assert torch.equal(got, want), s
        c.advance(s)


def test_attn_fwd_paged_checks_its_arguments():
    ext = ops.load_ext()
    q = torch.zeros(1, 20, 2, 64, dtype=torch.bfloat16, device=DEV)
    pool = torch.zeros(3, 2, 64, 64, dtype=torch.bfloat16, device=DEV)
    table = torch.zeros(1, 1, dtype=torch.int32, device=DEV)
    assert ext.attn_fwd_paged(q, pool, pool, table, 0, 0.125).shape == (1, 20, 2, 64)
    bad = {
        "q must be": lambda: ext.attn_fwd_paged(q.float(), pool, pool, table, 0, 0.125),
        "head dim must be 64 or 128": lambda: ext.attn_fwd_paged(q[..., :32], pool, pool, table, 0, 0.125),
        "k_pool must be": lambda: ext.attn_fwd_paged(q, pool[:, :, :32], pool[:, :, :32], table, 0, 0.125),
        "v_pool must be": lambda: ext.attn_fwd_paged(q, pool, pool[:2], table, 0, 0.125),
        "block_table must be": lambda: ext.attn_fwd_paged(q, pool, pool, table.long(), 0, 0.125),
        "multiple of the K/V heads": lambda: ext.attn_fwd_paged(q, pool[:, :1].expand(3, 3, 64, 64).contiguous(),
                                                                pool[:, :1].expand(3, 3, 64, 64).contiguous(),
                                                                table, 0, 0.125),
        "fit the block table": lambda: ext.attn_fwd_paged(q, pool, pool, table, 45, 0.125),
        "kv_start must be": lambda: ext.attn_fwd_paged(q, pool, pool, table, 0, 0.125, table[0, :1].long()),
        "must be on": lambda: ext.attn_fwd_paged(q, pool, pool, table.cpu(), 0, 0.125),
    }
    for match, call in bad.items():
        with pytest.raises(RuntimeError, match=match):
            call()
