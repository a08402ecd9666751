"""The paged flash prefill off the GPU: ``OF.attention_paged`` is the sm_90a kernel only, so without it the call raises
instead of falling back, and ``attention_paged_supported`` says so; a paged cache's prefill then takes the gather path,
whose output is the reference attention over the gathered rows."""
import pytest
import torch

from libai_b200.inference.kv_cache import PagedKVCache
from libai_b200.ops import functional as OF


def test_attention_paged_is_native_only():
    q = torch.randn(1, 20, 2, 64, dtype=torch.bfloat16)
    pool = torch.randn(2, 2, 64, 64, dtype=torch.bfloat16)
    table = torch.tensor([[1]], dtype=torch.int32)
    assert not OF.attention_paged_supported(q, pool)
    with pytest.raises(RuntimeError, match="attention_paged"):
        OF.attention_paged(q, pool, pool, table, 0, scale=0.125)


def test_paged_prefill_off_the_gpu_attends_over_the_gathered_rows():
    gen = torch.Generator().manual_seed(0)
    B, G, r, D, s = 2, 2, 2, 64, 70
    c = PagedKVCache(1, B, G, D, 128, torch.float32)
    c.reserve(s)
    layer = c.layer(0)
    q = layer.append(torch.randn(B, s, G, r + 2, D, generator=gen))
    k, v = layer.window(s, torch.float32)
    want = OF.attention(q.transpose(1, 2), k, v, causal=True, scale=D ** -0.5).transpose(1, 2)
    assert torch.equal(layer.attend(q, scale=D ** -0.5), want)
