"""Head-dim dispatch of the flash attention kernels, without a GPU: with the native path selected, bf16 attention with a
head dim that is a multiple of 8 from 8 to 128 reaches the extension (4-D q/k/v and the packed 4-D and grouped 5-D
projections), while other head dims, other dtypes and decode attention outside 64 / 128 keep the reference math."""
import pytest
import torch

from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.ops import functional as OF

FLASH_DIMS = list(range(8, 129, 8))
REF_DIMS = [4, 20, 36, 100, 136, 256]


class _Reached(RuntimeError):
    pass


@pytest.fixture
def native_without_ext(monkeypatch):
    def no_ext(*a, **k):
        raise _Reached("native extension reached")

    monkeypatch.setattr(OF, "use_native", lambda *t: True)
    monkeypatch.setattr(OF, "load_ext", no_ext)


def _qkv(d, dtype, B=2, A=4, G=4, S=5):
    g = torch.Generator().manual_seed(d)
    return tuple(torch.randn(B, h, S, d, generator=g).to(dtype) for h in (A, G, G))


def test_flash_head_dim_predicate():
    assert [d for d in range(0, 300) if OF.flash_head_dim_supported(d)] == FLASH_DIMS


@pytest.mark.parametrize("d", FLASH_DIMS)
def test_bf16_flash_head_dims_reach_the_extension(native_without_ext, d):
    q, k, v = _qkv(d, torch.bfloat16)
    assert OF.attention_supported(q, k)
    with pytest.raises(_Reached):
        OF.attention(q, k, v, causal=True)
    for qkv in (torch.randn(2, 5, 4, 3 * d).bfloat16(), torch.randn(2, 5, 2, 4, d).bfloat16()):   # [b, s, a, 3d], r = 2
        assert OF.attention_qkvpacked_supported(qkv, None, 0.0, True)
        with pytest.raises(_Reached):
            OF.attention_qkvpacked(qkv, causal=False, scale=d ** -0.5)


def _assert_reference(q, k, v, qkv):
    """OF.attention / OF.attention_qkvpacked dispatch give exactly attention_ref's result (the extension would raise)."""
    d = q.shape[-1]
    assert not OF.attention_supported(q, k)
    assert torch.equal(OF.attention(q, k, v, causal=True), OF.attention_ref(q, k, v, causal=True, scale=d ** -0.5))
    assert not OF.attention_qkvpacked_supported(qkv, None, 0.0, True)


@pytest.mark.parametrize("d", REF_DIMS)
def test_other_head_dims_run_the_reference(native_without_ext, d):
    q, k, v = _qkv(d, torch.bfloat16)
    _assert_reference(q, k, v, torch.randn(2, 5, 4, 3 * d).bfloat16())


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("d", [24, 64, 80])
def test_other_dtypes_run_the_reference(native_without_ext, dtype, d):
    q, k, v = _qkv(d, dtype)
    _assert_reference(q, k, v, torch.randn(2, 5, 4, 3 * d).to(dtype))


def test_decode_attention_at_head_dim_32_runs_the_reference(native_without_ext):
    d = 32
    c = StaticKVCache(1, 2, 2, d, 32, torch.bfloat16, "cpu")
    c.k[0].copy_(torch.randn(c.k[0].shape))
    c.v[0].copy_(torch.randn(c.v[0].shape))
    c.seqlens.fill_(3)
    qkv = torch.randn(2, 1, 2, 3 * d).bfloat16()
    OF.kv_cache_append(qkv, c.k[0], c.v[0], c.seqlens)
    q = qkv[..., :d]
    got = OF.decode_attention(q, c.k[0], c.v[0], c.seqlens, c.kv_start, scale=0.1)
    want = OF.decode_attention_ref(q, c.k[0], c.v[0], c.seqlens, c.kv_start, scale=0.1)
    assert torch.equal(got, want)
