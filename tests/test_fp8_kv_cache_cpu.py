"""FP8 (E4M3) KV cache without a GPU: the quantizer's rounding and range, the cache's bookkeeping of rows and scales,
and every model that decodes on the preallocated cache, whose cached logits with an FP8 cache must equal those of a
bf16 cache holding the dequantized rows, and whose native calls (under the stub extension of
``tests/test_cached_attention_cpu.py``) must be the FP8 append and decode ones."""
import copy
import sys

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import CASES, MODELS, TRACES, _expand, _prompt, _StubExt, _token

FP8 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


# ------------------------------------------------------------------------------------------------ quantizer
def _rows(seed, n=64, d=128):
    """bf16 rows spanning many magnitudes, with tiny elements (E4M3 subnormals after scaling), a zero row and a row
    at the bf16 maximum."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=g) * torch.logspace(-30, 30, n)[:, None]
    x[:, :8] *= 1e-4
    x[3] = 0
    x[5, 0] = 3.3895e38
    return x.bfloat16()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_quantizer_round_trip_and_range(seed):
    x = _rows(seed)
    e, s = OF.kv_cache_quantize_ref(x)
    assert e.dtype == FP8 and s.dtype == torch.float32 and s.shape == x.shape[:-1]
    ef = e.float()
    assert not torch.isnan(ef).any()
    zero = (x == 0).all(-1)
    assert bool((s[zero] == 1).all()) and not ef[zero].any()
    assert bool((ef[~zero].abs().amax(-1) == 448).all())                      # each row's largest element
    assert torch.equal(s[~zero], x.float().abs().amax(-1)[~zero] / 448)
    back, xf = ef * s[:, None], x.float()
    normal = (xf / s[:, None]).abs() >= 2.0 ** -6                             # E4M3's smallest normal
    err = (back - xf).abs()
    assert bool((err[normal] <= 2.0 ** -4 * xf.abs()[normal]).all())
    assert bool((err[~normal] <= 2.0 ** -10 * s[:, None].expand_as(err)[~normal]).all())
    assert (~normal & (xf != 0)).any()                                        # subnormals were exercised
    assert torch.equal(OF.kv_cache_dequant(e, s), back.bfloat16())
    assert OF.kv_cache_dequant(e, s, torch.float32).dtype == torch.float32


def test_quantizer_is_the_division_rule():
    """Stored byte = e4m3_rn_satfinite(x / s): the cast of the fp32 quotient, which never exceeds ±448."""
    x = _rows(7)
    e, s = OF.kv_cache_quantize_ref(x)
    q = x.float() / s[:, None]
    assert float(q.abs().max()) <= 448 * (1 + 2 ** -23)
    assert torch.equal(e.view(torch.uint8), q.to(FP8).view(torch.uint8))


# ------------------------------------------------------------------------------------------------ bookkeeping
def _cache(b=3, g=2, cap=10, d=8, layers=2):
    return StaticKVCache(layers, b, g, d, cap, torch.bfloat16, "cpu", kv_dtype=FP8)


def _window(c, i, L):
    return c.layer(i).window(L, torch.bfloat16)


def test_fp8_cache_layout():
    c = _cache(cap=10)
    assert c.capacity == 12 and c.fp8                                          # rounded to a multiple of 4
    assert c.k[0].dtype == FP8 and c.k[0].shape == (3, 2, 12, 8)
    assert c.k_scale[1].dtype == torch.float32 and c.k_scale[1].shape == (3, 2, 12)
    assert c.matches(3, torch.bfloat16, "cpu", FP8) and not c.matches(3, torch.bfloat16, "cpu")
    bf = StaticKVCache(1, 3, 2, 8, 10, torch.bfloat16, "cpu")
    assert bf.capacity == 10 and bf.k_scale == [None] and bf.matches(3, torch.bfloat16, "cpu")
    assert not bf.matches(3, torch.bfloat16, "cpu", FP8)
    with pytest.raises(ValueError):
        StaticKVCache(1, 3, 2, 8, 10, torch.bfloat16, "cpu", kv_dtype=torch.float16)


def test_rows_and_scales_move_together():
    g = torch.Generator().manual_seed(0)
    c = _cache(cap=5)
    k, v = (torch.randn(3, 2, 5, 8, generator=g) * 10).bfloat16(), torch.randn(3, 2, 5, 8, generator=g).bfloat16()
    for i in range(2):
        c.write_rows(i, k, v)
    c.advance(5)
    want_k = OF.kv_cache_dequant(*OF.kv_cache_quantize_ref(k))
    want_v = OF.kv_cache_dequant(*OF.kv_cache_quantize_ref(v))
    assert all(torch.equal(a, b) for a, b in zip(_window(c, 1, 5), (want_k, want_v)))
    # an append through the kernel's reference at rows 5 .. 6 (one grouped step of 2 tokens)
    assert c.capacity == 8
    c.reserve(4)
    assert c.capacity == 16
    assert all(torch.equal(a, b) for a, b in zip(_window(c, 1, 5), (want_k, want_v)))    # reserve copied scales
    qkv = torch.randn(3, 2, 2, 3, 8, generator=g).bfloat16()
    for i in range(2):
        c.layer(i).append(qkv)
    new_k = OF.kv_cache_dequant(*OF.kv_cache_quantize_ref(qkv[:, :, :, 1].transpose(1, 2)))
    assert torch.equal(_window(c, 0, 7)[0][:, :, 5:7], new_k)
    c.advance(2)
    # beam search: rows and scales gathered alike
    before = [_window(c, i, 7) for i in range(2)]
    idx = torch.tensor([2, 2, 0])
    c.reorder_(idx)
    for i in range(2):
        for got, old in zip(_window(c, i, 7), before[i]):
            assert torch.equal(got, old[idx])
    # reset keeps the buffers and scales; new rows overwrite them
    scales = c.k_scale[0].clone()
    c.reset()
    assert c.length == 0 and torch.equal(c.k_scale[0].view(torch.int32), scales.view(torch.int32))
    # fill (a cross-attention window) quantizes by the mirror
    c.fill(((k, v), (v, k)), 5, (torch.tensor([1, 0, 2], dtype=torch.int32), torch.tensor([5, 4, 5],
                                                                                       dtype=torch.int32)))
    assert c.length == 5 and c.seqlens.tolist() == [5, 4, 5] and c.kv_start.tolist() == [1, 0, 2]
    assert torch.equal(_window(c, 1, 5)[0], want_v) and torch.equal(_window(c, 0, 5)[1], want_v)


def test_scales_required_for_fp8_and_rejected_otherwise():
    c = _cache()
    qkv = torch.randn(3, 1, 2, 3, 8).bfloat16()
    with pytest.raises(ValueError):
        OF.kv_cache_append(qkv, c.k[0], c.v[0], c.seqlens)
    bf = StaticKVCache(1, 3, 2, 8, 10, torch.bfloat16, "cpu")
    with pytest.raises(ValueError):
        OF.kv_cache_append(qkv, bf.k[0], bf.v[0], bf.seqlens, k_scale=c.k_scale[0], v_scale=c.v_scale[0])
    q = torch.randn(3, 1, 2, 8).bfloat16()
    with pytest.raises(ValueError):
        OF.decode_attention(q, c.k[0], c.v[0], c.seqlens, c.kv_start, scale=0.3)
    with pytest.raises(ValueError):
        OF.decode_attention_ref(q, bf.k[0], bf.v[0], bf.seqlens, bf.kv_start, scale=0.3, k_scale=c.k_scale[0],
                                v_scale=c.v_scale[0])


# ------------------------------------------------------------------------------------------------ models
def _run(m, name, case, fp8):
    """The cases of test_cached_attention_cpu, returning what the model produced: per-step scores (generate) or logits
    (teacher forced)."""
    ids, am = _prompt(case)
    kv = FP8 if fp8 else None
    with torch.no_grad():
        if case == "teacher_forced":
            m.kv_cache_dtype = kv
            if name == "t5":
                dec = torch.randint(2, 100, (3, 20), generator=torch.Generator().manual_seed(3))
                m.allocate_kv_cache(3, 20)
                out = [m(ids, dec[:, :1], am, use_cache=True)["logits"],
                       m(ids, dec[:, 1:], am, use_cache=True)["logits"]]
            else:
                more = torch.randint(3, 100, (3, 18), generator=torch.Generator().manual_seed(3))
                m.allocate_kv_cache(3, 25)
                out = [m(ids, use_cache=True)["logits"], m(more, use_cache=True)["logits"]]
            m.kv_cache_dtype = None
            return torch.cat(out, dim=1).float()
        beams = 2 if case == "beams" else 1
        if name == "t5":
            res = m.generate(ids, encoder_attn_mask=am, max_length=5, eos_token_id=None, num_beams=beams,
                             output_scores=True, kv_cache_dtype=kv)
        else:
            kw = {} if am is None else {"attention_mask": am}
            res = m.generate(ids, max_length=ids.shape[1] + 4, eos_token_id=None, num_beams=beams, output_scores=True,
                             kv_cache_dtype=kv, **kw)
        seqs, scores = res[0], res[-1]
        return torch.cat([seqs.float().flatten()] + [s.float().flatten() for s in scores])


def _round_trip(x):
    return OF.kv_cache_dequant(*OF.kv_cache_quantize_ref(x), x.dtype)


@pytest.fixture
def dequantized_bf16_cache(monkeypatch):
    """bf16 caches that hold every row as it reads back from an FP8 cache: quantized and dequantized on writing."""
    real_append, real_write = OF.kv_cache_append_ref, StaticKVCache.write_rows

    def append(qkv, k_cache, v_cache, cache_seqlens, cos=None, sin=None, k_scale=None, v_scale=None):
        q = real_append(qkv, k_cache, v_cache, cache_seqlens, cos, sin, k_scale, v_scale)
        if k_scale is None:
            s = qkv.shape[1]
            for b, st in enumerate(cache_seqlens.tolist()):
                for c in (k_cache, v_cache):
                    c[b, :, st : st + s] = _round_trip(c[b, :, st : st + s])
        return q

    def write_rows(self, i, k, v, row0=0):
        if not self.fp8:
            k, v = _round_trip(k), _round_trip(v)
        real_write(self, i, k, v, row0)

    monkeypatch.setattr(OF, "kv_cache_append_ref", append)
    monkeypatch.setattr(StaticKVCache, "write_rows", write_rows)


@pytest.mark.parametrize("name,case", CASES)
def test_fp8_cache_equals_attention_over_dequantized_cache(dequantized_bf16_cache, name, case):
    m = MODELS[name]()
    want_model = copy.deepcopy(m)   # (ChatGLM's builder draws from the global generator: two builds differ)
    got = _run(m, name, case, fp8=True)
    want = _run(want_model, name, case, fp8=False)
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max()), float((got - want).abs().max())


class _Fp8Stub(_StubExt):
    """The stub extension with the FP8 append and the decode op's scales; FP8 calls are marked with an ``8``."""

    def kv_append_fp8(self, qkv, k_cache, v_cache, k_scale, v_scale, seqlens, cos, sin, write_q):
        self.calls.append("a8")
        return OF.kv_cache_append_ref(qkv, k_cache, v_cache, seqlens, cos, sin, k_scale, v_scale)

    def decode_attn(self, q, k_cache, v_cache, seqlens, kv_start, scale, splits, alibi_slopes=None, rel_bias=None,
                    causal=True, k_scale=None, v_scale=None):
        self.calls.append(_token("D", causal, kv_start is not None, False, alibi_slopes is not None,
                                 rel_bias is not None) + ("8" if k_scale is not None else ""))
        return OF.decode_attention_ref(q, k_cache, v_cache, seqlens, kv_start, scale=scale, alibi_slopes=alibi_slopes,
                                       rel_bias=rel_bias, causal=causal, k_scale=k_scale, v_scale=v_scale)


@pytest.fixture
def native_fp8(monkeypatch):
    from projects.BLOOM.modeling import bloom_model
    from projects.ChatGLM import chatglm

    ext = _Fp8Stub()
    attention_checks = {"_decode_native", "attention_supported", "attention_qkvpacked_supported"}
    monkeypatch.setattr(OF, "use_native", lambda *t: sys._getframe(1).f_code.co_name in attention_checks)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: ext)
    for mod in (bloom_model, chatglm):
        monkeypatch.setattr(mod, "use_native", lambda *t: True)
    return ext


def _fp8_trace(trace):
    """The bf16 trace with every append and decode call an FP8 one; the flash calls (prefill, continuations, the
    encoder, dense-bias cross-attention) read the dequantized window and are unchanged."""
    return [t + "8" if t == "a" or t.startswith("D") else t for t in _expand(trace)]


@pytest.mark.parametrize("name,case", CASES)
def test_kernel_calls_of_fp8_cached_generation(native_fp8, name, case):
    _run(MODELS[name](), name, case, fp8=True)
    assert native_fp8.calls == _fp8_trace(TRACES[name, case])


def test_generate_option_restored_and_cfg_default():
    m = MODELS["llama"]()
    ids, _ = _prompt("plain")
    m.generate(ids, max_length=9, eos_token_id=None, kv_cache_dtype=FP8)
    assert m.kv_cache.kv_dtype == FP8 and m.kv_cache_dtype is None
    m.generate(ids, max_length=9, eos_token_id=None)
    assert m.kv_cache.kv_dtype == torch.bfloat16                               # the default: the weights' dtype
    m.cfg.kv_cache_dtype = "fp8"
    m.generate(ids, max_length=9, eos_token_id=None)
    assert m.kv_cache.kv_dtype == FP8
    with pytest.raises(ValueError):
        m.generate(ids, max_length=9, eos_token_id=None, kv_cache_dtype="int8")


def test_generate_fp8_raises_on_a_tuple_cache_model(monkeypatch):
    """T5 under pipeline parallelism keeps tuple caches: no StaticKVCache to hold FP8 rows."""
    m = MODELS["t5"]()
    monkeypatch.setattr(dist.get_dist_util(), "pipeline_parallel_size", 2)
    ids, _ = _prompt("plain")
    with pytest.raises(ValueError, match="StaticKVCache"):
        m.generate(ids, max_length=5, eos_token_id=None, kv_cache_dtype="fp8")
    assert m.kv_cache_dtype is None
