"""BLOOM on the preallocated KV cache, without a GPU: the ALiBi reference of the decode attention against HF's absolute
ALiBi, cached greedy / beam generation against ``transformers.BloomForCausalLM``, cached teacher-forced logits against
the uncached forward, which kernels a bf16 model reaches with the native path selected, and tensor parallelism."""
import os
import re
import subprocess
import sys

import pytest
import torch

from libai_b200.config import DictConfig, LazyConfig
from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.layers._param import param_defaults
from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from projects.BLOOM.modeling import bloom_model
from projects.BLOOM.modeling.bloom_model import BloomForCausalLM, alibi_slopes, build_alibi_tensor
from tests.dist_utils import run_distributed


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


def _cfg(**kw):
    cfg = LazyConfig.load("projects/BLOOM/configs/bloom_inference.py").cfg
    cfg.update(dict(dict(vocab_size=96, hidden_size=64, hidden_layers=2, n_head=8), **kw))
    return cfg


def _model(dtype=torch.float32, seed=0, **kw):
    with param_defaults(dtype=dtype, device="cpu", seed=seed):
        return BloomForCausalLM(_cfg(**kw)).eval()


def _left_padded(b=3, s=7, pads=(0, 2, 4), seed=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(4, 96, (b, s), generator=g)
    am = torch.ones_like(ids)
    for i, p in enumerate(pads):
        ids[i, :p], am[i, :p] = 3, 0
    return ids, am


# ------------------------------------------------------------------------------------------------ reference math
def test_decode_reference_alibi_equals_hf_absolute_alibi():
    """Relative ALiBi over the cache window (``slope·(j − (len + i))``) gives HF's attention, whose bias counts key
    positions over the mask: the two differ by a constant along each query row."""
    g = torch.Generator().manual_seed(0)
    b, a, d, past, s, cap = 3, 6, 16, 9, 4, 20
    kv_start = torch.tensor([0, 3, 7], dtype=torch.int32)
    q = torch.randn(b, s, a, d, generator=g, dtype=torch.float64)
    k_cache = torch.randn(b, a, cap, d, generator=g, dtype=torch.float64)
    v_cache = torch.randn(b, a, cap, d, generator=g, dtype=torch.float64)
    lens = torch.full((b,), past, dtype=torch.int32)
    slopes = alibi_slopes(a)
    got = OF.decode_attention_ref(q, k_cache, v_cache, lens, kv_start, scale=0.25, alibi_slopes=slopes)

    L = past + s
    am = (torch.arange(L)[None, :] >= kv_start.long()[:, None]).long()       # [b, L]: zeros, then ones
    hf_bias = build_alibi_tensor(am, a, torch.float64)                         # [b, a, 1, L]
    want = OF.attention_ref(q.transpose(1, 2), k_cache[:, :, :L], v_cache[:, :, :L], causal=True, scale=0.25,
                            mask=am[:, None, None, :], bias=hf_bias).transpose(1, 2)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
    # the same call through the public entry point (which runs the reference here)
    torch.testing.assert_close(OF.decode_attention(q, k_cache, v_cache, lens, kv_start, scale=0.25,
                                                   alibi_slopes=slopes), got, rtol=0, atol=0)


# ------------------------------------------------------------------------------------------------ HF parity
def _hf_pair(tmp_path):
    transformers = pytest.importorskip("transformers")
    from projects.BLOOM.utils.model_loader import BlooMLoaderHuggerFace

    torch.manual_seed(0)
    hf = transformers.BloomForCausalLM(transformers.BloomConfig(
        vocab_size=96, hidden_size=64, n_layer=2, n_head=8, hidden_dropout=0.0, attention_dropout=0.0, pad_token_id=3,
        bos_token_id=1, eos_token_id=2)).eval()
    d = str(tmp_path / "bloom")
    hf.save_pretrained(d)
    cfg = LazyConfig.load("projects/BLOOM/configs/bloom_inference.py").cfg
    return hf, BlooMLoaderHuggerFace(BloomForCausalLM, cfg, d).load().eval()


@pytest.mark.parametrize("num_beams", [1, 2])
def test_cached_generate_matches_hf_on_a_left_padded_batch(tmp_path, num_beams, monkeypatch):
    hf, m = _hf_pair(tmp_path)
    reorders = []
    reorder = StaticKVCache.reorder_
    monkeypatch.setattr(StaticKVCache, "reorder_", lambda c, idx: (reorders.append(idx), reorder(c, idx)))
    ids, am = _left_padded()
    ours = m.generate(ids, attention_mask=am, max_length=16, eos_token_id=None, num_beams=num_beams)
    theirs = hf.generate(ids, attention_mask=am, max_length=16, do_sample=False, eos_token_id=None, pad_token_id=3,
                         num_beams=num_beams, early_stopping=False)
    assert ours.tolist() == theirs.tolist()
    assert isinstance(m.kv_cache, StaticKVCache)
    assert (len(reorders) > 0) == (num_beams > 1)   # beam search gathers the cache in place


# ------------------------------------------------------------------------------------------------ cached vs uncached
@pytest.mark.parametrize("padded", [False, True])
def test_teacher_forced_cached_logits_equal_uncached(padded):
    """Prefill, three single steps and one 17-token continuation (past the decode kernel's 16) through the cache give
    the uncached forward's logits at every non-padded position."""
    m = _model()
    ids, am = _left_padded(s=30, pads=(0, 3, 5) if padded else (0, 0, 0), seed=2)
    with torch.no_grad():
        want = m(ids, attention_mask=am)["logits"]
        m.allocate_kv_cache(3, 30)
        chunks = [(0, 10), (10, 11), (11, 12), (12, 13), (13, 30)]
        got = []
        for lo, hi in chunks:
            mask = am[:, :hi] if padded else None
            got.append(m(ids[:, lo:hi], attention_mask=mask, use_cache=True)["logits"])
        got = torch.cat(got, dim=1)
    assert m.kv_cache.length == 30
    keep = am.bool()
    torch.testing.assert_close(got[keep], want[keep], rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ dispatch
class _StubExt:
    """The extension's decode and flash ops, computed with the reference math; records every call."""

    def __init__(self):
        self.calls = []

    def kv_append(self, qkv, k_cache, v_cache, seqlens, cos, sin, write_q):
        self.calls.append(("kv_append", None))
        return OF.kv_cache_append_ref(qkv, k_cache, v_cache, seqlens)

    def decode_attn(self, q, k_cache, v_cache, seqlens, kv_start, scale, splits, alibi_slopes=None):
        self.calls.append(("decode_attn", alibi_slopes))
        return OF.decode_attention_ref(q, k_cache, v_cache, seqlens, kv_start, scale=scale, alibi_slopes=alibi_slopes)

    def attn_fwd(self, q, k, v, causal, scale, kv_lens, bias, alibi_slopes, p_drop, salt, kv_start=None,
                 doc_start=None):
        self.calls.append(("attn_fwd", alibi_slopes))
        sq, sk = q.shape[-2], k.shape[-2]
        vis = OF.visible_keys(sq, sk, causal=causal, kv_start=kv_start, kv_lens=kv_lens)
        rel = (torch.arange(sk)[None, :] - torch.arange(sk - sq, sk)[:, None]).float()
        o = OF.attention_ref(q, k, v, causal=False, scale=scale, mask=vis, bias=alibi_slopes[None, :, None, None] * rel)
        return o.masked_fill(~vis.any(-1, keepdim=True), 0), torch.empty(0), torch.empty(0)


@pytest.fixture
def native_attention(monkeypatch):
    """As if on the GPU for the attention ops only (the GEMMs and norms keep the PyTorch path)."""
    ext = _StubExt()
    attention_checks = {"_decode_native", "attention_supported", "attention_qkvpacked_supported"}
    monkeypatch.setattr(OF, "use_native", lambda *t: sys._getframe(1).f_code.co_name in attention_checks)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: ext)
    monkeypatch.setattr(bloom_model, "use_native", lambda *t: True)
    return ext


@pytest.mark.parametrize("padded", [False, True])
def test_bf16_head_dim_64_decodes_natively_with_slopes_in_every_layer(native_attention, padded):
    m = _model(torch.bfloat16, hidden_size=128, n_head=2)                  # head dim 64
    ids, am = _left_padded(pads=(0, 2, 4) if padded else (0, 0, 0))
    new = 5
    m.generate(ids, attention_mask=am, max_length=ids.shape[1] + new, eos_token_id=None)
    calls = native_attention.calls
    layers = 2
    assert [c[0] for c in calls].count("kv_append") == layers * new
    prefill = [c for c in calls if c[0] == "attn_fwd"]
    steps = [c for c in calls if c[0] == "decode_attn"]
    assert len(prefill) == layers and len(steps) == layers * (new - 1)
    full = alibi_slopes(2)
    for _, slopes in prefill + steps:
        assert slopes is not None and slopes.dtype == torch.float32 and torch.equal(slopes, full)


def test_bf16_head_dims_the_decode_kernel_does_not_take(native_attention):
    """Head dim 32: the flash kernel runs the prefill, the cache and the steps stay on the reference math; head dim
    36 (not a multiple of 8) never reaches the extension."""
    m = _model(torch.bfloat16, hidden_size=64, n_head=2)                   # head dim 32
    ids, am = _left_padded(pads=(0, 1, 2))
    m.generate(ids, attention_mask=am, max_length=ids.shape[1] + 4, eos_token_id=None)
    assert {c[0] for c in native_attention.calls} == {"attn_fwd"}
    native_attention.calls.clear()
    m = _model(torch.bfloat16, hidden_size=72, n_head=2)                   # head dim 36
    m.generate(ids, attention_mask=am, max_length=ids.shape[1] + 4, eos_token_id=None)
    assert native_attention.calls == []


# ------------------------------------------------------------------------------------------------ tensor parallel
def _generate_tp(rank, world):
    from libai_b200.utils import distributed as dutil

    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=world, pipeline_parallel_size=1,
                                          device_type="cpu")))
    m = _model(seed=7)
    ids, am = _left_padded()
    return m.generate(ids, attention_mask=am, max_length=16, eos_token_id=None)


def test_tensor_parallel_generation_matches_one_rank():
    one = run_distributed(_generate_tp, 1)[0]
    two = run_distributed(_generate_tp, 2)
    assert (two[0] == one).all() and (two[1] == one).all()


# ------------------------------------------------------------------------------------------------ build
@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_alibi_decode_kernels_compile_without_spills(tmp_path):
    src = "decode_attention_alibi_sm90.cu"
    assert src in ops_build.CU_SOURCES
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    spills = re.findall(r"Function properties for (\S+)\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                        res.stdout)
    # exactly the two ALiBi instances (head dims 64 and 128)
    assert sorted(name for name, _, _ in spills) == ["_ZN2lb3dec18decode_attn_kernelILi128ELb1EEEvNS0_6ParamsE",
                                                     "_ZN2lb3dec18decode_attn_kernelILi64ELb1EEEvNS0_6ParamsE"]
    assert all(st == "0" and ld == "0" for _, st, ld in spills), spills
