"""KV-cache decoding on the CPU: the preallocated cache, the reference decode attention and cached generation of the
Llama family and MagicPrompt's GPT-2; with nvcc, the decode kernels' build (no spills, wgmma never serialized)."""
import os
import re
import subprocess

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference.kv_cache import StaticKVCache, left_padding
from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF

LLAMA = dict(hidden_layers=2, vocab_size=100, hidden_size=64, intermediate_size=128, num_attention_heads=4,
             max_position_embeddings=64, rms_norm_eps=1e-5, initializer_range=0.02,
             use_scaled_init_for_output_weights=True, scale_mask_softmax_fusion=False, amp_enabled=False,
             bos_token_id=1, eos_token_id=2, pad_token_id=0, max_length=20)


def _llama(seed=0):
    from libai_b200.models import LlamaForCausalLM
    from libai_b200.utils import distributed as dutil

    dutil.reset_dist_util()
    torch.manual_seed(seed)
    return LlamaForCausalLM(DictConfig(LLAMA)).eval()


# ------------------------------------------------------------------------------------------------ cache semantics
def _filled_cache(b=3, a=2, cap=8, d=4, n=5, layers=2):
    c = StaticKVCache(layers, b, a, d, cap, torch.float32, "cpu")
    qkv = torch.randn(b, n, a, 3 * d)
    for i in range(layers):
        OF.kv_cache_append(qkv, c.k[i], c.v[i], c.seqlens)
    c.advance(n)
    return c, qkv


def test_append_and_advance():
    c, qkv = _filled_cache()
    d = 4
    assert c.length == 5 and c.seqlens.tolist() == [5, 5, 5]
    assert torch.equal(c.k[0][:, :, :5], qkv[..., d : 2 * d].transpose(1, 2))
    assert torch.equal(c.v[1][:, :, :5], qkv[..., 2 * d :].transpose(1, 2))
    more = torch.randn(3, 2, 2, 3 * d)
    OF.kv_cache_append(more, c.k[0], c.v[0], c.seqlens)
    assert torch.equal(c.k[0][:, :, 5:7], more[..., d : 2 * d].transpose(1, 2))


def test_append_rope_matches_apply_rotary_qkv():
    from libai_b200.models.llama_model import rotary_tables

    cos, sin = rotary_tables(8, 32)
    qkv = torch.randn(2, 3, 2, 24)
    c = StaticKVCache(1, 2, 2, 8, 16, torch.float32, "cpu")
    c.seqlens.fill_(4)
    q = OF.kv_cache_append(qkv, c.k[0], c.v[0], c.seqlens, cos, sin)
    want = OF.apply_rotary_qkv(qkv, cos, sin, 4)
    assert torch.equal(q, want[..., :8])
    assert torch.equal(c.k[0][:, :, 4:7], want[..., 8:16].transpose(1, 2))
    assert torch.equal(c.v[0][:, :, 4:7], want[..., 16:].transpose(1, 2))


def test_growth_keeps_contents():
    c, _ = _filled_cache(cap=6)
    before = [t[:, :, :5].clone() for t in c.k + c.v]
    c.reserve(4)
    assert c.capacity == 12
    assert all(torch.equal(t[:, :, :5], b) for t, b in zip(c.k + c.v, before))
    c.reserve(7)                                       # fits: no reallocation
    assert c.capacity == 12
    c.reserve(30)
    assert c.capacity == 35 and all(torch.equal(t[:, :, :5], b) for t, b in zip(c.k + c.v, before))


def test_reorder_equals_index_select_and_reset():
    c, _ = _filled_cache()
    c.kv_start.copy_(torch.tensor([0, 1, 2], dtype=torch.int32))
    idx = torch.tensor([2, 0, 0])
    want = [t[:, :, :5].index_select(0, idx) for t in c.k + c.v]
    c.reorder_(idx)
    assert all(torch.equal(t[:, :, :5], w) for t, w in zip(c.k + c.v, want))
    assert c.kv_start.tolist() == [2, 0, 0]
    c.reset()
    assert c.length == 0 and c.seqlens.tolist() == [0, 0, 0] and c.kv_start.tolist() == [0, 0, 0]


def test_pipeline_stage_allocates_only_its_layers():
    from libai_b200.utils import distributed as dutil

    model = _llama()
    topo = dutil.get_dist_util()
    topo._layer_stage_ids = [0, 1]                 # layer 1 on a second stage
    topo.pipeline_parallel_size, topo.pp_rank = 2, 0
    try:
        c = model.allocate_kv_cache(2, 8)
        assert c.owned == [0] and c.k[0] is not None and c.k[1] is None
    finally:
        dutil.reset_dist_util()


def test_layers_of_other_stages_get_no_buffers():
    c = StaticKVCache(4, 1, 2, 8, 4, torch.float32, "cpu", layers=[2, 3])
    assert c.k[0] is None and c.v[1] is None and c.k[2].shape == (1, 2, 4, 8)
    c.reserve(10)
    assert c.k[0] is None and c.k[3].shape[2] == 10


def test_left_padding():
    m = torch.tensor([[0, 0, 1, 1], [1, 1, 1, 1], [0, 1, 1, 1]])
    assert left_padding(m).tolist() == [2, 0, 1]
    assert left_padding(torch.tensor([[1, 1, 0, 0]])) is None        # right padding
    assert left_padding(torch.tensor([[0, 1, 0, 1]])) is None        # holes


# ------------------------------------------------------------------------------------------------ reference decode attention
@pytest.mark.parametrize("sq", [1, 3])
@pytest.mark.parametrize("starts", [[0, 0], [2, 5]])
def test_reference_decode_attention_equals_dense_mask(sq, starts):
    torch.manual_seed(0)
    b, a, d, cap, past = 2, 3, 8, 32, 9
    k_cache, v_cache = torch.randn(b, a, cap, d), torch.randn(b, a, cap, d)
    seqlens = torch.full((b,), past, dtype=torch.int32)
    kv_start = torch.tensor(starts, dtype=torch.int32)
    q = torch.randn(b, sq, a, d)
    got = OF.decode_attention(q, k_cache, v_cache, seqlens, kv_start, scale=0.3)
    L = past + sq                                                   # window shorter than the capacity
    j = torch.arange(L)
    i = torch.arange(sq)
    mask = (j[None, None, :] >= kv_start[:, None, None]) & (j[None, None, :] <= past + i[None, :, None])
    want = OF.attention_ref(q.transpose(1, 2), k_cache[:, :, :L], v_cache[:, :, :L], causal=False, scale=0.3,
                            mask=mask[:, None]).transpose(1, 2)
    assert got.shape == (b, sq, a, d) and got.is_contiguous()
    torch.testing.assert_close(got, want, rtol=0, atol=0)


def test_reference_decode_attention_no_visible_key_gives_zeros():
    k_cache, v_cache = torch.randn(1, 1, 8, 4), torch.randn(1, 1, 8, 4)
    got = OF.decode_attention(torch.randn(1, 1, 1, 4), k_cache, v_cache, torch.tensor([3], dtype=torch.int32),
                              torch.tensor([5], dtype=torch.int32), scale=1.0)
    assert torch.equal(got, torch.zeros_like(got))


def test_native_dispatch_only_for_bf16_head_dims_64_128(monkeypatch):
    """With the native path selected, the decode ops still run the reference math for other dtypes, head dims and more
    than 16 new tokens (as ``OF.attention`` does); only the supported case reaches the extension."""
    def no_ext(*a, **k):
        raise RuntimeError("native extension reached")

    monkeypatch.setattr(OF, "use_native", lambda *t: True)
    monkeypatch.setattr(OF, "load_ext", no_ext)
    for dtype, d, sq in ((torch.float32, 64, 1), (torch.float16, 128, 1), (torch.bfloat16, 32, 1),
                         (torch.bfloat16, 100, 1), (torch.bfloat16, 64, 17)):
        c = StaticKVCache(1, 2, 2, d, 32, dtype, "cpu")
        c.seqlens.fill_(3)
        qkv = torch.randn(2, sq, 2, 3 * d).to(dtype)
        if d != 64:                       # (the append kernel itself takes any number of new tokens)
            OF.kv_cache_append(qkv, c.k[0], c.v[0], c.seqlens)
        o = OF.decode_attention(qkv[..., :d], c.k[0], c.v[0], c.seqlens, c.kv_start, scale=0.1)
        assert o.shape == (2, sq, 2, d) and o.dtype == dtype
    c = StaticKVCache(1, 2, 2, 64, 32, torch.bfloat16, "cpu")
    with pytest.raises(RuntimeError, match="native extension reached"):
        OF.decode_attention(torch.randn(2, 1, 2, 64).bfloat16(), c.k[0], c.v[0], c.seqlens, c.kv_start, scale=0.1)


# ------------------------------------------------------------------------------------------------ models
def test_llama_long_continuation_keeps_left_padding():
    """More than 16 tokens appended after a left-padded prefill still exclude the padding keys."""
    model = _llama()
    ids = torch.randint(3, 100, (2, 26))
    am = torch.ones_like(ids)
    ids[1, :3], am[1, :3] = 0, 0
    with torch.no_grad():
        want = model(ids, attention_mask=am)["logits"][:, 6:]
        model.allocate_kv_cache(2, 26)
        model(ids[:, :6], attention_mask=am[:, :6], use_cache=True)
        got = model(ids[:, 6:], use_cache=True)["logits"]
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
    model.set_cache(None)


def test_llama_left_padded_greedy_equals_bruteforce():
    model = _llama()
    ids = torch.randint(3, 100, (3, 6))
    am = torch.ones_like(ids)
    ids[0, :2], am[0, :2] = 0, 0
    ids[2, :4], am[2, :4] = 0, 0
    out = model.generate(ids, attention_mask=am, max_length=14, pad_token_id=0)
    cur, mask = ids.clone(), am.clone()
    with torch.no_grad():
        for _ in range(8):
            nxt = model(cur, attention_mask=mask)["logits"][:, -1].argmax(-1, keepdim=True)
            cur, mask = torch.cat([cur, nxt], 1), torch.cat([mask, torch.ones_like(nxt)], 1)
    done = (out == LLAMA["eos_token_id"]).cumsum(1) > 0    # generate pads a sample after its eos
    done[:, :6] = False
    assert torch.equal(cur[~done], out[~done])
    assert model.kv_cache.length == 0 and model.past_length == 0       # generate resets the cache


def test_llama_cache_api():
    model = _llama()
    ids = torch.randint(3, 100, (2, 5))
    c = model.allocate_kv_cache(2, 7)
    assert model.past_key_values is c and c.capacity == 7
    with torch.no_grad():
        model(ids, use_cache=True)
        assert model.past_length == 5 and c.length == 5
        for _ in range(4):                                          # grows past the capacity
            model(ids[:, :1], use_cache=True)
    assert model.past_length == 9 and c.capacity == 14
    model.set_cache(None)
    assert model.past_length == 0 and c.length == 0
    with pytest.raises(ValueError):
        with torch.no_grad():
            model(torch.randint(3, 100, (2, 65)), use_cache=True)   # past the rotary tables


def test_llama_beam_search_cached_equals_uncached():
    model = _llama()
    ids = torch.randint(3, 100, (2, 4))
    a = model.generate(ids, max_length=10, num_beams=3, eos_token_id=None, pad_token_id=0)
    b = model.generate(ids, max_length=10, num_beams=3, eos_token_id=None, pad_token_id=0, use_cache=False)
    assert torch.equal(a, b)


def test_magicprompt_gpt2_cache_equals_no_cache():
    from projects.MagicPrompt.gpt2 import GPTModel
    from libai_b200.utils import distributed as dutil

    dutil.reset_dist_util()
    torch.manual_seed(0)
    m = GPTModel(DictConfig(dict(
        hidden_layers=2, vocab_size=96, hidden_size=64, ffn_hidden_size=128, num_attention_heads=4, max_seq_length=64,
        embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0, layernorm_epsilon=1e-5,
        initializer_range=0.02, use_scaled_init_for_output_weights=True, bias_gelu_fusion=True,
        bias_dropout_fusion=True, scale_mask_softmax_fusion=True, apply_query_key_layer_scaling=True,
        apply_residual_post_layernorm=False, amp_enabled=False, eos_token_id=95, pad_token_id=0, bos_token_id=95,
    ))).eval()
    ids = torch.randint(1, 90, (2, 6))
    a = m.generate(ids, max_length=16, eos_token_id=None)
    b = m.generate(ids, max_length=16, eos_token_id=None, use_cache=False)
    assert torch.equal(a, b)
    c = m.generate(ids, max_length=12, eos_token_id=None, num_beams=2)
    d = m.generate(ids, max_length=12, eos_token_id=None, num_beams=2, use_cache=False)
    assert torch.equal(c, d)


def _llama_tp(rank, world):
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM
    from libai_b200.utils import distributed as dutil

    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=world, pipeline_parallel_size=1,
                                          device_type="cpu")))
    with param_defaults(dtype=torch.float32, device="cpu", seed=11):
        model = LlamaForCausalLM(DictConfig(LLAMA)).eval()
    torch.manual_seed(5)
    ids = torch.randint(3, 100, (2, 5))
    am = torch.ones_like(ids)
    ids[1, :2], am[1, :2] = 0, 0
    return model.generate(ids, attention_mask=am, max_length=12, eos_token_id=None, pad_token_id=0)


def test_llama_tensor_parallel_generation_equals_single_process():
    from tests.dist_utils import run_distributed

    single = _llama_tp(0, 1)
    res = run_distributed(_llama_tp, 2, timeout=300)
    for r in res:
        assert (r == single.numpy()).all(), (r, single)


# ------------------------------------------------------------------------------------------------ build
@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_decode_kernels_compile_without_spills_or_serialization(tmp_path):
    src = "decode_attention_sm90.cu"
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    log = res.stdout
    assert src in ops_build.CU_SOURCES
    assert ops_build.serialized_wgmma(log) == []
    # one "Function properties" block per kernel instantiation: decode (64, 128), combine (64, 128), append
    spills = re.findall(r"Function properties for (\S+)\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 5, log
    assert all(st == "0" and ld == "0" for _, st, ld in spills), spills
