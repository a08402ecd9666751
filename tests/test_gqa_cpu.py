"""Grouped-query attention on the CPU: HuggingFace parity of GQA / MQA Llama and Qwen2 checkpoints, the grouped reference
ops against their MHA versions on expanded K/V, the model's grouped projection and cache, tensor parallelism over whole
key/value groups; with nvcc, the build of the grouped attention and decode kernels."""
import os
import re
import subprocess

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dutil

LLAMA = dict(hidden_layers=2, vocab_size=100, hidden_size=64, intermediate_size=128, num_attention_heads=4,
             max_position_embeddings=64, rms_norm_eps=1e-5, initializer_range=0.02,
             use_scaled_init_for_output_weights=True, scale_mask_softmax_fusion=False, amp_enabled=False,
             bos_token_id=1, eos_token_id=2, pad_token_id=0, max_length=20)


def _llama(seed=0, **kw):
    from libai_b200.models import LlamaForCausalLM

    dutil.reset_dist_util()
    torch.manual_seed(seed)
    return LlamaForCausalLM(DictConfig(dict(LLAMA, **kw))).eval()


def _expand(x, r, dim):
    return x.repeat_interleave(r, dim=dim)


def _grouped_to_mha(qkv):
    """A grouped projection [b, s, g, r + 2, d] → the MHA projection [b, s, a, 3d] with every K/V head repeated."""
    b, s, g, r2, d = qkv.shape
    r = r2 - 2
    q = qkv[..., :r, :].reshape(b, s, g * r, d)
    k, v = _expand(qkv[..., r, :], r, 2), _expand(qkv[..., r + 1, :], r, 2)
    return torch.cat([q, k, v], dim=-1)


# ------------------------------------------------------------------------------------------------ HuggingFace parity
transformers = pytest.importorskip("transformers")
BASE = dict(hidden_layers=1, vocab_size=1, hidden_size=8, intermediate_size=8, num_attention_heads=1,
            max_position_embeddings=8, rms_norm_eps=1e-6, initializer_range=0.02,
            use_scaled_init_for_output_weights=False, scale_mask_softmax_fusion=False, amp_enabled=False)


def _hf_greedy(hf, ids, n):
    with torch.no_grad():
        for _ in range(n):
            ids = torch.cat([ids, hf(ids).logits[:, -1].argmax(-1, keepdim=True)], 1)
    return ids


def _check_hf_parity(hf, ours_cls, loader_cls, tmp_path, name, **cfg):
    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                          device_type="cpu")))
    d = str(tmp_path / name)
    hf.save_pretrained(d)
    m = loader_cls(ours_cls, DictConfig(dict(BASE, **cfg)), d).load().eval()
    attn = m.model.layers[0].self_attn
    assert attn.num_kv_heads == hf.config.num_key_value_heads and attn.num_heads == hf.config.num_attention_heads
    torch.manual_seed(1)
    ids = torch.randint(3, hf.config.vocab_size, (2, 9))
    with torch.no_grad():
        assert (m(ids)["logits"] - hf(ids).logits).abs().max() < 1e-4
    ours = m.generate(ids, max_length=17, eos_token_id=None, pad_token_id=0)
    assert torch.equal(ours, _hf_greedy(hf, ids, 8))
    assert m.kv_cache is not None and m.kv_cache.heads == hf.config.num_key_value_heads


@pytest.mark.parametrize("kv_heads", [2, 1])
def test_llama_gqa_checkpoint_matches_hf(tmp_path, kv_heads):
    from libai_b200.models import LlamaForCausalLM
    from libai_b200.models.utils.model_loader.llama_loader import LlamaLoaderHuggerFace

    torch.manual_seed(0)
    hf = transformers.LlamaForCausalLM(transformers.LlamaConfig(
        vocab_size=96, hidden_size=64, intermediate_size=176, num_hidden_layers=2, num_attention_heads=4,
        num_key_value_heads=kv_heads, max_position_embeddings=64, rms_norm_eps=1e-6)).eval()
    _check_hf_parity(hf, LlamaForCausalLM, LlamaLoaderHuggerFace, tmp_path, f"llama_kv{kv_heads}")


def test_qwen2_gqa_checkpoint_with_biases_matches_hf(tmp_path):
    from projects.Qwen.qwen2 import Qwen2ForCausalLM
    from projects.Qwen.utils.qwen2_loader import Qwen2LoaderHuggerFace

    torch.manual_seed(0)
    hf = transformers.Qwen2ForCausalLM(transformers.Qwen2Config(
        vocab_size=96, hidden_size=64, intermediate_size=176, num_hidden_layers=2, num_attention_heads=4,
        num_key_value_heads=2, max_position_embeddings=64, rms_norm_eps=1e-6, tie_word_embeddings=False)).eval()
    with torch.no_grad():   # non-zero q/k/v biases, so their grouping is checked too
        for layer in hf.model.layers:
            for proj in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj):
                proj.bias.normal_(0, 0.5)
    _check_hf_parity(hf, Qwen2ForCausalLM, Qwen2LoaderHuggerFace, tmp_path, "qwen2_kv2", qkv_bias=True)


# ------------------------------------------------------------------------------------------------ reference ops
@pytest.mark.parametrize("r", [1, 2, 4])
@pytest.mark.parametrize("causal", [True, False])
def test_grouped_attention_ref_equals_mha_on_expanded_kv(r, causal):
    torch.manual_seed(0)
    b, g, s, d = 2, 2, 7, 8
    q = torch.randn(b, g * r, s, d)
    k, v = torch.randn(b, g, s, d), torch.randn(b, g, s, d)
    mask = torch.rand(b, 1, s, s) > 0.3
    for m in (None, mask):
        got = OF.attention(q, k, v, causal=causal, scale=0.3, mask=m)
        want = OF.attention_ref(q, _expand(k, r, 1), _expand(v, r, 1), causal=causal, scale=0.3, mask=m)
        assert torch.equal(got, want)


def test_attention_rejects_heads_that_do_not_group():
    with pytest.raises(ValueError):
        OF.attention(torch.randn(1, 6, 4, 8), torch.randn(1, 4, 4, 8), torch.randn(1, 4, 4, 8), causal=True)


@pytest.mark.parametrize("r", [1, 3])
def test_grouped_rotary_and_cache_append_equal_mha_on_expanded_inputs(r):
    from libai_b200.models.llama_model import rotary_tables

    torch.manual_seed(0)
    b, s, g, d, cap = 2, 3, 2, 8, 16
    cos, sin = rotary_tables(d, 32)
    qkv = torch.randn(b, s, g, r + 2, d)
    mha = _grouped_to_mha(qkv)
    rot = OF.apply_rotary_qkv(qkv, cos, sin, 5)
    assert torch.equal(_grouped_to_mha(rot), OF.apply_rotary_qkv(mha, cos, sin, 5))

    c = StaticKVCache(1, b, g, d, cap, torch.float32, "cpu")
    cm = StaticKVCache(1, b, g * r, d, cap, torch.float32, "cpu")
    for cache in (c, cm):
        cache.seqlens.copy_(torch.tensor([4, 6], dtype=torch.int32))
    q = OF.kv_cache_append(qkv, c.k[0], c.v[0], c.seqlens, cos, sin)
    qm = OF.kv_cache_append(mha, cm.k[0], cm.v[0], cm.seqlens, cos, sin)
    assert q.shape == (b, s, g * r, d) and torch.equal(q, qm)
    for bi, st in enumerate((4, 6)):
        assert torch.equal(_expand(c.k[0][bi, :, st : st + s], r, 0), cm.k[0][bi, :, st : st + s])
        assert torch.equal(_expand(c.v[0][bi, :, st : st + s], r, 0), cm.v[0][bi, :, st : st + s])


@pytest.mark.parametrize("r", [2, 4])
@pytest.mark.parametrize("sq", [1, 3])
def test_grouped_decode_attention_ref_equals_mha_on_expanded_cache(r, sq):
    torch.manual_seed(0)
    b, g, d, cap = 2, 2, 8, 32
    k, v = torch.randn(b, g, cap, d), torch.randn(b, g, cap, d)
    q = torch.randn(b, sq, g * r, d)
    lens = torch.tensor([9, 13], dtype=torch.int32)
    start = torch.tensor([0, 4], dtype=torch.int32)
    got = OF.decode_attention(q, k, v, lens, start, scale=0.3)
    want = OF.decode_attention_ref(q, _expand(k, r, 1), _expand(v, r, 1), lens, start, scale=0.3)
    assert torch.equal(got, want)


def test_r1_grouped_view_is_the_mha_layout():
    qkv = torch.randn(2, 5, 3, 3 * 8)
    grouped = qkv.view(2, 5, 3, 3, 8)
    assert grouped.data_ptr() == qkv.data_ptr()
    q4, k4, v4 = OF._packed_views(qkv)
    q5, k5, v5 = OF._packed_views(grouped)
    assert torch.equal(q5.reshape(q4.shape), q4) and q5.data_ptr() == q4.data_ptr()
    assert k5.stride() == k4.stride() and k5.data_ptr() == k4.data_ptr()
    assert v5.stride() == v4.stride() and v5.data_ptr() == v4.data_ptr()
    assert (q5.stride(0), q5.stride(1), q5.stride(3)) == (q4.stride(0), q4.stride(1), q4.stride(2))


def test_hf_qkv_fusion_groups_rows_per_kv_head():
    from libai_b200.models.utils.model_loader.base_loader import ModelLoaderHuggerFace

    a, g, d, h = 4, 2, 3, 5
    q, k, v = torch.randn(a * d, h), torch.randn(g * d, h), torch.randn(g * d, h)
    fused = ModelLoaderHuggerFace._fix_qkv_ordering(torch.cat([q, k, v]), d, a, num_kv_heads=g).view(g, a // g + 2, d, h)
    assert torch.equal(fused[:, :2].reshape(a * d, h), q)
    assert torch.equal(fused[:, 2].reshape(g * d, h), k) and torch.equal(fused[:, 3].reshape(g * d, h), v)
    mha = torch.randn(3 * a * d, h)
    assert torch.equal(ModelLoaderHuggerFace._fix_qkv_ordering(mha, d, a, num_kv_heads=a),
                       ModelLoaderHuggerFace._fix_qkv_ordering(mha, d, a))


# ------------------------------------------------------------------------------------------------ model
def test_equal_kv_heads_builds_the_mha_model():
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    dutil.reset_dist_util()
    a, b = [None, None]
    for i, kw in enumerate(({}, {"num_key_value_heads": 4})):
        with param_defaults(dtype=torch.float32, device="cpu", seed=11):
            m = LlamaForCausalLM(DictConfig(dict(LLAMA, **kw))).eval()
        a, b = (m, b) if i == 0 else (a, m)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(sa[n].shape == sb[n].shape for n in sa)
    assert all(torch.equal(sa[n], sb[n]) for n in sa)
    ids = torch.randint(3, 100, (2, 7))
    with torch.no_grad():
        assert torch.equal(a(ids)["logits"], b(ids)["logits"])


def test_gqa_model_shapes_and_cache():
    m = _llama(num_key_value_heads=2)
    attn = m.model.layers[0].self_attn
    assert attn.query_key_value.weight.shape == ((4 + 2 * 2) * 16, 64)
    assert attn.local_kv_heads == 2 and attn.local_heads == 4
    c = m.allocate_kv_cache(3, 10)
    assert c.heads == 2 and c.k[0].shape == (3, 2, 10, 16)


@pytest.mark.parametrize("kv_heads", [2, 1])
def test_gqa_beam_search_cached_equals_uncached(kv_heads):
    model = _llama(num_key_value_heads=kv_heads)
    ids = torch.randint(3, 100, (2, 4))
    a = model.generate(ids, max_length=10, num_beams=3, eos_token_id=None, pad_token_id=0)
    b = model.generate(ids, max_length=10, num_beams=3, eos_token_id=None, pad_token_id=0, use_cache=False)
    assert torch.equal(a, b)


def test_gqa_left_padded_greedy_equals_bruteforce():
    model = _llama(num_key_value_heads=2)
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
    done = (out == LLAMA["eos_token_id"]).cumsum(1) > 0
    done[:, :6] = False
    assert torch.equal(cur[~done], out[~done])


def test_gqa_legacy_tuple_cache_equals_full_forward():
    model = _llama(num_key_value_heads=2)
    ids = torch.randint(3, 100, (2, 9))
    with torch.no_grad():
        want = model(ids)["logits"][:, 5:]
        keep = lambda p: setattr(model, "_tuple_cache", p)
        model.model(ids[:, :5], use_cache=True, set_cache=keep)
        assert model._tuple_cache[0][0].shape == (2, 2, 5, 16)     # [b, g, s, d]
        got = []
        for i in range(5, 9):                                       # one new token per step
            h = model.model(ids[:, i : i + 1], past_key_values=model._tuple_cache, use_cache=True, set_cache=keep)
            got.append(model.lm_head(h))
        got = torch.cat(got, 1)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def test_adapter_refuses_grouped_query_attention():
    from projects.Llama.adapter.adapter_model import LlamaForCausalLM

    dutil.reset_dist_util()
    with pytest.raises(ValueError, match="num_key_value_heads"):
        LlamaForCausalLM(DictConfig(dict(LLAMA, num_key_value_heads=2, adapter_len=2, adapter_layer=1)))


# ------------------------------------------------------------------------------------------------ tensor parallel
def _gqa_tp(rank, world):
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=world, pipeline_parallel_size=1,
                                          device_type="cpu")))
    with param_defaults(dtype=torch.float32, device="cpu", seed=11):
        model = LlamaForCausalLM(DictConfig(dict(LLAMA, num_key_value_heads=2))).eval()
    torch.manual_seed(5)
    ids = torch.randint(3, 100, (2, 5))
    am = torch.ones_like(ids)
    ids[1, :2], am[1, :2] = 0, 0
    return model.generate(ids, attention_mask=am, max_length=12, eos_token_id=None, pad_token_id=0)


def test_gqa_tensor_parallel_generation_equals_single_process():
    from tests.dist_utils import run_distributed

    single = _gqa_tp(0, 1)
    res = run_distributed(_gqa_tp, 2, timeout=300)
    for r in res:
        assert (r == single.numpy()).all(), (r, single)


def _mqa_tp_error(rank, world):
    from libai_b200.models import LlamaForCausalLM

    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=world, pipeline_parallel_size=1,
                                          device_type="cpu")))
    try:
        LlamaForCausalLM(DictConfig(dict(LLAMA, num_key_value_heads=1)))
    except ValueError as e:
        return torch.tensor([int("tensor-parallel" in str(e))])
    return torch.tensor([0])


def test_kv_heads_not_divisible_by_tensor_parallel_size_raises():
    from tests.dist_utils import run_distributed

    res = run_distributed(_mqa_tp_error, 2, timeout=300)
    assert all(int(r[0]) == 1 for r in res), res


# ------------------------------------------------------------------------------------------------ build
@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
@pytest.mark.parametrize("src", ["attention_sm90.cu", "decode_attention_sm90.cu"])
def test_grouped_kernels_compile_for_sm90a(tmp_path, src):
    """The grouped kernels are the existing instantiations with a runtime group size: the sources compile for sm_90a,
    wgmma stays asynchronous, and the forward, decode and append kernels do not spill."""
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    log = res.stdout
    assert ops_build.serialized_wgmma(log) == []
    spills = dict((name, (st, ld)) for name, st, ld in re.findall(
        r"Function properties for (\S+)\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log))
    checked = {n: v for n, v in spills.items() if "attn_fwd_kernel" in n or "dec" in n}
    assert checked, log
    assert all(v == ("0", "0") for v in checked.values()), checked
