"""GLM as a prefix LM without a GPU: the mask classifier (``prefix_lm``), the exactness of running a right-padded
context with its padding first, and cached generation on a ``StaticKVCache`` against the hidden-state memories and
full recomputation.  ``_native_attention`` is patched to True where the test needs the flash path's structure (the
classifier, the reordering, the prefix prefill and the decode steps); the attention underneath is then the reference
math of the same rule."""
import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference.kv_cache import StaticKVCache
from projects.GLM import modeling_glm
from projects.GLM.modeling_glm import GLMForConditionalGeneration, GLMModel, prefix_lm
from projects.GLM.tokenizer.glm_tokenizer import GLMTokenizerMixin

GEN = dict(is_encoder_decoder=False, min_length=0, do_sample=False, early_stopping=False, num_beams=1,
           num_beam_groups=1, diversity_penalty=0.0, temperature=1.0, top_k=50, top_p=1.0, typical_p=1.0,
           repetition_penalty=1.0, length_penalty=1.0, no_repeat_ngram_size=0, encoder_no_repeat_ngram_size=0,
           num_return_sequences=1, chunk_size_feed_forward=0, output_scores=False, forced_bos_token_id=None,
           forced_eos_token_id=None, remove_invalid_values=False, exponential_decay_length_penalty=None,
           use_cache=True, bos_token_id=None, sep_token_id=None, decoder_start_token_id=None)


def tiny_cfg(**kw):
    return DictConfig(dict(GEN, num_layers=2, vocab_size=128, hidden_size=64, num_attention_heads=4,
                           max_sequence_length=64, embedding_dropout_prob=0.0, attention_dropout_prob=0.0,
                           output_dropout_prob=0.0, layernorm_epsilon=1e-5, initializer_range=0.02,
                           use_scaled_init_for_output_weights=True, bias_gelu_fusion=True, bias_dropout_fusion=True,
                           scale_mask_softmax_fusion=False, apply_query_key_layer_scaling=False, amp_enabled=False,
                           block_position_encoding=True, attention_scale=1.0, padding_idx=None, eos_token_id=None,
                           pad_token_id=0, max_length=30, **kw))


class _Host:
    mask_token_id, pad_token_id = 7, 0

    def convert_tokens_to_ids(self, t):
        return {"<|startofpiece|>": 9, "<|endofpiece|>": 5, "[gMASK]": 8, "[sMASK]": 6}[t]

    def encode(self, t):
        return [20, 21, 22]


class Tok(GLMTokenizerMixin, _Host):
    pass


def prompts():
    """Two contexts of different lengths, right-padded as the tokenizer lays them out."""
    ids = torch.tensor([[11, 12, 13, 7, 14, 15, 16], [31, 7, 33, 0, 0, 0, 0], [41, 42, 7, 43, 44, 0, 0]])
    am = (ids != 0).long()
    return {"input_ids": ids, "attention_mask": am}


@pytest.fixture
def native(monkeypatch):
    monkeypatch.setattr(modeling_glm, "_native_attention", lambda x, d: True)


# ------------------------------------------------------------------------------------------------ the classifier
def test_classifier_separator():
    p = prefix_lm(torch.tensor(4), 3, 6)
    assert p.prefix_lens.tolist() == [4, 4, 4] and p.kv_start is None and p.order is None
    p = prefix_lm(torch.tensor([1, 5, 0]), 3, 6, mem_len=7)
    assert p.prefix_lens.dtype == torch.int32 and p.prefix_lens.tolist() == [8, 12, 7]


def gen_mask(am, gen):
    return Tok().build_inputs_for_generation({"input_ids": torch.where(am > 0, 7, 0), "attention_mask": am},
                                             max_gen_length=gen)["generation_attention_mask"]


def test_classifier_left_and_right_padding():
    # left padded: kv_start is the padding, the prefix the context width, no reordering
    am = torch.tensor([[0, 0, 1, 1, 1], [1, 1, 1, 1, 1]])
    m = gen_mask(am, 4)[:, :, :7, :7]
    p = prefix_lm(m, 2, 7)
    assert p.kv_start.tolist() == [2, 0] and p.prefix_lens.tolist() == [5, 5] and p.order is None
    # right padded: the padding moves in front of the context
    am = torch.tensor([[1, 1, 1, 0, 0], [1, 1, 1, 1, 1], [1, 0, 0, 0, 0]])
    m = gen_mask(am, 4)[:, :, :8, :8]
    p = prefix_lm(m, 3, 8)
    assert p.kv_start.tolist() == [2, 0, 4] and p.prefix_lens.tolist() == [5, 5, 5]
    assert p.order[0].tolist() == [3, 4, 0, 1, 2, 5, 6, 7] and p.order[2].tolist() == [1, 2, 3, 4, 0, 5, 6, 7]
    mo = m[:, 0].gather(1, p.order[:, :, None].expand(-1, 8, 8)).gather(2, p.order[:, None, :].expand(-1, 8, 8))
    from libai_b200.ops import functional as OF
    assert torch.equal(mo, OF.visible_keys(8, 8, causal=True, kv_start=p.kv_start, prefix_lens=p.prefix_lens)[:, 0])


def test_classifier_keeps_holes_and_arbitrary_masks_dense():
    am = torch.tensor([[1, 0, 1, 1, 1]])   # a hole inside the context
    assert prefix_lm(gen_mask(am, 3)[:, :, :6, :6], 1, 6) is None
    assert prefix_lm(torch.rand(2, 1, 6, 6) > 0.5, 2, 6) is None
    m = gen_mask(torch.ones(1, 4, dtype=torch.long), 3)[:, :, :5, :5].clone()
    m[0, 0, 4, 0] = 0   # one generated row misses one context key
    assert prefix_lm(m, 1, 5) is None
    assert prefix_lm(torch.ones(2, 1, 1, 6), 2, 1, mem_len=5) is None   # a decode row over memories


# ------------------------------------------------------------------------------------------------ reordering
def test_reordered_forward_matches_dense_reference_and_trains(monkeypatch):
    torch.manual_seed(0)
    m = GLMForConditionalGeneration(tiny_cfg()).eval()
    tok = Tok()
    tr = tok.build_inputs_for_generation(prompts(), targets=["x", "y", "z"], max_gen_length=4)
    assert prefix_lm(tr["attention_mask"], 3, tr["input_ids"].shape[1]).order is not None
    m.zero_grad()
    ref = m.glm(tr["input_ids"], tr["position_ids"], tr["attention_mask"])[0]
    ref.float().square().mean().backward()
    ref_grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    monkeypatch.setattr(modeling_glm, "_native_attention", lambda x, d: True)
    m.zero_grad()
    got = m.glm(tr["input_ids"], tr["position_ids"], tr["attention_mask"])[0]
    torch.testing.assert_close(got, ref, atol=1e-5, rtol=1e-5)
    got.float().square().mean().backward()
    for n, p in m.named_parameters():
        torch.testing.assert_close(p.grad, ref_grads[n], atol=1e-6, rtol=1e-4, msg=n)
    loss = m.train()(**tr)["lm_loss"]
    loss.backward()
    assert torch.isfinite(loss)


# ------------------------------------------------------------------------------------------------ cached generation
def recompute_greedy(m, inp, steps):
    ids, pos, mask = inp["input_ids"], inp["position_ids"], inp["generation_attention_mask"]
    for _ in range(steps):
        L = ids.shape[1]
        logits = m(ids, pos[:, :, :L], mask[:, :, :L, :L])["logits"]
        ids = torch.cat([ids, logits[:, -1].argmax(-1, keepdim=True)], 1)
    return ids


@pytest.mark.parametrize("patched", [False, True])
def test_cached_greedy_equals_memories_and_recompute(monkeypatch, patched):
    if patched:
        monkeypatch.setattr(modeling_glm, "_native_attention", lambda x, d: True)
    torch.manual_seed(1)
    m = GLMForConditionalGeneration(tiny_cfg()).eval()
    inp = Tok().build_inputs_for_generation(prompts(), max_gen_length=10)
    kw = dict(position_ids=inp["position_ids"], generation_attention_mask=inp["generation_attention_mask"],
              max_length=inp["input_ids"].shape[1] + 8, eos_token_id=None)
    with torch.no_grad():
        cached = m.generate(inp["input_ids"], use_cache=True, **kw)
        assert isinstance(m.past_key_values, StaticKVCache)
        memory = m.generate(inp["input_ids"], use_cache=False, **kw)
        full = recompute_greedy(m, inp, 8)
    assert torch.equal(cached, memory)
    assert torch.equal(cached, full)


@pytest.mark.parametrize("patched", [False, True])
def test_cached_beam_search_equals_memories(monkeypatch, patched):
    if patched:
        monkeypatch.setattr(modeling_glm, "_native_attention", lambda x, d: True)
    torch.manual_seed(2)
    m = GLMForConditionalGeneration(tiny_cfg()).eval()
    inp = Tok().build_inputs_for_generation(prompts(), max_gen_length=10)
    beams = 3
    kw = dict(position_ids=inp["position_ids"].repeat_interleave(beams, 0),
              generation_attention_mask=inp["generation_attention_mask"].repeat_interleave(beams, 0),
              max_length=inp["input_ids"].shape[1] + 6, eos_token_id=None, num_beams=beams)
    with torch.no_grad():
        cached = m.generate(inp["input_ids"], use_cache=True, **kw)
        memory = m.generate(inp["input_ids"], use_cache=False, **kw)
    assert torch.equal(cached, memory)


def test_cached_sampling_and_fp8_cache_run(native):
    torch.manual_seed(3)
    m = GLMForConditionalGeneration(tiny_cfg()).eval()
    inp = Tok().build_inputs_for_generation(prompts(), max_gen_length=10)
    kw = dict(position_ids=inp["position_ids"], generation_attention_mask=inp["generation_attention_mask"],
              max_length=inp["input_ids"].shape[1] + 5, eos_token_id=None)
    with torch.no_grad():
        out = m.generate(inp["input_ids"], use_cache=True, do_sample=True, top_k=5, **kw)
        assert out.shape == (3, inp["input_ids"].shape[1] + 5)
        out = m.generate(inp["input_ids"], use_cache=True, kv_cache_dtype="fp8", **kw)
        assert out.shape == (3, inp["input_ids"].shape[1] + 5)
        assert m.past_key_values.kv_dtype == torch.float8_e4m3fn


def test_attend_rejects_prefix_on_a_warm_cache():
    c = StaticKVCache(1, 2, 2, 8, 16, dtype=torch.float32)
    layer = c.layer(0)
    qkv = torch.randn(2, 3, 2, 24)
    q = layer.append(qkv)
    out = layer.attend(q, scale=0.3, prefix_lens=torch.tensor([2, 3], dtype=torch.int32))
    assert out.shape == (2, 3, 2, 8)
    c.advance(3)
    with pytest.raises(ValueError):
        layer.attend(layer.append(qkv[:, :1]), scale=0.3, prefix_lens=torch.tensor([2, 3], dtype=torch.int32))


def test_memory_path_with_separator_matches_dense(native):
    """``memory_states`` with a ``sep`` go through the prefix rule: same logits as the dense mask."""
    torch.manual_seed(4)
    m = GLMModel(tiny_cfg()).eval()
    ids = torch.randint(10, 100, (2, 6))
    with torch.no_grad():
        _, mems = m(ids[:, :4], attention_mask=torch.tensor(3))
        got = m(ids[:, 4:], attention_mask=torch.tensor([1, 2]), memory_states=mems)[0]
        mask = GLMModel.build_mask_matrix(2, 2, torch.tensor([1, 2]), 4)
        want = m(ids[:, 4:], attention_mask=mask, memory_states=mems)[0]
    torch.testing.assert_close(got, want, atol=1e-5, rtol=1e-5)
