"""Which kernels cached generation runs, without a GPU: the decode and flash ops of the extension are replaced by a
stub that computes the reference math and records every call, and ``generate()`` / teacher-forced forwards of every
model that decodes on the preallocated cache are compared with a literal trace of those calls."""
import sys

import pytest
import torch

from libai_b200.config import DictConfig, LazyConfig, instantiate
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


def _token(op, causal=False, kv_start=False, bias=False, alibi=False, rel_bias=False):
    """One call: ``a`` (kv_append), ``F`` (flash attention) or ``D`` (decode attention), then a letter per argument:
    ``c`` causal, ``S`` kv_start, ``b`` dense bias, ``A`` ALiBi slopes, ``r`` relative-bias vector."""
    flags = zip("cSbAr", (causal, kv_start, bias, alibi, rel_bias))
    return op + "".join(f for f, on in flags if on)


class _StubExt:
    """The extension's cache, decode and flash ops, computed with the reference math; records every call."""

    def __init__(self):
        self.calls = []

    def kv_append(self, qkv, k_cache, v_cache, seqlens, cos, sin, write_q):
        self.calls.append("a")
        return OF.kv_cache_append_ref(qkv, k_cache, v_cache, seqlens, cos, sin)

    def decode_attn(self, q, k_cache, v_cache, seqlens, kv_start, scale, splits, alibi_slopes=None, rel_bias=None,
                    causal=True):
        self.calls.append(_token("D", causal, kv_start is not None, False, alibi_slopes is not None,
                                 rel_bias is not None))
        return OF.decode_attention_ref(q, k_cache, v_cache, seqlens, kv_start, scale=scale, alibi_slopes=alibi_slopes,
                                       rel_bias=rel_bias, causal=causal)

    def attn_fwd(self, q, k, v, causal, scale, kv_lens, bias, alibi_slopes, p_drop, salt, kv_start=None,
                 doc_start=None):
        self.calls.append(_token("F", causal, kv_start is not None, bias is not None, alibi_slopes is not None))
        sq, sk = q.shape[-2], k.shape[-2]
        vis = OF.visible_keys(sq, sk, causal=causal, kv_start=kv_start, kv_lens=kv_lens)
        total = None if bias is None else bias.float()
        if alibi_slopes is not None:
            rel = (torch.arange(sk)[None, :] - torch.arange(sk - sq, sk)[:, None]).float()
            ab = alibi_slopes[None, :, None, None] * rel
            total = ab if total is None else total + ab
        o = OF.attention_ref(q, k, v, causal=False, scale=scale, mask=vis, bias=total)
        return o.masked_fill(~vis.any(-1, keepdim=True), 0), torch.empty(0), torch.empty(0)


@pytest.fixture
def native_attention(monkeypatch):
    """As if on the GPU for the attention ops only (the GEMMs, norms and rotary keep the PyTorch path)."""
    from projects.BLOOM.modeling import bloom_model
    from projects.ChatGLM import chatglm

    ext = _StubExt()
    attention_checks = {"_decode_native", "attention_supported", "attention_qkvpacked_supported"}
    monkeypatch.setattr(OF, "use_native", lambda *t: sys._getframe(1).f_code.co_name in attention_checks)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: ext)
    for mod in (bloom_model, chatglm):   # their uncached forwards ask for the flash kernels themselves
        monkeypatch.setattr(mod, "use_native", lambda *t: True)
    return ext


# ------------------------------------------------------------------------------------------------ models (bf16, head dim 64)
LLAMA = dict(hidden_layers=2, vocab_size=100, hidden_size=128, intermediate_size=128, num_attention_heads=2,
             max_position_embeddings=64, rms_norm_eps=1e-5, initializer_range=0.02,
             use_scaled_init_for_output_weights=True, scale_mask_softmax_fusion=False, amp_enabled=False,
             bos_token_id=1, eos_token_id=2, pad_token_id=0, max_length=20)


def _llama(gqa):
    from libai_b200.models import LlamaForCausalLM

    kw = dict(hidden_size=256, num_attention_heads=4, num_key_value_heads=2) if gqa else {}
    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return LlamaForCausalLM(DictConfig(dict(LLAMA, **kw))).eval()


def _gpt2():
    from projects.MagicPrompt.gpt2 import GPTModel

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return GPTModel(DictConfig(dict(
            hidden_layers=2, vocab_size=100, hidden_size=128, ffn_hidden_size=128, num_attention_heads=2,
            max_seq_length=64, embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
            layernorm_epsilon=1e-5, initializer_range=0.02, use_scaled_init_for_output_weights=True,
            bias_gelu_fusion=True, bias_dropout_fusion=True, scale_mask_softmax_fusion=True,
            apply_query_key_layer_scaling=True, apply_residual_post_layernorm=False, amp_enabled=False,
            eos_token_id=2, pad_token_id=0, bos_token_id=1))).eval()


def _bloom():
    from projects.BLOOM.modeling.bloom_model import BloomForCausalLM

    cfg = LazyConfig.load("projects/BLOOM/configs/bloom_inference.py").cfg
    cfg.update(dict(vocab_size=100, hidden_size=128, hidden_layers=2, n_head=2))
    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return BloomForCausalLM(cfg).eval()


def _chatglm(prefix):
    c = LazyConfig.load("projects/ChatGLM/configs/chatglm_config.py")
    over = ["cfg.num_layers=2", "cfg.hidden_size=128", "cfg.ffn_hidden_size=128", "cfg.num_attention_heads=4",
            "cfg.kv_channels=64", "cfg.multi_query_group_num=2", "cfg.padded_vocab_size=100", "cfg.seq_length=64",
            "cfg.max_length=20", "cfg.pad_token_id=0"]
    if prefix:
        over += ["cfg.pre_seq_len=3", "cfg.prefix_projection=False"]
    c = LazyConfig.apply_overrides(c, over)
    c.model.cfg = c.cfg
    torch.manual_seed(0)
    return instantiate(c.model).to(torch.bfloat16).eval()


def _t5():
    from projects.MT5.mt5_model import MT5Model

    cfg = DictConfig(dict(
        is_encoder_decoder=True, max_length=12, min_length=0, do_sample=False, early_stopping=False, num_beams=1,
        num_beam_groups=1, diversity_penalty=0.0, temperature=1.0, top_k=50, top_p=1.0, typical_p=1.0,
        repetition_penalty=1.0, length_penalty=1.0, no_repeat_ngram_size=0, encoder_no_repeat_ngram_size=0,
        num_return_sequences=1, chunk_size_feed_forward=0, output_scores=False, use_cache=True, eos_token_id=1,
        pad_token_id=0, decoder_start_token_id=0, vocab_size=100, hidden_size=256, hidden_layers=2,
        num_attention_heads=4, head_size=64, intermediate_size=128, embedding_dropout_prob=0.0,
        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, relative_attention_num_buckets=8,
        initializer_range=0.5, layernorm_eps=1e-6, amp_enabled=False, model_type="mt5", padding_idx=0,
        tie_word_embeddings=False))
    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return MT5Model(cfg).eval()


MODELS = {"llama": lambda: _llama(False), "llama_gqa": lambda: _llama(True), "gpt2": _gpt2, "bloom": _bloom,
          "chatglm": lambda: _chatglm(False), "chatglm_prefix": lambda: _chatglm(True), "t5": _t5}


def _prompt(case, s=7):
    """Token ids ``[3, s]`` and their padding mask (None for an unpadded prompt)."""
    ids = torch.randint(3, 100, (3, s), generator=torch.Generator().manual_seed(1))
    if case not in ("left_padded", "hole"):
        return ids, None
    am = torch.ones_like(ids)
    if case == "left_padded":
        am[1, :2] = am[2, :4] = 0
    else:
        am[1, 3] = 0
    return ids.masked_fill(am == 0, 0), am


def _run(name, case):
    m = MODELS[name]()
    ids, am = _prompt(case)
    with torch.no_grad():
        if name == "t5":
            if case == "teacher_forced":   # one step, then 19 tokens at once (more than the decode kernel's 16)
                dec = torch.randint(2, 100, (3, 20), generator=torch.Generator().manual_seed(3))
                m.allocate_kv_cache(3, 20)
                m(ids, dec[:, :1], am, use_cache=True)
                m(ids, dec[:, 1:], am, use_cache=True)
            else:
                m.generate(ids, encoder_attn_mask=am, max_length=5, eos_token_id=None,
                           num_beams=2 if case == "beams" else 1)
        elif case == "teacher_forced":     # a 7-token prompt, then 18 tokens at once
            more = torch.randint(3, 100, (3, 18), generator=torch.Generator().manual_seed(3))
            m.allocate_kv_cache(3, 25)
            m(ids, use_cache=True)
            m(more, use_cache=True)
        else:
            kw = {} if am is None else {"attention_mask": am}
            m.generate(ids, max_length=ids.shape[1] + 4, eos_token_id=None, num_beams=2 if case == "beams" else 1,
                       **kw)


def _expand(trace):
    """``"tok*n"`` stands for ``n`` copies of ``tok``."""
    out = []
    for t in trace.split():
        tok, _, n = t.partition("*")
        out += [tok] * int(n or 1)
    return out


# Two layers per model.  A padded prompt takes kv_start, a mask with a hole the dense mask on the reference math (no
# attention call); the decode kernel runs every later step, and the flash kernel over the cache window a continuation
# of more than 16 tokens.
TRACES = {
    ("llama", "plain"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("llama", "left_padded"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("llama", "hole"): "a*8",
    ("llama", "teacher_forced"): "a FcS a FcS a FcS a FcS",
    ("llama", "beams"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("llama_gqa", "plain"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("llama_gqa", "left_padded"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("llama_gqa", "hole"): "a*8",
    ("llama_gqa", "teacher_forced"): "a FcS a FcS a FcS a FcS",
    ("llama_gqa", "beams"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    # GPT-2's prefill passes the cache's kv_start like every other causal prefill; it is all zeros (GPT-2 prompts are
    # never padded), so the visible keys are those of the plain causal call it made before
    ("gpt2", "plain"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("gpt2", "teacher_forced"): "a FcS a FcS a FcS a FcS",
    ("gpt2", "beams"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("bloom", "plain"): "a FcSA a FcSA a DcSA a DcSA a DcSA a DcSA a DcSA a DcSA",
    ("bloom", "left_padded"): "a FcSA a FcSA a DcSA a DcSA a DcSA a DcSA a DcSA a DcSA",
    ("bloom", "hole"): "a*8",
    ("bloom", "teacher_forced"): "a FcSA a FcSA a FcSA a FcSA",
    ("bloom", "beams"): "a FcSA a FcSA a DcSA a DcSA a DcSA a DcSA a DcSA a DcSA",
    ("chatglm", "plain"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("chatglm", "left_padded"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("chatglm", "hole"): "a*8",
    ("chatglm", "teacher_forced"): "a FcS a FcS a FcS a FcS",
    ("chatglm", "beams"): "a FcS a FcS a DcS a DcS a DcS a DcS a DcS a DcS",
    # the prefix rows are in the cache before the prompt: the prompt is a decoding step
    ("chatglm_prefix", "plain"): "a DcS a DcS a DcS a DcS a DcS a DcS a DcS a DcS",
    ("chatglm_prefix", "teacher_forced"): "a DcS a DcS a FcS a FcS",
    ("chatglm_prefix", "beams"): "a DcS a DcS a DcS a DcS a DcS a DcS a DcS a DcS",
    # the encoder (dense bias), then per layer and step self-attention with the relative-bias vector and
    # cross-attention over the encoder window, or the folded dense bias when the encoder mask has a hole
    ("t5", "plain"): "Fb*2 a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS",
    ("t5", "left_padded"): "Fb*2 a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS",
    ("t5", "hole"): "Fb*2 a DcSr Fb a DcSr Fb a DcSr Fb a DcSr Fb a DcSr Fb a DcSr Fb a DcSr Fb a DcSr Fb",
    ("t5", "teacher_forced"): "Fb*2 a DcSr DS a DcSr DS a FcSb FS a FcSb FS",
    ("t5", "beams"): "Fb*2 a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS a DcSr DS",
}

# GPT-2 takes no mask; ChatGLM's prompt mask does not cover the P-tuning prefix rows
CASES = [(name, case) for name in MODELS for case in ("plain", "left_padded", "hole", "teacher_forced", "beams")
         if not (name in ("gpt2", "chatglm_prefix") and case in ("left_padded", "hole"))]


@pytest.mark.parametrize("name,case", CASES)
def test_kernel_calls_of_cached_generation(native_attention, name, case):
    _run(name, case)
    assert native_attention.calls == _expand(TRACES[name, case])


# ------------------------------------------------------------------------------------------------ padding policy
def _mask(kind, b=3, n=6):
    am = torch.ones(b, n, dtype=torch.long)
    if kind == "left":
        am[1, :2] = am[2, :5] = 0
    elif kind == "right":
        am[1, 4:] = 0
    elif kind == "hole":
        am[0, 2] = 0
    return None if kind == "none" else am


@pytest.mark.parametrize("flash", [False, True])
@pytest.mark.parametrize("kv_start_ok", [False, True])
@pytest.mark.parametrize("kind", ["none", "ones", "left", "right", "hole"])
def test_step_needs_dense_mask(kind, kv_start_ok, flash):
    from libai_b200.inference.kv_cache import StaticKVCache

    c = StaticKVCache(1, 3, 1, 8, 16, torch.float32, "cpu")
    am = _mask(kind)
    in_kv_start = kind == "left" and kv_start_ok
    padded = kind in ("left", "right", "hole")
    assert c.step_needs_dense_mask(am, flash=flash, kv_start_ok=kv_start_ok) == (padded and not (in_kv_start and flash))
    assert c.dense_mask == (padded and not in_kv_start)
    assert c.kv_start.tolist() == ([0, 2, 5] if in_kv_start else [0, 0, 0])
    c.advance(6)
    for step in (None, torch.cat((am if am is not None else torch.ones(3, 6, dtype=torch.long),
                                  torch.ones(3, 1, dtype=torch.long)), dim=1)):
        assert c.step_needs_dense_mask(step, flash=flash, kv_start_ok=kv_start_ok) == (step is not None
                                                                                      and c.dense_mask)


def _old_bounds(am):
    """The classification ``padding_bounds`` replaces: a right-padded prefix first, then left padding."""
    from libai_b200.inference.kv_cache import left_padding
    from libai_b200.layers.attention import KeyPaddingMask

    keys = KeyPaddingMask(am)
    if keys.is_prefix():
        return keys.lengths, None
    kv_start = left_padding(am)
    return None if kv_start is None else (None, kv_start)


def _random_row(kind, n, g):
    row = torch.ones(n, dtype=torch.long)
    p, q = sorted(torch.randint(0, n + 1, (2,), generator=g).tolist())
    if kind == "left":
        row[:p] = 0
    elif kind == "right":
        row[q:] = 0
    elif kind == "both":
        row[:p], row[q:] = 0, 0
    elif kind == "hole":
        row[int(torch.randint(0, n, (1,), generator=g))] = 0
    elif kind == "zeros":
        row[:] = 0
    return row


@pytest.mark.parametrize("b,n", [(1, 1), (3, 1), (2, 5), (4, 9)])
def test_padding_bounds_routes_as_prefix_then_left_padding(b, n):
    from libai_b200.inference.kv_cache import padding_bounds

    g = torch.Generator().manual_seed(b * 100 + n)
    kinds = ["ones", "left", "right", "both", "hole", "zeros"]
    seen = set()
    for _ in range(100):
        am = torch.stack([_random_row(kinds[int(torch.randint(0, len(kinds), (1,), generator=g))], n, g)
                          for _ in range(b)])
        got, want = padding_bounds(am), _old_bounds(am)
        seen.add(None if want is None else tuple(t is None for t in want))
        assert (got is None) == (want is None), am
        if want is not None:
            for x, y in zip(got, want):
                assert (x is None) == (y is None) and (x is None or (x.dtype == torch.int32 and torch.equal(x, y))), am
    assert len(seen) == (1 if n == 1 else 3)   # every route is taken (with one key every row is a prefix)
