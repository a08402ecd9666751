"""KV-cache decoding on the H100: the split-KV decode attention kernel against the fp32 reference, its determinism and
CUDA-graph replay, the fused rotary cache append against rope_qkv, and cached generate() through the native kernels."""
import pytest
import torch

from libai_b200 import ops
from libai_b200.config import DictConfig
from libai_b200.ops import functional as OF

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def _case(B, A, D, sq, L, cap_extra=37, seed=0):
    """Packed projection qkv [B, sq, A, 3D] (q is a strided view of it), caches of capacity > length, per-sample
    lengths around L and non-zero left padding."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    C = L + sq + cap_extra
    k = torch.randn(B, A, C, D, device=DEV, generator=g).bfloat16()
    v = torch.randn(B, A, C, D, device=DEV, generator=g).bfloat16()
    qkv = torch.randn(B, sq, A, 3 * D, device=DEV, generator=g).bfloat16()
    lens = torch.tensor([max(L - 5 * b, 1) for b in range(B)], dtype=torch.int32, device=DEV)
    start = torch.tensor([(7 * b) % max(int(lens[b]), 1) if b % 2 else 0 for b in range(B)], dtype=torch.int32,
                         device=DEV)
    return qkv[..., :D], k, v, lens, start


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("sq", [1, 4, 16])
def test_decode_attention_matches_fp32_reference(D, sq):
    errs = {}
    for B in (1, 3, 8):
        for L in (1, 63, 64, 65, 1000, 4097):
            q, k, v, lens, start = _case(B, 4, D, sq, L, seed=B * 10000 + L)
            scale = D ** -0.5
            got = OF.decode_attention(q, k, v, lens, start, scale=scale)
            want = OF.decode_attention_ref(q, k, v, lens, start, scale=scale)
            assert got.shape == (B, sq, 4, D) and got.is_contiguous()
            errs[(B, L)] = rel_err(got, want)
    bad = {key: e for key, e in errs.items() if not e < 3e-2}
    assert not bad, bad


@pytest.mark.parametrize("splits", [1, 3, 32])
def test_decode_attention_any_split_count(splits):
    q, k, v, lens, start = _case(2, 4, 128, 4, 2000)
    got = OF.decode_attention(q, k, v, lens, start, scale=0.1, splits=splits)
    want = OF.decode_attention_ref(q, k, v, lens, start, scale=0.1)
    assert rel_err(got, want) < 3e-2


def test_decode_attention_no_visible_key_writes_zeros():
    q, k, v, lens, _ = _case(2, 4, 64, 4, 100)
    start = lens + 4                     # beyond the last key of every query
    for splits in (0, 1):
        o = OF.decode_attention(q, k, v, lens, start.contiguous(), scale=0.125, splits=splits)
        assert torch.equal(o, torch.zeros_like(o))


def test_decode_attention_is_bit_identical_between_calls():
    q, k, v, lens, start = _case(3, 8, 128, 4, 4097)
    a = OF.decode_attention(q, k, v, lens, start, scale=0.1)
    b = OF.decode_attention(q, k, v, lens, start, scale=0.1)
    assert torch.equal(a, b)


def test_decode_attention_graph_replay_after_lengths_bump():
    q, k, v, lens, start = _case(2, 4, 64, 1, 500, cap_extra=300)
    OF.decode_attention(q, k, v, lens, start, scale=0.125)          # configure the kernel outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = OF.decode_attention(q, k, v, lens, start, scale=0.125)
    lens.add_(200)                                                   # on the device, as StaticKVCache.advance does
    g.replay()
    eager = OF.decode_attention(q, k, v, lens, start, scale=0.125)
    assert torch.equal(out, eager)
    assert rel_err(out, OF.decode_attention_ref(q, k, v, lens, start, scale=0.125)) < 3e-2


@pytest.mark.parametrize("D", [64, 128])
def test_kv_append_rope_bit_identical_to_rope_qkv(D):
    from libai_b200.models.llama_model import rotary_tables

    B, sq, A, C = 3, 5, 4, 64
    cos, sin = rotary_tables(D, 128, device=DEV)
    qkv = torch.randn(B, sq, A, 3 * D, device=DEV).bfloat16()
    k = torch.zeros(B, A, C, D, device=DEV, dtype=torch.bfloat16)
    v = torch.zeros_like(k)
    lens = torch.tensor([0, 7, 40], dtype=torch.int32, device=DEV)
    before = ops.launch_count()
    q = OF.kv_cache_append(qkv, k, v, lens, cos, sin)
    assert ops.launch_count() == before + 1
    for b in range(B):
        p = int(lens[b])
        want = OF.apply_rotary_qkv(qkv[b : b + 1].contiguous(), cos, sin, p)[0]     # the rope_qkv kernel
        assert torch.equal(q[b], want[..., :D])
        assert torch.equal(k[b, :, p : p + sq], want[..., D : 2 * D].transpose(0, 1))
        assert torch.equal(v[b, :, p : p + sq], want[..., 2 * D :].transpose(0, 1))
    # without tables (GPT-2): plain copy, q not written
    k2, v2 = torch.zeros_like(k), torch.zeros_like(v)
    assert OF.kv_cache_append(qkv, k2, v2, lens, return_q=False) is None
    assert torch.equal(k2[1, :, 7 : 7 + sq], qkv[1, ..., D : 2 * D].transpose(0, 1))


# ------------------------------------------------------------------------------------------------ generate()
def _llama(head_dim):
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    heads = 256 // head_dim   # 64 / 128: native decode kernels; 32: reference math
    cfg = DictConfig(dict(hidden_layers=2, vocab_size=512, hidden_size=256, intermediate_size=512,
                          num_attention_heads=heads, max_position_embeddings=256, rms_norm_eps=1e-5,
                          initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return LlamaForCausalLM(cfg).eval()


def _gpt2():
    from libai_b200.layers._param import param_defaults
    from projects.MagicPrompt.gpt2 import GPTModel

    cfg = DictConfig(dict(
        hidden_layers=2, vocab_size=512, hidden_size=256, ffn_hidden_size=1024, num_attention_heads=4,
        max_seq_length=256, embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
        layernorm_epsilon=1e-5, initializer_range=0.02, use_scaled_init_for_output_weights=True, bias_gelu_fusion=True,
        bias_dropout_fusion=True, scale_mask_softmax_fusion=True, apply_query_key_layer_scaling=True,
        apply_residual_post_layernorm=False, amp_enabled=True, eos_token_id=511, pad_token_id=0, bos_token_id=511))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return GPTModel(cfg).eval()


def _native_decoding(model, monkeypatch, ids, **kw):
    """Greedy cached generation with every decode step on the native kernels: the reference attention raises once
    the cache holds the prompt.  Returns the sequences and the per-step logits."""
    real_ref = OF.attention_ref

    def guarded(*a, **k):
        if model.kv_cache is not None and model.kv_cache.length > 0:
            raise AssertionError("decode step fell back to the reference attention")
        return real_ref(*a, **k)

    launches = {"decode_attention": [], "kv_cache_append": []}

    def counting(name):
        real = getattr(OF, name)

        def fn(*a, **k):
            before = ops.launch_count()
            out = real(*a, **k)
            launches[name].append(ops.launch_count() - before)
            return out
        return fn

    monkeypatch.setattr(OF, "attention_ref", guarded)
    def refuse(*a, **k):
        raise AssertionError("a cached step ran the reference decode attention or cache append")

    monkeypatch.setattr(OF, "decode_attention_ref", refuse)
    monkeypatch.setattr(OF, "kv_cache_append_ref", refuse)
    for name in launches:
        monkeypatch.setattr(OF, name, counting(name))
    seqs, scores = model.generate(ids, max_length=ids.shape[1] + 12, eos_token_id=None, pad_token_id=0,
                                  output_scores=True, **kw)
    monkeypatch.undo()
    decode_steps = len(scores) - 1   # the first score comes from the prefill; both models have 2 layers
    dec, app = launches["decode_attention"], launches["kv_cache_append"]
    assert len(dec) == decode_steps * 2 and all(c > 0 for c in dec), dec
    assert len(app) == (decode_steps + 1) * 2 and all(c > 0 for c in app), app
    return seqs, torch.stack(scores, 1)


def _teacher_forced(model, seqs, prompt_len, attention_mask=None):
    with torch.no_grad():
        if attention_mask is None:
            logits = model(seqs[:, :-1])["logits"]
        else:
            logits = model(seqs[:, :-1], attention_mask=attention_mask[:, :-1])["logits"]
    return logits[:, prompt_len - 1 :].float()


@pytest.mark.parametrize("head_dim", [64, 128])
def test_llama_generate_runs_native_decode(head_dim, monkeypatch):
    model = _llama(head_dim)
    torch.manual_seed(0)
    ids = torch.randint(3, 512, (3, 16), device=DEV)
    seqs, steps = _native_decoding(model, monkeypatch, ids)
    ref = _teacher_forced(model, seqs, 16)
    assert rel_err(steps, ref) < 3e-2, rel_err(steps, ref)
    # left-padded batch: kv_start carries the padding into the decode kernel
    am = torch.ones_like(ids)
    ids[1, :5], am[1, :5] = 0, 0
    seqs, steps = _native_decoding(model, monkeypatch, ids, attention_mask=am)
    full_mask = torch.cat([am, torch.ones_like(seqs[:, 16:])], 1)
    ref = _teacher_forced(model, seqs, 16, full_mask)
    assert rel_err(steps, ref) < 3e-2, rel_err(steps, ref)


def test_llama_head_dim_32_decodes_through_the_reference():
    """Head dims the kernels do not take (and other dtypes) decode with the reference math, as they did before the
    cache existed, and match the uncached forward."""
    model = _llama(32)
    torch.manual_seed(0)
    ids = torch.randint(3, 512, (2, 16), device=DEV)
    seqs, scores = model.generate(ids, max_length=28, eos_token_id=None, pad_token_id=0, output_scores=True)
    ref = _teacher_forced(model, seqs, 16)
    assert rel_err(torch.stack(scores, 1), ref) < 3e-2


def test_gpt2_generate_runs_native_decode(monkeypatch):
    model = _gpt2()
    torch.manual_seed(0)
    ids = torch.randint(3, 500, (2, 16), device=DEV)
    seqs, steps = _native_decoding(model, monkeypatch, ids)
    with torch.no_grad():
        ref = model(seqs[:, :-1])["logits"][:, 15:].float()
    assert rel_err(steps, ref) < 3e-2, rel_err(steps, ref)
