"""Prefix caching on the H100: a call whose prompts start with cached pages reuses them (plain and left-padded prompts,
every decoder-only model with a paged cache except GLM), bit for bit what the same rows give in a contiguous cache,
and within bf16 tolerance of a full prefill; a chat turn reuses the pages of the previous turn's answer; decode graphs
replay the existing capture."""
import pytest
import torch

from libai_b200.config import DictConfig, LazyConfig, instantiate
from libai_b200.inference import decode_graph
from libai_b200.inference.kv_cache import PagedKVCache, StaticKVCache
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import LLAMA
from tests.test_decode_graphs_gpu import _Captures

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BUDGET = 1024


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


def _llama(**kw):
    from libai_b200.models import LlamaForCausalLM

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return LlamaForCausalLM(DictConfig(dict(LLAMA, max_position_embeddings=512, **kw))).eval()


def _adapter():
    from projects.Llama.adapter.adapter_model import LlamaForCausalLM

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        m = LlamaForCausalLM(DictConfig(dict(LLAMA, max_position_embeddings=512, hidden_size=256, num_attention_heads=4,
                                             adapter_len=4, adapter_layer=2))).eval()
    with torch.no_grad():
        for layer in m.model.layers:
            layer.self_attn.gate.copy_(torch.linspace(0.5, 2.0, layer.self_attn.gate.numel()).view_as(
                layer.self_attn.gate))
    return m


def _gpt2():
    from projects.MagicPrompt.gpt2 import GPTModel

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return GPTModel(DictConfig(dict(
            hidden_layers=2, vocab_size=100, hidden_size=128, ffn_hidden_size=128, num_attention_heads=2,
            max_seq_length=512, embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
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


def _chatglm():
    c = LazyConfig.load("projects/ChatGLM/configs/chatglm_config.py")
    c = LazyConfig.apply_overrides(c, [
        "cfg.num_layers=2", "cfg.hidden_size=128", "cfg.ffn_hidden_size=128", "cfg.num_attention_heads=4",
        "cfg.kv_channels=64", "cfg.multi_query_group_num=2", "cfg.padded_vocab_size=100", "cfg.seq_length=512",
        "cfg.max_length=20", "cfg.pad_token_id=0"])
    c.model.cfg = c.cfg
    torch.manual_seed(0)
    return instantiate(c.model).to(torch.bfloat16).eval()


BUILDERS = {"llama_gqa": lambda: _llama(hidden_size=256, num_attention_heads=4, num_key_value_heads=2),
            "qwen": lambda: _llama(qkv_bias=True), "gpt2": _gpt2, "bloom": _bloom, "chatglm": _chatglm,
            "llama_adapter": _adapter}
PADDED = ("llama_gqa", "qwen", "bloom", "chatglm", "llama_adapter")


def _ids(b, s, seed):
    # above every special id (BLOOM pads with 3): an unpadded prompt's mask is all ones
    return torch.randint(4, 100, (b, s), generator=torch.Generator().manual_seed(seed)).to(DEV)


def _gen(m, ids, mask=None, new=6, **kw):
    kw = dict(eos_token_id=None, output_scores=True, max_new_tokens=new, **kw)
    if mask is not None:
        kw["attention_mask"] = mask
    with torch.no_grad():
        return m.generate(ids, **kw)


def _prompts(case):
    a = _ids(3, 150, 1)
    b = torch.cat([a[:, :140], _ids(3, 30, 2)], dim=1)
    if case == "plain":
        return a, None, b, None
    ma, mb = torch.ones_like(a), torch.ones_like(b)
    for t, m in ((a, ma), (b, mb)):
        m[1, :2] = m[2, :5] = 0
        t.masked_fill_(m == 0, 0)
    return a, ma, b, mb


@pytest.mark.parametrize("case", ["plain", "left_padded"])
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_hit_reuses_pages_and_matches_a_full_prefill(name, case):
    if case == "left_padded" and name not in PADDED:
        pytest.skip("the model takes no padding mask")
    m = BUILDERS[name]().to(DEV)
    a, ma, b, mb = _prompts(case)
    full = _gen(m, b, mb, paged_kv_cache=True)
    _gen(m, a, ma, prefix_cache_tokens=BUDGET)
    assert m.kv_cache.reused_rows == 0
    hit = _gen(m, b, mb, prefix_cache_tokens=BUDGET)
    assert m.kv_cache.reused_rows == 128
    # the first logits: the suffix's GEMMs see another number of rows than a full prefill's
    x, y = hit[1][0], full[1][0]
    assert (x - y).abs().max() <= 0.03 * y.abs().max() + 0.02, (x - y).abs().max()


def test_hit_is_bit_identical_to_the_same_rows_in_a_contiguous_cache():
    m = BUILDERS["llama_gqa"]().to(DEV)
    a, _, b, _ = _prompts("plain")
    _gen(m, a, prefix_cache_tokens=BUDGET)
    ids, scores = _gen(m, b, prefix_cache_tokens=BUDGET)
    c = m.kv_cache
    assert c.reused_rows == 128
    table = []
    for row in b.tolist():
        parent, pages = -1, []
        for key in c._page_keys(row, [1] * b.shape[1], 2):
            parent = c._index[(parent, key)]
            pages.append(parent)
        table.append(pages)
    table = torch.tensor(table, dtype=torch.int32, device=DEV)
    ref = StaticKVCache(len(c.owned), 3, c.heads, c.head_dim, 256, torch.bfloat16, DEV)
    for i in c.owned:
        ref.write_rows(i, OF.kv_pages_gather(c.k[i], table, 128), OF.kv_pages_gather(c.v[i], table, 128))
    ref.advance(128)
    m.kv_cache = ref
    with torch.no_grad():
        seq, want = b, []
        out = m(seq[:, 128:], use_cache=True)
        for _ in range(6):
            logits = out["logits"][:, -1].float()
            want.append(logits)
            seq = torch.cat([seq, logits.argmax(-1, keepdim=True)], dim=1)
            out = m(seq[:, -1:], use_cache=True)
    assert torch.equal(ids, seq)
    assert all(torch.equal(x, y) for x, y in zip(scores, want))


def test_chat_turn_reuses_the_previous_answer():
    m = BUILDERS["llama_gqa"]().to(DEV)
    # both turns fit the first turn's pool (three pages per sequence), so it and its index are kept, as for chat()'s
    # calls with one max_length
    kw = dict(eos_token_id=None, output_scores=True, max_length=192, prefix_cache_tokens=BUDGET)
    turn1 = _ids(1, 120, 3)
    with torch.no_grad():
        out1, _ = m.generate(turn1, **dict(kw, max_length=160))   # 159 rows cached: the second page holds the answer
        turn2 = torch.cat([out1, _ids(1, 30, 4)], dim=1)
        m.generate(turn2, **kw)
    assert m.kv_cache.reused_rows == 128


def test_decode_graphs_with_a_hit(monkeypatch):
    m = BUILDERS["llama_gqa"]().to(DEV)
    a, _, b, _ = _prompts("plain")
    _gen(m, a, prefix_cache_tokens=BUDGET)
    eager = _gen(m, b, prefix_cache_tokens=BUDGET)
    captures = _Captures(monkeypatch)
    graphs = _gen(m, b, prefix_cache_tokens=BUDGET, decode_graphs=True)
    assert m.kv_cache.reused_rows == 128 and captures.n == 1
    assert torch.equal(eager[0], graphs[0]) and all(torch.equal(x, y) for x, y in zip(eager[1], graphs[1]))
    again = _gen(m, b, prefix_cache_tokens=BUDGET, decode_graphs=True)
    assert captures.n == 1 and isinstance(m.kv_cache, PagedKVCache) and decode_graph.current_graph(m) is not None
    assert torch.equal(again[0], graphs[0])
