"""``generate(decode_graphs=True)`` on the H100: small random models of every KV-cache family (Llama with GQA, Qwen with a
qkv bias, GPT-2, BLOOM, ChatGLM with multi-query attention, GLM and mT5) return the tokens and per-step scores of
eager decoding bit for bit, on bf16 and FP8 caches, FP8 weights, left-padded prompts and a prompt that needs the dense
mask; beam search keeps one capture through its in-place reorders; a replayed step launches nothing from Python, counts
the eager step's kernels and syncs nothing; and the device-position form of the GLM rotary kernel replays from a graph."""
import copy

import pytest
import torch

from libai_b200 import ops
from libai_b200.config import DictConfig
from libai_b200.inference import decode_graph, quantize_weights_fp8_
from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import LLAMA, MODELS, _prompt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


def _qwen():
    from libai_b200.models import LlamaForCausalLM

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        return LlamaForCausalLM(DictConfig(dict(LLAMA, qkv_bias=True))).eval()


def _glm():
    from projects.GLM.modeling_glm import GLMForConditionalGeneration
    from tests.test_glm_native_cpu import tiny_cfg

    cfg = tiny_cfg()
    cfg.update(dict(vocab_size=256, hidden_size=256, num_attention_heads=4, num_layers=2, max_sequence_length=128))
    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=5):
        return GLMForConditionalGeneration(cfg).eval()


def _adapter():
    """LLaMA-Adapter with non-zero gates (a fresh one's are zero, and its adapter path then adds nothing)."""
    from projects.Llama.adapter.adapter_model import LlamaForCausalLM

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        m = LlamaForCausalLM(DictConfig(dict(LLAMA, hidden_size=256, num_attention_heads=4, adapter_len=4,
                                             adapter_layer=2))).eval()
    with torch.no_grad():
        for layer in m.model.layers:
            gate = layer.self_attn.gate
            gate.copy_(torch.linspace(0.5, 2.0, gate.numel()).view_as(gate))
    return m


BUILDERS = {"llama_gqa": MODELS["llama_gqa"], "qwen": _qwen, "gpt2": MODELS["gpt2"], "bloom": MODELS["bloom"],
            "chatglm": MODELS["chatglm"], "glm": _glm, "t5": MODELS["t5"], "llama_adapter": _adapter}
# the models whose forward takes a padding mask
PADDED = ("llama_gqa", "qwen", "bloom", "chatglm", "t5", "llama_adapter")


def _model(name, fp8_weights=False):
    m = BUILDERS[name]().to(DEV)
    if name == "t5":   # as in the FP8 tests: T5's builder makes its logits chaotic at bf16 precision
        with torch.no_grad():
            for p in m.parameters():
                p.mul_(0.2)
    return quantize_weights_fp8_(m) if fp8_weights else m


def _glm_inputs(b=3):
    from tests.test_glm_native_cpu import Tok

    ids = torch.tensor([[11, 12, 13, 7, 14, 15, 16], [31, 7, 33, 34, 0, 0, 0], [41, 42, 7, 43, 44, 45, 0]])[:b]
    inp = Tok().build_inputs_for_generation({"input_ids": ids, "attention_mask": (ids != 0).long()}, max_gen_length=12)
    return {k: v.to(DEV) for k, v in inp.items()}


def _generate(m, name, graphs, case="plain", new=8, b=3, **kw):
    """``generate(..., output_scores=True)`` on prompt ``case`` (batch ``b``)."""
    kw = dict(eos_token_id=None, output_scores=True, decode_graphs=graphs, **kw)
    with torch.no_grad():
        if name == "glm":   # (beam search takes the per-sample inputs once per beam)
            inp = _glm_inputs(b)
            ids, beams = inp.pop("input_ids"), kw.get("num_beams", 1)
            inp = {k: v.repeat_interleave(beams, 0) for k, v in inp.items()}
            return m.generate(ids, position_ids=inp["position_ids"], max_length=ids.shape[1] + new, use_cache=True,
                              generation_attention_mask=inp["generation_attention_mask"], **kw)
        ids, am = _prompt(case)
        ids = ids[:b].to(DEV)
        am = None if am is None else am[:b].to(DEV)
        if name == "t5":
            return m.generate(ids, encoder_attn_mask=am, max_length=new, **kw)
        if am is not None:
            kw["attention_mask"] = am
        return m.generate(ids, max_length=ids.shape[1] + new, **kw)


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if torch.is_tensor(x):
            assert torch.equal(x, y)
        else:
            assert len(x) == len(y) and all(torch.equal(p, q) for p, q in zip(x, y))


class _Captures:
    """Counts the captures of decode graphs."""

    def __init__(self, monkeypatch):
        self.n = 0
        capture = decode_graph.DecodeGraph._capture

        def counted(graph, *a, **k):
            self.n += 1
            return capture(graph, *a, **k)

        monkeypatch.setattr(decode_graph.DecodeGraph, "_capture", counted)


# ------------------------------------------------------------------------------------------------ same tokens and scores
@pytest.mark.parametrize("kv", [None, "fp8"])
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_greedy_tokens_and_scores_are_bit_identical(monkeypatch, name, kv):
    m = _model(name)
    captures = _Captures(monkeypatch)
    eager = _generate(m, name, False, kv_cache_dtype=kv)
    graphs = _generate(m, name, True, kv_cache_dtype=kv)
    _same(eager, graphs)
    assert captures.n == 1 and decode_graph.current_graph(m).graph is not None


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_fp8_weights_are_bit_identical(monkeypatch, name):
    m = _model(name, fp8_weights=True)
    captures = _Captures(monkeypatch)
    _same(_generate(m, name, False, kv_cache_dtype="fp8"), _generate(m, name, True, kv_cache_dtype="fp8"))
    assert captures.n == 1


@pytest.mark.parametrize("name", PADDED)
def test_left_padded_prompt_is_bit_identical(monkeypatch, name):
    m = _model(name)
    captures = _Captures(monkeypatch)
    _same(_generate(m, name, False, "left_padded"), _generate(m, name, True, "left_padded"))
    assert captures.n == 1
    cache = m.cross_cache if name == "t5" else m.kv_cache
    assert not cache.dense_mask


@pytest.mark.parametrize("name", PADDED)
def test_dense_mask_prompt_falls_back_and_is_bit_identical(monkeypatch, caplog, name):
    m = _model(name)
    captures = _Captures(monkeypatch)
    eager = _generate(m, name, False, "hole")
    with caplog.at_level("INFO", logger=decode_graph.__name__):
        graphs = _generate(m, name, True, "hole")
    _same(eager, graphs)
    assert captures.n == 0
    lines = [r.getMessage() for r in caplog.records if r.name == decode_graph.__name__]
    assert len(lines) == 1 and "dense mask" in lines[0], lines


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_beam_search_is_bit_identical_with_one_capture(monkeypatch, name):
    m = _model(name)
    captures = _Captures(monkeypatch)
    reorders = []
    reorder = StaticKVCache.reorder_

    def counted(cache, idx):
        reorders.append(cache)
        return reorder(cache, idx)

    monkeypatch.setattr(StaticKVCache, "reorder_", counted)
    eager = _generate(m, name, False, num_beams=4)
    n_eager = len(reorders)
    graphs = _generate(m, name, True, num_beams=4)
    _same(eager, graphs)
    assert n_eager > 2 and len(reorders) == 2 * n_eager   # the in-place reorders kept the graph's key
    assert captures.n == 1


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_seeded_sampling_gives_identical_tokens(name):
    m = _model(name)
    out = []
    for graphs in (False, True):
        torch.manual_seed(7)
        out.append(_generate(m, name, graphs, do_sample=True, top_k=20, temperature=0.9))
    _same(out[0], out[1])


@pytest.mark.parametrize("name", ["llama_gqa", "t5", "glm"])
def test_graph_reuse_and_new_captures(monkeypatch, name):
    m = _model(name)
    captures = _Captures(monkeypatch)
    first = _generate(m, name, True)
    graph = decode_graph.current_graph(m)
    second = _generate(m, name, True)
    _same(first, second)
    assert captures.n == 1 and decode_graph.current_graph(m) is graph   # same batch, cache large enough: replayed
    _same(_generate(m, name, False, b=2), _generate(m, name, True, b=2))
    assert captures.n == 2 and decode_graph.current_graph(m) is not graph   # a new batch captures again
    _generate(m, name, True, b=2, kv_cache_dtype="fp8")
    assert captures.n == 3                                                 # so does a new KV dtype


def test_the_adapter_path_changes_the_tokens():
    """The adapter's gated attention reaches the logits in the adapter test model, so its tests compare something."""
    m = _model("llama_adapter")
    with_adapter = _generate(m, "llama_adapter", True)
    with torch.no_grad():
        for layer in m.model.layers:
            layer.self_attn.gate.zero_()
    without = _generate(m, "llama_adapter", True)
    assert not all(torch.equal(a, b) for a, b in zip(with_adapter[1], without[1]))


def test_a_reallocated_cache_captures_again(monkeypatch):
    """A cache that must grow runs that step eagerly (``reserve()`` reallocates its buffers); the next steps capture a
    new graph on the new buffers, and every step's logits are the eager ones."""
    m = _model("llama_gqa")
    twin = copy.deepcopy(m)
    captures = _Captures(monkeypatch)
    ids, _ = _prompt("plain")
    ids = ids.to(DEV)
    tokens = torch.randint(3, 100, (8, 3), generator=torch.Generator().manual_seed(2)).to(DEV)
    call = decode_graph.DecodeCall()
    with torch.no_grad():
        for model in (m, twin):
            model.allocate_kv_cache(3, 9)   # the prompt's 7 rows and 2 more
            model(ids, use_cache=True)
        for i in range(1, 8):
            want = twin(input_ids=tokens[i][:, None], use_cache=True)["logits"]
            got = decode_graph.step(m, {"input_ids": tokens[i][:, None], "use_cache": True}, call)["logits"]
            assert torch.equal(got, want)
            if i == 3:
                assert captures.n == 1 and m.kv_cache.capacity > 9   # the eager step grew the cache
    assert captures.n == 2 and "the cache must grow" in call.logged
    assert decode_graph.current_graph(m).key[2][0][1] == m.kv_cache.capacity


# ------------------------------------------------------------------------------------------------ a replayed step
def _step_inputs(name, m, tokens):
    if name == "t5":
        return {"encoder_input_ids": None, "decoder_input_ids": tokens[:, None], "use_cache": True}
    return {"input_ids": tokens[:, None], "use_cache": True}


@pytest.mark.parametrize("name", ["llama_gqa", "bloom", "chatglm", "t5", "llama_adapter"])
def test_replayed_step_launches_nothing_from_python_and_matches_the_eager_state(monkeypatch, name):
    m = _model(name)
    twin = copy.deepcopy(m)
    ids, _ = _prompt("plain")
    ids = ids.to(DEV)
    tokens = torch.randint(3, 100, (8, 3), generator=torch.Generator().manual_seed(2)).to(DEV)
    call = decode_graph.DecodeCall()
    with torch.no_grad():
        for model in (m, twin):
            model.allocate_kv_cache(3, 16)
        prefill = (lambda mm: mm(ids, tokens[0][:, None], None, use_cache=True)) if name == "t5" else \
            (lambda mm: mm(ids, use_cache=True))
        prefill(m)
        prefill(twin)
        eager_launches = []
        for i in range(1, 8):
            n0 = ops.launch_count()
            want = twin(**_step_inputs(name, twin, tokens[i]))["logits"]
            eager_launches.append(ops.launch_count() - n0)
            calls = {"decode_attention": 0, "kv_cache_append": 0}
            for fn in calls:
                def counted(*a, _fn=fn, _orig=getattr(OF, fn), **k):
                    calls[_fn] += 1
                    return _orig(*a, **k)
                monkeypatch.setattr(OF, fn, counted)
            replayed = i >= 3   # step 1 runs eagerly, step 2 is captured and replayed, later steps are replayed
            n0 = ops.launch_count()
            if replayed:
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode("error")
            try:
                got = decode_graph.step(m, _step_inputs(name, m, tokens[i]), call)["logits"]
            finally:
                torch.cuda.set_sync_debug_mode("default")
            launches = ops.launch_count() - n0
            monkeypatch.undo()
            assert torch.equal(got, want)
            if replayed:
                assert calls == {"decode_attention": 0, "kv_cache_append": 0}
                assert launches == eager_launches[-1] > 0
            # the invariant: the cache rows, lengths and host mirrors are those of eager decoding
            for c, t in zip(decode_graph._caches(m), decode_graph._caches(twin)):
                assert c.length == t.length and torch.equal(c.seqlens, t.seqlens)
                assert torch.equal(c.kv_start, t.kv_start)
                for i_layer in c.owned:
                    for a, b in ((c.k, t.k), (c.v, t.v)):
                        assert torch.equal(a[i_layer][:, :, : c.length], b[i_layer][:, :, : t.length])
            assert m.past_length == twin.past_length


# ------------------------------------------------------------------------------------------------ the kernel's device form
def test_glm_rotary_device_base_replays_from_a_graph():
    """``glm_rotary_qkv`` with ``pos_base`` (the decode step's form): bit for bit the host-offset form at every base, in
    one captured graph replayed after the base changed."""
    ext = ops.load_ext(required=True)
    torch.manual_seed(0)
    a, g, d, pre = 8, 2, 128, 3
    table = OF.glm_rope_table(64, d // 2, device=DEV)
    mixed = torch.randn(2, 1, (a + 2 * g) * d, device=DEV).to(torch.bfloat16)
    base = torch.full((2,), pre, dtype=torch.int32, device=DEV)
    for grouped in (True, False):
        ext.glm_rotary_qkv(mixed, a, g, table, -pre, None, grouped, base)   # warm-up
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = ext.glm_rotary_qkv(mixed, a, g, table, -pre, None, grouped, base)
        for length in (pre, pre + 1, pre + 17, 63 + pre):
            base.fill_(length)
            mixed.copy_(torch.randn_like(mixed, dtype=torch.float32).to(torch.bfloat16))
            graph.replay()
            want = ext.glm_rotary_qkv(mixed, a, g, table, length - pre, None, grouped)
            assert torch.equal(out, want)
            assert torch.equal(out, OF.apply_glm_rotary_qkv_ref(mixed, heads=a, kv_heads=g, table=table,
                                                                pos_offset=length - pre, grouped=grouped))
    with pytest.raises(RuntimeError, match="exclude each other"):
        ext.glm_rotary_qkv(mixed, a, g, table, 0, torch.zeros(2, 1, dtype=torch.int32, device=DEV), True, base)
    with pytest.raises(RuntimeError, match="pos_base"):
        ext.glm_rotary_qkv(mixed, a, g, table, 0, None, True, base.long())


def test_glm_rotary_device_base_backward_equals_the_host_offset():
    """The backward of ``pos_base`` (a cached ChatGLM forward with gradients) is bit for bit that of the host offset."""
    torch.manual_seed(1)
    a, g, d, pre = 8, 2, 128, 3
    table = OF.glm_rope_table(64, d // 2, device=DEV)
    base = torch.full((2,), 20, dtype=torch.int32, device=DEV)
    for grouped in (True, False):
        mixed = torch.randn(2, 3, (a + 2 * g) * d, device=DEV).to(torch.bfloat16)
        outs = []
        for kw in (dict(pos_offset=20 - pre), dict(pos_offset=-pre, pos_base=base)):
            x = mixed.clone().requires_grad_(True)
            y = OF.apply_glm_rotary_qkv(x, heads=a, kv_heads=g, table=table, grouped=grouped, **kw)
            y.backward(torch.linspace(-1, 1, y.numel(), device=DEV).view_as(y).to(y.dtype))
            outs.append((y.detach(), x.grad))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
