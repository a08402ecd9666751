"""``generate(decode_graphs=True)`` without a GPU: the option, the eligibility rule of every eager fallback, the same
tokens as eager decoding on CPU models (which fall back), and the device-side positions of GPT-2 and ChatGLM against
today's host-offset forms through the reference math."""
import copy
import logging
from types import SimpleNamespace

import pytest
import torch
from torch import nn

from libai_b200.config import DictConfig
from libai_b200.inference import decode_graph
from libai_b200.inference.generator.generation_utils import _DEFAULTS, Generator, _decode_graphs
from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import MODELS, _prompt


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


# ------------------------------------------------------------------------------------------------ the option
def test_option_parsing_and_default():
    assert _DEFAULTS["decode_graphs"] is False
    assert _decode_graphs(True) is True and _decode_graphs(False) is False
    for bad in ("yes", 1, None):
        with pytest.raises(ValueError, match="decode_graphs must be True or False"):
            _decode_graphs(bad)


class _NoCache(nn.Module, Generator):
    """A generator model with no StaticKVCache."""

    def __init__(self):
        super().__init__()
        self.cfg = DictConfig(dict(eos_token_id=None, pad_token_id=0, bos_token_id=1))
        self.w = nn.Parameter(torch.zeros(1))

    def forward(self, input_ids, use_cache=False):
        return {"logits": torch.zeros(*input_ids.shape, 10)}


def test_a_model_without_a_static_cache_raises():
    m = _NoCache().eval()
    ids = torch.ones(1, 3, dtype=torch.long)
    with pytest.raises(ValueError, match="decode_graphs=True: _NoCache does not decode on a StaticKVCache"):
        m.generate(ids, max_length=5, decode_graphs=True)
    m.cfg.decode_graphs = True   # the model cfg's default goes the same way
    with pytest.raises(ValueError, match="decode_graphs=True"):
        m.generate(ids, max_length=5)
    assert m.generate(ids, max_length=5, decode_graphs=False).shape == (1, 5)


# ------------------------------------------------------------------------------------------------ eligibility
def _eligible_step(monkeypatch, cross=False):
    """A model-like object on a (meta) cache that claims to be on the GPU, with every condition of a replay met."""
    monkeypatch.setattr(decode_graph, "use_native", lambda *t: True)

    def cache(capacity=16, dtype=torch.bfloat16, d=64):
        c = StaticKVCache(2, 3, 2, d, capacity, dtype, "meta")
        c.device, c.length = torch.device("cuda", 0), 5
        return c

    model = SimpleNamespace(kv_cache=cache(), max_cache_positions=None, past_length=5)
    if cross:
        model.cross_cache = cache()
    inputs = {"input_ids": torch.ones(3, 1, dtype=torch.long), "use_cache": True,
              "attention_mask": torch.ones(3, 6)}   # ignored: kv_start holds a left-padded prompt's padding
    return model, inputs, cache


def test_an_eligible_step(monkeypatch):
    model, inputs, _ = _eligible_step(monkeypatch, cross=True)
    assert decode_graph.fallback_reason(model, inputs) is None
    t5 = {"decoder_input_ids": torch.ones(3, 1, dtype=torch.long), "encoder_input_ids": torch.ones(3, 9),
          "encoder_attn_mask": torch.ones(3, 9), "use_cache": True}
    assert decode_graph.fallback_reason(model, t5) is None


def _reason(monkeypatch, change):
    model, inputs, cache = _eligible_step(monkeypatch, cross=True)
    change(model, inputs, cache)
    return decode_graph.fallback_reason(model, inputs)


def _tp(monkeypatch):
    monkeypatch.setattr(dist, "get_dist_util", lambda: SimpleNamespace(tensor_parallel_size=2, pipeline_parallel_size=1))


FALLBACKS = {
    "cpu": (lambda m, i, c: setattr(m.kv_cache, "device", torch.device("cpu")), "not on a CUDA device"),
    "fp32": (lambda m, i, c: setattr(m, "kv_cache", c(dtype=torch.float32)), "native bf16 kernels"),
    "head_dim": (lambda m, i, c: setattr(m, "kv_cache", c(d=32)), "native bf16 kernels"),
    "tokens": (lambda m, i, c: i.update(input_ids=torch.ones(3, 2, dtype=torch.long)), "more than one new token"),
    "dense": (lambda m, i, c: setattr(m.kv_cache, "dense_mask", True), "dense mask"),
    "cross_dense": (lambda m, i, c: setattr(m.cross_cache, "dense_mask", True), "dense mask"),
    "full": (lambda m, i, c: setattr(m.kv_cache, "length", 16), "the cache must grow"),
    "max_positions": (lambda m, i, c: setattr(m, "max_cache_positions", 5), "maximum length"),
    "input": (lambda m, i, c: i.update(labels=torch.ones(3, 1)), "input 'labels' is not a static buffer"),
}


@pytest.mark.parametrize("case", sorted(FALLBACKS) + ["parallel"])
def test_each_fallback_has_its_reason(monkeypatch, case):
    if case == "parallel":
        def change(m, i, c):
            _tp(monkeypatch)
        fragment = "tensor- or pipeline-parallel"
    else:
        change, fragment = FALLBACKS[case]
    reason = _reason(monkeypatch, change)
    assert reason is not None and fragment in reason, reason


def test_static_and_ignored_inputs_do_not_depend_on_values():
    a = {"input_ids": torch.ones(3, 1, dtype=torch.long), "attention_mask": torch.ones(3, 6), "use_cache": True}
    b = {"input_ids": torch.zeros(3, 1, dtype=torch.long), "attention_mask": torch.zeros(3, 7), "use_cache": True}
    assert decode_graph._signature(a) == decode_graph._signature(b)
    c = dict(b, input_ids=torch.zeros(4, 1, dtype=torch.long))
    assert decode_graph._signature(a) != decode_graph._signature(c)
    d = dict(a)
    del d["attention_mask"]
    assert decode_graph._signature(a) != decode_graph._signature(d)


# ------------------------------------------------------------------------------------------------ CPU models fall back
def _generate(m, name, graphs, case="plain", beams=1):
    ids, am = _prompt(case)
    with torch.no_grad():
        if name == "t5":
            return m.generate(ids, encoder_attn_mask=am, max_length=6, eos_token_id=None, num_beams=beams,
                              output_scores=True, decode_graphs=graphs)
        kw = {} if am is None else {"attention_mask": am}
        return m.generate(ids, max_length=ids.shape[1] + 5, eos_token_id=None, num_beams=beams, output_scores=True,
                          decode_graphs=graphs, **kw)


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if torch.is_tensor(x):
            assert torch.equal(x, y)
        else:
            assert len(x) == len(y) and all(torch.equal(p, q) for p, q in zip(x, y))


@pytest.mark.parametrize("beams", [1, 2])
@pytest.mark.parametrize("name", sorted(MODELS))
def test_cpu_models_fall_back_to_the_same_tokens(name, beams, caplog):
    m = MODELS[name]()
    eager = _generate(m, name, False, beams=beams)
    with caplog.at_level(logging.INFO, logger=decode_graph.__name__):
        graphs = _generate(m, name, True, beams=beams)
    _same(eager, graphs)
    lines = [r.getMessage() for r in caplog.records if r.name == decode_graph.__name__]
    assert len(lines) == 1 and "the cache is not on a CUDA device" in lines[0], lines
    assert decode_graph.current_graph(m) is None


# ------------------------------------------------------------------------------------------------ device positions
@pytest.mark.parametrize("name,case", [("chatglm", "plain"), ("chatglm", "left_padded"), ("chatglm_prefix", "plain")])
def test_chatglm_device_positions_equal_the_host_offset(monkeypatch, name, case):
    """The cached steps read their rotary positions from ``cache.seqlens`` (``pos_base``); converting that back into
    the host offset ``past - pre`` of the previous form gives bit-identical logits."""
    from projects.ChatGLM import chatglm

    m = MODELS[name]()
    device_form = _generate(m, name, False, case)
    rotary = OF.apply_glm_rotary_qkv
    seen = []

    def host_offset(mixed, pos_base=None, pos_offset=0, **kw):
        if pos_base is not None:
            seen.append(int(pos_base[0]) + pos_offset)
            pos_offset, pos_base = pos_offset + int(pos_base[0]), None
        return rotary(mixed, pos_offset=pos_offset, **kw)

    monkeypatch.setattr(chatglm.OF, "apply_glm_rotary_qkv", host_offset)
    host_form = _generate(m, name, False, case)
    _same(device_form, host_form)
    layers = m.cfg.num_layers
    assert seen == [p for p in [0] + list(range(7, 11)) for _ in range(layers)]   # the prompt, then 7, 8, ...


def test_glm_rotary_ref_with_a_device_base_equals_the_offset():
    torch.manual_seed(0)
    a, g, d, s = 4, 2, 64, 3
    mixed = torch.randn(2, s, (a + 2 * g) * d).to(torch.bfloat16)
    table = OF.glm_rope_table(32, d // 2)
    for grouped in (False, True):
        want = OF.apply_glm_rotary_qkv_ref(mixed, heads=a, kv_heads=g, table=table, pos_offset=9, grouped=grouped)
        base = torch.tensor([12, 12], dtype=torch.int32)
        got = OF.apply_glm_rotary_qkv(mixed, heads=a, kv_heads=g, table=table, pos_offset=-3, grouped=grouped,
                                      pos_base=base)
        assert torch.equal(want, got)
    with pytest.raises(ValueError, match="exclude each other"):
        OF.apply_glm_rotary_qkv(mixed, heads=a, kv_heads=g, table=table, pos_base=base,
                                position_ids=torch.zeros(2, s, dtype=torch.int32))


@pytest.mark.parametrize("beams", [1, 2])
def test_gpt2_device_positions_equal_the_host_offset(monkeypatch, beams):
    """GPT-2's cached steps take their position ids from ``cache.seqlens``; the previous form's host offset
    ``cache.length`` gives bit-identical logits."""
    m = MODELS["gpt2"]()
    device_form = _generate(m, "gpt2", False, beams=beams)
    embed = type(m.embeddings).forward
    seen = []

    def host_offset(self, input_ids, past_length=0, position_ids=None):
        if position_ids is not None:
            assert position_ids.dtype == torch.long and position_ids.shape == (input_ids.shape[1],)
            past_length = int(position_ids[0])
            seen.append(past_length)
        return embed(self, input_ids, past_length)

    monkeypatch.setattr(type(m.embeddings), "forward", host_offset)
    host_form = _generate(m, "gpt2", False, beams=beams)
    _same(device_form, host_form)
    assert seen == [0] + list(range(7, 11))


def _adapter(gates=True):
    from projects.Llama.adapter.adapter_model import LlamaForCausalLM
    from tests.test_cached_attention_cpu import LLAMA

    from libai_b200.layers._param import param_defaults

    with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
        m = LlamaForCausalLM(DictConfig(dict(LLAMA, adapter_len=4, adapter_layer=2))).eval()
    with torch.no_grad():
        for layer in m.model.layers:
            layer.self_attn.gate.fill_(0.8 if gates else 0.0)
    return m


@pytest.mark.parametrize("case", ["plain", "left_padded"])
def test_llama_adapter_device_positions_equal_the_host_offset(monkeypatch, case):
    """The adapter's query rotary in a cached step reads its positions from ``cache.seqlens``; converting them back
    into the host offset ``cache.length`` of the previous form gives bit-identical logits (gates non-zero)."""
    from projects.Llama.adapter import adapter_model

    m = _adapter()
    device_form = _generate(m, "llama", False, case)
    rotary = OF.apply_rotary_qkv
    seen = []

    def host_offset(qkv, cos, sin, pos_offset=0, position_ids=None):
        if position_ids is not None:
            assert position_ids.dtype == torch.int32 and bool((position_ids == position_ids[:1]).all())
            pos_offset, position_ids = int(position_ids[0, 0]), None
            seen.append(pos_offset)
        return rotary(qkv, cos, sin, pos_offset, position_ids)

    monkeypatch.setattr(adapter_model.OF, "apply_rotary_qkv", host_offset)
    host_form = _generate(m, "llama", False, case)
    _same(device_form, host_form)
    assert seen == [p for p in [0] + list(range(7, 11)) for _ in range(2)]
    gates_off = _generate(_adapter(gates=False), "llama", False, case)
    assert not all(torch.equal(a, b) for a, b in zip(device_form[1], gates_off[1]))   # the adapter path matters


@pytest.mark.parametrize("name", ["chatglm", "chatglm_prefix"])
def test_chatglm_cached_forward_with_gradients(monkeypatch, name):
    """A cached ChatGLM forward outside ``torch.no_grad()`` (``pos_base`` has a backward): the logits and the input
    gradients of the host-offset form, bit for bit."""
    from projects.ChatGLM import chatglm

    ids, _ = _prompt("plain")
    base = MODELS[name]()

    def run():
        m = copy.deepcopy(base)
        m.allocate_kv_cache(3, 12)
        emb = m.glm.embedding.word_embeddings.weight
        emb.requires_grad_(True)
        out = [m(ids, use_cache=True)["logits"], m(ids[:, :1], use_cache=True)["logits"]]
        assert all(o.requires_grad for o in out)
        torch.cat(out, 1).float().square().sum().backward()
        return [o.detach() for o in out] + [emb.grad]

    device_form = run()
    rotary = OF.apply_glm_rotary_qkv

    def host_offset(mixed, pos_base=None, pos_offset=0, **kw):
        if pos_base is not None:
            pos_offset, pos_base = pos_offset + int(pos_base[0]), None
        return rotary(mixed, pos_offset=pos_offset, **kw)

    monkeypatch.setattr(chatglm.OF, "apply_glm_rotary_qkv", host_offset)
    host_form = run()
    _same(device_form, host_form)


def test_a_new_cache_drops_the_decode_graph():
    m = MODELS["llama"]()
    m.allocate_kv_cache(3, 12)
    m._decode_graph = graph = object()
    m.allocate_kv_cache(3, 10)    # the same cache, large enough: kept
    assert decode_graph.current_graph(m) is graph
    m.allocate_kv_cache(2, 10)    # a new cache: the graph that wrote the old one goes with it
    assert decode_graph.current_graph(m) is None


class _FailingGraph:
    def __init__(self, *a, **k):
        pass


class _Capture:
    """Stands in for ``torch.cuda.graph``: marks the captured Python (which, on the GPU, would launch no kernel)."""

    active = False

    def __init__(self, graph):
        pass

    def __enter__(self):
        _Capture.active = True

    def __exit__(self, *exc):
        _Capture.active = False


def test_a_failed_capture_falls_back_to_eager_steps(monkeypatch, caplog):
    """A capture that raises (here: the step's Python changes host state, then fails, as a host sync would) rolls back
    the host mirrors, logs once, and every later step on that key runs eagerly, with the tokens of eager decoding."""
    m = MODELS["llama"]()
    eager = _generate(m, "llama", False)
    monkeypatch.setattr(decode_graph, "fallback_reason", lambda model, inputs: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _FailingGraph)
    monkeypatch.setattr(torch.cuda, "graph", _Capture)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "set_stream", lambda s: None)
    calls = []
    forward = type(m).forward

    def step(self, *a, **k):
        calls.append(self.kv_cache.length if self.kv_cache is not None else 0)
        if _Capture.active:
            self.kv_cache.length += 1
            self.past_length = 99
            raise RuntimeError("operation not permitted when stream is capturing")
        return forward(self, *a, **k)

    monkeypatch.setattr(type(m), "forward", step)
    with caplog.at_level(logging.INFO, logger=decode_graph.__name__):
        graphs = _generate(m, "llama", True)
    _same(eager, graphs)
    lines = [r.getMessage() for r in caplog.records if r.name == decode_graph.__name__]
    assert len(lines) == 1 and "the capture failed: RuntimeError" in lines[0], lines
    # the prefill, the eager first step, the failed capture, then an eager step for that step and every later one
    assert calls == [0, 7, 8, 8, 9, 10]
    assert decode_graph.current_graph(m).failed is not None
