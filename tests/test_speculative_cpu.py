"""Speculative decoding without a GPU: the iteration rule and both caches' invariant on a scripted model, speculative
output against ``greedy_search`` on tiny random models of every supported family, the prompt-lookup rule, the
acceptance mirror ``OF.spec_accept_ref`` against a loop written from the rule, every refusal, ``StaticKVCache.rollback``
and the decode-graph opt-in for steps of several tokens."""
import copy
from types import SimpleNamespace

import pytest
import torch
from torch import nn

from libai_b200.config import DictConfig
from libai_b200.inference import decode_graph
from libai_b200.inference.generator.generation_utils import _DEFAULTS, Generator, prompt_lookup
from libai_b200.inference.kv_cache import KVCacheOwner, StaticKVCache
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import MODELS, _prompt


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


V = 50


class Scripted(nn.Module, KVCacheOwner, Generator):
    """Logits are a table lookup: the token after ``tok`` at position ``pos`` of sample b is ``(7 tok + pos) % 40 + 3``,
    one more where ``pos + 1`` is in ``wrong[b]`` (a draft that is wrong there), or ``eos`` where ``(b, pos + 1)`` is in
    ``eos_at``.  Every step writes its token ids into the cache rows, so the rows can be checked."""

    speculative_decoding = True

    def __init__(self, wrong=((), ()), eos_at=(), max_positions=None, eos=None):
        super().__init__()
        self.cfg = DictConfig(dict(eos_token_id=eos, pad_token_id=0, bos_token_id=1))
        self.w = nn.Parameter(torch.zeros(1))
        self.wrong, self.eos_at, self.max_positions, self.eos = wrong, set(eos_at), max_positions, eos
        self.steps = []   # the new tokens of every call

    def allocate_kv_cache(self, batch, max_length):
        self.kv_cache = StaticKVCache(1, batch, 1, 1, max_length, torch.float32, "cpu")
        self.past_length = 0
        return self.kv_cache

    def forward(self, input_ids, attention_mask=None, use_cache=False):
        cache = self._prepare_cache(input_ids, max_positions=self.max_positions)
        cache.step_needs_dense_mask(attention_mask, flash=True)
        b, s = input_ids.shape
        p0 = cache.length
        self.steps.append(s)
        rows = input_ids.float().view(b, 1, s, 1)
        cache.write_rows(0, rows, rows, row0=p0)
        cache.advance(s)
        self.past_length = cache.length
        logits = torch.zeros(b, s, V)
        for i in range(b):
            for j in range(s):
                pos = p0 + j
                nxt = (7 * int(input_ids[i, j]) + pos) % 40 + 3
                if pos + 1 in self.wrong[i]:
                    nxt += 1
                if (i, pos + 1) in self.eos_at:
                    nxt = self.eos
                logits[i, j, nxt] = 10.0
        return {"logits": logits}


PROMPT = torch.tensor([[5, 6, 7, 8], [9, 10, 11, 12]])


class Recorder:
    """Records every iteration: n, and the lengths of both caches when the verify step starts (the invariant)."""

    def __init__(self, monkeypatch, target, draft=None):
        self.n, self.at_verify, self.blocks = [], [], []
        accept, verify = OF.spec_accept, Generator._verify_step

        def rec_accept(rows, proposals, unfinished, eos, pad):
            out = accept(rows, proposals, unfinished, eos, pad)
            self.n.append(int(out[0, 2 * rows.shape[1] + 1]))
            return out

        def rec_verify(model, block):
            c = model.kv_cache
            self.blocks.append(block.shape[1])
            self.at_verify.append((c.length, c.seqlens.tolist(), None if draft is None else
                                   (draft.kv_cache.length, draft.kv_cache.seqlens.tolist())))
            return verify(model, block)

        monkeypatch.setattr(OF, "spec_accept", rec_accept)
        monkeypatch.setattr(Generator, "_verify_step", rec_verify)


def _gen(m, **kw):
    return m.generate(PROMPT, max_length=19, output_scores=True, **kw)


def _same_scores(a, b, seq, eos, **tol):
    """Score rows equal where the sample has not finished: a finished sample's rows in the block where it emits EOS
    come from the proposals that follow it, greedy's from its pad tokens."""
    new = seq[:, seq.shape[1] - len(a):]
    done = torch.zeros(seq.shape[0], dtype=torch.bool)
    for j, (x, y) in enumerate(zip(a, b)):
        torch.testing.assert_close(x[~done], y[~done], **tol)
        if eos is not None:
            done |= new[:, j] == eos


def test_scripted_iterations_batch_minimum_and_cache_invariant(monkeypatch):
    target, draft = Scripted(), Scripted(wrong=({7, 12}, {9}))
    greedy = _gen(target)
    rec = Recorder(monkeypatch, target, draft)
    target.steps.clear()
    out = _gen(target, assistant_model=draft, num_assistant_tokens=3)
    assert torch.equal(out[0], greedy[0]) and len(out[1]) == len(greedy[1]) == 15
    assert all(torch.equal(a, b) for a, b in zip(out[1], greedy[1]))
    # sample 0's draft is wrong at position 7 and 12, sample 1's at 9: the batch advances by the minimum
    assert rec.n == [0, 2, 1, 2, 3, 3]
    # at every verify step each cache holds the sequence minus its last token (the target) plus the k proposals'
    # inputs (the draft): sequence lengths 5, 8, 10, 13, 17
    assert [a[0] for a in rec.at_verify] == [4, 7, 9, 12, 16]
    assert [a[1] for a in rec.at_verify] == [[4, 4], [7, 7], [9, 9], [12, 12], [16, 16]]
    assert [a[2][0] for a in rec.at_verify] == [7, 10, 12, 15, 19]
    assert [a[2][1] for a in rec.at_verify] == [[7, 7], [10, 10], [12, 12], [15, 15], [19, 19]]
    # the prompt, then 3 single-token draft steps per iteration and one catch-up after the n = k iteration (the 5th)
    assert draft.steps == [4] + [1] * 3 * 4 + [1] + [1] * 3
    assert target.steps == [4] + [4] * 5
    assert out[0].shape[1] == 19   # cut at max_length inside the last block (n + 1 = 4, 2 kept)


def test_scripted_cache_rows_are_the_sequence(monkeypatch):
    target, draft = Scripted(), Scripted(wrong=({7, 12}, {9}))
    seen = []
    verify = Generator._verify_step

    def check(model, block):
        c = model.kv_cache
        seen.append(c.k[0][:, 0, : c.length, 0].long().clone())
        return verify(model, block)

    monkeypatch.setattr(Generator, "_verify_step", check)
    out = _gen(target, assistant_model=draft, num_assistant_tokens=3)[0]
    for rows in seen:
        assert torch.equal(rows, out[:, : rows.shape[1]])


def test_scripted_eos_inside_an_accepted_block_and_finished_samples(monkeypatch):
    # sample 1 emits EOS (4) at position 6, inside a block the draft gets right, and then pads; it no longer limits n
    target = Scripted(eos_at={(1, 6)}, eos=4)
    draft = Scripted(wrong=({11}, {7, 8, 9, 10, 11}), eos_at={(1, 6)}, eos=4)
    greedy = _gen(target)
    rec = Recorder(monkeypatch, target, draft)
    out = _gen(target, assistant_model=draft, num_assistant_tokens=3)
    assert torch.equal(out[0], greedy[0]) and len(out[1]) == len(greedy[1])
    _same_scores(out[1], greedy[1], out[0], 4, atol=0, rtol=0)
    assert out[0][1, 6] == 4 and (out[0][1, 7:] == 0).all()
    assert rec.n[:3] == [0, 3, 2]


def test_scripted_stop_when_every_sample_finishes(monkeypatch):
    target = Scripted(eos_at={(0, 9), (1, 7)}, eos=4)
    draft = Scripted(eos_at={(0, 9), (1, 7)}, eos=4)
    greedy = _gen(target)
    out = _gen(target, assistant_model=draft, num_assistant_tokens=7)
    assert torch.equal(out[0], greedy[0]) and out[0].shape[1] == 10
    assert len(out[1]) == len(greedy[1]) == 6


def test_scripted_k_shrinks_at_the_position_limit(monkeypatch):
    # 14 positions: greedy's last step writes row 13; a verify step of k + 1 rows must stop there too
    target, draft = Scripted(max_positions=14), Scripted(max_positions=14)
    greedy = target.generate(PROMPT, max_length=14)
    rec = Recorder(monkeypatch, target, draft)
    out = target.generate(PROMPT, max_length=14, assistant_model=draft, num_assistant_tokens=7)
    assert torch.equal(out, greedy)
    assert rec.blocks == [8, 2]   # rows 4-11, then 12-19 would pass 14 at k = 7: the last step takes k = 1
    for (length, _, _), s in zip(rec.at_verify, rec.blocks):
        assert length + s <= 14
    pl = target.generate(PROMPT, max_length=14, prompt_lookup_num_tokens=7)
    assert torch.equal(pl, greedy)


# ------------------------------------------------------------------------------------------------ real families
def _llama_recipe(cls_path, **over):
    def build():
        import importlib

        from libai_b200.layers._param import param_defaults
        from tests.test_cached_attention_cpu import LLAMA

        module, name = cls_path.rsplit(".", 1)
        cls = getattr(importlib.import_module(module), name)
        with param_defaults(dtype=torch.bfloat16, device="cpu", seed=0):
            m = cls(DictConfig(dict(LLAMA, **over))).eval()
        if hasattr(m.model.layers[0].self_attn, "gate"):   # LLaMA-Adapter: a fresh model's zero gates add nothing
            with torch.no_grad():
                for layer in m.model.layers:
                    gate = layer.self_attn.gate
                    gate.copy_(torch.linspace(0.5, 2.0, gate.numel()).view_as(gate))
        return m
    return build


BUILDERS = dict(MODELS)
BUILDERS.update(
    qwen=_llama_recipe("projects.Qwen.qwen2.Qwen2ForCausalLM", qkv_bias=True),
    baichuan=_llama_recipe("projects.Baichuan.baichuan.BaichuanForCausalLM"),
    aquila=_llama_recipe("projects.Aquila.aquila.AquilaForCausalLM"),
    llama_adapter=_llama_recipe("projects.Llama.adapter.adapter_model.LlamaForCausalLM", hidden_size=256,
                                num_attention_heads=4, adapter_len=4, adapter_layer=2),
)
FAMILIES = ["llama", "llama_gqa", "gpt2", "bloom", "chatglm", "chatglm_prefix", "qwen", "baichuan", "aquila",
            "llama_adapter"]
PADDED = ("llama", "llama_gqa", "bloom", "chatglm", "qwen", "baichuan", "aquila", "llama_adapter")


def _verify_rounding(m, ids, am, seq, k):
    """The largest logit difference between a (k + 1)-token cached step and k + 1 single-token steps after the prompt
    of the greedy sequence ``seq``."""
    P = ids.shape[1]
    mask = {} if am is None else {"attention_mask": am}
    with torch.no_grad():
        m.allocate_kv_cache(ids.shape[0], seq.shape[1] + 1)
        m(seq[:, :P], use_cache=True, **mask)
        one = torch.cat([m(seq[:, P + i : P + i + 1], use_cache=True)["logits"] for i in range(k + 1)], 1)
        m.allocate_kv_cache(ids.shape[0], seq.shape[1] + 1)
        m(seq[:, :P], use_cache=True, **mask)
        block = m(seq[:, P : P + k + 1], use_cache=True)["logits"]
        m._reset_cache()
    return (one - block).abs().max().item()


def _check_family(name, case, dtype):
    if case == "left_padded" and name not in PADDED:
        pytest.skip("the model takes no padding mask (GPT-2), or pads behind its prefix with a dense mask")
    m = BUILDERS[name]().to(dtype)
    same = copy.deepcopy(m)
    other = BUILDERS[name]().to(dtype)
    with torch.no_grad():
        for p in other.parameters():
            p.add_(torch.randn(p.shape, generator=torch.Generator().manual_seed(9)).to(p.dtype) * 0.05)
    ids, am = _prompt("plain" if case == "batch1" else case)
    if case == "batch1":
        ids = ids[:1]
    kw = dict(eos_token_id=None, output_scores=True, max_length=ids.shape[1] + 12)
    if am is not None:
        kw["attention_mask"] = am
    greedy = m.generate(ids, **kw)
    top2 = torch.stack(greedy[1]).topk(2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1]).min().item()
    for k in (1, 3, 7):
        diff = _verify_rounding(m, ids, am, greedy[0], k)
        assert margin > 100 * max(diff, 1e-6), (margin, diff)   # no compared position is a near-tie
        for spec in (dict(assistant_model=same, num_assistant_tokens=k), dict(assistant_model=other,
                                                                              num_assistant_tokens=k),
                     dict(prompt_lookup_num_tokens=k)):
            out = m.generate(ids, **kw, **spec)
            assert torch.equal(out[0], greedy[0]), (k, spec.keys())
            assert len(out[1]) == len(greedy[1])
            tol = 1e-4 if dtype == torch.float32 else 1e-6   # fp64 models keep fp32 rotary tables
            _same_scores(out[1], greedy[1], out[0], m._gcfg("eos_token_id"), atol=tol, rtol=tol)


@pytest.mark.parametrize("case", ["plain", "left_padded", "batch1"])
@pytest.mark.parametrize("name", FAMILIES)
def test_families_equal_greedy(name, case):
    _check_family(name, case, torch.float32)


@pytest.mark.parametrize("name", ["llama", "gpt2", "bloom", "chatglm"])
def test_families_equal_greedy_fp64(name):
    _check_family(name, "left_padded" if name != "gpt2" else "plain", torch.float64)


def test_prompt_at_max_length_emits_one_token_as_greedy():
    target, draft = Scripted(), Scripted(wrong=({7}, {9}))
    for max_length in (2, 4):
        greedy = target.generate(PROMPT, max_length=max_length)
        assert greedy.shape[1] == 5
        assert torch.equal(target.generate(PROMPT, max_length=max_length, assistant_model=draft), greedy)
        assert torch.equal(target.generate(PROMPT, max_length=max_length, prompt_lookup_num_tokens=3), greedy)


def test_batch_one_and_the_model_state_is_restored():
    m, d = MODELS["llama"]().float(), MODELS["llama"]().float()
    m.train(), d.train()
    ids, _ = _prompt("plain")
    greedy = m.generate(ids[:1], max_length=15, eos_token_id=None)
    out = m.generate(ids[:1], max_length=15, eos_token_id=None, assistant_model=d, num_assistant_tokens=3,
                     decode_graphs=True)
    assert torch.equal(out, greedy)
    assert m.training and d.training and m._decode_graphs is None and d._decode_graphs is None
    assert m.kv_cache_dtype is None and d.kv_cache_dtype is None


# ------------------------------------------------------------------------------------------------ prompt lookup
def _lookup_rule(seq, k, N):
    L = len(seq)
    for n in range(N, 0, -1):
        if n >= L:
            continue
        for i in range(0, L - n):
            if seq[i : i + n] == seq[L - n :] and i + n < L:
                cont = seq[i + n : i + n + k]
                return cont + [cont[-1]] * (k - len(cont))
    return [seq[-1]] * k


@pytest.mark.parametrize("seq,k,N,want", [
    ([1, 2, 3, 4], 3, 2, [4, 4, 4]),                      # no match: x repeated
    ([1, 2, 3, 1, 2], 3, 2, [3, 1, 2]),                   # a bigram at the start
    ([1, 2, 3, 4, 2], 4, 2, [3, 4, 2, 2]),                # a unigram, short continuation padded
    ([5, 1, 2, 9, 1, 2, 7, 1, 2], 2, 2, [9, 1]),          # the earliest of several
    ([3, 3], 2, 3, [3, 3]),                               # the match's continuation is the tail itself
    ([7, 8, 7], 5, 1, [8, 7, 7, 7, 7]),                   # a continuation that reaches the end
])
def test_prompt_lookup_rule(seq, k, N, want):
    assert prompt_lookup(seq, k, N) == want == _lookup_rule(seq, k, N)


def test_prompt_lookup_random_sequences():
    g = torch.Generator().manual_seed(0)
    for _ in range(300):
        L = int(torch.randint(1, 20, (1,), generator=g))
        seq = torch.randint(0, 4, (L,), generator=g).tolist()
        k, N = int(torch.randint(1, 8, (1,), generator=g)), int(torch.randint(1, 4, (1,), generator=g))
        assert prompt_lookup(seq, k, N) == _lookup_rule(seq, k, N)


# ------------------------------------------------------------------------------------------------ the acceptance mirror
def _accept_loop(logits, draft, unfinished, eos, pad):
    b, R, _ = logits.shape
    k = R - 1
    t = [[int(torch.argmax(logits[i, j])) for j in range(R)] for i in range(b)]
    a = []
    for i in range(b):
        m = 0
        while m < k and int(draft[i, m]) == t[i][m]:
            m += 1
        a.append(m)
    limits = [k if eos is not None and eos in t[i][: a[i] + 1] else a[i] for i in range(b) if unfinished[i]]
    n = min(limits) if limits else k
    rows = []
    for i in range(b):
        u, e = int(unfinished[i]), []
        for j in range(R):
            if j > n:
                e.append(-1)
                continue
            tok = t[i][j] if eos is None or u else pad
            if eos is not None and tok == eos:
                u = 0
            e.append(tok)
        rows.append(t[i] + e + [a[i], n, u])
    return torch.tensor(rows)


@pytest.mark.parametrize("eos", [None, 3])
def test_spec_accept_ref_against_the_rule(eos):
    g = torch.Generator().manual_seed(1)
    for trial in range(200):
        b, k, Vv = int(torch.randint(1, 6, (1,), generator=g)), int(torch.randint(0, 8, (1,), generator=g)), 6
        logits = torch.randint(0, 3, (b, k + 1, Vv), generator=g).float()   # many ties
        if trial % 7 == 0:
            logits[0, 0] = float("-inf")
        t = logits.argmax(-1)
        draft = torch.where(torch.rand(b, k, generator=g) < 0.8, t[:, :k], torch.randint(0, Vv, (b, k), generator=g))
        unfinished = (torch.rand(b, generator=g) < 0.7).long()
        want = _accept_loop(logits, draft, unfinished, eos, 0)
        u = unfinished.clone()
        got = OF.spec_accept(logits, draft, u, eos, 0)   # CPU: the mirror
        assert torch.equal(got, want)
        assert torch.equal(u, want[:, -1])


def test_spec_accept_needs_pad_with_eos():
    with pytest.raises(ValueError, match="pad"):
        OF.spec_accept(torch.zeros(1, 2, 5), torch.zeros(1, 1, dtype=torch.long), torch.ones(1, dtype=torch.long), 2,
                       None)


# ------------------------------------------------------------------------------------------------ refusals
def test_defaults():
    for key in ("assistant_model", "num_assistant_tokens", "prompt_lookup_num_tokens", "max_matching_ngram_size"):
        assert key in _DEFAULTS and _DEFAULTS[key] is None


class _NoSpec(Scripted):
    speculative_decoding = False


REFUSALS = {
    "both": (dict(prompt_lookup_num_tokens=2, draft=True), "assistant_model and prompt_lookup_num_tokens"),
    "k0": (dict(prompt_lookup_num_tokens=0), "prompt_lookup_num_tokens"),
    "k16": (dict(num_assistant_tokens=16, draft=True), "num_assistant_tokens"),
    "ngram": (dict(prompt_lookup_num_tokens=2, max_matching_ngram_size=0), "max_matching_ngram_size"),
    "sample": (dict(prompt_lookup_num_tokens=2, do_sample=True), "do_sample"),
    "beams": (dict(prompt_lookup_num_tokens=2, num_beams=2), "num_beams"),
    "return": (dict(prompt_lookup_num_tokens=2, num_return_sequences=2), "num_return_sequences"),
    "penalty": (dict(prompt_lookup_num_tokens=2, repetition_penalty=1.2), "repetition_penalty"),
    "processor": (dict(prompt_lookup_num_tokens=2, logits_processor=[lambda i, s: s]), "logits_processor"),
    "prefix_fn": (dict(prompt_lookup_num_tokens=2, prefix_allowed_tokens_fn=lambda b, i: [1]),
                  "prefix_allowed_tokens_fn"),
    "criteria": (dict(prompt_lookup_num_tokens=2, stopping_criteria=[lambda i, s: False]), "stopping_criteria"),
    "use_cache": (dict(prompt_lookup_num_tokens=2, use_cache=False), "use_cache"),
    "self": (dict(num_assistant_tokens=2, draft="self"), "assistant_model must be another model"),
    "unsupported": (dict(num_assistant_tokens=2, draft="nospec"), "assistant_model"),
    "dense": (dict(prompt_lookup_num_tokens=2, attention_mask=torch.tensor([[1, 0, 1, 1], [1, 1, 1, 1]])),
              "attention_mask"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_each_refusal_names_its_argument(case):
    kw, fragment = REFUSALS[case]
    kw = dict(kw)
    m = Scripted()
    draft = kw.pop("draft", None)
    if draft is not None:
        kw["assistant_model"] = m if draft == "self" else _NoSpec() if draft == "nospec" else Scripted()
    with pytest.raises(ValueError, match=fragment):
        m.generate(PROMPT, max_length=10, **kw)


def test_refusals_of_models_and_parallelism(monkeypatch):
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens: the model"):
        _NoSpec().generate(PROMPT, max_length=10, prompt_lookup_num_tokens=2)
    t5 = MODELS["t5"]()
    ids, _ = _prompt("plain")
    with pytest.raises(ValueError, match="encoder-decoder"):
        t5.generate(ids, max_length=6, prompt_lookup_num_tokens=2)
    monkeypatch.setattr(dist, "get_dist_util", lambda: SimpleNamespace(tensor_parallel_size=2, pipeline_parallel_size=1,
                                                                       device=torch.device("cpu")))
    with pytest.raises(ValueError, match="tensor- or pipeline-parallel"):
        Scripted().generate(PROMPT, max_length=10, prompt_lookup_num_tokens=2)


def test_glm_is_refused():
    from projects.GLM.modeling_glm import GLMForConditionalGeneration

    assert not GLMForConditionalGeneration.speculative_decoding


# ------------------------------------------------------------------------------------------------ cache and graphs
def test_rollback():
    c = StaticKVCache(1, 2, 1, 4, 10, torch.float32, "cpu")
    c.advance(7)
    c.rollback(3)
    assert c.length == 4 and c.seqlens.tolist() == [4, 4]
    c.rollback(0)
    assert c.length == 4
    with pytest.raises(ValueError, match="rollback"):
        c.rollback(5)


def _fake_graph_model(monkeypatch, length=5):
    monkeypatch.setattr(decode_graph, "use_native", lambda *t: True)
    c = StaticKVCache(2, 3, 2, 64, 32, torch.bfloat16, "meta")
    c.device, c.length = torch.device("cuda", 0), length
    return SimpleNamespace(kv_cache=c, max_cache_positions=None, past_length=length)


def test_decode_graph_opt_in_for_several_tokens(monkeypatch):
    model = _fake_graph_model(monkeypatch)
    ids = {"input_ids": torch.ones(3, 4, dtype=torch.long), "use_cache": True}
    assert "more than one new token" in decode_graph.fallback_reason(model, ids)
    assert decode_graph.fallback_reason(model, ids, tokens=4) is None
    assert "not 5 new tokens" in decode_graph.fallback_reason(model, ids, tokens=5)
    model.max_cache_positions = 8
    assert "maximum length" in decode_graph.fallback_reason(model, ids, tokens=4)
    model.max_cache_positions, model.kv_cache.length = None, 29
    assert "must grow" in decode_graph.fallback_reason(model, ids, tokens=4)
    with pytest.raises(ValueError, match="tokens"):
        decode_graph.step(model, ids, decode_graph.DecodeCall(), tokens=17)


def test_a_replay_advances_by_the_step_tokens(monkeypatch):
    model = _fake_graph_model(monkeypatch)
    ids = {"input_ids": torch.ones(3, 4, dtype=torch.long)}
    g = decode_graph.DecodeGraph(None, ids, tokens=4)
    g.graph = SimpleNamespace(replay=lambda: None)
    g.outputs = {"logits": torch.zeros(3, 4, 5)}
    g.replay(model, ids)
    assert model.kv_cache.length == 9 and model.past_length == 9
