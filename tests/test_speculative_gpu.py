"""Speculative decoding on the H100: the acceptance kernel equals its PyTorch mirror bit for bit (ties, −inf rows, EOS at
every block position, finished samples, k 1..15, b 1..16, bf16 and fp32 logits, three vocabulary sizes, launches on
several streams) and checks its arguments; a replayed iteration runs no model Python, launches only the graph
replays and the acceptance kernel among the native kernels, and syncs once; ``generate()`` with decode graphs gives the tokens and scores of eager speculative decoding bit for bit on
every supported family, bf16 and FP8 caches, FP8 and INT4 weights on either model and both proposers; the tokens equal
plain greedy decoding wherever greedy's top-2 margin is far above the verify step's rounding; and the cache rows left
behind are those a prefill of the final sequence writes."""
import copy
import warnings

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200 import ops
from libai_b200.inference import decode_graph, quantize_weights_fp8_, quantize_weights_int4_
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import MODELS, _prompt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FAMILIES = ["llama", "llama_gqa", "gpt2", "bloom", "chatglm", "chatglm_prefix"]
PADDED = ("llama", "llama_gqa", "bloom", "chatglm")


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


# ------------------------------------------------------------------------------------------------ the kernel
def _case(b, k, V, dtype, seed, eos_pos=None, finished=False, ninf=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    logits = torch.randint(0, 4, (b, k + 1, V), device=DEV, generator=g).to(dtype)   # many exact ties
    logits += torch.randn(b, k + 1, V, device=DEV, generator=g).to(dtype) * (seed % 2)
    if ninf:
        logits[0, 0] = float("-inf")
        logits[-1, k, : V // 2] = float("-inf")
    t = logits.float().argmax(-1)
    draft = t[:, :k].clone()
    wrong = torch.rand(b, k, device=DEV, generator=g) < 0.15
    draft[wrong] = (draft[wrong] + 1) % V
    eos = 7
    if eos_pos is not None:   # EOS as the target's token at that block position of sample 0
        logits[0, eos_pos] = -1e4
        logits[0, eos_pos, eos] = 1e4
        draft[0, :eos_pos] = logits[0, :eos_pos].float().argmax(-1)
    unfinished = torch.zeros(b, dtype=torch.long, device=DEV) if finished else \
        (torch.rand(b, device=DEV, generator=g) < 0.8).long()
    return logits, draft, unfinished, eos


def _both(logits, draft, unfinished, eos, pad=0):
    u1, u2 = unfinished.clone(), unfinished.clone()
    got = OF.spec_accept(logits, draft, u1, eos, pad)
    want = OF.spec_accept_ref(logits, draft, u2, eos, pad)
    assert torch.equal(got, want)
    assert torch.equal(u1, u2)
    return got


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("V", [32000, 50257, 65024])
def test_kernel_equals_the_mirror(V, dtype):
    seed = 0
    for k in range(1, 16):
        for b in (1, 2, 5, 16):
            seed += 1
            for eos in (None, 7):
                logits, draft, unfinished, _ = _case(b, k, V, dtype, seed, ninf=seed % 3 == 0)
                _both(logits, draft, unfinished, eos)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_kernel_eos_at_every_position_and_all_finished(dtype):
    for k in (1, 4, 15):
        for pos in range(k + 1):
            logits, draft, unfinished, eos = _case(3, k, 32000, dtype, 100 + pos, eos_pos=pos)
            unfinished[0] = 1
            out = _both(logits, draft, unfinished, eos)
            assert out[0, pos] == eos
        logits, draft, unfinished, eos = _case(4, k, 50257, dtype, 7, finished=True)
        out = _both(logits, draft, unfinished, eos)
        assert (out[:, 2 * (k + 1) + 1] == k).all()   # nothing unfinished: n = k
        assert (out[:, k + 1 : 2 * (k + 1)] == 0).all()   # every token is pad


def test_kernel_is_deterministic_and_launches_on_other_streams_do_not_interfere():
    logits, draft, unfinished, eos = _case(16, 15, 65024, torch.bfloat16, 3)
    outs = [OF.spec_accept(logits, draft, unfinished.clone(), eos, 0) for _ in range(20)]
    assert all(torch.equal(o, outs[0]) for o in outs)
    streams = [torch.cuda.Stream() for _ in range(4)]
    got = []
    torch.cuda.synchronize()
    for st in streams * 5:   # every launch counts its blocks on a counter of its own
        with torch.cuda.stream(st):
            got.append(OF.spec_accept(logits, draft, unfinished.clone(), eos, 0))
    torch.cuda.synchronize()
    assert all(torch.equal(o, outs[0]) for o in got)


def test_kernel_argument_checks():
    from libai_b200 import ops

    ext = ops.load_ext(required=True)
    ok = dict(logits=torch.zeros(2, 4, 100, dtype=torch.bfloat16, device=DEV),
              draft=torch.zeros(2, 3, dtype=torch.long, device=DEV),
              unfinished=torch.ones(2, dtype=torch.long, device=DEV))
    assert ext.spec_accept(ok["logits"], ok["draft"], ok["unfinished"], 2, 0).shape == (2, 11)
    bad = {
        "logits": [ok["logits"].half(), torch.zeros(2, 4, 200, dtype=torch.bfloat16, device=DEV)[..., ::2],
                   ok["logits"].cpu(), torch.zeros(2, 17, 100, dtype=torch.bfloat16, device=DEV)],
        "draft": [ok["draft"].int(), ok["draft"][:, :2], ok["draft"].cpu()],
        "unfinished": [ok["unfinished"].int(), ok["unfinished"][:1], ok["unfinished"].cpu()],
    }
    for name, variants in bad.items():
        for v in variants:
            args = dict(ok, **{name: v})
            if name == "logits" and v.shape[1] == 17:
                args["draft"] = torch.zeros(2, 16, dtype=torch.long, device=DEV)
            with pytest.raises(RuntimeError, match="spec_accept"):
                ext.spec_accept(args["logits"], args["draft"], args["unfinished"], 2, 0)


# ------------------------------------------------------------------------------------------------ generate()
def _model(name, weights=None):
    m = MODELS[name]().to(DEV)
    if weights == "fp8":
        m = quantize_weights_fp8_(m)
    elif weights == "int4":
        m = quantize_weights_int4_(m)
    return m


def _other(name):
    m = MODELS[name]()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn(p.shape, generator=torch.Generator().manual_seed(9)).to(p.device, p.dtype) * 0.05)
    return m.to(DEV)


def _generate(m, name, case, graphs, **kw):
    ids, am = _prompt(case)
    ids = ids.to(DEV)
    kw = dict(eos_token_id=None, output_scores=True, max_length=ids.shape[1] + 16, decode_graphs=graphs, **kw)
    if am is not None:
        kw["attention_mask"] = am.to(DEV)
    with torch.no_grad():
        return m.generate(ids, **kw)


def _same(a, b):
    assert torch.equal(a[0], b[0])
    assert len(a[1]) == len(b[1]) and all(torch.equal(x, y) for x, y in zip(a[1], b[1]))


def _captured(*models):
    """Each model's decode graph was captured (a failed capture would leave eager steps behind)."""
    for mm in models:
        g = decode_graph.current_graph(mm)
        assert g is not None and g.graph is not None and g.failed is None, type(mm).__name__


@pytest.mark.parametrize("kv", [None, "fp8"])
@pytest.mark.parametrize("proposer", ["assistant", "lookup"])
@pytest.mark.parametrize("name", FAMILIES)
def test_graphs_equal_eager(name, proposer, kv):
    m = _model(name)
    for case in ("plain", "left_padded") if name in PADDED else ("plain",):
        for k in (3, 7):
            spec = dict(prompt_lookup_num_tokens=k) if proposer == "lookup" else \
                dict(assistant_model=_other(name), num_assistant_tokens=k)
            eager = _generate(m, name, case, False, kv_cache_dtype=kv, **spec)
            graphs = _generate(m, name, case, True, kv_cache_dtype=kv, **spec)
            _same(eager, graphs)
            _captured(m, *([spec["assistant_model"]] if proposer == "assistant" else []))


@pytest.mark.parametrize("target_w,draft_w", [("fp8", None), ("int4", None), (None, "fp8"), (None, "int4"),
                                              ("int4", "fp8")])
def test_quantized_weights_graphs_equal_eager(target_w, draft_w):
    m, d = _model("llama_gqa", target_w), _model("llama_gqa", draft_w)
    for case in ("plain", "left_padded"):
        eager = _generate(m, "llama_gqa", case, False, assistant_model=d, num_assistant_tokens=4)
        graphs = _generate(m, "llama_gqa", case, True, assistant_model=d, num_assistant_tokens=4)
        _same(eager, graphs)
    d.cfg.kv_cache_dtype = "fp8"   # the assistant's own cache format
    _same(_generate(m, "llama_gqa", "plain", False, assistant_model=d, num_assistant_tokens=4),
          _generate(m, "llama_gqa", "plain", True, assistant_model=d, num_assistant_tokens=4))
    _captured(m, d)


def _verify_rounding(m, seq, P, am, k):
    """The largest logit difference between a (k + 1)-token cached step and k + 1 single-token steps, over every block
    start of the greedy sequence ``seq`` after the prompt of ``P`` tokens."""
    worst = 0.0
    kw = {} if am is None else {"attention_mask": am}
    with torch.no_grad():
        for start in range(P, seq.shape[1] - k, k + 1):
            m.allocate_kv_cache(seq.shape[0], seq.shape[1] + 1)
            m(seq[:, :P], use_cache=True, **kw)
            if start > P:
                m(seq[:, P:start], use_cache=True)
            block = m(seq[:, start : start + k + 1], use_cache=True)["logits"].float()
            m.allocate_kv_cache(seq.shape[0], seq.shape[1] + 1)
            m(seq[:, :P], use_cache=True, **kw)
            if start > P:
                m(seq[:, P:start], use_cache=True)
            one = torch.cat([m(seq[:, i : i + 1], use_cache=True)["logits"].float()
                             for i in range(start, start + k + 1)], 1)
            worst = max(worst, (one - block).abs().max().item())
        m._reset_cache()
    return worst


@pytest.mark.parametrize("name", FAMILIES)
def test_tokens_equal_greedy_up_to_a_near_tie(name):
    m = _model(name)
    same = copy.deepcopy(m)   # a draft with the target's weights (copied before any graph exists)
    compared = 0
    for case in ("plain", "left_padded") if name in PADDED else ("plain",):
        ids, am = _prompt(case)
        am = None if am is None else am.to(DEV)
        greedy = _generate(m, name, case, True)
        P = ids.shape[1]
        top2 = torch.stack(greedy[1]).topk(2, dim=-1).values   # [steps, b, 2]
        margin = (top2[..., 0] - top2[..., 1]).min(dim=1).values   # the batch's smallest, per step
        for k in (1, 3, 7):
            diff = _verify_rounding(m, greedy[0], P, am, k)
            near = (margin < 4 * diff).nonzero()
            stop = int(near[0]) if len(near) else len(greedy[1])
            for spec in (dict(prompt_lookup_num_tokens=k), dict(assistant_model=same, num_assistant_tokens=k)):
                out = _generate(m, name, case, True, **spec)
                assert torch.equal(out[0][:, : P + stop], greedy[0][:, : P + stop]), (case, k, stop)
                compared += stop
    print(f"{name}: {compared} positions compared")
    assert compared >= 60


@pytest.mark.parametrize("name", ["llama_gqa", "chatglm"])
def test_cache_rows_after_generate_match_a_prefill(name):
    m = _model(name)
    twin = copy.deepcopy(m)
    d = _other(name)
    ids, _ = _prompt("plain")
    ids = ids.to(DEV)
    with torch.no_grad():
        out = m.generate(ids, max_length=ids.shape[1] + 13, eos_token_id=None, assistant_model=d,
                         num_assistant_tokens=3, decode_graphs=True)
        c = m.kv_cache
        L = out.shape[1] - 1   # the rows of every token but the last (the cache keeps its buffers after generate)
        got = [(c.k[i][:, :, :L].clone(), c.v[i][:, :, :L].clone()) for i in c.owned]
        twin.allocate_kv_cache(ids.shape[0], out.shape[1] + 1)
        twin(out[:, :-1], use_cache=True)
        tc = twin.kv_cache
        for i, (k, v) in zip(tc.owned, got):
            torch.testing.assert_close(k.float(), tc.k[i][:, :, :L].float(), atol=3e-2, rtol=3e-2)
            torch.testing.assert_close(v.float(), tc.v[i][:, :, :L].float(), atol=3e-2, rtol=3e-2)


@pytest.mark.parametrize("proposer", ["assistant", "lookup"])
def test_replayed_iteration_launches_the_graphs_and_syncs_once(monkeypatch, proposer):
    """Between two acceptance calls after the warm-up (the verify graph is captured in the second iteration, the
    draft's in the first) an iteration runs no model Python; its native launches are the replayed graphs' (the draft's
    k steps, one more after an iteration that accepted all k, and the verify step) and the acceptance kernel; and the
    host syncs once, on the readback."""
    m = _model("llama_gqa")
    d = _other("llama_gqa") if proposer == "assistant" else None
    k = 4
    spec = dict(assistant_model=d, num_assistant_tokens=k) if d is not None else dict(prompt_lookup_num_tokens=k)
    marks, outs, forwards = [], [], [0]
    accept = OF.spec_accept
    caught = []

    def recorded(rows, proposals, unfinished, eos, pad):
        syncs = sum("synchroniz" in str(w.message) for w in caught)
        marks.append((ops.launch_count(), syncs, forwards[0]))
        out = accept(rows, proposals, unfinished, eos, pad)
        outs.append(out)
        return out

    forward = type(m).forward

    def counted(self, *a, **kw):
        forwards[0] += 1
        return forward(self, *a, **kw)

    monkeypatch.setattr(OF, "spec_accept", recorded)
    monkeypatch.setattr(type(m), "forward", counted)
    ids, _ = _prompt("plain")
    ids = ids.to(DEV)
    with warnings.catch_warnings(record=True) as caught_now:
        warnings.simplefilter("always")
        caught = caught_now
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with torch.no_grad():
                m.generate(ids, max_length=ids.shape[1] + 40, eos_token_id=None, decode_graphs=True, **spec)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    verify = decode_graph.current_graph(m)
    assert verify.graph is not None and verify.failed is None and verify.tokens == k + 1
    step = 0
    if d is not None:
        draft = decode_graph.current_graph(d)
        assert draft.graph is not None and draft.failed is None and draft.tokens == 1
        step = draft.launches
    R = k + 1
    checked = 0
    for j in range(2, len(marks) - 1):   # the interval from acceptance j to j + 1 replays the verify step of j + 1
        launches = marks[j + 1][0] - marks[j][0]
        catch_up = d is not None and int(outs[j][0, 2 * R + 1]) == k
        assert launches == 1 + verify.launches + (k + catch_up) * step, (j, launches)
        assert marks[j + 1][1] - marks[j][1] == 1, j   # the readback
        assert marks[j + 1][2] == marks[j][2], j       # no model forward ran
        checked += 1
    assert checked >= 5
