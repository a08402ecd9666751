"""Speculative sampling on the H100: both sampling kernels against their fp64 mirrors (bf16 and fp32 logits, three
vocabulary sizes, b 1..16, k 1..15, four warps), equal except on decisions the mirror flags as within
``OF.SPEC_SAMPLE_MARGIN`` of a boundary, which must be rare and still valid; bit-identical results alone or in a batch,
on repeat launches and on several streams; the kernels' output distribution (chi-square, acceptance rate); and
``generate(do_sample=True, assistant_model=...)``: eager against decode graphs bit for bit on every supported family,
bf16 and FP8 caches and FP8/INT4 weights, one sync per replayed iteration, top_k=1 against greedy speculative decoding,
the acceptance of an exact copy, and the first two tokens' distributions."""
import copy
import warnings

import numpy as np
import pytest
import torch
from scipy import stats

from libai_b200 import ops
from libai_b200.config import DictConfig
from libai_b200.inference import decode_graph, quantize_weights_fp8_, quantize_weights_int4_
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import MODELS, _prompt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FAMILIES = ["llama", "llama_gqa", "gpt2", "bloom", "chatglm", "chatglm_prefix"]
WARPS = {"T": (0.7, 0, 1.0), "topk": (1.0, 50, 1.0), "topp": (1.0, 0, 0.8), "both": (0.8, 50, 0.8)}
# flagged rows, at most: 1 % over the full grids of 5610 rows (measured 0.1-0.3 %), 5 % over the 231 rows of the
# 250880-token subset (measured 0 and 3 %)
FLAG_BOUND = {32000: 0.01, 65024: 0.01, 250880: 0.05}


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


# ------------------------------------------------------------------------------------------------ the kernels
def _rows(shape, dtype, g, scale=2.0):
    """LM-like logits: a random tail and a head of 16 tokens per row raised by 8 to 14, which holds most of the mass
    (a flat row of 250880 tokens puts thousands of masses below the margin at a top-p boundary)."""
    x = torch.randn(*shape, device=DEV, generator=g) * scale
    head = torch.randint(0, shape[-1], (*shape[:-1], 16), device=DEV, generator=g)
    x.scatter_add_(-1, head, 8 + 6 * torch.rand(*shape[:-1], 16, device=DEV, generator=g))
    return x.to(dtype)


def _case(b, k, V, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    logits = _rows((b, k + 1, V), dtype, g)
    q = (logits.float()[:, :k] + torch.randn(b, k, V, device=DEV, generator=g) * 0.5).to(dtype)   # a close draft
    u = torch.rand(b, k + 1, 2, device=DEV, generator=g)
    ud = torch.rand(b, k, device=DEV, generator=g)
    unfinished = (torch.rand(b, device=DEV, generator=g) < 0.8).long()
    return logits, q, u, ud, unfinished


def _valid(row, tok, warp):
    """tok is a choice of the warped row when top_p is widened past the margin."""
    T, tk, tp = warp
    wide = OF.spec_warp_ref(row, T, tk, min(1.0, tp + 1e-3))
    return bool(wide[tok] > float("-inf"))


def _check_case(b, k, V, dtype, seed, warp, stats_):
    T, tk, tp = warp
    logits, qsrc, u, ud, unfinished = _case(b, k, V, dtype, seed)
    # the draft kernel: k steps on q's rows
    qk, qr = torch.empty_like(qsrc), torch.empty_like(qsrc)
    pk, pr = torch.empty(b, k, dtype=torch.long, device=DEV), torch.empty(b, k, dtype=torch.long, device=DEV)
    for j in range(k):
        row = qsrc[:, j].contiguous()
        OF.spec_sample(row, qk, j, ud, pk, T, tk, tp)
        near = OF.spec_sample_ref(row, qr, j, ud, pr, T, tk, tp, flags=True)
        same = pk[:, j] == pr[:, j]
        assert bool((same | near).all()), (seed, j)
        stats_["rows"] += b
        stats_["flagged"] += int(near.sum())
        for i in (~same).nonzero()[:, 0].tolist():
            assert _valid(row[i], int(pk[i, j]), warp)
    assert torch.equal(qk, qsrc)
    draft = pk
    # the acceptance kernel
    uk, ur = unfinished.clone(), unfinished.clone()
    sk = torch.empty(b, k + 1, V, device=DEV)
    sr = torch.empty_like(sk)
    out = OF.spec_accept_sample(logits, qk, draft, u, uk, T, tk, tp, 7, 0, sk)
    ref, near = OF.spec_accept_sample_ref(logits, qk, draft, u, ur, T, tk, tp, 7, 0, sr, flags=True)
    stats_["rows"] += b * (k + 1)
    stats_["flagged"] += int(near.sum())
    R = k + 1
    clean = ~near.any(dim=1)
    # every row's warped scores: equal where the top-p boundary is clear
    torch.testing.assert_close(sk[clean], sr[clean], atol=0, rtol=0)
    if bool(clean.all()):
        assert torch.equal(out, ref), seed
        assert torch.equal(uk, ur)
    else:   # the unflagged samples' own decisions agree; the flagged ones are valid choices
        cols = list(range(R)) + [2 * R]
        assert torch.equal(out[clean][:, cols], ref[clean][:, cols]), seed
        for i in (~clean).nonzero()[:, 0].tolist():
            a = int(out[i, 2 * R])
            for j in range(min(a + 1, R)):
                assert _valid(logits[i, j], int(out[i, j]), warp) or j < a
    return out


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("V", [32000, 65024, 250880])
def test_kernels_equal_the_mirrors(V, dtype):
    stats_ = dict(rows=0, flagged=0)
    seed = 0
    names = sorted(WARPS)
    for k in range(1, 16):
        for b in (1, 5, 16):
            seed += 1
            if V == 250880 and (b, k % 5) != (5, 1) and not (b == 1 and k in (2, 15)):
                continue   # the largest vocabulary: a subset, for time
            _check_case(b, k, V, dtype, seed, WARPS[names[seed % 4]], stats_)
    rate = stats_["flagged"] / stats_["rows"]
    print(f"V={V} {dtype}: {stats_['flagged']} of {stats_['rows']} rows flagged ({rate:.4f})")
    assert rate <= FLAG_BOUND[V]


def test_batch_invariance_repeats_and_streams():
    b, k, V = 16, 7, 65024
    T, tk, tp = WARPS["both"]
    logits, q, u, _, unfinished = _case(b, k, V, torch.bfloat16, 11)
    draft = torch.randint(0, V, (b, k), device=DEV)
    draft[:, :3] = logits[:, :3].float().argmax(-1)
    R = k + 1
    full = OF.spec_accept_sample(logits, q, draft, u, unfinished.clone(), T, tk, tp, None, None)
    for i in (0, 9, 15):   # a sample alone: its tokens and a_b are those it has in the batch
        alone = OF.spec_accept_sample(logits[i : i + 1].contiguous(), q[i : i + 1].contiguous(), draft[i : i + 1],
                                      u[i : i + 1].contiguous(), unfinished[i : i + 1].clone(), T, tk, tp, None, None)
        cols = list(range(R)) + [2 * R]
        assert torch.equal(alone[0, cols], full[i, cols])
    outs = [OF.spec_accept_sample(logits, q, draft, u, unfinished.clone(), T, tk, tp, None, None) for _ in range(10)]
    assert all(torch.equal(o, full) for o in outs)
    streams = [torch.cuda.Stream() for _ in range(4)]
    got = []
    torch.cuda.synchronize()
    for st in streams * 3:
        with torch.cuda.stream(st):
            got.append(OF.spec_accept_sample(logits, q, draft, u, unfinished.clone(), T, tk, tp, None, None))
    torch.cuda.synchronize()
    assert all(torch.equal(o, full) for o in got)
    qb = torch.empty_like(q)
    props = [torch.empty(b, k, dtype=torch.long, device=DEV) for _ in range(3)]
    ud = torch.rand(b, k, device=DEV)
    for p in props:
        OF.spec_sample(logits[:, 0].contiguous(), qb, 0, ud, p, T, tk, tp)
    assert torch.equal(props[0][:, 0], props[1][:, 0]) and torch.equal(props[0][:, 0], props[2][:, 0])


def test_argument_checks():
    ext = ops.load_ext(required=True)
    lg = torch.zeros(2, 4, 100, dtype=torch.bfloat16, device=DEV)
    q = torch.zeros(2, 3, 100, dtype=torch.bfloat16, device=DEV)
    d = torch.zeros(2, 3, dtype=torch.long, device=DEV)
    u = torch.rand(2, 4, 2, device=DEV)
    uf = torch.ones(2, dtype=torch.long, device=DEV)
    assert ext.spec_accept_sample(lg, q, d, u, uf, 1.0, 0, 1.0, 2, 0, None).shape == (2, 11)
    bad = [dict(u=u[:, :3]), dict(u=u.double()), dict(q=q[:, :2]), dict(d=d.int()), dict(T=0.0), dict(tp=0.0),
           dict(tp=1.5), dict(tk=-1), dict(lg=torch.zeros(2, 17, 100, dtype=torch.bfloat16, device=DEV))]
    for change in bad:
        a = dict(lg=lg, q=q, d=d, u=u, T=1.0, tk=0, tp=1.0)
        a.update(change)
        with pytest.raises(RuntimeError, match="spec_accept_sample"):
            ext.spec_accept_sample(a["lg"], a["q"], a["d"], a["u"], uf, a["T"], a["tk"], a["tp"], 2, 0, None)
    p = torch.zeros(2, 3, dtype=torch.long, device=DEV)
    for args in [(lg[:, 0].contiguous(), q, 3, u[:, :3, 0].contiguous(), p),
                 (lg[:, 0].contiguous(), q.float(), 0, u[:, :3, 0].contiguous(), p)]:
        with pytest.raises(RuntimeError, match="spec_sample"):
            ext.spec_sample(*args, 1.0, 0, 1.0)


# ------------------------------------------------------------------------------------------------ distributions
def _chi2(counts, probs, n):
    """Chi-square p-value of counts against probs, merging cells whose expected count is below 5."""
    exp = probs * n
    order = np.argsort(-exp)
    c, e = [], []
    acc_c = acc_e = 0.0
    for i in order:
        acc_c += counts[i]
        acc_e += exp[i]
        if acc_e >= 5:
            c.append(acc_c), e.append(acc_e)
            acc_c = acc_e = 0.0
    if acc_e > 0 and e:
        c[-1] += acc_c
        e[-1] += acc_e
    return stats.chisquare(np.array(c), np.array(e) * (sum(c) / sum(e))).pvalue


def _distribution(V, warp, n_samples, k=3, seed=0):
    T, tk, tp = warp
    g = torch.Generator(device=DEV).manual_seed(seed)
    p_rows = torch.randn(1, k + 1, V, device=DEV, generator=g) * 2
    q_rows = p_rows[:, :k] + torch.randn(1, k, V, device=DEV, generator=g)
    logits = p_rows.expand(n_samples, k + 1, V).contiguous()
    qsrc = q_rows.expand(n_samples, k, V).contiguous()
    torch.manual_seed(seed)
    ud = torch.rand(n_samples, k, device=DEV)
    qb = torch.empty_like(qsrc)
    props = torch.empty(n_samples, k, dtype=torch.long, device=DEV)
    for j in range(k):
        OF.spec_sample(qsrc[:, j].contiguous(), qb, j, ud, props, T, tk, tp)
    u = torch.rand(n_samples, k + 1, 2, device=DEV)
    out = OF.spec_accept_sample(logits, qb, props, u, torch.ones(n_samples, dtype=torch.long, device=DEV), T, tk, tp,
                                None, None).cpu()
    _, _, p, _ = OF._warp64(p_rows[0].cpu(), T, tk, tp)
    _, _, q, _ = OF._warp64(q_rows[0].cpu(), T, tk, tp)
    R = k + 1
    a = out[:, 2 * R]
    for j in range(R):
        sel = a >= j
        counts = np.bincount(out[sel, j].numpy(), minlength=V)
        pv = _chi2(counts, p[j].numpy(), int(sel.sum()))
        assert pv > 1e-3, (j, pv)
    rate = float((a >= 1).float().mean())
    want = float(torch.minimum(p[0], q[0]).sum())
    sigma = (want * (1 - want) / n_samples) ** 0.5
    assert abs(rate - want) <= 4 * sigma + 1e-9, (rate, want)


def test_kernel_distribution_top_k():
    _distribution(32000, (1.0, 50, 1.0), 20000)


def test_kernel_distribution_top_p_small_vocabulary():
    _distribution(40, (0.9, 0, 0.8), 20000)


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


def _sample(m, d, graphs, seed=0, case="plain", k=4, **kw):
    ids, am = _prompt(case)
    ids = ids.to(DEV)
    kw = dict(dict(eos_token_id=None, output_scores=True, max_length=ids.shape[1] + 16, decode_graphs=graphs,
                   do_sample=True, assistant_model=d, num_assistant_tokens=k, top_p=0.9, temperature=0.8), **kw)
    if am is not None:
        kw["attention_mask"] = am.to(DEV)
    torch.manual_seed(seed)
    with torch.no_grad():
        return m.generate(ids, **kw)


def _same(a, b):
    assert torch.equal(a[0], b[0])
    assert len(a[1]) == len(b[1]) and all(torch.equal(x, y) for x, y in zip(a[1], b[1]))


@pytest.mark.parametrize("kv", [None, "fp8"])
@pytest.mark.parametrize("name", FAMILIES)
def test_graphs_equal_eager(name, kv):
    m, d = _model(name), _other(name)
    for k in (3, 7):
        eager = _sample(m, d, False, seed=k, k=k, kv_cache_dtype=kv)
        graphs = _sample(m, d, True, seed=k, k=k, kv_cache_dtype=kv)
        _same(eager, graphs)
    g = decode_graph.current_graph(m)
    assert g is not None and g.graph is not None and g.failed is None


@pytest.mark.parametrize("target_w,draft_w", [("fp8", None), ("int4", None), (None, "fp8"), (None, "int4")])
def test_quantized_weights_graphs_equal_eager(target_w, draft_w):
    m, d = _model("llama_gqa", target_w), _model("llama_gqa", draft_w)
    for case in ("plain", "left_padded"):
        _same(_sample(m, d, False, case=case, num_return_sequences=2),
              _sample(m, d, True, case=case, num_return_sequences=2))


def test_replayed_iteration_launches_the_graphs_and_the_sampling_kernels_and_syncs_once(monkeypatch):
    m, d = _model("llama_gqa"), _other("llama_gqa")
    k = 4
    marks, outs, forwards = [], [], [0]
    accept = OF.spec_accept_sample
    caught = []

    def recorded(*a, **kw):
        marks.append((ops.launch_count(), sum("synchroniz" in str(w.message) for w in caught), forwards[0]))
        out = accept(*a, **kw)
        outs.append(out)
        return out

    forward = type(m).forward

    def counted(self, *a, **kw):
        forwards[0] += 1
        return forward(self, *a, **kw)

    monkeypatch.setattr(OF, "spec_accept_sample", recorded)
    monkeypatch.setattr(type(m), "forward", counted)
    ids, _ = _prompt("plain")
    # every sample runs to max_length: with the cfg's EOS the samples may all finish after a few iterations, leaving
    # too few replayed ones to count
    m.cfg.eos_token_id = None
    torch.manual_seed(0)
    with warnings.catch_warnings(record=True) as caught_now:
        warnings.simplefilter("always")
        caught = caught_now
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with torch.no_grad():
                m.generate(ids.to(DEV), max_length=ids.shape[1] + 40, eos_token_id=None, decode_graphs=True,
                           do_sample=True, assistant_model=d, num_assistant_tokens=k)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    verify, draft = decode_graph.current_graph(m), decode_graph.current_graph(d)
    assert verify.tokens == k + 1 and draft.tokens == 1
    R = k + 1
    checked = 0
    for j in range(2, len(marks) - 1):
        launches = marks[j + 1][0] - marks[j][0]
        catch_up = int(outs[j][0, 2 * R + 1]) == k
        # the acceptance kernel, the verify graph, k draft graphs (one more after a full acceptance), k draws
        want = 1 + verify.launches + (k + catch_up) * draft.launches + k
        info = (j, len(marks), launches, want, verify.launches, draft.launches, outs[j][:, 2 * R :].tolist())
        assert launches == want, info
        assert marks[j + 1][1] - marks[j][1] == 1, (marks[j + 1][1] - marks[j][1], info)
        assert marks[j + 1][2] == marks[j][2], (marks[j + 1][2] - marks[j][2], info)
        checked += 1
    assert checked >= 5


def test_top_k_one_is_greedy_speculative_decoding():
    """Per prompt (batch 1, so no other sample moves the blocks), up to its first step whose top two logits tie."""
    m, d = _model("llama_gqa"), _other("llama_gqa")
    ids, _ = _prompt("plain")
    compared = 0
    for i in range(ids.shape[0]):
        one = ids[i : i + 1].to(DEV)
        kw = dict(eos_token_id=None, max_length=one.shape[1] + 16, assistant_model=d, num_assistant_tokens=4,
                  output_scores=True)
        greedy = m.generate(one, **kw)
        sampled = m.generate(one, do_sample=True, top_k=1, **kw)
        top2 = torch.stack(greedy[1])[:, 0].float().topk(2, dim=-1).values
        ties = (top2[:, 0] == top2[:, 1]).nonzero()
        stop = int(ties[0]) if len(ties) else len(greedy[1])
        P = one.shape[1]
        assert torch.equal(sampled[0][:, : P + stop], greedy[0][:, : P + stop]), i
        compared += stop
    assert compared >= 16


def test_a_copy_of_the_target_accepts_nearly_everything(monkeypatch):
    m = _model("llama_gqa")
    d = copy.deepcopy(m)
    outs = []
    accept = OF.spec_accept_sample

    def recorded(*a, **kw):
        live = a[4] != 0   # the samples unfinished on entry (a finished one's proposals are pad tokens)
        out = accept(*a, **kw)
        outs.append((out[live], a[0].shape[1]))
        return out

    monkeypatch.setattr(OF, "spec_accept_sample", recorded)
    ids, _ = _prompt("plain")
    m.cfg.eos_token_id = None   # no sample finishes early: every iteration proposes for all of them
    torch.manual_seed(0)
    with torch.no_grad():
        m.generate(ids.to(DEV), max_length=ids.shape[1] + 40, eos_token_id=None, do_sample=True, assistant_model=d,
                   num_assistant_tokens=4)
    acc = tot = 0
    for out, R in outs[1:]:
        acc += int(out[:, 2 * R].sum())
        tot += out.shape[0] * (R - 1)
    rate = acc / tot
    print(f"acceptance of an exact copy: {rate:.4f} over {tot} proposals")
    # measured 1.0 over 96 proposals; below 1 only where the draft's single-token steps and the verify step round the
    # bf16 logits differently
    assert rate >= 0.9


def test_first_and_second_token_distributions():
    """A seeded chi-square on a tiny model: the first new token against the target's prefill distribution, the second
    (given the first) against the teacher-forced p(t2 | t1)."""
    m, d = _model("llama_gqa"), _other("llama_gqa")
    ids, _ = _prompt("plain")
    ids = ids[:1].to(DEV)
    warp = (0.9, 20, 0.95)
    n = 3000
    with torch.no_grad():
        torch.manual_seed(3)
        out = m.generate(ids, max_length=ids.shape[1] + 2, eos_token_id=None, do_sample=True, assistant_model=d,
                         num_assistant_tokens=2, temperature=warp[0], top_k=warp[1], top_p=warp[2],
                         num_return_sequences=n)
        P = ids.shape[1]
        first = m(ids, use_cache=False)["logits"][0, -1].float()
        _, _, p1, _ = OF._warp64(first.cpu(), *warp)
        assert _chi2(np.bincount(out[:, P].cpu().numpy(), minlength=p1.numel()), p1.numpy(), n) > 1e-3
        t1 = int(out[:, P].mode().values)
        sel = out[:, P] == t1
        second = m(torch.cat([ids, torch.tensor([[t1]], device=DEV)], 1), use_cache=False)["logits"][0, -1].float()
        _, _, p2, _ = OF._warp64(second.cpu(), *warp)
        c = np.bincount(out[sel, P + 1].cpu().numpy(), minlength=p2.numel())
        assert int(sel.sum()) >= 100
        assert _chi2(c, p2.numpy(), int(sel.sum())) > 1e-3
