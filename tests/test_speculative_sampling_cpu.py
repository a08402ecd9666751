"""Speculative sampling without a GPU: the warp rule ``OF.spec_warp_ref`` against an independent NumPy implementation
(and ``TopPLogitsWarper`` where no tie meets the boundary), the acceptance mirror against a loop written from the rule,
the output distribution of the mirrors (chi-square, acceptance rate), top_k=1 against greedy acceptance, and
``generate(do_sample=True, assistant_model=...)`` on the scripted model and tiny models of every supported family:
both caches' invariant, stops and padding, ``num_return_sequences``, ``output_scores``, seeded repeats and every
refusal."""
import numpy as np
import pytest
import torch
from scipy import stats

from libai_b200.config import DictConfig
from libai_b200.inference.generator.generation_logits_processor import TopKLogitsWarper, TopPLogitsWarper
from libai_b200.inference.generator.generation_utils import Generator
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_cached_attention_cpu import _prompt
from tests.test_speculative_cpu import BUILDERS, FAMILIES, PROMPT, Scripted

NINF = float("-inf")


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


# ------------------------------------------------------------------------------------------------ the warp rule
def _warp_np(row, T, top_k, top_p):
    """The rule, one row, NumPy: fp32 division, the k-th largest counting duplicates, mass strictly above <= top_p."""
    z = (np.asarray(row, np.float32) / np.float32(T)).astype(np.float32)
    V = z.size
    keep = np.ones(V, bool)
    if 0 < top_k < V:
        kth = np.sort(z)[::-1][top_k - 1]
        keep = z >= kth
    if np.float32(top_p) < 1:
        zk = np.where(keep, z.astype(np.float64), -np.inf)
        m = zk.max()
        with np.errstate(invalid="ignore"):   # −inf − −inf on a row of −inf only, where every token is the maximum
            e = np.where(keep, np.where(zk == m, 1.0, np.exp(zk - m)), 0.0)
        pi = e / e.sum()
        above = np.array([pi[(zk > zk[i]) & keep].sum() for i in range(V)])
        keep = keep & (above <= np.float64(np.float32(top_p)))
    return np.where(keep, z, -np.inf).astype(np.float32)


def _same_warp(row, T, k, p):
    got = OF.spec_warp_ref(torch.tensor(row, dtype=torch.float32)[None], T, k, p)[0].numpy()
    want = _warp_np(row, T, k, p)
    assert np.array_equal(got, want), (T, k, p)
    return got


def test_top_k_counts_ties_at_the_kth_value():
    row = [1.0, 3.0, 3.0, 2.0, 3.0, 0.5, 2.0]
    got = _same_warp(row, 1.0, 2, 1.0)
    assert (got > NINF).sum() == 3   # three tokens tie at the 2nd largest value: all kept
    got = _same_warp(row, 1.0, 4, 1.0)
    assert (got > NINF).sum() == 5
    torch.testing.assert_close(torch.tensor(got), TopKLogitsWarper(4)(None, torch.tensor([row]))[0])


def test_top_p_equals_top_p_warper_without_ties():
    g = torch.Generator().manual_seed(0)
    for trial in range(50):
        row = torch.randn(97, generator=g) * (1 + trial % 4)
        for p in (0.1, 0.5, 0.8, 0.95):
            got = _same_warp(row.tolist(), 1.0, 0, p)
            want = TopPLogitsWarper(p)(None, row[None].clone())[0]
            assert torch.equal(torch.tensor(got), want), (trial, p)


def test_top_p_keeps_every_tied_token_at_the_boundary():
    row = [2.0, 1.0, 1.0, 1.0, 0.0, -1.0]
    got = _same_warp(row, 1.0, 0, 0.5)
    # the top token alone has mass < 0.5 above the tied 1.0s: all three are kept
    assert list(got > NINF) == [True, True, True, True, False, False]


def test_top_k_at_or_past_the_vocabulary_and_ninf_entries():
    row = [0.5, NINF, 1.5, NINF, -2.0]
    for k in (0, 5, 9):
        got = _same_warp(row, 0.7, k, 1.0)
        assert list(got > NINF) == [True, False, True, False, True]
    _same_warp(row, 1.3, 2, 0.6)
    _same_warp([NINF] * 4, 1.0, 2, 0.5)   # −inf only: every token ties with the maximum


def test_random_rows_against_numpy():
    g = torch.Generator().manual_seed(1)
    for trial in range(60):
        V = int(torch.randint(2, 80, (1,), generator=g))
        row = torch.randint(-3, 4, (V,), generator=g).float() * 0.5 if trial % 2 else torch.randn(V, generator=g) * 2
        T = [1.0, 0.7, 1.6][trial % 3]
        k = [0, 1, 5, 50][trial % 4]
        p = [1.0, 0.9, 0.5, 0.2, 0.8][trial % 5]
        _same_warp(row.tolist(), T, k, p)


# ------------------------------------------------------------------------------------------------ the acceptance mirror
def _probs(row, T, k, p):
    z = _warp_np(row, T, k, p).astype(np.float64)
    m = z.max()
    e = np.where(z > -np.inf, np.where(z == m, 1.0, np.exp(z - m)), 0.0)
    return e / e.sum()


def _pick(w, u):
    cum = np.cumsum(w)
    return min(int(np.searchsorted(cum, u * cum[-1], side="right")), len(w) - 1)


def _accept_loop(logits, q, draft, u, unfinished, warp, eos, pad):
    b, R, _ = logits.shape
    k = R - 1
    t, a = [], []
    for i in range(b):
        ti, ai = [], None
        for j in range(R):
            p = _probs(logits[i, j].numpy(), *warp)
            if j < k:
                qq = _probs(q[i, j].numpy(), *warp)
                d = int(draft[i, j])
                ok = float(u[i, j, 0]) * qq[d] < p[d]
                r = np.maximum(p - qq, 0)
                c = _pick(r if r.sum() > 0 else p, float(u[i, j, 1]))
                if ai is None and not ok:
                    ai = j
                ti.append(d if ai is None else c)
            else:
                ti.append(_pick(p, float(u[i, j, 1])))
        t.append(ti)
        a.append(k if ai is None else ai)
    limits = [k if eos is not None and eos in t[i][: a[i] + 1] else a[i] for i in range(b) if unfinished[i]]
    n = min(limits) if limits else k
    rows = []
    for i in range(b):
        uu, e = int(unfinished[i]), []
        for j in range(R):
            if j > n:
                e.append(-1)
                continue
            tok = t[i][j] if eos is None or uu else pad
            if eos is not None and tok == eos:
                uu = 0
            e.append(tok)
        rows.append(t[i] + e + [a[i], n, uu])
    return torch.tensor(rows)


@pytest.mark.parametrize("eos", [None, 3])
def test_accept_mirror_against_the_rule(eos):
    g = torch.Generator().manual_seed(2)
    warps = [(1.0, 0, 1.0), (0.8, 4, 1.0), (1.0, 0, 0.7), (0.9, 5, 0.8)]
    for trial in range(120):
        b, k, V = int(torch.randint(1, 5, (1,), generator=g)), int(torch.randint(0, 6, (1,), generator=g)), 8
        logits = torch.randn(b, k + 1, V, generator=g) * 2
        q = logits[:, :k] + torch.randn(b, k, V, generator=g) * (trial % 3)
        if eos is not None and trial % 4 == 0:   # EOS likely at some block position
            logits[..., eos] += 4
        draft = torch.randint(0, V, (b, k), generator=g)
        draft[:, : k // 2] = logits[:, : k // 2].argmax(-1)
        u = torch.rand(b, k + 1, 2, generator=g)
        unfinished = (torch.rand(b, generator=g) < 0.7).long()
        warp = warps[trial % 4]
        want = _accept_loop(logits, q, draft, u, unfinished, warp, eos, 0)
        uf = unfinished.clone()
        got = OF.spec_accept_sample(logits, q, draft, u, uf, *warp, eos, 0 if eos is not None else None)
        assert torch.equal(got, want), trial
        assert torch.equal(uf, want[:, -1])


def test_top_k_one_gives_greedy_decisions():
    g = torch.Generator().manual_seed(3)
    for _ in range(50):
        b, k, V = 3, 4, 30
        logits = torch.randn(b, k + 1, V, generator=g)
        draft = logits[:, :k].argmax(-1)
        wrong = torch.rand(b, k, generator=g) < 0.3
        draft[wrong] = (draft[wrong] + 1) % V
        q = torch.randn(b, k, V, generator=g)
        q.scatter_(-1, draft[..., None], 100.0)   # the draft's own argmax is its proposal
        u = torch.rand(b, k + 1, 2, generator=g)
        greedy = OF.spec_accept(logits, draft, torch.ones(b, dtype=torch.long), None, None)
        sampled = OF.spec_accept_sample(logits, q, draft, u, torch.ones(b, dtype=torch.long), 1.0, 1, 1.0)
        assert torch.equal(sampled, greedy)


def _chi2(counts, probs, n):
    exp = probs * n
    c, e, acc_c, acc_e = [], [], 0.0, 0.0
    for i in np.argsort(-exp):
        acc_c += counts[i]
        acc_e += exp[i]
        if acc_e >= 5:
            c.append(acc_c), e.append(acc_e)
            acc_c = acc_e = 0.0
    c[-1] += acc_c
    e[-1] += acc_e
    return stats.chisquare(np.array(c), np.array(e) * (sum(c) / sum(e))).pvalue


@pytest.mark.parametrize("warp", [(1.0, 0, 1.0), (0.8, 6, 1.0), (1.0, 0, 0.8)])
def test_mirror_distribution(warp):
    torch.manual_seed(4)
    n, k, V = 20000, 3, 12
    p_rows = torch.randn(1, k + 1, V) * 1.5
    q_rows = p_rows[:, :k] + torch.randn(1, k, V)
    logits, qsrc = p_rows.expand(n, k + 1, V).contiguous(), q_rows.expand(n, k, V).contiguous()
    ud = torch.rand(n, k)
    qb, props = torch.empty_like(qsrc), torch.empty(n, k, dtype=torch.long)
    for j in range(k):
        OF.spec_sample(qsrc[:, j].contiguous(), qb, j, ud, props, *warp)
    out = OF.spec_accept_sample(logits, qb, props, torch.rand(n, k + 1, 2), torch.ones(n, dtype=torch.long), *warp)
    R = k + 1
    a = out[:, 2 * R]
    for j in range(R):
        sel = a >= j
        p = _probs(p_rows[0, j].numpy(), *warp)
        assert _chi2(np.bincount(out[sel, j].numpy(), minlength=V), p, int(sel.sum())) > 1e-3, j
    want = float(np.minimum(_probs(p_rows[0, 0].numpy(), *warp), _probs(q_rows[0, 0].numpy(), *warp)).sum())
    rate = float((a >= 1).float().mean())
    assert abs(rate - want) <= 4 * (want * (1 - want) / n) ** 0.5


# ------------------------------------------------------------------------------------------------ generate()
class Soft(Scripted):
    """The scripted model with soft logits: its table token gets +3, so sampling has somewhere to go."""

    def forward(self, input_ids, attention_mask=None, use_cache=False):
        out = super().forward(input_ids, attention_mask, use_cache)
        return {"logits": out["logits"] * 0.3}


def _sgen(m, seed=0, **kw):
    torch.manual_seed(seed)
    kw = dict(dict(max_length=19, output_scores=True, do_sample=True, top_k=0), **kw)
    return m.generate(PROMPT, **kw)


def test_scripted_cache_invariant_seeds_and_scores(monkeypatch):
    target, draft = Soft(), Soft(wrong=({7, 12}, {9}))
    seen = []
    verify = Generator._verify_step

    def check(model, block):
        c, dc = model.kv_cache, draft.kv_cache
        seen.append((c.k[0][:, 0, : c.length, 0].long().clone(), dc.length))
        return verify(model, block)

    monkeypatch.setattr(Generator, "_verify_step", check)
    out = _sgen(target, assistant_model=draft, num_assistant_tokens=3, temperature=0.9)
    for rows, dlen in seen:   # the target holds the sequence minus its last token; the draft k rows more
        assert torch.equal(rows, out[0][:, : rows.shape[1]])
        assert dlen == rows.shape[1] + 3
    assert out[0].shape[1] == 19 and len(out[1]) == 15
    again = _sgen(target, assistant_model=draft, num_assistant_tokens=3, temperature=0.9)
    assert torch.equal(again[0], out[0]) and all(torch.equal(x, y) for x, y in zip(again[1], out[1]))
    # the scores are the target's warped rows: z = logits / T at the emitted positions, teacher-forced
    for s in out[1]:
        assert s.dtype == torch.float32 and s.shape == (2, 50)
    tf = Soft()
    tf.allocate_kv_cache(2, 40)
    logits = tf(out[0][:, :-1], use_cache=True)["logits"]
    P = PROMPT.shape[1]
    for j, s in enumerate(out[1]):
        want = OF.spec_warp_ref(logits[:, P - 1 + j], 0.9, 0, 1.0)
        assert torch.equal(s, want), j


def test_scripted_stops_padding_and_return_sequences():
    target = Soft(eos_at={(0, 9), (1, 7)}, eos=4)
    draft = Soft(eos_at={(0, 9), (1, 7)}, eos=4)
    target.cfg.eos_token_id = 4
    out = _sgen(target, assistant_model=draft, num_assistant_tokens=4, top_k=1)   # greedy in effect
    greedy = target.generate(PROMPT, max_length=19, output_scores=False)
    assert torch.equal(out[0], greedy)
    for max_length in (2, 6, 11):
        o = _sgen(target, assistant_model=draft, num_assistant_tokens=4, max_length=max_length, output_scores=False)
        assert o.shape[1] <= max(max_length, 5)
    t6, d6 = Soft(wrong=((),) * 6), Soft(wrong=((7,),) * 6)
    o = _sgen(t6, assistant_model=d6, num_assistant_tokens=3, num_return_sequences=3, output_scores=False)
    assert o.shape == (6, 19)
    assert torch.equal(o[:, :4], PROMPT.repeat_interleave(3, 0))
    assert t6.kv_cache.seqlens.numel() == 6 and d6.kv_cache.seqlens.numel() == 6


@pytest.mark.parametrize("name", FAMILIES)
def test_families_sample_repeatably_and_top_k_one_is_greedy(name):
    m = BUILDERS[name]().float()
    other = BUILDERS[name]().float()
    with torch.no_grad():
        for p in other.parameters():
            p.add_(torch.randn(p.shape, generator=torch.Generator().manual_seed(9)) * 0.05)
    ids, _ = _prompt("plain")
    kw = dict(eos_token_id=None, max_length=ids.shape[1] + 10, assistant_model=other, num_assistant_tokens=3)
    torch.manual_seed(5)
    a = m.generate(ids, do_sample=True, top_p=0.9, temperature=0.8, output_scores=True, **kw)
    torch.manual_seed(5)
    b = m.generate(ids, do_sample=True, top_p=0.9, temperature=0.8, output_scores=True, **kw)
    assert torch.equal(a[0], b[0]) and a[0].shape == (ids.shape[0], ids.shape[1] + 10)
    for s in a[1]:   # warped rows: −inf off the kept set, which holds every emitted token
        assert (s > NINF).any(dim=-1).all()
    new = a[0][:, ids.shape[1]:]
    eos = m._gcfg("eos_token_id")
    done = torch.zeros(new.shape[0], dtype=torch.bool)
    for j, s in enumerate(a[1]):   # an unfinished sample's token is a choice of its warped row; then it pads
        assert (s.gather(1, new[:, j : j + 1])[~done] > NINF).all()
        if eos is not None:
            done |= new[:, j] == eos
    greedy = m.generate(ids, **kw)
    assert torch.equal(m.generate(ids, do_sample=True, top_k=1, **kw), greedy)


# ------------------------------------------------------------------------------------------------ refusals
REFUSALS = {
    "typical_p": dict(typical_p=0.9),
    "top_p": dict(top_p=0.0),
    "temperature": dict(temperature=0.0),
    "top_k": dict(top_k=-1),
    "renormalize_logits": dict(renormalize_logits=True),
    "repetition_penalty": dict(repetition_penalty=1.3),
    "num_beams": dict(num_beams=2),
}


@pytest.mark.parametrize("arg", sorted(REFUSALS))
def test_each_refusal_names_its_argument(arg):
    with pytest.raises(ValueError, match=arg if arg != "top_k" else "top_k"):
        Scripted().generate(PROMPT, max_length=10, do_sample=True, assistant_model=Scripted(), **REFUSALS[arg])


def test_prompt_lookup_does_not_sample():
    with pytest.raises(ValueError, match="do_sample"):
        Scripted().generate(PROMPT, max_length=10, do_sample=True, prompt_lookup_num_tokens=2)
    with pytest.raises(ValueError, match="num_return_sequences"):
        Scripted().generate(PROMPT, max_length=10, assistant_model=Scripted(), num_return_sequences=2)
