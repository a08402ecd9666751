"""The paged KV cache on the H100 against fp64, element by element: a real ``PagedKVCache`` walked through prefills,
forks, decode steps, continuations, beam reorders, rollbacks, prefix hits and graph replays, on the native appends, page
copy and paged kernels, beside an independent contiguous shadow.

After every operation the pages nobody may read hold NaN (every free page, and every row at or past the length in a
mapped page), the reference counts and free list are recounted from the host table and the prefix index, the device
table must equal the host one, and the logical rows gathered through the table must equal the shadow's bit for bit.
Every attention asserts which op ran and is checked within ``CR.expect``'s bound of fp64 computed over the shadow's
rows, never over the pool: an append to the wrong page, a stale device table, a missing copy on write or a page freed
while still mapped all show up as a difference with a cache the paging cannot touch.

The shadow is a ``StaticKVCache`` with a row per sequence, fed the same projections through the contiguous native
appends (their bytes have fp64 tests of their own); for prefix hits it is a fresh contiguous cache that prefills the
whole prompt."""
import random

import pytest
import torch

from libai_b200.inference.kv_cache import PagedKVCache, StaticKVCache
from libai_b200.ops import functional as OF
from tests import cached_attention_ref as CR
from tests.dense_ref import check
from tests.test_cached_attention_fp64_gpu import _check_out, _projection, _slopes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP8 = torch.float8_e4m3fn
BF16 = torch.bfloat16
P = OF.PAGE_ROWS

# BLOOM-like MHA with ALiBi, and a Llama-like grouping of 4 query heads per key/value head with rotary tables
HEADS = {"mha_alibi": dict(A=4, G=4, D=64, alibi=True, rotary=False),
         "gqa_rotary": dict(A=8, G=2, D=128, alibi=False, rotary=True)}
CACHES = ["bf16", "fp8"]


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


@pytest.fixture
def rec(ext, monkeypatch):
    r = CR.Recorder(ext)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: r)
    return r


# ------------------------------------------------------------------------------------------------------------- checks
def _poison(c):
    """NaN in every page on the free list and in every row at or past ``length`` of every mapped page: bf16 NaN, or
    for an FP8 pool the E4M3 NaN byte and NaN scales."""
    spots = [(p, 0) for p in set(c.free)]
    for slot in range(c.length // P, c.mapped):
        lo = max(c.length - slot * P, 0)
        spots += [(p, lo) for p in {row[slot] for row in c.host_table[: c.batch]}]
    for p, lo in spots:
        for t in c.arrays():
            if t.dtype == FP8:
                t.view(torch.uint8)[p, :, lo:] = 0x7F
            else:
                t[p, :, lo:] = float("nan")


def _check_books(c):
    """The reference counts recounted from the host table and the prefix index, the free list against them, and the
    device table against the host one."""
    refs = [1 if p in c._entry else 0 for p in range(c.num_pages)]
    for row in c.host_table[: c.batch]:
        assert all(p >= 0 for p in row[: c.mapped]) and all(p == -1 for p in row[c.mapped:])
        for p in row[: c.mapped]:
            refs[p] += 1
    assert refs == c.refs
    assert sorted(c.free) == [p for p in range(c.num_pages) if refs[p] == 0]
    assert torch.equal(c.block_table.cpu(), torch.tensor(c.host_table[: c.batch], dtype=torch.int32))


def _bytes(t):
    return t.view(torch.uint8) if t.dtype == FP8 else t


def _check_rows(c, sh, rows=slice(None)):
    """The paged logical rows ``[:length]`` equal the shadow's ``rows`` bit for bit (FP8: bytes and scales)."""
    L = c.length
    for pool, buf in zip(c.arrays(), [t[0] for t in (sh.k, sh.v, sh.k_scale, sh.v_scale) if t[0] is not None]):
        got, want = OF.kv_pages_gather(pool, c.block_table, L), buf[rows][:, :, :L]
        assert torch.equal(_bytes(got), _bytes(want)), f"paged rows differ from the shadow's (length {L})"


def _after(c, sh, rows=slice(None)):
    _poison(c)
    _check_books(c)
    _check_rows(c, sh, rows)


def _want(fp8, s, past, alibi):
    """The op a step of ``s`` new tokens after ``past`` rows must run, and which bound applies."""
    if s <= 16 and past > 0:
        return [("decode_attn_paged", fp8)], "decode"
    if not fp8:
        return [("attn_fwd_paged", alibi, past)], "flash"
    # an FP8 pool: its window gathered and dequantized to bf16, then the flash kernel
    return [("attn_fwd", False, alibi, True, past + s, BF16)], "flash"


def _check_attention(o, q, sh, rows, past, kv_start, *, scale, kernel, slopes=None, mask=None, what):
    """o against fp64 over the shadow's rows ``[:past + s]``; returns the largest ``|o - ref| / bound``."""
    B, s, A, D = q.shape
    L = past + s
    ks = None if sh.k_scale[0] is None else sh.k_scale[0][rows]
    vs = None if sh.v_scale[0] is None else sh.v_scale[0][rows]
    k64, v64 = CR.rows64(sh.k[0][rows], sh.v[0][rows], ks, vs, L, exact=kernel == "decode")
    if mask is not None:
        vis, slopes = mask.bool(), None
    else:
        vis = CR.visible(torch.full_like(kv_start, past), kv_start, s, L, True)
    eta, extra = CR.fp8_decode_terms(q, k64, scale) if kernel == "decode" and ks is not None else (None, 0.0)
    ref, bnd = CR.expect(q, k64, v64, scale=scale, vis=vis, alibi=slopes, tile=128 if kernel == "flash" else 64,
                         eta_extra=eta, extra_abs=extra)
    _check_out(o, B, s, A, D, what)
    check(o, ref, bnd, what)
    return float(((o.double() - ref).abs() / bnd).nan_to_num(0.0).max())


class _Setup:
    """Head layout, projections, rotary tables (for ``positions`` rows; none for 0) and ALiBi slopes of one case."""

    def __init__(self, heads, cache, seed, positions):
        self.__dict__.update(HEADS[heads])
        self.fp8 = cache == "fp8"
        self.kv_dtype = FP8 if self.fp8 else None
        self.scale = self.D ** -0.5
        self.g = torch.Generator(device=DEV).manual_seed(seed)
        self.slopes = _slopes(self.A) if self.alibi else None
        self.rope = ()
        if self.rotary and positions:
            ang = torch.arange(positions, dtype=torch.float32)[:, None] * torch.linspace(0.01, 1.0, self.D)[None]
            self.rope = (ang.cos().to(DEV), ang.sin().to(DEV))

    def proj(self, B, s, pad=None):
        return _projection(B, s, self.A, self.G, self.D, self.g, pad)

    def append(self, layer, qkv):
        return layer.append(qkv, *self.rope)

    def paged(self, batch, capacity, **kw):
        return PagedKVCache(1, batch, self.G, self.D, capacity, BF16, DEV, kv_dtype=self.kv_dtype, **kw)

    def static(self, batch, capacity):
        return StaticKVCache(1, batch, self.G, self.D, capacity, BF16, DEV, kv_dtype=self.kv_dtype)


# ----------------------------------------------------------------------------------------------------- 1. the walk
def _walk_ops(rnd):
    ops = ["d16", "rollback", "c17", "reorder_identity", "d1", "reorder_one", "boundary", "reorder_random", "d1",
           "c150", "reorder_random", "rollback", "d16", "dense", "reorder_random"]
    rnd.shuffle(ops)
    return ["d1"] + ops + ["d1"]


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("heads", sorted(HEADS))
@pytest.mark.parametrize("cache", CACHES)
def test_walk_matches_a_contiguous_shadow_and_fp64(rec, cache, heads, seed):
    """Two left-padded prompts (37, 128 or 300 rows: inside a page, on a boundary, past several) forked into three
    sequences each, then in a seeded order: 1- and 16-token decode steps, 17- and 150-token continuations, reorders
    (identity, random, every sequence continuing one), rollbacks of 0-5 rows and one across a page boundary, and a
    dense-mask step (the reference math)."""
    rnd = random.Random(seed)
    B, n, cap = 2, 3, 640
    u = _Setup(heads, cache, 100 * seed + 7 * len(heads) + (cache == "fp8"), cap)
    s0 = (37, 128, 300)[seed]
    c, sh = u.paged(B, cap, fork=n, prompt_len=s0), u.static(B * n, cap)
    layer, slayer = c.layer(0), sh.layer(0)
    worst = 0.0

    def step(s, pad=None, mask=None):
        nonlocal worst
        past, rows = c.length, slice(None) if c.batch == B * n else slice(None, None, n)
        x = u.proj(c.batch, s, pad)
        c.reserve(s)
        q = u.append(layer, x)
        sq = u.append(slayer, x.repeat_interleave(B * n // c.batch, 0))
        assert torch.equal(q, sq[rows])
        rec.take()
        o = layer.attend(q, scale=u.scale, alibi_slopes=u.slopes, mask=mask)
        want, kernel = ([], "ref") if mask is not None else _want(u.fp8, s, past, u.alibi)
        what = f"{cache} {heads} seed={seed} past={past} s={s} {kernel}"
        assert rec.take() == want, what
        c.advance(s)
        sh.advance(s)
        worst = max(worst, _check_attention(o, q, sh, rows, past, c.kv_start, scale=u.scale, kernel=kernel,
                                            slopes=u.slopes, mask=mask, what=what))
        _after(c, sh, rows)

    # the prompts: left padding in kv_start, the padding's k/v the sentinels a leak would show (short enough that the
    # rollbacks never take a sequence back into its padding)
    pad = [rnd.randrange(0, 3), rnd.randrange(1, min(s0 - 20, 90))]
    mask = torch.ones(B, s0, dtype=torch.long, device=DEV)
    for b, m in enumerate(pad):
        mask[b, :m] = 0
    assert c.step_needs_dense_mask(mask, flash=c.flash_attention()) is False
    assert sh.step_needs_dense_mask(mask.repeat_interleave(n, 0), flash=sh.flash_attention()) is False
    step(s0, pad=pad)
    c.fork(n)
    _after(c, sh)

    for op in _walk_ops(rnd):
        if op[0] in "dc" and op != "dense":   # a decode step or a continuation
            step(int(op[1:]))
        elif op == "boundary":   # two rows into a page, then back across its start
            t = (2 - c.length) % P or P
            step(t)
            k = rnd.randint(3, 5)
            c.rollback(k)
            sh.rollback(k)
            _after(c, sh)
        elif op == "rollback":
            k = rnd.randint(0, 5)
            c.rollback(k)
            sh.rollback(k)
            _after(c, sh)
        elif op == "dense":   # causality, the padding and a few holes: the reference math over the gathered window
            s, L = 5, c.length + 5
            vis = CR.visible(torch.full_like(c.seqlens, c.length), c.kv_start, s, L, True)
            holes = torch.rand(vis.shape, device=DEV, generator=u.g) < 0.2
            holes[..., c.length:] = False
            step(s, mask=(vis & ~holes).to(torch.uint8))
        else:
            N = B * n
            idx = {"reorder_identity": list(range(N)), "reorder_one": [rnd.randrange(N)] * N,
                   "reorder_random": [rnd.randrange(N) for _ in range(N)]}[op]
            idx = torch.tensor(idx, device=DEV)
            c.reorder_(idx)
            sh.reorder_(idx)
            _after(c, sh)
    print(f"\n[paged walk] {cache} {heads} seed={seed} prompt={s0}: max|o - ref| / bound = {worst:.3f}")


# ------------------------------------------------------------------------------------------- 2. prefix caching
class _Index:
    """What the prefix index must hold, by content: a full page is known by every (token, mask) pair from the start
    of its prompt to its end.  Lookup takes the longest run every prompt starts with; eviction takes the least recently
    used page no cached page continues (of two used at once, the one cached first)."""

    def __init__(self, budget):
        self.budget, self.used, self.order, self.tick, self.n = budget, {}, {}, 0, 0

    def lookup(self, rows, s):
        hit = min(next((j for j in range((s - 1) // P) if tuple(r[: (j + 1) * P]) not in self.used), (s - 1) // P)
                  for r in rows)
        if hit:
            self.tick += 1
            for r in rows:
                for j in range(hit):
                    self.used[tuple(r[: (j + 1) * P])] = self.tick
        return hit

    def insert(self, rows, L):
        self.tick += 1
        for r in rows:
            for j in range(L // P):
                key = tuple(r[: (j + 1) * P])
                if key not in self.used:
                    self.order[key], self.n = self.n, self.n + 1
                self.used[key] = self.tick
        while len(self.used) > self.budget:
            leaves = [k for k in self.used if not any(len(o) > len(k) and o[: len(k)] == k for o in self.used)]
            victim = min(leaves, key=lambda k: (self.used[k], self.order[k]))
            del self.used[victim], self.order[victim]


class _Model:
    """Projections as a model makes them: a function of (token id, position, mask) through seeded tables, so that
    equal prefixes give equal rows; a masked token's k/v are the sentinels."""

    def __init__(self, u, vocab, positions, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        r = u.A // u.G
        self.u, self.r = u, r
        self.tok = torch.randn(vocab, u.G, r + 2, u.D, device=DEV, generator=g)
        self.pos = 0.5 * torch.randn(positions, u.G, r + 2, u.D, device=DEV, generator=g)

    def __call__(self, ids, mask, p0):
        s = ids.shape[1]
        qkv = (self.tok[ids] + self.pos[p0 : p0 + s][None]).to(BF16)
        pad = mask == 0
        qkv[..., self.r, :][pad] = CR.SENT_K
        qkv[..., self.r + 1, :][pad] = CR.SENT_V
        return qkv


def _prefix_calls():
    """Six calls of two prompts: no hit; two shared pages; a prompt that differs inside its second page (one page
    shared); two left-padded prompts with the tokens of cached ones (no hit, and past the budget: every older page is
    evicted); the same again (three pages hit, left padded); and a shorter prompt whose rest is one decode step."""
    g = torch.Generator().manual_seed(5)
    X, Y, T = (torch.randint(4, 100, (256,), generator=g) for _ in range(3))
    c1 = torch.stack([X[:150], Y[:150]])
    c2 = torch.stack([torch.cat([X[:140], T[:60]]), torch.cat([Y[:140], T[60:120]])])
    row0 = torch.cat([X[:100], torch.tensor([3]), T[120:249]])   # X[100] >= 4: differs at row 100, page 1
    c3 = torch.stack([row0, torch.cat([c2[1], T[:30]])])
    m3 = torch.ones_like(c3)
    m4 = m3.clone()
    m4[0, :5] = m4[1, :9] = 0
    c4 = c3.masked_fill(m4 == 0, 0)
    return [(c1, None, 0), (c2, None, 2), (c3, None, 1), (c4, m4, 0), (c4, m4, 3), (c4[:, :200], m4[:, :200], 3)]


@pytest.mark.parametrize("cache", CACHES)
def test_prefix_hits_read_the_rows_of_a_full_prefill(rec, cache):
    """Calls on one pool with a six-page prefix budget: reset, lookup, the prefill of the rest, two decode steps and
    insert.  The pages the index held before a call are unchanged after it; the hits and the cached pages match the
    index's rule; every attention, the first after a hit included, is checked against fp64 over the rows a fresh
    contiguous cache holds after prefilling the whole prompt."""
    u = _Setup("gqa_rotary", cache, 41 + (cache == "fp8"), 0)   # no rotary: positions enter through the tables
    B, cap, budget = 2, 256, 6
    c = u.paged(B, cap, prefix_tokens=budget * P)
    layer = c.layer(0)
    model, index = _Model(u, 100, cap, 43), _Index(budget)
    g = torch.Generator().manual_seed(6)
    worst = 0.0
    for call, (ids, mask, hit_want) in enumerate(_prefix_calls()):
        ids = ids.to(DEV)
        s = ids.shape[1]
        full_mask = torch.ones_like(ids) if mask is None else mask.to(DEV)
        am = None if mask is None else full_mask   # the attention_mask a caller passes
        held = {p: [t[p].clone() for t in c.arrays()] for p in c._entry}
        c.reset()
        _poison(c)
        hit = c.lookup(ids, am)
        rows = [list(zip(r, m)) for r, m in zip(ids.tolist(), full_mask.tolist())]
        assert hit == index.lookup(rows, s) == hit_want, (call, hit)
        assert c.reused_rows == hit * P and c.length == hit * P
        # the reference: a fresh contiguous cache prefilled with the whole prompt
        fresh = u.static(B, cap)
        assert fresh.step_needs_dense_mask(am, flash=fresh.flash_attention()) is False
        u.append(fresh.layer(0), model(ids, full_mask, 0))
        fresh.advance(s)
        _check_books(c)
        _check_rows(c, fresh)
        assert c.step_needs_dense_mask(am, flash=c.flash_attention()) is False
        assert torch.equal(c.kv_start, fresh.kv_start)
        past, seq, seq_mask = hit * P, ids, full_mask
        for step, new in enumerate((s - past, 1, 1)):
            if step:   # a generated token
                tok = torch.randint(4, 100, (B, 1), generator=g).to(DEV)
                seq, seq_mask = torch.cat([seq, tok], 1), torch.cat([seq_mask, torch.ones_like(tok)], 1)
                u.append(fresh.layer(0), model(tok, seq_mask[:, -1:], fresh.length))
                fresh.advance(1)
            c.reserve(new)
            q = u.append(layer, model(seq[:, past:], seq_mask[:, past:], past))
            rec.take()
            o = layer.attend(q, scale=u.scale)
            want, kernel = _want(u.fp8, new, past, False)
            what = f"prefix {cache} call={call} hit={hit} past={past} s={new} {kernel}"
            assert rec.take() == want, what
            c.advance(new)
            worst = max(worst, _check_attention(o, q, fresh, slice(None), past, c.kv_start, scale=u.scale,
                                                kernel=kernel, what=what))
            _after(c, fresh)
            past = c.length
        c.insert(seq, None if mask is None else seq_mask)
        index.insert([list(zip(r, m)) for r, m in zip(seq.tolist(), seq_mask.tolist())], seq.shape[1])
        assert c.cached_pages() == len(index.used), call
        for p, before in held.items():   # a cached page is never written
            assert all(torch.equal(_bytes(t[p]), _bytes(x)) for t, x in zip(c.arrays(), before)), (call, p)
        _check_books(c)
    print(f"\n[prefix calls] {cache}: max|o - ref| / bound = {worst:.3f}")


# ---------------------------------------------------------------------------------------------- 3. graph replay
@pytest.mark.parametrize("cache", CACHES)
def test_graph_replays_follow_a_walking_cache(rec, cache):
    """One captured 1-token step (append, then attend), replayed after eager reorders, copies on write and
    rollbacks; ``reserve`` before the capture and before every replay, as decode graphs do."""
    rnd = random.Random(3)
    B, n, cap, s0 = 2, 3, 256, 100
    u = _Setup("gqa_rotary", cache, 61 + (cache == "fp8"), cap)
    c, sh = u.paged(B, cap, fork=n, prompt_len=s0), u.static(B * n, cap)
    layer, slayer = c.layer(0), sh.layer(0)
    x = u.proj(B, s0)
    c.reserve(s0)
    u.append(layer, x)
    u.append(slayer, x.repeat_interleave(n, 0))
    c.advance(s0)
    sh.advance(s0)
    c.fork(n)
    _after(c, sh)
    static = u.proj(B * n, 1)
    c.reserve(1)
    graph = torch.cuda.CUDAGraph()
    rec.take()
    with torch.cuda.graph(graph):
        q = u.append(layer, static)
        out = layer.attend(q, scale=u.scale)
    assert rec.take() == [("decode_attn_paged", u.fp8)]
    worst = 0.0
    for i in range(24):
        op = ("step", "reorder", "rollback", "step")[i % 4] if i else "step"
        if op == "reorder":
            idx = torch.tensor([rnd.randrange(B * n) for _ in range(B * n)], device=DEV)
            c.reorder_(idx)
            sh.reorder_(idx)
        elif op == "rollback":
            k = rnd.randint(0, 5)
            c.rollback(k)
            sh.rollback(k)
        if op != "step":
            _after(c, sh)
        past = c.length
        x = u.proj(B * n, 1)
        static.copy_(x)
        c.reserve(1)
        graph.replay()
        sq = u.append(slayer, x)
        c.advance(1)
        sh.advance(1)
        assert torch.equal(q, sq)
        what = f"graph {cache} replay={i} past={past}"
        worst = max(worst, _check_attention(out.clone(), sq, sh, slice(None), past, c.kv_start, scale=u.scale,
                                            kernel="decode", what=what))
        _after(c, sh)
    # outside the graph only the shadow's appends and the copies on write ran, and there were copies
    calls = [x[0] for x in rec.take()]
    assert set(calls) == {"kv_page_copy"}, calls
    print(f"\n[paged graph] {cache}: max|o - ref| / bound = {worst:.3f}")


# ----------------------------------------------------------------------------------------------- 4. a long window
@pytest.mark.parametrize("heads", sorted(HEADS))
@pytest.mark.parametrize("cache", CACHES)
def test_long_window_on_scattered_pages(rec, cache, heads):
    """A 1,990-row prefill on 32 pages taken from a shuffled free list (no two consecutive logical pages adjacent in
    the pool), then 5 new tokens read by the decode kernel at 1, 2, 7 and an automatic number of splits."""
    B, cap, s0, s = 2, 2048, 1990, 5
    u = _Setup(heads, cache, 71 + len(heads) + (cache == "fp8"), cap)
    c, sh = u.paged(B, cap), u.static(B, cap)
    layer, slayer = c.layer(0), sh.layer(0)
    # a shuffled free list (pages go from its end, slot by slot, sequence by sequence) on which no sequence gets two
    # adjacent pages for two consecutive slots; the table is checked after the prefill
    rnd, M = random.Random(8), -(-(s0 + s) // P)
    while True:
        rnd.shuffle(c.free)
        order = c.free[::-1]
        if all(abs(a - b) != 1 for r in range(B) for a, b in zip(order[r::B][:M], order[r::B][1:M])):
            break
    pad = [0, 77]
    mask = torch.ones(B, s0, dtype=torch.long, device=DEV)
    mask[1, : pad[1]] = 0
    assert c.step_needs_dense_mask(mask, flash=c.flash_attention()) is False
    assert sh.step_needs_dense_mask(mask, flash=sh.flash_attention()) is False
    worst = 0.0
    for new in (s0, s):
        past = c.length
        x = u.proj(B, new, pad if past == 0 else None)
        c.reserve(new)
        q = u.append(layer, x)
        assert torch.equal(q, u.append(slayer, x))
        rec.take()
        if past == 0:
            assert all(abs(a - b) != 1 for row in c.host_table[:B] for a, b in zip(row[: c.mapped], row[1: c.mapped]))
            o = layer.attend(q, scale=u.scale, alibi_slopes=u.slopes)
            want, kernel = _want(u.fp8, new, 0, u.alibi)
            assert rec.take() == want
            worst = max(worst, _check_attention(o, q, sh, slice(None), 0, c.kv_start, scale=u.scale, kernel=kernel,
                                                slopes=u.slopes, what=f"long prefill {cache} {heads}"))
        else:
            scales = {} if not u.fp8 else {"k_scale": c.k_scale[0], "v_scale": c.v_scale[0]}
            for splits in (1, 2, 7, 0):
                o = OF.decode_attention(q, c.k[0], c.v[0], c.seqlens, c.kv_start, scale=u.scale, splits=splits,
                                        past=past, alibi_slopes=u.slopes, block_table=c.block_table, **scales)
                assert rec.take() == [("decode_attn_paged", u.fp8)]
                worst = max(worst, _check_attention(o, q, sh, slice(None), past, c.kv_start, scale=u.scale,
                                                    kernel="decode", slopes=u.slopes,
                                                    what=f"long decode {cache} {heads} splits={splits}"))
        c.advance(new)
        sh.advance(new)
        _after(c, sh)
    print(f"\n[paged long window] {cache} {heads}: max|o - ref| / bound = {worst:.3f}")
