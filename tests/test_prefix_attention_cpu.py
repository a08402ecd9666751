"""Prefix-LM attention without a GPU: the visibility rule of ``prefix_lens`` (``OF.visible_keys``, the reference
path of ``OF.attention``) against brute force and GLM's ``build_mask_matrix``, and Python mirrors of the flash
kernels' schedule (libai_b200/csrc/attention_sm90.cu, PREFIX instances): the forward's key-tile range and element
mask, the backward's (key block, query block) visits, ``last_kb`` and the ordered dQ counter protocol."""
import itertools
import random

import pytest
import torch

from libai_b200.ops import functional as OF
from projects.GLM.modeling_glm import GLMModel

PREFIXES = (0, 1, 63, 64, 65, 127, 128)


def brute_visible(i, j, *, sq, sk, pre, kv_start=0, kv_len=None):
    kv_len = sk if kv_len is None else max(1, kv_len)
    return kv_start <= j < kv_len and (j <= i + sk - sq or j < pre)


def rule(sq, sk, pre, kv_start=None, kv_len=None):
    return torch.tensor([[[brute_visible(i, j, sq=sq, sk=sk, pre=p, kv_start=0 if kv_start is None else kv_start[b],
                                         kv_len=None if kv_len is None else kv_len[b])
                           for j in range(sk)] for i in range(sq)] for b, p in enumerate(pre)])


@pytest.mark.parametrize("sq,sk", [(1, 1), (5, 5), (7, 12), (1, 9), (70, 70), (33, 130)])
def test_visible_keys_matches_brute_force(sq, sk):
    pre = [0, 1, sk // 2, sk, sk + 5]
    kv_start, kv_len = [0, 2, 1, 0, 3], [sk, sk - 1, sk, 2, sk]
    got = OF.visible_keys(sq, sk, causal=True, prefix_lens=torch.tensor(pre, dtype=torch.int32),
                          kv_start=torch.tensor(kv_start, dtype=torch.int32), kv_lens=torch.tensor(kv_len, dtype=torch.int32))
    assert torch.equal(got[:, 0], rule(sq, sk, pre, kv_start, kv_len))
    got = OF.visible_keys(sq, sk, causal=True, prefix_lens=torch.tensor(pre, dtype=torch.int32))
    assert torch.equal(got[:, 0], rule(sq, sk, pre))


def test_visible_keys_prefix_needs_causal():
    with pytest.raises(ValueError):
        OF.visible_keys(4, 4, causal=False, prefix_lens=torch.zeros(1, dtype=torch.int32))
    q = torch.zeros(1, 1, 4, 8)
    with pytest.raises(ValueError):
        OF.attention(q, q, q, causal=False, prefix_lens=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError):
        OF.attention(q, q, q, causal=True, alibi_slopes=torch.ones(1), prefix_lens=torch.zeros(1, dtype=torch.int32))


@pytest.mark.parametrize("mem", [0, 3, 17])
@pytest.mark.parametrize("q", [1, 6, 20])
def test_visible_keys_equals_build_mask_matrix(q, mem):
    """GLM's context of ``sep`` tokens after ``mem`` memories is the prefix ``mem + sep`` in key coordinates."""
    for sep in (0, 1, q // 2, q, [0, q // 3, q, 1]):
        b = 4
        sep_t = torch.tensor(sep).expand(b) if isinstance(sep, int) else torch.tensor(sep)
        want = GLMModel.build_mask_matrix(b, q, torch.tensor(sep), mem)
        got = OF.visible_keys(q, q + mem, causal=True, prefix_lens=(sep_t + mem).to(torch.int32))
        assert torch.equal(got.expand_as(want), want), sep


@pytest.mark.parametrize("sq,sk,g", [(9, 9, 2), (5, 13, 1), (16, 40, 2)])
def test_reference_attention_with_prefix_matches_brute_force(sq, sk, g):
    torch.manual_seed(0)
    b, a, d = 3, 4, 8
    q, k, v = torch.randn(b, a, sq, d), torch.randn(b, g, sk, d), torch.randn(b, g, sk, d)
    pre, kv_start = [0, sk // 2, sk + 1], [0, 2, 1]
    o = OF.attention(q, k, v, causal=True, prefix_lens=torch.tensor(pre, dtype=torch.int32),
                     kv_start=torch.tensor(kv_start, dtype=torch.int32))
    vis = rule(sq, sk, pre, kv_start)
    kk, vv = k.double().repeat_interleave(a // g, 1), v.double().repeat_interleave(a // g, 1)
    s = (q.double() @ kk.transpose(-1, -2)) / d ** 0.5
    s = s.masked_fill(~vis[:, None], float("-inf"))
    p = torch.softmax(s, -1).nan_to_num(0.0)
    want = p @ vv
    torch.testing.assert_close(o.double(), want, atol=1e-5, rtol=1e-5)


# ------------------------------------------------------------------------------------------------ forward mirror
BM = BN = 128


def fwd_cta(q_blk, *, sq, sk, pre, kv_beg, kv_len):
    """The key tiles a forward CTA loads and, per tile, whether it applies the element mask (attn_fwd_cta)."""
    off, q0 = sk - sq, q_blk * BM
    pre = min(max(pre, 0), sk)
    key_end = min(kv_len, max(min(q0 + BM, sq) + off, pre))
    j0 = kv_beg // BN
    nkv = max(0, (key_end + BN - 1) // BN - j0)
    tiles = []
    for j in range(j0, j0 + nkv):
        kbase = j * BN
        need = kbase < kv_beg or kbase + BN > kv_len or (kbase + BN - 1 > q0 + off and kbase + BN > pre)
        tiles.append((j, need))
    return tiles


def fwd_row_limit(i, *, sq, sk, pre, kv_beg, kv_len):
    """keys kv_beg .. kv_beg + vis_len - 1 of row i (the kernel's one unsigned comparison per element)"""
    return kv_beg, max(0, min(kv_len, max(i + sk - sq + 1, min(max(pre, 0), sk))) - kv_beg)


FWD_SHAPES = [(1, 1), (5, 5), (128, 128), (129, 129), (200, 200), (64, 300), (300, 300), (1, 257), (130, 500)]


@pytest.mark.parametrize("sq,sk", FWD_SHAPES)
def test_forward_tiles_cover_every_visible_key(sq, sk):
    for pre in (*PREFIXES, sk // 4, sk // 2, sk, sk + 7):
        for kv_beg, kv_len in ((0, sk), (min(3, sk - 1), sk), (0, max(1, sk - 70)), (min(130, sk - 1), sk)):
            for q_blk in range((sq + BM - 1) // BM):
                tiles = dict(fwd_cta(q_blk, sq=sq, sk=sk, pre=pre, kv_beg=kv_beg, kv_len=kv_len))
                for i in range(q_blk * BM, min(sq, q_blk * BM + BM)):
                    beg, n = fwd_row_limit(i, sq=sq, sk=sk, pre=pre, kv_beg=kv_beg, kv_len=kv_len)
                    for j in range(sk):
                        vis = brute_visible(i, j, sq=sq, sk=sk, pre=pre, kv_start=kv_beg, kv_len=kv_len)
                        assert vis == (0 <= j - beg < n), (i, j, pre)
                        if vis:
                            assert j // BN in tiles, (q_blk, i, j, pre, kv_beg, kv_len)
                    for j, need in tiles.items():   # an unmasked tile is visible to every row in full
                        if not need:
                            assert all(brute_visible(i, jj, sq=sq, sk=sk, pre=pre, kv_start=kv_beg, kv_len=kv_len)
                                       for jj in range(j * BN, j * BN + BN)), (i, j, pre)


def test_forward_prefix_zero_and_full_match_causal_and_full_ranges():
    """The two bit-identities start here: with prefix 0 the tile range and masks are the causal kernel's, with a
    prefix >= Sk the non-causal kernel's."""
    for sq, sk in FWD_SHAPES:
        for q_blk in range((sq + BM - 1) // BM):
            q0, off = q_blk * BM, sk - sq
            causal_end = min(sk, min(q0 + BM, sq) + off)
            causal = [(j, j * BN + BN > sk or j * BN + BN - 1 > q0 + off) for j in range(max(0, (causal_end + BN - 1) // BN))]
            full = [(j, j * BN + BN > sk) for j in range((sk + BN - 1) // BN)]
            assert fwd_cta(q_blk, sq=sq, sk=sk, pre=0, kv_beg=0, kv_len=sk) == causal
            assert fwd_cta(q_blk, sq=sq, sk=sk, pre=sk, kv_beg=0, kv_len=sk) == full
            assert fwd_cta(q_blk, sq=sq, sk=sk, pre=sk + 9, kv_beg=0, kv_len=sk) == full


# ------------------------------------------------------------------------------------------------ backward mirror
B64 = 64


def first_qblock(kb, *, sq, sk, pre):
    if kb * B64 < pre:
        return 0
    return max(0, int((kb * B64 - (sk - sq)) / B64))   # C division truncates towards 0


def visits(kb, qb, *, sq, sk, pre):
    nkb = (sk + B64 - 1) // B64
    return kb < nkb and qb >= first_qblock(kb, sq=sq, sk=sk, pre=pre)


def last_kb(qb, *, sq, sk, pre):
    nkb = (sk + B64 - 1) // B64
    c = min(nkb - 1, int((qb * B64 + B64 - 1 + sk - sq) / B64))
    return min(nkb - 1, max(c, (pre + B64 - 1) // B64 - 1))


BWD_SHAPES = [(s, t) for s in (1, 5, 64, 65, 128, 130, 200) for t in (1, 7, 64, 65, 128, 129, 200, 257) if s <= t]


def clamp_pre(pre, sk):
    return min(max(pre, 0), sk)


@pytest.mark.parametrize("sq,sk", BWD_SHAPES)
def test_backward_visits_cover_every_visible_pair(sq, sk):
    nq, nkb = (sq + B64 - 1) // B64, (sk + B64 - 1) // B64
    for raw in (*PREFIXES, sk, sk + 5):
        pre = clamp_pre(raw, sk)
        for qb in range(nq):
            meet = [kb for kb in range(nkb) if visits(kb, qb, sq=sq, sk=sk, pre=pre)]
            # the issue's meeting rule, and monotone in the key block
            assert meet == [kb for kb in range(nkb) if 64 * kb <= 64 * qb + 63 + sk - sq or 64 * kb < pre]
            assert meet == list(range(len(meet)))
            if meet:
                assert last_kb(qb, sq=sq, sk=sk, pre=pre) == meet[-1]
        for i, j in itertools.product(range(sq), range(sk)):
            if brute_visible(i, j, sq=sq, sk=sk, pre=pre):
                assert visits(j // B64, i // B64, sq=sq, sk=sk, pre=pre), (i, j, pre)


@pytest.mark.parametrize("sq,sk", BWD_SHAPES)
def test_backward_prefix_zero_and_full_match_causal_and_full_schedules(sq, sk):
    nq, nkb = (sq + B64 - 1) // B64, (sk + B64 - 1) // B64
    for kb in range(nkb):
        assert first_qblock(kb, sq=sq, sk=sk, pre=0) == max(0, int((kb * B64 - (sk - sq)) / B64))
        assert first_qblock(kb, sq=sq, sk=sk, pre=sk) == 0
    for qb in range(nq):
        assert last_kb(qb, sq=sq, sk=sk, pre=0) == min(nkb - 1, int((qb * B64 + B64 - 1 + sk - sq) / B64))
        assert last_kb(qb, sq=sq, sk=sk, pre=sk) == nkb - 1


def simulate_dq_order(sq, sk, pre, nwg, r, seed):
    """Every CTA (NWG consecutive key blocks) walks its visit sequence; its writer adds the partials of a visit from
    the highest key block down, each after the counter of (query head, query block) reached last_kb - kb, and then
    releases it.  CTAs interleave at random; returns the order in which key blocks added to each query block, or
    raises on a state in which no CTA can move."""
    rng = random.Random(seed)
    nq, nkb = (sq + B64 - 1) // B64, (sk + B64 - 1) // B64
    ctas = []
    for cta in range((nkb + nwg - 1) // nwg):
        kb0 = nwg * cta
        i_begin = first_qblock(kb0, sq=sq, sk=sk, pre=pre)
        seq = []
        for hi in range(r):
            for qb in range(i_begin, nq):
                kbs = [kb0 + w for w in reversed(range(nwg)) if visits(kb0 + w, qb, sq=sq, sk=sk, pre=pre)]
                if kbs:
                    seq.append((hi, qb, kbs))
        ctas.append(seq)
    counter = {}
    added = {}
    pos = [0] * len(ctas)
    while any(pos[c] < len(ctas[c]) for c in range(len(ctas))):
        ready = []
        for c, seq in enumerate(ctas):
            if pos[c] < len(seq):
                hi, qb, kbs = seq[pos[c]]
                if counter.get((hi, qb), 0) >= last_kb(qb, sq=sq, sk=sk, pre=pre) - kbs[0]:
                    ready.append(c)
        assert ready, "every writer waits: the dQ order would never complete"
        c = rng.choice(ready)
        hi, qb, kbs = ctas[c][pos[c]]
        added.setdefault((hi, qb), []).extend(kbs)
        counter[(hi, qb)] = counter.get((hi, qb), 0) + len(kbs)
        pos[c] += 1
    return added, nq, nkb


@pytest.mark.parametrize("nwg", [1, 2])
@pytest.mark.parametrize("sq,sk", [(s, t) for s, t in BWD_SHAPES if t >= 64])
def test_backward_dq_counter_adds_in_decreasing_key_order(sq, sk, nwg):
    for raw in (*PREFIXES, sk, sk + 5):
        pre = clamp_pre(raw, sk)
        for seed in range(3):
            added, nq, nkb = simulate_dq_order(sq, sk, pre, nwg, r=2, seed=seed)
            for hi, qb in itertools.product(range(2), range(nq)):
                want = [kb for kb in reversed(range(nkb)) if visits(kb, qb, sq=sq, sk=sk, pre=pre)]
                assert added.get((hi, qb), []) == want, (pre, hi, qb)
