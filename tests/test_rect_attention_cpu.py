"""Rectangular attention on the CPU: the reference semantics of per-sample key windows (``kv_start`` / ``kv_lens``) and
bottom-right causal alignment against a brute-force per-element mask, a pure-Python mirror of the flash kernels' block
iteration (forward key-tile range and mask test, backward query-block range and the ordered-dQ counters) checked
exhaustively over small shapes, and, with nvcc, the sm_90a build of the attention kernels."""
import itertools
import math
import os
import re
import subprocess

import pytest
import torch

from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF


def _visible(i, j, sq, sk, causal, start, lens):
    """The visibility rule, one element at a time."""
    end = sk if lens is None else max(1, min(sk, lens))
    beg = 0 if start is None else min(max(start, 0), sk)
    return beg <= j < end and (not causal or j <= i + sk - sq)


# ------------------------------------------------------------------------------------------------ reference semantics
@pytest.mark.parametrize("sq,sk", [(1, 1), (1, 7), (5, 3), (3, 5), (6, 6), (9, 4)])
@pytest.mark.parametrize("causal", [False, True])
def test_visible_keys_matches_elementwise_rule(sq, sk, causal):
    for start, lens in itertools.product(range(sk + 1), [None, *range(sk + 1)]):
        st = torch.tensor([start, 0], dtype=torch.int32)
        ln = None if lens is None else torch.tensor([lens, sk], dtype=torch.int32)
        vis = OF.visible_keys(sq, sk, causal=causal, kv_start=st, kv_lens=ln)
        assert vis.shape == (2, 1, sq, sk)
        for i, j in itertools.product(range(sq), range(sk)):
            assert bool(vis[0, 0, i, j]) == _visible(i, j, sq, sk, causal, start, lens)
            assert bool(vis[1, 0, i, j]) == _visible(i, j, sq, sk, causal, 0, None if lens is None else sk)


def _bruteforce(q, k, v, scale, causal, start, lens, bias=None):
    """Per-row softmax over exactly the visible keys, in float64; zeros for a row without one."""
    b, a, sq, d = q.shape
    g, sk = k.shape[1], k.shape[2]
    out = torch.zeros(b, a, sq, d, dtype=torch.float64)
    for bi, h, i in itertools.product(range(b), range(a), range(sq)):
        keys = [j for j in range(sk) if _visible(i, j, sq, sk, causal, start[bi], None if lens is None else lens[bi])]
        if not keys:
            continue
        kh = h // (a // g)
        s = (k[bi, kh, keys].double() @ q[bi, h, i].double()) * scale
        if bias is not None:
            s = s + bias[bi % bias.shape[0], h % bias.shape[1], i, keys].double()
        out[bi, h, i] = torch.softmax(s, 0) @ v[bi, kh, keys].double()
    return out


@pytest.mark.parametrize("sq,sk", [(1, 9), (4, 11), (11, 4), (7, 7)])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("groups", [4, 2, 1])
def test_reference_with_kv_start_matches_bruteforce(sq, sk, causal, groups):
    torch.manual_seed(sq * 100 + sk)
    b, a, d = 3, 4, 8
    q, k, v = torch.randn(b, a, sq, d), torch.randn(b, groups, sk, d), torch.randn(b, groups, sk, d)
    start = [0, min(2, sk - 1), sk - 1]
    lens = [sk, sk, max(1, sk - 2)]
    bias = torch.randn(1, a, sq, sk)
    st, ln = torch.tensor(start, dtype=torch.int32), torch.tensor(lens, dtype=torch.int32)
    for bb in (None, bias):
        o = OF.attention(q, k, v, causal=causal, scale=0.3, kv_start=st, kv_lens=ln, bias=bb)
        ref = _bruteforce(q, k, v, 0.3, causal, start, lens, bb)
        torch.testing.assert_close(o.double(), ref, atol=1e-5, rtol=1e-5)
        assert torch.isfinite(o).all()


def test_reference_rows_without_keys_are_zero_with_zero_gradient():
    torch.manual_seed(0)
    q = torch.randn(2, 2, 6, 8, requires_grad=True)
    k = torch.randn(2, 2, 4, 8, requires_grad=True)
    v = torch.randn(2, 2, 4, 8, requires_grad=True)
    st = torch.tensor([0, 3], dtype=torch.int32)
    # causal with Sq > Sk: rows 0, 1 see no key (j <= i - 2); sample 1 also hides keys 0..2
    o = OF.attention(q, k, v, causal=True, scale=0.5, kv_start=st)
    assert (o[:, :, :2] == 0).all() and (o[1, :, :5] == 0).all()
    o.sum().backward()
    assert (q.grad[:, :, :2] == 0).all() and (q.grad[1, :, :5] == 0).all()
    assert (k.grad[1, :, :3] == 0).all() and (v.grad[1, :, :3] == 0).all()
    assert all(torch.isfinite(t.grad).all() for t in (q, k, v))


def test_reference_alibi_uses_bottom_right_alignment():
    torch.manual_seed(1)
    q, k, v = torch.randn(1, 2, 3, 8), torch.randn(1, 2, 7, 8), torch.randn(1, 2, 7, 8)
    slopes = torch.tensor([0.5, 0.25])
    o = OF.attention(q, k, v, causal=True, scale=0.2, alibi_slopes=slopes, kv_start=torch.zeros(1, dtype=torch.int32))
    rel = torch.arange(7)[None, :] - (torch.arange(3)[:, None] + 4)
    bias = slopes[None, :, None, None] * rel[None, None].float()
    torch.testing.assert_close(o.double(), _bruteforce(q, k, v, 0.2, True, [0], None, bias), atol=1e-5, rtol=1e-5)


def test_reference_without_kv_start_is_unchanged():
    torch.manual_seed(2)
    q, k, v = torch.randn(2, 2, 5, 8), torch.randn(2, 2, 9, 8), torch.randn(2, 2, 9, 8)
    for causal in (False, True):
        assert torch.equal(OF.attention(q, k, v, causal=causal, scale=0.3),
                           OF.attention_ref(q, k, v, causal=causal, scale=0.3))


def test_attention_supported_is_false_off_the_gpu():
    q = torch.randn(1, 2, 3, 64, dtype=torch.bfloat16)
    assert not OF.attention_supported(q, q)


def test_prep_bias_pads_rows_to_a_multiple_of_8():
    # contiguous, and heads innermost in memory (T5's relative-position bias is a permuted gather)
    for bias in (torch.randn(2, 3, 5, 13), torch.randn(2, 5, 13, 3).permute(0, 3, 1, 2)):
        b = OF._prep_bias(bias, None)
        assert b.dtype == torch.bfloat16 and b.shape == bias.shape and b.stride(-2) == 16 and b.stride(-1) == 1
        assert torch.equal(b.float(), bias.to(torch.bfloat16).float())
    aligned = torch.randn(1, 2, 4, 16, dtype=torch.bfloat16)
    assert OF._prep_bias(aligned, None) is aligned


# ------------------------------------------------------------------------------------------------ kernel mirror
# Integer arithmetic of attention_sm90.cu, written with C semantics (division truncates towards zero).
def _cdiv(a, b):
    return int(a / b) if (a < 0) != (b < 0) else a // b


def fwd_tiles(q_blk, sq, sk, causal, start, lens, bm, bn):
    """attn_fwd_kernel: the key tiles a CTA loads and, per tile, whether it applies the element mask."""
    q0 = q_blk * bm
    kv_len = max(1, min(sk, lens)) if lens is not None else sk
    kv_beg = min(max(start, 0), sk) if start is not None else 0
    off = sk - sq
    key_end = min(kv_len, min(q0 + bm, sq) + off) if causal else kv_len
    j0 = kv_beg // bn
    nkv = max(0, _cdiv(key_end + bn - 1, bn) - j0)
    tiles = []
    for j in range(j0, j0 + nkv):
        kbase = j * bn
        need_mask = kbase < kv_beg or kbase + bn > kv_len or (causal and kbase + bn - 1 > q0 + off)
        tiles.append((j, need_mask))
    return tiles


def bwd_query_blocks(kv_blk, sq, sk, causal, blk):
    """attn_bwd_kernel: the query blocks key block kv_blk visits (shapes only)."""
    nq = _cdiv(sq + blk - 1, blk)
    off = sk - sq
    i_begin = max(0, _cdiv(kv_blk * blk - off, blk)) if causal else 0
    return list(range(i_begin, nq))


def bwd_wait_target(kv_blk, q_blk, sq, sk, causal, blk):
    """attn_bwd_kernel: the dq_order count key block kv_blk waits for before adding its dQ share of query block q_blk."""
    nkb = _cdiv(sk + blk - 1, blk)
    off = sk - sq
    last_kb = min(nkb - 1, _cdiv(q_blk * blk + blk - 1 + off, blk)) if causal else nkb - 1
    return last_kb - kv_blk


def _shapes(limit):
    return [(sq, sk) for sq in range(1, limit) for sk in range(1, limit)]


@pytest.mark.parametrize("causal", [False, True])
def test_forward_tile_range_covers_every_visible_key(causal):
    bm = bn = 4
    for sq, sk in _shapes(14):
        for start, lens in itertools.product([None, *range(sk + 1)], [None, *range(sk + 1)]):
            for q_blk in range(_cdiv(sq + bm - 1, bm)):
                tiles = fwd_tiles(q_blk, sq, sk, causal, start, lens, bm, bn)
                loaded = {j for j, _ in tiles}
                rows = range(q_blk * bm, min(q_blk * bm + bm, sq))
                seen = {j for i in rows for j in range(sk) if _visible(i, j, sq, sk, causal, start, lens)}
                assert {j // bn for j in seen} <= loaded
                if seen:   # no tile outside [first visible, last visible] is loaded
                    assert min(loaded) == min(seen) // bn and max(loaded) == max(seen) // bn
                for j, need_mask in tiles:
                    if not need_mask:   # an unmasked tile is entirely visible to every row of the block
                        assert all(_visible(i, kk, sq, sk, causal, start, lens)
                                   for i in rows for kk in range(j * bn, j * bn + bn))


def _run_dq_order(sq, sk, causal, blk):
    """Simulate the backward's ordered dQ accumulation with every CTA resident: each CTA runs its steps in order and may
    add its share of query block i only once dq_order[i] reached its wait target.  Returns, per query block, the key
    blocks in the order they added, or raises on a deadlock or an overrun."""
    nkb = _cdiv(sk + blk - 1, blk)
    nq = _cdiv(sq + blk - 1, blk)
    steps = {kb: bwd_query_blocks(kb, sq, sk, causal, blk) for kb in range(nkb)}
    pos = {kb: 0 for kb in range(nkb)}
    order = [0] * nq
    added = [[] for _ in range(nq)]
    while any(pos[kb] < len(steps[kb]) for kb in range(nkb)):
        ran = False
        for kb in reversed(range(nkb)):   # highest key blocks are launched first
            if pos[kb] < len(steps[kb]):
                i = steps[kb][pos[kb]]
                target = bwd_wait_target(kb, i, sq, sk, causal, blk)
                assert order[i] <= target, (sq, sk, kb, i, "counter passed the wait target")
                if order[i] == target:
                    added[i].append(kb)
                    order[i] += 1
                    pos[kb] += 1
                    ran = True
        assert ran, (sq, sk, causal, "deadlock", pos, order)
    return added


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("blk", [4, 64])
def test_backward_dq_order_counting(causal, blk):
    limit = 14 if blk == 4 else 0
    shapes = _shapes(limit) if blk == 4 else [
        (sq, sk) for sq in (1, 7, 63, 64, 65, 127, 128, 129, 200, 512) for sk in (1, 9, 63, 64, 65, 128, 131, 400, 1000)]
    for sq, sk in shapes:
        nkb = _cdiv(sk + blk - 1, blk)
        added = _run_dq_order(sq, sk, causal, blk)
        for i, kbs in enumerate(added):
            # the visitors of query block i are key blocks 0 .. last, and they add in decreasing order
            assert kbs == list(range(len(kbs) - 1, -1, -1)), (sq, sk, i, kbs)
            if kbs:
                assert len(kbs) == bwd_wait_target(0, i, sq, sk, causal, blk) + 1
        for kb in range(nkb):   # every key block visits at least one query block, so it writes its dK / dV rows
            assert bwd_query_blocks(kb, sq, sk, causal, blk), (sq, sk, kb)


@pytest.mark.parametrize("causal", [False, True])
def test_backward_blocks_cover_every_visible_pair(causal):
    blk = 4
    for sq, sk in _shapes(14):
        visited = {(kb, i) for kb in range(_cdiv(sk + blk - 1, blk)) for i in bwd_query_blocks(kb, sq, sk, causal, blk)}
        for start, lens in itertools.product([None, *range(sk + 1)], [None, *range(sk + 1)]):
            for i, j in itertools.product(range(sq), range(sk)):
                if _visible(i, j, sq, sk, causal, start, lens):
                    assert (j // blk, i // blk) in visited


def test_square_problems_keep_the_original_iteration():
    """Sq == Sk: the key-tile count min(ceil(kv_len / 128), q_blk + 1), the query-block start k0 / 64 and the wait target
    q_blk - kv_blk (causal) of the square kernel."""
    for s in (64, 128, 192, 1024, 1000):
        for q_blk in range(math.ceil(s / 128)):
            for lens in (None, 1, 77, s):
                kv_len = s if lens is None else lens
                tiles = fwd_tiles(q_blk, s, s, True, None, lens, 128, 128)
                assert [j for j, _ in tiles] == list(range(min(math.ceil(kv_len / 128), q_blk + 1)))
                assert [m for _, m in tiles] == [j == q_blk or j * 128 + 128 > kv_len for j, _ in tiles]
        for kb in range(math.ceil(s / 64)):
            assert bwd_query_blocks(kb, s, s, True, 64)[0] == kb
            for i in bwd_query_blocks(kb, s, s, True, 64):
                assert bwd_wait_target(kb, i, s, s, True, 64) == i - kb


# ------------------------------------------------------------------------------------------------ build
@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_rectangular_attention_compiles_for_sm90a(tmp_path):
    """The rectangular kernels are the existing instantiations with runtime lengths and windows: the source compiles
    for sm_90a, wgmma stays asynchronous and the forward kernels do not spill."""
    src = "attention_sm90.cu"
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    assert ops_build.serialized_wgmma(res.stdout) == []
    spills = dict((name, (st, ld)) for name, st, ld in re.findall(
        r"Function properties for (\S+)\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads", res.stdout))
    fwd = {n: v for n, v in spills.items() if "attn_fwd_kernel" in n}
    assert len(fwd) == 12, res.stdout
    assert all(v == ("0", "0") for v in fwd.values()), fwd
