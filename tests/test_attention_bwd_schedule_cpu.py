"""The warp-specialised flash backward without a GPU: a mirror of which consumer warpgroup of a CTA makes or lets pass
which (query head, query block) visit, and of the dQ writer's ordering, run under random interleavings of the CTAs'
writers with a bounded number of resident CTAs; and the ptxas figures of the backward instances."""
import os
import random
import re
import subprocess

import pytest

from libai_b200.ops import build as ops_build

BN = BM = 64   # keys per consumer warpgroup, queries per visit
NWG = 2        # consumer warpgroups per CTA of the head-dim-64 instances without dropout


def _cdiv(a, b):
    return -(-a // b)


def first_qblock(kb, sq, sk, causal):
    """bwd_first_qblock: the first query block key block kb meets (C division truncates towards 0, then max 0)."""
    return max(0, int((kb * BN - (sk - sq)) / BM)) if causal else 0


def doc_begin(ds, i):
    return min(max(ds[i], 0), i)


def visit_empty(ds, sq, kb, qb):
    """doc_visit_empty: every row of the query block (rows past Sq repeat the last one) starts its document after the
    key block."""
    rows = [min(qb * BM + t, sq - 1) for t in range(BM)]
    return min(doc_begin(ds, i) for i in rows) >= kb * BN + BN


def visits(kb, qb, nkb, sq, sk, causal, ds):
    """bwd_visits: whether key block kb makes the visit of query block qb."""
    if kb >= nkb or qb < first_qblock(kb, sq, sk, causal):
        return False
    return ds is None or not visit_empty(ds, sq, kb, qb)


def wait_target(kb, qb, nkb, sq, sk, causal):
    last_kb = min(nkb - 1, (qb * BM + BM - 1 + sk - sq) // BN) if causal else nkb - 1
    return last_kb - kb


def cta_schedule(cta, r, sq, sk, causal, ds, nwg=NWG):
    """One CTA's visit sequence: (query head, query block, loaded, [key blocks that make it]).  The writer's tasks are
    the (head, query block, key block) triples in this order, the higher key block of a visit first."""
    nkb, nq = _cdiv(sk, BN), _cdiv(sq, BM)
    kb0 = nwg * cta
    out = []
    for hi in range(r):
        for qb in range(first_qblock(kb0, sq, sk, causal), nq):
            makers = [kb0 + w for w in reversed(range(nwg)) if visits(kb0 + w, qb, nkb, sq, sk, causal, ds)]
            out.append((hi, qb, bool(makers), makers))
    return out


def run_writers(r, sq, sk, causal, ds, rng, resident, nwg=NWG):
    """CTAs are dispatched in increasing linear index (highest key blocks first), at most `resident` at a time; a
    dispatched CTA's writer runs its visits in order: it waits until the (head, query block) counter reached the wait
    target of the visit's highest contributing key block, adds that block's partial and then the lower ones' (each
    complete before the next starts), and releases the counter once, by the number of partials.  Among the writers
    that can proceed one is picked at random.  Returns, per (head, query block), the key blocks in the order their
    partials landed; fails on a deadlock."""
    nkb, nq = _cdiv(sk, BN), _cdiv(sq, BM)
    ncta = _cdiv(nkb, nwg)
    tasks = []
    for idx in range(ncta):          # linear index idx runs CTA ncta - 1 - idx
        cta = ncta - 1 - idx
        tasks.append([(hi, qb, makers) for hi, qb, _, makers in cta_schedule(cta, r, sq, sk, causal, ds, nwg) if makers])
    counter = {}
    landed = {}
    nxt, live = 0, []
    while nxt < ncta or live:
        while len(live) < resident and nxt < ncta:
            live.append([nxt, 0])
            nxt += 1
        ready = []
        for slot in live:
            idx, pos = slot
            if pos == len(tasks[idx]):
                ready.append(slot)
                continue
            hi, qb, makers = tasks[idx][pos]
            if counter.get((hi, qb), 0) >= wait_target(makers[0], qb, nkb, sq, sk, causal):
                ready.append(slot)
        assert ready, ("deadlock", sq, sk, causal, live)
        slot = rng.choice(ready)
        idx, pos = slot
        if pos == len(tasks[idx]):
            live.remove(slot)
            continue
        hi, qb, makers = tasks[idx][pos]
        for i, kb in enumerate(makers):   # each partial lands exactly when its block's wait target is reached
            assert counter.get((hi, qb), 0) + i == wait_target(kb, qb, nkb, sq, sk, causal)
            landed.setdefault((hi, qb), []).append(kb)
        counter[(hi, qb)] = counter.get((hi, qb), 0) + len(makers)
        slot[1] += 1
    return landed


def doc_layout(S, rng):
    """Non-monotone document starts: runs of random length, some rows pointing anywhere (clamped by the kernel)."""
    ds, at = [], 0
    while at < S:
        n = rng.randint(1, 150)
        ds += [at] * min(n, S - at)
        at += n
    return [rng.randint(-10, S + 10) if rng.random() < 0.1 else x for x in ds]


SHAPES = [(1, 1), (65, 65), (129, 129), (300, 1), (77, 203), (203, 77), (1, 300), (200, 200), (64, 448), (517, 517)]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_each_key_block_makes_the_visits_it_made_alone(causal, shape):
    """Warpgroup w of CTA c makes exactly the visits its key block made as a CTA of its own, in the same order."""
    sq, sk = shape
    nkb = _cdiv(sk, BN)
    for cta in range(_cdiv(nkb, NWG)):
        sched = cta_schedule(cta, 2, sq, sk, causal, None)
        for w in range(NWG):
            kb = NWG * cta + w
            made = [(hi, qb) for hi, qb, _, makers in sched if kb in makers]
            alone = [(hi, qb) for hi in range(2) for qb in range(first_qblock(kb, sq, sk, causal), _cdiv(sq, BM))]
            assert made == (alone if kb < nkb else []), (shape, kb)
        # a visit is loaded iff some warpgroup makes it; the lowest key block makes every loaded visit without DOC
        assert all(loaded == bool(makers) for _, _, loaded, makers in sched)
        assert all(NWG * cta in makers for _, _, loaded, makers in sched if loaded)


@pytest.mark.parametrize("resident", [1, 2, 5])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_writers_land_partials_in_decreasing_key_block_order(resident, causal, shape):
    sq, sk = shape
    rng = random.Random(hash((resident, causal, shape)) & 0xFFFF)
    nkb = _cdiv(sk, BN)
    for _ in range(5):
        landed = run_writers(2, sq, sk, causal, None, rng, resident)
        for (hi, qb), kbs in landed.items():
            want = [kb for kb in reversed(range(nkb)) if visits(kb, qb, nkb, sq, sk, causal, None)]
            assert kbs == want, (shape, hi, qb, kbs)


@pytest.mark.parametrize("S", [65, 129, 256, 300, 517, 1000])
def test_writers_with_packed_documents(S):
    rng = random.Random(S)
    nkb = _cdiv(S, BN)
    for _ in range(3):
        ds = doc_layout(S, rng)
        for resident in (1, 3):
            landed = run_writers(1, S, S, True, ds, rng, resident)
            for (_, qb), kbs in landed.items():
                want = [kb for kb in reversed(range(nkb)) if visits(kb, qb, nkb, S, S, True, ds)]
                assert kbs == want and kbs, (S, qb, kbs)
                # a skipped visit lies below every contributing one, so the wait targets count contributors only
                skipped = [kb for kb in range(nkb) if kb <= wait_target(0, qb, nkb, S, S, True) and kb not in kbs]
                assert all(kb < min(kbs) for kb in skipped)


def test_one_warpgroup_per_cta_is_the_same_protocol():
    """The instances with one consumer warpgroup run the same writer protocol with one key block per CTA."""
    rng = random.Random(7)
    for sq, sk in SHAPES:
        landed = run_writers(2, sq, sk, True, None, rng, 1, nwg=1)
        nkb = _cdiv(sk, BN)
        for (_, qb), kbs in landed.items():
            assert kbs == [kb for kb in reversed(range(nkb)) if visits(kb, qb, nkb, sq, sk, True, None)]


# ------------------------------------------------------------------------------------------------ build
# spill stores (bytes) of the head-dim-128 backward instances with one consumer warpgroup per 64-key block and the
# lse / δ rows read from global memory, by (bias, dropout, packed)
PREVIOUS_D128_SPILLS = {(2, 0, 0): 84, (2, 1, 0): 172, (1, 0, 0): 108, (1, 1, 0): 208, (0, 0, 0): 76, (0, 1, 0): 152,
                        (0, 0, 1): 100}


@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_backward_instances_compile_without_new_spills(tmp_path):
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, "attention_sm90.cu"), "-o", str(tmp_path / "attn.o")],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    assert not ops_build.serialized_wgmma(res.stdout)
    spills, name = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r"Compiling entry function '\S*attn_bwd_kernelILi(\d+)ELi(\d)ELb(\d)ELb(\d)E", line)
        if m:
            name = tuple(int(x) for x in m.groups())
        elif "Compiling entry function" in line:
            name = None
        elif name and "spill stores" in line:
            spills[name] = int(re.search(r"(\d+) bytes spill stores", line).group(1))
            name = None
    assert len(spills) == 14, spills
    for (d, bias, drop, doc), n in spills.items():
        if d == 128:
            assert n <= PREVIOUS_D128_SPILLS[(bias, drop, doc)], (d, bias, drop, doc, n)
        else:
            assert n == 0, (d, bias, drop, doc, n)
