"""Packed-sequence SFT without a GPU: the reference semantics of a packed Llama batch (loss and gradients equal to the
same samples run one per row), a mirror of the flash kernels' tile-range and visit-skip arithmetic for ``doc_start``,
the packer, and ptxas figures of the packed-sequence kernel instances."""
import os
import random
import re
import subprocess

import pytest
import torch

from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF
from projects.common.sft import IGNORE_INDEX, PackedSFTDataset, pack_samples, sample_length

BM, BN = 128, 128          # forward: queries per CTA, keys per tile
BWD_BN, BWD_BM = 64, 64    # backward: keys per CTA, queries per visit


# ------------------------------------------------------------------------------------------------ kernel mirror
def doc_begin(doc_start, i):
    return min(max(doc_start[i], 0), i)


def fwd_tiles(doc_start, S, q_blk):
    """Key tiles a forward CTA loads: j0 from the minimum document start over the block's rows (rows past S repeat
    the last row), the end from the causal bound of the block's last row."""
    q0 = q_blk * BM
    blk_min = min(doc_begin(doc_start, min(q0 + t, S - 1)) for t in range(BM))
    j0 = blk_min // BN
    key_end = min(S, min(q0 + BM, S))
    return j0, max(0, (key_end + BN - 1) // BN - j0)


def bwd_visits(S):
    """(key block, query block) visits of the causal backward, as attn_bwd_kernel enumerates them."""
    nq, nk = (S + BWD_BM - 1) // BWD_BM, (S + BWD_BN - 1) // BWD_BN
    for kb in range(nk):
        i_begin = max(0, (kb * BWD_BN) // BWD_BM)
        for i in range(i_begin, nq):
            yield kb, i


def visit_empty(doc_start, S, kb, i):
    q0, k0 = i * BWD_BM, kb * BWD_BN
    m = min(doc_begin(doc_start, min(q0 + t, S - 1)) for t in range(BWD_BM))
    return m >= k0 + BWD_BN


def layouts(S, rng):
    """Document layouts of one row: packer-style (monotone) and arbitrary (non-monotone, out-of-range) doc_start."""
    out = [[0] * S, list(range(S))]   # one document; every token its own document
    for _ in range(3):
        ds, at = [], 0
        while at < S:
            n = rng.choice([1, 2, BN - 1, BN, BN + 1, rng.randint(1, 3 * BN)])
            ds += [at] * min(n, S - at)
            at += n
        out.append(ds)
    out.append([rng.randint(-5, S + 5) for _ in range(S)])
    out.append([i - rng.randint(0, 200) for i in range(S)])
    return out


@pytest.mark.parametrize("S", [1, 2, 63, 64, 65, 127, 128, 129, 255, 300, 517])
def test_mirror_tile_ranges_and_visit_skips(S):
    rng = random.Random(S)
    for ds in layouts(S, rng):
        vis = OF.visible_keys(S, S, causal=True, doc_start=torch.tensor([ds]))[0, 0]
        assert bool(vis.diagonal().all())   # every query sees itself
        # forward: every visible pair lies in a loaded tile
        for q_blk in range((S + BM - 1) // BM):
            j0, nkv = fwd_tiles(ds, S, q_blk)
            rows = vis[q_blk * BM : (q_blk + 1) * BM]
            keys = torch.nonzero(rows.any(0)).flatten()
            assert int(keys.min()) >= j0 * BN and int(keys.max()) < (j0 + nkv) * BN
        # backward: no visible pair in a skipped visit; every visit (skipped or not) counts once for the dQ order
        counts = {}
        for kb, i in bwd_visits(S):
            if visit_empty(ds, S, kb, i):
                assert not bool(vis[i * BWD_BM : (i + 1) * BWD_BM, kb * BWD_BN : (kb + 1) * BWD_BN].any())
            counts.setdefault(i, []).append(kb)
        for i, kbs in counts.items():
            last_kb = min((S + BWD_BN - 1) // BWD_BN - 1, (i * BWD_BM + BWD_BM - 1) // BWD_BN)
            # key block kb waits for last_kb - kb increments: exactly the visitors above it
            assert sorted(kbs) == list(range(last_kb + 1))


def dq_order_schedule(visitors, skipped, last_kb, rng, count_skipped=False):
    """One random interleaving of the CTAs that visit a query block under the dQ order protocol of attn_bwd_kernel: a
    contributing key block kb waits until the counter reaches last_kb - kb, adds its dQ share, then increments; a
    skipped visit does nothing (``count_skipped``: the rejected variant that increments without waiting).  Returns the
    key blocks in the order they added, or None when the remaining blocks can never proceed."""
    counter, order, todo = 0, [], list(visitors)
    while todo:
        ready = [kb for kb in todo if kb in skipped or counter >= last_kb - kb]
        if not ready:
            return None
        kb = rng.choice(ready)
        todo.remove(kb)
        if kb in skipped:
            counter += 1 if count_skipped else 0
        else:
            order.append(kb)
            counter += 1
    return order


@pytest.mark.parametrize("S", [65, 129, 256, 300, 517])
def test_mirror_dq_order_under_random_interleavings(S):
    rng = random.Random(1000 + S)
    for ds in layouts(S, rng):
        for i in range((S + BWD_BM - 1) // BWD_BM):
            visitors = [kb for kb, qi in bwd_visits(S) if qi == i]
            skipped = {kb for kb in visitors if visit_empty(ds, S, kb, i)}
            contrib = sorted(set(visitors) - skipped, reverse=True)
            assert contrib and all(kb < min(contrib) for kb in skipped)   # the skip is monotone in the key block
            last_kb = max(visitors)
            for _ in range(20):
                assert dq_order_schedule(visitors, skipped, last_kb, rng) == contrib


def test_mirror_counting_skipped_visits_would_break_the_order():
    """Why a skipped visit must not touch the counter: S = 256 in documents of 130 tokens, query block 3 (rows
    192..255) starts its documents at 130 and 260 -> min 130, so key blocks 3 and 2 contribute and 1 and 0 are
    skipped.  Counting the skipped visits lets key block 2 add before key block 3 in some interleaving."""
    S = 256
    ds = [i - i % 130 for i in range(S)]
    visitors = [kb for kb, qi in bwd_visits(S) if qi == 3]
    skipped = {kb for kb in visitors if visit_empty(ds, S, kb, 3)}
    assert skipped == {0, 1}
    rng = random.Random(0)
    orders = {tuple(dq_order_schedule(visitors, skipped, 3, rng, count_skipped=True)) for _ in range(200)}
    assert (2, 3) in orders
    assert {tuple(dq_order_schedule(visitors, skipped, 3, rng)) for _ in range(200)} == {(3, 2)}


def test_visible_keys_doc_start_clamps():
    ds = torch.tensor([[0, -3, 5, 1]])
    vis = OF.visible_keys(4, 4, causal=True, doc_start=ds)[0, 0]
    want = torch.tensor([[1, 0, 0, 0], [1, 1, 0, 0], [0, 0, 1, 0], [0, 1, 1, 1]], dtype=torch.bool)
    assert torch.equal(vis, want)


# ------------------------------------------------------------------------------------------------ packer
def _corpus(n, max_length, seed=0):
    g = torch.Generator().manual_seed(seed)
    data = []
    for k in range(n):
        full = int(torch.randint(2, max_length + 1, (1,), generator=g))
        prompt = int(torch.randint(1, full, (1,), generator=g)) if k % 7 else full   # every 7th: nothing trainable
        ids = torch.cat([torch.randint(3, 100, (full,), generator=g), torch.zeros(max_length - full, dtype=torch.long)])
        labels = torch.full((max_length,), IGNORE_INDEX)
        labels[prompt - 1 : full - 1] = ids[prompt:full]
        data.append({"input_ids": ids, "labels": labels})
    return data


def test_packer_places_every_trainable_label_once():
    L = 64
    data = _corpus(60, L)
    a, b = PackedSFTDataset(data, L), PackedSFTDataset(data, L)
    assert len(a) == len(b) and all(torch.equal(x, y) for ra, rb in zip(a.rows, b.rows) for x, y in zip(ra, rb))
    kept = [i for i, d in enumerate(data) if sample_length(d["labels"]) > 0]
    assert len(kept) < len(data)
    rows = [a[k] for k in range(len(a))]
    seen = []
    for inst in rows:
        ids, labels, pos = (inst.get(f).tensor for f in ("input_ids", "labels", "position_ids"))
        assert ids.shape == labels.shape == pos.shape == (L,)
        starts = torch.nonzero(pos == 0).flatten().tolist() + [L]
        for s, e in zip(starts[:-1], starts[1:]):
            assert torch.equal(pos[s:e], torch.arange(e - s))
            lab = labels[s:e]
            assert int(lab[-1]) <= 0          # no label crosses into the next document
            for t in torch.nonzero(lab > 0).flatten().tolist():
                assert int(lab[t]) == int(ids[s + t + 1])
            if (lab > 0).any():
                seen.append((ids[s:e], lab))
    # in order, each sample exactly once with its own tokens and labels
    assert len(seen) == len(kept)
    for (ids, lab), i in zip(seen, kept):
        n = sample_length(data[i]["labels"])
        assert len(ids) == n
        assert torch.equal(ids, data[i]["input_ids"][:n])
        assert torch.equal(lab[:-1], data[i]["labels"][: n - 1])
    assert a.fill_rate == pytest.approx(sum(sample_length(d["labels"]) for d in data) / (len(a) * L))
    print(f"fill rate {a.fill_rate:.3f}: {len(a)} packed rows for {len(kept)} samples of at most {L} tokens")


def test_pack_samples_rules():
    assert pack_samples([3, 0, 4, 2, 5], 8) == [[0, 2], [3, 4]]
    assert pack_samples([], 8) == []
    with pytest.raises(ValueError):
        pack_samples([9], 8)


# ------------------------------------------------------------------------------------------------ reference semantics
def _llama(g, qkv_bias, seed=0):
    from libai_b200.models.llama_model import LlamaForCausalLM

    torch.manual_seed(seed)
    return LlamaForCausalLM(hidden_layers=2, vocab_size=97, hidden_size=64, intermediate_size=96, num_attention_heads=4,
                            max_position_embeddings=64, qkv_bias=qkv_bias, num_key_value_heads=g).float()


def _docs(lengths, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in lengths:
        ids = torch.randint(1, 97, (n,), generator=g)
        lab = torch.full((n,), IGNORE_INDEX)
        lab[n // 3 : n - 1] = ids[n // 3 + 1 :]
        out.append((ids, lab))
    return out


def _packed(docs, L):
    ids, lab, pos = torch.zeros(L, dtype=torch.long), torch.full((L,), IGNORE_INDEX), torch.zeros(L, dtype=torch.long)
    at = 0
    for i, l in docs:
        n = len(i)
        ids[at : at + n], lab[at : at + n], pos[at : at + n] = i, l, torch.arange(n)
        at += n
    pos[at:] = torch.arange(L - at)
    return ids, lab, pos


def _grads(model, **batch):
    model.zero_grad()
    loss = model(**batch)["lm_loss"]
    loss.backward()
    return loss.detach(), {n: p.grad.detach().clone() for n, p in model.named_parameters()}


@pytest.mark.parametrize("g,qkv_bias", [(4, False), (2, False), (4, True), (1, True)])
def test_packed_batch_equals_one_sample_per_row(monkeypatch, g, qkv_bias):
    monkeypatch.setenv("LIBAI_B200_IMPL", "ref")
    L = 24
    docs = _docs([5, 1 + 1, 9, 3], seed=g)
    rows = [_packed(docs[:2], L), _packed(docs[2:], L)]
    model = _llama(g, qkv_bias)
    packed = _grads(model, input_ids=torch.stack([r[0] for r in rows]), labels=torch.stack([r[1] for r in rows]),
                    position_ids=torch.stack([r[2] for r in rows]))
    # the same samples, one per row: padded to L, and unpadded one at a time (summed with the loss's token weights)
    pad = [_packed([d], L) for d in docs]
    padded = _grads(model, input_ids=torch.stack([r[0] for r in pad]), labels=torch.stack([r[1] for r in pad]))
    for ref in (padded,):
        torch.testing.assert_close(packed[0], ref[0], rtol=1e-5, atol=1e-6)
        for n in ref[1]:
            torch.testing.assert_close(packed[1][n], ref[1][n], rtol=1e-4, atol=1e-6, msg=n)
    total = sum(int((l > 0).sum()) for _, l in docs)
    loss = torch.zeros(())
    grads = {n: torch.zeros_like(v) for n, v in packed[1].items()}
    for i, l in docs:
        w = int((l > 0).sum()) / total
        li, gi = _grads(model, input_ids=i[None], labels=l[None])
        loss += w * li
        for n in grads:
            grads[n] += w * gi[n]
    torch.testing.assert_close(packed[0], loss, rtol=1e-5, atol=1e-6)
    for n in grads:
        torch.testing.assert_close(packed[1][n], grads[n], rtol=1e-4, atol=1e-6, msg=n)


def test_position_ids_rejected_with_cache_or_mask(monkeypatch):
    monkeypatch.setenv("LIBAI_B200_IMPL", "ref")
    model = _llama(4, False)
    ids = torch.randint(1, 97, (1, 8))
    with pytest.raises(ValueError):
        model(ids, attention_mask=torch.ones_like(ids), position_ids=torch.arange(8)[None])


def test_rotary_reference_gathers_positions(monkeypatch):
    monkeypatch.setenv("LIBAI_B200_IMPL", "ref")
    from libai_b200.models.llama_model import rotary_tables

    cos, sin = rotary_tables(8, 32)
    for shape in ((2, 5, 3, 24), (2, 5, 2, 4, 8)):
        qkv = torch.randn(shape)
        off = OF.apply_rotary_qkv(qkv, cos, sin, 7)
        pos = OF.apply_rotary_qkv(qkv, cos, sin, 0, torch.arange(7, 12, dtype=torch.int32)[None].expand(2, 5))
        assert torch.equal(off, pos)


# ------------------------------------------------------------------------------------------------ build
@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_packed_sequence_kernels_compile_without_forward_spills(tmp_path):
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, "attention_sm90.cu"), "-o", str(tmp_path / "attn.o")],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    assert not ops_build.serialized_wgmma(res.stdout)
    reports, name = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
        elif name and "spill stores" in line:
            reports[name] = line
    fwd = {n: ln for n, ln in reports.items() if "attn_fwd_kernel" in n or "attn_fwd_doc_kernel" in n}
    doc = [n for n in reports if "attn_fwd_doc_kernel" in n or re.search(r"attn_bwd_kernelILi\d+ELi0ELb0ELb1E", n)]
    assert len(doc) == 4, doc    # forward and backward, head-dim tiles 64 and 128
    assert len(fwd) == 14
    for n, ln in fwd.items():
        assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", ln), (n, ln)


# ------------------------------------------------------------------------------------------------ pipeline
def _packed_batch(step):
    docs = _docs([5, 7, 2, 9, 4, 3, 6, 8], seed=100 + step)
    rows = [_packed(docs[:3], 16), _packed(docs[3:5], 16), _packed(docs[5:7], 16), _packed(docs[7:], 16)]
    return dict(input_ids=torch.stack([r[0] for r in rows]), labels=torch.stack([r[1] for r in rows]),
                position_ids=torch.stack([r[2] for r in rows]))


def _train_packed(rank, world, pp):
    """Two AdamW steps of a tiny GQA Llama on packed batches of two micro-batches each, on pp pipeline stages."""
    import torch.distributed as dist

    from libai_b200.config import DictConfig
    from libai_b200.layers._param import param_defaults
    from libai_b200.models.llama_model import LlamaForCausalLM
    from libai_b200.optim import AdamW, get_default_optimizer_params
    from libai_b200.parallel import state as pstate
    from libai_b200.parallel.pipeline import PipelineSchedule1F1B
    from libai_b200.utils import distributed as dutil

    topo = dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=pp,
                                                 pipeline_num_layers=2, device_type="cpu")))
    with param_defaults(dtype=torch.float32, device="cpu", seed=3):
        model = LlamaForCausalLM(hidden_layers=2, vocab_size=97, hidden_size=64, intermediate_size=96,
                                 num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=32)
    opt = AdamW(get_default_optimizer_params(model, clip_grad_max_norm=1.0, clip_grad_norm_type=2.0), lr=1e-2)
    opt.configure(zero_stage=0, param_names={id(p): n for n, p in model.named_parameters()})
    opt.setup()
    pipe = PipelineSchedule1F1B(model) if pp > 1 else None
    losses = []
    for step in range(2):
        full = _packed_batch(step)
        batches = [{k: v[i * 2:(i + 1) * 2] for k, v in full.items()} for i in range(2)]
        opt.zero_grad()
        if pipe is not None:
            out = pipe.run(batches)
            loss = out["lm_loss"] if out is not None else torch.zeros(())
        else:
            loss = torch.zeros(())
            for b in batches:
                o = model.forward_stage(b)
                (o["lm_loss"] / 2).backward()
                loss = loss + o["lm_loss"].detach() / 2
        opt.step()
        v = loss.detach().clone().float()
        if pp > 1:
            dist.all_reduce(v, group=topo.pp_group)
        losses.append(float(v))
    state = pstate.full_state_dict(model)
    return (losses, {k: v.clone() for k, v in state.items()}) if rank == 0 else None


def test_packed_pipeline_matches_single_process():
    """A 2-stage gloo pipeline run of packed batches (position_ids threaded to the blocks of both stages) trains like
    the single-process run."""
    from tests.dist_utils import run_distributed

    base_l, base_p = run_distributed(_train_packed, 1, 1)[0]
    pp_l, pp_p = run_distributed(_train_packed, 2, 2)[0]
    assert base_l == pytest.approx(pp_l, rel=1e-4, abs=1e-5), (base_l, pp_l)
    assert set(base_p) == set(pp_p)
    for k in base_p:
        a, b = torch.as_tensor(base_p[k]), torch.as_tensor(pp_p[k])
        assert torch.allclose(a, b, rtol=1e-3, atol=2e-5), f"{k}: {(a - b).abs().max()}"


def test_out_of_range_position_ids_are_rejected(monkeypatch):
    monkeypatch.setenv("LIBAI_B200_IMPL", "ref")
    model = _llama(4, False)
    ids = torch.randint(1, 97, (1, 8))
    for bad in (torch.arange(60, 68)[None], torch.arange(-1, 7)[None]):
        with pytest.raises(ValueError, match="position_ids"):
            model(ids, labels=ids, position_ids=bad)
