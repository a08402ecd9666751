"""The attention references of tests/attention_ref.py on the CPU: an fp32 emulation of the flash kernels' arithmetic
(tile-wise running max, bf16 P and dS, fp32 sums) passes the per-element bounds, and outputs with the defects a kernel
could have are rejected, at shapes the GPU tests use.  Also the Philox mirror: keep fractions and what the masks depend
on."""
import math

import numpy as np
import pytest
import torch

from libai_b200.ops import functional as OF
from tests import attention_ref as R
from tests.dense_ref import Mismatch


def bf16_rand(*shape, gen, scale=1.0):
    return (torch.randn(*shape, generator=gen, dtype=torch.float64) * scale).bfloat16()


def case(B, A, G, Sq, Sk, D=64, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return (bf16_rand(B, A, Sq, D, gen=gen), bf16_rand(B, G, Sk, D, gen=gen), bf16_rand(B, G, Sk, D, gen=gen),
            bf16_rand(B, A, Sq, D, gen=gen))


def emulate(q, k, v, do, *, scale, vis, bias=None, keep=None, inv_keep=1.0):
    """The flash kernels' arithmetic in fp32: 128-key tiles with a running max, unrounded P summed into l, bf16 P (dropped)
    into P.V, bf16 O; backward from that O and lse with bf16 P * inv_keep and bf16 dS.  Returns bf16 o, dq, dk, dv and
    fp32 lse, dbias."""
    B, A, Sq, D = q.shape
    G, Sk = k.shape[1], k.shape[2]
    r = A // G
    L2E = np.float32(1.4426950408889634)
    o = torch.zeros(B, A, Sq, D, dtype=torch.bfloat16)
    lse = torch.zeros(B, A, Sq)
    dq = torch.zeros(B, A, Sq, D)
    dk, dv = torch.zeros(B, G, Sk, D), torch.zeros(B, G, Sk, D)
    dbias = None if bias is None else torch.zeros(bias.shape)
    sl2 = float(np.float32(scale) * L2E)
    for b in range(B):
        for h in range(A):
            g = h // r
            vm = vis[min(b, vis.shape[0] - 1), 0]
            x = (q[b, h].float() @ k[b, g].float().t()) * sl2
            if bias is not None:
                x = x + bias[min(b, bias.shape[0] - 1), min(h, bias.shape[1] - 1)].float() * float(L2E)
            x = torch.where(vm, x, torch.full_like(x, -math.inf))
            kp = torch.ones(Sq, Sk) if keep is None else keep[b, h].float()
            m = torch.full((Sq, 1), -math.inf)
            l = torch.zeros(Sq, 1)
            acc = torch.zeros(Sq, D)
            for t0 in range(0, Sk, 128):
                xt = x[:, t0:t0 + 128]
                m_new = torch.maximum(m, xt.max(-1, keepdim=True).values)
                m_use = torch.where(torch.isinf(m_new), torch.zeros_like(m_new), m_new)
                alpha = torch.exp2(m - m_use)
                p = torch.exp2(xt - m_use)
                l = l * alpha + p.sum(-1, keepdim=True)
                acc = acc * alpha + (p * kp[:, t0:t0 + 128]).bfloat16().float() @ v[b, g, t0:t0 + 128].float()
                m = m_new
            inv = torch.where(l > 0, inv_keep / l, torch.zeros_like(l))
            o[b, h] = (acc * inv).bfloat16()
            lse[b, h] = torch.where(torch.isinf(m), torch.zeros_like(m), (m + torch.log2(l)) * math.log(2.0))[:, 0]
            # backward
            P = torch.where(vm, torch.exp2(x - lse[b, h][:, None] * float(L2E)), torch.zeros_like(x))
            dP = do[b, h].float() @ v[b, g].float().t()
            delta = (do[b, h].float() * o[b, h].float()).sum(-1, keepdim=True)
            ds = P * (kp * inv_keep * dP * scale - delta * scale)
            dsb = ds.bfloat16().float()
            dq[b, h] = dsb @ k[b, g].float()
            dk[b, g] += dsb.t() @ q[b, h].float()
            dv[b, g] += (P * kp * inv_keep).bfloat16().float().t() @ do[b, h].float()
            if bias is not None:
                dbias[min(b, bias.shape[0] - 1), min(h, bias.shape[1] - 1)] += ds / scale
    out = dict(o=o, lse=lse, dq=dq.bfloat16(), dk=dk.bfloat16(), dv=dv.bfloat16())
    if bias is not None:
        out["dbias"] = dbias
    return out


def refs(q, k, v, do, *, scale, vis, o_in, lse_in, **kw):
    (o, ob), (lse, lseb) = R.attention_fwd_ref(q, k, v, scale=scale, vis=vis, tile=128, **kw)
    out = dict(o=(o, ob), lse=(lse, lseb))
    out.update(R.attention_bwd_ref(q, k, v, do, o_in, lse_in, scale=scale, vis=vis, **kw))
    return out


def rejected(got, ref, name):
    with pytest.raises(Mismatch):
        R.check(got, ref[name][0], ref[name][1], name)


# ---------------------------------------------------------------------------------------------- square causal, D = 64
@pytest.fixture(scope="module")
def square():
    B, A, S, D = 2, 4, 1000, 64
    q, k, v, do = case(B, A, A, S, S, D, seed=1)
    scale = D ** -0.5
    vis = OF.visible_keys(S, S, causal=True)
    em = emulate(q, k, v, do, scale=scale, vis=vis)
    ref = refs(q, k, v, do, scale=scale, vis=vis, o_in=em["o"], lse_in=em["lse"])
    return q, k, v, do, scale, vis, em, ref


def test_emulated_kernel_passes_the_bounds(square):
    *_, em, ref = square
    R.check_all(em, ref, "square causal")


def test_late_rows_scaled_by_3_percent_are_rejected(square):
    *_, em, ref = square
    o = em["o"].clone()
    o[:, :, 250:] = (o[:, :, 250:].float() * 1.03).bfloat16()
    rejected(o, ref, "o")


def test_last_query_block_of_dq_scaled_by_5_percent_is_rejected(square):
    *_, em, ref = square
    dq = em["dq"].clone()
    dq[:, :, 960:] = (dq[:, :, 960:].float() * 1.05).bfloat16()
    rejected(dq, ref, "dq")


def test_a_key_tile_missing_from_late_rows_is_rejected(square):
    q, k, v, do, scale, vis, em, ref = square
    vis2 = vis.clone()
    vis2[..., 512:, 128:256] = False
    (o, _), _ = R.attention_fwd_ref(q, k, v, scale=scale, vis=vis2)
    rejected(o, ref, "o")


def test_a_key_block_missing_from_one_query_blocks_dq_is_rejected(square):
    q, k, v, do, scale, vis, em, ref = square
    vis2 = vis.clone()
    vis2[..., 640:704, 192:256] = False                # P is recomputed from the lse: only that block's terms go
    got = R.attention_bwd_ref(q, k, v, do, em["o"], em["lse"], scale=scale, vis=vis2)
    rejected(got["dq"][0], ref, "dq")


# ------------------------------------------------------------------------------- rectangular, grouped, key windows
RECT = dict(B=2, A=8, G=2, Sq=65, Sk=129)


@pytest.fixture(scope="module")
def rect():
    B, A, G, Sq, Sk = RECT.values()
    q, k, v, do = case(B, A, G, Sq, Sk, 64, seed=2)
    kv_start = torch.tensor([0, 5], dtype=torch.int32)
    kv_lens = torch.tensor([129, 100], dtype=torch.int32)
    vis = OF.visible_keys(Sq, Sk, causal=True, kv_start=kv_start, kv_lens=kv_lens)
    em = emulate(q, k, v, do, scale=0.125, vis=vis)
    ref = refs(q, k, v, do, scale=0.125, vis=vis, o_in=em["o"], lse_in=em["lse"])
    return q, k, v, do, kv_start, kv_lens, em, ref


def test_rect_emulated_kernel_passes(rect):
    *_, em, ref = rect
    R.check_all(em, ref, "rect")


def test_top_left_causal_alignment_is_rejected(rect):
    q, k, v, do, kv_start, kv_lens, em, ref = rect
    Sq, Sk = q.shape[2], k.shape[2]
    tl = torch.arange(Sk)[None, :] <= torch.arange(Sq)[:, None]
    vis = OF.visible_keys(Sq, Sk, causal=False, kv_start=kv_start, kv_lens=kv_lens) & tl
    (o, _), _ = R.attention_fwd_ref(q, k, v, scale=0.125, vis=vis)
    rejected(o, ref, "o")


def test_kv_start_off_by_one_is_rejected(rect):
    q, k, v, do, kv_start, kv_lens, em, ref = rect
    vis = OF.visible_keys(q.shape[2], k.shape[2], causal=True, kv_start=kv_start + 1, kv_lens=kv_lens)
    (o, _), _ = R.attention_fwd_ref(q, k, v, scale=0.125, vis=vis)
    rejected(o, ref, "o")


def test_grouped_dk_dv_missing_one_query_head_are_rejected(rect):
    q, k, v, do, kv_start, kv_lens, em, ref = rect
    vis = OF.visible_keys(q.shape[2], k.shape[2], causal=True, kv_start=kv_start, kv_lens=kv_lens)
    do2 = do.clone()
    do2[:, 3] = 0                       # the last query head of group 0 adds nothing to that group's dK / dV
    got = R.attention_bwd_ref(q, k, v, do2, em["o"], em["lse"], scale=0.125, vis=vis)
    rejected(got["dk"][0], ref, "dk")
    rejected(got["dv"][0], ref, "dv")


def test_empty_rows_must_be_exactly_zero():
    q, k, v, do = case(1, 2, 2, 77, 203, 64, seed=3)
    kv_start = torch.tensor([150], dtype=torch.int32)     # rows i < 24 see no key (j <= i + 126)
    vis = OF.visible_keys(77, 203, causal=True, kv_start=kv_start)
    em = emulate(q, k, v, do, scale=0.125, vis=vis)
    ref = refs(q, k, v, do, scale=0.125, vis=vis, o_in=em["o"], lse_in=em["lse"])
    R.check_all(em, ref, "empty rows")
    assert not vis[0, 0, :24].any() and vis[0, 0, 24:].any(-1).all()
    o = em["o"].clone()
    o[0, 1, 5, 7] = 1e-3
    rejected(o, ref, "o")
    lse = em["lse"].clone()
    lse[0, 0, 23] = 0.25
    rejected(lse, ref, "lse")


# ------------------------------------------------------------------------------------------------------------ dropout
DROP = dict(B=2, A=4, G=2, S=203)
SEED, OFFSET, SALT = 0x1234_5678_9ABC_DEF0, 0x1_0000_0008, 3


@pytest.fixture(scope="module")
def drop():
    B, A, G, S = DROP.values()
    q, k, v, do = case(B, A, G, S, S, 64, seed=4)
    thr, ik = R.attn_drop_threshold(0.1)
    seed = R.salted_seed(SEED, SALT)
    keep = R.attn_keep_mask(seed, OFFSET, B, A, S, S, thr)
    vis = OF.visible_keys(S, S, causal=False)
    em = emulate(q, k, v, do, scale=0.125, vis=vis, keep=keep, inv_keep=ik)
    ref = refs(q, k, v, do, scale=0.125, vis=vis, o_in=em["o"], lse_in=em["lse"], keep=keep, inv_keep=ik)
    return q, k, v, do, vis, thr, ik, keep, em, ref


def _bwd_with(drop, keep):
    q, k, v, do, vis, thr, ik, _, em, _ = drop
    return R.attention_bwd_ref(q, k, v, do, em["o"], em["lse"], scale=0.125, vis=vis, keep=keep, inv_keep=ik)


def test_dropout_emulated_kernel_passes(drop):
    *_, em, ref = drop
    R.check_all(em, ref, "dropout")


def test_backward_mask_differing_in_one_16_key_group_is_rejected(drop):
    *_, keep, em, ref = drop
    k2 = keep.clone()
    k2[1, 2, :, 96:112] = ~k2[1, 2, :, 96:112]
    got = _bwd_with(drop, k2)
    for name in ("dq", "dk", "dv"):
        rejected(got[name][0], ref, name)


def test_backward_mask_keyed_by_the_kv_head_is_rejected(drop):
    B, A, G, S = DROP.values()
    *_, keep, em, ref = drop
    thr = R.attn_drop_threshold(0.1)[0]
    full = R.attn_keep_mask(R.salted_seed(SEED, SALT), OFFSET, B, A, S, S, thr)
    # the kernel's bh = b A + h with h the query head; a wrong one would use the K/V head h / r
    wrong = torch.stack([full[:, h // (A // G)] for h in range(A)], 1)
    got = _bwd_with(drop, wrong)
    for name in ("dq", "dk", "dv"):
        rejected(got[name][0], ref, name)


@pytest.mark.parametrize("defect", ["ij_swapped", "unsalted_seed"])
def test_wrong_mask_in_forward_and_backward_is_rejected(drop, defect):
    B, A, G, S = DROP.values()
    q, k, v, do, vis, thr, ik, keep, em, ref = drop
    if defect == "ij_swapped":
        wrong = R.attn_keep_mask(R.salted_seed(SEED, SALT), OFFSET, B, A, S, S, thr).transpose(-1, -2)
    else:
        wrong = R.attn_keep_mask(SEED, OFFSET, B, A, S, S, thr)
    assert not torch.equal(wrong, keep)
    (o, _), _ = R.attention_fwd_ref(q, k, v, scale=0.125, vis=vis, keep=wrong, inv_keep=ik)
    rejected(o, ref, "o")
    got = _bwd_with(drop, wrong)
    rejected(got["dv"][0], ref, "dv")


# ------------------------------------------------------------------------------------------------------- Philox mirror
def test_philox_known_answer():
    # Random123's published known-answer vector for philox4x32 with 7 rounds (kat_vectors: counter 0, key 0)
    words = R.philox4x32_7(0, 0, 0, 0, 0, 0)
    assert [int(w) for w in words] == [0x5F6FB709, 0x0D893F64, 0x4F121F81, 0x4F730A48]


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_attention_keep_fraction(p):
    thr, ik = R.attn_drop_threshold(p)
    keep = R.attn_keep_mask(R.salted_seed(7, 0), 12, 2, 4, 300, 300, thr)
    n = keep.numel()
    q = 1.0 - thr / 256.0
    # binomial: the kept count lies within 6 standard deviations of n q
    assert abs(int(keep.sum()) - n * q) < 6 * math.sqrt(n * q * (1 - q))
    assert ik == pytest.approx(256.0 / (256 - thr), rel=2 ** -23)


def test_bias_dropout_keep_fraction():
    thr, scale = R.bdr_drop_threshold(0.3)
    keep = R.bdr_keep_mask(R.salted_seed(11, 0), 40, 1 << 20, thr)
    n, q = keep.numel(), 1.0 - thr / 65536.0
    assert abs(int(keep.sum()) - n * q) < 6 * math.sqrt(n * q * (1 - q))
    assert scale == pytest.approx(65536.0 / (65536 - thr), rel=2 ** -23)


def test_thresholds():
    assert R.attn_drop_threshold(0.1)[0] == 26
    assert R.attn_drop_threshold(0.5)[0] == 128
    assert R.attn_drop_threshold(0.999)[0] == 255
    # below 1/512 the rounding gives 0, which the kernels raise to 1: 1/256 of the probabilities are dropped
    assert R.attn_drop_threshold(0.001)[0] == 1
    assert R.bdr_drop_threshold(0.1)[0] == 6554
    assert R.bdr_drop_threshold(0.99999999)[0] == 65535


def test_mask_changes_with_salt_offset_and_head():
    thr = R.attn_drop_threshold(0.5)[0]
    base = R.attn_keep_mask(R.salted_seed(5, 0), 8, 1, 2, 64, 64, thr)
    for other in (R.attn_keep_mask(R.salted_seed(5, 1), 8, 1, 2, 64, 64, thr),
                  R.attn_keep_mask(R.salted_seed(5, 0), 12, 1, 2, 64, 64, thr),
                  R.attn_keep_mask(R.salted_seed(5, 0), 8 + (1 << 32), 1, 2, 64, 64, thr)):
        assert (base != other).float().mean() > 0.4
    assert (base[0, 0] != base[0, 1]).float().mean() > 0.4
    # j counts from key 0: a mask over more keys extends, rather than shifts, the one over fewer
    wide = R.attn_keep_mask(R.salted_seed(5, 0), 8, 1, 2, 64, 100, thr)
    assert torch.equal(wide[..., :64], base)
