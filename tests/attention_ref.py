"""Element-by-element references for the attention kernels (flash forward / backward, decode) and the Philox dropout
masks, in fp64 from the exact bf16 inputs the kernels saw.  The comparator, the rounding units and the measured
approximation constants are those of ``tests/dense_ref.py``.

Every check is ``|out - ref| <= bound`` per element.  The bound follows the kernels' rounding points
(attention_sm90.cu, decode_attention_sm90.cu); each term is derived in a comment where it is formed.

Forward: ``O = sum_j P_ij keep_ij inv_keep V_j`` with ``P = softmax(scale * Q K^T + bias)`` over the visible keys.  The
kernels round each unnormalised probability to bf16 before P.V but sum the unrounded ones into the normaliser, so the
bf16 rounding of P gives the dominant term ``2^-8 * sum_j |P_ij keep_ij inv_keep V_jd|``.

Backward: the kernel takes the forward's bf16 O and fp32 lse as inputs, and so does this reference: delta = rowsum(dO * O)
and P = exp(z - lse) are formed from them.  The kernel rounds ``P * inv_keep`` (for dV) and ``dS`` (for dK, dQ) to bf16.
Those roundings are emulated here: the fp64 value is rounded through fp32 to bf16, and where the kernel's fp32 value
(known to within its error bound) could round to a different bf16 neighbour, the difference between the two is added to
the bound.  What is left is fp32 accumulation and the output rounding, so a wrong row or block is seen at the percent
level even where |dQ| is much smaller than sum |dS K|.
"""
import math

import numpy as np
import torch

from tests.dense_ref import ACC, FLUSH, ROUND, check  # noqa: F401  (check is re-exported for the tests)

# ex2.approx.ftz.f32 (fast_exp2 in common.cuh): every exponent the attention kernels feed it is <= 0 (a score minus a
# running max or the lse, or the difference of two running maxima).  max |ex2.approx(x) / 2^x - 1| over every fp32 x in
# [-126, 0] was 1.44e-7 = 2^-22.73, measured once on an H100 80GB HBM3 by dev/measure_ex2.py, which sweeps all those
# bit patterns against the fp64 2^x on the device (the power limit of that card was not recorded; the result of one
# SFU instruction does not depend on clocks); the constant rounds it up to the next power of two.
EX2_APPROX = 2.0 ** -22
LN2 = math.log(2.0)


# ------------------------------------------------------------------------------------------------------------- Philox
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_U32 = np.uint64(0xFFFFFFFF)
_GOLDEN = 0x9E3779B97F4A7C15


def philox4x32_7(c0, c1, c2, c3, k0, k1):
    """Philox4x32 with 7 rounds, as ``philox4x32_7`` in common.cuh: per round (hi, lo) of 0xD2511F53 * c0 and of
    0xCD9E8D57 * c2, output (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0), then the key is bumped by the Weyl constants.
    Arguments are broadcastable integer arrays holding uint32 values; returns the four uint32 words (as uint64 arrays)."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _U32 for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for _ in range(7):
        p0, p1 = _M0 * c0, _M1 * c2            # 32 x 32 -> 64 bits: exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _U32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _U32
        k0, k1 = (k0 + _W0) & _U32, (k1 + _W1) & _U32
    return c0, c1, c2, c3


def salted_seed(seed: int, salt: int) -> int:
    """The Philox key the kernels use: rng_resolve's seed ^ salt * 0x9E3779B97F4A7C15 (mod 2^64)."""
    return (int(seed) ^ (int(salt) * _GOLDEN)) & 0xFFFFFFFFFFFFFFFF


def attn_drop_threshold(p: float):
    """(thr, inv_keep) of the attention kernels: keep <=> byte >= thr, thr = clamp((uint32)(256 p + 0.5f), 1, 255) in
    fp32, inv_keep = 256 / (256 - thr) in fp32.  (So any p below 1/512 drops 1/256 of the probabilities.)"""
    thr = int(np.float32(p) * np.float32(256.0) + np.float32(0.5))
    thr = min(max(thr, 1), 255)
    return thr, float(np.float32(256.0) / np.float32(256 - thr))


def attn_keep_mask(seed: int, offset: int, B: int, A: int, Sq: int, Sk: int, thr: int, device=None):
    """Keep-mask [B, A, Sq, Sk] of the flash kernels for the stored (seed, offset) (seed already salted).  keep(b, h, i, j)
    is byte j mod 16 (little endian across x, y, z, w) of philox(c = (i, j div 16, (b A + h) ^ ((offset >> 32) << 20),
    offset mod 2^32), k = seed), compared with >= thr; h is the query head, i and j absolute indices."""
    seed, offset = int(seed) & 0xFFFFFFFFFFFFFFFF, int(offset) & 0xFFFFFFFFFFFFFFFF
    ng = (Sk + 15) // 16
    i = np.arange(Sq, dtype=np.uint64)[None, :, None]
    g = np.arange(ng, dtype=np.uint64)[None, None, :]
    bh = np.arange(B * A, dtype=np.uint64)[:, None, None] ^ np.uint64(((offset >> 32) << 20) & 0xFFFFFFFF)
    words = philox4x32_7(i, g, bh, offset & 0xFFFFFFFF, seed & 0xFFFFFFFF, seed >> 32)
    w = np.stack(words, -1)                                              # [BA, Sq, ng, 4]
    by = (w[..., None] >> (np.arange(4, dtype=np.uint64) * np.uint64(8))) & np.uint64(0xFF)
    by = by.reshape(B * A, Sq, ng * 16)[..., :Sk]                       # byte 4 * word + k is key 16 g + 4 word + k
    return torch.from_numpy(by >= np.uint64(thr)).reshape(B, A, Sq, Sk).to(device)


def bdr_drop_threshold(p: float):
    """(thr, scale) of bias_dropout_residual: keep <=> u16 >= thr, thr = min((uint32)(65536 p + 0.5f), 65535),
    scale = 65536 / (65536 - thr), both in fp32."""
    thr = min(int(np.float32(p) * np.float32(65536.0) + np.float32(0.5)), 65535)
    return thr, float(np.float32(65536.0) / np.float32(65536 - thr))


def bdr_keep_mask(seed: int, offset: int, numel: int, thr: int, device=None):
    """Keep-mask of bias_dropout_residual over the flattened tensor: element e uses 16-bit lane e mod 8 of
    philox(c = (n lo, n hi, offset lo, offset hi), k = seed) with n = e div 8."""
    seed, offset = int(seed) & 0xFFFFFFFFFFFFFFFF, int(offset) & 0xFFFFFFFFFFFFFFFF
    n = np.arange((numel + 7) // 8, dtype=np.uint64)
    w = np.stack(philox4x32_7(n & _U32, n >> np.uint64(32), offset & 0xFFFFFFFF, offset >> 32, seed & 0xFFFFFFFF,
                              seed >> 32), -1)                           # [n, 4]
    u = (w[..., None] >> (np.arange(2, dtype=np.uint64) * np.uint64(16))) & np.uint64(0xFFFF)
    return torch.from_numpy(u.reshape(-1)[:numel] >= np.uint64(thr)).to(device)


# ------------------------------------------------------------------------------------------------------------ helpers
def alibi_bias(slopes, Sq: int, Sk: int, device=None):
    """[1, A, Sq, Sk] ALiBi bias slope * (j - i - (Sk - Sq)) in fp64."""
    rel = (torch.arange(Sk, device=device)[None, :] - torch.arange(Sq, device=device)[:, None] - (Sk - Sq)).double()
    return slopes.double().to(device)[None, :, None, None] * rel[None, None]


def _bf16_emulate(x, err):
    """A kernel's fp32 value is known to lie within ``x +- err``; it is then rounded to bf16.  Returns the bf16 rounding
    of x (through fp32, as the kernel's value was formed) and how far the kernel's bf16 value can be from it: fp32 and
    bf16 rounding are both monotone, so the kernel's lies between the roundings of x - err and x + err."""
    r = x.float().bfloat16().double()
    lo = (x - err).float().bfloat16().double()
    hi = (x + err).float().bfloat16().double()
    return r, torch.maximum(hi - r, r - lo)


def _head_scores(q, k, scale, bias_h):
    """fp64 z = scale * q k^T + bias and the bound of the kernel's fp32 S = q k^T: a sum of D products accumulated in
    fp32, D * 2^-23 * sum |q||k| (dense_ref.ACC)."""
    qd, kd = q.double(), k.double()
    z = scale * (qd @ kd.t())
    ds = q.shape[-1] * ACC * (qd.abs() @ kd.abs().t())
    if bias_h is not None:
        z = z + bias_h
    return z, ds


def _bias_head(bias, alibi, b, h, Sq, Sk, device):
    if bias is not None:
        return bias[min(b, bias.shape[0] - 1), min(h, bias.shape[1] - 1)].double().to(device)
    if alibi is not None:
        return alibi_bias(alibi[h:h + 1], Sq, Sk, device)[0, 0]
    return None


# ------------------------------------------------------------------------------------------------------------ forward
def attention_fwd_ref(q, k, v, *, scale, vis, bias=None, alibi=None, keep=None, inv_keep=1.0, tile=64,
                      eta_extra=None):
    """Reference O [B, A, Sq, D] and lse [B, A, Sq] with their bounds, as ((o, o_bound), (lse, lse_bound)).

    q [B, A, Sq, D]; k, v [B, G, Sk, D] (query head h reads K/V head h / (A / G)); vis: bool [B|1, 1|A, Sq, Sk]
    (``OF.visible_keys``); bias: dense [B|1, A|1, Sq, Sk] or ``alibi`` slopes [A]; keep: bool [B, A, Sq, Sk] and its
    ``inv_keep``.  A row without a visible key has O = 0 and lse = 0, with a zero bound.  ``tile``: the smallest number
    of keys after which a kernel rescales its running sums (64 in decode, 128 in the flash forward).  ``eta_extra``
    (fp64 [B|1, A|1, Sq, Sk], or a number): a relative error of each unnormalised probability beyond the kernel's own
    roundings, e.g. from inputs the kernel saw rounded where the reference holds them exact."""
    B, A, Sq, D = q.shape
    G, Sk = k.shape[1], k.shape[2]
    r = A // G
    dev = q.device
    o = torch.zeros(B, A, Sq, D, dtype=torch.float64, device=dev)
    ob = torch.zeros_like(o)
    lse = torch.zeros(B, A, Sq, dtype=torch.float64, device=dev)
    lseb = torch.zeros_like(lse)
    # rescales of a row's running max / sum: one per tile, plus the merges of decode's warps and splits
    n_resc = (Sk + tile - 1) // tile + 4
    for b in range(B):
        for h in range(A):
            g = h // r
            z, dS = _head_scores(q[b, h], k[b, g], scale, _bias_head(bias, alibi, b, h, Sq, Sk, dev))
            vm = vis[min(b, vis.shape[0] - 1), min(h, vis.shape[1] - 1)].to(dev)
            zm = torch.where(vm, z, torch.full_like(z, -math.inf))
            m = zm.max(-1, keepdim=True).values
            empty = torch.isinf(m)
            m = torch.where(empty, torch.zeros_like(m), m)
            e = torch.where(vm, torch.exp(zm - m), torch.zeros_like(z))
            l = e.sum(-1, keepdim=True)
            P = e / torch.where(empty, torch.ones_like(l), l)
            T = P if keep is None else P * keep[b, h].to(dev) * inv_keep
            vd = v[b, g].double()
            ov = T @ vd
            M = torch.where(vm, z.abs(), torch.zeros_like(z)).max(-1, keepdim=True).values
            # relative error of one unnormalised probability before its bf16 rounding, natural-log units:
            #   scale * dS: the fp32 S;
            #   2^-21 (n_resc + 2) (|z| + M): the fp32 roundings of x = S scale log2e (+ bias log2e), of x - m and of
            #     the n_resc running-max differences, each 2^-24 of a value below |z| + M (log2 e / ln 2 absorbed in 2^3);
            #   (n_resc + 2) EX2_APPROX: its own ex2.approx and the ex2.approx of every rescale applied to it
            eta = scale * dS + 2.0 ** -21 * (n_resc + 2) * (z.abs() + M) + (n_resc + 2) * EX2_APPROX
            if eta_extra is not None:
                ex = eta_extra if not torch.is_tensor(eta_extra) else \
                    eta_extra[min(b, eta_extra.shape[0] - 1), min(h, eta_extra.shape[1] - 1)].to(dev)
                eta = eta + ex
            eta = torch.where(vm, eta, torch.zeros_like(eta))
            eta_max = eta.max(-1, keepdim=True).values
            # O = N / l with N = sum_j T_j V_j: each term of N carries eta, its bf16 rounding 2^-8 and the fp32 sum over
            # Sk keys (Sk * 2^-23); l carries eta and its own fp32 sum, and the epilogue's inv_keep / l and o * inv two
            # more roundings, which move O by |O| (eta_max + (Sk + n_resc + 4) 2^-23).  1.01 covers the second-order
            # products of these relative errors; the output rounding is ROUND of |O| plus that bound.
            bnd = (T.abs() * (eta + ROUND[torch.bfloat16] + Sk * ACC)) @ vd.abs() \
                + ov.abs() * (eta_max + (Sk + n_resc + 4) * ACC)
            bnd = 1.01 * bnd * (1 + ROUND[torch.bfloat16]) + ROUND[torch.bfloat16] * ov.abs()
            o[b, h] = torch.where(empty, torch.zeros_like(ov), ov)
            ob[b, h] = torch.where(empty, torch.zeros_like(ov), bnd + FLUSH)
            lv = (m + torch.log(torch.where(empty, torch.ones_like(l), l)))[:, 0]
            # lse = (m2 + log2f(l)) ln 2: errors of the max cancel to first order; l carries eta_max and its fp32 sum;
            # lg2.approx errs by at most 2^-21 absolute (bounded like ex2.approx on [1, 2), with room); the product with
            # ln 2 and the sum round at 2^-24 of |m| + |log l| each
            lb = eta_max[:, 0] + (Sk + 4) * ACC + 2.0 ** -21 + 2.0 ** -22 * (M[:, 0] + lv.abs() + m[:, 0].abs())
            lse[b, h] = torch.where(empty[:, 0], torch.zeros_like(lv), lv)
            lseb[b, h] = torch.where(empty[:, 0], torch.zeros_like(lb), lb + FLUSH)
    return (o, ob), (lse, lseb)


# ----------------------------------------------------------------------------------------------------------- backward
def attention_bwd_ref(q, k, v, do, o, lse, *, scale, vis, bias=None, alibi=None, keep=None, inv_keep=1.0):
    """Reference gradients of the flash backward for its inputs: dQ [B, A, Sq, D], dK, dV [B, G, Sk, D] and, with a dense
    ``bias``, dbias of the bias' shape (fp32 in the kernel, summed over its broadcast dimensions).  ``o`` (bf16) and
    ``lse`` (fp32) are the forward's outputs, which the kernel reads: delta = rowsum(dO * o), P = exp(z - lse).  Returns
    {name: (ref, bound)}."""
    B, A, Sq, D = q.shape
    G, Sk = k.shape[1], k.shape[2]
    r = A // G
    dev = q.device
    bf = ROUND[torch.bfloat16]
    dq = torch.zeros(B, A, Sq, D, dtype=torch.float64, device=dev)
    dqb = torch.zeros_like(dq)
    dk = torch.zeros(B, G, Sk, D, dtype=torch.float64, device=dev)
    dkb, dv, dvb = torch.zeros_like(dk), torch.zeros_like(dk), torch.zeros_like(dk)
    dkabs, dvabs = torch.zeros_like(dk), torch.zeros_like(dk)
    if bias is not None:
        dbias = torch.zeros(bias.shape, dtype=torch.float64, device=dev)
        dbiasb, dbiasabs = torch.zeros_like(dbias), torch.zeros_like(dbias)
        n_bcast = (B // bias.shape[0]) * (A // bias.shape[1])
    for b in range(B):
        for h in range(A):
            g = h // r
            bh = _bias_head(bias, alibi, b, h, Sq, Sk, dev)
            z, dS = _head_scores(q[b, h], k[b, g], scale, bh)
            vm = vis[min(b, vis.shape[0] - 1), min(h, vis.shape[1] - 1)].to(dev)
            L = lse[b, h].double().to(dev)[:, None]
            P = torch.where(vm, torch.exp(z - L), torch.zeros_like(z))
            # relative error of the kernel's P: its fp32 S (scale * dS); the fp32 roundings of x, lse * log2e and x - lse2,
            # each 2^-24 of |z|, |lse| or |bias| in log2 units (2^-21 with room); ex2.approx
            beta = bh.abs() if bh is not None else 0.0
            eta = scale * dS + 2.0 ** -21 * (z.abs() + L.abs() + beta) + EX2_APPROX
            kp = 1.0 if keep is None else keep[b, h].to(dev).double() * inv_keep
            dod, vd = do[b, h].double(), v[b, g].double()
            dP = dod @ vd.t()
            dPb = D * ACC * (dod.abs() @ vd.abs().t())                       # fp32 sum of D products
            od = o[b, h].double()
            delta = (dod * od).sum(-1, keepdim=True)
            deltab = D * ACC * (dod * od).abs().sum(-1, keepdim=True)        # the delta kernel's fp32 sum
            ds = P * (kp * dP - delta)                                       # natural units (without scale)
            # error of the kernel's fp32 dS / scale: dP and delta as above, plus 2^-23 of each for dP * inv_keep and
            # delta * scale; P's eta on the whole; 2^-22 for the fmaf and the product with P
            dse = P * (kp * (dPb + 2.0 ** -23 * dP.abs()) + deltab + 2.0 ** -23 * delta.abs()) \
                + ds.abs() * (eta + 2.0 ** -22)
            E, U = _bf16_emulate(scale * ds, scale * dse)                  # dS as the dK / dQ products see it
            Pd = P * kp
            EP, UP = _bf16_emulate(Pd, Pd * (eta + 2.0 ** -23))             # P * inv_keep rounded for dV
            kd, qd = k[b, g].double(), q[b, h].double()
            # dQ: sum over Sk keys of bf16 dS * K, fp32 products accumulated in the MMA and by red.add (Sk * 2^-23 of
            # sum |terms|), plus where dS's rounding could go either way U * |K|
            dq[b, h] = E @ kd
            dqb[b, h] = U @ kd.abs() + Sk * ACC * (E.abs() @ kd.abs())
            dk[b, g] += E.t() @ qd
            dkb[b, g] += U.t() @ qd.abs()
            dkabs[b, g] += E.abs().t() @ qd.abs()
            dv[b, g] += EP.t() @ dod
            dvb[b, g] += UP.t() @ dod.abs()
            dvabs[b, g] += EP.abs().t() @ dod.abs()
            if bias is not None:
                # fp32 dS * (1 / scale) (two roundings) added with fp32 atomics over the broadcast dimensions
                bi = (min(b, bias.shape[0] - 1), min(h, bias.shape[1] - 1))
                dbias[bi] += ds
                dbiasb[bi] += dse + 2.0 ** -22 * ds.abs()
                dbiasabs[bi] += ds.abs()
    # dK / dV sum r * Sq terms per element (the group's query heads): fp32 accumulation r Sq 2^-23 of sum |terms|
    dkb += r * Sq * ACC * dkabs
    dvb += r * Sq * ACC * dvabs
    out = {}
    for name, ref, bnd in (("dq", dq, dqb), ("dk", dk, dkb), ("dv", dv, dvb)):
        # output rounding to bf16 of a value within bnd of ref; 1.001 covers the second-order terms
        out[name] = (ref, 1.001 * bnd * (1 + bf) + bf * ref.abs() + FLUSH)
    if bias is not None:
        out["dbias"] = (dbias, 1.001 * dbiasb + (n_bcast + 2) * ACC * dbiasabs + FLUSH)
    return out


def check_all(got: dict, ref: dict, what: str):
    """check() for every name in ``ref`` ({name: (ref, bound)}) against ``got[name]``."""
    for name, (rv, bnd) in ref.items():
        check(got[name], rv, bnd, f"{what} {name}")
