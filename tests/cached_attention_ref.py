"""fp64 references for cached attention (``OF.decode_attention`` and ``KVCacheLayer.attend``), built from the cache rows
each branch's kernel saw, with the per-element bound of ``tests/attention_ref.attention_fwd_ref``.

* bf16 cache: the rows themselves.
* FP8 cache read by the decode kernel: ``float(e)·s`` in fp64 — the kernel widens the bytes exactly and folds the
  scales into its scores and probabilities (``fp8_decode_terms`` bounds what that folding adds).
* FP8 cache on every other branch: the bf16 rounding of ``float(e)·s`` (``OF.kv_cache_dequant``'s window).

Rows that a branch must never read hold NaN (``poison``); masked rows inside the window hold ``SENT_K`` / ``SENT_V``, so
that a leak of one of them moves the output far past any bound.
"""
import torch

from tests import attention_ref as R

FP8 = torch.float8_e4m3fn
# masked rows inside the window: a zero key scores like an ordinary one, and a leaked probability p then adds about
# p·2^14 to the output (p is ~1/L for a window of L keys without ALiBi: far above any bound here)
SENT_K, SENT_V = 0.0, 2.0 ** 14


def i32(xs, device):
    return torch.tensor(xs, dtype=torch.int32, device=device)


def poison(k, v, ks, vs, b, lo, hi=None):
    """Rows ``lo:hi`` of sample ``b`` become NaN: bf16 NaN, or for an FP8 cache the E4M3 NaN byte and a NaN scale."""
    for t in (k, v):
        if t.dtype == FP8:
            t.view(torch.uint8)[b, :, lo:hi] = 0x7F
        else:
            t[b, :, lo:hi] = float("nan")
    for s in (ks, vs):
        if s is not None:
            s[b, :, lo:hi] = float("nan")


def sentinel_rows(k, v, b, lo, hi):
    """Rows ``lo:hi`` of sample ``b`` of bf16 ``[B, G, n, D]`` rows (before quantization) become the sentinels."""
    k[b, :, lo:hi] = SENT_K
    v[b, :, lo:hi] = SENT_V


def rows64(k, v, ks, vs, L, exact):
    """fp64 K, V rows ``[:L]`` as the kernel saw them: a bf16 cache's rows; an FP8 cache's ``float(e)·s`` (``exact``, the
    decode kernel) or its bf16 rounding (what ``OF.kv_cache_dequant`` hands the flash kernel and the reference math).
    NaN rows (never visible) become zeros."""
    out = []
    for t, s in ((k, ks), (v, vs)):
        t = t[:, :, :L]
        if s is None:
            x = t.double()
        elif exact:
            x = t.double() * s[:, :, :L, None].double()
        else:
            x = (t.float() * s[:, :, :L, None]).to(torch.bfloat16).double()
        out.append(torch.nan_to_num(x, nan=0.0))
    return out


def visible(lens, kv_start, s, L, causal):
    """bool ``[B, 1, s, L]``: query ``i`` of sample ``b`` sees ``kv_start[b] <= j <= lens[b] + i`` (causal) or
    ``kv_start[b] <= j < lens[b]`` (cross-attention)."""
    dev = lens.device
    j = torch.arange(L, device=dev)[None, None, :]
    i = torch.arange(s, device=dev)[None, :, None]
    end = lens.long()[:, None, None] + i if causal else lens.long()[:, None, None] - 1
    return ((j >= kv_start.long()[:, None, None]) & (j <= end))[:, None]


def rel_dense(rel_bias, lens, s, L):
    """fp32 ``[B, A, s, L]``: T5's ``rel_bias[h, min(lens[b] + i - j, R - 1)]`` (0 for keys after the query)."""
    dev = rel_bias.device
    j = torch.arange(L, device=dev)[None, None, :]
    i = torch.arange(s, device=dev)[None, :, None]
    dist = (lens.long()[:, None, None] + i - j).clamp(0, rel_bias.shape[1] - 1)               # [B, s, L]
    return rel_bias[:, dist].permute(1, 0, 2, 3)


def bf16_bias_term(bias):
    """The relative error of each unnormalised probability when a kernel scores with the bf16 rounding of the fp32
    ``bias``: rounding to nearest moves every score by at most half a unit in the last place, ``|δ| <= 2^-9 |b|`` (eight
    significant bits), and ``e^(z + δ) = e^z (1 + ε)`` with ``|ε| <= e^|δ| - 1``.  The normaliser is a sum of the same
    probabilities, so ``attention_fwd_ref`` carries this term through ``O = N / l`` like its own roundings.  Over a
    window, the largest is ``expm1(2^-9·max|bias|)``."""
    return torch.expm1(2.0 ** -9 * bias.double().abs())


def fp8_decode_terms(q, k64, scale):
    """What the FP8 decode kernel adds to ``attention_fwd_ref``'s bound over ``float(e)·s``, as (``eta_extra``
    [B, A, s, L], an absolute term).  q ``[B, s, A, D]`` bf16, k64 ``[B, G, L, D]`` the fp64 ``float(e)·s`` rows.

    Scores: the kernel widens the bytes ``ê_j`` to bf16 exactly and sums ``q·ê_j`` in fp32, an error of
    ``D 2^-23 Σ|q||ê_j|``; it then multiplies by ``s^k_j``, which scales that error to exactly the reference's
    ``D 2^-23 Σ|q||k_j|`` (``k_j = ê_j s^k_j``), and rounds once more: ``2^-24 |q·k_j|`` (to first order), i.e. a score
    error of at most ``2^-24 scale Σ|q||k_j|``, a relative error of the probability of the same size.
    Probabilities: the kernel rounds ``P_j s^v_j`` to bf16 where the bf16 kernel rounds ``P_j``.  ``T_j |V_j|`` in the
    reference's bound is ``P_j s^v_j |ê_j| / l``, so its ``2^-8`` term covers that rounding; the fp32 product before it
    adds ``2^-24``.  Below ``2^-126`` the product is flushed to zero (fast math): at most ``2^-126 |ê_j| <= 448 2^-126``
    per key and output element, after the division by ``l >= 1``; over ``L`` keys ``L 448 2^-126`` in all."""
    B, s, A, D = q.shape
    G, L = k64.shape[1], k64.shape[2]
    kx = k64.abs().repeat_interleave(A // G, dim=1)                                           # [B, A, L, D]
    qk = torch.einsum("bqhd,bhkd->bhqk", q.double().abs(), kx)
    return 2.0 ** -24 * (scale * qk + 1.0), L * 448.0 * 2.0 ** -126


def expect(q, k64, v64, *, scale, vis, bias=None, alibi=None, tile, eta_extra=None, extra_abs=0.0):
    """(ref, bound) ``[B, s, A, D]`` of the attention of q ``[B, s, A, D]`` over the fp64 rows (``attention_fwd_ref``)."""
    (o, ob), _ = R.attention_fwd_ref(q.permute(0, 2, 1, 3), k64, v64, scale=scale, vis=vis, bias=bias, alibi=alibi,
                                     tile=tile, eta_extra=eta_extra)
    ob = torch.where(vis.any(-1)[..., None].expand_as(ob), ob + extra_abs, ob)
    return o.permute(0, 2, 1, 3), ob.permute(0, 2, 1, 3)


class Recorder:
    """The extension with every call recorded.  Attention calls are described: ``("decode_attn", fp8)``,
    ``("attn_fwd", bias, alibi, kv_start, key rows, key dtype)`` (the first three: whether the argument was given), and
    over a paged cache ``("decode_attn_paged", fp8)`` and ``("attn_fwd_paged", alibi, past)``."""

    APPENDS = ("kv_append", "kv_append_fp8", "kv_append_paged", "kv_append_fp8_paged")

    def __init__(self, ext):
        self.ext, self.calls = ext, []

    def __getattr__(self, name):
        fn = getattr(self.ext, name)
        if not callable(fn):
            return fn

        def wrapped(*a, **k):
            if name == "decode_attn":
                self.calls.append(("decode_attn", len(a) > 10 and a[10] is not None))
            elif name == "attn_fwd":
                kv_start = a[10] if len(a) > 10 else k.get("kv_start")
                self.calls.append(("attn_fwd", a[6] is not None, a[7] is not None, kv_start is not None,
                                   a[1].shape[-2], a[1].dtype))
            elif name == "decode_attn_paged":   # (q, k, v, table, seqlens, kv_start, scale, splits, alibi, k_scale, ..)
                self.calls.append(("decode_attn_paged", a[9] is not None))
            elif name == "attn_fwd_paged":      # (q, k, v, table, past, scale, kv_start, alibi)
                self.calls.append(("attn_fwd_paged", a[7] is not None, int(a[4])))
            else:
                self.calls.append((name,))
            return fn(*a, **k)
        return wrapped

    def take(self):
        """The calls since the last ``take`` other than cache appends."""
        out = [c for c in self.calls if c[0] not in self.APPENDS]
        self.calls = []
        return out
