"""Seeded flash-attention backward cases whose dq / dk / dv (and dbias) bytes are pinned in
tests/golden/attn_bwd_parent.json.  The file was written by dev/attn_bwd_golden.py with the backward kernel as it was
before the warp-specialised schedule (one consumer warpgroup per 64-key block), so every later schedule must reproduce
those bytes exactly: the per-visit arithmetic and the order of every fp32 dQ addition are part of the kernel's
contract.  Inputs come from a CPU torch.Generator, so they do not depend on the device's random number generator."""
import hashlib

import torch

GOLDEN = "tests/golden/attn_bwd_parent.json"

# name: B, A, G, Sq, Sk, d, causal, extra
CASES = {
    "d64_mha_causal_s1024": (2, 8, 8, 1024, 1024, 64, True, None),
    "d64_gqa4_causal_s203": (2, 8, 2, 203, 203, 64, True, None),
    "d64_mqa_full_s129": (2, 8, 1, 129, 129, 64, False, None),
    "d24_mha_causal_s129": (2, 4, 4, 129, 129, 24, True, None),
    "d80_mqa_causal_rect_77x203": (2, 4, 1, 77, 203, 80, True, None),
    "d128_mha_causal_rect_203x77": (2, 4, 4, 203, 77, 128, True, None),
    "d128_gqa4_causal_s1000": (1, 8, 2, 1000, 1000, 128, True, None),
    "d64_full_rect_300x1": (2, 4, 4, 300, 1, 64, False, None),
    "d64_causal_s65_windows": (2, 4, 2, 65, 65, 64, True, "windows"),
    "d64_full_rect_77x203_dense_bias": (2, 8, 2, 77, 203, 64, False, "bias"),
    "d128_causal_s129_dense_bias": (2, 4, 4, 129, 129, 128, True, "bias"),
    "d64_causal_s203_alibi": (2, 8, 8, 203, 203, 64, True, "alibi"),
    "d64_causal_s203_dropout": (2, 4, 2, 203, 203, 64, True, "dropout"),
    "d128_full_s129_dropout_bias": (2, 4, 4, 129, 129, 128, False, "dropout_bias"),
    "d64_doc_start_s1000": (2, 4, 2, 1000, 1000, 64, True, "doc"),
    "d128_doc_start_s203": (2, 4, 4, 203, 203, 128, True, "doc"),
    # the attention shape of the GPT-2 medium training step
    "bench_b8_h16_s1024_d64": (8, 16, 16, 1024, 1024, 64, True, None),
}
DROPOUT_RNG_STATE = (0x5DEECE66D, 0x1234)   # (seed, offset) of the dropout stream


def _randn(gen, *shape, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).bfloat16()


def make_inputs(name, device):
    """The arguments of ext.attn_fwd / ext.attn_bwd for one case, on `device`."""
    B, A, G, Sq, Sk, d, causal, extra = CASES[name]
    gen = torch.Generator().manual_seed(int.from_bytes(hashlib.sha256(name.encode()).digest()[:4], "little"))
    q = _randn(gen, B, A, Sq, d).to(device)
    k = _randn(gen, B, G, Sk, d).to(device)
    v = _randn(gen, B, G, Sk, d).to(device)
    do = _randn(gen, B, A, Sq, d).to(device)
    kw = dict(kv_start=None, kv_lens=None, bias=None, alibi=None, p=0.0, rng_state=None, doc_start=None)
    if extra == "windows":
        kw["kv_start"] = torch.tensor([3, 20], dtype=torch.int32).to(device)
        kw["kv_lens"] = torch.tensor([Sk, 50], dtype=torch.int32).to(device)
    if extra in ("bias", "dropout_bias"):
        pad = (Sk + 7) // 8 * 8   # row stride a multiple of 8 elements, as the kernel requires
        bias = torch.zeros(1, A, Sq, pad, dtype=torch.bfloat16)
        bias[..., :Sk] = _randn(gen, 1, A, Sq, Sk, scale=2.0)
        kw["bias"] = bias.to(device)[..., :Sk]
    if extra == "alibi":
        kw["alibi"] = torch.tensor([2.0 ** (-8 * (h + 1) / A) for h in range(A)]).to(device)
    if extra in ("dropout", "dropout_bias"):
        kw["p"] = 0.1
        kw["rng_state"] = torch.tensor(DROPOUT_RNG_STATE, dtype=torch.int64).to(device)
    if extra == "doc":
        # non-monotone document starts: runs of random length, some rows pointing anywhere (clamped by the kernel)
        g = torch.Generator().manual_seed(Sq)
        rows = []
        for _ in range(B):
            ds, at = [], 0
            while at < Sq:
                n = int(torch.randint(1, 150, (1,), generator=g))
                ds += [at] * min(n, Sq - at)
                at += n
            wild = torch.rand(Sq, generator=g) < 0.1
            noise = torch.randint(-10, Sq + 10, (Sq,), generator=g)
            rows.append(torch.where(wild, noise, torch.tensor(ds)))
        kw["doc_start"] = torch.stack(rows).to(torch.int32).to(device)
    return q, k, v, do, causal, d ** -0.5, kw


def run_backward(ext, name, device):
    """Forward (without dropout: o and lse only feed the backward) then the backward; returns the gradients."""
    q, k, v, do, causal, scale, kw = make_inputs(name, device)
    o, lse, _ = ext.attn_fwd(q, k, v, causal, scale, kw["kv_lens"], kw["bias"], kw["alibi"], 0.0, 0, kw["kv_start"],
                             kw["doc_start"])
    dbias = None
    if kw["bias"] is not None:
        b = kw["bias"]
        dbias = torch.empty_strided(b.shape, b.stride(), dtype=torch.float32, device=device).zero_()
    dq, dk, dv, _ = ext.attn_bwd(do, q, k, v, o, lse, causal, scale, kw["kv_lens"], kw["bias"], kw["alibi"], dbias,
                                 kw["p"], kw["rng_state"], kw["kv_start"], kw["doc_start"])
    out = dict(dq=dq, dk=dk, dv=dv)
    if dbias is not None:
        out["dbias"] = dbias
    return out


def digests(out):
    """SHA-256 of each gradient's bytes in a fixed (contiguous) layout."""
    res = {}
    for n, t in out.items():
        t = t.contiguous()
        raw = t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)
        res[n] = hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest()
    return res
