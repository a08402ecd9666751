"""Every branch of cached attention on the H100 against fp64, element by element (tests/cached_attention_ref.py builds
the references, tests/attention_ref.py states the bounds): ``OF.decode_attention`` on bf16 and FP8 caches across the
16/17-token switch between the split-KV decode kernel and the flash kernel, for causal, ALiBi, T5 relative-bias and
cross-attention scores, and ``KVCacheLayer.attend`` on a real ``StaticKVCache`` from a left-padded prompt through
chunked prefill, decode steps, dense-mask and dense-bias steps, a cross-attention window and T5's relative bias.

Every case asserts which kernel ran (a silent fall-back to the reference math fails), a contiguous ``[b, s, a, d]``
output, and a finite one: rows at or past the window end hold NaN, and masked rows inside it hold sentinels that a leak
would carry far past the bound."""
import pytest
import torch

from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.ops import functional as OF
from tests import cached_attention_ref as CR
from tests.dense_ref import check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP8 = torch.float8_e4m3fn
BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


@pytest.fixture
def rec(ext, monkeypatch):
    r = CR.Recorder(ext)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: r)
    return r


def _slopes(A):
    from projects.BLOOM.modeling.bloom_model import alibi_slopes

    return alibi_slopes(A).to(DEV)


def _rand(*shape, g, scale=1.0):
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(BF16)


def _quantized(k, v, fp8):
    """The cache buffers holding the bf16 rows ``k``, ``v``: as they are, or quantized with their row scales."""
    if not fp8:
        return k, v, None, None
    (k8, ks), (v8, vs) = OF.kv_cache_quantize_ref(k), OF.kv_cache_quantize_ref(v)
    return k8, v8, ks, vs


def _check_out(o, B, s, A, D, what):
    assert o.shape == (B, s, A, D) and o.is_contiguous(), (what, o.shape, o.stride())
    assert bool(torch.isfinite(o).all()), f"{what}: non-finite output"


def _flash_bias_checks(o, q, k64, v64, *, scale, vis, bias32, what):
    """A flash branch scoring with the dense bias rounded to bf16: against fp64 with that bias (the kernel's input),
    and against fp64 with the fp32 bias the decode kernel uses plus the rounding's term (``CR.bf16_bias_term``)."""
    ref, bnd = CR.expect(q, k64, v64, scale=scale, vis=vis, bias=bias32.to(BF16).double(), tile=128)
    check(o, ref, bnd, what + " (bf16 bias)")
    ref, bnd = CR.expect(q, k64, v64, scale=scale, vis=vis, bias=bias32.double(), tile=128,
                         eta_extra=CR.bf16_bias_term(bias32))
    check(o, ref, bnd, what + " (fp32 bias)")


# ------------------------------------------------------------------------------------------------ OF.decode_attention
KINDS = ["causal", "alibi", "rel_small", "rel_large", "window"]
CACHES = ["bf16", "fp8"]
SQ = [1, 15, 16, 17, 64, 200]
PASTS = [0, 1, 63, 1037]
CROSS_PASTS = [5, 1, 63, 1037]   # a cross-attention window holds a row at least; none ends on a 64-row tile
HEADS = [(8, 8), (8, 2)]         # MHA, and grouped-query with 4 query heads per key/value head


def _cases():
    # every (kind, cache, s) meets two pasts; across the kinds every s meets every past, both head dims and both
    # head groupings
    out = []
    for ki, kind in enumerate(KINDS):
        for ci, cache in enumerate(CACHES):
            for si, s in enumerate(SQ):
                for j in range(2):
                    past = (CROSS_PASTS if kind == "window" else PASTS)[(si + ki + 2 * j) % 4]
                    D = (64, 128)[(si + ci + j) % 2]
                    A, G = HEADS[(ki + ci + si // 2 + j) % 2]
                    out.append((kind, cache, s, past, D, A, G))
    return out


CASES = _cases()


def _decode_case(kind, fp8, s, past, D, A, G, seed, lens=None, starts=None):
    """q and caches of three samples.  Causal kinds: every sample holds ``past`` rows; sample 0 sees from row 0, sample
    1 is left padded and sample 2's ``kv_start`` is the window end (no visible key: zeros).  Cross-attention
    (``window``): the cache holds ``past`` rows, sample 1 sees a shorter window ``[7, past - 20)``, sample 2 none.
    Masked rows inside the window hold sentinels, rows from the window end to the capacity (not a multiple of 64, a
    multiple of 4 for FP8) NaN.  Returns the caches, their bf16 rows, lens, kv_start, the window end ``L`` and the
    rows each sample's NaN starts at."""
    B = 3
    causal = kind != "window"
    if lens is None:
        if causal:
            lens = [past] * B
            starts = [0, min(37, (past + s) // 2), past + s]
        else:
            lens = [past, max(1, past - 20), past]
            starts = [0, min(7, lens[1] - 1), past]
    L = max(lens) + (s if causal else 0)
    C = L + 13
    C += -C % 4 if fp8 else 0
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = _rand(B, s, A, D, g=g)
    k, v = _rand(B, G, C, D, g=g, scale=2.0), _rand(B, G, C, D, g=g)
    ends = [n + s if causal else past for n in lens]
    for b in range(B):
        CR.sentinel_rows(k, v, b, 0, starts[b])
        if not causal:
            CR.sentinel_rows(k, v, b, lens[b], past)
    kc, vc, ks, vs = _quantized(k, v, fp8)
    for b in range(B):
        CR.poison(kc, vc, ks, vs, b, ends[b])
    return q, kc, vc, ks, vs, CR.i32(lens, DEV), CR.i32(starts, DEV), L


def _bias_of(kind, A, L, seed):
    if kind == "alibi":
        return _slopes(A)
    if kind.startswith("rel"):
        R = 33 if kind == "rel_small" else L + 50
        return torch.randn(A, R, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    return None


def _call(q, kc, vc, ks, vs, lens, starts, *, kind, scale, past, bias):
    kw = dict(scale=scale, past=past, causal=kind != "window")
    if ks is not None:
        kw.update(k_scale=ks, v_scale=vs)
    if kind == "alibi":
        kw["alibi_slopes"] = bias
    elif kind.startswith("rel"):
        kw["rel_bias"] = bias
    return OF.decode_attention(q, kc, vc, lens, starts, **kw)


def _check_decode_attention(o, q, kc, vc, ks, vs, lens, starts, *, kind, scale, bias, L, kernel, what):
    """o against fp64 over the rows the branch read: ``kernel`` is "decode", "flash" or "ref" (the reference math)."""
    B, s, A, D = q.shape
    causal = kind != "window"
    k64, v64 = CR.rows64(kc, vc, ks, vs, L, exact=kernel == "decode")
    vis = CR.visible(lens, starts, s, L, causal)
    tile = 128 if kernel == "flash" else 64   # the reference math rounds less than either kernel
    eta, extra = (CR.fp8_decode_terms(q, k64, scale) if kernel == "decode" and ks is not None else (None, 0.0))
    kw = dict(scale=scale, vis=vis, tile=tile, eta_extra=eta, extra_abs=extra)
    if kind == "alibi":
        # the kernels' slope·(j - lens[b] - i); with equal lens it is attention_fwd_ref's slope·(j - i - (L - s))
        rel = (torch.arange(L, device=DEV)[None, None, :] - lens.long()[:, None, None]
               - torch.arange(s, device=DEV)[None, :, None]).double()
        kw["bias"] = bias.double()[None, :, None, None] * rel[:, None]
    if kind.startswith("rel"):
        dense = CR.rel_dense(bias, lens, s, L)
        if kernel == "flash":
            _flash_bias_checks(o, q, k64, v64, scale=scale, vis=vis, bias32=dense, what=what)
            return
        kw["bias"] = dense.double()
    ref, bnd = CR.expect(q, k64, v64, **kw)
    check(o, ref, bnd, what)


@pytest.mark.parametrize("kind,cache,s,past,D,A,G", CASES,
                         ids=[f"{k}-{c}-s{s}-past{p}-D{d}-A{a}G{g}" for k, c, s, p, d, a, g in CASES])
def test_decode_attention_matches_fp64(rec, kind, cache, s, past, D, A, G):
    fp8 = cache == "fp8"
    seed = CASES.index((kind, cache, s, past, D, A, G))
    q, kc, vc, ks, vs, lens, starts, L = _decode_case(kind, fp8, s, past, D, A, G, seed)
    bias = _bias_of(kind, A, L, seed)
    scale = D ** -0.5
    o = _call(q, kc, vc, ks, vs, lens, starts, kind=kind, scale=scale, past=past, bias=bias)
    what = f"{kind} {cache} s={s} past={past} D={D} A/G={A}/{G}"
    _check_out(o, 3, s, A, D, what)
    if s <= 16:
        kernel, want = "decode", [("decode_attn", fp8)]
    else:
        # the flash kernel over the window [:past + s] (causal) or [:past] (cross), an FP8 one dequantized to bf16
        kernel = "flash"
        want = [("attn_fwd", kind.startswith("rel"), kind == "alibi", True, L, BF16)]
    assert rec.take() == want, what
    _check_decode_attention(o, q, kc, vc, ks, vs, lens, starts, kind=kind, scale=scale, bias=bias, L=L, kernel=kernel,
                            what=what)
    assert torch.equal(o[2], torch.zeros_like(o[2])), what   # kv_start at the window end


FALLBACK = [(k, c, s) for k in ("causal", "alibi", "rel_small") for c in CACHES for s in (17, 40)]


@pytest.mark.parametrize("kind,cache,s", FALLBACK)
def test_decode_attention_without_past_runs_the_reference_math(rec, kind, cache, s):
    """More than 16 causal tokens without ``past=`` and unequal lengths: the reference math over ``[:max(lens) + s]``,
    in which the shorter samples' rows past their own window end hold NaN."""
    fp8 = cache == "fp8"
    A, G, D = 8, 2, 64
    seed = 500 + FALLBACK.index((kind, cache, s))
    q, kc, vc, ks, vs, lens, starts, L = _decode_case(kind, fp8, s, None, D, A, G, seed, lens=[300, 41, 150],
                                                      starts=[0, 9, 150 + s])
    bias = _bias_of(kind, A, L, seed)
    scale = D ** -0.5
    o = _call(q, kc, vc, ks, vs, lens, starts, kind=kind, scale=scale, past=None, bias=bias)
    what = f"fallback {kind} {cache} s={s}"
    _check_out(o, 3, s, A, D, what)
    assert rec.take() == [], what
    _check_decode_attention(o, q, kc, vc, ks, vs, lens, starts, kind=kind, scale=scale, bias=bias, L=L, kernel="ref",
                            what=what)


@pytest.mark.parametrize("kind", ["causal", "alibi", "rel_small", "rel_large"])
@pytest.mark.parametrize("D", [64, 128])
def test_decode_and_flash_agree_across_the_switch(rec, kind, D):
    """The first 16 of 17 new tokens see the same keys as 16 new tokens: the decode kernel (16) and the flash kernel
    (17) must agree within the sum of their bounds against one fp64 reference.  With T5's relative bias the flash side
    scores with its bf16 rounding and the decode side with the fp32 bias; ``CR.bf16_bias_term`` states that part."""
    A, G, past = 8, 2, 1037
    seed = 900 + D + len(kind)
    q, kc, vc, ks, vs, lens, starts, L17 = _decode_case(kind, False, 17, past, D, A, G, seed, lens=[past] * 3,
                                                        starts=[0, 37, 500])
    bias = _bias_of(kind, A, L17, seed)
    scale = D ** -0.5
    o17 = _call(q, kc, vc, ks, vs, lens, starts, kind=kind, scale=scale, past=past, bias=bias)
    o16 = _call(q[:, :16].contiguous(), kc, vc, ks, vs, lens, starts, kind=kind, scale=scale, past=past, bias=bias)
    assert [c[0] for c in rec.take()] == ["attn_fwd", "decode_attn"]
    k64, v64 = CR.rows64(kc, vc, None, None, L17, exact=True)
    vis = CR.visible(lens, starts, 17, L17, True)
    kw = dict(scale=scale, vis=vis)
    if kind == "alibi":
        kw["alibi"] = bias
    if kind.startswith("rel"):
        dense = CR.rel_dense(bias, lens, 17, L17)
        kw["bias"] = dense.double()
    ref17, bnd17 = CR.expect(q, k64, v64, tile=128, eta_extra=CR.bf16_bias_term(dense) if "bias" in kw else None, **kw)
    ref16, bnd16 = CR.expect(q, k64, v64, tile=64, **kw)
    diff = (o17[:, :16].double() - o16.double()).abs()
    check(o16, ref16[:, :16], bnd16[:, :16], f"{kind} D={D} decode side")
    check(o17, ref17, bnd17, f"{kind} D={D} flash side")
    check(diff, torch.zeros_like(diff), bnd16[:, :16] + bnd17[:, :16], f"{kind} D={D} decode vs flash")
    print(f"\n[switch 16/17] {kind} D={D}: max|o17 - o16| = {float(diff.max()):.3e}, "
          f"max|o17 - o16| / bound = {float((diff / (bnd16[:, :16] + bnd17[:, :16])).nan_to_num(0).max()):.3f}")


# ------------------------------------------------------------------------------------------------ KVCacheLayer.attend
def _cache(B, G, D, capacity, fp8, S=0):
    """A one-layer StaticKVCache whose every row is NaN until written."""
    c = StaticKVCache(1, B, G, D, capacity, BF16, DEV, kv_dtype=FP8 if fp8 else None)
    assert c.capacity % 64 and (not fp8 or c.capacity % 4 == 0)
    for b in range(B):
        CR.poison(c.k[0], c.v[0], c.k_scale[0], c.v_scale[0], b, 0)
    return c


def _projection(B, s, A, G, D, g, pad=None):
    """A packed projection — per-head ``[B, s, A, 3D]`` for MHA, grouped ``[B, s, G, r + 2, D]`` otherwise — whose k
    and v of sample b's first ``pad[b]`` tokens are the sentinels."""
    r = A // G
    if r == 1:
        qkv = _rand(B, s, A, 3 * D, g=g)
        ksl, vsl = (Ellipsis, slice(D, 2 * D)), (Ellipsis, slice(2 * D, 3 * D))
    else:
        qkv = _rand(B, s, G, r + 2, D, g=g)
        ksl, vsl = (Ellipsis, r, slice(None)), (Ellipsis, r + 1, slice(None))
    for b, n in enumerate(pad or []):
        qkv[b, :n][ksl] = CR.SENT_K
        qkv[b, :n][vsl] = CR.SENT_V
    return qkv


def _layer_rows(c, L, exact):
    return CR.rows64(c.k[0], c.v[0], c.k_scale[0], c.v_scale[0], L, exact)


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("alibi", [False, True], ids=["plain", "alibi"])
def test_attend_walks_a_static_cache(rec, cache, alibi):
    """A left-padded prompt (flash prefill, the padding in kv_start), a 150-token continuation (chunked prefill), 1-
    and 16-token decode steps, a dense-mask step (the reference math) and a dense-bias step (the flash kernel with the
    bias), each against fp64 over the rows the appends stored."""
    fp8 = cache == "fp8"
    B, D = 3, 64 if alibi else 128
    A, G = (8, 8) if alibi else (8, 2)    # BLOOM is MHA; the Llama family groups its heads
    scale = D ** -0.5
    c = _cache(B, G, D, 301, fp8)
    layer = c.layer(0)
    slopes = _slopes(A) if alibi else None
    g = torch.Generator(device=DEV).manual_seed(11 + alibi + 2 * fp8)
    pad = [0, 5, 20]
    s0 = 37
    mask = torch.ones(B, s0, dtype=torch.long, device=DEV)
    for b, n in enumerate(pad):
        mask[b, :n] = 0
    assert c.step_needs_dense_mask(mask, flash=c.flash_attention()) is False
    assert c.kv_start.tolist() == pad

    def step(s, want, kernel, **kw):
        past = c.length
        q = layer.append(_projection(B, s, A, G, D, g, pad if past == 0 else None))
        rec.take()
        o = layer.attend(q, scale=scale, **kw)
        what = f"{cache} alibi={alibi} past={past} s={s} {kernel}"
        _check_out(o, B, s, A, D, what)
        assert rec.take() == want, what
        L = past + s
        k64, v64 = _layer_rows(c, L, exact=kernel == "decode")
        if "mask" in kw:
            vis = kw["mask"].bool()
        elif "bias" in kw:
            # the model's padding and causality folded into the bias as -30000: the kernel's exp2 of such a score is
            # exactly 0, so those keys are the reference's invisible ones
            vis = (kw["bias"] > -1000)[:, :1]
        else:
            vis = CR.visible(torch.full_like(c.seqlens, past), c.kv_start, s, L, True)
        eta, extra = CR.fp8_decode_terms(q, k64, scale) if kernel == "decode" and fp8 else (None, 0.0)
        bias = kw["bias"].to(BF16).double() if "bias" in kw else None
        ref, bnd = CR.expect(q, k64, v64, scale=scale, vis=vis, bias=bias, alibi=kw.get("alibi_slopes"),
                             tile=128 if kernel == "flash" else 64, eta_extra=eta, extra_abs=extra)
        check(o, ref, bnd, what)
        c.advance(s)

    al = (slopes is not None)
    step(s0, [("attn_fwd", False, al, True, s0, BF16)], "flash", alibi_slopes=slopes)
    step(150, [("attn_fwd", False, al, True, s0 + 150, BF16)], "flash", alibi_slopes=slopes)
    step(1, [("decode_attn", fp8)], "decode", alibi_slopes=slopes)
    step(16, [("decode_attn", fp8)], "decode", alibi_slopes=slopes)
    # a dense 0/1 mask [b, 1, s, L] (causality, the padding and a few holes) runs the reference math
    L = c.length + 5
    vis = CR.visible(torch.full_like(c.seqlens, c.length), c.kv_start, 5, L, True)
    holes = torch.rand(vis.shape, device=DEV, generator=g) < 0.2
    holes[..., c.length :] = False                       # every query still sees itself
    step(5, [], "ref", mask=(vis & ~holes).to(torch.uint8))
    L = c.length + 3
    vis = CR.visible(torch.full_like(c.seqlens, c.length), c.kv_start, 3, L, True).expand(B, A, 3, L)
    bias = torch.randn(B, A, 3, L, device=DEV, generator=g).masked_fill(~vis, -30000.0)
    step(3, [("attn_fwd", True, False, False, L, BF16)], "flash", bias=bias)


@pytest.mark.parametrize("cache", CACHES)
def test_attend_cross_attention_window(rec, cache):
    """A cross-attention cache of S = 75 rows (capacity past S, every row past S NaN) made by ``fill(window=)``: sample
    0 sees all S rows, sample 1 rows [3, S - 10), sample 2 none.  Read at 1 (decode kernel) and 40 (flash) queries."""
    fp8 = cache == "fp8"
    B, A, G, D, S = 3, 8, 2, 64, 75
    scale = D ** -0.5
    c = _cache(B, G, D, S + 30, fp8)
    g = torch.Generator(device=DEV).manual_seed(21 + fp8)
    starts, ends = [0, 3, 50], [S, S - 10, 50]
    k, v = _rand(B, G, S, D, g=g, scale=2.0), _rand(B, G, S, D, g=g)
    for b in range(B):
        CR.sentinel_rows(k, v, b, 0, starts[b])
        CR.sentinel_rows(k, v, b, ends[b], S)
    c.fill([(k, v)], S, window=(CR.i32(starts, DEV), CR.i32(ends, DEV)))
    layer = c.layer(0)
    for s in (1, 40):
        q = _rand(B, s, A, D, g=g)
        rec.take()
        o = layer.attend(q, scale=scale, causal=False)
        what = f"cross {cache} s={s}"
        _check_out(o, B, s, A, D, what)
        kernel = "decode" if s <= 16 else "flash"
        want = [("decode_attn", fp8)] if s <= 16 else [("attn_fwd", False, False, True, S, BF16)]
        assert rec.take() == want, what
        k64, v64 = _layer_rows(c, S, exact=kernel == "decode")
        vis = CR.visible(c.seqlens, c.kv_start, s, S, False)
        eta, extra = CR.fp8_decode_terms(q, k64, scale) if kernel == "decode" and fp8 else (None, 0.0)
        ref, bnd = CR.expect(q, k64, v64, scale=scale, vis=vis, tile=64 if kernel == "decode" else 128, eta_extra=eta,
                             extra_abs=extra)
        check(o, ref, bnd, what)
        assert torch.equal(o[2], torch.zeros_like(o[2])), what


@pytest.mark.parametrize("cache", CACHES)
def test_attend_t5_relative_bias(rec, cache):
    """T5's causal self-attention with ``rel_bias``: a 20-token first step (the flash kernel with the dense bias, even
    though the cache was empty), then a 1-token step (the decode kernel with the fp32 bias)."""
    fp8 = cache == "fp8"
    B, A, G, D = 3, 8, 8, 64
    scale = D ** -0.5
    c = _cache(B, G, D, 59, fp8)
    layer = c.layer(0)
    g = torch.Generator(device=DEV).manual_seed(31 + fp8)
    rel = torch.randn(A, 32, device=DEV, generator=g)
    for s, want in ((20, [("attn_fwd", True, False, True, 20, BF16)]), (1, [("decode_attn", fp8)])):
        past = c.length
        q = layer.append(_projection(B, s, A, G, D, g))
        rec.take()
        o = layer.attend(q, scale=scale, rel_bias=rel)
        what = f"t5 {cache} past={past} s={s}"
        _check_out(o, B, s, A, D, what)
        assert rec.take() == want, what
        L = past + s
        lens = torch.full_like(c.seqlens, past)
        vis = CR.visible(lens, c.kv_start, s, L, True)
        dense = CR.rel_dense(rel, lens, s, L)
        if s > 16:
            k64, v64 = _layer_rows(c, L, exact=False)
            _flash_bias_checks(o, q, k64, v64, scale=scale, vis=vis, bias32=dense, what=what)
        else:
            k64, v64 = _layer_rows(c, L, exact=True)
            eta, extra = CR.fp8_decode_terms(q, k64, scale) if fp8 else (None, 0.0)
            ref, bnd = CR.expect(q, k64, v64, scale=scale, vis=vis, bias=dense.double(), tile=64, eta_extra=eta,
                                 extra_abs=extra)
            check(o, ref, bnd, what)
        c.advance(s)
