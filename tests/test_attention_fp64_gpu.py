"""The attention kernels on the H100 against fp64, element by element (tests/attention_ref.py states the bounds): the
flash forward and backward over ragged and rectangular shapes, grouped heads, key windows, dense and ALiBi bias and
dropout (masks rebuilt from the Philox mirror, also under CUDA-graph replay); the decode kernel at every split count;
bias_dropout_residual against the mirror; rope, rope_qkv and kv_append."""
import struct

import pytest
import torch

from libai_b200.ops import functional as OF
from tests import attention_ref as R
from tests.dense_ref import FLUSH, ROUND, check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF = ROUND[torch.bfloat16]


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def rand(*shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).bfloat16()


def generator_state():
    """(seed, offset) of the default CUDA generator: get_rng_state() is the 8-byte seed then the 8-byte offset."""
    st = bytes(torch.cuda.get_rng_state(DEV).tolist())
    assert len(st) == 16
    return struct.unpack("<QQ", st)


def stored_state(rng_state):
    s, o = (int(x) for x in rng_state.cpu().tolist())
    return s & 0xFFFFFFFFFFFFFFFF, o & 0xFFFFFFFFFFFFFFFF


def windows(kind, B, Sq, Sk, causal):
    """(kv_start, kv_lens) of a window kind for B = 2 samples."""
    def t(xs):
        return torch.tensor(xs, dtype=torch.int32, device=DEV)
    if kind == "none":
        return None, None
    if kind == "lens":                      # the second sample's 0 is clamped to 1 key
        return None, t([max(1, Sk - 37), 0])
    if kind == "start_lens":
        return t([min(3, Sk - 1), Sk // 3]), t([Sk, max(1, Sk - 5)])
    # "empty": rows without a visible key (all of sample 1 without causality, its early rows with it)
    if causal:
        return t([0, max(0, Sk - (Sq + 1) // 2)]), None
    return t([0, min(10, Sk - 1)]), t([Sk, min(10, Sk - 1)])


def run_flash(ext, q, k, v, do, *, causal, scale, kv_start=None, kv_lens=None, bias=None, alibi=None, p=0.0, salt=0,
              want_dbias=False):
    o, lse, st = ext.attn_fwd(q, k, v, causal, scale, kv_lens, bias, alibi, p, salt, kv_start)
    # fp32 with the strides of the (possibly row-padded) bias, as the binding requires
    dbias = torch.empty_strided(bias.shape, bias.stride(), dtype=torch.float32, device=DEV).zero_() if want_dbias else None
    dq, dk, dv, _ = ext.attn_bwd(do, q, k, v, o, lse, causal, scale, kv_lens, bias, alibi, dbias, p,
                                 st if p > 0 else None, kv_start)
    out = dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv)
    if want_dbias:
        out["dbias"] = dbias
    return out, st


def check_flash(ext, q, k, v, do, *, causal, scale, what, kv_start=None, kv_lens=None, bias=None, alibi=None, p=0.0,
                salt=0):
    """Runs the flash kernels and checks O, lse, dQ, dK, dV (and dbias) per element; q is [B, A, Sq, D] or the grouped
    [B, G, r, Sq, D].  With dropout the mask is rebuilt from the stored state, which must be the generator's."""
    B, G, Sk = k.shape[0], k.shape[1], k.shape[2]
    q4 = q if q.dim() == 4 else q.reshape(B, -1, q.shape[-2], q.shape[-1])
    A, Sq = q4.shape[1], q4.shape[2]
    gen = generator_state()
    got, st = run_flash(ext, q, k, v, do, causal=causal, scale=scale, kv_start=kv_start, kv_lens=kv_lens, bias=bias,
                        alibi=alibi, p=p, salt=salt, want_dbias=bias is not None)
    keep, ik = None, 1.0
    if p > 0:
        seed, off = stored_state(st)
        assert (seed, off) == (R.salted_seed(gen[0], salt), gen[1]), "rng_state is not the generator's (seed ^ salt, offset)"
        assert generator_state() == (gen[0], gen[1] + 4), "the generator offset must advance by 4 per call"
        thr, ik = R.attn_drop_threshold(p)
        keep = R.attn_keep_mask(seed, off, B, A, Sq, Sk, thr, device=DEV)
    got["dq"] = got["dq"].reshape(B, A, Sq, -1)
    vis = OF.visible_keys(Sq, Sk, causal=causal, kv_start=kv_start, kv_lens=kv_lens, device=DEV)
    (o, ob), (lse, lseb) = R.attention_fwd_ref(q4, k, v, scale=scale, vis=vis, bias=bias, alibi=alibi, keep=keep,
                                               inv_keep=ik, tile=128)
    check(got["o"], o, ob, what + " o")
    check(got["lse"], lse, lseb, what + " lse")
    ref = R.attention_bwd_ref(q4, k, v, do, got["o"], got["lse"], scale=scale, vis=vis, bias=bias, alibi=alibi,
                              keep=keep, inv_keep=ik)
    R.check_all(got, ref, what)
    return got, st


# ------------------------------------------------------------------------------------------------ flash, per element
SHAPES = [(1, 300), (63, 63), (65, 129), (77, 203), (203, 77), (128, 1000), (1000, 1000)]
HEADS = [(8, 8), (8, 2), (8, 1)]
WINDOWS = ["none", "lens", "start_lens", "empty"]


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("si", range(len(SHAPES)))
def test_flash_per_element(ext, D, causal, si):
    Sq, Sk = SHAPES[si]
    # every shape meets every head grouping and window kind across the (D, causal) combinations
    n = 2 * si + (D == 128) * 1 + causal * 3
    A, G = HEADS[n % 3]
    wk = WINDOWS[n % 4]
    B = 2
    seed = 1000 * si + 10 * D + causal
    q, k, v, do = rand(B, A, Sq, D, seed=seed), rand(B, G, Sk, D, seed=seed + 1), rand(B, G, Sk, D, seed=seed + 2), \
        rand(B, A, Sq, D, seed=seed + 3)
    kv_start, kv_lens = windows(wk, B, Sq, Sk, causal)
    check_flash(ext, q, k, v, do, causal=causal, scale=D ** -0.5, kv_start=kv_start, kv_lens=kv_lens,
                what=f"Sq={Sq} Sk={Sk} D={D} causal={causal} A/G={A}/{G} window={wk}")


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("heads", HEADS)
def test_flash_grouped_packed_projection(ext, D, heads):
    """q read in place as the 5-D [B, G, r, S, D] view of the packed projection [B, S, G, r + 2, D]."""
    A, G = heads
    r, B, S = A // G, 2, 203
    qkv = rand(B, S, G, r + 2, D, seed=7 + D + A * G)
    q = qkv[:, :, :, :r].permute(0, 2, 3, 1, 4)
    k = qkv[:, :, :, r].permute(0, 2, 1, 3)
    v = qkv[:, :, :, r + 1].permute(0, 2, 1, 3)
    do = rand(B, A, S, D, seed=99)
    for causal in (False, True):
        check_flash(ext, q, k, v, do, causal=causal, scale=D ** -0.5, what=f"packed D={D} A/G={A}/{G} causal={causal}")


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("bshape", [(1, 1), (1, 8), (2, 1), (2, 8)])
def test_flash_dense_bias_and_dbias(ext, D, bshape):
    B, A, G, Sq, Sk = 2, 8, 2, 77, 203
    q, k, v, do = rand(B, A, Sq, D, seed=1), rand(B, G, Sk, D, seed=2), rand(B, G, Sk, D, seed=3), rand(B, A, Sq, D, seed=4)
    bias = OF._prep_bias(rand(*bshape, Sq, Sk, seed=5, scale=2.0), q)
    kv_start, kv_lens = windows("start_lens", B, Sq, Sk, True)
    for causal in (False, True):
        check_flash(ext, q, k, v, do, causal=causal, scale=D ** -0.5, bias=bias, kv_start=kv_start, kv_lens=kv_lens,
                    what=f"bias {bshape} D={D} causal={causal}")


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("shape", [(203, 203), (65, 129), (203, 77)])
def test_flash_alibi(ext, D, shape):
    Sq, Sk = shape
    B, A, G = 2, 8, 8
    q, k, v, do = rand(B, A, Sq, D, seed=11), rand(B, G, Sk, D, seed=12), rand(B, G, Sk, D, seed=13), \
        rand(B, A, Sq, D, seed=14)
    slopes = torch.tensor([2.0 ** (-8 * (h + 1) / A) for h in range(A)], device=DEV)
    for causal in (False, True):
        check_flash(ext, q, k, v, do, causal=causal, scale=D ** -0.5, alibi=slopes, what=f"alibi {shape} D={D} causal={causal}")


# ------------------------------------------------------------------------------------------------------------ dropout
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("bias_kind", ["none", "dense", "alibi"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True])
def test_flash_dropout_per_element(ext, p, bias_kind, D, causal):
    B, A, G, S = 2, 4, 4, 203
    seed = int(p * 10) + 3 * D + 7 * causal
    q, k, v, do = rand(B, A, S, D, seed=seed), rand(B, G, S, D, seed=seed + 1), rand(B, G, S, D, seed=seed + 2), \
        rand(B, A, S, D, seed=seed + 3)
    bias = OF._prep_bias(rand(1, A, S, S, seed=seed + 4), q) if bias_kind == "dense" else None
    alibi = torch.tensor([0.5 ** (h + 1) for h in range(A)], device=DEV) if bias_kind == "alibi" else None
    check_flash(ext, q, k, v, do, causal=causal, scale=D ** -0.5, bias=bias, alibi=alibi, p=p,
                what=f"dropout p={p} {bias_kind} D={D} causal={causal}")


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("case", ["gqa4", "mqa", "rect_kv_start", "salted"])
def test_flash_dropout_grouped_rect_salted(ext, p, case):
    B, A, D = 2, 8, 64
    G, Sq, Sk, salt, kv_start, kv_lens = 8, 203, 203, 0, None, None
    if case == "gqa4":
        G = 2
    elif case == "mqa":
        G = 1
    elif case == "rect_kv_start":
        G, Sq, Sk = 2, 77, 203
        kv_start, kv_lens = windows("start_lens", B, Sq, Sk, True)
    else:
        salt = 3
    q, k, v, do = rand(B, A, Sq, D, seed=21), rand(B, G, Sk, D, seed=22), rand(B, G, Sk, D, seed=23), \
        rand(B, A, Sq, D, seed=24)
    check_flash(ext, q, k, v, do, causal=True, scale=D ** -0.5, kv_start=kv_start, kv_lens=kv_lens, p=p, salt=salt,
                what=f"dropout {case} p={p}")


def test_flash_dropout_under_cuda_graph_replay(ext):
    """Forward and backward with dropout captured once; each replay draws a fresh mask, which the outputs must follow."""
    B, A, G, S, D, p = 2, 4, 2, 203, 64, 0.1
    q, k, v, do = rand(B, A, S, D, seed=31), rand(B, G, S, D, seed=32), rand(B, G, S, D, seed=33), rand(B, A, S, D, seed=34)
    scale = D ** -0.5

    def step():
        return run_flash(ext, q, k, v, do, causal=True, scale=scale, p=p, salt=2)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got, st = step()
    thr, ik = R.attn_drop_threshold(p)
    vis = OF.visible_keys(S, S, causal=True, device=DEV)
    states = []
    for rep in range(2):
        graph.replay()
        torch.cuda.synchronize()
        seed, off = stored_state(st)
        states.append((seed, off))
        keep = R.attn_keep_mask(seed, off, B, A, S, S, thr, device=DEV)
        (o, ob), (lse, lseb) = R.attention_fwd_ref(q, k, v, scale=scale, vis=vis, keep=keep, inv_keep=ik, tile=128)
        check(got["o"], o, ob, f"replay {rep} o")
        check(got["lse"], lse, lseb, f"replay {rep} lse")
        ref = R.attention_bwd_ref(q, k, v, do, got["o"], got["lse"], scale=scale, vis=vis, keep=keep, inv_keep=ik)
        R.check_all({n: got[n].reshape(ref[n][0].shape) for n in ref}, ref, f"replay {rep}")
    assert states[0] != states[1], states
    assert states[0][0] == states[1][0] and states[1][1] > states[0][1]
    del graph


# ------------------------------------------------------------------------------------------------------------- decode
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("splits", [1, 2, 7, 0])
@pytest.mark.parametrize("heads_sq", [(8, 8, 1), (8, 2, 4), (8, 1, 2), (4, 4, 16)])
def test_decode_per_element(ext, D, splits, heads_sq):
    A, G, Sq = heads_sq
    B, C = 3, 1100
    lens = torch.tensor([1000, 37, 0], dtype=torch.int32, device=DEV)
    kv_start = torch.tensor([0, 5, 0], dtype=torch.int32, device=DEV)
    seed = D + splits * 7 + A * G + Sq
    q, kc, vc = rand(B, Sq, A, D, seed=seed), rand(B, G, C, D, seed=seed + 1), rand(B, G, C, D, seed=seed + 2)
    scale = D ** -0.5
    o = ext.decode_attn(q, kc, vc, lens, kv_start, scale, splits)
    j = torch.arange(C, device=DEV)[None, None, :]
    i = torch.arange(Sq, device=DEV)[None, :, None]
    vis = (j >= kv_start.long()[:, None, None]) & (j <= lens.long()[:, None, None] + i)
    (ref, bnd), _ = R.attention_fwd_ref(q.permute(0, 2, 1, 3), kc, vc, scale=scale, vis=vis[:, None], tile=64)
    check(o.permute(0, 2, 1, 3), ref, bnd, f"decode D={D} splits={splits} A/G/Sq={heads_sq}")


# ------------------------------------------------------------------------------------------------ bias_dropout_residual
# past the grid cap of the elementwise kernels (SMs * 8 blocks of 256 threads, 8 elements each), so that the grid-stride
# loop runs more than once
BDR_ROWS, BDR_N = 2560, 1024


def test_bias_dropout_all_bf16_values_exact(ext):
    """With bias = residual = None: y = keep ? bf16(fp32(x) * scale) : 0, over every bf16 bit pattern, to the bit."""
    n = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert BDR_ROWS * BDR_N > n * 8 * 256 * 8
    pat = torch.arange(-32768, 32768, dtype=torch.int32, device=DEV).to(torch.int16)
    x = pat.repeat(BDR_ROWS * BDR_N // 65536).view(torch.bfloat16).reshape(BDR_ROWS, BDR_N)
    p, salt = 0.1, 5
    gen = generator_state()
    y, st = ext.bias_dropout_residual(x, None, None, p, salt, None)
    seed, off = stored_state(st)
    assert (seed, off) == (R.salted_seed(gen[0], salt), gen[1])
    assert generator_state() == (gen[0], gen[1] + 4)
    thr, scale = R.bdr_drop_threshold(p)
    keep = R.bdr_keep_mask(seed, off, x.numel(), thr, device=DEV).reshape(x.shape)
    xf = x.float()
    want = (xf * scale).bfloat16()
    # --use_fast_math flushes subnormal fp32 operands and results to zero
    sub = (xf != 0) & (xf.abs() < 2.0 ** -126)
    yb, wb = y.view(torch.int16), want.view(torch.int16)
    dropped_ok = (yb == 0)
    kept_ok = (yb == wb) | (torch.isnan(y) & torch.isnan(want)) | (sub & (y == 0)) | \
        ((want.float().abs() < 2.0 ** -126) & (y == 0))
    ok = torch.where(keep, kept_ok, dropped_ok)
    bad = (~ok).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} elements differ, first at {bad[0].tolist()}: x={x[tuple(bad[0])].item()} " \
                             f"y={y[tuple(bad[0])].item()} keep={keep[tuple(bad[0])].item()}"
    # the backward regenerates the mask from the stored state
    gy = rand(BDR_ROWS, BDR_N, seed=41)
    gx, st2 = ext.bias_dropout_residual(gy, None, None, p, 0, st)
    assert torch.equal(st2, st)
    gw = torch.where(keep, (gy.float() * scale).bfloat16(), torch.zeros_like(gy))
    assert torch.equal(gx.view(torch.int16), gw.view(torch.int16))


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_bias_dropout_residual_per_element(ext, p):
    x = rand(BDR_ROWS, BDR_N, seed=51, scale=3.0)
    bias = rand(BDR_N, seed=52)
    res = rand(BDR_ROWS, BDR_N, seed=53)
    y, st = ext.bias_dropout_residual(x, bias, res, p, 0, None)
    seed, off = stored_state(st)
    thr, scale = R.bdr_drop_threshold(p)
    keep = R.bdr_keep_mask(seed, off, x.numel(), thr, device=DEV).reshape(x.shape)
    xb = x.double() + bias.double()
    ref = torch.where(keep, xb * scale, torch.zeros_like(xb)) + res.double()
    # fp32 x + b, * scale and + residual each round at 2^-24 of their result (2^-23 per term with room); bf16 output
    dev = 2.0 ** -23 * (2 * xb.abs() * scale * keep + ref.abs())
    check(y, ref, BF * ref.abs() + (1 + BF) * dev + FLUSH, f"bias_dropout_residual p={p}")


# ---------------------------------------------------------------------------------------------------- rotary embedding
def rope_ref(x1, x2, c1, c2, s1, s2, backward):
    """fp64 rotate-half rotation of the pair (x1, x2) and its bound: two fp32 products and a sum, each rounding at 2^-24
    of a value below |x1 c| + |x2 s| (2^-22 in all), then the bf16 output rounding."""
    if not backward:
        y1, y2 = x1 * c1 - x2 * s1, x2 * c2 + x1 * s2
        m1, m2 = (x1 * c1).abs() + (x2 * s1).abs(), (x2 * c2).abs() + (x1 * s2).abs()
    else:
        y1, y2 = x1 * c1 + x2 * s2, x2 * c2 - x1 * s1
        m1, m2 = (x1 * c1).abs() + (x2 * s2).abs(), (x2 * c2).abs() + (x1 * s1).abs()
    ref = torch.cat([y1, y2], -1)
    m = torch.cat([m1, m2], -1)
    return ref, BF * ref.abs() + (1 + BF) * 2.0 ** -22 * m + FLUSH


def tables(P, D, base=10000.0):
    inv = 1.0 / base ** (torch.arange(0, D, 2, device=DEV, dtype=torch.float64) / D)
    ang = torch.arange(P, device=DEV, dtype=torch.float64)[:, None] * inv[None]
    emb = torch.cat([ang, ang], -1)
    return emb.cos().float(), emb.sin().float()


def rotate(x, cos, sin, backward):
    """x [..., S, D] against tables already indexed to [S, D]."""
    h = x.shape[-1] // 2
    xd, c, s = x.double(), cos.double(), sin.double()
    return rope_ref(xd[..., :h], xd[..., h:], c[..., :h], c[..., h:], s[..., :h], s[..., h:], backward)


@pytest.mark.parametrize("r", [1, 4])
@pytest.mark.parametrize("backward", [False, True])
def test_rope_qkv_per_element(ext, r, backward):
    B, S, G, D, off = 2, 45, 2, 128, 17
    qkv = rand(B, S, G, r + 2, D, seed=63 + r, scale=4.0)
    cos, sin = tables(S + off + 5, D)
    y = ext.rope_qkv(qkv, cos, sin, off, backward, False)
    c, s = cos[off:off + S][None, :, None, None], sin[off:off + S][None, :, None, None]
    ref, bnd = rotate(qkv[:, :, :, :r + 1], c, s, backward)
    check(y[:, :, :, :r + 1], ref, bnd, f"rope_qkv r={r} backward={backward}")
    assert torch.equal(y[:, :, :, r + 1], qkv[:, :, :, r + 1])


@pytest.mark.parametrize("r", [1, 4])
def test_kv_append_per_element(ext, r):
    B, Sq, G, D, C = 2, 5, 2, 64, 64
    qkv = rand(B, Sq, G, r + 2, D, seed=71 + r, scale=4.0)
    kc = torch.zeros(B, G, C, D, dtype=torch.bfloat16, device=DEV)
    vc = torch.zeros_like(kc)
    lens = torch.tensor([3, 40], dtype=torch.int32, device=DEV)
    cos, sin = tables(C, D)
    q = ext.kv_append(qkv, kc, vc, lens, cos, sin, True)
    for b in range(B):
        pos = int(lens[b])
        c, s = cos[pos:pos + Sq][:, None, None], sin[pos:pos + Sq][:, None, None]
        ref, bnd = rotate(qkv[b, :, :, :r + 1], c, s, False)       # [Sq, G, r + 1, D]
        check(q[b].reshape(Sq, G, r, D), ref[:, :, :r], bnd[:, :, :r], f"kv_append q r={r}")
        check(kc[b, :, pos:pos + Sq].transpose(0, 1), ref[:, :, r], bnd[:, :, r], f"kv_append k r={r}")
        assert torch.equal(vc[b, :, pos:pos + Sq].transpose(0, 1), qkv[b, :, :, r + 1])
        # rows outside [pos, pos + Sq) are untouched
        mask = torch.ones(C, dtype=torch.bool, device=DEV)
        mask[pos:pos + Sq] = False
        assert not kc[b, :, mask].any() and not vc[b, :, mask].any()
