"""Prefix-LM flash attention (prefix_lens, the PREFIX kernel instances) on the H100 against fp64, element by element
(tests/attention_ref.py states the bounds): head dims 64 and 128, MHA and GQA, square and rectangular, with key
windows and dropout, at prefixes on both sides of the 64- and 128-key tile edges.  Then the two bit-identities (a
prefix of 0 is the causal kernel, a prefix >= Sk the non-causal one), run-to-run determinism, CUDA-graph replay after
the prefix changes on the device, and every rejection of the bindings."""
import pytest
import torch

from libai_b200.ops import functional as OF
from tests import attention_ref as R
from tests.dense_ref import check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def rand(*shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, device=DEV, generator=g).bfloat16()


def i32(xs):
    return torch.tensor(xs, dtype=torch.int32, device=DEV)


def run(ext, q, k, v, do, pre, *, kv_start=None, kv_lens=None, p=0.0, causal=True, with_prefix=True):
    extra = {"prefix_lens": pre} if with_prefix else {}
    o, lse, st = ext.attn_fwd(q, k, v, causal, q.shape[-1] ** -0.5, kv_lens, None, None, p, 0, kv_start, **extra)
    dq, dk, dv, _ = ext.attn_bwd(do, q, k, v, o, lse, causal, q.shape[-1] ** -0.5, kv_lens, None, None, None, p,
                                 st if p > 0 else None, kv_start, **extra)
    return dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv), st


def prefixes(sk):
    return [x for x in (0, 1, 63, 64, 65, 127, 128, sk // 4, sk // 2, sk, sk + 9)]


SHAPES = [(63, 63), (130, 130), (200, 200), (77, 203), (1, 300), (256, 256)]
HEADS = [(4, 4), (4, 1), (8, 2)]


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("si", range(len(SHAPES)))
@pytest.mark.parametrize("drop", [False, True])
def test_prefix_per_element(ext, D, si, drop):
    Sq, Sk = SHAPES[si]
    A, G = HEADS[(si + (D == 128)) % 3]
    B = 2
    seed = 100 * si + D + drop
    q, k, v, do = rand(B, A, Sq, D, seed=seed), rand(B, G, Sk, D, seed=seed + 1), rand(B, G, Sk, D, seed=seed + 2), \
        rand(B, A, Sq, D, seed=seed + 3)
    pres = prefixes(Sk)
    for n, p0 in enumerate(pres):
        pre = i32([p0, pres[(n + 5) % len(pres)]])
        # every other prefix meets a key window: the second sample left padded and shortened
        kv_start, kv_lens = (i32([0, min(5, Sk - 1)]), i32([Sk, max(1, Sk - 3)])) if n % 2 else (None, None)
        p = 0.2 if drop else 0.0
        got, st = run(ext, q, k, v, do, pre, kv_start=kv_start, kv_lens=kv_lens, p=p)
        keep, ik = None, 1.0
        if drop:
            seed_s, off = (int(x) & 0xFFFFFFFFFFFFFFFF for x in st.cpu().tolist())
            thr, ik = R.attn_drop_threshold(p)
            keep = R.attn_keep_mask(seed_s, off, B, A, Sq, Sk, thr, device=DEV)
        vis = OF.visible_keys(Sq, Sk, causal=True, kv_start=kv_start, kv_lens=kv_lens, prefix_lens=pre, device=DEV)
        what = f"D{D} {Sq}x{Sk} A{A} G{G} prefix {pre.tolist()} window {n % 2} drop {drop}"
        (o, ob), (lse, lseb) = R.attention_fwd_ref(q, k, v, scale=D ** -0.5, vis=vis, keep=keep, inv_keep=ik, tile=128)
        check(got["o"], o, ob, what + " o")
        check(got["lse"], lse, lseb, what + " lse")
        ref = R.attention_bwd_ref(q, k, v, do, got["o"], got["lse"], scale=D ** -0.5, vis=vis, keep=keep, inv_keep=ik)
        R.check_all(got, ref, what)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("Sq,Sk", [(200, 200), (77, 203), (256, 256)])
def test_prefix_bit_identities(ext, D, drop, Sq, Sk):
    """prefix 0 == the causal kernel and prefix >= Sk == the non-causal kernel, outputs and gradients bit for bit
    (with dropout, under the same generator state)."""
    A, G, B = 4, 2, 2
    q, k, v, do = rand(B, A, Sq, D, seed=1), rand(B, G, Sk, D, seed=2), rand(B, G, Sk, D, seed=3), rand(B, A, Sq, D, seed=4)
    p = 0.1 if drop else 0.0
    kv_start, kv_lens = i32([0, 3]), i32([Sk, Sk - 2])
    for pre, causal in ((i32([0, 0]), True), (i32([Sk, Sk + 40]), False)):
        state = torch.cuda.get_rng_state(DEV)
        got, _ = run(ext, q, k, v, do, pre, kv_start=kv_start, kv_lens=kv_lens, p=p)
        torch.cuda.set_rng_state(state, DEV)
        want, _ = run(ext, q, k, v, do, None, kv_start=kv_start, kv_lens=kv_lens, p=p, causal=causal, with_prefix=False)
        for name in got:
            assert torch.equal(got[name], want[name]), (name, causal)


def test_prefix_deterministic(ext):
    B, A, G, S, D = 2, 8, 2, 700, 64
    q, k, v, do = rand(B, A, S, D, seed=5), rand(B, G, S, D, seed=6), rand(B, G, S, D, seed=7), rand(B, A, S, D, seed=8)
    pre = i32([130, 450])
    a, _ = run(ext, q, k, v, do, pre)
    b, _ = run(ext, q, k, v, do, pre)
    for name in a:
        assert torch.equal(a[name], b[name]), name


def test_prefix_cuda_graph_replay_reads_the_device_prefix(ext):
    B, A, S, D = 2, 4, 300, 64
    q, k, v, do = rand(B, A, S, D, seed=9), rand(B, A, S, D, seed=10), rand(B, A, S, D, seed=11), rand(B, A, S, D, seed=12)
    pre = i32([10, 20])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(ext, q, k, v, do, pre)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got, _ = run(ext, q, k, v, do, pre)
    for val in ([10, 20], [0, 299], [150, 64]):
        pre.copy_(i32(val))
        graph.replay()
        torch.cuda.synchronize()
        want, _ = run(ext, q, k, v, do, i32(val))
        for name in want:
            assert torch.equal(got[name], want[name]), (val, name)


def test_prefix_native_path_runs_the_kernels():
    """OF.attention with prefix_lens runs _FlashAttnFn (no reference math) and matches the dense reference."""
    from libai_b200 import ops

    B, A, S, D = 2, 4, 100, 64
    q, k, v = (rand(B, A, S, D, seed=s).requires_grad_() for s in (13, 14, 15))
    pre = i32([30, 70])
    ops.reset_launch_count()
    o = OF.attention(q, k, v, causal=True, prefix_lens=pre)
    assert ops.launch_count() == 1 and o.grad_fn.name().startswith("_FlashAttnFn")
    vis = OF.visible_keys(S, S, causal=True, prefix_lens=pre, device=DEV)
    ref = OF.attention_ref(q.float(), k.float(), v.float(), causal=False, scale=D ** -0.5, mask=vis)
    assert float((o.detach().float() - ref.detach()).abs().max()) < 2e-2


def test_prefix_binding_rejections(ext):
    B, A, S, D = 2, 4, 64, 64
    q, k, v = rand(B, A, S, D, seed=1), rand(B, A, S, D, seed=2), rand(B, A, S, D, seed=3)
    pre = i32([3, 4])
    allowed = "supported for causal attention, with kv_lens, kv_start, grouped-query heads and dropout, without bias"

    def fwd(*, causal=True, bias=None, alibi=None, doc=None, prefix=pre):
        return ext.attn_fwd(q, k, v, causal, 0.125, None, bias, alibi, 0.0, 0, None, doc, prefix)

    with pytest.raises(RuntimeError, match=allowed):
        fwd(causal=False)
    with pytest.raises(RuntimeError, match=allowed):
        fwd(bias=torch.zeros(1, 1, S, S, dtype=torch.bfloat16, device=DEV))
    with pytest.raises(RuntimeError, match=allowed):
        fwd(alibi=torch.ones(A, device=DEV))
    with pytest.raises(RuntimeError):
        fwd(doc=torch.zeros(B, S, dtype=torch.int32, device=DEV))
    with pytest.raises(RuntimeError, match="attn_fwd: prefix_lens"):
        fwd(prefix=pre.long())
    with pytest.raises(RuntimeError, match="attn_fwd: prefix_lens"):
        fwd(prefix=i32([3, 4, 5]))
    with pytest.raises(RuntimeError, match="attn_fwd: prefix_lens"):
        fwd(prefix=pre.cpu())
    with pytest.raises(RuntimeError, match="attn_fwd: prefix_lens"):
        fwd(prefix=i32([3, 4, 5, 6])[::2])
    o, lse, _ = fwd()
    with pytest.raises(RuntimeError, match=allowed):
        ext.attn_bwd(q, q, k, v, o, lse, False, 0.125, None, None, None, None, 0.0, None, None, None, pre)
    with pytest.raises(RuntimeError, match="attn_bwd: prefix_lens"):
        ext.attn_bwd(q, q, k, v, o, lse, True, 0.125, None, None, None, None, 0.0, None, None, None, pre.float())
