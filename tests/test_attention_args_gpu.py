"""The flash-attention op wrappers: the forward against the bytes it produced before its arguments were gathered into
one lb::AttnArgs (tests/golden/attn_fwd_parent.json, see tests/attn_bwd_cases.py), and the inputs that both
directions reject before any kernel reads them."""
import json
import os

import pytest
import torch

from tests import attn_bwd_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(REPO, C.FWD_GOLDEN)) as f:
        return json.load(f)["cases"]


def test_golden_file_covers_every_case(golden):
    assert set(golden) == set(C.FWD_CASES)


@pytest.mark.parametrize("name", sorted(C.FWD_CASES))
def test_forward_matches_parent_bit_for_bit(ext, golden, name):
    assert C.digests(C.run_forward(ext, name, DEV)) == golden[name]


B, A, S, D = 2, 4, 64, 64


def _qkv():
    g = torch.Generator(device=DEV).manual_seed(0)
    return [torch.randn(B, A, S, D, generator=g, device=DEV).bfloat16() for _ in range(3)]


def _fwd(ext, q, k, v, alibi=None, p=0.0):
    return ext.attn_fwd(q, k, v, True, D ** -0.5, None, None, alibi, p, 0, None)


def _bwd(ext, do, q, k, v, o, lse, alibi=None, p=0.0, rng_state=None):
    return ext.attn_bwd(do, q, k, v, o, lse, True, D ** -0.5, None, None, alibi, None, p, rng_state, None)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("which", [0, 1, 2])
def test_rejects_non_bf16_qkv(ext, dtype, which):
    t = _qkv()
    t[which] = t[which].to(dtype)
    with pytest.raises(RuntimeError, match="bf16"):
        _fwd(ext, *t)
    q, k, v = _qkv()
    o, lse, _ = _fwd(ext, q, k, v)
    t = [q, k, v]
    t[which] = t[which].to(dtype)
    with pytest.raises(RuntimeError, match="bf16"):
        _bwd(ext, torch.ones_like(o), *t, o, lse)


def test_rejects_k_on_the_cpu(ext):
    q, k, v = _qkv()
    with pytest.raises(RuntimeError, match="device"):
        _fwd(ext, q, k.cpu(), v)
    o, lse, _ = _fwd(ext, q, k, v)
    with pytest.raises(RuntimeError, match="device"):
        _bwd(ext, torch.ones_like(o), q, k.cpu(), v, o, lse)


@pytest.mark.parametrize("bad", ["fp16", "short", "cpu"])
def test_backward_rejects_bad_alibi_slopes(ext, bad):
    q, k, v = _qkv()
    slopes = torch.tensor([2.0 ** (-8 * (h + 1) / A) for h in range(A)], device=DEV)
    o, lse, _ = _fwd(ext, q, k, v, alibi=slopes)
    wrong = {"fp16": slopes.half(), "short": slopes[:-1], "cpu": slopes.cpu()}[bad]
    with pytest.raises(RuntimeError, match="alibi_slopes"):
        _bwd(ext, torch.ones_like(o), q, k, v, o, lse, alibi=wrong)


def test_backward_with_dropout_needs_rng_state(ext):
    q, k, v = _qkv()
    o, lse, rng_state = _fwd(ext, q, k, v, p=0.1)
    do = torch.ones_like(o)
    for wrong in (None, rng_state[:1], rng_state.int(), rng_state.cpu()):
        with pytest.raises(RuntimeError, match="rng_state"):
            _bwd(ext, do, q, k, v, o, lse, p=0.1, rng_state=wrong)


@pytest.mark.parametrize("bad", ["o", "lse", "dout"])
def test_backward_rejects_misshaped_forward_tensors(ext, bad):
    q, k, v = _qkv()
    o, lse, _ = _fwd(ext, q, k, v)
    do = torch.ones_like(o)
    if bad == "o":
        o = o[:, :, : S // 2]
    elif bad == "lse":
        lse = lse[:, :, : S // 2].contiguous()
    else:
        do = do[:, : A // 2]
    with pytest.raises(RuntimeError, match=f"attn_bwd: {bad} must be"):
        _bwd(ext, do, q, k, v, o, lse)
