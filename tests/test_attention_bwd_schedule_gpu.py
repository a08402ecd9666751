"""The flash backward against the bytes it produced before the warp-specialised schedule (tests/golden/
attn_bwd_parent.json, see tests/attn_bwd_cases.py): every case, the GPT-2 training shape included, must give the same
dq / dk / dv (and dbias) bits; repeated runs and CUDA-graph replays must agree bit for bit."""
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
    with open(os.path.join(REPO, C.GOLDEN)) as f:
        return json.load(f)["cases"]


def test_golden_file_covers_every_case(golden):
    assert set(golden) == set(C.CASES)


@pytest.mark.parametrize("name", sorted(C.CASES))
def test_matches_parent_bit_for_bit(ext, golden, name):
    assert C.digests(C.run_backward(ext, name, DEV)) == golden[name]


@pytest.mark.parametrize("name", ["d64_gqa4_causal_s203", "d128_mha_causal_rect_203x77", "d64_doc_start_s1000"])
def test_two_runs_identical(ext, name):
    a, b = C.run_backward(ext, name, DEV), C.run_backward(ext, name, DEV)
    for n in a:
        assert torch.equal(a[n].view(torch.int16) if a[n].dtype == torch.bfloat16 else a[n],
                           b[n].view(torch.int16) if b[n].dtype == torch.bfloat16 else b[n]), n


@pytest.mark.parametrize("name", ["d64_causal_s203_alibi", "d128_gqa4_causal_s1000"])
def test_cuda_graph_replay_matches_eager(ext, golden, name):
    q, k, v, do, causal, scale, kw = C.make_inputs(name, DEV)
    o, lse, _ = ext.attn_fwd(q, k, v, causal, scale, kw["kv_lens"], kw["bias"], kw["alibi"], 0.0, 0, kw["kv_start"],
                             kw["doc_start"])

    def bwd():
        return ext.attn_bwd(do, q, k, v, o, lse, causal, scale, kw["kv_lens"], kw["bias"], kw["alibi"], None, 0.0,
                            None, kw["kv_start"], kw["doc_start"])[:3]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        bwd()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = bwd()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert C.digests(dict(zip(("dq", "dk", "dv"), out))) == golden[name]
    del graph
