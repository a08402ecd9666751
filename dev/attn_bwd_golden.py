"""Writes tests/golden/attn_bwd_parent.json: the SHA-256 of the flash backward's dq / dk / dv (and dbias) bytes for the
seeded cases of tests/attn_bwd_cases.py, as the current build computes them.  Run it on an H100 from the repository
root (`python dev/attn_bwd_golden.py [--out PATH]`) when the file has to be regenerated from a kernel that is known to
be right; tests/test_attention_bwd_schedule_gpu.py then holds every later kernel to those bytes."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from libai_b200.ops import load_ext  # noqa: E402
from tests import attn_bwd_cases as C  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=C.GOLDEN)
    args = ap.parse_args()
    ext = load_ext(required=True)
    res = {}
    for name in C.CASES:
        first = C.digests(C.run_backward(ext, name, "cuda:0"))
        second = C.digests(C.run_backward(ext, name, "cuda:0"))
        assert first == second, f"{name}: two runs differ"
        res[name] = first
    props = torch.cuda.get_device_properties(0)
    doc = {"device": props.name, "cases": res}
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(doc, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps({"cases": len(res), "out": args.out}))


if __name__ == "__main__":
    main()
