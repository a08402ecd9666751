"""The outputs of the rotate-half rotary kernels on fixed seeded inputs, for comparing two builds bit for bit.

    python dev/rotary_bits.py --out DIR [--lib path/to/_C.so]
    python dev/rotary_bits.py --compare DIR_A DIR_B

rope_qkv (forward and backward, at s + pos_offset and at per-token positions, out of place and in place), kv_append
(with and without tables, q returned) and kv_append_fp8 (the same) at head dims 64 and 128, in the per-head
[q|k|v] and grouped layouts.  ``--lib`` loads another build of the extension (one build per process: both register
the same operators).  ``--compare`` exits non-zero unless every tensor of the two runs is torch.equal.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DEV = "cuda"


def rand(*shape, seed, scale=4.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).bfloat16()


def tables(P, D):
    inv_freq = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    emb = torch.outer(torch.arange(P, dtype=torch.float32), inv_freq).repeat(1, 2)
    return emb.cos().to(DEV), emb.sin().to(DEV)


def outputs(ext):
    out = {}
    for D in (64, 128):
        for r in (1, 4):
            B, S, G, off = 3, 67, 2, 11
            shape = (B, S, G, 3 * D) if r == 1 else (B, S, G, r + 2, D)
            qkv = rand(*shape, seed=D + r)
            cos, sin = tables(S + off + 5, D)
            pos = torch.randint(-3, S + off + 8, (B, S), device=DEV, dtype=torch.int32,
                                generator=torch.Generator(device=DEV).manual_seed(D * r))   # clamped by the kernel
            for bwd in (False, True):
                tag = f"D{D}_r{r}_{'bwd' if bwd else 'fwd'}"
                out[f"rope_qkv_offset_{tag}"] = ext.rope_qkv(qkv, cos, sin, off, bwd, False)
                out[f"rope_qkv_positions_{tag}"] = ext.rope_qkv(qkv, cos, sin, off, bwd, False, pos)
                out[f"rope_qkv_inplace_{tag}"] = ext.rope_qkv(qkv.clone(), cos, sin, off, bwd, True)
            Sq, C = 5, 64
            step = rand(B, Sq, G, 3 * D, seed=7 + D + r) if r == 1 else rand(B, Sq, G, r + 2, D, seed=7 + D + r)
            lens = torch.tensor([0, 17, C - Sq], dtype=torch.int32, device=DEV)
            cos, sin = tables(C, D)
            for rot, (c, s) in (("rope", (cos, sin)), ("plain", (None, None))):
                tag = f"D{D}_r{r}_{rot}"
                kc = torch.zeros(B, G, C, D, dtype=torch.bfloat16, device=DEV)
                vc = torch.zeros_like(kc)
                out[f"kv_append_q_{tag}"] = ext.kv_append(step, kc, vc, lens, c, s, True)
                out[f"kv_append_k_{tag}"], out[f"kv_append_v_{tag}"] = kc, vc
                k8 = torch.zeros(B, G, C, D, dtype=torch.float8_e4m3fn, device=DEV)
                v8 = torch.zeros_like(k8)
                ks = torch.zeros(B, G, C, dtype=torch.float32, device=DEV)
                vs = torch.zeros_like(ks)
                out[f"kv_append_fp8_q_{tag}"] = ext.kv_append_fp8(step, k8, v8, ks, vs, lens, c, s, True)
                out[f"kv_append_fp8_k_{tag}"] = k8.view(torch.uint8)
                out[f"kv_append_fp8_v_{tag}"] = v8.view(torch.uint8)
                out[f"kv_append_fp8_kscale_{tag}"], out[f"kv_append_fp8_vscale_{tag}"] = ks, vs
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--lib", default="")
    ap.add_argument("--compare", nargs=2, metavar="DIR")
    a = ap.parse_args()
    if a.compare:
        x, y = (torch.load(os.path.join(d, "rotary_bits.pt")) for d in a.compare)
        bad = sorted(set(x) ^ set(y)) + [k for k in sorted(set(x) & set(y)) if not torch.equal(x[k], y[k])]
        print(f"{len(x)} / {len(y)} tensors, {len(bad)} differ{': ' + ', '.join(bad) if bad else ''}")
        sys.exit(1 if bad else 0)
    if a.lib:
        torch.ops.load_library(a.lib)
        ext = torch.ops.libai_b200
    else:
        from libai_b200 import ops

        ext = ops.load_ext(required=True)
    os.makedirs(a.out, exist_ok=True)
    res = outputs(ext)
    torch.save(res, os.path.join(a.out, "rotary_bits.pt"))
    print(f"{len(res)} tensors -> {a.out}")


if __name__ == "__main__":
    main()
