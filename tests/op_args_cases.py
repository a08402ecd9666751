"""Argument cases of the single-device native ops (``libai_b200/csrc/bindings.cpp``).

Every op gets one structurally valid argument set, built on a given device, and a list of mutations.  A mutation
changes one argument and names the ``"<op>: <arg>"`` fragment the op's error must carry.  The kinds are:

* ``dtype=<torch dtype name>``: the argument in another dtype;
* ``short``: one row fewer (dim 0); ``narrow``: one column fewer (last dim);
* ``rank``: one more leading dimension;
* ``noncontig``: same shape and values, every other element of a buffer twice as wide;
* ``misalign``: same shape and values, one element past a 16-byte boundary;
* ``device``: on another device (``other`` in ``mutate``);
* ``none``: left out (a missing companion, such as ``sin`` without ``cos``).

``outputs`` lists the shapes a valid call returns (``None`` for ops that return nothing).
"""
from dataclasses import dataclass, field

import torch

BF, F32, I32, I64, FP8 = torch.bfloat16, torch.float32, torch.int32, torch.int64, torch.float8_e4m3fn


@dataclass
class Case:
    op: str
    args: list                    # (name, value) pairs in the op's positional order
    mutations: list = field(default_factory=list)   # (name, kind, fragment)
    outputs: list = None
    label: str = ""

    @property
    def id(self):
        return self.op + (f"-{self.label}" if self.label else "")

    def values(self):
        return [v for _, v in self.args]


def _misalign(t):
    flat = torch.empty(t.numel() + 16, dtype=t.dtype, device=t.device)
    out = flat[1:1 + t.numel()].view(t.shape)
    out.copy_(t)
    return out


def mutate(t, kind, other):
    if kind.startswith("dtype="):
        return t.to(getattr(torch, kind[6:]))
    return {
        "short": lambda: t[:-1],
        "narrow": lambda: t[..., :-1].contiguous(),
        "rank": lambda: t.unsqueeze(0),
        "noncontig": lambda: torch.stack([t, t], -1)[..., 0],
        "misalign": lambda: _misalign(t),
        "device": lambda: t.to(other),
        "none": lambda: None,
    }[kind]()


def mutated(case, name, kind, other):
    return [mutate(v, kind, other) if n == name else v for n, v in case.args]


def _c(op, args, muts, outputs, label=""):
    """muts: "name:kind" or ("name:kind", fragment); the default fragment is "<op>: <name>" ("<op>: <name> must be
    on" for ``device``)."""
    out = []
    for m in muts:
        spec, frag = (m, None) if isinstance(m, str) else m
        name, kind = spec.split(":")
        if frag is None:
            frag = f"{op}: {name}" + (" must be on" if kind == "device" else "")
        out.append((name, kind, frag))
    return Case(op, list(args.items()), out, outputs, label)


def cases(dev):
    g = torch.Generator().manual_seed(0)

    def r(*shape, dtype=BF):
        return torch.randn(*shape, generator=g).to(dtype).to(dev)

    def z(*shape, dtype=I32):
        return torch.zeros(*shape, dtype=dtype, device=dev)

    def ar(n, dtype=I32):
        return torch.arange(n, dtype=dtype, device=dev)

    M, N, K = 128, 64, 64
    main_grad = torch.zeros(M, 2 * N, device=dev)
    qkv_att = r(1, 64, 2, 3, 64)                      # packed [b, s, a, 3, d]: q, k, v are strided views of it
    q, k, v = (qkv_att[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))
    o_att = torch.empty(1, 64, 2, 64, dtype=BF, device=dev).permute(0, 2, 1, 3)
    qkv_dec = r(2, 1, 4, 192)                         # decode q: a strided view of the packed projection
    fp8_cache = r(2, 4, 16, 64, dtype=FP8)
    L = [
        _c("gemm", dict(a=r(M, K), b=r(N, K), layout=0, bias=r(N), out=None, accumulate=False, out_dtype=BF),
           ["a:dtype=float32", "a:noncontig", "b:narrow", "b:device", "bias:short", "bias:dtype=float32",
            "bias:noncontig", "bias:device", "a:rank"], [(M, N)]),
        _c("gemm", dict(a=r(K, M), b=r(K, N), layout=2, bias=None, out=main_grad[:, 8:8 + N], accumulate=True,
                        out_dtype=F32),
           ["out:short", "out:dtype=float16", "out:device", "b:short"], [(M, N)], "wgrad-into-slice"),
        _c("gemm_tuned", dict(a=r(M, K), b=r(N, K), layout=0, bn=0, splits=1, fp32_out=False),
           ["a:dtype=float16", "b:device", "b:narrow", "a:rank"], [(M, N)]),
        _c("linear_fwd", dict(x=r(M, K), w=r(N, K), bias=r(N), act=1, need_pre=True),
           ["x:dtype=float32", "w:narrow", "w:device", "bias:short", "bias:noncontig", "bias:device"],
           [(M, N), (M, N)]),
        _c("linear_bias_residual", dict(x=r(M, K), w=r(N, K), bias=r(N), residual=r(M, N)),
           ["residual:short", "residual:noncontig", "residual:device", "bias:dtype=float32", "w:device"], [(M, N)]),
        _c("dgrad_actgrad", dict(gy=r(M, K), w=r(K, N), pre=r(M, N), act=1, bias_grad=z(N, dtype=F32)),
           ["gy:dtype=float32", "w:device", "pre:short", "pre:noncontig", "pre:device", "bias_grad:dtype=bfloat16",
            "bias_grad:device"], [(M, N)]),
        _c("act_bwd", dict(gy=r(M, N), pre=r(M, N), act=1),
           ["gy:dtype=float32", "gy:rank", "pre:short", "pre:misalign", "pre:device"], [(M, N)]),
        _c("colsum", dict(x=r(M, N), accum=z(N, dtype=F32)),
           ["x:noncontig", "accum:short", "accum:dtype=bfloat16", "accum:device"], [(0,)]),
        _c("quantize_e4m3", dict(x=r(M, K)), ["x:dtype=float32", "x:noncontig", "x:misalign"], [(M, K), (1,)]),
        _c("linear_fp8_fwd", dict(xq=r(M, K, dtype=FP8), wq=r(N, K, dtype=FP8), deq_x=r(1, dtype=F32).abs(),
                                  deq_w=r(1, dtype=F32).abs(), bias=r(N), act=0, need_pre=False, residual=r(M, N), bn=0),
           ["xq:dtype=bfloat16", "wq:narrow", "wq:device", "deq_x:rank", "deq_w:device", "bias:noncontig",
            "bias:device", "residual:short", "residual:device"], [(M, N), (0,)]),
        _c("linear_fp8w", dict(x=r(4, 256), w=r(128, 256, dtype=FP8), w_scale=r(128, dtype=F32).abs(), bias=r(128),
                               act=0),
           ["x:misalign", "w:misalign", "w:device", "w_scale:short", "w_scale:device", "bias:device"], [(4, 128)]),
        _c("dequant_e4m3_rows", dict(w=r(128, 256, dtype=FP8), w_scale=r(128, dtype=F32).abs()),
           ["w:noncontig", "w_scale:dtype=float64", "w_scale:device"], [(128, 256)]),
        _c("embedding_fwd", dict(ids=(ar(16, I64) * 5).view(2, 8), table=r(100, 64), vocab_start=0),
           ["ids:dtype=int32", "ids:noncontig", "ids:device", "table:misalign"], [(16, 64)]),
        _c("embedding_bwd", dict(ids=ar(16, I64) * 5, gy=r(16, 64), grad=z(100, 64, dtype=F32), vocab_start=0),
           ["gy:short", "ids:device", "grad:dtype=bfloat16", "grad:misalign", "grad:device"], None),
        _c("norm_fwd", dict(x=r(16, 256), gamma=r(256), beta=r(256), eps=1e-5, rms=False),
           ["x:dtype=float16", "x:noncontig", "gamma:short", ("gamma:device", "norm_fwd: gamma must be contiguous"),
            ("beta:device", "norm_fwd: beta must be contiguous")],
           [(16, 256), (16,), (16,)]),
        _c("norm_bwd", dict(gy=r(16, 256), x=r(16, 256), gamma=r(256), mean=r(16, dtype=F32),
                            rstd=r(16, dtype=F32).abs(), rms=False, has_bias=True, dgamma_accum=z(256, dtype=F32),
                            dbeta_accum=z(256, dtype=F32), gadd=r(16, 256)),
           ["gy:short", "gy:device", "mean:dtype=bfloat16", "rstd:short", "rstd:device", "dgamma_accum:short",
            "dgamma_accum:device", "dbeta_accum:none", "gadd:short", "gadd:device"], [(16, 256), (0,), (0,)]),
        _c("bias_act_fwd", dict(x=r(16, 64), bias=r(64), act=1),
           ["x:dtype=float32", "bias:dtype=float32", "bias:short", "bias:misalign", "bias:device"], [(16, 64)]),
        _c("bias_act_bwd", dict(gy=r(16, 64), x=r(16, 64), bias=r(64), act=1),
           ["gy:short", "gy:dtype=float32", "gy:device", "bias:device"], [(16, 64)]),
        _c("bias_residual_fwd", dict(x=r(16, 64), bias=r(64), res=r(16, 64)),
           ["bias:dtype=float32", "res:short", "res:noncontig", "res:device"], [(16, 64)]),
        _c("bias_dropout_residual", dict(x=r(16, 64), bias=r(64), res=r(16, 64), p=0.1, salt=0, rng_state=None),
           ["bias:dtype=float32", "bias:device", "res:short", "res:device", "x:misalign"], [(16, 64), (2,)]),
        _c("bias_dropout_residual", dict(x=r(16, 64), bias=None, res=None, p=0.1, salt=0, rng_state=z(2, dtype=I64)),
           ["rng_state:dtype=int32", "rng_state:short", "rng_state:device"], [(16, 64), (2,)], "replay"),
        _c("swiglu_fwd", dict(gate=r(16, 64), up=r(16, 64)),
           ["gate:noncontig", "up:short", "up:dtype=float32", "up:device"], [(16, 64)]),
        _c("swiglu_bwd", dict(gy=r(16, 64), gate=r(16, 64), up=r(16, 64)),
           ["gy:short", "gy:device", "up:dtype=float32"], [(16, 64), (16, 64)]),
        _c("swiglu_packed_fwd", dict(gu=r(16, 128)), ["gu:dtype=float32", "gu:misalign", "gu:noncontig"], [(16, 64)]),
        _c("swiglu_packed_bwd", dict(gy=r(16, 64), gu=r(16, 128)),
           ["gy:short", "gy:dtype=float32", "gy:device"], [(16, 128)]),
        _c("rope_qkv", dict(qkv=r(1, 16, 2, 192), cos=r(16, 64, dtype=F32), sin=r(16, 64, dtype=F32), pos_offset=0,
                            backward=False, inplace=False, positions=ar(16).view(1, 16)),
           ["qkv:dtype=float32", "qkv:noncontig", "positions:dtype=int64", "positions:narrow", "positions:device",
            ("cos:narrow", "rope_qkv: cos/sin"), ("sin:short", "rope_qkv: cos/sin"),
            ("sin:dtype=float64", "rope_qkv: cos/sin"), ("cos:device", "rope_qkv: cos/sin must be on")],
           [(1, 16, 2, 192)]),
        _c("glm_rotary_qkv", dict(mixed=r(1, 8, 512), heads=4, kv_heads=2, table=r(16, 16, 2, dtype=F32),
                                  pos_offset=0, position_ids=ar(8).view(1, 8), grouped=False),
           [("mixed:noncontig", "glm_rotary_qkv: contiguous"), "table:dtype=float64", "table:device",
            "position_ids:narrow", "position_ids:device"], [(1, 8, 4, 192)]),
        _c("glm_rotary_qkv_bwd", dict(grad=r(1, 8, 4, 192), heads=4, kv_heads=2, table=r(16, 16, 2, dtype=F32),
                                      pos_offset=0, position_ids=ar(8).view(1, 8)),
           [("grad:noncontig", "glm_rotary_qkv_bwd: contiguous"), "table:device", "position_ids:narrow"],
           [(1, 8, 512)]),
        _c("ce_stats", dict(logits=r(16, 100), labels=ar(16, I64), vocab_start=0),
           ["logits:dtype=float16", "logits:noncontig", "labels:short", "labels:dtype=int32", "labels:device"],
           [(16,), (16,), (16,)]),
        _c("ce_bwd", dict(logits=r(16, 100), labels=ar(16, I64), lse=r(16, dtype=F32), gloss=r(16, dtype=F32),
                          vocab_start=0),
           ["labels:noncontig", "lse:short", "lse:dtype=bfloat16", "gloss:device"], [(16, 100)]),
        _c("fused_adamw", dict(master=r(1024, dtype=F32), grad=r(1024, dtype=F32), m=z(1024, dtype=F32),
                               v=z(1024, dtype=F32), lp_out=z(1024, dtype=BF), scale=r(1, dtype=F32).abs(), lr=1e-3,
                               b1=0.9, b2=0.999, eps=1e-8, wd=0.0, bc1=0.1, bc2=0.001, decoupled=True),
           ["grad:short", "m:device", "v:misalign", "lp_out:dtype=float32", "lp_out:misalign", "lp_out:device",
            "scale:rank", "scale:device"], None),
        _c("sqnorm", dict(x=r(1000, dtype=F32)), ["x:dtype=bfloat16", "x:misalign", "x:noncontig"], [(1,)]),
        _c("attn_fwd", dict(q=q, k=k, v=v, causal=True, scale=0.125, kv_lens=torch.full((1,), 64, dtype=I32, device=dev),
                            bias=None, alibi_slopes=r(2, dtype=F32), p_drop=0.0, salt=0, kv_start=z(1), doc_start=None),
           ["q:dtype=float32", "k:dtype=float32", "v:device", "kv_lens:dtype=int64", "kv_lens:device", "kv_start:rank",
            "alibi_slopes:short", "alibi_slopes:device"], [(1, 2, 64, 64), (1, 2, 64), (0,)]),
        _c("attn_fwd", dict(q=q, k=k, v=v, causal=True, scale=0.125, kv_lens=None, bias=r(1, 2, 64, 64),
                            alibi_slopes=None, p_drop=0.1, salt=0, kv_start=None, doc_start=None),
           ["bias:narrow", "bias:dtype=float32", "bias:device", "k:short"], [(1, 2, 64, 64), (1, 2, 64), (2,)],
           "bias"),
        _c("attn_fwd", dict(q=q, k=k, v=v, causal=True, scale=0.125, kv_lens=None, bias=None, alibi_slopes=None,
                            p_drop=0.0, salt=0, kv_start=None, doc_start=z(1, 64)),
           ["doc_start:narrow", "doc_start:dtype=int64", "doc_start:device"], [(1, 2, 64, 64), (1, 2, 64), (0,)],
           "doc_start"),
        _c("attn_bwd", dict(dout=r(1, 2, 64, 64), q=q, k=k, v=v, o=o_att, lse=z(1, 2, 64, dtype=F32), causal=True,
                            scale=0.125, kv_lens=None, bias=r(1, 2, 64, 64), alibi_slopes=None,
                            dbias=z(1, 2, 64, 64, dtype=F32), p_drop=0.1, rng_state=z(2, dtype=I64), kv_start=None,
                            doc_start=None),
           ["dout:narrow", "dout:device", "o:narrow", "o:device", "lse:short", "lse:device", "rng_state:dtype=int32",
            "rng_state:device", "dbias:dtype=bfloat16", "dbias:device", "bias:device", "q:dtype=float16"],
           [(1, 2, 64, 64), (1, 2, 64, 64), (1, 2, 64, 64), (1, 64, 2, 3, 64)]),
        _c("kv_append", dict(qkv=r(2, 1, 4, 192), k_cache=r(2, 4, 16, 64), v_cache=r(2, 4, 16, 64),
                             cache_seqlens=z(2), cos=r(16, 64, dtype=F32), sin=r(16, 64, dtype=F32), write_q=True),
           ["qkv:noncontig", "k_cache:dtype=float32", "k_cache:misalign", "v_cache:short", "v_cache:device",
            "cache_seqlens:dtype=int64", "cache_seqlens:device", ("cos:device", "kv_append: cos/sin must be on"),
            ("sin:none", "kv_append: cos and sin")], [(2, 1, 4, 64)]),
        _c("kv_append_fp8", dict(qkv=r(2, 1, 4, 192), k_cache=fp8_cache.clone(), v_cache=fp8_cache.clone(),
                                 k_scale=z(2, 4, 16, dtype=F32), v_scale=z(2, 4, 16, dtype=F32), cache_seqlens=z(2),
                                 cos=r(16, 64, dtype=F32), sin=r(16, 64, dtype=F32), write_q=True),
           ["k_cache:dtype=bfloat16", "v_cache:device", "k_scale:short", "k_scale:misalign", "v_scale:device",
            "cache_seqlens:device", ("cos:none", "kv_append_fp8: cos and sin")], [(2, 1, 4, 64)]),
        _c("decode_attn", dict(q=qkv_dec[..., :64], k_cache=r(2, 4, 16, 64), v_cache=r(2, 4, 16, 64),
                               cache_seqlens=torch.full((2,), 4, dtype=I32, device=dev), kv_start=z(2), scale=0.125,
                               splits=0, alibi_slopes=r(4, dtype=F32), rel_bias=None, causal=True, k_scale=None,
                               v_scale=None),
           ["q:narrow", "k_cache:device", "v_cache:dtype=float32", "cache_seqlens:device", "kv_start:dtype=int64",
            "alibi_slopes:short", "alibi_slopes:device"], [(2, 1, 4, 64)]),
        _c("decode_attn", dict(q=qkv_dec[..., :64], k_cache=fp8_cache, v_cache=fp8_cache,
                               cache_seqlens=torch.full((2,), 4, dtype=I32, device=dev), kv_start=z(2), scale=0.125,
                               splits=0, alibi_slopes=None, rel_bias=r(4, 8, dtype=F32), causal=True,
                               k_scale=r(2, 4, 16, dtype=F32).abs(), v_scale=r(2, 4, 16, dtype=F32).abs()),
           ["k_scale:short", "v_scale:device", ("k_scale:none", "decode_attn: an FP8 cache"),
            ("rel_bias:device", "decode_attn: rel_bias")], [(2, 1, 4, 64)], "fp8-rel_bias"),
        _c("window_attn_fwd", dict(qkv=r(1, 64, 192), H=8, W=8, window=4, shift=2, heads=2, scale=0.17,
                                   table=r(49, 2, dtype=F32), tau=r(2, dtype=F32).abs()),
           ["qkv:misalign", "table:short", "table:device", "tau:dtype=bfloat16", "tau:device"],
           [(1, 64, 64), (4, 2, 16)]),
        _c("window_attn_bwd", dict(dout=r(1, 64, 64), qkv=r(1, 64, 192), lse=z(4, 2, 16, dtype=F32), H=8, W=8,
                                   window=4, shift=2, heads=2, scale=0.17, table=r(49, 2, dtype=F32),
                                   tau=r(2, dtype=F32).abs()),
           ["dout:narrow", "dout:device", "lse:short", "lse:device"], [(1, 64, 192), (49, 2), (2,)]),
    ]
    return L

