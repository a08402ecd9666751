"""Same-box comparator: GPT-2 pre-training step in plain PyTorch, the way a competent user would write it today.

NOT the reference (that needs OneFlow) and nothing from ``libai_b200`` — only stock PyTorch pieces:
``F.scaled_dot_product_attention`` (flash / cuDNN backend picked by PyTorch), ``F.layer_norm``, ``F.gelu``, cuBLAS
matmuls under bf16 autocast, ``torch.optim.AdamW(fused=True)`` on fp32 parameters, ``DistributedDataParallel`` over
NCCL (bucketed all-reduce overlapped with backward) when world > 1.  ``bench.py`` runs it in the same process launch
as the native arm and prints its number as ``ref_same_box``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn


class Block(nn.Module):
    def __init__(self, h: int, heads: int):
        super().__init__()
        self.ln1 = nn.LayerNorm(h)
        self.qkv = nn.Linear(h, 3 * h)
        self.proj = nn.Linear(h, h)
        self.ln2 = nn.LayerNorm(h)
        self.fc = nn.Linear(h, 4 * h)
        self.out = nn.Linear(4 * h, h)
        self.heads = heads

    def forward(self, x):
        b, s, h = x.shape
        q, k, v = self.qkv(self.ln1(x)).view(b, s, 3, self.heads, h // self.heads).permute(2, 0, 3, 1, 4)
        a = F.scaled_dot_product_attention(q, k, v, is_causal=True)
        x = x + self.proj(a.transpose(1, 2).reshape(b, s, h))
        return x + self.out(F.gelu(self.fc(self.ln2(x))))


class GPT2(nn.Module):
    def __init__(self, layers=24, hidden=1024, heads=16, vocab=50304, max_seq=1024):
        super().__init__()
        self.wte = nn.Embedding(vocab, hidden)
        self.wpe = nn.Embedding(max_seq, hidden)
        self.blocks = nn.ModuleList(Block(hidden, heads) for _ in range(layers))
        self.ln_f = nn.LayerNorm(hidden)
        for m in self.modules():
            if isinstance(m, (nn.Linear, nn.Embedding)):
                nn.init.normal_(m.weight, std=0.02)
        for blk in self.blocks:
            for lin in (blk.proj, blk.out):
                nn.init.normal_(lin.weight, std=0.02 / math.sqrt(2 * layers))

    def forward(self, ids, labels):
        b, s = ids.shape
        x = self.wte(ids) + self.wpe(torch.arange(s, device=ids.device))
        for blk in self.blocks:
            x = blk(x)
        logits = F.linear(self.ln_f(x), self.wte.weight)          # tied LM head
        return F.cross_entropy(logits.float().view(b * s, -1), labels.reshape(-1))


def build(layers, hidden, heads, vocab, seq, device, world, local_rank):
    model = GPT2(layers, hidden, heads, vocab, seq).to(device)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01, fused=True)
    if world > 1:
        model = nn.parallel.DistributedDataParallel(model, device_ids=[local_rank], gradient_as_bucket_view=True,
                                                    static_graph=True)
    return model, opt


def train_step(model, opt, ids, labels, clip: float = 1.0):
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = model(ids, labels)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), clip, foreach=True)
    opt.step()
    return loss.detach()
