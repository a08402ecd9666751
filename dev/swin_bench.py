"""Shifted-window attention of the Swin and SwinV2 recipes on one GPU: native kernel against the PyTorch window path.

    python dev/swin_bench.py [--out output/swin_bench.json] [--iters 10] [--steps 10] [--rounds 3]

Per op (``ops`` rows): the attention half of one block at the recipe layer shapes, batch 128, bf16, forward + backward.
  * ``native``: qkv Linear -> ``OF.window_attention`` -> proj Linear on the image-ordered tokens (``forward_image``);
  * ``window``: roll -> window_partition -> ``WindowAttention`` (qkv, scores, softmax, proj) -> window_reverse -> roll,
    the path every Swin block took before.
  Both arms include the qkv and proj GEMMs.  Medians of CUDA-event times with the arms alternated, the peak memory
  allocated during one forward + backward, and the kernels alone: ``window_attn_fwd`` and ``window_attn_bwd`` timed
  on their own, with the bytes they must move (qkv and O forward; qkv, dO and dqkv backward, plus the lse) over
  their time against the H100 SXM's 3.35 TB/s.  Stages whose map is no larger than the window run the whole map as one
  window without a shift, as the models do; the others use the shifted (odd) block.
Per step (``steps`` rows): training-step images/s of Swin-T 224 and SwinV2-T 256 at batch 128 (bf16 parameters, AdamW,
seeded synthetic images), native against the window path forced by patching ``OF.window_attention_supported``; the
two arms alternate ``--rounds`` times, ``--steps`` timed steps each after three warm-up steps.

The card name, power limit and SM clock are printed with the figures and stored in the JSON output.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from dev.decode_bench import gpu_info  # noqa: E402
from libai_b200 import ops  # noqa: E402
from libai_b200.layers._param import param_defaults  # noqa: E402
from libai_b200.models import swin_transformer as v1  # noqa: E402
from libai_b200.models import swin_transformer_v2 as v2  # noqa: E402
from libai_b200.ops import functional as OF  # noqa: E402

HBM_TBS = 3.35

# name, version, image, window, embed, heads per stage
MODELS = [
    ("swin-t 224/ws7", 1, 224, 7, 96, [3, 6, 12, 24]),
    ("swin-t-c24 256/ws8", 1, 256, 8, 96, [4, 8, 16, 32]),
    ("swinv2-t 256/ws8", 2, 256, 8, 96, [3, 6, 12, 24]),
    ("swinv2-t 256/ws16", 2, 256, 16, 96, [3, 6, 12, 24]),
    ("swin-b 384/ws12", 1, 384, 12, 128, [4, 8, 16, 32]),
]


def _block(version, dim, res, heads, window):
    mod = v1 if version == 1 else v2
    with param_defaults(dtype=torch.bfloat16, device="cuda", seed=0):
        blk = mod.SwinTransformerBlock(dim=dim, input_resolution=(res, res), num_heads=heads, window_size=window,
                                       shift_size=window // 2)
    return blk.to(device="cuda", dtype=torch.bfloat16)   # buffers


def _window_path(blk, x):
    """The PyTorch window path of a block's attention half (the same for v1 and v2)."""
    H, W = blk.input_resolution
    B, L, C = x.shape
    ws, s = blk.window_size, blk.shift_size
    x = x.view(B, H, W, C)
    if s > 0:
        x = torch.roll(x, shifts=(-s, -s), dims=(1, 2))
    win = v1.window_partition(x, ws).view(-1, ws * ws, C)
    win = blk.attn(win, blk._attn_mask(x.device)).view(-1, ws, ws, C)
    x = v1.window_reverse(win, ws, H, W)
    if s > 0:
        x = torch.roll(x, shifts=(s, s), dims=(1, 2))
    return x.reshape(B, H * W, C)


def _peak_gib(run):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    run()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def _time_alternated(arms, iters):
    for run in arms.values():
        run()
    times = {name: [] for name in arms}
    for _ in range(iters):
        for name, run in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            run()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    return {name: statistics.median(t) for name, t in times.items()}


def op_rows(iters, B):
    ext = ops.load_ext(required=True)
    rows = []
    for name, version, img, window, embed, heads in MODELS:
        for stage, h in enumerate(heads):
            res, dim = img // 4 // 2 ** stage, embed * 2 ** stage
            blk = _block(version, dim, res, h, window)
            ws, s, d = blk.window_size, blk.shift_size, dim // h
            assert OF.window_attention_supported(torch.empty(1, device="cuda", dtype=torch.bfloat16), H=res, W=res,
                                                 window=ws, shift=s, head_dim=d)
            g = torch.Generator(device="cuda").manual_seed(stage)
            x = torch.randn(B, res * res, dim, device="cuda", generator=g, dtype=torch.bfloat16).requires_grad_()
            go = torch.randn(B, res * res, dim, device="cuda", generator=g, dtype=torch.bfloat16)

            def fwd_bwd(fn):
                def run():
                    x.grad = None
                    for p in blk.parameters():
                        p.grad = None
                    fn().backward(go)
                return run

            arms = {"native": fwd_bwd(lambda: blk.attn.forward_image(x, res, res, s)),
                    "window": fwd_bwd(lambda: _window_path(blk, x))}
            ms = _time_alternated(arms, iters)
            peak = {arm: _peak_gib(run) for arm, run in arms.items()}

            # the kernels alone, on the projection of x
            with torch.no_grad():
                qkv = blk.attn.qkv(x).contiguous()
                if version == 2:
                    table = (16 * torch.sigmoid(blk.attn.cpb_mlp(blk.attn.relative_coords_table.bfloat16())
                                                .view(-1, h).float())).contiguous()
                    tau = torch.full((h,), 10.0, device="cuda")
                else:
                    table, tau = blk.attn.relative_position_bias_table.float().contiguous(), None
            o, lse = ext.window_attn_fwd(qkv, res, res, ws, s, h, d ** -0.5, table, tau)
            kern = _time_alternated({
                "fwd": lambda: ext.window_attn_fwd(qkv, res, res, ws, s, h, d ** -0.5, table, tau),
                "bwd": lambda: ext.window_attn_bwd(go, qkv, lse, res, res, ws, s, h, d ** -0.5, table, tau),
            }, iters)
            tokens, lse_bytes = B * res * res, lse.numel() * 4
            fwd_bytes = tokens * 4 * dim * 2 + lse_bytes
            bwd_bytes = tokens * 7 * dim * 2 + lse_bytes
            row = dict(model=name, stage=stage + 1, B=B, map=res, window=ws, shift=s, heads=h, head_dim=d,
                       cosine=version == 2, native_ms=round(ms["native"], 3), window_ms=round(ms["window"], 3),
                       speedup=round(ms["window"] / ms["native"], 2),
                       native_peak_gib=round(peak["native"], 3), window_peak_gib=round(peak["window"], 3),
                       kernel_fwd_ms=round(kern["fwd"], 3), kernel_bwd_ms=round(kern["bwd"], 3),
                       kernel_fwd_gbs=round(fwd_bytes / kern["fwd"] / 1e6, 1),
                       kernel_bwd_gbs=round(bwd_bytes / kern["bwd"] / 1e6, 1),
                       kernel_fwd_hbm_share=round(fwd_bytes / kern["fwd"] / 1e9 / HBM_TBS, 3),
                       kernel_bwd_hbm_share=round(bwd_bytes / kern["bwd"] / 1e9 / HBM_TBS, 3))
            rows.append(row)
            print(json.dumps(row), flush=True)
            del blk, x, go, arms, qkv, o, lse
            torch.cuda.empty_cache()
    return rows


def _model(version, img, window, embed, heads):
    from libai_b200.optim import AdamW, get_default_optimizer_params

    M = v1.SwinTransformer if version == 1 else v2.SwinTransformerV2
    kw = {} if version == 1 else {"pretrained_window_sizes": [0, 0, 0, 0]}
    with param_defaults(dtype=torch.bfloat16, device="cuda", seed=1234):
        model = M(img_size=img, num_classes=1000, embed_dim=embed, depths=[2, 2, 6, 2], num_heads=heads,
                  window_size=window, drop_path_rate=0.1, **kw)
    model.to(device="cuda", dtype=torch.bfloat16)   # the patch-embedding convolution and the buffers
    opt = AdamW(get_default_optimizer_params(model, weight_decay_norm=0.0, weight_decay_bias=0.0,
                                             clip_grad_max_norm=5.0, clip_grad_norm_type=2.0), lr=1e-4)
    opt.setup()
    return model, opt


def step_rows(steps, rounds, B):
    rows = []
    native_pred = OF.window_attention_supported
    for name, version, img, window, embed, heads in (MODELS[0], MODELS[2]):
        model, opt = _model(version, img, window, embed, heads)
        model.train()
        g = torch.Generator(device="cuda").manual_seed(0)
        images = torch.randn(B, 3, img, img, device="cuda", generator=g)
        labels = torch.randint(0, 1000, (B,), device="cuda", generator=g)

        def step():
            opt.zero_grad()
            model(images, labels)["losses"].backward()
            opt.step()

        rates = {"native": [], "window": []}
        try:
            for _ in range(rounds):
                for arm in rates:
                    OF.window_attention_supported = native_pred if arm == "native" else (lambda *a, **k: False)
                    for _ in range(3):
                        step()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(steps):
                        step()
                    torch.cuda.synchronize()
                    rates[arm].append(B * steps / (time.perf_counter() - t0))
        finally:
            OF.window_attention_supported = native_pred
        row = dict(model=name, B=B, steps=steps, rounds=rounds,
                   native_images_s=[round(r, 1) for r in rates["native"]],
                   window_images_s=[round(r, 1) for r in rates["window"]],
                   native_median=round(statistics.median(rates["native"]), 1),
                   window_median=round(statistics.median(rates["window"]), 1))
        row["speedup"] = round(row["native_median"] / row["window_median"], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del model, opt, images, labels
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join("output", "swin_bench.json"))
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--skip-steps", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("swin_bench needs a GPU")
    info = gpu_info()
    print(json.dumps(info), flush=True)
    out = dict(info, ops=op_rows(a.iters, a.batch))
    if not a.skip_steps:
        out["steps"] = step_rows(a.steps, a.rounds, a.batch)
    out["after"] = gpu_info()
    print(json.dumps(out["after"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
