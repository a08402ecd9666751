"""Multi-GPU check of the fused NVLink collectives against NCCL (run under torchrun, 2+ GPUs).

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/gpu_comm_check.py

Every case prints one JSON line from rank 0 (max error over ranks, device time = max over ranks)."""
import json
import os
import sys
import traceback

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

RESULTS = []


def rel_err(a, b):
    return float((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6))


def max_over_ranks(x):
    t = torch.tensor([float(x)], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def timeit(fn, iters=20, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return max_over_ranks(ts[len(ts) // 2])


def record(name, fn):
    try:
        info = fn() or {}
        info.setdefault("ok", True)
    except Exception as e:  # noqa
        info = {"ok": False, "error": f"{type(e).__name__}: {e}", "trace": traceback.format_exc()[-1200:]}
    info["ok"] = bool(max_over_ranks(0.0 if info["ok"] else 1.0) == 0.0)
    RESULTS.append({"name": name, **info})
    if dist.get_rank() == 0:
        print(json.dumps(RESULTS[-1]), flush=True)


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    from libai_b200.config import DictConfig
    from libai_b200.ops import comm_gemm, load_ext
    from libai_b200.parallel import mappings
    from libai_b200.parallel.symm_mem import get_workspace
    from libai_b200.utils import distributed as dutil

    ext = load_ext()
    topo = dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=world, pipeline_parallel_size=1,
                                                 sequence_parallel=True, fused_tp_comm=True)))
    group = topo.tp_group
    torch.manual_seed(1234)  # same on all ranks

    def symm():
        ws = get_workspace(group)
        for i in range(3):
            ext.device_barrier(ws.flags.peer_ptrs(0), world, rank, 5, ws.next_epoch())
        torch.cuda.synchronize()
        return {"peer_access": bool(ext.can_access_peer(rank, (rank + 1) % world))}

    record("symmetric memory + device barrier", symm)

    M, K, N = 8192, 1024, 4096
    Nl, Kl = N // world, N // world

    def aggemm():
        xfull = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(Nl, K, device="cuda") * 0.05).bfloat16()
        b = torch.randn(Nl, device="cuda").bfloat16()
        xs = xfull[rank * (M // world): (rank + 1) * (M // world)].contiguous()
        y, _, _ = comm_gemm.ag_gemm(xs, w, b, None, group)
        ref = xfull.float() @ w.float().t() + b.float()
        err = rel_err(y, ref)
        for _ in range(3):  # repeated calls exercise the parity/double buffering + the device-side call counters
            y2, _, _ = comm_gemm.ag_gemm(xs, w, b, None, group)
        err2 = rel_err(y2, ref)
        # fill_local: the gathered buffer itself must equal the all-gather
        _, _, xg = comm_gemm.ag_gemm(xs, w, b, None, group, fill_local=True)
        torch.cuda.synchronize()
        gather_ok = torch.equal(xg, xfull)
        # fused GELU epilogue with the pre-activation copy
        yg, pre, _ = comm_gemm.ag_gemm(xs, w, b, "gelu", group, need_pre=True)
        err_act = max(rel_err(pre, ref), rel_err(yg, torch.nn.functional.gelu(ref)))
        ms = timeit(lambda: comm_gemm.ag_gemm(xs, w, b, None, group))

        def nccl():
            g = torch.empty(M, K, device="cuda", dtype=torch.bfloat16)
            dist.all_gather_into_tensor(g, xs, group=group)
            return torch.nn.functional.linear(g, w, b)

        ms_ref = timeit(nccl)
        ms_gemm = timeit(lambda: ext.linear_fwd(xfull, w, b, 0, False))
        flops = 2.0 * M * Nl * K
        link_bytes = (world - 1) * (M // world) * K * 2       # this rank's shard to every peer
        roof_ms = max(flops / 1.6e15, link_bytes / 770e9) * 1e3
        return {"ok": err < 2e-2 and err2 < 2e-2 and gather_ok and err_act < 2e-2, "rel_err": err, "rel_err_repeat": err2,
                "gathered_buffer_exact": gather_ok, "rel_err_gelu_pre": err_act, "fused_ms": ms,
                "nccl_plus_cublas_ms": ms_ref, "gemm_only_ms": ms_gemm, "copy_ctas": comm_gemm._n_comm_ctas(world),
                "roofline_ms": roof_ms, "roofline_fraction": roof_ms / ms}

    record(f"AG->GEMM M{M} N{Nl} K{K}", aggemm)

    def gemmrs():
        x = torch.randn(M, Kl, device="cuda").bfloat16()
        w = (torch.randn(K, Kl, device="cuda") * 0.05).bfloat16()   # out features = K (=h), in = f/t
        b = torch.randn(K, device="cuda").bfloat16()
        res = torch.randn(M // world, K, device="cuda").bfloat16()
        y = comm_gemm.gemm_rs(x, w, b, res, group)
        part = (x.float() @ w.float().t())
        dist.all_reduce(part, group=group)
        ref = part[rank * (M // world): (rank + 1) * (M // world)] + b.float() + res.float()
        err = rel_err(y, ref)
        for _ in range(3):
            y2 = comm_gemm.gemm_rs(x, w, b, res, group)
        err2 = rel_err(y2, ref)
        ms = timeit(lambda: comm_gemm.gemm_rs(x, w, b, res, group))

        def nccl():
            p = torch.nn.functional.linear(x, w)
            o = torch.empty(M // world, K, device="cuda", dtype=torch.bfloat16)
            dist.reduce_scatter_tensor(o, p, group=group)
            return o + b + res

        ms_ref = timeit(nccl)
        ms_gemm = timeit(lambda: ext.linear_fwd(x, w, None, 0, False))
        flops = 2.0 * M * K * Kl
        link_bytes = (world - 1) * (M // world) * K * 2
        roof_ms = max(flops / 1.6e15, link_bytes / 770e9) * 1e3
        return {"ok": err < 3e-2 and err2 < 3e-2, "rel_err": err, "rel_err_repeat": err2, "fused_ms": ms,
                "cublas_plus_nccl_ms": ms_ref, "gemm_only_ms": ms_gemm, "roofline_ms": roof_ms,
                "roofline_fraction": roof_ms / ms}

    record(f"GEMM->RS M{M} N{K} K{Kl}", gemmrs)

    def gemmrs_odd_n():
        """N not a multiple of the tile width (Llama-7B tp4: ffn/t = 2752)."""
        Mo, No, Ko = 2048, 2752, 512
        x = torch.randn(Mo, Ko, device="cuda").bfloat16()
        w = (torch.randn(No, Ko, device="cuda") * 0.05).bfloat16()
        y = comm_gemm.gemm_rs(x, w, None, None, group)
        part = (x.float() @ w.float().t())
        dist.all_reduce(part, group=group)
        ref = part[rank * (Mo // world): (rank + 1) * (Mo // world)]
        err = rel_err(y, ref)
        xs = x[rank * (Mo // world): (rank + 1) * (Mo // world)].contiguous()
        xfull = torch.empty(Mo, Ko, device="cuda", dtype=torch.bfloat16)
        dist.all_gather_into_tensor(xfull, xs, group=group)
        y2, _, _ = comm_gemm.ag_gemm(xs, w, None, None, group)
        err2 = rel_err(y2, xfull.float() @ w.float().t())
        return {"ok": err < 3e-2 and err2 < 2e-2, "rs_rel_err": err, "ag_rel_err": err2}

    record("AG->GEMM / GEMM->RS with N = 2752", gemmrs_odd_n)

    def agwgrad():
        """dW = dyᵀ · all_gather(x_shard) with the all-gather inside the split-K wgrad kernel."""
        T, h, Nloc = 8192, 1024, 3072 // world
        xfull = torch.randn(T, h, device="cuda").bfloat16()
        dist.broadcast(xfull, 0)
        gy = (torch.randn(T, Nloc, device="cuda") * 0.1).bfloat16()
        xs = xfull[rank * (T // world): (rank + 1) * (T // world)].contiguous()
        out = torch.zeros(Nloc, h, device="cuda", dtype=torch.float32)
        comm_gemm.ag_wgrad(gy, xs, out, True, group)
        comm_gemm.ag_wgrad(gy, xs, out, True, group)      # accumulates
        ref = 2.0 * (gy.float().t() @ xfull.float())
        err = rel_err(out, ref)
        ms = timeit(lambda: comm_gemm.ag_wgrad(gy, xs, out, True, group))

        def nccl():
            g = torch.empty(T, h, device="cuda", dtype=torch.bfloat16)
            dist.all_gather_into_tensor(g, xs, group=group)
            return ext.gemm(gy, g, 2, None, out, True, torch.float32)

        ms_ref = timeit(nccl)
        ms_gemm = timeit(lambda: ext.gemm(gy, xfull, 2, None, out, True, torch.float32))
        return {"ok": err < 2e-2, "rel_err": err, "fused_ms": ms, "nccl_allgather_plus_native_wgrad_ms": ms_ref,
                "wgrad_only_ms": ms_gemm}

    record("AG->wgrad (gathered B, split-K) T8192", agwgrad)

    def graph_replay():
        """The fused kernels inside a CUDA graph: call counters / arrival targets live in device memory, so the SAME
        captured launches are replayed with fresh data and must keep producing the right result."""
        T, h = 4096, 1024
        fl = 4096 // world
        w1 = (torch.randn(fl, h, device="cuda") * 0.03).bfloat16()
        w2 = (torch.randn(h, fl, device="cuda") * 0.03).bfloat16()
        xs = torch.randn(T // world, h, device="cuda").bfloat16()
        static_x = xs.clone()

        def body():
            hmid, _, _ = comm_gemm.ag_gemm(static_x, w1, None, "gelu", group)
            return comm_gemm.gemm_rs(hmid, w2, None, None, group)

        for _ in range(3):
            body()
        torch.cuda.synchronize()
        dist.barrier()
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            with torch.cuda.graph(g, stream=side):
                static_y = body()
        torch.cuda.current_stream().wait_stream(side)
        errs = []
        for it in range(6):
            xnew = torch.randn(T // world, h, device="cuda").bfloat16() * (1 + it)
            static_x.copy_(xnew)
            g.replay()
            if it % 2 == 1:
                body()        # eager calls interleaved with replays keep working (shared device-side counters)
            xfull = torch.empty(T, h, device="cuda", dtype=torch.bfloat16)
            dist.all_gather_into_tensor(xfull, xnew, group=group)
            part = torch.nn.functional.gelu(xfull.float() @ w1.float().t()).bfloat16().float() @ w2.float().t()
            dist.all_reduce(part, group=group)
            errs.append(rel_err(static_y, part[rank * (T // world): (rank + 1) * (T // world)]))
        ms = timeit(lambda: g.replay())
        return {"ok": max(errs) < 3e-2, "errs": errs, "replay_ms": ms}

    record("fused AG->GEMM + GEMM->RS replayed from a CUDA graph", graph_replay)

    def autograd_parity():
        """Column + row fused linears and the fused TP MLP (fwd + bwd) against the NCCL mappings path."""
        T, h, f = 2048, 1024, 4096
        x = torch.randn(T // world, h, device="cuda").bfloat16()
        w1 = (torch.randn(f // world, h, device="cuda") * 0.03).bfloat16()
        b1 = (torch.randn(f // world, device="cuda") * 0.1).bfloat16()
        w2 = (torch.randn(h, f // world, device="cuda") * 0.03).bfloat16()
        b2 = (torch.randn(h, device="cuda") * 0.1).bfloat16()
        res = torch.randn(T // world, h, device="cuda").bfloat16()
        outs = []
        for mode in ("mlp", "colrow", "nccl"):
            xx = x.clone().requires_grad_(True)
            a1, a2 = w1.clone().requires_grad_(True), w2.clone().requires_grad_(True)
            bb, bb2 = b1.clone().requires_grad_(True), b2.clone().requires_grad_(True)
            rr = res.clone().requires_grad_(True)
            if mode == "mlp":
                y = comm_gemm.tp_mlp(xx, a1, bb, a2, bb2, rr, "gelu", group)
            elif mode == "colrow":
                hmid = comm_gemm.column_parallel_linear(xx, a1, bb, "gelu", group)
                y = comm_gemm.row_parallel_linear(hmid, a2, bb2, rr, group)
            else:
                os.environ["LIBAI_B200_IMPL"] = "ref"
                g = mappings.gather_from_sp(xx)
                hmid = torch.nn.functional.gelu(torch.nn.functional.linear(g, a1, bb))
                y = mappings.reduce_scatter_to_sp(torch.nn.functional.linear(hmid, a2)) + bb2 + rr
                os.environ["LIBAI_B200_IMPL"] = "native"
            gy = torch.randn(y.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7 + rank)).bfloat16() * 0.01
            y.backward(gy)
            outs.append((y.detach(), xx.grad, a1.grad, a2.grad, bb.grad, bb2.grad, rr.grad))
        errs_mlp = [rel_err(a, b) for a, b in zip(outs[0], outs[2])]
        errs_cr = [rel_err(a, b) for a, b in zip(outs[1], outs[2])]
        return {"ok": max(errs_mlp) < 4e-2 and max(errs_cr) < 4e-2, "errs_tp_mlp": errs_mlp, "errs_col_row": errs_cr}

    record("fused column/row linear + TP-MLP autograd vs NCCL", autograd_parity)

    def _grid(x):
        # Gradients on a 2^-10 grid: their sum over ranks is exact in fp32 whatever the order of the additions.  Without
        # this the check is ill-conditioned, not the kernels: the first Adam step moves every element by
        # lr * g / (|g| + 1e-8), i.e. by +-lr with the SIGN of the reduced gradient, and among 4 M elements there is
        # (with these fixed seeds: at 8 ranks) one whose 8-term sum is ~1e-8 — the rotated summation order of the pull
        # kernel, NCCL's ring order and the sequential local reference then disagree by half a step on that element
        # (0.5 * lr = 0.005 against max|p| = 0.13, a 0.0385 max-norm "error"; commutative at 2 ranks, hence bitwise equal
        # there).
        return (x * 1024.0).round() / 1024.0

    def zero():
        """ZeRO-1 with fused RS+Adam+AG kernels vs the NCCL sequence (dp = world)."""
        from libai_b200.optim import AdamW

        dutil.reset_dist_util()
        dutil.setup_dist_util(DictConfig(dict(data_parallel_size=world, tensor_parallel_size=1, pipeline_parallel_size=1)))
        finals = []
        times = []
        nvls = False
        for arm in ("fused", "fused_nvls", "nccl"):
            fused = arm != "nccl"
            os.environ["LIBAI_B200_NVLS"] = "1" if arm == "fused_nvls" else "0"
            torch.manual_seed(5)
            params = [torch.nn.Parameter((torch.randn(1 << 22, device="cuda") * 0.02).bfloat16()),
                      torch.nn.Parameter((torch.randn(1000, 333, device="cuda") * 0.02).bfloat16())]
            opt = AdamW(params, lr=1e-2, weight_decay=0.01)
            opt.fused_zero_comm = fused
            opt.configure(zero_stage=1)
            opt.setup()

            def step(i):
                opt.zero_grad()
                g = torch.Generator(device="cuda").manual_seed(100 * i + rank)
                for p in params:
                    p.main_grad.copy_(_grid(torch.randn(p.shape, device="cuda", generator=g)))
                opt.step()

            for i in range(3):
                step(i)
            torch.cuda.synchronize()
            finals.append([p.detach().float().clone() for p in params])
            times.append(timeit(lambda: opt.step(), iters=10, warmup=2))
            if arm == "fused_nvls":
                nvls = bool(opt._groups[0].symm is not None and opt._groups[0].symm["grad"].mc_ptr)
        os.environ["LIBAI_B200_NVLS"] = "0"
        errs = [rel_err(a, b) for a, b in zip(finals[0], finals[2])] + [rel_err(a, b) for a, b in zip(finals[1], finals[2])]
        # third opinion: the same three AdamW steps computed locally in fp32 from every rank's (seeded) gradients,
        # so a mismatch can be attributed to one arm
        torch.manual_seed(5)
        p0 = (torch.randn(1 << 22, device="cuda") * 0.02).bfloat16().float()
        m = torch.zeros_like(p0)
        v = torch.zeros_like(p0)
        for i in range(3):
            g = torch.zeros_like(p0)
            for r in range(world):
                gen = torch.Generator(device="cuda").manual_seed(100 * i + r)
                g += _grid(torch.randn(p0.shape, device="cuda", generator=gen))
            g /= world
            m.mul_(0.9).add_(g, alpha=0.1)
            v.mul_(0.999).addcmul_(g, g, value=0.001)
            upd = (m / (1 - 0.9 ** (i + 1))) / ((v / (1 - 0.999 ** (i + 1))).sqrt() + 1e-8) + 0.01 * p0
            p0 -= 1e-2 * upd
        ref_errs = [rel_err(finals[0][0], p0), rel_err(finals[2][0], p0), rel_err(finals[1][0], p0)]
        return {"ok": max(errs) < 1e-2 and max(ref_errs) < 2e-2, "errs": errs, "fused_vs_local_ref": ref_errs[0],
                "nccl_vs_local_ref": ref_errs[1], "nvls_vs_local_ref": ref_errs[2], "fused_step_ms": times[0],
                "fused_nvls_step_ms": times[1], "nccl_step_ms": times[2], "nvls_multicast_available": nvls}

    record("ZeRO fused RS+Adam+AG vs NCCL", zero)

    def overlap():
        """Early reduce-scatter launched from the backward pass (side stream) == end-of-step reduce-scatter on a small
        GPT trained data-parallel for three steps."""
        from libai_b200.layers._param import param_defaults
        from libai_b200.models.gpt_model import GPTForPreTraining
        from libai_b200.optim import AdamW, get_default_optimizer_params

        cfg = DictConfig(dict(
            hidden_layers=6, vocab_size=512, hidden_size=256, ffn_hidden_size=1024, num_attention_heads=4,
            max_seq_length=256, embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
            layernorm_epsilon=1e-5, initializer_range=0.02, use_scaled_init_for_output_weights=True,
            bias_gelu_fusion=True, bias_dropout_fusion=True, scale_mask_softmax_fusion=True,
            apply_query_key_layer_scaling=False, apply_residual_post_layernorm=False, amp_enabled=True))
        finals, launched = [], []
        for use_overlap in (True, False):
            dutil.reset_dist_util()
            dutil.setup_dist_util(DictConfig(dict(data_parallel_size=world, tensor_parallel_size=1, pipeline_parallel_size=1)))
            with param_defaults(dtype=torch.bfloat16, device="cuda", seed=11):
                model = GPTForPreTraining(cfg)
            opt = AdamW(get_default_optimizer_params(model, clip_grad_max_norm=1.0, clip_grad_norm_type=2.0), lr=1e-3,
                        weight_decay=0.01)
            opt.configure(zero_stage=1, param_names={id(p): n for n, p in model.named_parameters()})
            opt.setup()
            triggers = opt.plan_overlap() if use_overlap else ()
            model.grad_ready_layers = tuple(triggers)
            n_early = 0
            for step in range(3):
                g = torch.Generator(device="cuda").manual_seed(1000 * step + rank)
                ids = torch.randint(0, 512, (4, 256), device="cuda", generator=g)
                opt.zero_grad()
                model.grad_ready_callback = opt.on_grads_ready if use_overlap else None
                model(ids, ids)["lm_loss"].backward()
                n_early += int(getattr(opt, "_early_launched", False))
                if step == 0:   # the reduced gradients themselves (before Adam turns tiny differences into sign flips)
                    opt.sync_gradients()
                    torch.cuda.synchronize()
                    grads0 = torch.cat([fg.grad_shard().clone() for fg in opt._groups if fg is not None])
                opt.step()
            torch.cuda.synchronize()
            finals.append((grads0, torch.cat([p.detach().float().reshape(-1) for p in model.parameters()])))
            launched.append((list(triggers), n_early))
        # (split-K wgrad accumulates with fp32 atomics, so two runs agree to rounding, not bit for bit)
        g_err = rel_err(finals[0][0], finals[1][0])
        p_diff = float((finals[0][1] - finals[1][1]).abs().mean())
        return {"ok": g_err < 1e-4 and p_diff < 1e-4 and launched[0][1] == 3 and len(launched[0][0]) > 0,
                "reduced_grad_rel_err": g_err, "param_mean_abs_diff": p_diff, "trigger_layers": launched[0][0],
                "steps_with_early_reduce": launched[0][1]}

    record("overlapped grad reduce-scatter == end-of-step", overlap)

    if rank == 0:
        out = "output/comm_check.json"
        if "--out" in sys.argv:
            out = sys.argv[sys.argv.index("--out") + 1]
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            json.dump(RESULTS, f, indent=1)
        bad = [r["name"] for r in RESULTS if not r["ok"]]
        print(f"SUMMARY: {len(RESULTS) - len(bad)}/{len(RESULTS)} ok; failed: {bad}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
