"""Steady-state cost of the fused comm+GEMM kernels at the benchmark model's tensor-parallel shapes: every op is issued
back to back (no host barrier between iterations, like inside a training step) and compared with the plain GEMM of the
same shape.  Run under torchrun with 2+ GPUs; rank 0 writes output/comm_bench.json."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    from libai_b200.config import DictConfig
    from libai_b200.ops import comm_gemm, load_ext
    from libai_b200.utils import distributed as dutil

    ext = load_ext()
    topo = dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=world, pipeline_parallel_size=1,
                                                 sequence_parallel=True, fused_tp_comm=True)))
    g = topo.tp_group
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else "output/comm_bench.json"
    tag = os.environ.get("LIBAI_B200_DEBUG_COMM_NO_PAYLOAD", "0")

    def bench(fn, iters=40):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return round(float(t) * 1e3, 1)   # us

    res = {"world": world, "no_payload": tag}
    h = 1024
    for T in (8192 * world // 2, 16384 * world // 2):          # tokens of the TP group: mb8 and mb16 per 2 ranks
        rows = T // world
        xs = torch.randn(rows, h, device="cuda").bfloat16()
        r = {}
        for name, Nl in (("qkv", 3 * h // world), ("fc1", 4 * h // world)):
            w = (torch.randn(Nl, h, device="cuda") * 0.03).bfloat16()
            b = torch.zeros(Nl, device="cuda").bfloat16()
            xfull = torch.randn(T, h, device="cuda").bfloat16()
            act = "gelu" if name == "fc1" else None
            r[f"ag_nt_{name}"] = bench(lambda: comm_gemm.ag_gemm(xs, w, b, act, g, need_pre=act is not None))
            r[f"plain_nt_{name}"] = bench(lambda: ext.linear_fwd(xfull, w, b, 1 if act else 0, act is not None))
            # column backward: dgrad GEMM->RS (NN) and the gathered-B wgrad
            gy = torch.randn(T, Nl, device="cuda").bfloat16()
            r[f"rs_nn_{name}_dgrad"] = bench(lambda: comm_gemm.gemm_rs(gy, w, None, None, g, layout=1))
            r[f"plain_nn_{name}_dgrad"] = bench(lambda: ext.gemm(gy, w, 1, None, None, False, torch.bfloat16))
            mg = torch.zeros(Nl, h, device="cuda")
            r[f"ag_wgrad_{name}"] = bench(lambda: comm_gemm.ag_wgrad(gy, xs, mg, True, g))
            r[f"plain_wgrad_{name}"] = bench(lambda: ext.gemm(gy, xfull, 2, None, mg, True, torch.float32))
        for name, Kl in (("proj", h // world), ("fc2", 4 * h // world)):
            w = (torch.randn(h, Kl, device="cuda") * 0.03).bfloat16()
            b = torch.zeros(h, device="cuda").bfloat16()
            x = torch.randn(T, Kl, device="cuda").bfloat16()
            res_t = torch.randn(rows, h, device="cuda").bfloat16()
            r[f"rs_nt_{name}"] = bench(lambda: comm_gemm.gemm_rs(x, w, b, res_t, g))
            r[f"plain_nt_{name}"] = bench(lambda: ext.linear_fwd(x, w, b, 0, False))
            gys = torch.randn(rows, h, device="cuda").bfloat16()
            r[f"ag_nn_{name}_dgrad"] = bench(lambda: comm_gemm.ag_gemm(gys, w, None, None, g, layout=1, fill_local=True))
            gyf = torch.randn(T, h, device="cuda").bfloat16()
            r[f"plain_nn_{name}_dgrad"] = bench(lambda: ext.gemm(gyf, w, 1, None, None, False, torch.bfloat16))
        # copy-CTA count sweep on the qkv AG->GEMM
        w = (torch.randn(3 * h // world, h, device="cuda") * 0.03).bfloat16()
        orig = comm_gemm._n_comm_ctas
        for n in (8, 24, 32, 48):
            comm_gemm._n_comm_ctas = lambda world, n=n: n
            r[f"ag_nt_qkv_copyctas{n}"] = bench(lambda: comm_gemm.ag_gemm(xs, w, None, None, g))
        comm_gemm._n_comm_ctas = orig
        # NCCL reference for the payloads
        full = torch.empty(T, h, device="cuda", dtype=torch.bfloat16)
        r["nccl_allgather_Txh"] = bench(lambda: dist.all_gather_into_tensor(full, xs, group=g))
        o = torch.empty(rows, h, device="cuda", dtype=torch.bfloat16)
        r["nccl_reducescatter_Txh"] = bench(lambda: dist.reduce_scatter_tensor(o, full, group=g))
        res[f"T{T}"] = r
        if rank == 0:
            print(T, json.dumps(r), flush=True)
    if rank == 0:
        os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
