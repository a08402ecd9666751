"""Spawn ``world`` CPU processes with a gloo process group and run ``fn(rank, world, *args)`` in each
("multi-node without a cluster").  Return values of all ranks are collected."""
import os
import socket
import traceback

import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _plain(obj):
    """Tensors -> numpy so results cross the process boundary by value (no fd passing)."""
    import torch

    if isinstance(obj, torch.Tensor):
        return obj.detach().cpu().float().numpy() if obj.dtype.is_floating_point else obj.detach().cpu().numpy()
    if isinstance(obj, dict):
        return {k: _plain(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_plain(v) for v in obj)
    return obj


def _worker(rank, world, port, fn, args, queue):
    os.environ.update(
        RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world),
        MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="1",
    )
    import torch
    import torch.distributed as dist

    torch.set_num_threads(1)
    try:
        dist.init_process_group("gloo", rank=rank, world_size=world)
        out = fn(rank, world, *args)
        queue.put((rank, "ok", _plain(out)))
    except Exception:
        queue.put((rank, "err", traceback.format_exc()))
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def run_distributed(fn, world, *args, timeout=300):
    ctx = mp.get_context("spawn")
    queue = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, fn, args, queue)) for r in range(world)]
    for p in procs:
        p.start()
    results = {}
    try:
        for _ in range(world):
            rank, status, payload = queue.get(timeout=timeout)
            if status != "ok":
                raise RuntimeError(f"rank {rank} failed:\n{payload}")
            results[rank] = payload
    finally:
        for p in procs:
            p.join(timeout=10)
            if p.is_alive():
                p.terminate()
    return [results[r] for r in range(world)]
