"""Distributed topology: one process per GPU, explicit process groups for TP / DP / PP.

Behavioural spec: reference libai/utils/distributed.py — size clamping and derivation (:88-147),
rank mesh "PP outermost, DP middle, TP innermost" (:149-159, :246-252), the layer→stage map with
the "middle stages get more layers" rule (:161-195), ``custom_pipeline_stage_id`` (:115-130),
helpers (:366-494).

Design (H100-first, not a port): the reference expresses placement through OneFlow SBP/placement
objects and lets the runtime insert collectives.  Here the topology is a plain object that owns
``torch.distributed`` process groups (NCCL for device collectives, gloo for host objects) built
from the same rank formula

    rank = stage * (D * t) + dp_idx * t + tp_idx

and the layers / engine call collectives (or fused comm kernels over NVLink symmetric memory)
explicitly.  ``get_layer_stage_id(layer_idx)`` carries the placement information that
``get_layer_placement`` carried in the reference.
"""
from __future__ import annotations

import io
import logging
import os
import pickle
from datetime import timedelta
from typing import Any, List, Optional

import torch
import torch.distributed as dist

from libai_b200.config.config import try_get_key
from libai_b200.config.dictconfig import DictConfig, ListConfig

logger = logging.getLogger(__name__)

_DIST_UTIL: Optional["DistributedTopology"] = None


# --------------------------------------------------------------------------------------
# process-level helpers (valid before/without init_process_group)
# --------------------------------------------------------------------------------------
def get_rank() -> int:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank()
    return int(os.environ.get("RANK", 0))


def get_world_size() -> int:
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size()
    return int(os.environ.get("WORLD_SIZE", 1))


def get_local_rank() -> int:
    return int(os.environ.get("LOCAL_RANK", get_rank()))


def get_num_nodes() -> int:
    lws = int(os.environ.get("LOCAL_WORLD_SIZE", 0)) or get_world_size()
    return max(1, get_world_size() // max(1, lws))


def is_main_process() -> bool:
    return get_rank() == 0


def is_last_process() -> bool:
    return get_rank() == get_world_size() - 1


def init_process_group(device_type: str = "cuda", timeout_s: int = 1800) -> None:
    """Initialise ``torch.distributed`` from the torchrun environment (no-op if world==1 and
    no rendezvous variables are present, so single-process use needs no launcher)."""
    if dist.is_initialized():
        return
    world = int(os.environ.get("WORLD_SIZE", 1))
    if world == 1 and "MASTER_ADDR" not in os.environ:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ.setdefault("MASTER_PORT", str(29400 + os.getpid() % 2000))
        os.environ.setdefault("RANK", "0")
        os.environ.setdefault("WORLD_SIZE", "1")
    use_cuda = device_type == "cuda" and torch.cuda.is_available()
    if use_cuda:
        torch.cuda.set_device(get_local_rank() % torch.cuda.device_count())
    backend = "cpu:gloo,cuda:nccl" if use_cuda else "gloo"
    kwargs = {}
    if use_cuda:
        kwargs["device_id"] = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group(backend=backend, timeout=timedelta(seconds=timeout_s), **kwargs)


# --------------------------------------------------------------------------------------
# layer → stage map
# --------------------------------------------------------------------------------------
def compute_layer_stage_ids(num_layers: int, pp: int) -> List[int]:
    """Stage id of every layer index.

    Even split when ``num_layers % pp != 0`` puts the *extra* layers on the later stages; when
    ``pp >= 4 and num_layers >= 8 and num_layers % pp == 0`` the first stage (embedding) and the
    last stage (head + loss) get fewer layers and the middle ones more — e.g. L=24, p=4 →
    6/7/7/4 (reference: libai/utils/distributed.py:161-195).
    """
    if pp >= 4 and num_layers >= 8 and num_layers % pp == 0:
        virtual = num_layers + min(pp - 1, num_layers // pp)
    else:
        virtual = num_layers
    per_stage, extra = divmod(virtual, pp)
    ids: List[int] = []
    for stage in range(pp):
        n = per_stage + (1 if stage >= pp - extra else 0)
        ids.extend([stage] * n)
    return ids[:num_layers]


class DistributedTopology:
    """Sizes, coordinates and process groups of the (pp, dp, tp) mesh of this job."""

    def __init__(self, cfg: DictConfig):
        self._cfg = cfg
        world = get_world_size()
        nodes = get_num_nodes()
        gpus_per_node = world // nodes
        for key, actual in (("num_gpus_per_node", gpus_per_node), ("num_nodes", nodes)):
            if try_get_key(cfg, key, default=actual) != actual:
                logger.warning(
                    f"'train.dist.{key}' differs from the launch environment: {cfg[key]} != {actual}"
                )
        cfg.num_nodes, cfg.num_gpus_per_node = nodes, gpus_per_node
        self.num_nodes, self.num_gpus_per_node, self.world_size = nodes, gpus_per_node, world

        self._device_type = try_get_key(cfg, "device_type", default="cuda")
        if self._device_type not in ("cuda", "cpu"):
            raise NotImplementedError(
                f"Unsupported device {self._device_type}: this framework targets H100 ('cuda'); "
                "'cpu' is kept for gloo plumbing tests"
            )
        if self._device_type == "cuda" and not torch.cuda.is_available():
            self._device_type = "cpu"

        # ---- sizes (clamped like the reference) --------------------------------------
        tp = min(int(try_get_key(cfg, "tensor_parallel_size", default=1)), world)
        assert world % tp == 0, f"world size ({world}) is not divisible by tensor parallel size ({tp})"
        pp = min(int(try_get_key(cfg, "pipeline_parallel_size", default=1)), world // tp)
        cfg.tensor_parallel_size, cfg.pipeline_parallel_size = tp, pp
        if pp > 1:
            assert (
                try_get_key(cfg, "pipeline_num_layers") is not None
            ), "cfg.train.dist.pipeline_num_layers must be set when run pipeline parallel"
            assert cfg.pipeline_num_layers >= pp, (
                f"number of layers ({cfg.pipeline_num_layers}) is less than"
                f" pipeline model parallel size ({pp})"
            )
        elif try_get_key(cfg, "pipeline_num_layers") is None:
            cfg.pipeline_num_layers = 10000
        assert world % (tp * pp) == 0, f"world size ({world}) is not divisible by tp*pp ({tp}*{pp})"
        dp = world // (tp * pp)
        cfg.data_parallel_size = dp
        self.tensor_parallel_size, self.pipeline_parallel_size, self.data_parallel_size = tp, pp, dp
        # Megatron-style sequence parallelism inside the TP region (new vs. the reference):
        # activations between TP blocks are sharded over tokens, col/row linears become
        # all-gather->GEMM / GEMM->reduce-scatter.
        # "auto" (the default of configs/common/train.py) is resolved by `engine.default_setup` from the model class
        # (`supports_sequence_parallel`); an unresolved "auto" counts as off.
        def _flag(key):
            v = try_get_key(cfg, key, default=False)
            return False if isinstance(v, str) else bool(v)

        self.sequence_parallel = _flag("sequence_parallel") and tp > 1
        # run the SP collectives inside the GEMM kernels (AG->GEMM / GEMM->RS over NVLink peer memory)
        self.fused_tp_comm = _flag("fused_tp_comm") and self.sequence_parallel

        # ---- layer → stage -------------------------------------------------------------
        self._layer_stage_ids = compute_layer_stage_ids(int(cfg.pipeline_num_layers), pp)
        if pp > 1:
            cfg.auto_pipeline_stage_id = list(self._layer_stage_ids)
            custom = try_get_key(cfg, "custom_pipeline_stage_id")
            if custom is not None:
                assert isinstance(custom, (list, ListConfig)), (
                    "type of cfg.train.dist.custom_pipeline_stage_id must be list"
                )
                custom = [int(x) for x in custom]
                assert max(custom) < pp, (
                    f"the element {max(custom)} in cfg.train.dist.custom_pipeline_stage_id "
                    f"is out of range for {pp} stages"
                )
                assert len(custom) == cfg.pipeline_num_layers, (
                    f"the length of cfg.train.dist.custom_pipeline_stage_id {len(custom)} must be "
                    f"equal to cfg.train.dist.pipeline_num_layers {cfg.pipeline_num_layers}"
                )
                self._layer_stage_ids = custom
            cfg.actual_pipeline_stage_id = list(self._layer_stage_ids)

        # ---- coordinates of this rank ---------------------------------------------------
        rank = get_rank()
        self.rank = rank
        self.pp_rank = rank // (dp * tp)
        self.dp_rank = (rank // tp) % dp
        self.tp_rank = rank % tp

        # ---- process groups ---------------------------------------------------------------
        self.tp_group = self.dp_group = self.pp_group = None
        self.embedding_group = None  # first+last stage, for tied embeddings
        self.tp_ranks = [self.pp_rank * dp * tp + self.dp_rank * tp + i for i in range(tp)]
        self.dp_ranks = [self.pp_rank * dp * tp + j * tp + self.tp_rank for j in range(dp)]
        self.pp_ranks = [s * dp * tp + self.dp_rank * tp + self.tp_rank for s in range(pp)]
        if dist.is_initialized() and world > 1:
            self._build_groups()

    def _build_groups(self):
        tp, dp, pp = self.tensor_parallel_size, self.data_parallel_size, self.pipeline_parallel_size
        # every rank must create every group, in the same order
        for s in range(pp):
            for j in range(dp):
                ranks = [s * dp * tp + j * tp + i for i in range(tp)]
                g = dist.new_group(ranks) if tp > 1 else None
                if self.rank in ranks:
                    self.tp_group = g
        for s in range(pp):
            for i in range(tp):
                ranks = [s * dp * tp + j * tp + i for j in range(dp)]
                g = dist.new_group(ranks) if dp > 1 else None
                if self.rank in ranks:
                    self.dp_group = g
        for j in range(dp):
            for i in range(tp):
                ranks = [s * dp * tp + j * tp + i for s in range(pp)]
                g = dist.new_group(ranks) if pp > 1 else None
                if self.rank in ranks:
                    self.pp_group = g
                if pp > 1:
                    er = [ranks[0], ranks[-1]]
                    eg = dist.new_group(er)
                    if self.rank in er:
                        self.embedding_group = eg

    # ---- reference-compatible accessors ----------------------------------------------------
    @property
    def model_parallel_size(self):
        # NB: the reference returns the *tensor* parallel size here (distributed.py:230-232)
        return self.tensor_parallel_size

    @property
    def device_type(self):
        return self._device_type

    def set_device_type(self, device_type):
        self._device_type = device_type

    @property
    def device(self) -> torch.device:
        if self._device_type == "cuda":
            return torch.device("cuda", torch.cuda.current_device())
        return torch.device("cpu")

    def get_layer_stage_id(self, layer_idx: int) -> int:
        return self._layer_stage_ids[layer_idx]

    def get_layer_ranks(self, layer_idx: int):
        """Ranks of the stage owning ``layer_idx`` as a ``[dp][tp]`` nested list."""
        s = self.get_layer_stage_id(layer_idx)
        dp, tp = self.data_parallel_size, self.tensor_parallel_size
        return [[s * dp * tp + j * tp + i for i in range(tp)] for j in range(dp)]

    def owns_layer(self, layer_idx: int) -> bool:
        return self.pipeline_parallel_size == 1 or self.get_layer_stage_id(layer_idx) == self.pp_rank

    @property
    def is_first_stage(self) -> bool:
        return self.pp_rank == 0

    @property
    def is_last_stage(self) -> bool:
        return self.pp_rank == self.pipeline_parallel_size - 1

    def is_tensor_model_parallel(self):
        return self.tensor_parallel_size > 1

    def is_data_parallel(self):
        return self.data_parallel_size > 1

    def is_pipeline_model_parallel(self):
        return self.pipeline_parallel_size > 1

    def is_data_model_parallel(self):
        return self.is_tensor_model_parallel() and self.is_data_parallel()

    def __repr__(self):
        return (
            f"DistributedTopology(world={self.world_size}, dp={self.data_parallel_size}, "
            f"tp={self.tensor_parallel_size}, pp={self.pipeline_parallel_size}, rank={self.rank} -> "
            f"(pp={self.pp_rank}, dp={self.dp_rank}, tp={self.tp_rank}), device={self._device_type})"
        )


_DistributeUtil = DistributedTopology  # reference name


def setup_dist_util(cfg) -> DistributedTopology:
    """Create the global topology from ``cfg.train.dist`` (initialises torch.distributed when
    launched under torchrun)."""
    global _DIST_UTIL
    device_type = try_get_key(cfg, "device_type", default="cuda")
    if int(os.environ.get("WORLD_SIZE", 1)) > 1 or "MASTER_ADDR" in os.environ:
        init_process_group(device_type)
    _DIST_UTIL = DistributedTopology(cfg)
    return _DIST_UTIL


def get_dist_util() -> DistributedTopology:
    """The global topology; lazily defaults to dp = world, tp = pp = 1."""
    global _DIST_UTIL
    if _DIST_UTIL is None:
        _DIST_UTIL = DistributedTopology(
            DictConfig(
                dict(data_parallel_size=get_world_size(), tensor_parallel_size=1, pipeline_parallel_size=1)
            )
        )
    return _DIST_UTIL


def reset_dist_util() -> None:
    global _DIST_UTIL
    _DIST_UTIL = None


# thin functional accessors -------------------------------------------------------------------
def model_parallel_seed(base_seed: int) -> int:
    """Seed of the *device* RNG (dropout): identical on all tensor-parallel ranks of one model replica — replicated
    activations must see identical masks, sharded ones add the TP rank as Philox salt (``ops.functional.tp_rng_salt``)
    — and different across data-parallel replicas and pipeline stages.  (The reference gets this from OneFlow's global
    generator; Megatron from its CudaRNGStatesTracker.)"""
    topo = get_dist_util()
    return int(base_seed) + 100003 * topo.dp_rank + 7919 * topo.pp_rank


def get_layer_stage_id(layer_idx: int) -> int:
    return get_dist_util().get_layer_stage_id(layer_idx)


def owns_layer(layer_idx: int) -> bool:
    return get_dist_util().owns_layer(layer_idx)


def get_data_parallel_rank() -> int:
    return get_dist_util().dp_rank


def get_data_parallel_size() -> int:
    return get_dist_util().data_parallel_size


def get_tensor_parallel_rank() -> int:
    return get_dist_util().tp_rank


def get_tensor_parallel_size() -> int:
    return get_dist_util().tensor_parallel_size


def get_pipeline_parallel_rank() -> int:
    return get_dist_util().pp_rank


def get_pipeline_parallel_size() -> int:
    return get_dist_util().pipeline_parallel_size


def get_tp_group():
    return get_dist_util().tp_group


def get_dp_group():
    return get_dist_util().dp_group


def get_pp_group():
    return get_dist_util().pp_group


def get_device() -> torch.device:
    return get_dist_util().device


def set_device_type(device_type):
    get_dist_util().set_device_type(device_type)


# host-object collectives ------------------------------------------------------------------------
def broadcast_py_object(obj: Any, src: int = 0) -> Any:
    """Broadcast an arbitrary picklable python object from ``src`` to every rank (gloo/CPU path)."""
    if get_world_size() == 1 or not dist.is_initialized():
        return obj
    box = [obj if get_rank() == src else None]
    dist.broadcast_object_list(box, src=src)
    return box[0]


def all_gather_py_object(obj: Any) -> List[Any]:
    if get_world_size() == 1 or not dist.is_initialized():
        return [obj]
    out = [None] * get_world_size()
    dist.all_gather_object(out, obj)
    return out


def synchronize() -> None:
    """Barrier across all ranks (no-op for a single process)."""
    if get_world_size() == 1 or not dist.is_initialized():
        return
    if torch.cuda.is_available() and get_dist_util().device_type == "cuda":
        dist.barrier(device_ids=[torch.cuda.current_device()])
    else:
        dist.barrier()


def all_reduce_scalar(t: torch.Tensor, group=None, op=dist.ReduceOp.SUM) -> torch.Tensor:
    if dist.is_initialized() and get_world_size() > 1:
        dist.all_reduce(t, op=op, group=group)
    return t


def dp_mean_to_rank0(value: torch.Tensor) -> torch.Tensor:
    """Average a last-stage scalar over the DP group; every rank of the DP group gets it."""
    topo = get_dist_util()
    v = value.detach().float().clone()
    if topo.dp_group is not None:
        dist.all_reduce(v, group=topo.dp_group)
        v /= topo.data_parallel_size
    return v


def tensor_to_rank0(tensor: torch.Tensor, device="cpu", to_local: bool = True) -> torch.Tensor:
    """Gather a DP-sharded (dim 0) tensor from the DP group and return it on ``device``.

    The reference moves a *global* tensor to rank 0 (distributed.py:472-482); with explicit
    process groups the equivalent is "concatenate the dp shards".  Returned on every caller.
    """
    topo = get_dist_util()
    t = tensor.detach()
    if topo.dp_group is not None and t.dim() > 0:
        parts = [torch.empty_like(t) for _ in range(topo.data_parallel_size)]
        dist.all_gather(parts, t.contiguous(), group=topo.dp_group)
        t = torch.cat(parts, dim=0)
    return t.to(device)


def ttol(tensor, pure_local=False, ranks=None):
    """Reference-API shim: tensors are already process-local in this design."""
    return tensor


def tton(tensor, local_only=False, ranks=None):
    return ttol(tensor).detach().cpu().numpy()


def convert_to_distributed_default_setting(t):
    """Reference-API shim (distributed.py:434-447): move a tensor to this rank's device."""
    return t.to(get_device()) if isinstance(t, torch.Tensor) else t


# --------------------------------------------------------------------------------------------------------------
# Placement / SBP vocabulary of the reference (libai/utils/distributed.py:317-393), mapped onto the process-group
# world: a *placement* is "device type + the ranks of the pipeline stage that owns a layer"; an *sbp signature* is the
# pair of strings (data-parallel axis, tensor-parallel axis) that `DistTensorData` already carries
# ("split_<dim>" | "broadcast" | "partial_sum").  Code ported from the reference can keep asking these questions.
# --------------------------------------------------------------------------------------------------------------
class Placement:
    """Device type + global ranks of one pipeline stage (the reference's ``flow.placement`` restricted to what LiBai
    uses it for: "where does layer *i* live")."""

    __slots__ = ("device_type", "ranks", "mesh")

    def __init__(self, device_type: str, ranks):
        self.device_type = device_type
        rows = [list(r) if isinstance(r, (list, tuple)) else [r] for r in ranks]
        self.mesh = tuple(tuple(int(x) for x in row) for row in rows)       # [dp][tp]
        self.ranks = tuple(x for row in self.mesh for x in row)

    def __contains__(self, rank: int) -> bool:
        return int(rank) in self.ranks

    @property
    def is_local(self) -> bool:
        """True when the calling process belongs to this placement."""
        return get_rank() in self.ranks

    @property
    def device(self) -> torch.device:
        """The calling process' device for tensors of this placement."""
        if self.device_type == "cuda":
            return torch.device("cuda", get_local_rank())
        return torch.device(self.device_type)

    def __eq__(self, other):
        return isinstance(other, Placement) and (self.device_type, self.ranks) == (other.device_type, other.ranks)

    def __hash__(self):
        return hash((self.device_type, self.ranks))

    def __repr__(self):
        return f"Placement(type={self.device_type!r}, ranks={list(self.ranks)})"


def get_layer_placement(layer_idx: int, device_type: Optional[str] = None) -> Placement:
    """Placement of layer ``layer_idx`` (negative indices count from the last layer, ``-1`` = last stage)."""
    topo = get_dist_util()
    device_type = topo.device_type if device_type is None else device_type
    if device_type == "cuda" and not torch.cuda.is_available():
        device_type = "cpu"
    return Placement(device_type, topo.get_layer_ranks(layer_idx))


def get_nd_sbp(sbp_list):
    """Trim a 2-entry signature ``[dp_axis, tp_axis]`` to the axes that exist in the current layout: both for dp×tp,
    the first for pure data parallel, the second for pure tensor parallel, ``["broadcast"]`` on a single device."""
    assert isinstance(sbp_list, (list, tuple)) and len(sbp_list) == 2, "a 2-D (data, tensor) signature is expected"
    assert all(isinstance(s, str) and (s in ("broadcast", "partial_sum") or s.startswith("split_")) for s in sbp_list), sbp_list
    topo = get_dist_util()
    if topo.is_data_model_parallel():
        return list(sbp_list)
    if topo.is_data_parallel():
        return list(sbp_list[:1])
    if topo.is_tensor_model_parallel():
        return list(sbp_list[1:])
    return ["broadcast"]


def get_hidden_sbp():
    """Signature of the hidden states between blocks: batch-split over data parallel, replicated over tensor parallel
    (with ``train.dist.sequence_parallel`` the token dimension is additionally sharded over the TP group inside the
    blocks — see parallel/mappings.py)."""
    return get_nd_sbp(["split_0", "broadcast"])


def same_sbp(lhs_sbp, rhs_sbp) -> bool:
    assert len(lhs_sbp) == len(rhs_sbp)
    return all(a == b for a, b in zip(lhs_sbp, rhs_sbp))
