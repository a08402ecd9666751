"""Symmetric (peer-mapped) device memory: the substrate of the in-kernel NVLink collectives.

Each rank of a process group allocates the same number of bytes with ``cudaMalloc`` (outside the
caching allocator), the 64-byte CUDA IPC handles are exchanged through ``torch.distributed``, and
every rank maps all peers' buffers.  Kernels receive the table of peer pointers and use plain
``ld/st/red`` on them – the traffic goes over NVLink 5 / NVSwitch. 
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from libai_b200.ops import load_ext


class SymmetricBuffer:
    """``nbytes`` of zero-initialised device memory mapped by every rank of ``group``."""

    def __init__(self, nbytes: int, group=None, tag: str = "", multicast: bool = False):
        ext = load_ext()
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.nbytes = int((nbytes + 255) // 256 * 256)
        self.tag = tag
        self.mc_ptr = 0          # NVSwitch multicast address of the buffer (0 = none: unicast peer pointers only)
        self._torch_handle = None
        if multicast and self.world > 1 and self._init_multicast():
            return
        self.local = ext.symm_alloc(self.nbytes)  # uint8 tensor owning the allocation
        if self.world == 1:
            self.ptrs = [self.local.data_ptr()]
            return
        handle = ext.symm_export(self.local)
        payload = bytes(handle.numpy().tobytes())
        gathered: List[Optional[bytes]] = [None] * self.world
        dist.all_gather_object(gathered, payload, group=group)
        self.ptrs = []
        for r, h in enumerate(gathered):
            if r == self.rank:
                self.ptrs.append(self.local.data_ptr())
            else:
                ht = torch.frombuffer(bytearray(h), dtype=torch.uint8)
                self.ptrs.append(int(ext.symm_open(ht)))
        dist.barrier(group=group)

    def _init_multicast(self) -> bool:
        """Allocate through PyTorch's symmetric-memory allocator (CUDA VMM: ``cuMemCreate`` + file-descriptor exchange +
        ``cuMulticastBindMem``), which hands back the peers' unicast addresses AND the multicast address of the NVSwitch
        multicast object the buffers are bound to.  Only the plumbing is PyTorch's; the kernels that use the addresses
        (``multimem.ld_reduce`` / ``multimem.st``, csrc/comm_kernels.cu) are ours.  Every rank takes the same decision:
        the outcome is agreed with a MIN all-reduce, a rank-local failure falls back to the CUDA-IPC path everywhere."""
        ok, t, hdl = 1, None, None
        try:
            import torch.distributed._symmetric_memory as tsm

            dev = torch.device("cuda", torch.cuda.current_device())
            group = self.group if self.group is not None else dist.group.WORLD
            try:
                tsm.enable_symm_mem_for_group(group.group_name)
            except Exception:   # noqa: BLE001 - newer releases enable groups implicitly
                pass
            t = tsm.empty(self.nbytes, dtype=torch.uint8, device=dev)
            hdl = tsm.rendezvous(t, group)
            if not (getattr(hdl, "has_multicast_support", False) or int(getattr(hdl, "multicast_ptr", 0)) != 0):
                ok = 0
            if int(getattr(hdl, "multicast_ptr", 0)) == 0:
                ok = 0
        except Exception as e:   # noqa: BLE001
            import logging

            logging.getLogger(__name__).info("NVLS multicast unavailable for %s (%s: %s)", self.tag, type(e).__name__, str(e)[:200])
            ok = 0
        flag = torch.tensor([ok], device="cuda")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            return False
        t.zero_()
        torch.cuda.synchronize()
        self.local = t
        self._torch_handle = hdl
        self.ptrs = [int(p) for p in hdl.buffer_ptrs]
        self.ptrs[self.rank] = t.data_ptr()
        self.mc_ptr = int(hdl.multicast_ptr)
        dist.barrier(group=self.group)
        return True

    def close(self) -> None:
        """Unmap the peers' allocations and free the local one.  Collective over ``group``: nobody frees memory a
        peer may still have mapped (a later ``cudaMalloc`` can hand the same range out again, and re-opening its IPC
        handle while the stale mapping exists fails with "resource already mapped")."""
        if self.local is None:
            return
        ext = load_ext()
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(group=self.group)           # every rank's kernels on these buffers have retired
            if self._torch_handle is None:
                for r, p in enumerate(self.ptrs):
                    if r != self.rank:
                        ext.symm_close(int(p))
            dist.barrier(group=self.group)           # every mapping is gone before any owner frees
        self.ptrs = []
        self.local = None
        self._torch_handle = None
        self.mc_ptr = 0

    def view(self, dtype: torch.dtype, shape, offset_bytes: int = 0) -> torch.Tensor:
        """Typed view of the *local* buffer."""
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty((), dtype=dtype).element_size()
        return self.local[offset_bytes : offset_bytes + nb].view(dtype).view(*shape)

    def peer_ptrs(self, offset_bytes: int = 0) -> List[int]:
        return [p + offset_bytes for p in self.ptrs]


class CommWorkspace:
    """Per-group bookkeeping for the fused collectives: handshake flags, arrival counters, epochs and
    shape-keyed data buffers (all symmetric)."""

    FLAG_BYTES = 1 << 16

    def __init__(self, group):
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.flags = SymmetricBuffer(self.FLAG_BYTES, group, "flags")
        self._flag_cursor = 64 * 4 * self.world  # first slots are reserved for the handshake rows
        self.epoch = 0
        self.device = self.flags.local.device
        self.done_counter = torch.zeros(4, dtype=torch.int32, device=self.device)
        self._bufs: Dict[Tuple, object] = {}

    def next_epoch(self) -> int:
        self.epoch += 1
        return self.epoch

    def alloc_flags(self, n_words: int) -> int:
        """Reserve ``n_words`` uint32 counters in the symmetric flag buffer; returns the byte offset
        (identical on every rank because all ranks allocate in the same order)."""
        off = self._flag_cursor
        self._flag_cursor += (n_words * 4 + 63) // 64 * 64
        assert self._flag_cursor <= self.FLAG_BYTES, "symmetric flag buffer exhausted"
        return off

    def buffer(self, key: Tuple, nbytes: int, multicast: bool = False) -> SymmetricBuffer:
        if key not in self._bufs:
            self._bufs[key] = SymmetricBuffer(nbytes, self.group, str(key), multicast=multicast)
        return self._bufs[key]

    def close(self) -> None:
        """Release every buffer of this workspace (collective; same order on every rank of the group)."""
        for key in list(self._bufs):
            buf = self._bufs.pop(key)
            if isinstance(buf, SymmetricBuffer):
                buf.close()
        self.flags.close()


_WORKSPACES: Dict[int, CommWorkspace] = {}


def get_workspace(group) -> CommWorkspace:
    key = id(group)
    if key not in _WORKSPACES:
        _WORKSPACES[key] = CommWorkspace(group)
    return _WORKSPACES[key]


def release_workspaces() -> None:
    """Tear down every workspace (before the process groups they belong to are destroyed or re-made).  Must be called
    by all ranks at the same point; objects still holding views of the buffers must be dropped first."""
    for key in list(_WORKSPACES):
        _WORKSPACES.pop(key).close()
