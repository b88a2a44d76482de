"""Symmetric (peer-mapped) device memory for in-kernel NVLink communication.

Native part: ``csrc/symm.cpp`` — ``cudaMalloc`` + CUDA-IPC handle exchange; every rank ends up
with a table of device pointers to all peers' buffers plus a flags region, which the fused
GEMM+collective kernels (``csrc/gemm_sm90.cu``) and the ZeRO-1 reduce-scatter kernel dereference
directly (P2P ld/st over NVSwitch).  Handles travel over the gloo control group.

A :class:`SymmWorkspace` is created lazily per (process group, purpose) and reused; kernels use
monotonically increasing epochs with double-buffered payload so no extra barrier is needed
between consecutive calls (see DESIGN.md §symmetric memory protocol).
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from . import _ext

_WORKSPACES: Dict[Tuple[int, str], "SymmWorkspace"] = {}


def reset() -> None:
    for ws in list(_WORKSPACES.values()) + list(_VMM_WORKSPACES.values()):
        ws.close()
    _WORKSPACES.clear()
    _VMM_WORKSPACES.clear()
    from . import _fused_impl, allreduce, nvls

    allreduce.reset()
    nvls.reset()
    _fused_impl.reset()


def available() -> bool:
    e = _ext.ext()
    return e is not None and hasattr(e, "symm_alloc") and torch.cuda.is_available()


@dataclass
class SymmWorkspace:
    """``nbytes`` of payload + ``nflags`` 32-bit flags on every rank of ``group``; ``ptrs``/``flag_ptrs``
    are device-resident tables (int64) of all ranks' base addresses, indexed by group rank."""

    group: object
    rank: int
    world: int
    nbytes: int
    nflags: int
    handle: int = 0                       # native handle id
    ptrs: Optional[torch.Tensor] = None   # [world] int64 on device
    flag_ptrs: Optional[torch.Tensor] = None
    local_ptr: int = 0
    local_flag_ptr: int = 0
    epoch: Dict[str, int] = field(default_factory=dict)

    def next_epoch(self, key: str) -> int:
        self.epoch[key] = self.epoch.get(key, 0) + 1
        return self.epoch[key]

    def local_tensor(self, offset: int, shape, dtype) -> torch.Tensor:
        """A torch view over this rank's payload (for debugging / eager reads)."""
        return _ext.ext().symm_view(self.handle, int(offset), list(shape), dtype)

    def close(self) -> None:
        if self.handle:
            try:
                _ext.ext().symm_free(self.handle)
            except Exception:
                pass
            self.handle = 0


def _control_group_for(group):
    """gloo group with the same membership as ``group`` for handle exchange."""
    from ..parallel_layers import parallel_state as ps

    ranks = dist.get_process_group_ranks(group)
    key = ("symm_ctl", tuple(ranks))
    cache = getattr(_control_group_for, "_cache", {})
    _control_group_for._cache = cache
    if key not in cache:
        # every rank of the WORLD must participate in new_group; callers guarantee collective use
        cache[key] = None
    return ranks


def get_workspace(group, purpose: str, nbytes: int, nflags: int = 4096) -> SymmWorkspace:
    """Collective over ``group``: allocate (or fetch) a symmetric workspace of at least ``nbytes``."""
    key = (id(group), purpose)
    ws = _WORKSPACES.get(key)
    if ws is not None and ws.nbytes >= nbytes and ws.nflags >= nflags:
        return ws
    if ws is not None:
        ws.close()
    e = _ext.ext()
    assert e is not None, "symmetric memory needs the CUDA extension"
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    nbytes = (int(nbytes) + (1 << 21) - 1) & ~((1 << 21) - 1)
    handle, ipc_payload, ipc_flags = e.symm_alloc(nbytes, int(nflags))
    gathered: List[Optional[tuple]] = [None] * world
    dist.all_gather_object(gathered, (os.getpid(), ipc_payload, ipc_flags), group=group)
    ptrs, flag_ptrs = e.symm_open(handle, rank, [g[1] for g in gathered], [g[2] for g in gathered])
    dev = torch.device("cuda", torch.cuda.current_device())
    ws = SymmWorkspace(
        group=group, rank=rank, world=world, nbytes=nbytes, nflags=nflags, handle=handle,
        ptrs=torch.tensor(ptrs, dtype=torch.int64, device=dev),
        flag_ptrs=torch.tensor(flag_ptrs, dtype=torch.int64, device=dev),
        local_ptr=ptrs[rank], local_flag_ptr=flag_ptrs[rank],
    )
    # nobody may touch a peer buffer before every rank has mapped everything
    torch.cuda.synchronize()
    dist.barrier(group=group)
    _WORKSPACES[key] = ws
    return ws


# ------------------------------------------------------------------------------------------------------------------
# v2: VMM allocations shared by POSIX fd + NVLS multicast mapping (csrc/symm_vmm.cpp)
_VMM_WORKSPACES: Dict[Tuple[int, str], "VmmWorkspace"] = {}


@dataclass
class VmmWorkspace:
    """One ``cuMemCreate`` allocation per rank of ``group``, every peer's allocation mapped locally (``ptrs``: device table
    of unicast base addresses) and — if the fabric supports it — bound to one NVLS multicast object (``mc_ptr``: a store
    to ``mc_ptr + off`` lands at ``off`` in every rank's allocation; a ``multimem.ld_reduce`` returns the sum over ranks).
    ``mc_ptr == 0`` means unicast only (single-device loopback tests, no NVSwitch multicast): kernels then use ``ptrs``."""

    group: object
    rank: int
    world: int
    nbytes: int
    handle: int = 0
    ptrs: Optional[torch.Tensor] = None
    ptr_list: Optional[List[int]] = None
    local_ptr: int = 0
    mc_ptr: int = 0
    mc_error: str = ""

    @property
    def has_multicast(self) -> bool:
        return self.mc_ptr != 0

    def local_tensor(self, offset: int, shape, dtype) -> torch.Tensor:
        return _ext.ext().vmm_view(self.handle, int(offset), list(shape), dtype)

    def close(self) -> None:
        if self.handle:
            try:
                _ext.ext().vmm_free(self.handle)
            except Exception:
                pass
            self.handle = 0


def vmm_available() -> bool:
    e = _ext.ext()
    return e is not None and hasattr(e, "vmm_begin") and torch.cuda.is_available()


def get_vmm_workspace(group, purpose: str, nbytes: int, multicast: Optional[bool] = None) -> VmmWorkspace:
    """Collective over ``group``: allocate (or fetch) a VMM symmetric workspace of at least ``nbytes`` bytes.  The phases of
    the handle exchange are separated by host barriers over ``group``'s control plane; a multicast failure on ANY rank
    makes every rank fall back to unicast together (the reason is kept in ``mc_error`` and logged once)."""
    key = (id(group), purpose)
    ws = _VMM_WORKSPACES.get(key)
    if ws is not None and ws.nbytes >= nbytes:
        return ws
    if ws is not None:
        _sync()
        dist.barrier(group=group)
        ws.close()
    e = _ext.ext()
    assert e is not None and hasattr(e, "vmm_begin"), "VMM symmetric memory needs the CUDA extension"
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    want_mc = (os.environ.get("NXD_NVLS", "1") != "0") if multicast is None else bool(multicast)
    handle, sock, mc_ok, size = e.vmm_begin(int(nbytes), rank, world, want_mc)
    infos: List[Optional[tuple]] = [None] * world
    dist.all_gather_object(infos, (sock, bool(mc_ok), _device_uuid()), group=group)
    same_device = len({i[2] for i in infos}) < world          # two ranks on one GPU (loopback tests): no multicast team
    use_mc = all(i[1] for i in infos) and not same_device and world > 1
    err = e.vmm_send(handle, [i[0] for i in infos], use_mc)
    err = e.vmm_recv(handle) or err
    oks: List[Optional[tuple]] = [None] * world
    dist.all_gather_object(oks, (err == "", err), group=group)      # doubles as the barrier: every device added
    everyone = use_mc and all(o[0] for o in oks)
    err2 = e.vmm_bind(handle, everyone) if use_mc else ""
    oks2: List[Optional[tuple]] = [None] * world
    dist.all_gather_object(oks2, (err2 == "", err2), group=group)
    mc_everywhere = everyone and all(o[0] for o in oks2)
    ptrs, mc_ptr, size = e.vmm_ptrs(handle, mc_everywhere)
    reasons = [o[1] for o in oks + oks2 if o[1]]
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    ws = VmmWorkspace(group=group, rank=rank, world=world, nbytes=int(size), handle=handle,
                      ptrs=torch.tensor(ptrs, dtype=torch.int64, device=dev), ptr_list=list(ptrs), local_ptr=ptrs[rank],
                      mc_ptr=int(mc_ptr), mc_error="; ".join(sorted(set(reasons))))
    if want_mc and not ws.has_multicast and world > 1:
        from ..utils.logger import get_logger

        why = ws.mc_error or ("ranks share a device" if same_device else "device reports no multicast support")
        get_logger("symm").warning("NVLS multicast unavailable for workspace '%s' (%s): using unicast peer accesses", purpose, why)
    _sync()
    dist.barrier(group=group)
    _VMM_WORKSPACES[key] = ws
    return ws


def _sync() -> None:
    if torch.cuda.is_available():
        torch.cuda.synchronize()


def _device_uuid() -> str:
    try:
        return str(torch.cuda.get_device_properties(torch.cuda.current_device()).uuid)
    except Exception:                                    # noqa: BLE001 - no uuid attribute / no CUDA (host-logic tests)
        return f"dev{os.environ.get('LOCAL_RANK', os.environ.get('RANK', '0'))}"
