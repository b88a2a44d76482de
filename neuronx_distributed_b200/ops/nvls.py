"""Stand-alone collectives on the NVLS symmetric region (``csrc/nvls_coll.cu``): in-switch all-reduce
(``multimem.ld_reduce``), multicast all-gather (``multimem.st``) and reduce-scatter — one kernel each, CUDA-graph
capturable (the call counter lives in device memory), no NCCL call.  Without a multicast mapping (two ranks on one GPU in
the loopback tests, fabrics without NVLS) the same kernels run over unicast peer pointers.

Used by ``parallel_layers.comm.all_reduce`` for latency-bound tensors (decode-time RowParallelLinear /
ParallelEmbedding outputs without sequence parallel — reference layers.py:1040-1043, mappings.py:196-211) and by
``tools/nvls_probe.py`` to measure the link bandwidth.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch
import torch.distributed as dist

from ..utils.plan_registry import plan_op
from . import _ext, symm

_FLAG_BYTES = 4096                     # 1024 per-CTA barrier counters
_STATE: Dict[tuple, "_Coll"] = {}


class _Coll:
    def __init__(self, group, kind: str, half_bytes: int):
        self.group = group
        self.half_bytes = int(half_bytes)
        self.ws = symm.get_vmm_workspace(group, f"nvls_{kind}", _FLAG_BYTES + 2 * self.half_bytes)
        dev = torch.device("cuda", torch.cuda.current_device())
        # the device-side call / barrier counters belong to the REGION (its flag words count the same events): when a larger
        # request is served by the same (already big enough) region, the counters must carry over, not restart at zero
        st = getattr(self.ws, "_coll_state", None)
        if st is None:
            st = self.ws._coll_state = torch.zeros(2 + 1024, dtype=torch.int32, device=dev)
        self.state = st

    @property
    def args(self):
        ws = self.ws
        return (ws.ptrs, ws.mc_ptr, ws.local_ptr, 0, _FLAG_BYTES, self.half_bytes, self.state, ws.rank, ws.world)


def _coll(group, kind: str, need_bytes: int, default_mb: int) -> _Coll:
    key = (id(group), kind)
    c = _STATE.get(key)
    if c is None or c.half_bytes < need_bytes:
        half = max(int(need_bytes), default_mb << 20)
        half = (half + (1 << 21) - 1) & ~((1 << 21) - 1)
        c = _STATE[key] = _Coll(group, kind, half)
    return c


def reset() -> None:
    _STATE.clear()


def available(group=None) -> bool:
    e = _ext.ext()
    return e is not None and hasattr(e, "nvls_allreduce") and symm.vmm_available()


def has_multicast(group) -> bool:
    """True when ``group``'s NVLS workspace got a multicast mapping (allocates the all-reduce workspace on first use)."""
    return _coll(group, "ar", 0, int(os.environ.get("NXD_NVLS_AR_MAX_MB", "8"))).ws.has_multicast


@plan_op("nvls.all_reduce_sum", pure=True)
def all_reduce_sum(x: torch.Tensor, group, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``sum_over_ranks(x) (+ residual)`` as a new tensor.  bf16 / fp32, contiguous, bytes % 16 == 0."""
    nbytes = x.numel() * x.element_size()
    c = _coll(group, "ar", nbytes, int(os.environ.get("NXD_NVLS_AR_MAX_MB", "8")))
    _ext.count_launch()
    return _ext.ext().nvls_allreduce(x, residual, *c.args)


@plan_op("nvls.gemv_all_reduce", pure=True)
def gemv_all_reduce(x: torch.Tensor, weight: torch.Tensor, group, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``sum_over_ranks(x @ weightᵀ) (+ residual)`` for ``x`` [M<=8, K] bf16, ``weight`` [N, K] bf16 in ONE kernel (decode-time
    RowParallelLinear): the GEMV's fp32 partials are reduced in the switch, never rounded to bf16 in between."""
    M, N = x.shape[0], weight.shape[0]
    c = _coll(group, "gemv_ar", M * N * 4, 1)
    _ext.count_launch()
    return _ext.ext().gemv_allreduce(x, weight, residual, *c.args)


def gemv_all_reduce_eligible(x2d: torch.Tensor, weight: torch.Tensor) -> bool:
    return (x2d.is_cuda and x2d.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and x2d.shape[0] <= 8
            and weight.shape[0] % 8 == 0 and weight.shape[1] % 8 == 0 and x2d.is_contiguous() and weight.is_contiguous()
            and available() and os.environ.get("NXD_GEMV_AR", "1") == "1")


@plan_op("nvls.all_gather", pure=True)
def all_gather(x: torch.Tensor, group, ctas: int = 32) -> torch.Tensor:
    """Concatenation over ranks along dim 0 (the shard is multicast into every rank's symmetric buffer, then copied out)."""
    world = dist.get_world_size(group)
    nbytes = x.numel() * x.element_size()
    c = _coll(group, "ag", nbytes * world, 64)
    out = torch.empty((world * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    _ext.count_launch()
    _ext.ext().nvls_all_gather(x.contiguous(), out, *c.args, int(ctas))
    return out


@plan_op("nvls.reduce_scatter_sum", pure=True)
def reduce_scatter_sum(x: torch.Tensor, group, ctas: int = 32) -> torch.Tensor:
    """``x`` = [world * n, ...] on every rank → this rank's [n, ...] chunk of the sum."""
    world = dist.get_world_size(group)
    nbytes = x.numel() * x.element_size()
    c = _coll(group, "rs", nbytes, 64)
    _ext.count_launch()
    out = _ext.ext().nvls_reduce_scatter(x.contiguous(), *c.args, int(ctas))
    return out.view((x.shape[0] // world,) + tuple(x.shape[1:]))


@plan_op("nvls.embedding_gather", pure=True)
def embedding_gather(ids: torch.Tensor, table: torch.Tensor, group, ctas: int = 64) -> torch.Tensor:
    """Rows ``ids`` (GLOBAL vocabulary ids, any shape) of a vocabulary-sharded table (``table`` = this rank's equal-sized shard
    ``[V/world, H]``) → ``[*ids.shape, H]``.  CUDA: every rank publishes its shard in its symmetric slot and pulls the rows it
    needs straight from the owners over NVLink (``csrc/nvls_coll.cu`` ``nvls_publish_kernel`` + ``peer_row_gather_kernel``) — no
    masked partial lookups, no reduction.  Ids outside the vocabulary give zero rows.  CPU: all-gather of the shards + index."""
    world = dist.get_world_size(group)
    flat = ids.reshape(-1).long().contiguous()
    if table.is_cuda and _ext.use_cuda(table) and hasattr(_ext.ext(), "nvls_embedding_gather") and available():
        nbytes = table.numel() * table.element_size()
        c = _coll(group, "emb", nbytes, 64)
        _ext.count_launch(2)
        out = _ext.ext().nvls_embedding_gather(table.contiguous(), flat, *c.args, int(ctas))
    else:
        from ..parallel_layers import comm

        full = comm.all_gather(table.contiguous(), dim=0, group=group) if world > 1 else table
        ok = (flat >= 0) & (flat < full.shape[0])
        out = full[torch.where(ok, flat, torch.zeros_like(flat))] * ok.unsqueeze(-1).to(full.dtype)
    return out.view(*ids.shape, table.shape[1])


def embedding_gather_eligible(table: torch.Tensor) -> bool:
    return (table.is_cuda and table.dtype in (torch.bfloat16, torch.float32, torch.float16) and table.is_contiguous()
            and (table.shape[1] * table.element_size()) % 16 == 0 and available())


@plan_op("nvls.all_to_all", pure=True)
def all_to_all(x: torch.Tensor, group, ctas: int = 64) -> torch.Tensor:
    """Equal-split all-to-all along dim 0 (``x`` = ``[world * n, …]``: rows ``[p*n, (p+1)*n)`` go to rank ``p``; the result holds
    at the same place what rank ``p`` sent here) over peer memory: publish the send buffer in the symmetric slot, pull the own
    chunk of every peer (``csrc/nvls_coll.cu``).  No NCCL, CUDA-graph capturable."""
    nbytes = x.numel() * x.element_size()
    c = _coll(group, "a2a", nbytes, 64)
    _ext.count_launch(2)
    return _ext.ext().nvls_all_to_all(x.contiguous(), *c.args, int(ctas))


def all_to_all_eligible(x: torch.Tensor, group) -> bool:
    if os.environ.get("NXD_NVLS_A2A", "0") != "1":             # opt-in until the kernels have run on hardware
        return False
    world = dist.get_world_size(group)
    return (x.is_cuda and x.dim() >= 1 and x.shape[0] % world == 0 and (x.numel() * x.element_size()) % (16 * world) == 0
            and x.numel() > 0 and available() and hasattr(_ext.ext(), "nvls_all_to_all"))


def publish(x: torch.Tensor, group, ctas: int = 64):
    """Make ``x`` readable by every rank of ``group``: returns one tensor per rank, entry ``p`` viewing rank ``p``'s ``x``.
    CUDA: ``x`` is copied into this rank's symmetric slot (halves alternate per call), all ranks meet, and the returned
    tensors are VIEWS of the peers' slots — a kernel that takes them (e.g. flash attention, through TMA) loads straight over
    NVLink.  They stay valid until this rank's NEXT ``publish`` on the same group (once a rank has arrived there its peers may
    run one call further and rewrite this half — `tools/sim_nvls_protocol.py::simulate_publish` shows the interleaving).  The half is chosen on the host (the
    addresses are needed to build the views), so a call is not CUDA-graph capturable.  CPU: an all-gather."""
    world = dist.get_world_size(group)
    if not (x.is_cuda and _ext.use_cuda(x) and hasattr(_ext.ext(), "nvls_publish") and available()):
        from ..parallel_layers import comm

        full = comm.all_gather(x.contiguous().unsqueeze(0), dim=0, group=group) if world > 1 else x.unsqueeze(0)
        return list(full.unbind(0))
    nbytes = x.numel() * x.element_size()
    c = _coll(group, "publish", nbytes, 64)
    calls = getattr(c, "calls", 0)
    c.calls = calls + 1
    parity = calls & 1
    _ext.count_launch()
    _ext.ext().nvls_publish(x.contiguous(), *c.args, parity, int(ctas))
    off = _FLAG_BYTES + parity * c.half_bytes
    return [_ext.ext().ptr_view(int(p) + off, list(x.shape), x.dtype) for p in c.ws.ptr_list]
