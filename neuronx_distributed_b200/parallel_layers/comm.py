"""Collective wrappers used by the cold paths and the ``nccl`` (library) backend.

Same surface as reference ``parallel_layers/comm.py:124-220`` (``all_reduce`` accepting a tensor
*bucket*, ``all_gather``/``reduce_scatter`` along an arbitrary dim).  On CUDA these are NCCL
calls issued through ``torch.distributed``; in CPU mode they run on gloo, which lacks
reduce-scatter, so that one is emulated (all-reduce + local slice — simpler and deterministic
compared with the reference's reduce-to-root + scatter :82-121).

The hot tensor-parallel paths do NOT go through this file on H100: they use the fused
GEMM+collective kernels in ``ops/tp_fused.py``.
"""
from __future__ import annotations

import os
from typing import Optional, Sequence, Union

import torch
import torch.distributed as dist

from ..utils.plan_registry import plan_op
from . import parallel_state as ps

_REDUCE_OPS = {
    "sum": dist.ReduceOp.SUM,
    "max": dist.ReduceOp.MAX,
    "min": dist.ReduceOp.MIN,
    "avg": dist.ReduceOp.SUM,  # divided afterwards: gloo has no AVG
    "product": dist.ReduceOp.PRODUCT,
}


def _tp(group):
    return group if group is not None else ps.get_tensor_model_parallel_group()


def _is_gloo(group) -> bool:
    try:
        return dist.get_backend(group) == "gloo"
    except Exception:
        return False


def group_size(group=None) -> int:
    return dist.get_world_size(_tp(group))


def group_rank(group=None) -> int:
    return dist.get_rank(_tp(group))


@plan_op("comm.all_reduce")
def all_reduce(
    tensors: Union[torch.Tensor, Sequence[torch.Tensor]],
    op: str = "sum",
    group=None,
    async_op: bool = False,
):
    """In-place all-reduce of a tensor or a bucket (list) of tensors.

    A bucket is flattened into one buffer so a single collective is launched
    (reference comm.py:200-220 coalesces likewise)."""
    group = _tp(group)
    rop = _REDUCE_OPS[op]
    n = dist.get_world_size(group)
    if isinstance(tensors, torch.Tensor):
        if n == 1:
            return None if async_op else tensors
        if op == "sum" and not async_op and tensors.is_cuda:
            from ..ops import allreduce as _oneshot     # small tensors: one-shot peer-memory kernel instead of NCCL

            red = _oneshot.all_reduce_sum(tensors, group)
            if red is not None:
                tensors.copy_(red)
                return tensors
        work = dist.all_reduce(tensors, op=rop, group=group, async_op=async_op)
        if op == "avg":
            assert not async_op
            tensors.div_(n)
        return work if async_op else tensors
    tensors = list(tensors)
    if not tensors or n == 1:
        return tensors
    assert not async_op, "bucketed all_reduce is synchronous"
    flat = torch.cat([t.reshape(-1) for t in tensors])
    dist.all_reduce(flat, op=rop, group=group)
    if op == "avg":
        flat.div_(n)
    off = 0
    for t in tensors:
        t.copy_(flat[off : off + t.numel()].view_as(t))
        off += t.numel()
    return tensors


@plan_op("comm.all_gather", pure=True)
def all_gather(x: torch.Tensor, dim: int = 0, group=None) -> torch.Tensor:
    """Concatenate every rank's ``x`` along ``dim``."""
    group = _tp(group)
    n = dist.get_world_size(group)
    if n == 1:
        return x
    if x.dim() == 0:
        x = x.view(1)
    dim = dim % x.dim()
    xc = x.contiguous()
    out = torch.empty((n,) + tuple(xc.shape), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(out.view(-1, *xc.shape[1:]), xc, group=group)
    if dim == 0:
        return out.view(n * xc.shape[0], *xc.shape[1:])
    # [n, d0, ..., dk, ...] -> move n in front of dk and merge
    out = out.movedim(0, dim)  # [..., n, dk, ...]
    shape = list(xc.shape)
    shape[dim] = n * shape[dim]
    return out.reshape(shape)


@plan_op("comm.reduce_scatter", pure=True)
def reduce_scatter(x: torch.Tensor, dim: int = 0, group=None, op: str = "sum") -> torch.Tensor:
    """Sum ``x`` over the group and return this rank's 1/n slice along ``dim``."""
    group = _tp(group)
    n = dist.get_world_size(group)
    if n == 1:
        return x
    dim = dim % x.dim()
    assert x.shape[dim] % n == 0, f"dim {dim} of {tuple(x.shape)} not divisible by group size {n}"
    r = dist.get_rank(group)
    if _is_gloo(group):
        full = x.contiguous().clone() if not x.is_cuda else x.detach().cpu()    # gloo control plane next to CUDA data (loopback)
        dist.all_reduce(full, op=_REDUCE_OPS[op], group=group)
        out = full.chunk(n, dim=dim)[r].contiguous().to(x.device)
    else:
        xin = x if dim == 0 else x.movedim(dim, 0)
        xin = xin.contiguous()
        out = torch.empty((xin.shape[0] // n,) + tuple(xin.shape[1:]), dtype=x.dtype, device=x.device)
        dist.reduce_scatter_tensor(out, xin, op=_REDUCE_OPS[op], group=group)
        if dim != 0:
            out = out.movedim(0, dim).contiguous()
    if op == "avg":
        out = out / n
    return out


@plan_op("comm.all_to_all", pure=True)
def all_to_all(x: torch.Tensor, split_dim: int, concat_dim: int, group=None) -> torch.Tensor:
    """Split ``x`` into n pieces along ``split_dim``, exchange, concatenate along ``concat_dim``
    (semantics of ``xm.all_to_all`` used at reference mappings.py:160-172)."""
    group = group if group is not None else ps.get_expert_model_parallel_group()
    n = dist.get_world_size(group)
    if n == 1:
        return x
    if x.is_cuda and x.shape[split_dim] % n == 0 and os.environ.get("NXD_NVLS_A2A", "0") == "1":
        from ..ops import nvls as _nvls

        # EP dispatch / combine over peer memory (opt-in NXD_NVLS_A2A=1): one publish + one pull kernel instead of NCCL
        send = x.movedim(split_dim, 0).contiguous() if split_dim != 0 else x.contiguous()
        if _nvls.all_to_all_eligible(send, group):
            recv = _nvls.all_to_all(send, group)                       # [n * c, …rest] with the split dim in front
            chunks = recv.chunk(n, dim=0)
            if split_dim != 0:
                chunks = [c.movedim(0, split_dim) for c in chunks]
            return torch.cat(chunks, dim=concat_dim)
    pieces = [p.contiguous() for p in x.chunk(n, dim=split_dim)]
    outs = [torch.empty_like(pieces[0]) for _ in range(n)]
    if _is_gloo(group):
        # gloo all_to_all support is uneven across versions → use all_gather of the stacked pieces
        stacked = torch.stack(pieces)  # [n, ...]
        gathered = [torch.empty_like(stacked) for _ in range(n)]
        dist.all_gather(gathered, stacked, group=group)
        r = dist.get_rank(group)
        outs = [gathered[src][r] for src in range(n)]
    else:
        dist.all_to_all(outs, pieces, group=group)
    return torch.cat(outs, dim=concat_dim)


@plan_op("comm.broadcast")
def broadcast(x: torch.Tensor, src: int, group=None) -> torch.Tensor:
    group = _tp(group)
    if dist.get_world_size(group) > 1:
        dist.broadcast(x, src=src, group=group)
    return x


def barrier(group=None) -> None:
    if dist.is_initialized():
        dist.barrier(group=group)


def send(x: torch.Tensor, dst: int, group=None):
    return dist.send(x.contiguous(), dst=dst, group=group)


def recv(x: torch.Tensor, src: int, group=None):
    return dist.recv(x, src=src, group=group)


def gloo_reduce_scatter(output: torch.Tensor, input: torch.Tensor, op="sum", group=None, async_op: bool = False):  # noqa: A002
    """gloo has no reduce-scatter: reduce to the group's first rank, then scatter equal chunks of dim 0 into ``output``
    (reference comm.py:82-130).  ``reduce_scatter`` above uses all-reduce + slice instead (one collective, no root
    hot-spot); this form is kept for callers that need the out-parameter signature."""
    group = _tp(group)
    n = dist.get_world_size(group)
    ranks = dist.get_process_group_ranks(group)
    red = _REDUCE_OPS[op] if isinstance(op, str) else op
    buf = input.contiguous().clone()
    dist.reduce(buf, dst=ranks[0], op=red, group=group)
    chunks = [c.contiguous() for c in buf.chunk(n, dim=0)] if dist.get_rank() == ranks[0] else None
    dist.scatter(output, chunks, src=ranks[0], group=group)
    return output


def cpu_reduce_scatter(reduce_type: str, input: torch.Tensor, scale: float = 1, scatter_dim: int = 0, shard_count=None,  # noqa: A002
                       groups=None, output: Optional[torch.Tensor] = None, pin_layout: bool = True) -> torch.Tensor:
    """``xm.reduce_scatter`` signature on CPU tensors (reference comm.py:32-79)."""
    group = _tp(groups)
    n = dist.get_world_size(group)
    assert shard_count is None or shard_count == n, f"shard_count {shard_count} must equal the group size {n}"
    res = reduce_scatter(input, scatter_dim, group, reduce_type if reduce_type in _REDUCE_OPS else "sum")
    if scale != 1:
        res = res * scale
    if output is not None:
        output.copy_(res)
        return output
    return res
