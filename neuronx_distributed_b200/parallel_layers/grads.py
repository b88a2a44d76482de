"""Gradient norm / clipping and data-parallel gradient reduction.

Capability parity with reference ``parallel_layers/grads.py`` (``get_grad_norm`` :41-189,
``clip_grad_norm`` :192, ``clip_grads_with_norm`` :238-256, ``bucket_allreduce_gradients``
:259-327, ``allreduce_sequence_parallel_gradients`` :330-346,
``allreduce_context_parallel_gradients`` :348-366).

H100 design: squared norms are produced by ONE multi-tensor kernel launch
(``ops.optim.multi_tensor_sq_norm`` → a single fp32 scalar on device) instead of a python loop of
``torch.norm`` calls, the scalar all-reduces stay on device (no host sync; the clip coefficient is
applied with a device-side ``clamp`` exactly as the reference's ``torch.where(coeff<1)`` trick),
and SP/CP parameter-gradient all-reduces are coalesced into one bucket per dtype.
"""
from __future__ import annotations

import os
from typing import Dict, Iterable, List, Optional, Sequence, Union

import torch

from ..utils.logger import get_logger
from . import comm
from . import parallel_state as ps
from .utils import param_is_not_shared

logger = get_logger()
_ALLREDUCE_BUCKET_CAP_MB = 512


def _is_ep(obj) -> bool:
    return bool(getattr(obj, "expert_model_parallel", False))


def _sq_norm(tensors: Sequence[torch.Tensor], device) -> torch.Tensor:
    from .. import ops

    if not tensors:
        return torch.zeros((), dtype=torch.float32, device=device)
    return ops.optim.multi_tensor_sq_norm(list(tensors))


def _p_norm_pow(tensors: Sequence[torch.Tensor], p: float, device) -> torch.Tensor:
    if p == 2:
        return _sq_norm(tensors, device)
    total = torch.zeros((), dtype=torch.float32, device=device)
    for t in tensors:
        total = total + torch.norm(t.float(), p) ** p
    return total


def get_grad_norm(
    parameters: Union[Iterable[torch.Tensor], torch.Tensor],
    norm_type: Union[float, int] = 2,
    zero1_optimizer: bool = False,
    zero1_optimizer_groups: Optional[List[List[int]]] = None,
    force_spmd: bool = True,
    zero1_group=None,
) -> torch.Tensor:
    """Global p-norm of the gradients of ``parameters`` across TP / EP / PP (and ZeRO shards).

    Tensor-parallel *duplicates* (replicated params such as norms) are counted once: with
    ``force_spmd`` every rank contributes duplicated grads scaled by 1/tp (same program on all
    ranks), otherwise only tp-rank 0 contributes.  ``shared`` (tied across PP stages) params
    are counted only where ``param.shared`` is False.  Expert-parallel params get their own
    accumulator reduced over the EP group.
    """
    params = [parameters] if isinstance(parameters, torch.Tensor) else list(parameters)
    if zero1_optimizer_groups is not None and not zero1_optimizer:
        raise ValueError("zero1_optimizer_groups given while zero1_optimizer is False")
    if not params:
        return torch.zeros((), dtype=torch.float32)
    device = params[0].device
    norm_type = float(norm_type)
    is_inf = norm_type == float("inf")
    if is_inf:
        force_spmd = True
    tp, ep, pp = (
        ps.get_tensor_model_parallel_size(),
        ps.get_expert_model_parallel_size(),
        ps.get_pipeline_model_parallel_size(),
    )
    tp_rank = ps.get_tensor_model_parallel_rank()

    sharded, duplicated, ep_sharded, ep_duplicated = [], [], [], []
    for p in params:
        g = p.grad if p.grad is not None else getattr(p, "main_grad", None)
        if g is None or not param_is_not_shared(p):
            continue
        is_dup = not getattr(p, "tensor_model_parallel", False)
        if _is_ep(p):
            (ep_duplicated if is_dup else ep_sharded).append(g.detach())
        else:
            (duplicated if is_dup else sharded).append(g.detach())

    def _acc(shard_list, dup_list):
        if is_inf:
            vals = [t.abs().max().float() for t in shard_list + dup_list]
            return torch.stack(vals).max() if vals else torch.zeros((), dtype=torch.float32, device=device)
        total = _p_norm_pow(shard_list, norm_type, device)
        if dup_list:
            if force_spmd:
                total = total + _p_norm_pow(dup_list, norm_type, device) / tp
            elif tp_rank == 0:
                total = total + _p_norm_pow(dup_list, norm_type, device)
        return total

    total = _acc(sharded, duplicated)
    ep_total = _acc(ep_sharded, ep_duplicated)
    op = "max" if is_inf else "sum"

    if zero1_optimizer and zero1_optimizer_groups is None and zero1_group is None:
        # grads are ZeRO shards: everything lives somewhere in the world exactly once
        comm.all_reduce(total, op=op, group=ps.get_world_group())
        if ep > 1:
            comm.all_reduce(ep_total, op=op, group=ps.get_world_group())
            total = torch.maximum(total, ep_total) if is_inf else total + ep_total
    else:
        if ep > 1:
            comm.all_reduce(ep_total, op=op, group=ps.get_expert_model_parallel_group())
        total = torch.maximum(total, ep_total) if is_inf else total + ep_total
        if tp > 1:
            comm.all_reduce(total, op=op, group=ps.get_tensor_model_parallel_group())
        if pp > 1:
            comm.all_reduce(total, op=op, group=ps.get_pipeline_model_parallel_group())
        if zero1_group is not None or zero1_optimizer_groups is not None:
            comm.all_reduce(total, op=op, group=zero1_group if zero1_group is not None else ps.get_zero1_sharding_group())
    return total if is_inf else total ** (1.0 / norm_type)


def clip_grads_with_norm(
    parameters: Union[Iterable[torch.Tensor], torch.Tensor],
    max_norm: Union[float, int],
    total_norm: torch.Tensor,
) -> None:
    """Scale grads by ``min(1, max_norm/(norm+eps))`` without a host sync."""
    from .. import ops

    params = [parameters] if isinstance(parameters, torch.Tensor) else list(parameters)
    coeff = torch.clamp(float(max_norm) / (total_norm.float() + 1.0e-6), max=1.0)
    grads = []
    for p in params:
        g = p.grad if p.grad is not None else getattr(p, "main_grad", None)
        if g is not None:
            grads.append(g.detach())
    ops.optim.multi_tensor_scale_(grads, coeff)


def clip_grad_norm(
    parameters: Union[Iterable[torch.Tensor], torch.Tensor],
    max_norm: Union[float, int],
    norm_type: Union[float, int] = 2,
    zero1_optimizer: bool = False,
    zero1_optimizer_groups: Optional[List[List[int]]] = None,
    force_spmd: bool = True,
) -> torch.Tensor:
    params = [parameters] if isinstance(parameters, torch.Tensor) else list(parameters)
    total_norm = get_grad_norm(params, norm_type, zero1_optimizer, zero1_optimizer_groups, force_spmd)
    clip_grads_with_norm(params, max_norm, total_norm)
    return total_norm


def _bucketize(tensors: Sequence[torch.Tensor], cap_bytes: int) -> List[List[torch.Tensor]]:
    """Greedy buckets in the given order; an over-cap tensor gets a bucket of its own."""
    buckets: List[List[torch.Tensor]] = []
    cur: List[torch.Tensor] = []
    total = 0
    for t in tensors:
        nbytes = t.numel() * t.element_size()
        if nbytes > cap_bytes:
            if cur:
                buckets.append(cur)
                cur, total = [], 0
            buckets.append([t])
            continue
        if total + nbytes > cap_bytes and cur:
            buckets.append(cur)
            cur, total = [], 0
        cur.append(t)
        total += nbytes
    if cur:
        buckets.append(cur)
    return buckets


def bucket_allreduce_gradients(grads_list: Sequence[torch.Tensor], reduce_over_ep_group: bool = False) -> None:
    """Average gradients over data parallel replicas: scale by 1/dp, group by dtype, walk in
    *reverse* (last layer first) and all-reduce coalesced buckets of at most
    ``ALLREDUCE_BUCKET_CAP_MB`` (default 512) over the expert-data-parallel group; a second call
    with ``reduce_over_ep_group=True`` finishes the non-expert params over EP."""
    cap = int(os.getenv("ALLREDUCE_BUCKET_CAP_MB", _ALLREDUCE_BUCKET_CAP_MB)) * 1024 * 1024
    group = ps.get_expert_model_parallel_group() if reduce_over_ep_group else ps.get_expert_data_parallel_group()
    size = 1.0 if reduce_over_ep_group else float(ps.get_data_parallel_size())
    by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
    for g in grads_list:
        by_dtype.setdefault(g.dtype, []).append(g)
    for grads in by_dtype.values():
        ordered = list(reversed(grads))
        if size != 1.0:
            from .. import ops

            ops.optim.multi_tensor_scale_(ordered, 1.0 / size)
        for bucket in _bucketize(ordered, cap):
            comm.all_reduce(bucket, op="sum", group=group)


def _optimizer_grads(optimizer, predicate) -> List[torch.Tensor]:
    grads = []
    for pg in optimizer.param_groups:
        for p in pg["params"]:
            if isinstance(p, torch.Tensor) and predicate(p):
                if p.grad is not None:
                    grads.append(p.grad.data)
                elif hasattr(p, "main_grad"):
                    grads.append(p.main_grad.data)
    return grads


def allreduce_sequence_parallel_gradients(optimizer) -> None:
    """Norm/bias params tagged ``sequence_parallel_enabled`` saw only S/tp of the tokens on each
    TP rank → sum their grads over TP (coalesced per dtype)."""
    if ps.get_tensor_model_parallel_size() == 1:
        return
    # `_nxd_sp_reduced`: the ZeRO-1 optimizer already summed this gradient over TP in its gradient hook (overlapped
    # reduce-scatter mode), once, on the fully accumulated value
    grads = _optimizer_grads(optimizer, lambda p: getattr(p, "sequence_parallel_enabled", False)
                             and not getattr(p, "_nxd_sp_reduced", False))
    by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
    for g in grads:
        by_dtype.setdefault(g.dtype, []).append(g)
    for bucket in by_dtype.values():
        comm.all_reduce(bucket, op="sum", group=ps.get_tensor_model_parallel_group())


def allreduce_context_parallel_gradients(optimizer) -> None:
    """Every param saw S/cp of the sequence on each CP rank → average grads over CP."""
    cp = ps.get_context_model_parallel_size()
    if cp <= 1:
        return
    from .. import ops

    grads = _optimizer_grads(optimizer, lambda p: True)
    by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
    for g in grads:
        by_dtype.setdefault(g.dtype, []).append(g)
    for bucket in by_dtype.values():
        ops.optim.multi_tensor_scale_(bucket, 1.0 / cp)
        for b in _bucketize(bucket, _ALLREDUCE_BUCKET_CAP_MB * 1024 * 1024):
            comm.all_reduce(b, op="sum", group=ps.get_context_model_parallel_group())
