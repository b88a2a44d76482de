"""Stage-to-stage communication for the pipeline engine.

Role parity with reference ``pipeline/comm.py`` (tensor send/recv :41-106, python-object metadata
exchange :114-211).  XLA has no point-to-point primitive, so the reference emulates send/recv with
2-rank all-gathers; on H100 these are real NCCL ``isend``/``irecv`` issued as ONE batched group per
schedule step (``batch_isend_irecv``) on NCCL's own stream, so activation traffic overlaps compute.
Shape/dtype metadata travels once per (direction, chunk) over the gloo PP group and is cached.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, List, Optional, Tuple

import torch
import torch.distributed as dist

from ..parallel_layers import parallel_state as ps
from ..utils import get_device


@dataclass
class TensorMeta:
    tensor_index: int
    dtype: torch.dtype
    shape: torch.Size
    requires_grad: bool
    device: Optional[torch.device] = None


class P2PBatch:
    """Collects isend/irecv ops and launches them as one NCCL group."""

    def __init__(self, group):
        self.group = group
        self.ops: List[dist.P2POp] = []
        self.kinds: List[str] = []
        self.keep: List[torch.Tensor] = []

    def send(self, t: torch.Tensor, dst: int) -> None:
        t = t.contiguous()
        self.keep.append(t)
        self.ops.append(dist.P2POp(dist.isend, t, dst, self.group))
        self.kinds.append("send")

    def recv(self, meta: TensorMeta, src: int) -> torch.Tensor:
        buf = torch.empty(meta.shape, dtype=meta.dtype, device=get_device())
        self.ops.append(dist.P2POp(dist.irecv, buf, src, self.group))
        self.kinds.append("recv")
        return buf

    def launch(self) -> Tuple[List[Any], List[Any]]:
        """Start everything queued; returns (works that gate received data, works that only gate sends).
        gloo yields one work per op; NCCL coalesces the group into one work (a stream dependency, never a
        host block), which gates the receives if the group has any."""
        if not self.ops:
            return [], []
        works = dist.batch_isend_irecv(self.ops)
        kinds, self.ops, self.kinds = self.kinds, [], []
        if len(works) == len(kinds):
            return ([w for w, k in zip(works, kinds) if k == "recv"], [w for w, k in zip(works, kinds) if k == "send"])
        return (works, []) if "recv" in kinds else ([], works)


MAX_LENGTH = 2 ** 20          # largest pickled object the reference's fixed-size exchange accepts; objects here have no bound
MAX_RETRY = 3                 # attempts of the reference's store-based receive; the gloo exchange below blocks instead


def send_python_object(obj: Any, dst: Any = True, method: str = "gloo") -> None:
    """Send a picklable object over the pipeline's CPU (gloo) group.  ``dst``: a global rank, or the reference's
    ``send_next`` flag (``True`` → next pipeline rank, ``False`` → previous; comm.py:114-123).  ``method`` is accepted for
    source compatibility — there is one transport."""
    if isinstance(dst, bool):
        dst = ps.get_pipeline_model_parallel_next_rank() if dst else ps.get_pipeline_model_parallel_prev_rank()
    dist.send_object_list([obj], dst=dst, group=ps.get_pp_gloo_group())


def recv_python_object(src: Any = True, method: str = "gloo") -> Any:
    """Counterpart of :func:`send_python_object`.  ``src``: a global rank, or the reference's ``recv_prev`` flag (``True`` →
    from the previous pipeline rank; comm.py:160-169)."""
    if isinstance(src, bool):
        src = ps.get_pipeline_model_parallel_prev_rank() if src else ps.get_pipeline_model_parallel_next_rank()
    box: List[Any] = [None]
    dist.recv_object_list(box, src=src, group=ps.get_pp_gloo_group())
    return box[0]


# reference-compatible blocking helpers --------------------------------------------------
def send(tensor: torch.Tensor, send_next: bool = True, all_reduce_send_recv: bool = False) -> torch.Tensor:
    dst = ps.get_pipeline_model_parallel_next_rank() if send_next else ps.get_pipeline_model_parallel_prev_rank()
    dist.send(tensor.contiguous(), dst=dst, group=ps.get_pipeline_model_parallel_group())
    return tensor


def recv_from(tensor_meta: TensorMeta, recv_prev: bool = True, tracing: bool = False,
              all_reduce_send_recv: bool = False) -> torch.Tensor:
    """``tracing`` (reference: record the receive in a lazy graph instead of executing it) has no meaning with eager NCCL."""
    src = ps.get_pipeline_model_parallel_prev_rank() if recv_prev else ps.get_pipeline_model_parallel_next_rank()
    buf = torch.empty(tensor_meta.shape, dtype=tensor_meta.dtype, device=get_device())
    dist.recv(buf, src=src, group=ps.get_pipeline_model_parallel_group())
    buf.requires_grad_(tensor_meta.requires_grad and buf.is_floating_point())
    return buf
