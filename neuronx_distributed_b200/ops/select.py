"""Row-wise arg-max / top-k on the sm_90a selection kernels (``csrc/select.cu``) with plain PyTorch as the CPU path and the
numerics oracle.  ``index_offset`` shifts the returned indices (global id of a vocab shard's first column)."""
from __future__ import annotations

from typing import Tuple

import torch

from . import _ext


def _kernel_ok(x: torch.Tensor) -> bool:
    return (x.is_cuda and x.dtype in (torch.bfloat16, torch.float16, torch.float32) and x.shape[-1] > 0
            and _ext.ext() is not None and hasattr(_ext.ext(), "row_argmax"))


def row_max(x: torch.Tensor, index_offset: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """``x`` [..., V] → (max fp32 [...], argmax int64 [...] + index_offset); ties → smallest index."""
    lead = x.shape[:-1]
    if _kernel_ok(x):
        x2 = x.reshape(-1, x.shape[-1])
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        _ext.count_launch()
        v, i = _ext.ext().row_argmax(x2, int(index_offset))
        return v.view(lead), i.view(lead)
    v, i = torch.max(x.float(), dim=-1)
    return v, i + index_offset


def row_topk(x: torch.Tensor, k: int, index_offset: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """``x`` [..., V] → (values fp32 [..., k], indices int64 [..., k] + index_offset), sorted descending."""
    lead = x.shape[:-1]
    V = x.shape[-1]
    if _kernel_ok(x) and _ext.ext().row_topk_supported(V, k):
        x2 = x.reshape(-1, V)
        if x2.stride(-1) != 1:
            x2 = x2.contiguous()
        _ext.count_launch()
        v, i = _ext.ext().row_topk(x2, int(k), int(index_offset))
        return v.view(*lead, k), i.view(*lead, k)
    v, i = torch.topk(x.float(), k, dim=-1)
    return v, i + index_offset
