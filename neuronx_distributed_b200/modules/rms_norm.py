"""RMSNorm with fp32 statistics and a sequence-parallel-tagged weight
(reference ``modules/rms_norm.py:10-72``).  Forward/backward run the sm_90a kernels in
``csrc/elementwise.cu`` via :func:`ops.norm.rms_norm`."""
from __future__ import annotations

import numbers
from typing import Optional

import torch
from torch import nn

from ..ops.norm import rms_norm


def manual_rms_norm(input: torch.Tensor, *args) -> torch.Tensor:   # noqa: A002  (reference argument name)
    """Plain-PyTorch form (kept for numerics tests).  ``manual_rms_norm(x, weight, eps)`` or the reference's
    ``manual_rms_norm(input, normalized_shape, weight, eps)`` (rms_norm.py:10-33; statistics over the trailing
    ``len(normalized_shape)`` dims)."""
    if len(args) == 3:
        normalized_shape, weight, eps = args
        dims = tuple(range(-len(tuple(normalized_shape)), 0))
    else:
        (weight, eps), dims = args, (-1,)
    dt = input.dtype
    xf = input.float()
    return (weight.float() * (xf * torch.rsqrt(xf.pow(2).mean(dims, keepdim=True) + eps))).to(dt)


class RMSNorm(nn.Module):
    def __init__(self, normalized_shape=None, eps: float = 1e-5, sequence_parallel_enabled: bool = False,
                 dtype: torch.dtype = torch.float32, device=None, hidden_size: Optional[int] = None, **kwargs):
        """``normalized_shape``: int or shape of the trailing dims (``hidden_size=`` is the same thing by keyword).  Signature
        and the 1e-5 default of reference rms_norm.py:36-62; ``elementwise_affine=False`` is refused as there."""
        super().__init__()
        if kwargs.pop("elementwise_affine", True) is False:
            raise RuntimeError("RMSNorm does not support `elementwise_affine = False`")
        if kwargs:
            raise TypeError(f"unexpected arguments {sorted(kwargs)}")
        shape = normalized_shape if normalized_shape is not None else hidden_size
        assert shape is not None, "normalized_shape (or hidden_size) is required"
        self.normalized_shape = torch.Size((shape,) if isinstance(shape, numbers.Integral) else tuple(shape))
        assert len(self.normalized_shape) == 1, "the kernels normalise over the last dimension"
        self.elementwise_affine = True
        self.weight = nn.Parameter(torch.ones(self.normalized_shape, dtype=dtype, device=device))
        self.eps = self.variance_epsilon = eps
        self.sequence_parallel_enabled = sequence_parallel_enabled
        setattr(self.weight, "sequence_parallel_enabled", sequence_parallel_enabled)

    def reset_parameters(self) -> None:
        """Re-initialise after meta-device materialisation (``reinit_model`` calls it): unit gain."""
        with torch.no_grad():
            self.weight.fill_(1.0)
        setattr(self.weight, "sequence_parallel_enabled", self.sequence_parallel_enabled)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        hidden_states = input      # reference parameter names in the signature
        return rms_norm(hidden_states, self.weight, self.variance_epsilon)

    def extra_repr(self) -> str:
        return f"{tuple(self.weight.shape)}, eps={self.variance_epsilon}"
