"""Rotary position embedding, HF "rotate-half" convention, applied in place to q and k
(kernel: ``csrc/elementwise.cu`` rope_apply).  Backward is the same rotation with −sin.
Reference: ``overrides/transformer_overrides.py:20-32``, ``modules/attention/utils.py:50-80``.

Layout: q/k ``[B, S, H, D]`` (any strides on B/S/H as long as D is contiguous); cos/sin ``[S, D/2]``
fp32 (position ``s`` of the *global* sequence; callers slice for CP/SP offsets).
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _ext


def rotate(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, sign: float = 1.0) -> torch.Tensor:
    """Rotate-half RoPE in fp32 torch math (the reference of the kernel, and the decode-time rotation off the kernels):
    x ``[B, S, H, D]``; cos/sin ``[S, D/2]`` shared by the batch, or ``[B, S, D/2]`` per row (each sequence at its own
    positions).  ``sign`` −1 rotates backwards (the gradient)."""
    d2 = x.shape[-1] // 2
    xf = x.float()
    x1, x2 = xf[..., :d2], xf[..., d2:]
    c = cos.unsqueeze(-2).float()
    s = sin.unsqueeze(-2).float() * sign
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1).to(x.dtype)


class _Rope(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cos, sin):
        ctx.save_for_backward(cos, sin)
        if _ext.use_cuda(x, cos, sin) and x.dtype in (torch.bfloat16, torch.float16, torch.float32) \
                and x.stride(-1) == 1 and x.shape[-1] % 2 == 0:
            ctx.cuda = True
            _ext.count_launch()
            return _ext.ext().rope_apply(x, cos.contiguous().float(), sin.contiguous().float(), 1.0)
        ctx.cuda = False
        return rotate(x, cos, sin)

    @staticmethod
    def backward(ctx, g):
        cos, sin = ctx.saved_tensors
        if ctx.cuda:
            _ext.count_launch()
            g = g if g.stride(-1) == 1 else g.contiguous()        # autograd may hand a gradient with a strided head dim
            return _ext.ext().rope_apply(g, cos.contiguous().float(), sin.contiguous().float(), -1.0), None, None
        return rotate(g, cos, sin, -1.0), None, None


def apply_rotary(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    return _Rope.apply(x, cos, sin)


def rope_tables(seq_len: int, dim: int, base: float = 10000.0, device=None, offset: int = 0,
                scaling: float = 1.0, rope_scaling: Optional[dict] = None):
    """cos / sin ``[seq_len, dim/2]`` fp32 for positions ``offset ..``.  ``scaling``: linear position scaling.
    ``rope_scaling``: Llama-3 frequency rescaling (the ``"llama3"`` keys of a Hugging Face ``rope_scaling``: ``factor``,
    ``low_freq_factor``, ``high_freq_factor``, ``original_max_position_embeddings``), applied to the inverse frequencies
    by :func:`~neuronx_distributed_b200.modules.attention.utils.apply_scaling`."""
    inv = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.float32, device=device) / dim))
    if rope_scaling is not None:
        from ..modules.attention.utils import apply_scaling      # not at module level: ``modules`` imports ``ops``

        inv = apply_scaling(inv, **rope_scaling)
    t = (torch.arange(offset, offset + seq_len, dtype=torch.float32, device=device)) / scaling
    fr = torch.outer(t, inv)
    return fr.cos(), fr.sin()
