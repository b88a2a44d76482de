"""Flash-attention entry points with the reference's call conventions (``kernels/flash_attn.py:15-214``).

Layout convention of ``nki_flash_attn_func`` (same as the reference):

* ``transpose_nki_inputs=True`` (default) — the caller hands ``q`` and ``k`` already transposed to ``[B, H, D, S]`` and
  ``v`` as ``[B, H, S, D]`` (what ``overrides.transformer_overrides.apply_rotary_pos_emb(…, flash_attn=True)`` produces);
* ``transpose_nki_inputs=False`` — ``q``, ``k``, ``v`` are all ``[B, H, S, D]``.

The result is ``[B, H, S, D]`` in both cases.  The math runs in ``ops.attention.flash_attention`` (own forward /
backward kernels for bf16 with head_dim 64, 80, 96 or 128, library flash attention otherwise), which wants ``[B, S, H, D]``
*views* — the transposes below are stride changes the kernels' strided ``cp.async`` tile loads consume, not copies."""
from __future__ import annotations

from typing import Optional

import torch

from ..ops.attention import flash_attention, flash_kernels_apply
from .kernel_utils import cast


def get_flash_attn_kernels(use_sharded: bool = False):
    """(forward, backward) callables.  There is one kernel pair; ``use_sharded`` (LNC2 sharding on Trn2) has no meaning on
    a GPU whose two dies are one device."""
    from .. import ops

    def forward(q, k, v, causal, scale):
        return ops.attention._FlashAttn.apply(q, k, v, causal, scale, None, 0, 0, True)[0]

    return forward, None


class NKIAttnFunc(torch.autograd.Function):
    """Name kept for code that calls ``NKIAttnFunc.apply`` directly.  Delegates to the differentiable
    ``flash_attention`` op (its own autograd node carries the backward kernel).

    ``dropout_p`` > 0 is the fused kernel's attention dropout, as in the reference: it needs inputs the flash kernels take
    (CUDA bf16, head_dim 64, 80, 96 or 128) and raises ``AssertionError`` otherwise.  ``seed`` (a one-element integer
    tensor) or, when None, one drawn from the default generator on the device (``kernel_utils.get_seed``).  Attention
    dropout on any other input is ``ops.attention.flash_attention(dropout_p=…)``."""

    @staticmethod
    def apply(q, k, v, softmax_scale=None, causal: bool = True, mixed_precision: bool = True, seed=None, dropout_p: float = 0.0,  # noqa: D102
              use_sharded: bool = False, transpose_nki_inputs: bool = True, lnc: int = 1):
        if transpose_nki_inputs:                              # q, k arrive as [B, H, D, S]
            q, k = q.permute(0, 1, 3, 2), k.permute(0, 1, 3, 2)
        q, k, v = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
        if dropout_p > 0.0:
            assert flash_kernels_apply(q, k, v, causal), \
                "attention dropout runs in the fused kernel: CUDA bf16 q, k, v with head_dim 64, 80, 96 or 128"
        out = flash_attention(q, k, v, causal, softmax_scale, dropout_p=dropout_p, dropout_seed=seed)
        return out.transpose(1, 2)


def nki_flash_attn_func(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, lnc: int = 1, dropout_p: float = 0.0,
                        softmax_scale: Optional[float] = None, causal: bool = True, mixed_precision: bool = True, seed=None,
                        hardware_type=None, transpose_nki_inputs: bool = True) -> torch.Tensor:
    seqlen = q.shape[-1] if transpose_nki_inputs else q.shape[-2]
    if seqlen % 128 != 0 and q.is_cuda:
        raise NotImplementedError(f"sequence length must be a multiple of 128 for the fused kernel, got {seqlen}")
    q, k, v = cast(q, k, v)
    return NKIAttnFunc.apply(q, k, v, softmax_scale, causal, mixed_precision, seed, dropout_p, lnc == 2, transpose_nki_inputs, lnc)
