"""Small helpers around the attention entry points (reference ``kernels/kernel_utils.py:8-58``)."""
from __future__ import annotations

import os

import torch


def check_xla_bf16_flags() -> bool:
    """The reference's global bf16 switches (``XLA_USE_BF16`` / ``XLA_DOWNCAST_BF16``) are honoured by ``cast`` so that
    launch scripts that export them keep producing bf16 attention."""
    return os.getenv("XLA_USE_BF16") == "1" or os.getenv("XLA_DOWNCAST_BF16") == "1"


def get_seed(dropout_p: float, device) -> torch.Tensor | None:
    """Dropout seed for the attention kernels: a one-element int32 tensor drawn on ``device`` from (and advancing) its
    default generator, without a host sync.  TP ranks draw the same seed (the default stream is seeded alike inside a TP
    group) and differ through their global head indices; activation checkpointing restores the generator, so a recompute
    draws the same seed."""
    if dropout_p <= 0.0:
        return None
    return torch.randint(0, 2 ** 31 - 1, (1,), device=device, dtype=torch.int32)


def move_seed(dropout_p: float) -> None:
    """``get_seed`` already advanced the generator; kept for call-site parity."""


def permute(q, k, v):
    """``[B, H, S, D] → [B, H, D, S]`` for all three (the reference kernel's operand layout)."""
    return tuple(t.permute(0, 1, 3, 2) for t in (q, k, v))


def cast(q, k, v):
    if check_xla_bf16_flags():
        return tuple(t.to(torch.bfloat16) for t in (q, k, v))
    return q, k, v


def torch_to_nki_dtype(dtype: torch.dtype):
    """Kernels here take torch dtypes directly; validates that the dtype is one the own kernels support."""
    if dtype not in (torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn, torch.float8_e5m2):
        raise ValueError(f"Invalid dtype '{dtype}'. Not supported by the sm_90a kernels.")
    return dtype
