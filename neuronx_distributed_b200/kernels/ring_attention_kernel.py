"""Context-parallel ring attention entry points (reference ``kernels/ring_attention_kernel.py:36-167``)."""
from __future__ import annotations

from typing import Optional

import torch

from ..modules.attention.ring import ring_attention
from .kernel_utils import cast


def get_seq_tile_size(seqlen: int) -> int:
    """K/V tile length used per ring step: the local sequence is processed in tiles of at most 2048 and at least 1024
    positions (same rule as the reference, which sizes its SBUF tiles with it; here it bounds the per-step score tile the
    block kernel keeps in registers)."""
    return max(2048 if seqlen >= 4096 else seqlen // 2, 1024)


class NkiRingAttnFunc:
    """``apply(q, k, v, rank_id, src_tgt_pairs, softmax_scale, causal, …)`` with q/k/v in the kernel layout ``[B, H, D, S]``
    (what ``nki_ring_attn_func`` passes after ``permute``).  ``rank_id`` / ``src_tgt_pairs`` describe the ring in the
    reference; here the ring is the context-parallel process group of ``parallel_state``."""

    @staticmethod
    def apply(q, k, v, rank_id=None, src_tgt_pairs=None, softmax_scale=None, causal: bool = True, mixed_precision: bool = True,
              seed=None, dropout_p: float = 0.0):
        assert dropout_p == 0.0, "attention dropout is not supported by the ring kernel"
        q, k, v = (t.permute(0, 3, 1, 2) for t in (q, k, v))            # [B, H, D, S] → [B, S, H, D]
        return ring_attention(q, k, v, causal=causal, scale=softmax_scale).transpose(1, 2)


def nki_ring_attn_func(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, rank_id=None, src_tgt_pairs=None, dropout_p: float = 0.0,
                       softmax_scale: Optional[float] = None, causal: bool = True, mixed_precision: bool = True, seed=None,
                       lnc: int = 1, transpose_nki_inputs: bool = True) -> torch.Tensor:
    """q/k/v: this rank's ``[B, H, S_local, D]`` slices → ``[B, H, S_local, D]``."""
    assert dropout_p == 0.0, "attention dropout is not supported by the ring kernel"
    q, k, v = cast(q, k, v)
    out = ring_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), causal=causal, scale=softmax_scale)
    return out.transpose(1, 2)
