"""Causal self-attention (flash style).  Kernel: ``csrc/attention_sm90.cu`` (tensor-core QK^T / PV with
register accumulators, online softmax) when built; otherwise the PyTorch SDPA library call, which is
flagged as a *library* path in DESIGN.md.  Reference call sites: ``kernels/flash_attn.py:162-212``
(``nki_flash_attn_func``), ``modeling_llama_nxd.py:468-475``.

Layout: q ``[B, S, Hq, D]``, k/v ``[B, S, Hkv, D]`` → out ``[B, S, Hq, D]``.
"""
from __future__ import annotations

import math
import os
from typing import Optional

import torch
import torch.nn.functional as F

from . import _ext


def _sdpa(q, k, v, causal: bool, scale: Optional[float]):
    hq, hkv = q.shape[2], k.shape[2]
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    if hq != hkv:
        kt = kt.repeat_interleave(hq // hkv, dim=1)
        vt = vt.repeat_interleave(hq // hkv, dim=1)
    o = F.scaled_dot_product_attention(qt, kt, vt, is_causal=causal, scale=scale)
    return o.transpose(1, 2)


def _own_kernel_ok(q, k, v) -> bool:
    if os.environ.get("NXD_DISABLE_OWN_ATTENTION", "0") == "1":
        return False
    if not (q.is_cuda and q.dtype == torch.bfloat16 and k.dtype == torch.bfloat16 and v.dtype == torch.bfloat16
            and q.shape[-1] == 128 and q.dim() == 4):
        return False
    e = _ext.ext()
    return e is not None and hasattr(e, "flash_attn_fwd")


def _tma_view(t: torch.Tensor) -> torch.Tensor:
    """The kernels address q/k/v as ``base + b·sb + s·ss + h·sh + d`` with 16-byte row loads: head_dim must be contiguous, the
    base 16-byte aligned and the (b, s, h) strides multiples of 8 elements (true for [B,S,H,D], [S,B,H,D], [B,H,S,D] memory
    and for slices of a fused projection output); anything else is copied once."""
    if t.stride(3) != 1 or t.data_ptr() % 16 or any(t.stride(i) % 8 for i in range(3)):
        return t.contiguous()
    return t


class _FlashAttn(torch.autograd.Function):
    """Flash attention (``csrc/attention_sm90.cu``): forward saves (q, k, v, o, lse); backward is a dK/dV kernel and a dQ
    kernel.  Outputs/gradients are laid out ``[S,B,H,D]`` in memory (returned as ``[B,S,H,D]`` views) so the
    model's ``[S,B,H·D]`` reshape is free."""

    @staticmethod
    def forward(ctx, q, k, v, causal, scale):
        e = _ext.ext()
        q, k, v = _tma_view(q), _tma_view(k), _tma_view(v)
        _ext.count_launch()
        o, lse = e.flash_attn_fwd(q, k, v, bool(causal), float(scale), True)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.causal, ctx.scale = causal, scale
        return o

    @staticmethod
    def backward(ctx, go):
        q, k, v, o, lse = ctx.saved_tensors
        e = _ext.ext()
        _ext.count_launch(3)   # δ prep + dK/dV + dQ
        dq, dk, dv = e.flash_attn_bwd(_tma_view(go), q, k, v, o, lse, bool(ctx.causal), float(ctx.scale), True)
        return dq, dk, dv, None, None


class _FlashAttnLse(torch.autograd.Function):
    """Same kernels, but LSE is a differentiable output: ring attention merges per-block results through their LSEs, and
    a gradient into LSE only shifts δ in the backward kernel (``dS = P∘(dP − (δ − g_lse))``)."""

    @staticmethod
    def forward(ctx, q, k, v, causal, scale):
        q, k, v = _tma_view(q), _tma_view(k), _tma_view(v)
        _ext.count_launch()
        o, lse = _ext.ext().flash_attn_fwd(q, k, v, bool(causal), float(scale), False)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.causal, ctx.scale = causal, scale
        return o, lse

    @staticmethod
    def backward(ctx, go, g_lse):
        q, k, v, o, lse = ctx.saved_tensors
        _ext.count_launch(3)
        go = torch.zeros_like(o) if go is None else go
        dlse = None if g_lse is None else g_lse.float().contiguous()
        dq, dk, dv = _ext.ext().flash_attn_bwd(_tma_view(go.to(o.dtype)), q, k, v, o, lse, bool(ctx.causal), float(ctx.scale), False, dlse)
        return dq, dk, dv, None, None


def flash_attention_with_lse(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool, scale: float):
    """``(out [B,S,H,D], lse [B,H,S] fp32)`` on the own kernels, or ``None`` when they do not apply."""
    if _own_kernel_ok(q, k, v) and (not causal or q.shape[1] == k.shape[1]) and hasattr(_ext.ext(), "flash_attn_bwd"):
        return _FlashAttnLse.apply(q, k, v, causal, scale)
    return None


def flash_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True,
                    scale: Optional[float] = None) -> torch.Tensor:
    scale = scale if scale is not None else 1.0 / math.sqrt(q.shape[-1])
    if _own_kernel_ok(q, k, v) and (not causal or q.shape[1] == k.shape[1]):
        return _FlashAttn.apply(q, k, v, causal, scale)
    return _sdpa(q, k, v, causal, scale)


def decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, positions: torch.Tensor,
                     scale: Optional[float] = None) -> torch.Tensor:
    """One new token per sequence against a KV cache: ``q [B,1,H,D]``, caches ``[B,L,Hkv,D]`` (any batch / sequence / head
    strides), ``positions [B]`` = cache index of the newest token (keys ≤ position are visible).  CUDA bf16 with head_dim 128:
    the split-KV flash-decoding kernel (``csrc/decode.cu``); otherwise SDPA with a length mask."""
    B, _, H, D = q.shape
    Hkv, L = k_cache.shape[2], k_cache.shape[1]
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    e = _ext.ext() if q.is_cuda else None
    if (e is not None and hasattr(e, "decode_attention") and D == 128 and q.dtype == torch.bfloat16 and k_cache.dtype == torch.bfloat16
            and H // Hkv in (1, 2, 4, 8) and k_cache.stride(3) == 1 and v_cache.stride(3) == 1):
        _ext.count_launch(2)
        return e.decode_attention(q.contiguous(), k_cache, v_cache, positions.to(torch.long).contiguous(), float(scale))
    qt, kt, vt = q.transpose(1, 2), k_cache.transpose(1, 2), v_cache.transpose(1, 2)
    if H != Hkv:
        kt, vt = kt.repeat_interleave(H // Hkv, 1), vt.repeat_interleave(H // Hkv, 1)
    mask = (torch.arange(L, device=q.device)[None, :] <= positions[:, None])[:, None, None, :]
    return torch.nn.functional.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, scale=scale).transpose(1, 2)
