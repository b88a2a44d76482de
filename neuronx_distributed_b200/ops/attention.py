"""Self-attention (flash style), causal or not, with an optional key-padding mask and, when causal, an optional sliding window.  Kernel: ``csrc/attention_sm90.cu``
(tensor-core QK^T / PV with register accumulators, online softmax) for bf16 CUDA tensors with head_dim 64, 80, 96 or 128;
otherwise the PyTorch SDPA library call, which is flagged as a *library* path in DESIGN.md.  Reference call sites:
``kernels/flash_attn.py:162-212`` (``nki_flash_attn_func``), ``modeling_llama_nxd.py:468-475``.

Layout: q ``[B, S, Hq, D]``, k/v ``[B, S, Hkv, D]`` → out ``[B, S, Hq, D]``.

Attention dropout follows one rule on every path, :func:`attention_dropout_keep`, so a seed drops the same (b, h, i, j) on
the kernels and off them.
"""
from __future__ import annotations

import math
import os
from typing import Optional, Union

import numpy as np
import torch
import torch.nn.functional as F

from . import _ext


#: head sizes the flash kernels are compiled for
FLASH_HEAD_DIMS = (64, 80, 96, 128)

#: GQA group sizes H / Hkv the token-generation kernels (decode, flash-decoding, verification) are compiled for; they keep
#: the group's query rows in registers, so larger groups take :func:`speculation_attention_torch`
DECODE_GQA_GROUPS = (1, 2, 3, 4, 5, 6, 7, 8)

#: fp8 KV-cache dtypes: stored as k / k_scale and v / v_scale, de-quantised off the kernels (the decode kernels read e4m3)
FP8_KV_DTYPES = (torch.float8_e4m3fn, torch.float8_e5m2)


def window_visibility(s_q: int, s_kv: int, window: Optional[int], device=None, q_offset: int = 0) -> torch.Tensor:
    """``[S_q, S_kv]`` bool: causal visibility, limited to the last ``window`` keys (query i sees i − W < j ≤ i) when
    ``window`` is set.  ``q_offset``: global position of query row 0 minus that of key row 0 (a context-parallel block whose
    queries come after its keys); query i then sees i + q_offset − W < j ≤ i + q_offset."""
    i = torch.arange(s_q, device=device)[:, None] + q_offset
    j = torch.arange(s_kv, device=device)[None, :]
    vis = j <= i
    return vis if window is None else vis & (j > i - window)


_PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_PHILOX_W = (np.uint64(0x9E3779B9), np.uint64(0xBB67AE85))
_U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., SC'11; the generator of torch's CUDA RNG) on numpy arrays: ``counter`` is four
    broadcastable arrays of 32-bit words, ``key`` two 32-bit words → the four output words as uint64 arrays.  32×32-bit
    products are exact in uint64."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _U32 for c in counter)
    k0, k1 = np.uint64(key[0]) & _U32, np.uint64(key[1]) & _U32
    for r in range(10):
        if r:
            k0, k1 = (k0 + _PHILOX_W[0]) & _U32, (k1 + _PHILOX_W[1]) & _U32
        p0, p1 = c0 * _PHILOX_M[0], c2 * _PHILOX_M[1]
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _U32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _U32
    return c0, c1, c2, c3


def dropout_keep_threshold(p: float) -> int:
    """round((1 − p)·2³²), at most 2³² − 1: a Philox word below it keeps its element (the kernels compute it alike)."""
    return min(math.floor((1.0 - p) * 4294967296.0 + 0.5), 4294967295)


def attention_dropout_keep(seed, B: int, H: int, S_q: int, S_kv: int, p: float, head_offset: int = 0) -> torch.Tensor:
    """``[B, H, S_q, S_kv]`` bool (CPU): which attention probabilities dropout with probability ``p`` keeps.  The rule of
    the flash kernels (``csrc/attention_sm90.cu``): element (b, h, i, j) — query row i, key row j, global head
    g = ``head_offset`` + h — is kept iff word 2·((i >> 3) & 1) + ((j >> 3) & 1) of Philox4x32-10 with key (seed low word,
    seed high word) and counter (j & ~8, i & ~8, g, b) is below :func:`dropout_keep_threshold`.  It depends on nothing
    else, so tensor-parallel ranks, which hold heads ``head_offset`` … ``head_offset + H − 1``, together drop what one
    unsharded run drops.  ``seed``: an int or a one-element integer tensor."""
    if isinstance(seed, torch.Tensor):
        seed = int(seed.reshape(-1)[0].item())
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    i = np.arange(S_q, dtype=np.uint64)[None, None, :, None]
    j = np.arange(S_kv, dtype=np.uint64)[None, None, None, :]
    g = np.arange(head_offset, head_offset + H, dtype=np.uint64)[None, :, None, None]
    b = np.arange(B, dtype=np.uint64)[:, None, None, None]
    not8 = np.uint64(~8 & 0xFFFFFFFF)
    words = philox4x32_10((j & not8, i & not8, g, b), (seed & 0xFFFFFFFF, seed >> 32))
    sel = (((i >> np.uint64(3)) & np.uint64(1)) * np.uint64(2) + ((j >> np.uint64(3)) & np.uint64(1)))
    w = np.where(sel == 0, words[0], np.where(sel == 1, words[1], np.where(sel == 2, words[2], words[3])))
    return torch.from_numpy(np.broadcast_to(w < np.uint64(dropout_keep_threshold(p)), (B, H, S_q, S_kv)).copy())


def _check_dropout(p: float) -> float:
    if not 0.0 <= float(p) < 1.0:
        raise ValueError(f"dropout_p must be in [0, 1), got {p}")
    return float(p)


def _dropout_seed(seed, p: float, device) -> torch.Tensor:
    """The seed as the kernels read it (a one-element integer tensor on ``device``); ``None`` draws one from the default
    generator of ``device`` without a host sync."""
    if seed is None:
        from ..kernels.kernel_utils import get_seed
        return get_seed(p, device)
    if isinstance(seed, torch.Tensor):
        return seed.to(device)
    return torch.tensor([int(seed)], dtype=torch.int64, device=device)


def _dropout_attention(q, k, v, causal: bool, scale: float, key_padding_mask, window: Optional[int], p: float, seed,
                       head_offset: int):
    """Attention with dropout off the kernels: the explicit softmax in fp32, with the mask of
    :func:`attention_dropout_keep`.  A query row that sees no key gets 0, as on the kernels."""
    B, sq, H, _ = q.shape
    sk, hkv = k.shape[1], k.shape[2]
    qt, kt, vt = q.transpose(1, 2).float(), k.transpose(1, 2).float(), v.transpose(1, 2).float()
    if H != hkv:
        kt, vt = kt.repeat_interleave(H // hkv, dim=1), vt.repeat_interleave(H // hkv, dim=1)
    visible = torch.ones(1, 1, 1, sk, dtype=torch.bool, device=q.device)
    if key_padding_mask is not None:
        visible = key_padding_mask.to(q.device).bool()[:, None, None, :]
    if causal:
        visible = visible & window_visibility(sq, sk, window, q.device)
    s = (qt @ kt.transpose(-1, -2) * scale).masked_fill(~visible, torch.finfo(torch.float32).min)
    probs = torch.softmax(s, dim=-1).masked_fill(~visible, 0.0)
    keep = attention_dropout_keep(seed, B, H, sq, sk, p, head_offset).to(q.device)
    probs = probs * (keep.float() * (1.0 / (1.0 - p)))
    return (probs @ vt).transpose(1, 2).to(q.dtype)


def _sdpa(q, k, v, causal: bool, scale: Optional[float], key_padding_mask: Optional[torch.Tensor] = None,
          window: Optional[int] = None):
    hq, hkv = q.shape[2], k.shape[2]
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    if hq != hkv:
        kt = kt.repeat_interleave(hq // hkv, dim=1)
        vt = vt.repeat_interleave(hq // hkv, dim=1)
    if key_padding_mask is None and window is None:
        o = F.scaled_dot_product_attention(qt, kt, vt, is_causal=causal, scale=scale)
    else:
        # additive bias [B or 1, 1, 1 or S_q, S_kv]: 0 where visible, −inf where masked (or above the diagonal when causal, or
        # outside the window)
        sq, sk = q.shape[1], k.shape[1]
        visible = torch.ones(1, 1, 1, sk, dtype=torch.bool, device=q.device)
        if key_padding_mask is not None:
            visible = key_padding_mask.bool()[:, None, None, :]
        if causal:
            visible = visible & window_visibility(sq, sk, window, q.device)
        bias = torch.zeros(visible.shape, dtype=q.dtype, device=q.device).masked_fill(~visible, float("-inf"))
        o = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=bias, scale=scale)
    return o.transpose(1, 2)


def flash_kernels_apply(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = False) -> bool:
    """True when the own flash kernels handle these tensors: bf16 CUDA, 4-D ``[B, S, H, D]`` with D in
    :data:`FLASH_HEAD_DIMS` (the same for q, k and v), S_q == S_kv when ``causal``, and the extension loaded.
    ``NXD_DISABLE_OWN_ATTENTION=1`` turns them off (the SDPA path is then used, e.g. as a comparison baseline)."""
    if os.environ.get("NXD_DISABLE_OWN_ATTENTION", "0") == "1":
        return False
    if not (q.is_cuda and q.dtype == torch.bfloat16 and k.dtype == torch.bfloat16 and v.dtype == torch.bfloat16
            and q.dim() == 4 and k.dim() == 4 and v.dim() == 4 and q.shape[-1] in FLASH_HEAD_DIMS
            and k.shape[-1] == q.shape[-1] and v.shape[-1] == q.shape[-1] and (not causal or q.shape[1] == k.shape[1])):
        return False
    e = _ext.ext()
    return e is not None and hasattr(e, "flash_attn_fwd") and hasattr(e, "flash_attn_bwd")


def _kernel_mask(m: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """Key-padding mask as the kernels read it: bool / uint8 ``[B, S_kv]`` with a contiguous key dimension."""
    if m is None:
        return None
    if m.dtype not in (torch.bool, torch.uint8):
        m = m != 0
    return m if m.stride(-1) == 1 else m.contiguous()


def _tma_view(t: torch.Tensor) -> torch.Tensor:
    """The kernels address q/k/v as ``base + b·sb + s·ss + h·sh + d`` with 16-byte ``cp.async`` row loads: head_dim must be
    contiguous, the base 16-byte aligned and the (b, s, h) strides multiples of 8 elements (true for [B,S,H,D], [S,B,H,D],
    [B,H,S,D] memory and for slices of a fused projection output); anything else is copied once."""
    if t.stride(3) != 1 or t.data_ptr() % 16 or any(t.stride(i) % 8 for i in range(3)):
        return t.contiguous()
    return t


def _flash_backward(go, q, k, v, o, lse, causal: bool, scale: float, mask=None, window: int = 0, q_offset: int = 0,
                    sbhd_out: bool = False, dlse=None, dropout_p: float = 0.0, seed=None, head_offset: int = 0):
    """``(dq, dk, dv)`` of the flash kernels for the rows' output ``o`` and log-normaliser ``lse``: a δ pre-pass, a dK/dV
    kernel and a dQ kernel.  ``dlse``: the gradient into ``lse``, or None.  ``dropout_p`` / ``seed`` / ``head_offset``:
    those of the forward."""
    _ext.count_launch(3)
    tv = _tma_view
    return _ext.ext().flash_attn_bwd(tv(go.to(o.dtype)), tv(q), tv(k), tv(v), tv(o), lse.contiguous(), bool(causal),
                                     float(scale), sbhd_out, dlse, mask, int(window), int(q_offset), float(dropout_p), seed,
                                     int(head_offset))


class _FlashAttn(torch.autograd.Function):
    """Flash attention (``csrc/attention_sm90.cu``) → ``(o, lse)``; forward saves (q, k, v, o, lse, mask).  LSE is a
    differentiable output: ring attention merges per-block results through their LSEs, and a gradient into LSE only shifts
    δ in the backward kernel (``dS = P∘(dP − (δ − g_lse))``).  ``sbhd_out``: outputs and gradients are laid out ``[S,B,H,D]``
    in memory (returned as ``[B,S,H,D]`` views), so a model's ``[S,B,H·D]`` reshape is free.  ``dropout_p`` > 0: attention
    dropout with the device ``seed`` (saved for the backward) and global head offset ``head_offset``."""

    @staticmethod
    def forward(ctx, q, k, v, causal, scale, mask, window, q_offset, sbhd_out, dropout_p=0.0, seed=None, head_offset=0):
        ctx.set_materialize_grads(False)
        q, k, v = _tma_view(q), _tma_view(k), _tma_view(v)
        _ext.count_launch()
        o, lse = _ext.ext().flash_attn_fwd(q, k, v, bool(causal), float(scale), sbhd_out, mask, int(window), int(q_offset),
                                           float(dropout_p), seed, int(head_offset))
        ctx.save_for_backward(q, k, v, o, lse, mask, seed)
        ctx.args = (causal, scale, window, q_offset, sbhd_out, dropout_p, head_offset)
        return o, lse

    @staticmethod
    def backward(ctx, go, g_lse):
        q, k, v, o, lse, mask, seed = ctx.saved_tensors
        causal, scale, window, q_offset, sbhd_out, dropout_p, head_offset = ctx.args
        go = torch.zeros_like(o) if go is None else go
        dlse = None if g_lse is None else g_lse.float().contiguous()
        dq, dk, dv = _flash_backward(go, q, k, v, o, lse, causal, scale, mask, window, q_offset, sbhd_out, dlse, dropout_p,
                                     seed, head_offset)
        return dq, dk, dv, None, None, None, None, None, None, None, None, None


def _window_args(name: str, causal: bool, sliding_window: Optional[int], q_offset: int = 0) -> int:
    """Checks ``sliding_window`` / ``q_offset`` and returns the kernels' integer window (0 = none)."""
    if sliding_window is not None and not causal:
        raise ValueError(f"{name}: sliding_window needs causal=True")
    window = check_window(sliding_window)
    if q_offset < 0 or (q_offset > 0 and window == 0):
        raise ValueError(f"{name}: q_offset must be 0, or > 0 with a sliding_window; got {q_offset}")
    return window


def flash_attention_with_lse(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool, scale: float,
                             sliding_window: Optional[int] = None, q_offset: int = 0):
    """``(out [B,S,H,D], lse [B,H,S] fp32)`` on the own kernels, or ``None`` when they do not apply.

    ``sliding_window`` as in :func:`flash_attention`.  ``q_offset`` ≥ 0 (causal, with a window): the global position of query
    row 0 minus that of key row 0, as in one off-diagonal block of context-parallel attention; query i then sees keys
    i + q_offset − W < j ≤ i + q_offset.  A row that sees no key gets O = 0 and LSE = −inf."""
    window = _window_args("flash_attention_with_lse", causal, sliding_window, q_offset)
    if flash_kernels_apply(q, k, v, causal):
        return _FlashAttn.apply(q, k, v, causal, scale, None, window, q_offset, False)
    return None


def flash_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True,
                    scale: Optional[float] = None, key_padding_mask: Optional[torch.Tensor] = None,
                    sliding_window: Optional[int] = None, dropout_p: float = 0.0,
                    dropout_seed: Optional[Union[int, torch.Tensor]] = None, head_offset: int = 0) -> torch.Tensor:
    """softmax(q·kᵀ·scale)·v for q ``[B, S_q, H, D]``, k/v ``[B, S_kv, Hkv, D]`` (H a multiple of Hkv) → ``[B, S_q, H, D]``.

    ``causal``: query i sees keys ≤ i (needs S_q == S_kv on the own kernels).  ``key_padding_mask``: ``[B, S_kv]`` bool
    (or integer, nonzero = visible); key j of batch b is visible iff ``key_padding_mask[b, j]``.  It combines with
    ``causal`` and GQA and is never read on the host, so the call stays capturable in CUDA graphs and launch plans.
    ``sliding_window``: W ≥ 1 (causal only) limits query i to keys i − W < j ≤ i, the last W keys including its own (the rule
    of Mistral / Mixtral); ``None`` means no window, and W ≥ S_kv is plain causal attention.  On the own kernels key tiles
    wholly outside the window are skipped, so the work grows as S·W instead of S²/2.

    On the own kernels a masked key contributes nothing and gets dK = dV = 0, and a query row that sees no key at all gets
    O = 0 and dQ = 0.  The SDPA fallback (CPU, other dtypes or head sizes) follows SDPA's rule for such a row, which is NaN
    on some SDPA backends and versions.

    ``dropout_p`` ∈ [0, 1): attention dropout on the probabilities, by the rule of :func:`attention_dropout_keep` for
    ``dropout_seed`` (an int or a one-element int32 / int64 tensor) and global heads ``head_offset`` … ``head_offset + H − 1``
    (a tensor-parallel rank passes rank · H).  Without a seed one is drawn from the default generator of q's device, on the
    device, so activation checkpointing, which restores that generator, recomputes the same mask.  Off the kernels, p > 0
    runs the explicit softmax with that mask (a host computation), so a seed drops the same elements on every path."""
    window = _window_args("flash_attention", causal, sliding_window)
    dropout_p = _check_dropout(dropout_p)
    scale = scale if scale is not None else 1.0 / math.sqrt(q.shape[-1])
    if flash_kernels_apply(q, k, v, causal):
        seed = _dropout_seed(dropout_seed, dropout_p, q.device) if dropout_p > 0 else None
        return _FlashAttn.apply(q, k, v, causal, scale, _kernel_mask(key_padding_mask), window, 0, True, dropout_p, seed,
                                head_offset)[0]
    if dropout_p > 0:
        seed = _dropout_seed(dropout_seed, dropout_p, q.device)
        return _dropout_attention(q, k, v, causal, scale, key_padding_mask, window or None, dropout_p, seed, head_offset)
    return _sdpa(q, k, v, causal, scale, key_padding_mask, window or None)


def check_window(sliding_window: Optional[int]) -> int:
    """``sliding_window`` (``None`` or ≥ 1) → the kernels' integer form (0 = no window); raises ``ValueError`` otherwise."""
    if sliding_window is None:
        return 0
    if int(sliding_window) < 1:
        raise ValueError(f"sliding_window must be >= 1 or None, got {sliding_window}")
    return int(sliding_window)


def check_kv_scales(k_cache: torch.Tensor, v_cache: torch.Tensor, k_scale: float, v_scale: float) -> dict:
    """The decode kernels' ``k_scale`` / ``v_scale`` keyword arguments: ``{}`` when both are 1.0 (what a bf16 cache always
    has), else both.  Raises ``ValueError`` for scales other than 1.0 on a cache that is not fp8, or for k and v caches of
    different dtypes."""
    if k_cache.dtype != v_cache.dtype:
        raise ValueError(f"k and v caches must have the same dtype, got {k_cache.dtype} and {v_cache.dtype}")
    if k_scale == 1.0 and v_scale == 1.0:
        return {}
    if k_cache.dtype not in FP8_KV_DTYPES:
        raise ValueError(f"k_scale / v_scale apply to fp8 caches only; got a {k_cache.dtype} cache with scales "
                         f"({k_scale}, {v_scale})")
    return {"k_scale": float(k_scale), "v_scale": float(v_scale)}


def check_rolling(name: str, rolling: bool, window: int, length: int, W: Optional[int] = None) -> None:
    """A rolling cache of L = ``length`` rows (position t in row t mod L) needs a sliding window: 0 < window < L for one
    token per sequence (``W`` None), window + W − 1 ≤ L for W verified tokens.  Token w of a window writes row (p + w) mod L
    over position p + w − L, which must be invisible to every token of the window, and each sees only positions
    > p − window.  Raises ``ValueError``."""
    if not rolling:
        return
    if W is None and not 0 < window < length:
        raise ValueError(f"{name}: a rolling cache of {length} rows needs 0 < sliding_window < {length}, got {window or None}")
    if W is not None and not (window > 0 and window + W - 1 <= length):
        raise ValueError(f"{name}: a rolling cache of {length} rows needs a sliding_window with sliding_window + W - 1 <= "
                         f"{length} for W = {W} tokens, got {window or None}")


def decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, positions: torch.Tensor,
                     scale: Optional[float] = None, sliding_window: Optional[int] = None, k_scale: float = 1.0,
                     v_scale: float = 1.0, rolling: bool = False) -> torch.Tensor:
    """One new token per sequence against a KV cache: ``q [B,1,H,D]``, caches ``[B,L,Hkv,D]`` (any batch / sequence / head
    strides), ``positions [B]`` = cache index of the newest token (keys ≤ position are visible; with ``sliding_window`` W only
    keys position − W < j ≤ position, and the kernel reads only those rows).  An fp8 cache holds k / ``k_scale`` and
    v / ``v_scale`` (one scale per tensor, as ``inference.kv_cache.KVCacheManager`` stores it).  ``rolling``: the cache is a
    ring of L rows holding position j in row j mod L (``KVCacheManager`` in rolling mode); needs 0 < W < L.

    This is the W = 1 chain of :func:`speculation_attention` (one token in slot p = position, seeing slots ≤ p), with the
    stricter ring condition of a single token.  CUDA bf16 q with a bf16 or fp8 e4m3 cache and a head_dim in
    :data:`FLASH_HEAD_DIMS`: the split-KV flash-decoding kernel (``csrc/decode.cu``), which reads the e4m3 bytes directly;
    otherwise :func:`speculation_attention_torch`."""
    B, _, H, D = q.shape
    Hkv, L = k_cache.shape[2], k_cache.shape[1]
    window = check_window(sliding_window)
    check_rolling("decode_attention", rolling, window, L)
    kw = check_kv_scales(k_cache, v_cache, k_scale, v_scale)
    if rolling:
        kw["rolling"] = True
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    e = _ext.ext() if q.is_cuda else None
    if (e is not None and hasattr(e, "decode_attention") and D in FLASH_HEAD_DIMS and q.dtype == torch.bfloat16
            and k_cache.dtype in (torch.bfloat16, torch.float8_e4m3fn) and H // Hkv in DECODE_GQA_GROUPS and k_cache.stride(3) == 1
            and v_cache.stride(3) == 1):
        _ext.count_launch(2)
        return e.decode_attention(q.contiguous(), k_cache, v_cache, positions.to(torch.long).contiguous(), float(scale), window,
                                  **kw)
    return speculation_attention_torch(q, k_cache, v_cache, positions, sliding_window=sliding_window, scale=scale,
                                       k_scale=k_scale, v_scale=v_scale, rolling=rolling)


#: most new tokens per sequence the speculation kernel verifies in one call
SPEC_MAX_TOKENS = 64


def _check_spec_args(q, k_cache, v_cache, tree_mask, tree_depth, sliding_window, k_scale, v_scale, rolling=False):
    """Argument checks of :func:`speculation_attention` → ``(window, scale kwargs)``; raises ``ValueError``."""
    if q.dim() != 4 or k_cache.dim() != 4 or v_cache.shape != k_cache.shape:
        raise ValueError(f"speculation_attention: expected q [B,W,H,D] and caches [B,L,Hkv,D], got {tuple(q.shape)}, "
                         f"{tuple(k_cache.shape)} and {tuple(v_cache.shape)}")
    B, W, H, D = q.shape
    if k_cache.shape[0] != B or k_cache.shape[3] != D or H % k_cache.shape[2]:
        raise ValueError(f"speculation_attention: q {tuple(q.shape)} does not match the caches {tuple(k_cache.shape)}")
    if (tree_mask is None) != (tree_depth is None):
        raise ValueError("speculation_attention: tree_mask and tree_depth go together")
    if tree_mask is not None and (tuple(tree_mask.shape) != (W, W) or tuple(tree_depth.shape) != (W,)):
        raise ValueError(f"speculation_attention: tree_mask must be [W, W] and tree_depth [W] for W = {W}, got "
                         f"{tuple(tree_mask.shape)} and {tuple(tree_depth.shape)}")
    window = check_window(sliding_window)
    check_rolling("speculation_attention", rolling, window, k_cache.shape[1], W)
    return window, check_kv_scales(k_cache, v_cache, k_scale, v_scale)


def speculation_visibility(positions: torch.Tensor, length: int, W: int, tree_mask: Optional[torch.Tensor] = None,
                           tree_depth: Optional[torch.Tensor] = None, window: int = 0, rolling: bool = False) -> torch.Tensor:
    """``[B, W, length]`` bool: which cache slots each of W new tokens sees (the rule of :func:`speculation_attention`; at
    W = 1 that of one-token decode: slot c is seen iff c ≤ p and, with a window, c > p − window).  ``rolling``: slot c is a
    row of a ring of ``length`` rows: window column (c − p) mod length when that is < W, else the newest committed position
    p − 1 − ((p − 1 − c) mod length), which is seen only when ≥ 0."""
    dev = positions.device
    p = positions.long()[:, None]                                                          # [B, 1]
    d = torch.arange(W, device=dev) if tree_depth is None else tree_depth.to(dev).long()
    m = torch.ones(W, W, dtype=torch.bool, device=dev).tril() if tree_mask is None else tree_mask.to(dev).bool()
    c = torch.arange(length, device=dev)[None, :]                                          # [1, L]
    if rolling:
        u = (c - p) % length                                                               # [B, L] window column of slot c
        inside = u < W
        cpos = p - 1 - (p - 1 - c) % length                                                # committed position of slot c
        committed = ~inside & (cpos >= 0)
    else:
        u = c - p
        inside = (u >= 0) & (u < W)
        cpos, committed = c, u < 0
    uc = u.clamp(0, W - 1)
    vis = committed[:, None, :] | (inside[:, None, :] & m[:, uc].permute(1, 0, 2))        # [B, W, L]
    if window > 0:
        kpos = torch.where(inside, p + d[uc], cpos)                                        # sequence position of slot c
        vis = vis & (kpos[:, None, :] > (p + d[None, :])[:, :, None] - window)
    return vis


def speculation_attention_torch(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, positions: torch.Tensor,
                                tree_mask: Optional[torch.Tensor] = None, tree_depth: Optional[torch.Tensor] = None,
                                sliding_window: Optional[int] = None, scale: Optional[float] = None, k_scale: float = 1.0,
                                v_scale: float = 1.0, rolling: bool = False) -> torch.Tensor:
    """The torch path of :func:`speculation_attention` (any device and dtype): SDPA with a ``[B, 1, W, L]`` mask on the
    de-quantised cache, K / V repeated over the GQA group."""
    window, _ = _check_spec_args(q, k_cache, v_cache, tree_mask, tree_depth, sliding_window, k_scale, v_scale, rolling)
    B, W, H, D = q.shape
    Hkv, L = k_cache.shape[2], k_cache.shape[1]
    if k_cache.dtype in FP8_KV_DTYPES:
        k_cache, v_cache = (k_cache.float() * k_scale).to(q.dtype), (v_cache.float() * v_scale).to(q.dtype)
    qt, kt, vt = q.transpose(1, 2), k_cache.transpose(1, 2), v_cache.transpose(1, 2)
    if H != Hkv:
        kt, vt = kt.repeat_interleave(H // Hkv, 1), vt.repeat_interleave(H // Hkv, 1)
    mask = speculation_visibility(positions, L, W, tree_mask, tree_depth, window, rolling)[:, None]
    return F.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, scale=scale).transpose(1, 2)


def speculation_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, positions: torch.Tensor,
                          tree_mask: Optional[torch.Tensor] = None, tree_depth: Optional[torch.Tensor] = None,
                          sliding_window: Optional[int] = None, scale: Optional[float] = None, k_scale: float = 1.0,
                          v_scale: float = 1.0, rolling: bool = False) -> torch.Tensor:
    """W new tokens per sequence against a KV cache, as speculative decoding and Medusa verify them: ``q [B,W,H,D]``,
    caches ``[B,L,Hkv,D]`` (any batch / sequence / head strides), ``positions [B]``.  Token w of sequence b occupies cache
    slot p + w (p = ``positions[b]``) and sits at sequence position p + d[w], with d = ``tree_depth`` (a chain: d[w] = w).
    Its window mask row is ``tree_mask[w]`` ([W, W], True = sees that window column; a chain: the lower triangle).

    Token w sees slot c iff c < p (the committed sequence) and, with ``sliding_window`` SW, c > p + d[w] − SW; or
    c = p + u with ``tree_mask[w, u]`` and, with SW, d[u] > d[w] − SW.  Slots ≥ p + W and ≥ L are never seen; a token that
    sees nothing gets 0.  An fp8 cache holds k / ``k_scale`` and v / ``v_scale``.  ``rolling``: the cache is a ring of L
    rows holding slot c in row c mod L (``KVCacheManager`` in rolling mode); needs SW > 0 and SW + W − 1 ≤ L, and the rule
    above then applies to logical slots without the bound at L.

    CUDA bf16 q with a head_dim in :data:`FLASH_HEAD_DIMS`, W ≤ 64, H / Hkv in :data:`DECODE_GQA_GROUPS` and a bf16 or fp8 e4m3 cache whose
    rows are aligned as :func:`decode_attention` needs: the kernel in ``csrc/attention_sm90.cu``, which reads each K / V
    row once for all W tokens and the GQA group, reads e4m3 as stored, and with a window only the slots some token can see.
    ``tree_mask`` and ``tree_depth`` are never read on the host there, so the call can be captured in a CUDA graph.  Otherwise
    :func:`speculation_attention_torch`."""
    window, kw = _check_spec_args(q, k_cache, v_cache, tree_mask, tree_depth, sliding_window, k_scale, v_scale, rolling)
    if rolling:
        kw["rolling"] = True
    B, W, H, D = q.shape
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    e = _ext.ext() if q.is_cuda else None
    align = 16 if k_cache.dtype == torch.bfloat16 else 8
    if (e is not None and hasattr(e, "speculation_attention") and D in FLASH_HEAD_DIMS and q.dtype == torch.bfloat16
            and k_cache.dtype in (torch.bfloat16, torch.float8_e4m3fn) and W <= SPEC_MAX_TOKENS
            and H // k_cache.shape[2] in DECODE_GQA_GROUPS
            and all(t.stride(3) == 1 and t.data_ptr() % align == 0 and all(s % 8 == 0 for s in t.stride()[:3])
                    for t in (k_cache, v_cache))):
        if tree_mask is not None:
            tree_mask, tree_depth = tree_mask.to(q.device).contiguous(), tree_depth.to(q.device, torch.long).contiguous()
        _ext.count_launch(2)
        return e.speculation_attention(_tma_view(q), k_cache, v_cache, positions.to(torch.long).contiguous(), tree_mask,
                                       tree_depth, scale=float(scale), window=window, **kw)
    return speculation_attention_torch(q, k_cache, v_cache, positions, tree_mask, tree_depth, sliding_window, scale, k_scale,
                                       v_scale, rolling)
