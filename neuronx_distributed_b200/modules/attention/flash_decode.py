"""Distributed flash-decoding: the KV cache of a GQA head that is replicated over several TP ranks is *sharded along the sequence*
inside that KV-replica group instead of being stored ``n`` times (reference ``examples/inference/modules/attention/
flashdecode_attention.py:190-235``, masks ``flashdecode/util.py:9-77``, cache shape ``kv_cache_manager.py:60-88``).

Per decode step, inside a group of ``n`` ranks that share the same KV heads:
  1. all-gather the queries of the group (every rank attends for all ``n·H_local`` query heads over ITS sequence shard),
  2. local partial attention → un-normalised output, row max ``m`` and row sum ``l`` (fp32),
  3. combine across the group with the log-sum-exp rule: all-reduce(max) of ``m``, rescale, reduce-scatter(sum) of the
     outputs and of ``l`` over the head axis — each rank ends with the finished output of its own heads.
Rank ``r`` of the group owns cache positions ``[r·L_local, (r+1)·L_local)``; the new token's K/V is written only by its owner.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.distributed as dist

from ...ops.attention import FP8_KV_DTYPES


def owner_and_offset(positions: torch.Tensor, l_local: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Global cache position → (owning rank in the group, offset inside that rank's shard)."""
    return positions // l_local, positions % l_local


def write_decode_sharded(k_cache: torch.Tensor, v_cache: torch.Tensor, k_new: torch.Tensor, v_new: torch.Tensor,
                         positions: torch.Tensor, rank_in_group: int) -> None:
    """k/v_cache ``[B, L_local, Hkv, D]`` (this rank's shard); k/v_new ``[B, 1, Hkv, D]`` in the cache's dtype (already
    quantised for an fp8 cache); only the owner writes (mask, no sync)."""
    l_local = k_cache.shape[1]
    owner, off = owner_and_offset(positions, l_local)
    mine = (owner == rank_in_group)
    b = torch.arange(k_cache.shape[0], device=k_cache.device)
    off = torch.where(mine, off, torch.zeros_like(off))
    if k_cache.dtype in FP8_KV_DTYPES:                     # torch has no float8 arithmetic; a select moves the bytes unchanged
        keep = mine.view(-1, 1, 1)
        k_cache[b, off] = torch.where(keep, k_new[:, 0], k_cache[b, off])
        v_cache[b, off] = torch.where(keep, v_new[:, 0], v_cache[b, off])
        return
    keep = mine.view(-1, 1, 1).to(k_cache.dtype)
    k_cache[b, off] = keep * k_new[:, 0] + (1 - keep) * k_cache[b, off]
    v_cache[b, off] = keep * v_new[:, 0] + (1 - keep) * v_cache[b, off]


def _local_partial(q_all: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, local_pos: torch.Tensor, scale: float,
                   sliding_window: Optional[int] = None, k_scale: float = 1.0, v_scale: float = 1.0):
    """Partial attention of ``q_all [B, 1, H, D]`` over this rank's cache shard, cache index ≤ ``local_pos[b]`` visible
    (``local_pos`` may be negative: nothing visible yet), and with ``sliding_window`` W only indices > ``local_pos[b]`` − W
    (both ends shift by the shard offset, so local positions need no other change).  Returns un-normalised ``o [B, H, D]`` relative to the row maximum
    ``m [B, H]`` (natural-log units, −inf when nothing is visible) and the row sum ``l [B, H]``, all fp32.

    An fp8 cache holds k / ``k_scale`` and v / ``v_scale`` (one scale per tensor).

    CUDA / bf16 q / bf16 or e4m3 cache / head_dim in ``FLASH_HEAD_DIMS`` / H / Hkv in ``DECODE_GQA_GROUPS``: the split-KV
    decode kernel (``csrc/decode.cu`` ``decode_attn_kernel`` + the partial combine): K/V are read once per KV head for the whole GQA group.  Otherwise fp32 torch math."""
    from ...ops import _ext
    from ...ops.attention import DECODE_GQA_GROUPS, FLASH_HEAD_DIMS, check_kv_scales, check_window, speculation_visibility

    window = check_window(sliding_window)
    kw = check_kv_scales(k_cache, v_cache, k_scale, v_scale)
    B, _, H, D = q_all.shape
    l_local, Hkv = k_cache.shape[1], k_cache.shape[2]
    if (_ext.use_cuda(q_all, k_cache, v_cache) and q_all.dtype == torch.bfloat16 and k_cache.dtype in (torch.bfloat16, torch.float8_e4m3fn)
            and D in FLASH_HEAD_DIMS and H % Hkv == 0 and (H // Hkv) in DECODE_GQA_GROUPS and hasattr(_ext.ext(), "decode_attention_partial")):
        _ext.count_launch(2)
        o, ml = _ext.ext().decode_attention_partial(q_all.contiguous(), k_cache, v_cache, local_pos.to(torch.long).contiguous(),
                                                    float(scale), window, **kw)
        return o, ml[..., 0], ml[..., 1]
    g = H // Hkv
    kf = (k_cache.float() * k_scale if kw else k_cache.float()).repeat_interleave(g, dim=2)    # [B, L_local, H, D]
    vf = (v_cache.float() * v_scale if kw else v_cache.float()).repeat_interleave(g, dim=2)
    s = torch.einsum("bhd,blhd->bhl", q_all[:, 0].float(), kf) * scale  # [B, H, L_local]
    valid = speculation_visibility(local_pos, l_local, 1, window=window)[:, 0]                  # [B, L_local]
    s = s.masked_fill(~valid[:, None, :], float("-inf"))
    m = s.max(dim=-1).values                                            # [B, H]  (−inf if this shard has nothing yet)
    p = torch.exp(s - torch.where(torch.isinf(m), torch.zeros_like(m), m).unsqueeze(-1))
    p = torch.where(valid[:, None, :], p, torch.zeros_like(p))
    return torch.einsum("bhl,blhd->bhd", p, vf), m, p.sum(-1)


def flash_decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, positions: torch.Tensor,
                           group, scale: Optional[float] = None, sliding_window: Optional[int] = None, k_scale: float = 1.0,
                           v_scale: float = 1.0) -> torch.Tensor:
    """q ``[B, 1, H_local, D]`` (this rank's query heads), caches ``[B, L_local, Hkv, D]`` (this rank's sequence shard of the
    shared KV heads), ``positions`` ``[B]`` = index of the newest token (attend to ≤ position; with ``sliding_window`` W only
    to the last W positions).  An fp8 cache holds k / ``k_scale`` and v / ``v_scale``.  Returns ``[B, 1, H_local, D]``.
    Collectives go through ``parallel_layers.comm`` (NCCL / gloo; recordable in launch plans)."""
    from ...parallel_layers import comm

    n = dist.get_world_size(group)
    r = dist.get_rank(group)
    B, _, Hl, D = q.shape
    l_local = k_cache.shape[1]
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    # 1. every rank needs the queries of the whole group.  Heads are ordered (local head, rank): the group members share the
    #    same Hkv local KV heads and local query head j belongs to KV head j // (Hl / Hkv) on every member, so this order keeps
    #    the GQA mapping "head i → KV head i // (n·Hl / Hkv)" valid for any number of local KV heads
    if n > 1:
        q_all = comm.all_gather(q.unsqueeze(3).contiguous(), dim=3, group=group).reshape(B, 1, Hl * n, D)
    else:
        q_all = q
    # 2. partial attention over the local shard: global position p is local index p − r·L_local
    o, m, l = _local_partial(q_all, k_cache, v_cache, positions - r * l_local, scale, sliding_window, k_scale, v_scale)
    # 3. combine across the group
    if n > 1:
        m_glob = comm.all_reduce(m.clone(), op="max", group=group)
        w = torch.where(torch.isinf(m), torch.zeros_like(m), torch.exp(m - m_glob))
        ol = torch.cat([o * w.unsqueeze(-1), (l * w).unsqueeze(-1)], dim=-1)             # [B, Hl·n, D+1]: ONE reduce-scatter
        mine = comm.reduce_scatter(ol.view(B, Hl, n, D + 1), dim=2, group=group)[:, :, 0]  # this rank's column of (head, rank)
        o_mine, l_mine = mine[..., :D], mine[..., D]
    else:
        o_mine, l_mine = o, l
    return (o_mine / l_mine.clamp(min=1e-30).unsqueeze(-1)).to(q.dtype).unsqueeze(1)
