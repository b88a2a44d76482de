"""KV-cache manager (role of reference ``examples/inference/modules/kvcache/kv_cache_manager.py:60-199``):
persistent per-layer K/V buffers ``[B, S_max, H_kv_local, D]`` allocated once (CUDA-graph safe), prefill writes a
whole prompt, decode scatters one position per sequence; optional fp8 storage (``KVQuantizationConfig``) and
flash-decoding layout where the sequence axis is additionally sharded inside a KV-replica group.

Rolling mode (``rolling_window`` = the model's sliding window SW): the cache keeps R = min(max_seq_len, SW + 64) rows and
logical position t lives in row t mod R.  64 is ``ops.attention.SPEC_MAX_TOKENS``: a verification window of W ≤ 64 tokens
at position p writes row (p + w) mod R over position p + w − R ≤ p − SW, and no token of the window sees a position
≤ p − SW (each sees committed positions > p + d − SW ≥ p − SW), so R ≥ SW + W − 1 keeps every visible position in the
ring.  Positions stay bounded by max_seq_len (the RoPE tables).  When R == max_seq_len the layout is the linear one and
the cache is not rolling.  This class is the only place that maps positions to rows."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from ..ops.attention import SPEC_MAX_TOKENS
from ..quantization.quantization_config import KVQuantizationConfig, QuantizationType


def per_tensor(kv_quant: KVQuantizationConfig) -> bool:
    """True when ``kv_quant`` asks for one scale per tensor, the only granularity this cache implements."""
    return (not kv_quant.per_key and kv_quant.k_quant_method == QuantizationType.PER_TENSOR_SYMMETRIC
            and kv_quant.v_quant_method == QuantizationType.PER_TENSOR_SYMMETRIC)


class KVCacheManager:
    def __init__(self, num_layers: int, batch_size: int, max_seq_len: int, num_kv_heads_local: int, head_dim: int,
                 dtype: torch.dtype = torch.bfloat16, device=None, kv_quant: Optional[KVQuantizationConfig] = None,
                 num_cores_per_group: int = 1, rolling_window: Optional[int] = None):
        """``rolling_window``: keep a ring of ``min(max_seq_len, rolling_window + 64)`` rows (module docstring); ``rolling``
        is True when that is shorter than ``max_seq_len``, and ``rows`` is the row count either way."""
        self.num_layers, self.batch_size, self.max_seq_len = num_layers, batch_size, max_seq_len
        self.kv_quant = kv_quant
        self.seq_shards = num_cores_per_group
        store = kv_quant.quant_dtype if kv_quant is not None else dtype
        self.dtype = dtype
        s_local = max_seq_len // num_cores_per_group
        if rolling_window is not None:
            if int(rolling_window) < 1 or num_cores_per_group != 1:
                raise ValueError(f"rolling_window must be >= 1 on an unsharded cache, got {rolling_window} with "
                                 f"{num_cores_per_group} sequence shards")
            s_local = min(max_seq_len, int(rolling_window) + SPEC_MAX_TOKENS)
        self.rows = s_local
        self.rolling = rolling_window is not None and s_local < max_seq_len
        shape = (batch_size, s_local, num_kv_heads_local, head_dim)
        self.k: List[torch.Tensor] = [torch.zeros(shape, dtype=store, device=device) for _ in range(num_layers)]
        self.v: List[torch.Tensor] = [torch.zeros(shape, dtype=store, device=device) for _ in range(num_layers)]

    def _q(self, x: torch.Tensor) -> torch.Tensor:
        if self.kv_quant is None:
            return x
        return (x.float() / self.kv_quant.scale).to(self.kv_quant.quant_dtype)

    def _dq(self, x: torch.Tensor) -> torch.Tensor:
        if self.kv_quant is None:
            return x
        return (x.float() * self.kv_quant.scale).to(self.kv_quant.dequant_dtype)

    def _row(self, positions: torch.Tensor) -> torch.Tensor:
        """Cache row of each position (the identity unless rolling)."""
        return positions % self.rows if self.rolling else positions

    def _ring(self, cache: torch.Tensor, x: torch.Tensor, lengths: Optional[torch.Tensor]) -> torch.Tensor:
        """Rolling prefill of ``cache [B, R, H, D]`` from ``x [B, S, H, D]``: ring row j of sequence b takes the newest prompt
        position t < lengths[b] (default S) with t ≡ j (mod R) and keeps its content when there is none.  One gather of
        static shape, no host sync: right-padding past a prompt never reaches the ring."""
        B, S = x.shape[:2]
        R = self.rows
        last = (torch.full((B,), S, device=x.device, dtype=torch.long) if lengths is None
                else lengths.to(x.device, torch.long)).clamp(max=S)[:, None] - 1
        t = last - (last - torch.arange(R, device=x.device)[None, :]) % R          # [B, R]
        src = self._q(x.gather(1, t.clamp(min=0)[:, :, None, None].expand(B, R, *x.shape[2:])))
        keep = (t < 0)[:, :, None, None]
        if src.element_size() == 1:                                                 # where() has no fp8 kernels
            return torch.where(keep, cache.view(torch.uint8), src.view(torch.uint8)).view(cache.dtype)
        return torch.where(keep, cache, src)

    def write_prefill(self, layer: int, k: torch.Tensor, v: torch.Tensor, seq_ids: Optional[torch.Tensor] = None,
                      lengths: Optional[torch.Tensor] = None) -> None:
        """k/v ``[B, S, H, D]`` → cache rows ``seq_ids`` (default 0..B-1), positions 0..S-1.  ``lengths`` ``[B]``: the
        prompt lengths (the rest is right-padding); only a rolling cache uses them (:meth:`_ring`)."""
        S = k.shape[1]
        if self.rolling:
            rows = slice(0, k.shape[0]) if seq_ids is None else seq_ids
            for cache, x in ((self.k[layer], k), (self.v[layer], v)):
                cache[rows] = self._ring(cache[rows], x, lengths)
            return
        if seq_ids is None:
            self.k[layer][: k.shape[0], :S].copy_(self._q(k))
            self.v[layer][: v.shape[0], :S].copy_(self._q(v))
        else:
            self.k[layer][seq_ids, :S] = self._q(k)
            self.v[layer][seq_ids, :S] = self._q(v)

    def write_prefill_sharded(self, layer: int, k: torch.Tensor, v: torch.Tensor, shard_rank: int) -> None:
        """Flash-decoding layout: this rank keeps prompt positions ``[shard_rank·L_local, (shard_rank+1)·L_local)`` of the
        k/v ``[B, S, H, D]`` every member of the KV-replica group computed (reference ``kv_cache_manager.py:60-88``)."""
        self._not_rolling("write_prefill_sharded")
        l_local = self.k[layer].shape[1]
        lo = shard_rank * l_local
        hi = min(k.shape[1], lo + l_local)
        if hi > lo:
            self.k[layer][: k.shape[0], : hi - lo].copy_(self._q(k[:, lo:hi]))
            self.v[layer][: v.shape[0], : hi - lo].copy_(self._q(v[:, lo:hi]))

    def write_decode_sharded(self, layer: int, k: torch.Tensor, v: torch.Tensor, positions: torch.Tensor,
                             shard_rank: int) -> None:
        """Flash-decoding layout: k/v ``[B, 1, H, D]`` of global ``positions``, written only by the rank whose sequence
        shard holds each position."""
        from ..modules.attention.flash_decode import write_decode_sharded

        self._not_rolling("write_decode_sharded")
        write_decode_sharded(self.k[layer], self.v[layer], self._q(k), self._q(v), positions, shard_rank)

    def _not_rolling(self, name: str) -> None:
        if self.rolling:
            raise ValueError(f"KVCacheManager.{name}: the flash-decoding layout does not take a rolling cache")

    def write_window(self, layer: int, k: torch.Tensor, v: torch.Tensor, positions: torch.Tensor) -> None:
        """k/v ``[B, W, H, D]`` written at positions ``positions[b] + 0..W-1`` (decode at W = 1, speculative verification,
        chunked prefill); ``positions`` ``[B]`` is a device tensor (no host sync → graph capturable)."""
        B, W = k.shape[0], k.shape[1]
        b = torch.arange(B, device=k.device).unsqueeze(1).expand(B, W)
        pos = positions.unsqueeze(1) + torch.arange(W, device=k.device).unsqueeze(0)
        pos = self._row(pos) if self.rolling else pos.clamp(max=self.k[layer].shape[1] - 1)
        self.k[layer].index_put_((b, pos), self._q(k))
        self.v[layer].index_put_((b, pos), self._q(v))

    def compact_window(self, positions: torch.Tensor, src_offsets: torch.Tensor) -> None:
        """After tree verification: entry ``positions[b] + src_offsets[b, i]`` (an accepted tree node) moves to
        ``positions[b] + i`` for every layer, so the accepted path becomes a contiguous continuation of the sequence."""
        B, n = src_offsets.shape
        b = torch.arange(B, device=positions.device).unsqueeze(1).expand(B, n)
        src = self._row(positions.unsqueeze(1) + src_offsets)
        dst = self._row(positions.unsqueeze(1) + torch.arange(n, device=positions.device).unsqueeze(0))
        for layer in range(self.num_layers):
            self.k[layer].index_put_((b, dst), self.k[layer][b, src])
            self.v[layer].index_put_((b, dst), self.v[layer][b, src])

    def kernel_scales(self) -> Optional[Tuple[float, float]]:
        """``(k_scale, v_scale)`` when the decode kernels (``csrc/decode.cu``) can read this cache as stored, else ``None``.
        They read a bf16 cache (scales 1.0) and an fp8 e4m3 cache with one scale per tensor that de-quantises to bf16, on
        CUDA; there ``stored`` holds k / k_scale and v / v_scale, rounded by ``_q``."""
        if not self.k or not self.k[0].is_cuda:
            return None
        q = self.kv_quant
        if q is None:
            return (1.0, 1.0) if self.dtype == torch.bfloat16 else None
        if q.quant_dtype == torch.float8_e4m3fn and per_tensor(q) and q.dequant_dtype == torch.bfloat16:
            return (q.scale, q.scale)
        return None

    def stored(self, layer: int, length: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """The cache tensors of ``layer`` as stored (fp8 when quantised), positions ``[0, length)`` (a rolling cache has no
        prefix of positions: ``length`` must be None)."""
        k, v = self.k[layer], self.v[layer]
        if length is not None and self.rolling:
            raise ValueError("KVCacheManager.stored: a rolling cache has no prefix of positions; pass length=None")
        if length is not None:
            k, v = k[:, :length], v[:, :length]
        return k, v

    def get(self, layer: int, length: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        k, v = self.stored(layer, length)
        return self._dq(k), self._dq(v)

    def reset(self) -> None:
        for t in self.k + self.v:
            t.zero_()
