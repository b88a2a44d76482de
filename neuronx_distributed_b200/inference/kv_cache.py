"""KV-cache manager (role of reference ``examples/inference/modules/kvcache/kv_cache_manager.py:60-199``):
persistent per-layer K/V buffers ``[B, S_max, H_kv_local, D]`` allocated once (CUDA-graph safe), prefill writes a
whole prompt, decode scatters one position per sequence; optional fp8 storage (``KVQuantizationConfig``) and
flash-decoding layout where the sequence axis is additionally sharded inside a KV-replica group."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from ..quantization.quantization_config import KVQuantizationConfig, QuantizationType


def per_tensor(kv_quant: KVQuantizationConfig) -> bool:
    """True when ``kv_quant`` asks for one scale per tensor, the only granularity this cache implements."""
    return (not kv_quant.per_key and kv_quant.k_quant_method == QuantizationType.PER_TENSOR_SYMMETRIC
            and kv_quant.v_quant_method == QuantizationType.PER_TENSOR_SYMMETRIC)


class KVCacheManager:
    def __init__(self, num_layers: int, batch_size: int, max_seq_len: int, num_kv_heads_local: int, head_dim: int,
                 dtype: torch.dtype = torch.bfloat16, device=None, kv_quant: Optional[KVQuantizationConfig] = None,
                 num_cores_per_group: int = 1):
        self.num_layers, self.batch_size, self.max_seq_len = num_layers, batch_size, max_seq_len
        self.kv_quant = kv_quant
        self.seq_shards = num_cores_per_group
        store = kv_quant.quant_dtype if kv_quant is not None else dtype
        self.dtype = dtype
        s_local = max_seq_len // num_cores_per_group
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

    def write_prefill(self, layer: int, k: torch.Tensor, v: torch.Tensor, seq_ids: Optional[torch.Tensor] = None) -> None:
        """k/v ``[B, S, H, D]`` → cache rows ``seq_ids`` (default 0..B-1), positions 0..S-1."""
        S = k.shape[1]
        if seq_ids is None:
            self.k[layer][: k.shape[0], :S].copy_(self._q(k))
            self.v[layer][: v.shape[0], :S].copy_(self._q(v))
        else:
            self.k[layer][seq_ids, :S] = self._q(k)
            self.v[layer][seq_ids, :S] = self._q(v)

    def write_prefill_sharded(self, layer: int, k: torch.Tensor, v: torch.Tensor, shard_rank: int) -> None:
        """Flash-decoding layout: this rank keeps prompt positions ``[shard_rank·L_local, (shard_rank+1)·L_local)`` of the
        k/v ``[B, S, H, D]`` every member of the KV-replica group computed (reference ``kv_cache_manager.py:60-88``)."""
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

        write_decode_sharded(self.k[layer], self.v[layer], self._q(k), self._q(v), positions, shard_rank)

    def write_decode(self, layer: int, k: torch.Tensor, v: torch.Tensor, positions: torch.Tensor) -> None:
        """k/v ``[B, 1, H, D]``; ``positions`` ``[B]`` (device tensor; no host sync → graph capturable)."""
        b = torch.arange(k.shape[0], device=k.device)
        self.k[layer].index_put_((b, positions), self._q(k[:, 0]))
        self.v[layer].index_put_((b, positions), self._q(v[:, 0]))

    def write_window(self, layer: int, k: torch.Tensor, v: torch.Tensor, positions: torch.Tensor) -> None:
        """k/v ``[B, W, H, D]`` written at positions ``positions[b] + 0..W-1`` (speculative verification / chunked prefill)."""
        B, W = k.shape[0], k.shape[1]
        b = torch.arange(B, device=k.device).unsqueeze(1).expand(B, W)
        pos = (positions.unsqueeze(1) + torch.arange(W, device=k.device).unsqueeze(0)).clamp(max=self.k[layer].shape[1] - 1)
        self.k[layer].index_put_((b, pos), self._q(k))
        self.v[layer].index_put_((b, pos), self._q(v))

    def compact_window(self, positions: torch.Tensor, src_offsets: torch.Tensor) -> None:
        """After tree verification: entry ``positions[b] + src_offsets[b, i]`` (an accepted tree node) moves to
        ``positions[b] + i`` for every layer, so the accepted path becomes a contiguous continuation of the sequence."""
        B, n = src_offsets.shape
        b = torch.arange(B, device=positions.device).unsqueeze(1).expand(B, n)
        src = positions.unsqueeze(1) + src_offsets
        dst = positions.unsqueeze(1) + torch.arange(n, device=positions.device).unsqueeze(0)
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
        """The cache tensors of ``layer`` as stored (fp8 when quantised), positions ``[0, length)``."""
        k, v = self.k[layer], self.v[layer]
        if length is not None:
            k, v = k[:, :length], v[:, :length]
        return k, v

    def get(self, layer: int, length: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        k, v = self.stored(layer, length)
        return self._dq(k), self._dq(v)

    def reset(self) -> None:
        for t in self.k + self.v:
            t.zero_()
