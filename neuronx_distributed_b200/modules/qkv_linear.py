"""Grouped-query-attention QKV projection with KV-head replication.

Capability parity with reference ``modules/qkv_linear.py:371-713`` and ``qkv_linear_utils.py``:
one module produces (q, k, v); when ``num_kv_heads < tp`` the K/V weights are replicated
``kv_size_multiplier`` times so every TP rank owns a KV head, and the K/V gradients are summed
over the *KV-shared group* (the ranks holding replicas of the same head).

H100 design: Q, K and V are computed by ONE fused column-parallel GEMM (one AG→GEMM launch
under sequence parallelism) over the concatenated ``[q/tp + 2·kv·m/tp, in]`` weight.  With
``fuse_qkv=True`` that concatenation *is* the stored parameter (``weight_qkv``).  The KV-group
gradient reduction is a separate identity-forward / all-reduce-backward node on the k and v
outputs, so it composes with the fused kernels unchanged.

Replication layout: ``"tile"`` (K0..Kn-1 repeated m times → replicas are tp/m apart; the
reference's Trn1 layout and its default KV groups) or ``"adjacent"`` (each head repeated m
times consecutively; the reference's Trn2 layout).
"""
from __future__ import annotations

import math
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch.nn import init
from torch.nn.parameter import Parameter

from ..parallel_layers import comm, mappings
from ..parallel_layers import parallel_state as ps
from ..parallel_layers.layers import BaseParallelLayer, _group_info, tp_linear
from ..parallel_layers.utils import create_local_weight, divide, set_tensor_model_parallel_attributes


class _KVGradSum(torch.autograd.Function):
    """identity forward; backward all-reduces (sum) over the KV-shared group in ``reduce_dtype``
    (reference qkv_linear_utils.py:117-144)."""

    @staticmethod
    def forward(ctx, x, group, reduce_dtype):
        ctx.group, ctx.reduce_dtype = group, reduce_dtype
        return x

    @staticmethod
    def backward(ctx, g):
        if dist.get_world_size(ctx.group) == 1:
            return g, None, None
        od = g.dtype
        gr = g.to(ctx.reduce_dtype) if ctx.reduce_dtype is not None else g.clone()
        comm.all_reduce(gr, group=ctx.group)
        return gr.to(od), None, None


def replicate_kv(weight: torch.Tensor, multiplier: int, head_dim_rows: Optional[int] = None,
                 layout: str = "tile") -> torch.Tensor:
    """Replicate a full ``[kv_size, in]`` weight ``multiplier`` times along dim 0."""
    if multiplier == 1:
        return weight
    if layout == "tile":
        return weight.repeat(multiplier, *([1] * (weight.dim() - 1)))
    assert head_dim_rows is not None
    kv_heads = weight.shape[0] // head_dim_rows
    w = weight.view(kv_heads, head_dim_rows, *weight.shape[1:])
    return w.repeat_interleave(multiplier, dim=0).reshape(kv_heads * multiplier * head_dim_rows, *weight.shape[1:])


class GQAQKVColumnParallelLinear(BaseParallelLayer):
    #: run the fused q/k/v GEMMs as row-wise scaled e4m3 products (``tp_linear(fp8=True)``), as on ``BaseParallelLinear``
    fp8_training: bool = False

    def __init__(
        self,
        input_size: int,
        output_sizes: List[int],
        bias: bool = True,
        gather_output: bool = True,
        dtype: torch.dtype = torch.float32,
        device: Optional[torch.device] = None,
        init_method: Optional[Callable[..., Any]] = None,
        sequence_parallel_enabled: bool = False,
        keep_master_weight: bool = False,
        kv_size_multiplier: int = 1,
        fuse_qkv: bool = True,
        reduce_dtype: torch.dtype = torch.float32,
        sequence_dimension: Optional[int] = 0,
        tensor_model_parallel_group=None,
        kv_replication_layout: str = "tile",
        head_dim: Optional[int] = None,
    ):
        super().__init__(device=device)
        self.input_size, self.output_sizes = input_size, list(output_sizes)
        self.gather_output, self.arg_init_method = gather_output, init_method
        self.tensor_parallel_group, tp, self._tp_rank = _group_info(tensor_model_parallel_group)
        self.tensor_model_parallel_size = tp
        self.kv_size_multiplier = kv_size_multiplier
        assert tp % kv_size_multiplier == 0, "tp size must be divisible by kv_size_multiplier"
        assert (output_sizes[1] * kv_size_multiplier) % tp == 0, "kv_size*multiplier must be divisible by tp"
        self.kv_replication_layout = kv_replication_layout
        self.head_dim = head_dim
        if kv_replication_layout == "adjacent":
            assert head_dim is not None, "adjacent replication needs head_dim"
        ps.initialize_kv_group(kv_size_multiplier, sequential_ranks_in_group=(kv_replication_layout == "adjacent"))
        self.kv_group = ps.get_kv_shared_group()
        self.q_output_size_per_partition = divide(output_sizes[0], tp)
        self.kv_output_size_per_partition = divide(output_sizes[1] * kv_size_multiplier, tp)
        self.dtype, self.keep_master_weight = dtype, keep_master_weight
        self.device = device if device is not None else torch.device("cpu")
        self.use_bias, self.fuse_qkv = bias, fuse_qkv
        self.sequence_parallel_enabled = sequence_parallel_enabled
        self.sequence_dimension = 0 if sequence_dimension is None else sequence_dimension
        self.reduce_dtype = reduce_dtype
        self.async_tensor_model_parallel_allreduce = not sequence_parallel_enabled and tp > 1
        qp, kvp = self.q_output_size_per_partition, self.kv_output_size_per_partition
        if fuse_qkv:
            # layout of the fused shard: [q_local ; k_local ; v_local] along dim 0.  The full fused
            # tensor is [Q ; K_rep ; V_rep] with stride-3-like semantics expressed by
            # `fused_qkv`/`num_attention_heads`… attrs used by the checkpoint sharder.
            self.weight_qkv = Parameter(torch.empty(qp + 2 * kvp, input_size, dtype=dtype, device=self.device))
            if bias:
                self.bias_qkv = Parameter(torch.zeros(qp + 2 * kvp, dtype=dtype, device=self.device))
            else:
                self.register_parameter("bias_qkv", None)
        else:
            self.weight_q = Parameter(torch.empty(qp, input_size, dtype=dtype, device=self.device))
            self.weight_k = Parameter(torch.empty(kvp, input_size, dtype=dtype, device=self.device))
            self.weight_v = Parameter(torch.empty(kvp, input_size, dtype=dtype, device=self.device))
            if bias:
                self.bias_q = Parameter(torch.zeros(qp, dtype=dtype, device=self.device))
                self.bias_k = Parameter(torch.zeros(kvp, dtype=dtype, device=self.device))
                self.bias_v = Parameter(torch.zeros(kvp, dtype=dtype, device=self.device))
            else:
                for n in ("bias_q", "bias_k", "bias_v"):
                    self.register_parameter(n, None)
        self.master_weights: Dict[str, torch.Tensor] = {}
        self.initialize_weight_biases()

    # ------------------------------------------------------------------ init
    def _init_full(self, rows: int) -> torch.Tensor:
        w = torch.empty(rows, self.input_size, dtype=torch.float32, device=self.device)
        if self.arg_init_method is None:
            init.kaiming_uniform_(w, a=math.sqrt(5))
        else:
            self.arg_init_method(w)
        return w

    def _rep(self, w: torch.Tensor) -> torch.Tensor:
        rows = self.head_dim if self.head_dim is not None else None
        return replicate_kv(w, self.kv_size_multiplier, rows, self.kv_replication_layout)

    def initialize_weight_biases(self) -> None:
        tp, r = self.tensor_model_parallel_size, self._tp_rank
        qp, kvp = self.q_output_size_per_partition, self.kv_output_size_per_partition
        meta = (self.weight_qkv if self.fuse_qkv else self.weight_q).device.type == "meta"
        if self.fuse_qkv:
            set_tensor_model_parallel_attributes(self.weight_qkv, True, 0, 1, num_partitions=tp)
            # extra attrs that tell sharders this is [Q;K;V]-fused with per-section sharding
            self.weight_qkv.fused_qkv = True
            self.weight_qkv.qkv_sections = (self.output_sizes[0], self.output_sizes[1] * self.kv_size_multiplier,
                                            self.output_sizes[1] * self.kv_size_multiplier)
            if self.bias_qkv is not None:
                set_tensor_model_parallel_attributes(self.bias_qkv, True, 0, 1, num_partitions=tp)
                self.bias_qkv.fused_qkv = True
                self.bias_qkv.qkv_sections = self.weight_qkv.qkv_sections
        else:
            for n in ("q", "k", "v"):
                set_tensor_model_parallel_attributes(getattr(self, f"weight_{n}"), True, 0, 1, num_partitions=tp)
                b = getattr(self, f"bias_{n}")
                if b is not None:
                    set_tensor_model_parallel_attributes(b, True, 0, 1, num_partitions=tp)
        if meta or ps.get_aot_mode():
            return
        full_q = self._init_full(self.output_sizes[0]).to(self.dtype)
        full_k = self._rep(self._init_full(self.output_sizes[1]).to(self.dtype))
        full_v = self._rep(self._init_full(self.output_sizes[1]).to(self.dtype))
        loc = {
            "q": create_local_weight(full_q, 0, qp, 1, rank=r, world_size=tp),
            "k": create_local_weight(full_k, 0, kvp, 1, rank=r, world_size=tp),
            "v": create_local_weight(full_v, 0, kvp, 1, rank=r, world_size=tp),
        }
        with torch.no_grad():
            if self.fuse_qkv:
                self.weight_qkv.copy_(torch.cat([loc["q"], loc["k"], loc["v"]], dim=0))
            else:
                for n in ("q", "k", "v"):
                    getattr(self, f"weight_{n}").copy_(loc[n])
        if self.keep_master_weight:
            self.master_weights = {"q": full_q, "k": full_k, "v": full_v}

    # --------------------------------------------------------------- forward
    def _weights(self) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        if self.fuse_qkv:
            return self.weight_qkv, self.bias_qkv
        w = torch.cat([self.weight_q, self.weight_k, self.weight_v], dim=0)
        b = torch.cat([self.bias_q, self.bias_k, self.bias_v], dim=0) if self.use_bias else None
        return w, b

    def forward(self, input: torch.Tensor):  # noqa: A002
        tp = self.tensor_model_parallel_size
        w, b = self._weights()
        in_mode = "gather" if self.sequence_parallel_enabled else ("copy" if tp > 1 else "none")
        qp, kvp = self.q_output_size_per_partition, self.kv_output_size_per_partition
        m = self.kv_size_multiplier
        out = tp_linear(input, w, None, in_mode, "none", self.sequence_dimension, self.tensor_parallel_group,
                        self.reduce_dtype, dgrad_col_scale=(qp, 1.0 / m) if m > 1 else None, fp8=self.fp8_training)
        if b is not None:
            out = out + b
        q, k, v = torch.split(out, [qp, kvp, kvp], dim=-1)
        if self.kv_size_multiplier > 1:
            k = _KVGradSum.apply(k, self.kv_group, self.reduce_dtype)
            v = _KVGradSum.apply(v, self.kv_group, self.reduce_dtype)
        if self.gather_output:
            q = mappings.gather_from_tensor_model_parallel_region(q, self.tensor_parallel_group)
            k = mappings.gather_from_tensor_model_parallel_region(k, self.tensor_parallel_group)
            v = mappings.gather_from_tensor_model_parallel_region(v, self.tensor_parallel_group)
        return q, k, v

    # ------------------------------------------------------ checkpoint hooks
    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> bool:
        """Bring a full (unsharded, un-replicated) checkpoint into the layout this module shards
        from: replicate K/V ``kv_size_multiplier`` times and, for ``fuse_qkv``, build the fused
        tensor whose dim-0 sharding yields ``[q_r; k_r; v_r]`` on rank r (reference :640-713)."""
        base = prefix.rsplit(".", 1)[0] if prefix.endswith(("weight", "bias", "weight_qkv", "weight_q")) else prefix.rstrip(".")
        tp = self.tensor_model_parallel_size

        def _get(*names):
            for n in names:
                if f"{base}.{n}" in model_state_dict:
                    return f"{base}.{n}"
            return None

        changed = False
        for kind in ("weight", "bias"):
            kq, kk, kv = _get(f"{kind}_q"), _get(f"{kind}_k"), _get(f"{kind}_v")
            if kq is None or kk is None or kv is None:
                continue
            q = model_state_dict[kq]
            k, v = model_state_dict[kk], model_state_dict[kv]
            if k.shape[0] == self.output_sizes[1]:
                k, v = self._rep(k), self._rep(v)
            if self.fuse_qkv:
                qs, ks, vs = q.chunk(tp, 0), k.chunk(tp, 0), v.chunk(tp, 0)
                fused = torch.cat([torch.cat([qs[i], ks[i], vs[i]], 0) for i in range(tp)], 0)
                model_state_dict[f"{base}.{kind}_qkv"] = fused
                for key in (kq, kk, kv):
                    del model_state_dict[key]
            else:
                model_state_dict[kk], model_state_dict[kv] = k, v
            changed = True
        return changed


# ---------------------------------------------------------------------------------------------------------------------
# functional form (reference qkv_linear.py:43-368)
# ---------------------------------------------------------------------------------------------------------------------
def gqa_qkv_linear_with_async_allreduce(input: torch.Tensor, weight_q, weight_k, weight_v, bias_q, bias_k, bias_v,  # noqa: A002
                                        async_grad_allreduce: bool, sequence_parallel_enabled: bool, kv_size_multiplier: int = 1,
                                        weight_qkv=None, bias_qkv=None, fuse_qkv: bool = False, output_size_q: Optional[int] = None,
                                        output_size_kv: Optional[int] = None, reduce_dtype: torch.dtype = torch.float32,
                                        sequence_dimension: int = 0, process_group=None, kv_group=None, fp8: bool = False):
    """``(q, k, v) = split(x · [Wq; Wk; Wv]ᵀ)`` as ONE GEMM on the local shards.

    * ``sequence_parallel_enabled`` — the input is all-gathered along the sequence dim inside the GEMM kernel (fused
      AG→GEMM over NVLink peer memory) and its gradient is reduce-scattered; otherwise ``async_grad_allreduce`` all-reduces
      the input gradient over the TP group, overlapped with the weight-gradient GEMM;
    * ``kv_size_multiplier > 1`` — K/V heads are replicated across groups of TP ranks: the K and V gradients are summed over
      the KV-shared group (``parallel_state.get_kv_shared_group``) so the replicas stay identical;
    * ``fp8`` — the GEMMs are row-wise scaled e4m3 products (``tp_linear(fp8=True)``)."""
    group = process_group if process_group is not None else ps.get_tensor_model_parallel_group()
    tp = dist.get_world_size(group)
    if fuse_qkv:
        w, b = weight_qkv, bias_qkv
        qp = output_size_q if output_size_q is not None else None
        kvp = output_size_kv
        assert qp is not None and kvp is not None, "output_size_q / output_size_kv (per-partition sizes) are required with fuse_qkv"
    else:
        w = torch.cat([weight_q, weight_k, weight_v], dim=0)
        b = torch.cat([bias_q, bias_k, bias_v], dim=0) if bias_q is not None else None
        qp, kvp = weight_q.shape[0], weight_k.shape[0]
    in_mode = "gather" if sequence_parallel_enabled else ("copy" if (async_grad_allreduce and tp > 1) else "none")
    out = tp_linear(input, w, None, in_mode, "none", sequence_dimension, group, reduce_dtype,
                    dgrad_col_scale=(qp, 1.0 / kv_size_multiplier) if kv_size_multiplier > 1 else None, fp8=fp8)
    if b is not None:
        out = out + b
    q, k, v = torch.split(out, [qp, kvp, kvp], dim=-1)
    if kv_size_multiplier > 1:
        kvg = kv_group if kv_group is not None else ps.get_kv_shared_group()
        k, v = _KVGradSum.apply(k, kvg, reduce_dtype), _KVGradSum.apply(v, kvg, reduce_dtype)
    return q, k, v


class GQAQKVLinearWithAsyncCommunication:
    """Name-compatible façade (reference :43-327): ``apply`` takes the reference's positional arguments."""

    @staticmethod
    def apply(input, weight_q, weight_k, weight_v, bias_q, bias_k, bias_v, async_grad_allreduce, sequence_parallel_enabled,  # noqa: A002
              kv_size_multiplier=1, weight_qkv=None, bias_qkv=None, fuse_qkv=False, output_size_q=None, output_size_kv=None,
              reduce_dtype=torch.float32):
        return gqa_qkv_linear_with_async_allreduce(input, weight_q, weight_k, weight_v, bias_q, bias_k, bias_v, async_grad_allreduce,
                                                   sequence_parallel_enabled, kv_size_multiplier, weight_qkv, bias_qkv, fuse_qkv,
                                                   output_size_q, output_size_kv, reduce_dtype)
