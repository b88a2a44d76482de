"""Tensor-parallel layers.

Capability parity with reference ``parallel_layers/layers.py`` (``ParallelEmbedding`` :186,
``LinearWithAsyncCommunication`` :434, ``ColumnParallelLinear`` :561, ``RowParallelLinear``
:815, conv layers :1309/:1432, ``SPMDRank`` :1543) and ``layers_utils.py:16-140``.

H100 design notes
-----------------
* A TP linear is ONE autograd node (:class:`_TPLinear`) covering gather → GEMM → reduce in
  both directions, so the forward and backward each map to a single fused GEMM+collective
  kernel (``ops/tp_fused.py``: AG→GEMM, GEMM→RS, GEMM→AR over NVLink peer memory) instead of
  an autograd chain of separate collective and matmul nodes.  The same node falls back to
  NCCL/gloo collectives + ``torch.matmul`` for CPU mode, unsupported shapes/dtypes, and the
  ``nccl`` baseline backend.
* Weight init is TP-degree independent: build the full fp32 master weight from the default
  RNG, cast, keep this rank's (strided) slice.
* Row-parallel reductions honour ``reduce_dtype`` (fp32 default, as the reference) on the
  library path; the fused path accumulates in fp32 and moves bf16 on the wire (documented in
  DESIGN.md).
"""
from __future__ import annotations

import math
import os
import warnings
from typing import Any, Callable, Dict, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import nn
from torch.nn import init
from torch.nn.parameter import Parameter

from ..utils.logger import get_logger
from . import comm, mappings
from . import parallel_state as ps
from .random import get_rng_tracker
from .utils import (
    EmbeddingUtility,
    create_local_weight,
    divide,
    get_padding_length,
    set_tensor_model_parallel_attributes,
)

logger = get_logger()

_SP_ATTR = "sequence_parallel_enabled"


def _tag_sequence_parallel(param: torch.Tensor, enabled: bool) -> None:
    setattr(param, _SP_ATTR, enabled)


# --------------------------------------------------------------------------------------
# parameter initialisation
# --------------------------------------------------------------------------------------
def _initialize_parameter_from_master(
    param: torch.Tensor,
    partition_dim: int,
    num_partitions: int,
    init_method: Callable[[torch.Tensor], Any],
    return_master_param: bool = False,
    param_dtype: torch.dtype = torch.float32,
    stride: int = 1,
    rank: Optional[int] = None,
) -> Optional[torch.Tensor]:
    """Initialise the *full* fp32 weight (identical on all ranks) and copy this rank's slice
    into ``param`` — results do not depend on the TP degree (reference layers.py:111-164)."""
    if not hasattr(param, "tensor_model_parallel"):          # re-initialisation keeps the attributes it already has
        set_tensor_model_parallel_attributes(param, True, partition_dim, stride, num_partitions)
    if ps.get_aot_mode() or param.device.type == "meta":
        return None
    shape = list(param.shape)
    shape[partition_dim] *= num_partitions
    # the full weight is drawn from the *default* generator of the parameter's device: identical on
    # every TP rank (same seed), on the GPU when the layer was constructed with device=cuda (fast path
    # for multi-billion-parameter models), on the CPU otherwise.
    master = torch.empty(shape, dtype=torch.float32, device=param.device)
    init_method(master)
    master = master.to(param_dtype)
    with torch.no_grad():
        local = create_local_weight(
            master, partition_dim, param.shape[partition_dim], stride, rank=rank, world_size=num_partitions
        )
        param.copy_(local.to(param.device))
    return master if return_master_param else None


def _initialize_parameter_sharded(
    param: torch.Tensor, partition_dim: int, num_partitions: int, init_method, stride: int = 1
) -> None:
    """Initialise only the local shard under the TP-forked RNG stream (cheaper; results depend
    on TP degree) — reference ``_initialize_affine_weight_neuron`` layers.py:60-84."""
    set_tensor_model_parallel_attributes(param, True, partition_dim, stride, num_partitions)
    if param.device.type == "meta":
        return
    with get_rng_tracker().fork():
        init_method(param)


class ProcessGroupSafeDeepcopy:
    """Mixin: ``copy.deepcopy`` of a module that stores process groups.  Groups are shared by reference (they cannot be
    pickled / copied) and the parallel attributes on parameters survive the copy (``Parameter.__deepcopy__`` drops custom
    attributes; bound-method attributes such as state-dict hooks are re-bound to nothing and simply carried over)."""

    def __deepcopy__(self, memo):
        import copy

        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if isinstance(v, dist.ProcessGroup):
                new.__dict__[k] = v
            else:
                new.__dict__[k] = copy.deepcopy(v, memo)
        for (_, p_old), (_, p_new) in zip(self.named_parameters(recurse=False), new.named_parameters(recurse=False)):
            for ak, av in p_old.__dict__.items():
                if not hasattr(p_new, ak):
                    setattr(p_new, ak, av)
        return new


class BaseParallelLayer(ProcessGroupSafeDeepcopy, nn.Module):
    """Brings up a single-rank parallel state if the user never initialised one
    (reference layers.py:167-183)."""

    def __init__(self, device: Optional[torch.device] = None):
        super().__init__()
        if not ps.model_parallel_is_initialized():
            warnings.warn("parallel state is not initialized; falling back to a single-rank world")
            ps.initialize_fallback_parallel_state()


class BaseParallelLinear(BaseParallelLayer):
    """Common base of the TP linears (reference layers.py:535-558): default initialisers and the inference-only guard for
    padded layers."""

    arg_init_method: Optional[Callable[..., Any]] = None
    pad: bool = False
    #: run the layer's GEMMs as row-wise scaled e4m3 products (``tp_linear(fp8=True)``); parameters and checkpoints are unchanged
    fp8_training: bool = False

    def _init_weight(self, w: torch.Tensor) -> None:
        if self.arg_init_method is None:
            init.kaiming_uniform_(w, a=math.sqrt(5))
        else:
            self.arg_init_method(w)

    def _check_pad_false_for_training(self) -> None:
        if self.pad and self.training:
            raise RuntimeError("`pad=True` is only supported for inference. Set model.eval()")


def _group_info(group) -> Tuple[Any, int, int]:
    if group is None:
        # default TP group: honour the cached size/rank overrides (reference parallel_state.py:895-926), which is how
        # ``inference.NxDParallelState`` builds any rank's shard in a single process for offline checkpoint sharding
        return ps.get_tensor_model_parallel_group(), ps.get_tensor_model_parallel_size(), ps.get_tensor_model_parallel_rank()
    return group, dist.get_world_size(group), dist.get_rank(group)


# --------------------------------------------------------------------------------------
# SPMDRank
# --------------------------------------------------------------------------------------
class SPMDRank(nn.Module):
    """Holds this rank's index as a *weight* so one captured program can be replayed on all
    ranks with only the weights differing (reference layers.py:1543-1603)."""

    def __init__(self, world_size: int, tensor_model_parallel_size: Optional[int] = None):
        super().__init__()
        self.world_size = world_size
        tp = tensor_model_parallel_size or world_size
        self.rank = Parameter(torch.zeros(1, dtype=torch.int32), requires_grad=False)
        set_tensor_model_parallel_attributes(self.rank, True, 0, 1, num_partitions=tp)
        try:
            self.rank.data.fill_(ps.get_tensor_model_parallel_rank())
        except AssertionError:
            pass

    def get_rank(self) -> torch.Tensor:
        return self.rank

    def initialize_expert_indices(self, num_local_experts: int) -> Parameter:
        """Per-rank list of the expert ids this rank owns, kept as a WEIGHT ``[1, num_local_experts]`` (dim 0 sharded over
        the world) so that one captured program serves every rank (reference layers.py:1571-1593).  Filled for the current
        EP rank; a full checkpoint provides ``[world, num_local_experts]``."""
        self.local_expert_indices = Parameter(torch.zeros((1, num_local_experts), dtype=torch.int32), requires_grad=False)
        set_tensor_model_parallel_attributes(self.local_expert_indices, True, 0, 1, num_partitions=self.world_size)
        try:
            ep, r = ps.get_expert_model_parallel_size(), ps.get_expert_model_parallel_rank()
            ids = ps.get_experts_for_expert_parallel_rank(r, num_local_experts * ep, ep)
            self.local_expert_indices.data.copy_(torch.as_tensor(ids, dtype=torch.int32).view(1, -1))
        except AssertionError:
            pass
        return self.local_expert_indices

    def get_local_expert_indices(self) -> torch.Tensor:
        return self.local_expert_indices

    def forward(self) -> torch.Tensor:
        return self.rank

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        # full tensor is arange(world) so that sharding dim 0 hands every rank its id
        key = prefix if prefix.endswith("rank") else prefix + "rank"
        model_state_dict[key] = torch.arange(0, self.world_size, dtype=torch.int32)


# --------------------------------------------------------------------------------------
# Embedding
# --------------------------------------------------------------------------------------
class _EmbeddingRS(torch.autograd.Function):
    """``embedding_rs``: ids ``[B, S]`` → this rank's sequence shard ``[S/tp, B, H]`` of the vocabulary-parallel lookup, by
    pulling each row from the rank that owns it (``ops.nvls.embedding_gather``) instead of a masked local lookup of all S·B
    rows + reduce-scatter (reference layers.py:334-378).  Backward = the transpose of the reference path: all-gather the
    output gradient along the sequence, scatter-add the rows of the locally owned ids into the shard's gradient."""

    @staticmethod
    def forward(ctx, ids, weight, group, start):
        from .. import ops

        n, r = dist.get_world_size(group), dist.get_rank(group)
        B, S = ids.shape
        assert S % n == 0, f"sequence length {S} is not divisible by the tensor-parallel size {n}"
        mine = ids[:, r * (S // n):(r + 1) * (S // n)].t().contiguous()            # [S/tp, B]
        out = ops.nvls.embedding_gather(mine, weight, group)                      # [S/tp, B, H]
        ctx.save_for_backward(ids)
        ctx.group, ctx.start, ctx.shape, ctx.dtype = group, start, weight.shape, weight.dtype
        return out

    @staticmethod
    def backward(ctx, gy):
        (ids,) = ctx.saved_tensors
        g_full = comm.all_gather(gy.contiguous(), dim=0, group=ctx.group)          # [S, B, H]
        local = ids.t().reshape(-1) - ctx.start                                    # [S·B] in (s, b) order
        ok = (local >= 0) & (local < ctx.shape[0])
        gw = torch.zeros(ctx.shape, dtype=g_full.dtype, device=g_full.device)
        gw.index_add_(0, torch.where(ok, local, torch.zeros_like(local)),
                      g_full.reshape(-1, g_full.shape[-1]) * ok.unsqueeze(-1).to(g_full.dtype))
        return None, gw.to(ctx.dtype), None, None


_EMBEDDING_RS = os.environ.get("NXD_EMBEDDING_RS", "0") == "1"     # opt-in until the kernels have run on hardware


class ParallelEmbedding(BaseParallelLayer):
    """Embedding sharded along the vocabulary (default) or the embedding dim.

    Vocab sharding: ids outside ``[start, end)`` are looked up as row 0 and zeroed, then the
    partial embeddings are summed across TP — by all-reduce, or by reduce-scatter straight into
    the sequence-parallel ``[S/tp, B, H]`` layout (reference layers.py:334-378)."""

    def __init__(
        self,
        num_embeddings: int,
        embedding_dim: int,
        padding_idx: Optional[int] = None,
        max_norm: Optional[float] = None,
        norm_type: float = 2.0,
        scale_grad_by_freq: bool = False,
        sparse: bool = False,
        init_method: Callable[[Any], Any] = init.normal_,
        device: Optional[torch.device] = None,
        dtype: torch.dtype = torch.float32,
        shard_across_embedding: bool = False,
        pad: bool = False,
        sequence_parallel_enabled: bool = False,
        tensor_model_parallel_group=None,
        use_spmd_rank: bool = False,
        sequence_dimension: Optional[int] = None,
        tile_cc: bool = False,
        rank_ordering: Optional[Sequence[int]] = None,
        collect_output: bool = True,
    ):
        super().__init__(device=device)
        self.num_embeddings, self.embedding_dim = num_embeddings, embedding_dim
        self.padding_idx, self.max_norm, self.norm_type = padding_idx, max_norm, norm_type
        self.scale_grad_by_freq, self.sparse = scale_grad_by_freq, sparse
        self.tensor_model_parallel_group, self.tensor_model_parallel_size, tp_rank = _group_info(
            tensor_model_parallel_group
        )
        self.shard_across_embedding = shard_across_embedding
        self.pad, self.pad_size = pad, 0
        self.sequence_parallel_enabled = sequence_parallel_enabled
        self.sequence_dim = sequence_dimension
        self.rank_ordering = rank_ordering
        self.collect_output = collect_output
        self.dtype, self.init_method, self.stride = dtype, init_method, 1
        self.rank_util = SPMDRank(self.tensor_model_parallel_size) if use_spmd_rank else None
        tp = self.tensor_model_parallel_size
        if shard_across_embedding:
            if pad:
                self.pad_size = get_padding_length(embedding_dim, tp)
                self.embedding_dim += self.pad_size
            self.num_embeddings_per_partition = num_embeddings
            self.embedding_dim_per_partition = divide(self.embedding_dim, tp)
            self.weight_partition_dim = 1
            shape = (num_embeddings, self.embedding_dim_per_partition)
        else:
            if pad:
                self.pad_size = get_padding_length(num_embeddings, tp)
                self.num_embeddings += self.pad_size
            self.start_index, self.end_index = EmbeddingUtility.range_from_global_vocab_size(
                self.num_embeddings, tp_rank, tp
            )
            self.num_embeddings_per_partition = self.end_index - self.start_index
            self.embedding_dim_per_partition = embedding_dim
            self.weight_partition_dim = 0
            shape = (self.num_embeddings_per_partition, embedding_dim)
        device = device if device is not None else torch.device("cpu")
        self.weight = Parameter(torch.empty(*shape, device=device, dtype=dtype))
        self.init_method, self.dtype, self._tp_rank = init_method, dtype, tp_rank
        self.init_weight_cpu()
        if rank_ordering is not None:
            self.weight.rank_ordering = list(rank_ordering)

    def init_weight_cpu(self) -> None:
        """(Re-)initialise from a full master table drawn identically on every rank (reference layers.py:325-332)."""
        _initialize_parameter_from_master(
            self.weight, self.weight_partition_dim, self.tensor_model_parallel_size, self.init_method,
            param_dtype=self.dtype, rank=self._tp_rank
        )

    def _embed(self, ids: torch.Tensor) -> torch.Tensor:
        return F.embedding(
            ids.long(), self.weight, self.padding_idx, self.max_norm, self.norm_type, self.scale_grad_by_freq, self.sparse
        )

    def forward(self, input_: torch.Tensor) -> torch.Tensor:
        if self.pad and self.training:
            raise RuntimeError("`pad=True` is only supported for inference. Set model.eval()")
        if self.shard_across_embedding:
            out = self._embed(input_)
            if self.collect_output:
                out = mappings.gather_from_tensor_model_parallel_region(out, self.tensor_model_parallel_group)
            if self.pad and self.pad_size > 0 and self.collect_output:
                out = out.narrow(-1, 0, self.embedding_dim - self.pad_size)
            return out
        tp = self.tensor_model_parallel_size
        if self._use_embedding_rs(input_):
            return _EmbeddingRS.apply(input_, self.weight, self.tensor_model_parallel_group, self.start_index)
        if tp > 1:
            if self.rank_util is not None:
                start = self.num_embeddings_per_partition * self.rank_util.get_rank().to(input_.device).long()
                end = start + self.num_embeddings_per_partition
            else:
                start, end = self.start_index, self.end_index
            mask = (input_ >= start) & (input_ < end)
            ids = (input_ - start) * mask
        else:
            mask, ids = None, input_
        out = self._embed(ids)
        if mask is not None:
            out = out * mask.unsqueeze(-1).to(out.dtype)
        if not self.collect_output:
            return out
        if self.sequence_parallel_enabled:
            if self.sequence_dim is not None:
                return mappings.reduce_scatter_to_sequence_parallel_region(
                    out, self.sequence_dim, self.tensor_model_parallel_group
                )
            # default layout contract: [B, S] ids → [S/tp, B, H]
            return mappings.reduce_scatter_to_sequence_parallel_region(
                out.transpose(0, 1).contiguous(), 0, self.tensor_model_parallel_group
            )
        return mappings.reduce_from_tensor_model_parallel_region(out, self.tensor_model_parallel_group)

    def _use_embedding_rs(self, input_: torch.Tensor) -> bool:
        """The remote-gather path covers the default training contract: vocab sharding with equal shards, sequence parallel,
        ``[B, S]`` ids → ``[S/tp, B, H]``, no ``F.embedding`` extras.  CPU tensors take it too when forced (tests)."""
        if not (_EMBEDDING_RS or getattr(self, "force_embedding_rs", False)):
            return False
        if (self.tensor_model_parallel_size == 1 or not self.sequence_parallel_enabled or self.sequence_dim is not None
                or not self.collect_output or self.rank_util is not None or input_.dim() != 2
                or input_.shape[1] % self.tensor_model_parallel_size
                or self.padding_idx is not None or self.max_norm is not None or self.scale_grad_by_freq or self.sparse
                or self.num_embeddings % self.tensor_model_parallel_size):
            return False
        if input_.is_cuda:
            from .. import ops

            return ops.nvls.embedding_gather_eligible(self.weight)
        return True

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        """Pad a full (unsharded) checkpoint weight so it divides by tp (reference :404-431)."""
        if not self.pad or self.pad_size == 0:
            return
        w = model_state_dict[prefix]
        if self.shard_across_embedding:
            if self.embedding_dim != w.shape[1] + self.pad_size:
                raise RuntimeError(f"State dict {prefix} has unexpected shape {tuple(w.shape)}")
            model_state_dict[prefix] = F.pad(w, (0, self.pad_size))
        else:
            if self.num_embeddings != w.shape[0] + self.pad_size:
                raise RuntimeError(f"State dict {prefix} has unexpected shape {tuple(w.shape)}")
            model_state_dict[prefix] = F.pad(w, (0, 0, 0, self.pad_size))


# --------------------------------------------------------------------------------------
# The single autograd node behind Column/Row linear layers
# --------------------------------------------------------------------------------------
def _flat2d(x: torch.Tensor) -> torch.Tensor:
    return x.reshape(-1, x.shape[-1])


def _add_to_main_grad(weight: torch.Tensor, product: Callable[[torch.Tensor, bool], Any]) -> bool:
    """The ZeRO-1 ``main_grad`` protocol of a weight gradient.  If the optimizer gave the weight an fp32 ``main_grad``,
    ``product(main_grad, accumulate)`` writes the gradient into it (overwriting while ``main_grad_fresh`` is set, the first
    contribution since ``zero_grad``), and ``_nxd_grad_ready`` tells the overlapped reduce-scatter that it is final.  Returns
    False, with nothing done, when there is no such buffer."""
    mg = getattr(weight, "main_grad", None)
    if not (mg is not None and mg.dtype == torch.float32 and mg.is_contiguous() and mg.shape == weight.shape):
        return False
    product(mg, not getattr(weight, "main_grad_fresh", False))
    weight.main_grad_fresh = False
    cb = getattr(weight, "_nxd_grad_ready", None)      # ZeRO-1 overlapped reduce-scatter: this gradient is final
    if cb is not None:
        cb(weight)
    return True


def wgrad(go2d: torch.Tensor, x2d: torch.Tensor, weight: torch.Tensor, fp8: bool = False):
    """``dW = goᵀ @ x``.  If the optimizer gave the weight an fp32 ``main_grad`` buffer (ZeRO-1 with fp32 gradient
    accumulation) the GEMM epilogue accumulates straight into it — no bf16 gradient tensor, no cast, no separate
    add kernel — and ``None`` is returned to autograd (Megatron-style gradient-accumulation fusion).

    ``fp8``: the row-wise scaled e4m3 product ``cols_t(go) · cols_t(x)ᵀ`` (``ops.gemm_fp8.fp8_wgrad``), reduce-added into the
    ``main_grad`` in fp32, or without one a fresh fp32 result cast to the weight's dtype."""
    from .. import ops
    from ..ops import gemm_fp8

    if fp8:
        if _add_to_main_grad(weight, lambda mg, acc: gemm_fp8.fp8_wgrad(go2d, x2d, out=mg, accumulate=acc)):
            return None
        return gemm_fp8.fp8_wgrad(go2d, x2d).to(weight.dtype)
    if (go2d.is_cuda and go2d.dtype == torch.bfloat16 and ops.gemm.fused_wgrad_enabled()
            and _add_to_main_grad(weight, lambda mg, acc: ops.gemm.matmul(go2d, x2d, True, False, out=mg, accumulate=acc))):
        return None
    return ops.gemm.matmul(go2d, x2d, True, False)


class _TPLinear(torch.autograd.Function):
    """``y = collective_out( collective_in(x) @ W^T )`` with its transposed backward.

    modes (``in_mode`` → ``out_mode``):
      * ``"gather"`` → ``"none"``   : Column + SP. fwd AG(seq)→GEMM ; bwd GEMM→RS(seq) + wgrad on re-gathered x
      * ``"copy"``   → ``"none"``   : Column, no SP. fwd GEMM ; bwd GEMM→AR (overlapped with wgrad)
      * ``"none"``   → ``"none"``   : plain linear on already-parallel data
      * ``"none"``   → ``"scatter"``: Row + SP. fwd GEMM→RS(seq) ; bwd AG(seq)→GEMM
      * ``"none"``   → ``"reduce"`` : Row, no SP. fwd GEMM→AR ; bwd GEMM
    Semantics follow reference layers.py:434-532 and layers_utils.py:16-140 (input is saved
    *sharded* and re-gathered in backward; dgrad collective overlaps wgrad).

    ``fp8``: the three GEMMs are the row-wise scaled e4m3 products of ``ops.gemm_fp8`` (``fp8_forward`` / ``fp8_dgrad`` /
    ``fp8_wgrad``) around the library collectives; the fused TP kernels are bf16, so they are not dispatched.
    """

    @staticmethod
    def forward(ctx, x, weight, bias, in_mode, out_mode, seq_dim, group, reduce_dtype, save_for_backward, dgrad_col_scale=None,
                fp8=False):
        from .. import ops
        from ..ops import gemm_fp8

        ctx.in_mode, ctx.out_mode, ctx.seq_dim, ctx.group = in_mode, out_mode, seq_dim, group
        ctx.dgrad_col_scale = dgrad_col_scale
        ctx.reduce_dtype = reduce_dtype
        ctx.has_bias = bias is not None
        ctx.x_requires_grad = x.requires_grad
        ctx.fp8 = fp8
        n = dist.get_world_size(group)
        fused = None if fp8 else ops.tp_fused.dispatch(x, weight, in_mode, out_mode, seq_dim, group)
        if fused is not None:
            ctx.fused = True
            y = fused.forward(x, weight)
            gathered = getattr(fused, "gathered", None)
            ctx.has_gathered = gathered is not None
            if save_for_backward:
                if gathered is not None:
                    ctx.save_for_backward(x, weight, gathered)
                else:
                    ctx.save_for_backward(x, weight)
        else:
            ctx.fused = False
            if save_for_backward:
                ctx.save_for_backward(x, weight)
            total = comm.all_gather(x, dim=seq_dim, group=group) if (in_mode == "gather" and n > 1) else x
            if (n > 1 and out_mode == "reduce" and not fp8 and not torch.is_grad_enabled() and total.is_cuda
                    and total.numel() // total.shape[-1] <= 8 and ops.tp_fused.get_backend() == "fused"
                    and ops.nvls.gemv_all_reduce_eligible(total.reshape(-1, total.shape[-1]), weight)):
                # decode-time Row-parallel linear: GEMV and the all-reduce of its fp32 partials in ONE kernel
                # (csrc/nvls_coll.cu gemv_allreduce_kernel; in-switch reduction when the group has an NVLS mapping)
                y = ops.nvls.gemv_all_reduce(total.reshape(-1, total.shape[-1]), weight, group).view(*total.shape[:-1], weight.shape[0])
                if bias is not None:
                    y = y + bias
                return y
            if fp8:
                y = gemm_fp8.fp8_forward(_flat2d(total), weight).view(*total.shape[:-1], weight.shape[0])
            else:
                y = ops.gemm.linear_nt(total, weight)      # wgmma kernel on CUDA bf16, torch.matmul otherwise
            if n > 1 and out_mode in ("scatter", "reduce"):
                od = y.dtype
                yr = y.to(reduce_dtype) if reduce_dtype is not None else y
                if out_mode == "scatter":
                    yr = comm.reduce_scatter(yr, dim=seq_dim, group=group)
                else:
                    comm.all_reduce(yr, group=group)
                y = yr.to(od)
        if bias is not None:
            y = y + bias
        return y

    @staticmethod
    def backward(ctx, gy):
        from .. import ops
        from ..ops import gemm_fp8

        group, seq_dim = ctx.group, ctx.seq_dim
        n = dist.get_world_size(group)
        in_mode, out_mode = ctx.in_mode, ctx.out_mode
        gbias = None
        gy = gy.contiguous()
        # GQA with replicated KV heads: the K/V output gradients arrive summed over the KV-shared group (needed by wgrad);
        # the input gradient is later summed over the whole TP group, so the dgrad GEMM sees those columns scaled by
        # 1/multiplier (reference qkv_linear.py:183-198).
        gy_d = gy
        if ctx.dgrad_col_scale is not None and ctx.x_requires_grad:
            start, scale = ctx.dgrad_col_scale
            gy_d = gy.clone()
            gy_d[..., start:] *= scale
        if ctx.fused:
            if ctx.has_gathered:
                x, weight, gathered = ctx.saved_tensors
            else:
                (x, weight), gathered = ctx.saved_tensors, None
            fused = ops.tp_fused.dispatch(x, weight, in_mode, out_mode, seq_dim, group)
            gx, gw, gbias = fused.backward(x, weight, gy, ctx.has_bias, ctx.x_requires_grad, weight.requires_grad,
                                           gathered, gy_dgrad=(gy_d if gy_d is not gy else None))
            return gx, gw, gbias, None, None, None, None, None, None, None, None
        x, weight = ctx.saved_tensors

        # ---- grad wrt the GEMM output (undo the output collective) -----------------
        if out_mode == "scatter" and n > 1:
            g_out = comm.all_gather(gy, dim=seq_dim, group=group)
        else:
            g_out = gy  # "reduce": identity backward; "none"
        if ctx.has_bias:
            # bias is added after the collective → its grad uses the *local* gy
            gbias = _flat2d(gy).sum(0)
        # ---- dgrad --------------------------------------------------------------------
        gx = None
        work = None
        if ctx.x_requires_grad:
            g_d = g_out if gy_d is gy else gy_d          # dgrad_col_scale is only used with out_mode "none" (g_out is gy)
            if ctx.fp8:
                gx = gemm_fp8.fp8_dgrad(_flat2d(g_d), weight)
            else:
                gx = ops.gemm.matmul(_flat2d(g_d), weight, False, False)
            gx = gx.view(*g_out.shape[:-1], weight.shape[1])
            if n > 1 and in_mode == "copy":
                work = comm.all_reduce(gx, group=group, async_op=True)  # overlaps wgrad
            elif n > 1 and in_mode == "gather":
                od = gx.dtype
                rd = ctx.reduce_dtype
                gx = comm.reduce_scatter(gx.to(rd) if rd is not None else gx, dim=seq_dim, group=group).to(od)
        # ---- wgrad ----------------------------------------------------------------------
        gw = None
        if weight.requires_grad:
            total = comm.all_gather(x, dim=seq_dim, group=group) if (in_mode == "gather" and n > 1) else x
            gw = wgrad(_flat2d(g_out), _flat2d(total), weight, fp8=ctx.fp8)
        if work is not None:
            work.wait()
        return gx, gw, gbias, None, None, None, None, None, None, None, None


def tp_linear(
    x: torch.Tensor,
    weight: torch.Tensor,
    bias: Optional[torch.Tensor],
    in_mode: str,
    out_mode: str,
    seq_dim: int = 0,
    group=None,
    reduce_dtype: Optional[torch.dtype] = None,
    save_for_backward: bool = True,
    autocast: bool = False,
    dgrad_col_scale=None,
    fp8: bool = False,
) -> torch.Tensor:
    """``dgrad_col_scale=(first_col, scale)``: output-gradient columns ``>= first_col`` are multiplied by ``scale`` for the
    input-gradient GEMM only (weight gradient sees them unscaled) — the GQA KV-replication correction.

    ``fp8``: forward, input-gradient and weight-gradient GEMMs in e4m3 with one absmax scale per row of each operand
    (``ops.gemm_fp8``: rows(x)·rows(W)ᵀ, rows(g)·cols_t(W)ᵀ, cols_t(g)·cols_t(x)ᵀ); the bias, the collectives and the tensors
    saved for backward stay bf16."""
    assert dgrad_col_scale is None or out_mode == "none"
    group = group if group is not None else ps.get_tensor_model_parallel_group()
    if autocast or torch.is_autocast_enabled():
        dt = torch.get_autocast_dtype("cuda" if x.is_cuda else "cpu") if torch.is_autocast_enabled() else x.dtype
        x = x.to(dt)
        weight = weight.to(dt)
        bias = bias.to(dt) if bias is not None else None
        with torch.autocast(device_type="cuda" if x.is_cuda else "cpu", enabled=False):
            return _TPLinear.apply(x, weight, bias, in_mode, out_mode, seq_dim, group, reduce_dtype, save_for_backward,
                                   dgrad_col_scale, fp8)
    return _TPLinear.apply(x, weight, bias, in_mode, out_mode, seq_dim, group, reduce_dtype, save_for_backward, dgrad_col_scale,
                           fp8)


class LinearWithAsyncCommunication:
    """Name-compatible façade (reference layers.py:434): ``apply`` maps the reference's flag
    combination onto :class:`_TPLinear` modes."""

    @staticmethod
    def apply(
        input,  # noqa: A002
        weight,
        bias,
        async_grad_allreduce: bool,
        sequence_parallel_enabled: bool,
        sequence_dimension: Optional[int] = 0,
        save_for_backward: bool = True,
        process_group=None,
        reduce_dtype: torch.dtype = torch.float32,
    ):
        if sequence_parallel_enabled:
            assert not async_grad_allreduce
            in_mode = "gather"
        else:
            in_mode = "copy" if async_grad_allreduce else "none"
        return tp_linear(
            input, weight, bias, in_mode, "none", sequence_dimension or 0, process_group, reduce_dtype, save_for_backward
        )


def linear_with_async_allreduce(
    input: torch.Tensor,  # noqa: A002
    weight: torch.Tensor,
    bias: Optional[torch.Tensor],
    async_grad_allreduce: bool,
    sequence_parallel_enabled: bool,
    sequence_dimension: Optional[int] = 0,
    autograd_func_class: Any = None,
    save_for_backward: bool = True,
    process_group=None,
    reduce_dtype: torch.dtype = torch.float32,
    autocast: bool = False,
) -> torch.Tensor:
    """Seventh positional argument as in the reference (layers.py:507-532): an autograd class whose ``apply`` takes
    ``(input, weight, bias, async_grad_allreduce, sequence_parallel_enabled, sequence_dimension, save_for_backward,
    process_group, reduce_dtype)`` — a custom class is called as is, the default / ``None`` runs the fused TP linear.  A bool in
    that position is this package's earlier ``autocast`` flag."""
    if isinstance(autograd_func_class, bool):
        autocast, autograd_func_class = autograd_func_class, None
    if autograd_func_class is not None and autograd_func_class is not LinearWithAsyncCommunication:
        return autograd_func_class.apply(input, weight, bias, async_grad_allreduce, sequence_parallel_enabled, sequence_dimension,
                                         save_for_backward, process_group, reduce_dtype)
    if sequence_parallel_enabled:
        in_mode = "gather"
    else:
        in_mode = "copy" if async_grad_allreduce else "none"
    return tp_linear(
        input, weight, bias, in_mode, "none", sequence_dimension or 0, process_group, reduce_dtype,
        save_for_backward, autocast,
    )


# --------------------------------------------------------------------------------------
# Column / Row parallel linear
# --------------------------------------------------------------------------------------
class ColumnParallelLinear(BaseParallelLinear):
    """``Y = X A^T + b`` with ``A`` split along its output dim: ``A = [A_1; …; A_p]``.

    Arguments mirror reference layers.py:587-607.  ``stride`` >1 interleaves fused matrices
    (gate/up, q/k/v) so each rank's shard holds matching slices of each."""

    def __init__(
        self,
        input_size: int,
        output_size: int,
        bias: bool = True,
        gather_output: bool = True,
        dtype: torch.dtype = torch.float32,
        device: Optional[torch.device] = None,
        stride: int = 1,
        init_method: Optional[Callable[..., Any]] = None,
        sequence_parallel_enabled: bool = False,
        sequence_dimension: Optional[int] = None,
        keep_master_weight: bool = False,
        skip_bias_add: bool = False,
        pad: bool = False,
        pad_alignment_size_per_rank: int = 1,
        keep_padded_output: bool = False,
        tensor_model_parallel_group=None,
        reduce_dtype: torch.dtype = torch.float32,
        rank_ordering: Optional[Sequence[int]] = None,
    ):
        super().__init__(device=device)
        self.input_size, self.output_size = input_size, output_size
        self.gather_output, self.stride = gather_output, stride
        self.tensor_parallel_group, tp, self._tp_rank = _group_info(tensor_model_parallel_group)
        self.tensor_model_parallel_size = tp
        self.pad, self.pad_size, self.keep_padded_output = pad, 0, keep_padded_output
        self.pad_alignment_size_per_rank = pad_alignment_size_per_rank
        if pad:
            self.pad_size = get_padding_length(output_size, tp * pad_alignment_size_per_rank)
            self.output_size = output_size + self.pad_size
        self.output_size_per_partition = divide(self.output_size, tp)
        self.dtype = dtype
        self.device = device if device is not None else torch.device("cpu")
        self.keep_master_weight, self.skip_bias_add = keep_master_weight, skip_bias_add
        self.sequence_parallel_enabled = sequence_parallel_enabled
        self.sequence_dimension = 0 if sequence_dimension is None else sequence_dimension
        self.reduce_dtype, self.rank_ordering = reduce_dtype, rank_ordering
        self.arg_init_method = init_method
        self.async_tensor_model_parallel_allreduce = not sequence_parallel_enabled and tp > 1
        self.master_weight: Optional[torch.Tensor] = None
        self.add_bias = bias
        self.set_weight_and_bias_config()
        self.weight = Parameter(torch.empty(*self.weight_shape, dtype=dtype, device=self.device))
        if bias:
            # bias is sharded like the weight unless the output is gathered (then it is
            # replicated and added after the gather) — reference :700-722
            self.bias = Parameter(torch.zeros(*self.bias_shape, dtype=dtype, device=self.device))
            if not gather_output:
                set_tensor_model_parallel_attributes(self.bias, True, 0, stride, num_partitions=tp)
            else:
                set_tensor_model_parallel_attributes(self.bias, False, 0, 1, num_partitions=1)
        else:
            self.register_parameter("bias", None)
        self.initialize_weight_and_bias()

    def set_weight_and_bias_config(self) -> None:
        """Shapes / partition dims of this rank's parameters — the override point for layers with another weight layout
        (reference layers.py:660-671)."""
        self.weight_shape = (self.output_size_per_partition, self.input_size)
        self.weight_partition_dim = 0
        self.bias_shape = ((self.output_size,) if self.gather_output else (self.output_size_per_partition,))
        self.bias_partition_dim = 0

    def init_weight_cpu(self) -> None:
        """Draw the FULL weight (identical on every rank) and keep this rank's slice — TP-degree independent init."""
        master = _initialize_parameter_from_master(
            self.weight, self.weight_partition_dim, self.tensor_model_parallel_size, self._init_weight,
            return_master_param=self.keep_master_weight, param_dtype=self.dtype, stride=self.stride, rank=self._tp_rank,
        )
        if self.keep_master_weight:
            self.master_weight = master

    def initialize_weight_and_bias(self) -> None:
        tp = self.tensor_model_parallel_size
        self.init_weight_cpu()
        if self.rank_ordering is not None:
            self.weight.rank_ordering = list(self.rank_ordering)
        if self.bias is not None and self.arg_init_method is None and self.weight.device.type != "meta":
            bound = 1 / math.sqrt(self.input_size) if self.input_size > 0 else 0
            with torch.no_grad():
                full = torch.empty(self.output_size, dtype=torch.float32)
                init.uniform_(full, -bound, bound)
                if self.gather_output:
                    self.bias.copy_(full.to(self.dtype))
                else:
                    self.bias.copy_(create_local_weight(
                        full.to(self.dtype), 0, self.output_size_per_partition, self.stride,
                        rank=self._tp_rank, world_size=tp))

    def forward(self, input: torch.Tensor, slice_indices: Optional[torch.Tensor] = None, *_: Any):  # noqa: A002
        self._check_pad_false_for_training()
        tp = self.tensor_model_parallel_size
        weight = self.weight if slice_indices is None else self.weight.index_select(0, slice_indices)
        if self.sequence_parallel_enabled:
            in_mode = "gather"
        else:
            in_mode = "copy" if tp > 1 else "none"
        out = tp_linear(
            input, weight, None, in_mode, "none", self.sequence_dimension, self.tensor_parallel_group, self.reduce_dtype,
            fp8=self.fp8_training,
        )
        if self.gather_output:
            out = mappings.gather_from_tensor_model_parallel_region(out, self.tensor_parallel_group)
            if self.pad and self.pad_size > 0 and not self.keep_padded_output:
                out = out.narrow(-1, 0, self.output_size - self.pad_size)
        if self.skip_bias_add:
            return out, self.bias
        if self.bias is not None:
            b = self.bias
            if self.gather_output and self.pad and self.pad_size > 0 and not self.keep_padded_output:
                b = b.narrow(0, 0, self.output_size - self.pad_size)
            out = out + b
        return out

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        """Zero-pad a full checkpoint weight/bias along the output dim (reference :770-783)."""
        if not self.pad or self.pad_size == 0:
            return
        w = model_state_dict[prefix]
        if w.shape[0] + self.pad_size != self.output_size:
            raise RuntimeError(f"State dict {prefix} has unexpected shape {tuple(w.shape)}")
        model_state_dict[prefix] = F.pad(w, (0, 0, 0, self.pad_size))
        bkey = prefix.replace("weight", "bias")
        if self.bias is not None and bkey in model_state_dict:
            model_state_dict[bkey] = F.pad(model_state_dict[bkey], (0, self.pad_size))


class RowParallelLinear(BaseParallelLinear):
    """``Y = X A^T + b`` with ``A`` split along its input dim; partial products are summed
    across TP — all-reduce, or reduce-scatter along the sequence dim under SP (reference
    layers.py:815-1063)."""

    def __init__(
        self,
        input_size: int,
        output_size: int,
        bias: bool = True,
        input_is_parallel: bool = False,
        dtype: torch.dtype = torch.float32,
        device: Optional[torch.device] = None,
        stride: int = 1,
        init_method: Optional[Callable[..., Any]] = None,
        sequence_parallel_enabled: bool = False,
        sequence_dimension: Optional[int] = None,
        keep_master_weight: bool = False,
        skip_bias_add: bool = False,
        pad: bool = False,
        reduce_output: bool = True,
        reduce_dtype: torch.dtype = torch.float32,
        tensor_model_parallel_group=None,
        tile_cc: bool = False,
        rank_ordering: Optional[Sequence[int]] = None,
    ):
        super().__init__(device=device)
        self.input_size, self.output_size = input_size, output_size
        self.input_is_parallel, self.stride = input_is_parallel, stride
        self.tensor_parallel_group, tp, self._tp_rank = _group_info(tensor_model_parallel_group)
        self.tensor_model_parallel_size = tp
        self.pad, self.pad_size = pad, 0
        if pad:
            self.pad_size = get_padding_length(input_size, tp)
            self.input_size = input_size + self.pad_size
        self.input_size_per_partition = divide(self.input_size, tp)
        self.dtype = dtype
        self.device = device if device is not None else torch.device("cpu")
        self.keep_master_weight, self.skip_bias_add = keep_master_weight, skip_bias_add
        self.sequence_parallel_enabled = sequence_parallel_enabled
        self.sequence_dimension = 0 if sequence_dimension is None else sequence_dimension
        self.reduce_output, self.reduce_dtype = reduce_output, reduce_dtype
        self.rank_ordering = rank_ordering
        self.arg_init_method = init_method
        if sequence_parallel_enabled and not input_is_parallel:
            raise RuntimeError("To enable `sequence_parallel_enabled`, `input_is_parallel` must be `True`")
        self.master_weight: Optional[torch.Tensor] = None
        self.add_bias = bias
        self.set_weight_and_bias_config()
        self.weight = Parameter(torch.empty(*self.weight_shape, dtype=dtype, device=self.device))
        if bias:
            self.bias = Parameter(torch.zeros(*self.bias_shape, dtype=dtype, device=self.device))
            _tag_sequence_parallel(self.bias, sequence_parallel_enabled)
        else:
            self.register_parameter("bias", None)
        self.initialize_weight_and_bias()

    def _init_weight(self, w: torch.Tensor) -> None:
        if self.arg_init_method is None:
            init.kaiming_uniform_(w, a=math.sqrt(5))
        else:
            self.arg_init_method(w)

    def set_weight_and_bias_config(self) -> None:
        """Override point (reference layers.py:909-918)."""
        self.weight_shape = (self.output_size, self.input_size_per_partition)
        self.weight_partition_dim = 1
        self.bias_shape = (self.output_size,)

    def init_weight_cpu(self) -> None:
        master = _initialize_parameter_from_master(
            self.weight, self.weight_partition_dim, self.tensor_model_parallel_size, self._init_weight,
            return_master_param=self.keep_master_weight, param_dtype=self.dtype, stride=self.stride,
            rank=self._tp_rank,
        )
        if self.keep_master_weight:
            self.master_weight = master

    def initialize_weight_and_bias(self) -> None:
        self.init_weight_cpu()
        if self.rank_ordering is not None:
            self.weight.rank_ordering = list(self.rank_ordering)
        if self.bias is not None and self.arg_init_method is None and self.weight.device.type != "meta":
            bound = 1 / math.sqrt(self.input_size) if self.input_size > 0 else 0
            with torch.no_grad():
                init.uniform_(self.bias, -bound, bound)

    def forward(self, input_: torch.Tensor, slice_indices: Optional[torch.Tensor] = None, *_: Any):
        """``slice_indices`` selects input-feature columns of the local weight (decode-time slicing of replicated weights,
        reference layers.py:971-1000)."""
        self._check_pad_false_for_training()
        tp = self.tensor_model_parallel_size
        if self.input_is_parallel:
            x = input_
        else:
            if self.pad and self.pad_size > 0:
                input_ = F.pad(input_, (0, self.pad_size))
            x = mappings.scatter_to_tensor_model_parallel_region(input_, self.tensor_parallel_group)
        if not self.reduce_output or tp == 1:
            out_mode = "none"
        else:
            out_mode = "scatter" if self.sequence_parallel_enabled else "reduce"
        weight = self.weight if slice_indices is None else self.weight.index_select(1, slice_indices)
        out = tp_linear(
            x, weight, None, "none", out_mode, self.sequence_dimension, self.tensor_parallel_group,
            self.reduce_dtype, fp8=self.fp8_training,
        )
        if self.skip_bias_add:
            return out, self.bias
        if self.bias is not None:
            out = out + self.bias
        return out

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        if not self.pad or self.pad_size == 0:
            return
        w = model_state_dict[prefix]
        if w.shape[1] + self.pad_size != self.input_size:
            raise RuntimeError(f"State dict {prefix} has unexpected shape {tuple(w.shape)}")
        model_state_dict[prefix] = F.pad(w, (0, self.pad_size))


# --------------------------------------------------------------------------------------
# Conv2d
# --------------------------------------------------------------------------------------
def _pair(v) -> Tuple[int, int]:
    return (v, v) if isinstance(v, int) else tuple(v)


class _ConvWithAsyncAllReduce(torch.autograd.Function):
    """conv2d whose input-grad all-reduce overlaps the weight-grad computation
    (reference layers.py:1066-1150)."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation, groups, allreduce_dgrad, group):
        ctx.save_for_backward(x, weight)
        ctx.conf = (stride, padding, dilation, groups)
        ctx.has_bias, ctx.allreduce_dgrad, ctx.group = bias is not None, allreduce_dgrad, group
        return F.conv2d(x, weight, bias, stride, padding, dilation, groups)

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        stride, padding, dilation, groups = ctx.conf
        gx = gw = gb = None
        work = None
        if ctx.needs_input_grad[0]:
            gx = torch.nn.grad.conv2d_input(x.shape, weight, gy, stride, padding, dilation, groups)
            if ctx.allreduce_dgrad and dist.get_world_size(ctx.group) > 1:
                work = comm.all_reduce(gx, group=ctx.group, async_op=True)
        if ctx.needs_input_grad[1]:
            gw = torch.nn.grad.conv2d_weight(x, weight.shape, gy, stride, padding, dilation, groups)
        if ctx.has_bias:
            gb = gy.sum((0, 2, 3))
        if work is not None:
            work.wait()
        return gx, gw, gb, None, None, None, None, None, None


Conv2dWithInputGradAllReduce = _ConvWithAsyncAllReduce        # reference name (layers.py:1066)


def conv2d_with_weight_grad_allreduce(input: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor],  # noqa: A002
                                      stride: Tuple[int, int], padding: Tuple[int, int], allreduce_weight_grad: bool,
                                      dilation: Tuple[int, int] = (1, 1), groups: int = 1, group=None) -> torch.Tensor:
    """Functional form (reference layers.py:1132-1150).  The flag's name is historical: the collective it enables is the
    all-reduce of the *input* gradient over the TP group (output-channel-parallel convolutions), issued before the
    weight-gradient kernel so the two overlap."""
    from .utils import cast_if_autocast_enabled

    input, weight, bias = cast_if_autocast_enabled(input, weight, bias)  # noqa: A001
    group = group if group is not None else ps.get_tensor_model_parallel_group()
    with torch.autocast(device_type="cuda" if input.is_cuda else "cpu", enabled=False):
        return _ConvWithAsyncAllReduce.apply(input, weight, bias, _pair(stride), _pair(padding), _pair(dilation), groups,
                                             allreduce_weight_grad, group)


class BaseParallelConv(BaseParallelLayer):
    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                 padding_mode, partition_dim, dtype, device, init_method, keep_master_weight, group, partition_pad=False):
        super().__init__(device=device)
        if groups != 1:
            raise NotImplementedError("grouped convolution is not supported by the parallel conv layers")
        if padding_mode != "zeros":
            raise NotImplementedError("only zero padding is supported")
        self.kernel_size, self.stride = _pair(kernel_size), _pair(stride)
        self.padding, self.dilation, self.groups = _pair(padding), _pair(dilation), groups
        self.tensor_parallel_group, self.tensor_model_parallel_size, self._tp_rank = _group_info(group)
        # ``partition_pad``: zero-pad the partitioned channel count up to a multiple of tp (reference layers.py:1195-1211);
        # padded output channels are cut after the gather, padded input channels see zero input
        self.partition_pad, self.partition_pad_size = partition_pad, 0
        if partition_pad:
            n = out_channels if partition_dim == 0 else in_channels
            self.partition_pad_size = get_padding_length(n, self.tensor_model_parallel_size)
            if partition_dim == 0:
                out_channels += self.partition_pad_size
            else:
                in_channels += self.partition_pad_size
        self.in_channels, self.out_channels = in_channels, out_channels
        self.partition_dim, self.dtype = partition_dim, dtype
        self.arg_init_method, self.keep_master_weight = init_method, keep_master_weight
        self.device = device if device is not None else torch.device("cpu")
        tp = self.tensor_model_parallel_size
        oc = divide(out_channels, tp) if partition_dim == 0 else out_channels
        ic = divide(in_channels, tp) if partition_dim == 1 else in_channels
        self.weight = Parameter(torch.empty(oc, ic, *self.kernel_size, dtype=dtype, device=self.device))
        self.master_weight = _initialize_parameter_from_master(
            self.weight, partition_dim, tp, self._init_weight, keep_master_weight, dtype, 1, self._tp_rank)
        if bias:
            self.bias = Parameter(torch.zeros(oc if partition_dim == 0 else out_channels, dtype=dtype, device=self.device))
            fan_in = in_channels * self.kernel_size[0] * self.kernel_size[1]
            bound = 1 / math.sqrt(fan_in)
            with torch.no_grad():
                full = torch.empty(out_channels, dtype=torch.float32)
                init.uniform_(full, -bound, bound)
                if partition_dim == 0:
                    self.bias.copy_(create_local_weight(full.to(dtype), 0, oc, 1, rank=self._tp_rank, world_size=tp))
                    set_tensor_model_parallel_attributes(self.bias, True, 0, 1, num_partitions=tp)
                else:
                    self.bias.copy_(full.to(dtype))
        else:
            self.register_parameter("bias", None)

    def _init_weight(self, w):
        if self.arg_init_method is None:
            init.kaiming_uniform_(w, a=math.sqrt(5))
        else:
            self.arg_init_method(w)


CONV_KERNEL_OUTPUT_CHANNEL_DIMENSION = 0             # Conv2d weight is [out, in / groups, kh, kw]
CONV_KERNEL_INPUT_CHANNEL_DIMENSION = 1


class OutputChannelParallelConv2d(BaseParallelConv):
    """Conv2d sharded along output channels; optional all-gather on the channel dim
    (reference layers.py:1309-1430)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", gather_output=True, dtype=torch.float32, device=None,
                 init_method=None, keep_master_weight=False, partition_pad=False, tensor_model_parallel_group=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         padding_mode, CONV_KERNEL_OUTPUT_CHANNEL_DIMENSION, dtype, device, init_method, keep_master_weight,
                         tensor_model_parallel_group, partition_pad)
        self.gather_output = gather_output

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        """Zero-pad a full checkpoint's weight / bias along the output-channel dim (reference :1419-1429)."""
        if not self.partition_pad or self.partition_pad_size == 0:
            return
        w = model_state_dict[prefix]
        if self.out_channels != w.shape[0] + self.partition_pad_size:
            raise RuntimeError(f"State dict {prefix} is of an unexpected size {w.shape[0]} expected "
                               f"{self.out_channels - self.partition_pad_size}")
        model_state_dict[prefix] = F.pad(w, (0, 0) * (w.dim() - 1) + (0, self.partition_pad_size))

    def forward(self, in_tensor: torch.Tensor) -> torch.Tensor:
        x = in_tensor      # reference parameter names in the signature
        tp = self.tensor_model_parallel_size
        out = _ConvWithAsyncAllReduce.apply(x, self.weight, self.bias, self.stride, self.padding, self.dilation,
                                            self.groups, tp > 1, self.tensor_parallel_group)
        if self.gather_output:
            out = mappings.gather_from_tensor_model_parallel_region_with_dim(out, 1, self.tensor_parallel_group)
            if self.partition_pad and self.partition_pad_size > 0:
                out = out.narrow(1, 0, self.out_channels - self.partition_pad_size)
        return out


class InputChannelParallelConv2d(BaseParallelConv):
    """Conv2d sharded along input channels; partial outputs all-reduced
    (reference layers.py:1432-1540)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias=True, padding_mode="zeros", input_is_parallel=False, dtype=torch.float32, device=None,
                 init_method=None, keep_master_weight=False, partition_pad=False, tensor_model_parallel_group=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias,
                         padding_mode, CONV_KERNEL_INPUT_CHANNEL_DIMENSION, dtype, device, init_method, keep_master_weight,
                         tensor_model_parallel_group, partition_pad)
        self.input_is_parallel = input_is_parallel

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        if not self.partition_pad or self.partition_pad_size == 0 or not prefix.endswith("weight"):
            return
        w = model_state_dict[prefix]
        if self.in_channels != w.shape[1] + self.partition_pad_size:
            raise RuntimeError(f"State dict {prefix} is of an unexpected size {w.shape[1]}")
        model_state_dict[prefix] = F.pad(w, (0, 0, 0, 0, 0, self.partition_pad_size))

    def forward(self, in_tensor: torch.Tensor) -> torch.Tensor:
        x = in_tensor      # reference parameter names in the signature
        if not self.input_is_parallel:
            if self.partition_pad and self.partition_pad_size > 0:
                x = F.pad(x, (0, 0, 0, 0, 0, self.partition_pad_size))
            x = mappings.scatter_input_channels_to_tensor_model_parallel_region(x, self.tensor_parallel_group)
        out = _ConvWithAsyncAllReduce.apply(x, self.weight, None, self.stride, self.padding, self.dilation,
                                            self.groups, False, self.tensor_parallel_group)
        out = mappings.reduce_from_tensor_model_parallel_region(out, self.tensor_parallel_group)
        if self.bias is not None:
            out = out + self.bias.view(1, -1, 1, 1)
        return out
