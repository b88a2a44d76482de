"""Blockwise (dropless) expert MLP.

Role of the reference's NKI blockwise kernels K6/K7/K9 (``modules/moe/blockwise.py:180-468,1037-1127``,
``expert_mlps_v2.py:691-917,1079-1206``).  Tokens are grouped by expert, every expert's group is padded to a multiple
of ``block_size`` and each block is multiplied by exactly one expert's weights:

    num_blocks            = ceil((T·k − (E−1)) / B) + (E−1)          (static upper bound)
    block_to_expert[b]    : expert owning block b
    token_position_to_id  : flat [num_blocks·B] token id feeding each block slot (−1 = padding)

On CUDA the two projections are grouped wgmma GEMMs (``ops.gemm.grouped_matmul`` → MODE 3/4 of
``csrc/gemm_sm90.cu``): the block's expert only shifts the TMA coordinate of the weight tile, the backward runs the
grouped dgrad and a per-expert segmented wgrad, and nothing syncs with the host.  On CPU it is a gathered einsum.
Quantised expert layers run their own ``grouped_linear``: W8A8 block-wise e4m3 experts quantise each projection's input
per token and run the grouped block-scaled FP8 GEMM (``ops.gemm_fp8.grouped_blockscaled_linear``); weight-only experts
are de-quantised to the activation dtype once per call and run the bf16 grouped GEMM (inference only).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Optional, Tuple

import torch

from .moe_configs import (  # noqa: F401  (re-exported here as in the reference, blockwise.py:83-87)
    ActFnType,
    ActivationFunction,
    BlockShardStrategy,
    ExpertAffinityScaleMode,
    SkipMode,
)


def get_num_blocks(total_tokens: int, top_k: int, num_experts: int, block_size: int) -> int:
    return max(1, math.ceil(max(total_tokens * top_k - (num_experts - 1), 0) / block_size) + (num_experts - 1))


def build_block_metadata(expert_index: torch.Tensor, num_experts: int, block_size: int
                         ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """From ``expert_index [T, k]`` build ``(block_to_expert [nb], token_position_to_id [nb·B], tokens_per_expert [E])``.
    Entirely on device (sort + cumsum), no host sync."""
    T, k = expert_index.shape
    nb = get_num_blocks(T, k, num_experts, block_size)
    if expert_index.is_cuda and num_experts <= 256 and expert_index.dtype in (torch.int32, torch.int64):
        from ... import ops

        e = ops._ext.ext()
        if e is not None and hasattr(e, "moe_block_metadata"):
            # one launch, no sort (csrc/select.cu moe_block_metadata_kernel — role of the reference's index-build NKI kernels)
            ops._ext.count_launch()
            return e.moe_block_metadata(expert_index.contiguous(), int(num_experts), int(block_size), int(nb))
    flat_e = expert_index.reshape(-1)
    token_ids = torch.arange(T, device=expert_index.device).repeat_interleave(k)
    order = torch.argsort(flat_e, stable=True)
    se, st = flat_e[order], token_ids[order]
    counts = torch.bincount(flat_e, minlength=num_experts)
    blocks_per_e = (counts + block_size - 1) // block_size
    block_start = torch.cumsum(blocks_per_e, 0) - blocks_per_e                      # first block of each expert
    seg_start = torch.cumsum(counts, 0) - counts
    pos_in_e = torch.arange(se.numel(), device=se.device) - seg_start[se]
    slot = block_start[se] * block_size + pos_in_e
    tp2id = torch.full((nb * block_size,), -1, dtype=torch.long, device=se.device)
    tp2id[slot] = st
    b_idx = torch.arange(nb, device=se.device)
    ends = torch.cumsum(blocks_per_e, 0)
    block_to_expert = torch.searchsorted(ends, b_idx, right=True).clamp(max=num_experts - 1)
    return block_to_expert, tp2id, counts


def _weight_of(proj) -> torch.Tensor:
    return proj if isinstance(proj, torch.Tensor) else proj.weight


def _grouped(x: torch.Tensor, proj, b2e: torch.Tensor, seg_first: torch.Tensor, block_size: int) -> torch.Tensor:
    if isinstance(proj, torch.Tensor):
        from ... import ops

        return ops.gemm.grouped_matmul(x, proj, b2e, seg_first, block_size)
    return proj.grouped_linear(x, b2e, seg_first, block_size)


def _projection(layer):
    """What the grouped path multiplies by: a float expert layer's weight, or a quantised layer itself."""
    return layer if hasattr(layer, "grouped_linear") else layer.weight


def blockwise_mlp_from_metadata(hidden: torch.Tensor, expert_affinities_masked: torch.Tensor, gate_up_proj_weight: torch.Tensor,
                                down_proj_weight: torch.Tensor, token_position_to_id: torch.Tensor, block_to_expert: torch.Tensor,
                                block_size: int, activation, gate_up_proj_bias: Optional[torch.Tensor] = None,
                                down_proj_bias: Optional[torch.Tensor] = None, pre_scale: bool = False) -> torch.Tensor:
    """The dropless computation for a GIVEN block layout: ``out[t] += aff[t, e(b)] · MLP_{e(b)}(hidden[t])`` for every slot of
    every block ``b`` holding token ``t`` (``-1`` slots are padding).  ``expert_affinities_masked`` is ``[T, E]``.
    ``pre_scale`` multiplies the expert input by the affinity instead of the output (early affinity modulation).  A projection
    is a ``[E, K, N]`` weight or a quantised expert-fused layer, which runs its own ``grouped_linear``."""
    T, H = hidden.shape
    E = _weight_of(gate_up_proj_weight).shape[0]
    nb = block_to_expert.numel()
    tp2id = token_position_to_id[: nb * block_size].long()
    b2e = block_to_expert.long()
    blocks_per_e = torch.bincount(b2e, minlength=E)
    seg_first = torch.cat([blocks_per_e.new_zeros(1), torch.cumsum(blocks_per_e, 0)])          # [E+1] block prefix sum
    valid = tp2id >= 0
    gather_ids = tp2id.clamp(min=0)
    slot_e = b2e.repeat_interleave(block_size)
    aff = expert_affinities_masked[gather_ids, slot_e] * valid.to(expert_affinities_masked.dtype)
    x = hidden[gather_ids] * valid.unsqueeze(-1).to(hidden.dtype)                   # [nb·B, H]
    if pre_scale:
        x = x * aff.unsqueeze(-1).to(x.dtype)
    h = _grouped(x, gate_up_proj_weight, b2e, seg_first, block_size)
    if gate_up_proj_bias is not None:
        h = h + gate_up_proj_bias[slot_e].to(h.dtype)
    h = activation(h)
    y = _grouped(h.contiguous(), down_proj_weight, b2e, seg_first, block_size)
    if down_proj_bias is not None:
        y = y + down_proj_bias[slot_e].to(y.dtype)
    scale = (aff > 0).to(y.dtype) if pre_scale else aff.to(y.dtype)
    out = torch.zeros(T, H, dtype=y.dtype, device=y.device)
    out.index_add_(0, gather_ids, y * (scale * valid.to(y.dtype)).unsqueeze(-1))
    return out


def blockwise_expert_mlp(hidden: torch.Tensor, expert_affinities: torch.Tensor, expert_index: torch.Tensor,
                         experts, block_size: int, normalize: bool = False) -> torch.Tensor:
    """Dropless MoE MLP: ``out[t] = Σ_j aff[t, e_j] · MLP_{e_j}(hidden[t])``."""
    E = expert_affinities.shape[-1]
    b2e, tp2id, _ = build_block_metadata(expert_index, E, block_size)
    if normalize:
        denom = expert_affinities.gather(1, expert_index).sum(-1, keepdim=True).clamp(min=1e-9)
        expert_affinities = expert_affinities / denom
    proj = experts.gate_up_proj if experts.glu_mlp else experts.up_proj
    return blockwise_mlp_from_metadata(hidden, expert_affinities, _projection(proj), _projection(experts.down_proj), tp2id, b2e,
                                       block_size, experts.activation, proj.bias,
                                       None if experts.down_proj.bias is None else experts.down_proj.bias / experts.down_proj.tp)


# ---------------------------------------------------------------------------------------------------------------------
# Reference-named surface (modules/moe/blockwise.py:136-1127).  The reference selects among a family of NKI kernels
# (block-parallel, shard-on-hidden / -intermediate / -block, MX) by hardware generation; here there is ONE grouped
# wgmma GEMM (MODE 3 forward/dgrad, MODE 4 segmented wgrad) and a PyTorch path, so the selection helpers reduce to
# "is the CUDA extension usable for these shapes".
# ---------------------------------------------------------------------------------------------------------------------
DEFAULT_PADDING_VALUE = -1


_TORCH_TO_KERNEL_DTYPE = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32", torch.float8_e4m3fn: "e4m3",
                          torch.float8_e5m2: "e5m2", torch.uint8: "u8", torch.int8: "s8", torch.int32: "s32", torch.int64: "s64"}


def torch_to_nki_dtype(dtype: torch.dtype) -> str:
    """torch dtype → the element-type name the kernels' tensor maps / epilogues are specialised on (reference
    ``blockwise.py:33-40`` maps to ``nki.language`` dtypes)."""
    name = _TORCH_TO_KERNEL_DTYPE.get(dtype)
    if name is None:
        raise ValueError(f"Unsupported torch dtype for kernel conversion: {dtype}")
    return name


def _resolve(imports) -> dict:
    import warnings

    from .nki_import import import_kernel

    out = {}
    for key, cfg in imports.items():
        obj, err = import_kernel(cfg)
        if err:
            warnings.warn(f"Warning: {err}")
        out[key] = obj
    return out


def initialize_nki_components() -> dict:
    """Inference-side building blocks by the reference's component names (``blockwise.py:43-87``): the grouped wgmma GEMM that
    every blockwise variant runs on, the device-side block-metadata build, the fused decode block, and the enums."""
    from .nki_import import KernelImport as K

    return _resolve({
        "bwmm_shard_on_block": K("blockwise_mlp_from_metadata", module_name="modules.moe.blockwise"),
        "bwmm_shard_on_block_mx": K("BlockwiseMatmulMXNKIFunc", module_name="modules.moe.blockwise"),
        "blockwise_mm_baseline_shard_intermediate": K("blockwise_mlp_from_metadata", module_name="modules.moe.blockwise"),
        "blockwise_mm_baseline_shard_intermediate_hybrid": K("blockwise_mlp_from_metadata", module_name="modules.moe.blockwise"),
        "blockwise_mm_shard_intermediate_dropping": K("blockwise_mlp_from_metadata", module_name="modules.moe.blockwise"),
        "moe_cte": K("blockwise_expert_mlp", module_name="modules.moe.blockwise"),
        "grouped_gemm": K("grouped_gemm", is_kernel=True),
        "moe_block_metadata": K("moe_block_metadata", is_kernel=True),
        "moe_block_tkg": K("moe_block_tkg", is_kernel=True),
        "block_shard_strategy": K("BlockShardStrategy", module_name="modules.moe.moe_configs"),
        "skip_mode": K("SkipMode", module_name="modules.moe.moe_configs"),
        "affinity_scale_mode": K("ExpertAffinityScaleMode", module_name="modules.moe.moe_configs"),
        "act_fn_type": K("ActFnType", module_name="modules.moe.moe_configs"),
    })


def initialize_training_kernels() -> dict:
    """Training-side kernels by the reference's names (``blockwise.py:90-104``): forward = grouped GEMMs over the block list,
    backward = the grouped dgrad (same kernel, transposed weights) + ``grouped_wgrad``."""
    from .nki_import import KernelImport as K

    return _resolve({
        "blockwise_mm_training": K("TorchBlockwiseTraining", module_name="modules.moe.blockwise"),
        "blockwise_mm_baseline_shard_hidden": K("TorchBlockwiseTraining", module_name="modules.moe.blockwise"),
        "blockwise_mm_bwd": K("grouped_wgrad", is_kernel=True),
        "blockwise_mm_bwd_baseline_shard_hidden": K("grouped_wgrad", is_kernel=True),
    })


class KernelAvailabilityError(RuntimeError):
    """Raised when the grouped-GEMM kernel cannot serve a configuration (reference :88)."""


@dataclass
class KernelConfig:
    logical_nc_config: int = 1
    use_block_parallel: bool = False
    use_shard_on_intermediate: bool = False
    use_shard_on_block_dynamic_while: bool = False


@dataclass
class BlockwiseMatmulArgs:
    """Everything one blockwise call needs (reference :136-178)."""

    hidden_states: torch.Tensor
    expert_affinities_masked: torch.Tensor
    gate_up_proj_weight: torch.Tensor
    down_proj_weight: torch.Tensor
    token_position_to_id: torch.Tensor
    block_to_expert: torch.Tensor
    block_size: int = 512
    gate_up_proj_scale: Optional[torch.Tensor] = None
    down_proj_scale: Optional[torch.Tensor] = None
    output: Optional[torch.Tensor] = None
    dtype: torch.dtype = torch.bfloat16
    expert_affinities_scaling_mode: Any = ExpertAffinityScaleMode.POST_SCALE      # enum, its int, or "post_scale" / "pre_scale"
    skip_dma: Any = SkipMode(False, False)
    block_sharding_strategy: Any = BlockShardStrategy.HI_LO
    gate_clamp_upper_limit: Optional[float] = None
    gate_clamp_lower_limit: Optional[float] = None
    up_clamp_upper_limit: Optional[float] = None
    up_clamp_lower_limit: Optional[float] = None
    gate_up_proj_bias: Optional[torch.Tensor] = None
    down_proj_bias: Optional[torch.Tensor] = None
    kernel_act_fn: Any = None
    is_tensor_update_accumulating: bool = False


def check_kernel_availability(device: Optional[torch.device] = None) -> bool:
    from ...ops import _ext

    if device is not None and device.type != "cuda":
        return False
    e = _ext.ext() if torch.cuda.is_available() else None
    return e is not None and hasattr(e, "grouped_gemm")


def check_blockwise_mm_kernel_compatibility(hidden_size: int, block_size: int, intermediate_size_tp: int) -> None:
    """The grouped GEMM tiles need 128-row blocks and 16-element (32-byte) aligned K / N (reference :683-716)."""
    if block_size % 128 != 0:
        raise KernelAvailabilityError(f"block_size {block_size} must be a multiple of 128 for the grouped wgmma GEMM")
    if hidden_size % 16 != 0 or intermediate_size_tp % 16 != 0:
        raise KernelAvailabilityError(f"hidden ({hidden_size}) and intermediate/tp ({intermediate_size_tp}) must be multiples of 16")


def can_use_blockwise_matmul_nki(hidden_size: int, intermediate_size_tp: int, block_size: int, glu_mlp: bool = True,
                                 glu_type: Any = "glu", use_torch_block_wise: bool = False,
                                 device: Optional[torch.device] = None, logical_nc_config: int = 1, **_unused) -> bool:
    """True when the CUDA grouped GEMM will run the blockwise MLP (name kept from the reference, :719-802)."""
    if use_torch_block_wise or not check_kernel_availability(device):
        return False
    try:
        check_blockwise_mm_kernel_compatibility(hidden_size, block_size, intermediate_size_tp)
    except KernelAvailabilityError:
        return False
    return True


def augment_inputs_for_padded_blockwise_matmul(output: torch.Tensor, hidden_states: torch.Tensor,
                                               token_position_to_id: torch.Tensor, expert_affinities_masked: torch.Tensor):
    """Append one all-zero token row and point the ``-1`` padding slots at it (reference :804-850): lets a gather-based
    kernel run without a validity mask."""
    T = hidden_states.shape[0]
    zrow = lambda t: torch.cat([t, t.new_zeros(1, *t.shape[1:])])   # noqa: E731
    return (zrow(output), zrow(hidden_states), token_position_to_id.masked_fill(token_position_to_id == DEFAULT_PADDING_VALUE, T),
            zrow(expert_affinities_masked))


def _glu_act(args: BlockwiseMatmulArgs):
    import torch.nn.functional as F

    act = args.kernel_act_fn
    if isinstance(act, ActFnType):
        act = act.fn()
    elif not callable(act):
        act = F.silu

    def f(h):
        g, u = h.chunk(2, -1)
        if args.gate_clamp_upper_limit is not None or args.gate_clamp_lower_limit is not None:
            g = g.clamp(min=args.gate_clamp_lower_limit, max=args.gate_clamp_upper_limit)
        if args.up_clamp_upper_limit is not None or args.up_clamp_lower_limit is not None:
            u = u.clamp(min=args.up_clamp_lower_limit, max=args.up_clamp_upper_limit)
        return act(g) * u
    return f


def blockwise_matmul(args: BlockwiseMatmulArgs) -> torch.Tensor:
    """Run one blockwise MLP described by ``args`` (autograd-enabled: the grouped GEMM op has its own backward)."""
    mode = ExpertAffinityScaleMode.coerce(args.expert_affinities_scaling_mode)
    aff = args.expert_affinities_masked
    if mode is ExpertAffinityScaleMode.NO_SCALE:                    # plain sum of the chosen experts: weight 1 wherever routed
        aff = (aff != 0).to(aff.dtype)
    out = blockwise_mlp_from_metadata(args.hidden_states, aff, args.gate_up_proj_weight,
                                      args.down_proj_weight, args.token_position_to_id, args.block_to_expert, args.block_size,
                                      _glu_act(args), args.gate_up_proj_bias, args.down_proj_bias,
                                      pre_scale=mode is ExpertAffinityScaleMode.PRE_SCALE)
    if args.output is not None and args.is_tensor_update_accumulating:
        out = out + args.output
    return out


class BlockwiseMatmulNKIFunc:
    """Reference entry point name (:853-1035).  ``apply`` takes the reference's positional arguments and runs the grouped
    wgmma path; gradients flow through ``ops.gemm.grouped_matmul``'s autograd function."""

    @staticmethod
    def apply(hidden_states, expert_affinities_masked, gate_up_proj_weight, down_proj_weight, token_position_to_id,
              block_to_expert, block_size: int = 512, *extra, **kw):
        known = {k: v for k, v in kw.items() if k in BlockwiseMatmulArgs.__dataclass_fields__}
        return blockwise_matmul(BlockwiseMatmulArgs(hidden_states, expert_affinities_masked, gate_up_proj_weight,
                                                    down_proj_weight, token_position_to_id, block_to_expert, block_size, **known))


class TorchBlockwiseTraining(torch.autograd.Function):
    """Pure-PyTorch blockwise MLP with a hand-written backward (reference :470-680): the oracle the grouped kernel is
    tested against; block loop over gathered rows, SiLU-GLU only."""

    @staticmethod
    def forward(ctx, hidden_states, expert_affinities_masked, token_position_to_id, block_to_expert, gate_up_proj_weight,
                down_proj_weight):
        T, H = hidden_states.shape
        nb = block_to_expert.numel()
        B = token_position_to_id.numel() // nb
        ids = token_position_to_id.view(nb, B).long()
        out = torch.zeros(T, H, dtype=torch.float32, device=hidden_states.device)
        for b in range(nb):
            e = int(block_to_expert[b])
            valid = ids[b] >= 0
            if not bool(valid.any()):
                continue
            t = ids[b][valid]
            gu = hidden_states[t].float() @ gate_up_proj_weight[e].float()
            g, u = gu.chunk(2, -1)
            y = (torch.nn.functional.silu(g) * u) @ down_proj_weight[e].float()
            out.index_add_(0, t, y * expert_affinities_masked[t, e].float().unsqueeze(-1))
        ctx.save_for_backward(hidden_states, expert_affinities_masked, ids, block_to_expert, gate_up_proj_weight, down_proj_weight)
        return out.to(hidden_states.dtype)

    @staticmethod
    def backward(ctx, grad_out):
        x, aff, ids, b2e, w1, w2 = ctx.saved_tensors
        gx, gaff = torch.zeros_like(x, dtype=torch.float32), torch.zeros_like(aff, dtype=torch.float32)
        gw1, gw2 = torch.zeros_like(w1, dtype=torch.float32), torch.zeros_like(w2, dtype=torch.float32)
        for b in range(b2e.numel()):
            e = int(b2e[b])
            valid = ids[b] >= 0
            if not bool(valid.any()):
                continue
            t = ids[b][valid]
            xt, go = x[t].float(), grad_out[t].float()
            gu = xt @ w1[e].float()
            g, u = gu.chunk(2, -1)
            sg = torch.sigmoid(g)
            act = g * sg
            hmid = act * u
            y = hmid @ w2[e].float()
            a = aff[t, e].float().unsqueeze(-1)
            gaff[t, e] += (go * y).sum(-1)
            gy = go * a
            gw2[e] += hmid.t() @ gy
            ghm = gy @ w2[e].float().t()
            gg = ghm * u * (sg * (1 + g * (1 - sg)))
            ggu = torch.cat([gg, ghm * act], -1)
            gw1[e] += xt.t() @ ggu
            gx.index_add_(0, t, ggu @ w1[e].float().t())
        return gx.to(x.dtype), gaff.to(aff.dtype), None, None, gw1.to(w1.dtype), gw2.to(w2.dtype)


def _dyn_slice(tensor: torch.Tensor, starts, sizes) -> torch.Tensor:
    """Slice with start offsets that may be 0-d device tensors WITHOUT reading them on the host (CUDA-graph safe): gather
    along each dim with ``start + arange(size)``; python ints take the free ``narrow`` path."""
    out = tensor
    for d, (st, sz) in enumerate(zip(starts, sizes)):
        if isinstance(st, torch.Tensor):
            out = out.index_select(d, st.reshape(()).to(torch.long) + torch.arange(sz, device=out.device))
        else:
            out = out.narrow(d, int(st), sz)
    return out


def dynamic_slice_3D(tensor, start0, start1, start2, size0, size1, size2):  # noqa: N802
    return _dyn_slice(tensor, (start0, start1, start2), (size0, size1, size2))


def dynamic_slice_2D(tensor, start0, start1, size0, size1):  # noqa: N802
    return _dyn_slice(tensor, (start0, start1), (size0, size1))


def dynamic_slice_1D(tensor, start0, size0):  # noqa: N802
    return _dyn_slice(tensor, (start0,), (size0,))


def get_data(tensor, transform=None):
    """``tensor.data`` (optionally transformed), ``None`` passing through."""
    if tensor is None:
        return None
    return transform(tensor.data) if transform else tensor.data


class BlockwiseMatmulMXNKIFunc:
    """Blockwise MLP on MXFP4 expert weights (reference :1037-1127).  ``gate_up_proj_weight`` / ``down_proj_weight`` are
    K-major x4-packed ``[E, N, K/4]`` (uint16) with E8M0 ``*_scale`` ``[E, N, K/32]`` — the layout of
    ``moe_fused_tkg_mx.pack_expert_weight_mxfp4``.  Inference only: the weights are expanded to bf16 ``[E, K, N]`` once per
    call and fed to the grouped GEMM (a block-scaled grouped UMMA would consume them packed)."""

    @staticmethod
    def apply(hidden_states, expert_affinities_masked, gate_up_proj_weight, down_proj_weight, token_position_to_id,
              block_to_expert, gate_up_proj_scale=None, down_proj_scale=None, block_size: int = 512, **kw):
        from .moe_fused_tkg_mx import _dequant

        dt = hidden_states.dtype if hidden_states.dtype in (torch.bfloat16, torch.float16, torch.float32) else torch.bfloat16
        w1 = _dequant(gate_up_proj_weight, gate_up_proj_scale).transpose(1, 2).to(dt).contiguous()
        w2 = _dequant(down_proj_weight, down_proj_scale).transpose(1, 2).to(dt).contiguous()
        known = {k: v for k, v in kw.items() if k in BlockwiseMatmulArgs.__dataclass_fields__}
        with torch.no_grad():
            return blockwise_matmul(BlockwiseMatmulArgs(hidden_states, expert_affinities_masked, w1, w2, token_position_to_id,
                                                        block_to_expert, block_size, **known))
