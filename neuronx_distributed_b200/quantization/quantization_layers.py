"""Quantised tensor-parallel layers (inference; reference ``quantization/quantization_layers.py:73-1414``).

``ColumnParallelLinear → QuantizedColumnParallel``, ``RowParallelLinear → QuantizedRowParallel`` and the expert-fused
MoE pair.  A layer owns ``weight`` (int8 / fp8 / x4-packed MX, ``requires_grad=False``), ``scale`` (fp32 or E8M0),
optionally ``input_scale`` (static activation quantisation) and ``bias``; all of them carry the tensor-parallel
attributes the checkpoint sharder needs, plus ``get_tensor_from_state_dict`` hooks so that torch ``qint8`` packed
checkpoints load directly (``QuantizedParallelLinearLayerStateDictAdaptor``).

Execution on H100:

* weight-only, per-tensor / per-channel — the quantised values are exact in bf16, so the GEMM runs on the upcast weight
  and the scale is a per-output-feature multiply in the epilogue (no de-quantised copy of the weight is scaled);
* blockwise / MX — block scales are expanded once per call into a bf16 weight, then the bf16 GEMM;
* fp8 weights with dynamic or static fp8 activations — ``ops.gemm_fp8``: e4m3 wgmma GEMM with the
  (per-token × per-channel) scale product applied in the epilogue;
* blockwise e4m3 weights with K-blocks of 32, 64 or 128 and dynamic activations — W8A8 with the activations quantised per
  token and per K-block (``ops.gemm_fp8.quantize_groups``) and the block-scaled FP8 GEMM (``ops.gemm_fp8.blockscaled_linear``):
  per-group wgmma partial sums promoted into fp32 with both scales, no de-quantised copy of the weight.  1-D (per output row)
  and 2-D (e.g. 128 × 128) blocks, fp32 and E8M0 block scales; the same numerics on CPU (fp32 oracle);
* MXFP8 weights with ``NXD_GEMM_MX=1`` on CUDA (more than 8 rows) — ``ops.gemm_mx.linear_mx``: MXFP8 activations and the
  block-scaled FP8 GEMM.

Layers can be built empty (``QuantizedColumnParallel(in, out, …)`` → load a quantised checkpoint) or from a float layer
(``from_float``), which — a superset of the reference — also quantises the float layer's weights when they are
materialised, so ``convert(model, q_config)`` yields a working quantised model without an offline step.
"""
from __future__ import annotations

import warnings
from abc import ABCMeta, abstractmethod
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.distributed as dist
from torch import nn
from torch.nn.parameter import Parameter

from ..modules.moe.moe_parallel_layers import ExpertFusedLinear, ExpertFusedLinearWithAsyncCommunication
from ..parallel_layers import mappings
from ..parallel_layers import parallel_state as ps
from ..parallel_layers.layers import LinearWithAsyncCommunication, ProcessGroupSafeDeepcopy, _group_info
from ..parallel_layers.utils import divide, get_padding_length, set_tensor_model_parallel_attributes
from .dequantize import blockwise_scale_dequantize, direct_cast_dequantize, scale_dequantize
from .microscaling.mx_torch import quantize_mx
from .quantization_config import (_DEFAULT_CUSTOM_QCONFIG_DICT, BASE_QCONFIG_DICT_TYPE, ActivationQuantizationType,
                                  DtypeBound, QuantizationType, QuantizedDtype, ScaleDtype, is_ocp_mx_quantized,
                                  validate_block_axis_size)
from .quantization_utils import (_cast, extract_q_scale, quantize_activation_dynamic, quantize_static_quant_activations)

_FP8 = (torch.float8_e4m3fn, torch.float8_e5m2)


def _qmax(dtype: torch.dtype) -> float:
    return 127.0 if dtype == torch.int8 else float(DtypeBound.from_torch_dtype(dtype)[0])


def _index_experts(t: torch.Tensor, idx: Optional[torch.Tensor]) -> torch.Tensor:
    if idx is None:
        return t
    if t.dtype in _FP8 and not t.is_cuda:          # CPU has no fp8 gather: index the byte view
        return t.view(torch.int8)[idx].view(t.dtype)
    return t[idx]


class QuantizedParallelLinearLayerStateDictAdaptor:
    """Reads a layer's tensors from either a plain (``weight`` / ``scale`` / ``bias`` / ``input_scale``) or a torch
    dynamic-quantisation (``_packed_params``) state dict (reference :356-463)."""

    @staticmethod
    def _packed(prefix: str, state_dict: Dict[str, Any]):
        return state_dict[prefix + "_packed_params._packed_params"] if (prefix + "_packed_params.dtype") in state_dict else None

    @staticmethod
    def get_weight_from_state_dict(prefix: str, state_dict: Dict[str, Any]) -> torch.Tensor:
        if (prefix + "weight") in state_dict:
            return state_dict[prefix + "weight"]
        packed = QuantizedParallelLinearLayerStateDictAdaptor._packed(prefix, state_dict)
        if packed is None:
            raise RuntimeError(f"Cannot find {prefix + 'weight'} in the state_dict")
        return torch.int_repr(packed[0])

    @staticmethod
    def set_weight_to_state_dict(prefix: str, tensor: torch.Tensor, state_dict: Dict[str, Any]) -> None:
        if (prefix + "weight") in state_dict:
            state_dict[prefix + "weight"] = tensor
        elif (prefix + "_packed_params.dtype") in state_dict:
            packed = list(state_dict[prefix + "_packed_params._packed_params"])
            packed[0] = tensor
            state_dict[prefix + "_packed_params._packed_params"] = tuple(packed)
        else:
            raise RuntimeError(f"Cannot find {prefix + 'weight'} in the state_dict")

    @staticmethod
    def get_bias_from_state_dict(prefix: str, state_dict: Dict[str, Any]) -> Optional[torch.Tensor]:
        if (prefix + "bias") in state_dict:
            return state_dict[prefix + "bias"]
        packed = QuantizedParallelLinearLayerStateDictAdaptor._packed(prefix, state_dict)
        if packed is None or len(packed) < 2:
            warnings.warn(f"Cannot find {prefix + 'bias'} in the state_dict")
            return None
        return packed[1].data if isinstance(packed[1], Parameter) else packed[1]

    @staticmethod
    def set_bias_to_state_dict(prefix: str, tensor: torch.Tensor, state_dict: Dict[str, Any]) -> None:
        state_dict[prefix + "bias"] = tensor

    @staticmethod
    def get_scale_from_state_dict(prefix: str, state_dict: Dict[str, Any]) -> torch.Tensor:
        packed = QuantizedParallelLinearLayerStateDictAdaptor._packed(prefix, state_dict)
        if packed is not None and packed[0].dtype == torch.qint8:
            return extract_q_scale(packed[0])
        if (prefix + "scale") in state_dict:
            return state_dict[prefix + "scale"]
        raise RuntimeError(f"Cannot find {prefix + 'scale'} in state_dict")

    @staticmethod
    def get_input_scale_from_state_dict(prefix: str, state_dict: Dict[str, Any]) -> torch.Tensor:
        if (prefix + "input_scale") in state_dict:
            return state_dict[prefix + "input_scale"]
        raise RuntimeError(f"Cannot find {prefix + 'input_scale'} in state_dict")


class BaseQuantizeParallelLinear(ProcessGroupSafeDeepcopy, nn.Module, metaclass=ABCMeta):
    """Parameter set-up shared by all quantised parallel layers (reference :73-354)."""

    autograd_func_class = LinearWithAsyncCommunication

    def __init__(self, quantization_type: Union[QuantizationType, str] = "per_tensor_symmetric",
                 dequantized_dtype: torch.dtype = torch.bfloat16,
                 quantized_dtype: Union[QuantizedDtype, torch.dtype] = QuantizedDtype.INT8,
                 device: Optional[torch.device] = None, tensor_model_parallel_group=None,
                 rank_ordering: Optional[Sequence[int]] = None,
                 scale_dtype: Union[ScaleDtype, torch.dtype] = ScaleDtype.F32) -> None:
        super().__init__()
        assert quantization_type in QuantizationType, \
            f"{quantization_type} quantization is not supported. Specify from {[e.value for e in QuantizationType]}"
        assert quantized_dtype in QuantizedDtype, \
            f"{quantized_dtype} quantization is not supported. Specify from {[e.value for e in QuantizedDtype]}"
        if not ps.model_parallel_is_initialized():
            ps.initialize_fallback_parallel_state()
        self.quantization_type = QuantizationType(quantization_type)
        self.dequantized_dtype = dequantized_dtype
        self.quantized_dtype = quantized_dtype if isinstance(quantized_dtype, QuantizedDtype) else QuantizedDtype(quantized_dtype)
        self.scale_dtype = scale_dtype if isinstance(scale_dtype, ScaleDtype) else ScaleDtype(scale_dtype)
        self.device = device
        self.tensor_parallel_group, self._tp, self._tp_rank = _group_info(tensor_model_parallel_group)
        self.rank_ordering = rank_ordering
        self.register_parameter("scale", None)
        self.keep_master_weight: Optional[bool] = None
        self.weight_shape: Optional[Sequence[int]] = None
        self.weight_partition_dim: Optional[int] = None
        self.stride: int = 1
        self.bias_shape: Optional[Sequence[int]] = None
        self.mx_swizzle = False
        self.block_axis: Optional[List[int]] = None
        self.block_size: Optional[List[int]] = None
        self.per_channel_axis: Optional[int] = None
        self.activation_quantization_type = ActivationQuantizationType.NONE
        self.clamp_bound = float("inf")

    # ------------------------------------------------------------------------------------------------ parameters
    def _setup_for_weight(self) -> None:
        assert self.weight_shape is not None and self.weight_partition_dim is not None
        packed = list(self.weight_shape)
        n = self.quantized_dtype.get_packed_count()
        assert packed[-1] % n == 0, f"last weight dim {packed[-1]} must be divisible by the packed count {n}"
        packed[-1] //= n
        w = torch.zeros(*packed, dtype=torch.uint8 if self.quantized_dtype.value.itemsize == 1 else torch.int16
                        if self.quantized_dtype.value.itemsize == 2 else torch.int32,
                        device=self.device or torch.device("cpu")).view(self.quantized_dtype.value)
        self.weight = Parameter(w, requires_grad=False)
        self.device = self.weight.device
        set_tensor_model_parallel_attributes(self.weight, True, self.weight_partition_dim, self.stride, num_partitions=self._tp)
        if self.rank_ordering is not None:
            self.weight.rank_ordering = list(self.rank_ordering)
        self.weight.get_tensor_from_state_dict = self.get_weight_from_state_dict
        self.weight.set_tensor_to_state_dict = self.set_weight_to_state_dict
        self.master_weight = None

    def _base_setup_for_bias(self, bias: bool) -> None:
        if not bias:
            self.register_parameter("bias", None)
            return
        assert self.bias_shape is not None
        self.bias = Parameter(torch.zeros(*self.bias_shape, dtype=self.dequantized_dtype, device=self.device), requires_grad=False)
        self.bias.get_tensor_from_state_dict = self.get_bias_from_state_dict
        self.bias.set_tensor_to_state_dict = self.set_bias_to_state_dict

    def _new_scale(self, shape: Sequence[int]) -> Parameter:
        return Parameter(torch.full(tuple(shape), self.scale_dtype.get_default_scale(), device=self.weight.device,
                                    dtype=self.scale_dtype.value), requires_grad=False)

    def _setup_for_scale(self, weight_shape: Sequence[int], quantization_type: QuantizationType,
                         weight_partition_dim: Optional[int] = None, per_channel_axis: Optional[int] = None,
                         block_axis: Optional[List[int]] = None, block_size: Optional[List[int]] = None,
                         activation_quantization_type: Optional[ActivationQuantizationType] = None) -> None:
        """Scale shapes (reference :205-303): per-tensor ``[1]``; per-channel ``[1,…,C,…,1]`` (``[E,…]`` expert-wise);
        blockwise ``weight_shape // block_size`` on the blocked axes.  A scale is tensor-parallel exactly when the
        axis it varies along is the weight's partition axis."""
        nd = len(weight_shape)
        replicated = dict(is_parallel=False, dim=0, stride=1, num_partitions=1)
        if quantization_type == QuantizationType.PER_TENSOR_SYMMETRIC:
            self.scale = self._new_scale([1])
            set_tensor_model_parallel_attributes(self.scale, **replicated)
            if activation_quantization_type == ActivationQuantizationType.STATIC:
                self.input_scale = self._new_scale([1])
                set_tensor_model_parallel_attributes(self.input_scale, **replicated)
                self.input_scale.get_tensor_from_state_dict = BaseQuantizeParallelLinear.get_input_scale_from_state_dict
        elif quantization_type in (QuantizationType.PER_CHANNEL_SYMMETRIC, QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC):
            assert per_channel_axis is not None, "per_channel_axis cannot be None for per_channel_symmetric quantization"
            per_channel_axis %= nd
            shape = [1] * nd
            shape[per_channel_axis] = weight_shape[per_channel_axis]
            if quantization_type == QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC:
                shape[0] = self._n_local_experts
            self.scale = self._new_scale(shape)
            if weight_partition_dim == per_channel_axis:
                set_tensor_model_parallel_attributes(self.scale, True, weight_partition_dim, self.stride, num_partitions=self._tp)
                if self.rank_ordering is not None:
                    self.scale.rank_ordering = list(self.rank_ordering)
            else:
                set_tensor_model_parallel_attributes(self.scale, **replicated)
        elif quantization_type == QuantizationType.BLOCKWISE_SYMMETRIC:
            block_axis, block_size = validate_block_axis_size(block_axis, block_size)
            block_axis = [a % nd for a in block_axis]
            shape = list(weight_shape)
            for ax, sz in zip(block_axis, block_size):
                if weight_shape[ax] < sz:
                    assert ax == weight_partition_dim, (f"dim {ax} of weight {tuple(weight_shape)} is smaller than block size "
                                                        f"{sz} and is not the partition dim {weight_partition_dim}")
                    shape[ax] = 1
                else:
                    assert weight_shape[ax] % sz == 0, f"weight dim {ax} ({weight_shape[ax]}) not divisible by block size {sz}"
                    shape[ax] = weight_shape[ax] // sz
            self.block_axis, self.block_size = block_axis, list(block_size)
            self.scale = self._new_scale(shape)
            set_tensor_model_parallel_attributes(self.scale, True, weight_partition_dim, self.stride, num_partitions=self._tp)
        else:
            raise ValueError(f"scale for quantization_type: {quantization_type} not supported")
        self.per_channel_axis = per_channel_axis
        self.scale.get_tensor_from_state_dict = BaseQuantizeParallelLinear.get_scale_from_state_dict

    # state-dict hooks ------------------------------------------------------------------------------------------
    get_weight_from_state_dict = staticmethod(QuantizedParallelLinearLayerStateDictAdaptor.get_weight_from_state_dict)
    set_weight_to_state_dict = staticmethod(QuantizedParallelLinearLayerStateDictAdaptor.set_weight_to_state_dict)
    get_bias_from_state_dict = staticmethod(QuantizedParallelLinearLayerStateDictAdaptor.get_bias_from_state_dict)
    set_bias_to_state_dict = staticmethod(QuantizedParallelLinearLayerStateDictAdaptor.set_bias_to_state_dict)
    get_scale_from_state_dict = staticmethod(QuantizedParallelLinearLayerStateDictAdaptor.get_scale_from_state_dict)
    get_input_scale_from_state_dict = staticmethod(QuantizedParallelLinearLayerStateDictAdaptor.get_input_scale_from_state_dict)

    @staticmethod
    def _apply_post_quantization_hook(mod: nn.Module, new_mod: nn.Module) -> nn.Module:
        hook = getattr(mod, "post_create_quantized_module_hook", None)
        if hook is not None:
            hook(new_mod)
        return new_mod

    @classmethod
    @abstractmethod
    def from_float(cls, mod, q_config: BASE_QCONFIG_DICT_TYPE = _DEFAULT_CUSTOM_QCONFIG_DICT):
        """Create the quantised counterpart of a float parallel layer."""

    # ------------------------------------------------------------------------------------------------ quantisation
    def _is_mx(self) -> bool:
        return is_ocp_mx_quantized(self.quantization_type, self.quantized_dtype, self.scale_dtype)

    def _allreduce_max(self, t: torch.Tensor) -> torch.Tensor:
        if self._tp > 1 and self.tensor_parallel_group is not None:
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.tensor_parallel_group)
        return t

    def _to_scale_dtype(self, scale_f32: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """(stored scale, fp32 scale actually applied) — E8M0 rounds the scale UP to a power of two (no saturation)."""
        if self.scale_dtype == ScaleDtype.F32:
            return scale_f32, scale_f32
        e = torch.ceil(torch.log2(scale_f32.clamp(min=2.0 ** -126)))
        return (e + 127).clamp(0, 254).to(torch.uint8), torch.pow(2.0, e)

    @torch.no_grad()
    def quantize_from_float_weight(self, w: torch.Tensor) -> None:
        """Fill ``weight`` / ``scale`` from this rank's float shard ``w`` (same logical shape as ``weight_shape``).
        Scales that are replicated across TP are computed from the all-reduced absmax so every rank stores the same."""
        qd = self.quantized_dtype.value
        wf = w.detach().float()
        if self.clamp_bound != float("inf"):
            wf = wf.clamp(-self.clamp_bound, self.clamp_bound)
        qt = self.quantization_type
        if self._is_mx():
            assert self.block_axis == [wf.dim() - 1] and self.block_size == [32], "MX blocks are 32 along the last dim"
            kind = "mxfp4" if self.quantized_dtype == QuantizedDtype.F4E2M1FN_X4 else "mxfp8"
            packed, e8m0 = quantize_mx(wf, kind)
            self.weight.data.copy_(packed.view(self.weight.dtype))
            self.scale.data.copy_(e8m0)
            return
        if qt == QuantizationType.BLOCKWISE_SYMMETRIC:
            view, red = [], []
            for d, n in enumerate(wf.shape):
                if d in self.block_axis:
                    b = min(self.block_size[self.block_axis.index(d)], n)
                    view += [n // b, b]
                    red.append(len(view) - 1)
                else:
                    view.append(n)
            wv = wf.reshape(view)
            stored, s = self._to_scale_dtype((wv.abs().amax(dim=red, keepdim=True) / _qmax(qd)).clamp(min=1e-12))
            self.weight.data.copy_(_cast(wv / s, qd).reshape(wf.shape))
            self.scale.data.copy_(stored.reshape(self.scale.shape))
            return
        if qt == QuantizationType.PER_TENSOR_SYMMETRIC:
            amax = wf.abs().max().reshape(1)
        else:
            keep = {self.per_channel_axis} | ({0} if qt == QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC else set())
            amax = wf.abs().amax(dim=[d for d in range(wf.dim()) if d not in keep], keepdim=True)
        if not getattr(self.scale, "tensor_model_parallel", False):
            amax = self._allreduce_max(amax.contiguous())
        stored, s = self._to_scale_dtype((amax / _qmax(qd)).clamp(min=1e-12))
        self.weight.data.copy_(_cast(wf / s, qd))
        self.scale.data.copy_(stored.reshape(self.scale.shape))

    def _maybe_quantize_from(self, mod: nn.Module) -> None:
        w = getattr(mod, "weight", None)
        if w is None or w.device.type == "meta" or tuple(w.shape) != tuple(self.weight_shape):
            return
        self.quantize_from_float_weight(w.data)
        if self.bias is not None and getattr(mod, "bias", None) is not None and mod.bias.device.type != "meta":
            self.bias.data.copy_(mod.bias.data.to(self.bias.dtype))

    # ------------------------------------------------------------------------------------------------ math
    def _scale_f32(self, scale: torch.Tensor) -> torch.Tensor:
        if scale.dtype == torch.uint8:
            return torch.pow(2.0, scale.float() - 127.0)
        return scale.float()

    def _dequantized_weight(self, weight: torch.Tensor, scale: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
        if self.quantization_type == QuantizationType.BLOCKWISE_SYMMETRIC:
            return blockwise_scale_dequantize(weight, scale, dtype, mx_swizzle=self.mx_swizzle)
        return (direct_cast_dequantize(weight, torch.float32) * self._scale_f32(scale)).to(dtype)

    def _scale_is_output_only(self, out_axis: int) -> bool:
        """True when the scale varies along the output-feature axis only → it can be applied after the GEMM."""
        if self.quantization_type == QuantizationType.BLOCKWISE_SYMMETRIC:
            return False
        if self.quantization_type == QuantizationType.PER_TENSOR_SYMMETRIC:
            return True
        return self.per_channel_axis == out_axis % len(self.weight_shape)

    def _blockscaled_group(self) -> int:
        """Size G of the K-blocks when the layer runs W8A8 on the block-scaled FP8 GEMM (block-wise e4m3 weight, dynamic
        activations, G ∈ {32, 64, 128} dividing this rank's K so row-parallel shards keep whole blocks), else 0.  K is
        axis 1 of both a dense ``[N, K]`` and an expert-fused ``[E, K, N]`` weight; expert scales must be per expert."""
        if (self.quantization_type != QuantizationType.BLOCKWISE_SYMMETRIC
                or self.activation_quantization_type != ActivationQuantizationType.DYNAMIC
                or self.weight.dtype != torch.float8_e4m3fn or self.weight.dim() not in (2, 3) or self.mx_swizzle
                or 1 not in self.block_axis):
            return 0
        G, K = self.block_size[self.block_axis.index(1)], self.weight.shape[1]
        if (G not in (32, 64, 128) or K % G or self.scale.dim() != self.weight.dim() or self.scale.shape[1] != K // G
                or (self.weight.dim() == 3 and self.scale.shape[0] != self.weight.shape[0])):
            return 0
        return G

    def _linear_2d(self, x: torch.Tensor) -> torch.Tensor:
        """``x [..., K] @ weight[N, K]ᵀ`` with the layer's quantisation scheme; returns ``[..., N]`` in x's dtype class."""
        out_dtype = x.dtype if x.dtype in (torch.bfloat16, torch.float16, torch.float32) else self.dequantized_dtype
        qd = self.weight.dtype
        act = self.activation_quantization_type
        w_scale = self._scale_f32(self.scale)
        if act != ActivationQuantizationType.NONE and self._scale_is_output_only(0) and qd in _FP8 + (torch.int8,):
            if act == ActivationQuantizationType.DYNAMIC:
                aq_dtype = qd if qd in _FP8 else torch.float8_e4m3fn
                xq, xs = quantize_activation_dynamic(x, aq_dtype, None if self.clamp_bound == float("inf") else self.clamp_bound)
            else:
                assert self.quantization_type == QuantizationType.PER_TENSOR_SYMMETRIC, \
                    "Static activation quantization is only supported for PER TENSOR quantization type."
                xq = quantize_static_quant_activations(x, self._scale_f32(self.input_scale), qd)
                xs = self._scale_f32(self.input_scale).reshape(1).expand(*x.shape[:-1], 1)
            ws = w_scale.reshape(-1) if w_scale.numel() > 1 else w_scale.reshape(1).expand(self.weight.shape[0])
            if qd in _FP8 and xq.dtype == qd:
                from ..ops import gemm_fp8

                return gemm_fp8.scaled_linear(xq, xs, self.weight, ws, out_dtype=out_dtype)
            y = torch.matmul(xq.float(), self.weight.float().t()) * xs.float() * ws.reshape(1, -1)
            return y.to(out_dtype)
        G = self._blockscaled_group()
        if G:
            from ..ops import gemm_fp8

            xq, xs = gemm_fp8.quantize_groups(x, G, "absmax", None if self.clamp_bound == float("inf") else self.clamp_bound)
            return gemm_fp8.blockscaled_linear(xq, xs, self.weight, self.scale, G, out_dtype=out_dtype)
        if self._scale_is_output_only(0):
            y = torch.nn.functional.linear(x.to(out_dtype), direct_cast_dequantize(self.weight, out_dtype))
            return scale_dequantize(y, w_scale.reshape(1, -1) if w_scale.numel() > 1 else w_scale, out_dtype)
        if self._is_mx() and x.is_cuda and self.weight.dim() == 2 and not self.mx_swizzle:
            from ..ops import gemm_mx

            x2 = x.reshape(-1, x.shape[-1])
            if gemm_mx.gemv_eligible(x2.contiguous(), self.weight, self.scale):
                # token generation on MX weights: decode the codes in registers, read 4.25 / 8.25 bits per weight
                return gemm_mx.linear_mx(x, self.weight, self.scale).to(out_dtype)
            if gemm_mx.gemm_mx_eligible(x2, self.weight, self.scale, gemm_mx.kind_of(self.weight)):
                # prefill on MXFP8 weights (opt-in): MXFP8 activations and the block-scaled FP8 GEMM
                return gemm_mx.linear_mx(x, self.weight, self.scale).to(out_dtype)
        return torch.nn.functional.linear(x.to(out_dtype), self._dequantized_weight(self.weight, self.scale, out_dtype))

    def _linear_experts(self, x: torch.Tensor, expert_indices: Optional[torch.Tensor]) -> torch.Tensor:
        """``x [E, …, K] · weight[E, K, N]`` → ``[E, …, N]`` (expert-fused layers).  W8A8 expert layers quantise ``x`` per
        token and K-block as the grouped path does and run the fp32 oracle of the quantised operands."""
        weight, scale = _index_experts(self.weight, expert_indices), _index_experts(self.scale, expert_indices) \
            if self.scale.shape[0] > 1 else self.scale
        dt = x.dtype
        G = self._blockscaled_group()
        if G:
            from ..ops import gemm_fp8

            K = x.shape[-1]
            xq, xs = gemm_fp8.quantize_groups(x, G, "absmax", None if self.clamp_bound == float("inf") else self.clamp_bound)
            xd = gemm_fp8._dequant_groups(xq.reshape(-1, K), xs.reshape(-1, K // G), G).reshape(x.shape)
            return torch.einsum("e...h,ehi->e...i", xd, blockwise_scale_dequantize(weight, scale, torch.float32)).to(dt)
        if self._scale_is_output_only(2):
            y = torch.einsum("e...h,ehi->e...i", x, direct_cast_dequantize(weight, dt))
            s = self._scale_f32(scale)
            s = s.reshape(s.shape[0], *([1] * (y.dim() - 2)), s.shape[-1])
            return (y.float() * s).to(dt)
        return torch.einsum("e...h,ehi->e...i", x, self._dequantized_weight(weight, scale, dt))


# =====================================================================================================================
# Column / Row
# =====================================================================================================================
class QuantizedColumnParallel(BaseQuantizeParallelLinear):
    """``Y = X Aᵀ`` with A ``[out, in]`` split along ``out`` (reference :465-742)."""

    def __init__(self, input_size: int, output_size: int, bias: bool = True,
                 quantization_type: Union[QuantizationType, str] = "per_tensor_symmetric", gather_output: bool = True,
                 dtype: torch.dtype = torch.float32, quantized_dtype: Union[QuantizedDtype, torch.dtype] = QuantizedDtype.INT8,
                 device: Optional[torch.device] = None, stride: int = 1, sequence_parallel_enabled: bool = False,
                 sequence_dimension: Optional[int] = None, keep_master_weight: bool = False,
                 quantization_per_channel_axis: Optional[int] = None, block_axis: Optional[List[int]] = None,
                 block_size: Optional[List[int]] = None, scale_dtype: Union[torch.dtype, ScaleDtype] = torch.float32,
                 tensor_model_parallel_group=None, pad: bool = False,
                 activation_quantization_type: Optional[Union[ActivationQuantizationType, str]] = None,
                 clamp_bound: float = float("inf"), rank_ordering: Optional[Sequence[int]] = None):
        if QuantizationType(quantization_type) == QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC and \
                "_n_local_experts" not in self.__dict__:
            # a model-wide expert-wise config also reaches the dense layers (router-side / shared experts): per-channel there
            quantization_type = QuantizationType.PER_CHANNEL_SYMMETRIC
        super().__init__(quantization_type=quantization_type, dequantized_dtype=dtype, quantized_dtype=quantized_dtype,
                         device=device, tensor_model_parallel_group=tensor_model_parallel_group,
                         rank_ordering=rank_ordering, scale_dtype=scale_dtype)
        self.activation_quantization_type = ActivationQuantizationType(activation_quantization_type)
        self.clamp_bound = clamp_bound
        self.input_size, self.output_size, self.gather_output = input_size, output_size, gather_output
        self.pad, self.pad_size = pad, 0
        if pad:
            self.pad_size = get_padding_length(output_size, self._tp)
            self.output_size = output_size + self.pad_size
        self.output_size_per_partition = divide(self.output_size, self._tp)
        self.stride, self.keep_master_weight = stride, keep_master_weight
        if sequence_parallel_enabled and sequence_dimension is None:
            sequence_dimension = 0
        self.sequence_parallel_enabled, self.sequence_dimension = sequence_parallel_enabled, sequence_dimension
        self._setup_for_weight_and_bias_config(bias)
        self._setup_for_weight()
        self._setup_for_bias(bias)
        if self.quantization_type == QuantizationType.PER_CHANNEL_SYMMETRIC and quantization_per_channel_axis is None:
            quantization_per_channel_axis = self._default_channel_axis
        self._setup_for_scale(self.weight_shape, self.quantization_type, self.weight_partition_dim,
                              quantization_per_channel_axis, block_axis, block_size, self.activation_quantization_type)
        self._setup_for_parallelism(self._tp)

    _default_channel_axis = 0

    def _setup_for_weight_and_bias_config(self, bias: bool) -> None:
        self.weight_shape = (self.output_size_per_partition, self.input_size)
        self.weight_partition_dim = 0
        self.bias_shape = ((self.output_size if self.gather_output else self.output_size_per_partition),) if bias else None

    def _setup_for_bias(self, bias: bool) -> None:
        self._base_setup_for_bias(bias)
        if bias and not self.gather_output:
            set_tensor_model_parallel_attributes(self.bias, True, 0, self.stride, num_partitions=self._tp)

    def _setup_for_parallelism(self, world_size: int) -> None:
        self.async_tensor_model_parallel_allreduce = not self.sequence_parallel_enabled and world_size > 1
        if self.sequence_parallel_enabled and world_size <= 1:
            warnings.warn(f"`sequence_parallel_enabled` is set to `True`, but got world_size of {world_size}")

    def forward(self, input: torch.Tensor, *args: Any, **kwargs: Any) -> torch.Tensor:  # noqa: A002
        x = input
        if self.sequence_parallel_enabled:
            x = mappings.gather_from_sequence_parallel_region(x, self.sequence_dimension, True, self.tensor_parallel_group)
        y = self._linear_2d(x)
        if self.gather_output:
            assert not self.sequence_parallel_enabled
            y = mappings.gather_from_tensor_model_parallel_region(y, self.tensor_parallel_group)
            if self.pad and self.pad_size > 0:
                y = y.narrow(-1, 0, self.output_size - self.pad_size)
        if self.bias is None:
            return y
        b = self.bias
        if self.gather_output and self.pad and self.pad_size > 0:
            b = b.narrow(0, 0, self.output_size - self.pad_size)
        return y + b.to(y.dtype)

    @classmethod
    def from_float(cls, mod, q_config: BASE_QCONFIG_DICT_TYPE = _DEFAULT_CUSTOM_QCONFIG_DICT):
        assert mod.__class__.__name__ == "ColumnParallelLinear", "ColumnParallelLinear expected"
        new_mod = cls(
            input_size=mod.input_size, output_size=mod.output_size - (mod.pad_size if mod.pad else 0),
            bias=mod.bias is not None, quantization_type=q_config["quantization_type"],
            quantized_dtype=q_config["quantized_dtype"], gather_output=mod.gather_output, dtype=mod.dtype,
            device=mod.weight.device, stride=mod.stride, sequence_parallel_enabled=mod.sequence_parallel_enabled,
            sequence_dimension=mod.sequence_dimension, keep_master_weight=mod.keep_master_weight,
            quantization_per_channel_axis=q_config.get("quantization_per_channel_axis"),
            tensor_model_parallel_group=mod.tensor_parallel_group, pad=mod.pad,
            activation_quantization_type=q_config.get("activation_quantization_type"),
            clamp_bound=q_config.get("clamp_bound", float("inf")), block_axis=q_config.get("block_axis"),
            block_size=q_config.get("block_size"), scale_dtype=q_config.get("scale_dtype", torch.float32),
            rank_ordering=getattr(mod, "rank_ordering", None))
        new_mod._maybe_quantize_from(mod)
        return cls._apply_post_quantization_hook(mod, new_mod)

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        """Zero-pad the full quantised weight (and its per-channel scale) along the output dim (reference :731-742)."""
        if not self.pad or self.pad_size == 0:
            return
        w = model_state_dict[prefix]
        if self.output_size != w.shape[0] + self.pad_size:
            raise RuntimeError(f"State dict {prefix} is of an unexpected size {w.shape[0]} expected {self.output_size - self.pad_size}")
        model_state_dict[prefix] = _pad_rows(w, self.pad_size)
        assert prefix.endswith(".weight") or prefix == "weight"
        sk = prefix[: -len("weight")] + "scale"
        if sk in model_state_dict and model_state_dict[sk].dim() == 2 and model_state_dict[sk].shape[0] == w.shape[0]:
            model_state_dict[sk] = torch.nn.functional.pad(model_state_dict[sk], (0, 0, 0, self.pad_size), value=1.0)


def _pad_rows(w: torch.Tensor, n: int) -> torch.Tensor:
    if w.dtype in _FP8:                 # no fp8 pad kernel on CPU: pad the byte view (0x00 is +0 in both formats)
        return torch.nn.functional.pad(w.view(torch.uint8), (0, 0, 0, n)).view(w.dtype)
    return torch.nn.functional.pad(w, (0, 0, 0, n))


class QuantizedRowParallel(BaseQuantizeParallelLinear):
    """``Y = X Aᵀ`` with A ``[out, in]`` split along ``in``; partial sums all-reduced / reduce-scattered
    (reference :744-1011)."""

    def __init__(self, input_size: int, output_size: int, bias: bool = True,
                 quantization_type: Union[QuantizationType, str] = "per_tensor_symmetric", input_is_parallel: bool = False,
                 dtype: torch.dtype = torch.float32, quantized_dtype: Union[QuantizedDtype, torch.dtype] = QuantizedDtype.INT8,
                 device: Optional[torch.device] = None, stride: int = 1, sequence_parallel_enabled: bool = False,
                 sequence_dimension: Optional[int] = None, keep_master_weight: bool = False,
                 quantization_per_channel_axis: Optional[int] = None, reduce_output: bool = True,
                 block_axis: Optional[List[int]] = None, block_size: Optional[List[int]] = None,
                 scale_dtype: Union[torch.dtype, ScaleDtype] = torch.float32, tensor_model_parallel_group=None,
                 pad: bool = False, activation_quantization_type: Optional[Union[ActivationQuantizationType, str]] = None,
                 clamp_bound: float = float("inf"), rank_ordering: Optional[Sequence[int]] = None):
        if QuantizationType(quantization_type) == QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC and \
                "_n_local_experts" not in self.__dict__:
            # a model-wide expert-wise config also reaches the dense layers (router-side / shared experts): per-channel there
            quantization_type = QuantizationType.PER_CHANNEL_SYMMETRIC
        super().__init__(quantization_type=quantization_type, dequantized_dtype=dtype, quantized_dtype=quantized_dtype,
                         device=device, tensor_model_parallel_group=tensor_model_parallel_group,
                         rank_ordering=rank_ordering, scale_dtype=scale_dtype)
        self.activation_quantization_type = ActivationQuantizationType(activation_quantization_type)
        self.clamp_bound = clamp_bound
        self.input_size, self.output_size, self.input_is_parallel = input_size, output_size, input_is_parallel
        self.pad, self.pad_size = pad, 0
        if pad:
            self.pad_size = get_padding_length(input_size, self._tp)
            self.input_size = input_size + self.pad_size
        self.input_size_per_partition = divide(self.input_size, self._tp)
        self.stride, self.keep_master_weight, self.reduce_output = stride, keep_master_weight, reduce_output
        if sequence_parallel_enabled and sequence_dimension is None:
            sequence_dimension = 0
        self.sequence_parallel_enabled, self.sequence_dimension = sequence_parallel_enabled, sequence_dimension
        if sequence_parallel_enabled and not input_is_parallel:
            raise RuntimeError("To enable `sequence_parallel_enabled`, `input_is_parallel` must be `True`")
        self._setup_for_weight_and_bias_config(bias)
        self._setup_for_weight()
        self._setup_for_bias(bias)
        if self.quantization_type == QuantizationType.PER_CHANNEL_SYMMETRIC and quantization_per_channel_axis is None:
            quantization_per_channel_axis = self._default_channel_axis
        self._setup_for_scale(self.weight_shape, self.quantization_type, self.weight_partition_dim,
                              quantization_per_channel_axis, block_axis, block_size, self.activation_quantization_type)

    _default_channel_axis = 0

    def _setup_for_weight_and_bias_config(self, bias: bool) -> None:
        self.weight_shape = (self.output_size, self.input_size_per_partition)
        self.weight_partition_dim = 1
        self.bias_shape = (self.output_size,) if bias else None

    def _setup_for_bias(self, bias: bool) -> None:
        self._base_setup_for_bias(bias)
        if bias:
            self.bias.sequence_parallel_enabled = self.sequence_parallel_enabled

    def _reduce(self, y: torch.Tensor) -> torch.Tensor:
        if not self.reduce_output:
            return y
        if self.sequence_parallel_enabled:
            return mappings.reduce_scatter_to_sequence_parallel_region(y, self.sequence_dimension, self.tensor_parallel_group)
        return mappings.reduce_from_tensor_model_parallel_region(y, self.tensor_parallel_group)

    def forward(self, input_: torch.Tensor, *args: Any, **kwargs: Any) -> torch.Tensor:
        x = input_
        if not self.input_is_parallel:
            assert not self.sequence_parallel_enabled
            if self.pad and self.pad_size > 0:
                x = torch.nn.functional.pad(x, (0, self.pad_size))
            x = mappings.scatter_to_tensor_model_parallel_region(x, self.tensor_parallel_group)
        y = self._reduce(self._linear_2d(x))
        return y if self.bias is None else y + self.bias.to(y.dtype)

    @classmethod
    def from_float(cls, mod, q_config: BASE_QCONFIG_DICT_TYPE = _DEFAULT_CUSTOM_QCONFIG_DICT):
        assert mod.__class__.__name__ == "RowParallelLinear", "RowParallelLinear expected"
        new_mod = cls(
            input_size=mod.input_size - (mod.pad_size if mod.pad else 0), output_size=mod.output_size,
            bias=mod.bias is not None, quantization_type=q_config["quantization_type"],
            input_is_parallel=mod.input_is_parallel, dtype=mod.dtype, quantized_dtype=q_config["quantized_dtype"],
            device=mod.weight.device, stride=mod.stride, sequence_parallel_enabled=mod.sequence_parallel_enabled,
            sequence_dimension=mod.sequence_dimension, keep_master_weight=mod.keep_master_weight,
            quantization_per_channel_axis=q_config.get("quantization_per_channel_axis"), reduce_output=mod.reduce_output,
            tensor_model_parallel_group=mod.tensor_parallel_group, pad=mod.pad,
            activation_quantization_type=q_config.get("activation_quantization_type"),
            clamp_bound=q_config.get("clamp_bound", float("inf")), block_axis=q_config.get("block_axis"),
            block_size=q_config.get("block_size"), scale_dtype=q_config.get("scale_dtype", torch.float32),
            rank_ordering=getattr(mod, "rank_ordering", None))
        new_mod._maybe_quantize_from(mod)
        return cls._apply_post_quantization_hook(mod, new_mod)

    def preshard_hook(self, model_state_dict: Dict[str, Any], prefix: str) -> None:
        """Zero-pad the full quantised weight along the input dim (reference :1005-1011)."""
        if not self.pad or self.pad_size == 0:
            return
        w = model_state_dict[prefix]
        if self.input_size != w.shape[1] + self.pad_size:
            raise RuntimeError(f"State dict {prefix} is of an unexpected size {w.shape[1]} expected {self.input_size - self.pad_size}")
        if w.dtype in _FP8:
            model_state_dict[prefix] = torch.nn.functional.pad(w.view(torch.uint8), (0, self.pad_size)).view(w.dtype)
        else:
            model_state_dict[prefix] = torch.nn.functional.pad(w, (0, self.pad_size))


# =====================================================================================================================
# Expert-fused (MoE)
# =====================================================================================================================
def _check_expert_activation_quantization(t) -> None:
    if ActivationQuantizationType(t) == ActivationQuantizationType.STATIC:
        raise ValueError("expert-fused layers take no static input scale: activation quantisation must be none or dynamic")


def _expert_activation_quantization(q_config: BASE_QCONFIG_DICT_TYPE) -> ActivationQuantizationType:
    """The q_config's activation quantisation for expert-fused layers.  A static input scale belongs to one dense layer
    and the fused experts have none, so a static config leaves the experts weight-only."""
    t = ActivationQuantizationType(q_config.get("activation_quantization_type"))
    return ActivationQuantizationType.NONE if t == ActivationQuantizationType.STATIC else t


class _QuantizedExpertMixin(ExpertFusedLinear):
    autograd_func_class = ExpertFusedLinearWithAsyncCommunication
    _default_channel_axis = 2

    def _expert_setup(self, num_experts: int, expert_model_parallel_group, is_prefill: bool, is_fused_gate_up: bool) -> None:
        self.num_experts = num_experts
        if expert_model_parallel_group is not None:
            self.ep = dist.get_world_size(expert_model_parallel_group)
        else:
            self.ep = ps.get_expert_model_parallel_size()
        self.expert_model_parallel_group = expert_model_parallel_group
        self._n_local_experts = self.num_local_experts = divide(num_experts, self.ep)
        r = dist.get_rank(expert_model_parallel_group) if expert_model_parallel_group is not None else \
            ps.get_expert_model_parallel_rank()
        self.local_expert_ids = ps.get_experts_for_expert_parallel_rank(r, num_experts, self.ep)
        self.is_prefill, self.is_fused_gate_up = is_prefill, is_fused_gate_up

    def _k_major_weight(self) -> torch.Tensor:
        """The weight with its storage K-major (strides ``(N·K, 1, K)``), the layout Hopper's e4m3 wgmma reads, keeping its
        logical ``[E, K, N]`` shape and values: every einsum path and ``state_dict()`` see the same tensor.  The expert
        constructors relayout a W8A8 weight once; loading a checkpoint or moving the layer to another device copies into
        that layout.  Only a weight whose storage was replaced since is relaid out here, once, and never under CUDA-graph
        capture."""
        w = self.weight
        if not w.transpose(1, 2).is_contiguous():
            if w.is_cuda and torch.cuda.is_current_stream_capturing():
                raise RuntimeError("W8A8 expert weight is not K-major: run one forward before CUDA-graph capture")
            w.data = w.data.transpose(1, 2).contiguous().transpose(1, 2)
        return w

    def _expert_scales_kn(self, G: int) -> torch.Tensor:
        """fp32 ``[E, K/G, N]`` weight scales of the grouped block-scaled GEMM.  2-D blocks and E8M0 scales are expanded once
        per scale tensor (and again only after it is written); fp32 ``[E, K/G, N]`` scales are used as they are."""
        from ..ops import gemm_fp8

        s = self.scale
        key = (s.data_ptr(), s._version, s.device, s.dtype, tuple(s.shape))
        cached = self.__dict__.get("_scales_kn")
        if cached is None or cached[0] != key:
            cached = (key, gemm_fp8.expert_weight_scales_kn(s, self.weight.shape[2], self.weight.shape[1], G))
            self.__dict__["_scales_kn"] = cached
        return cached[1]

    def grouped_linear(self, x: torch.Tensor, block_to_expert: torch.Tensor, seg_first_block: torch.Tensor,
                       block_size: int) -> torch.Tensor:
        """Dropless block layout: ``x [nb·B, K]``, block i through local expert ``block_to_expert[i]`` → ``[nb·B, N]``.
        W8A8 layers quantise ``x`` per token and K-block and run the grouped block-scaled FP8 GEMM (two launches, no
        de-quantised weight); weight-only layers de-quantise their experts to ``x``'s dtype once and run the grouped GEMM."""
        from ..ops import gemm

        G = self._blockscaled_group()
        if G:
            from ..ops import gemm_fp8

            xq, xs = gemm_fp8.quantize_groups(x, G, "absmax", None if self.clamp_bound == float("inf") else self.clamp_bound)
            return gemm_fp8.grouped_blockscaled_linear(xq, xs, self._k_major_weight(), self._expert_scales_kn(G),
                                                       block_to_expert, block_size, G, out_dtype=x.dtype)
        w = self._dequantized_weight(self.weight, self.scale, x.dtype)
        return gemm.grouped_matmul(x, w, block_to_expert, seg_first_block, block_size)

    def _expert_bias(self, y: torch.Tensor, expert_indices: Optional[torch.Tensor], scale: float = 1.0) -> torch.Tensor:
        if self.bias is None:
            return y
        b = self.bias if expert_indices is None else self.bias[expert_indices]
        b = b.reshape(b.shape[0], *([1] * (y.dim() - 2)), b.shape[1])
        return y + (b * scale).to(y.dtype)


class QuantizedExpertFusedColumnParallel(QuantizedColumnParallel, _QuantizedExpertMixin):
    """Quantised ``[E_local, in, out/tp]`` expert weights (reference :1013-1213)."""

    def __init__(self, num_experts: int, input_size: int, output_size: int, bias: bool = False,
                 quantization_type: Union[QuantizationType, str] = "per_tensor_symmetric", dtype: torch.dtype = torch.float32,
                 quantized_dtype: Union[QuantizedDtype, torch.dtype] = QuantizedDtype.INT8,
                 device: Optional[torch.device] = None, stride: int = 1, keep_master_weight: bool = False,
                 quantization_per_channel_axis: Optional[int] = None, tensor_model_parallel_group=None,
                 block_axis: Optional[List[int]] = None, block_size: Optional[List[int]] = None,
                 scale_dtype: Union[torch.dtype, ScaleDtype] = torch.float32, expert_model_parallel_group=None,
                 is_prefill: bool = True, rank_ordering: Optional[Sequence[int]] = None, is_fused_gate_up: bool = False,
                 activation_quantization_type: Optional[Union[ActivationQuantizationType, str]] = None,
                 clamp_bound: float = float("inf")):
        _check_expert_activation_quantization(activation_quantization_type)
        nn.Module.__init__(self)                    # attributes needed by the config hooks before the parent ctor runs
        self._expert_setup(num_experts, expert_model_parallel_group, is_prefill, is_fused_gate_up)
        qt = QuantizationType(quantization_type)
        if qt in (QuantizationType.PER_CHANNEL_SYMMETRIC, QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC):
            quantization_per_channel_axis = 2 if quantization_per_channel_axis is None else quantization_per_channel_axis
            assert quantization_per_channel_axis == 2, "Only per_channel_axis=2 (output features) is supported"
        saved = dict(self.__dict__)
        super().__init__(input_size=input_size, output_size=output_size, bias=bias, quantization_type=qt,
                         gather_output=False, dtype=dtype, quantized_dtype=quantized_dtype, device=device, stride=stride,
                         sequence_parallel_enabled=False, keep_master_weight=keep_master_weight,
                         quantization_per_channel_axis=quantization_per_channel_axis,
                         tensor_model_parallel_group=tensor_model_parallel_group, block_axis=block_axis,
                         block_size=block_size, scale_dtype=scale_dtype, rank_ordering=rank_ordering,
                         activation_quantization_type=activation_quantization_type, clamp_bound=clamp_bound)
        for k in ("num_experts", "ep", "expert_model_parallel_group", "_n_local_experts", "num_local_experts",
                  "is_prefill", "is_fused_gate_up", "local_expert_ids"):
            self.__dict__[k] = saved[k]
        self._mark_expert_parallel_weights(expert_parallel_group_size=self.ep, is_prefill=is_prefill)
        if self._blockscaled_group():
            self._k_major_weight()

    def _setup_for_weight_and_bias_config(self, bias: bool) -> None:
        self.weight_shape = (self._n_local_experts, self.input_size, self.output_size_per_partition)
        self.weight_partition_dim = 2
        self.bias_shape = (self._n_local_experts, self.output_size_per_partition) if bias else None

    def _setup_for_bias(self, bias: bool) -> None:
        self._base_setup_for_bias(bias)
        if bias:
            set_tensor_model_parallel_attributes(self.bias, True, 1, self.stride, num_partitions=self._tp)

    def forward(self, input: torch.Tensor, expert_indices: Optional[torch.Tensor] = None, *_: Any) -> torch.Tensor:  # noqa: A002
        return self._expert_bias(self._linear_experts(input, expert_indices), expert_indices)

    @classmethod
    def from_float(cls, mod, q_config: BASE_QCONFIG_DICT_TYPE = _DEFAULT_CUSTOM_QCONFIG_DICT):
        assert mod.__class__.__name__ == "ExpertFusedColumnParallelLinear", "ExpertFusedColumnParallelLinear expected"
        new_mod = cls(
            num_experts=mod.num_experts, input_size=mod.input_size, output_size=mod.output_size, bias=mod.bias is not None,
            quantization_type=q_config["quantization_type"], quantized_dtype=q_config["quantized_dtype"], dtype=mod.dtype,
            device=mod.weight.device, stride=mod.stride, keep_master_weight=mod.keep_master_weight,
            quantization_per_channel_axis=q_config.get("quantization_per_channel_axis"),
            tensor_model_parallel_group=mod.tensor_parallel_group, expert_model_parallel_group=mod.expert_model_parallel_group,
            is_prefill=mod.is_prefill, block_axis=q_config.get("block_axis"), block_size=q_config.get("block_size"),
            scale_dtype=q_config.get("scale_dtype", torch.float32), is_fused_gate_up=mod.is_fused_gate_up,
            activation_quantization_type=_expert_activation_quantization(q_config),
            clamp_bound=q_config.get("clamp_bound", float("inf")))
        new_mod._maybe_quantize_from(mod)
        return cls._apply_post_quantization_hook(mod, new_mod)


class QuantizedExpertFusedRowParallel(QuantizedRowParallel, _QuantizedExpertMixin):
    """Quantised ``[E_local, in/tp, out]`` expert weights (reference :1215-1414)."""

    def __init__(self, num_experts: int, input_size: int, output_size: int, reduce_output: bool = False, bias: bool = False,
                 quantization_type: Union[QuantizationType, str] = "per_tensor_symmetric", dtype: torch.dtype = torch.float32,
                 quantized_dtype: Union[QuantizedDtype, torch.dtype] = QuantizedDtype.INT8,
                 device: Optional[torch.device] = None, stride: int = 1, keep_master_weight: bool = False,
                 quantization_per_channel_axis: Optional[int] = None, tensor_model_parallel_group=None,
                 block_axis: Optional[List[int]] = None, block_size: Optional[List[int]] = None,
                 scale_dtype: Union[torch.dtype, ScaleDtype] = torch.float32, expert_model_parallel_group=None,
                 is_prefill: bool = True, rank_ordering: Optional[Sequence[int]] = None, is_fused_gate_up: bool = False,
                 activation_quantization_type: Optional[Union[ActivationQuantizationType, str]] = None,
                 clamp_bound: float = float("inf")):
        _check_expert_activation_quantization(activation_quantization_type)
        nn.Module.__init__(self)
        self._expert_setup(num_experts, expert_model_parallel_group, is_prefill, is_fused_gate_up)
        qt = QuantizationType(quantization_type)
        if qt in (QuantizationType.PER_CHANNEL_SYMMETRIC, QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC):
            quantization_per_channel_axis = 2 if quantization_per_channel_axis is None else quantization_per_channel_axis
            assert quantization_per_channel_axis == 2, "Only per_channel_axis=2 (output features) is supported"
        saved = dict(self.__dict__)
        super().__init__(input_size=input_size, output_size=output_size, bias=bias, quantization_type=qt,
                         input_is_parallel=True, dtype=dtype, quantized_dtype=quantized_dtype, device=device, stride=stride,
                         sequence_parallel_enabled=False, keep_master_weight=keep_master_weight,
                         quantization_per_channel_axis=quantization_per_channel_axis, reduce_output=reduce_output,
                         tensor_model_parallel_group=tensor_model_parallel_group, block_axis=block_axis,
                         block_size=block_size, scale_dtype=scale_dtype, rank_ordering=rank_ordering,
                         activation_quantization_type=activation_quantization_type, clamp_bound=clamp_bound)
        for k in ("num_experts", "ep", "expert_model_parallel_group", "_n_local_experts", "num_local_experts",
                  "is_prefill", "is_fused_gate_up", "local_expert_ids"):
            self.__dict__[k] = saved[k]
        self._mark_expert_parallel_weights(expert_parallel_group_size=self.ep, is_prefill=is_prefill)
        if self._blockscaled_group():
            self._k_major_weight()

    def _setup_for_weight_and_bias_config(self, bias: bool) -> None:
        self.weight_shape = (self._n_local_experts, self.input_size_per_partition, self.output_size)
        self.weight_partition_dim = 1
        self.bias_shape = (self._n_local_experts, self.output_size) if bias else None

    def forward(self, input_: torch.Tensor, expert_indices: Optional[torch.Tensor] = None, *_: Any) -> torch.Tensor:
        y = self._linear_experts(input_, expert_indices)
        if self.reduce_output:
            y = mappings.reduce_from_tensor_model_parallel_region(y, self.tensor_parallel_group)
        return self._expert_bias(y, expert_indices, 1.0 if self.reduce_output else 1.0 / self._tp)

    @classmethod
    def from_float(cls, mod, q_config: BASE_QCONFIG_DICT_TYPE = _DEFAULT_CUSTOM_QCONFIG_DICT):
        assert mod.__class__.__name__ == "ExpertFusedRowParallelLinear", "ExpertFusedRowParallelLinear expected"
        new_mod = cls(
            num_experts=mod.num_experts, input_size=mod.input_size, output_size=mod.output_size,
            reduce_output=mod.reduce_output, bias=mod.bias is not None, quantization_type=q_config["quantization_type"],
            dtype=mod.dtype, quantized_dtype=q_config["quantized_dtype"], device=mod.weight.device, stride=mod.stride,
            keep_master_weight=mod.keep_master_weight,
            quantization_per_channel_axis=q_config.get("quantization_per_channel_axis"),
            tensor_model_parallel_group=mod.tensor_parallel_group, expert_model_parallel_group=mod.expert_model_parallel_group,
            is_prefill=mod.is_prefill, block_axis=q_config.get("block_axis"), block_size=q_config.get("block_size"),
            scale_dtype=q_config.get("scale_dtype", torch.float32), is_fused_gate_up=mod.is_fused_gate_up,
            activation_quantization_type=_expert_activation_quantization(q_config),
            clamp_bound=q_config.get("clamp_bound", float("inf")))
        new_mod._maybe_quantize_from(mod)
        return cls._apply_post_quantization_hook(mod, new_mod)
