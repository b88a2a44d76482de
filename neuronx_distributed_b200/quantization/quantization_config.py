"""Quantization configuration (reference ``quantization/quantization_config.py:10-256``).

Same enums / config dictionaries as the reference so that model code written against it ports unchanged; the dtype table
is the OCP / NVIDIA one: e4m3 saturates at 448 (``float8_e4m3fn``, the e4m3 wgmma operand format — the
reference clamps to the Trainium e4m3 range of 240), microscaling blocks are 32 elements along K with UE8M0 scales
(the OCP MX block-scale format).
"""
from __future__ import annotations

import enum
import os
from typing import List, Optional, Tuple, TypedDict, Union

import torch


class MyEnumMeta(enum.EnumMeta):
    """``value in EnumClass`` answers for raw values as well as members (reference :10-17)."""

    def __contains__(cls, item) -> bool:
        if isinstance(item, cls):
            return True
        try:
            cls(item)
        except (ValueError, TypeError):
            return False
        return True


class DtypeBound(enum.Enum):
    """(max, min) representable magnitude per storage dtype (reference :20-65)."""

    INT8_MAX = 127
    INT8_MIN = -128
    F8E4M3FN_MAX = torch.finfo(torch.float8_e4m3fn).max          # 448
    F8E4M3FN_MIN = torch.finfo(torch.float8_e4m3fn).min
    F8E4M3_MAX = torch.finfo(torch.float8_e4m3fn).max            # alias: Trainium's e4m3 tops out at 240, Blackwell has only "fn"
    F8E4M3_MIN = torch.finfo(torch.float8_e4m3fn).min
    F8E5M2_MAX = torch.finfo(torch.float8_e5m2).max              # 57344
    F8E5M2_MIN = torch.finfo(torch.float8_e5m2).min
    F4E2M1FN_X2_MAX = 6.0
    F4E2M1FN_X2_MIN = -6.0
    F8E8M0_MAX = 2.0 ** (255.0 - 127.0)
    F8E8M0_MIN = 2.0 ** (-127.0)
    BFLOAT16_MAX = torch.finfo(torch.bfloat16).max
    BFLOAT16_MIN = torch.finfo(torch.bfloat16).min
    FLOAT16_MAX = torch.finfo(torch.float16).max
    FLOAT16_MIN = torch.finfo(torch.float16).min

    @staticmethod
    def from_torch_dtype(dtype: torch.dtype) -> Tuple[float, float]:
        table = {
            torch.float8_e4m3fn: (DtypeBound.F8E4M3FN_MAX, DtypeBound.F8E4M3FN_MIN),
            torch.float8_e5m2: (DtypeBound.F8E5M2_MAX, DtypeBound.F8E5M2_MIN),
            torch.int8: (DtypeBound.INT8_MAX, DtypeBound.INT8_MIN),
            torch.bfloat16: (DtypeBound.BFLOAT16_MAX, DtypeBound.BFLOAT16_MIN),
            torch.float16: (DtypeBound.FLOAT16_MAX, DtypeBound.FLOAT16_MIN),
        }
        if dtype not in table:
            raise ValueError(f"Unsupported dtype: {dtype}")
        hi, lo = table[dtype]
        return hi.value, lo.value


class QuantizationType(enum.Enum, metaclass=MyEnumMeta):
    PER_TENSOR_SYMMETRIC = "per_tensor_symmetric"
    PER_CHANNEL_SYMMETRIC = "per_channel_symmetric"
    PER_KEY_SYMMETRIC = "per_key_symmetric"
    BLOCKWISE_SYMMETRIC = "blockwise_symmetric"
    EXPERT_WISE_PER_CHANNEL_SYMMETRIC = "expert_wise_per_channel_symmetric"


class ActivationQuantizationType(enum.Enum, metaclass=MyEnumMeta):
    DYNAMIC = "dynamic"      # absmax scale per token computed on the fly
    STATIC = "static"        # calibrated ``input_scale`` loaded from the checkpoint
    NONE = None

    @classmethod
    def _missing_(cls, value):
        if value in ("none", "None"):
            return cls.NONE
        return None


def get_float4x4_torch_dtype() -> torch.dtype:
    """Storage dtype of four packed e2m1 values.  ``NEURON_FLOAT4X4_IS_FLOAT16`` (reference :93-103) is honoured for
    checkpoints that were written with the float16 carrier."""
    return torch.float16 if int(os.environ.get("NEURON_FLOAT4X4_IS_FLOAT16", "0")) > 0 else torch.uint16


class QuantizedDtype(enum.Enum, metaclass=MyEnumMeta):
    INT8 = torch.int8
    F8E4M3 = torch.float8_e4m3fn
    F8E4M3FN = torch.float8_e4m3fn        # alias
    F8E5M2 = torch.float8_e5m2
    F4E2M1FN_X4 = get_float4x4_torch_dtype()   # 4 × e2m1 per 16-bit word
    F8E4M3FN_X4 = torch.uint32                 # 4 × e4m3 per 32-bit word
    F8E5M2_X4 = torch.uint32                   # alias of the carrier (the element format is a layer attribute)

    @classmethod
    def has_dtype(cls, dtype_string: str) -> None:
        assert dtype_string.upper() in cls.__members__, f"{dtype_string} is not a valid QuantizedDtype."

    @classmethod
    def get_dtype(cls, dtype_string) -> torch.dtype:
        """torch dtype for a name (``"f8e4m3"``), member or torch dtype."""
        if isinstance(dtype_string, cls):
            return dtype_string.value
        if isinstance(dtype_string, torch.dtype):
            return cls(dtype_string).value
        name = {"MXFP4": "F4E2M1FN_X4", "MXFP8": "F8E4M3FN_X4"}.get(str(dtype_string).upper(), str(dtype_string).upper())
        cls.has_dtype(name)
        return cls[name].value

    def is_float(self) -> bool:
        return self != QuantizedDtype.INT8

    def get_packed_count(self) -> int:
        return 4 if self in (QuantizedDtype.F4E2M1FN_X4, QuantizedDtype.F8E4M3FN_X4, QuantizedDtype.F8E5M2_X4) else 1

    def storage_dtype(self) -> torch.dtype:
        return self.value


class ScaleDtype(enum.Enum, metaclass=MyEnumMeta):
    F32 = torch.float32
    F8E8M0 = torch.uint8          # power-of-two scale stored as a biased exponent (OCP microscaling)
    E8M0 = torch.uint8            # alias

    def get_default_scale(self):
        return 127 if self == ScaleDtype.F8E8M0 else 1.0

    @classmethod
    def has_dtype(cls, dtype_string: str) -> None:
        assert dtype_string.upper() in cls.__members__, f"{dtype_string} is not a valid ScaleDtype."

    @classmethod
    def get_dtype(cls, dtype_string) -> torch.dtype:
        if isinstance(dtype_string, cls):
            return dtype_string.value
        if isinstance(dtype_string, torch.dtype):
            return cls(dtype_string).value
        name = {"E8M0": "F8E8M0"}.get(str(dtype_string).upper(), str(dtype_string).upper())
        cls.has_dtype(name)
        return cls[name].value


class KVQuantizationConfig:
    """KV-cache quantisation (reference :74-84) + the static-scale options of ``inference.kv_cache.KVCacheManager``."""

    def __init__(self, **kwargs):
        self.k_quant_method = QuantizationType(kwargs.pop("k_quant_method", QuantizationType.PER_TENSOR_SYMMETRIC))
        self.v_quant_method = QuantizationType(kwargs.pop("v_quant_method", QuantizationType.PER_TENSOR_SYMMETRIC))
        self.quant_dtype: torch.dtype = kwargs.pop("quant_dtype", torch.float8_e4m3fn)
        self.dequant_dtype: torch.dtype = kwargs.pop("dequant_dtype", torch.bfloat16)
        self.scale: float = float(kwargs.pop("scale", 1.0))
        self.per_key: bool = bool(kwargs.pop("per_key", self.k_quant_method == QuantizationType.PER_KEY_SYMMETRIC))
        self.direct_cast: bool = kwargs.pop("direct_cast", self.scale == 1.0 and not self.per_key)
        if kwargs:
            raise TypeError(f"unexpected KVQuantizationConfig arguments: {sorted(kwargs)}")
        if self.direct_cast:
            assert self.k_quant_method == QuantizationType.PER_TENSOR_SYMMETRIC and \
                self.v_quant_method == QuantizationType.PER_TENSOR_SYMMETRIC, \
                "When using direct cast both K and V quantization strategies must be PER_TENSOR_SYMMETRIC"


class BASE_QCONFIG_DICT_TYPE(TypedDict, total=False):
    quantization_type: QuantizationType
    quantized_dtype: QuantizedDtype
    activation_quantization_type: ActivationQuantizationType
    clamp_bound: float
    quantization_per_channel_axis: Optional[int]
    block_axis: Optional[List[int]]
    block_size: Optional[List[int]]
    scale_dtype: ScaleDtype


class PER_CHANNEL_QCONFIG_DICT_TYPE(BASE_QCONFIG_DICT_TYPE, total=False):
    pass


class EXPERT_WISE_PER_CHANNEL_QCONFIG_DICT_TYPE(BASE_QCONFIG_DICT_TYPE, total=False):
    pass


class BLOCKWISE_QCONFIG_DICT_TYPE(BASE_QCONFIG_DICT_TYPE, total=False):
    pass


_DEFAULT_CUSTOM_QCONFIG_DICT: BASE_QCONFIG_DICT_TYPE = {
    "quantization_type": QuantizationType.PER_TENSOR_SYMMETRIC,
    "quantized_dtype": QuantizedDtype.INT8,
    "activation_quantization_type": ActivationQuantizationType.NONE,
    "clamp_bound": float("inf"),
}

_DEFAULT_PER_CHANNEL_QCONFIG_DICT: PER_CHANNEL_QCONFIG_DICT_TYPE = {
    "quantization_type": QuantizationType.PER_CHANNEL_SYMMETRIC,
    "quantized_dtype": QuantizedDtype.INT8,
    "quantization_per_channel_axis": None,       # every layer picks its own output-feature axis
    "activation_quantization_type": ActivationQuantizationType.NONE,
    "clamp_bound": float("inf"),
}

_DEFAULT_BLOCKWISE_QCONFIG_DICT: BLOCKWISE_QCONFIG_DICT_TYPE = {
    "quantization_type": QuantizationType.BLOCKWISE_SYMMETRIC,
    "quantized_dtype": QuantizedDtype.F8E4M3,
    "block_axis": [1],
    "block_size": [128],
    "scale_dtype": ScaleDtype.F32,
    "activation_quantization_type": ActivationQuantizationType.NONE,
    "clamp_bound": float("inf"),
}

_DEFAULT_EXPERT_WISE_PER_CHANNEL_QCONFIG_DICT: EXPERT_WISE_PER_CHANNEL_QCONFIG_DICT_TYPE = {
    "quantization_type": QuantizationType.EXPERT_WISE_PER_CHANNEL_SYMMETRIC,
    "quantized_dtype": QuantizedDtype.F8E4M3,
    "quantization_per_channel_axis": None,
    "activation_quantization_type": ActivationQuantizationType.NONE,
    "clamp_bound": float("inf"),
}


def validate_block_axis_size(block_axis: Optional[List[int]], block_size: Optional[List[int]]) -> Tuple[List[int], List[int]]:
    assert block_size is not None and block_axis is not None, \
        "block_axis and block_size must be specified for blockwise quantization"
    assert len(block_size) == len(block_axis), "block_axis and block_size list arguments must have the same length"
    return list(block_axis), list(block_size)


def get_default_custom_qconfig_dict() -> BASE_QCONFIG_DICT_TYPE:
    return dict(_DEFAULT_CUSTOM_QCONFIG_DICT)  # type: ignore[return-value]


get_default_per_tensor_custom_qconfig_dict = get_default_custom_qconfig_dict


def get_default_per_channel_custom_qconfig_dict() -> PER_CHANNEL_QCONFIG_DICT_TYPE:
    return dict(_DEFAULT_PER_CHANNEL_QCONFIG_DICT)  # type: ignore[return-value]


def get_default_blockwise_custom_qconfig_dict() -> BLOCKWISE_QCONFIG_DICT_TYPE:
    d = dict(_DEFAULT_BLOCKWISE_QCONFIG_DICT)
    d["block_axis"], d["block_size"] = list(d["block_axis"]), list(d["block_size"])
    return d  # type: ignore[return-value]


def get_default_expert_wise_per_channel_custom_qconfig_dict() -> EXPERT_WISE_PER_CHANNEL_QCONFIG_DICT_TYPE:
    return dict(_DEFAULT_EXPERT_WISE_PER_CHANNEL_QCONFIG_DICT)  # type: ignore[return-value]


def is_ocp_mx_quantized(q_type: QuantizationType, q_dtype: Union[QuantizedDtype, torch.dtype],
                        scale_dtype: Union[ScaleDtype, torch.dtype]) -> bool:
    """OCP microscaling = blockwise + x4-packed fp4/fp8 elements + E8M0 scales (reference :239-256)."""
    try:
        qd, sd = QuantizedDtype(q_dtype), ScaleDtype(scale_dtype)
    except ValueError:
        return False
    return (QuantizationType(q_type) == QuantizationType.BLOCKWISE_SYMMETRIC
            and qd in (QuantizedDtype.F4E2M1FN_X4, QuantizedDtype.F8E4M3FN_X4, QuantizedDtype.F8E5M2_X4)
            and sd == ScaleDtype.F8E8M0)
