"""MoE enums / defaults shared by the expert implementations (reference ``modules/moe/model_utils.py:11-119``)."""
from __future__ import annotations

from enum import Enum
from typing import Any, Callable, Dict

import torch
import torch.nn.functional as F

from ...utils.logger import get_logger

logger = get_logger()

ACT2FN: Dict[str, Callable] = {
    "gelu": F.gelu,
    "leaky_relu": F.leaky_relu,
    "relu": F.relu,
    "sigmoid": torch.sigmoid,
    "silu": F.silu,
    "swish": F.silu,
    "tanh": torch.tanh,
    "gelu_new": lambda x: F.gelu(x, approximate="tanh"),
    "gelu_pytorch_tanh": lambda x: F.gelu(x, approximate="tanh"),
    "gelu_tanh_approx": lambda x: F.gelu(x, approximate="tanh"),
    "quick_gelu": lambda x: x * torch.sigmoid(1.702 * x),
}


class GLUType(Enum):
    """``glu``: act(gate)·up.  ``swiglu``: gate·σ(α·gate)·(up + β) with clamps (gpt-oss)."""

    GLU = "glu"
    SWIGLU = "swiglu"

    @classmethod
    def validate(cls, glu_type) -> "GLUType":
        if isinstance(glu_type, cls):
            return glu_type
        if glu_type is None:
            logger.warning("glu_type is None, default to basic GLU")
            return cls.GLU
        try:
            return cls(glu_type)
        except ValueError:
            raise ValueError(f"glu_type={glu_type} not supported, must be one of {[e.value for e in cls]}") from None


class ACTFunc(Enum):
    """Activation id / name pairs; the ids are what the grouped-GEMM epilogue (``csrc/gemm_sm90.cu`` MODE 3) switches
    on when the activation is fused — same numbering as the reference's kernel enum so configs port unchanged."""

    def __new__(cls, ident: int, name: str):
        obj = object.__new__(cls)
        obj._value_ = ident
        obj.id, obj.name_str = ident, name
        return obj

    SILU = (0, "silu")
    GELU = (1, "gelu")
    GELU_TANH_APPROX = (2, "gelu_tanh_approx")
    SIGMOID = (3, "sigmoid")
    RELU = (4, "relu")
    TANH = (5, "tanh")
    LEAKY_RELU = (6, "leaky_relu")

    @classmethod
    def validate(cls, act_func) -> "ACTFunc":
        if isinstance(act_func, cls):
            return act_func
        if act_func is None:
            logger.warning("act_func is None, default to SIGMOID")
            return cls.SIGMOID
        if isinstance(act_func, str):
            for member in cls:
                if member.name_str == act_func:
                    return member
            raise ValueError(f"act_func={act_func} not supported, must be one of: {[e.name_str for e in cls]}")
        raise ValueError(f"Invalid type for act_func: {type(act_func)}")

    @property
    def fn(self) -> Callable:
        return ACT2FN[self.name_str]


def get_kernel_activation_func_id(act_fn: ACTFunc, glu_type: GLUType) -> int:
    """Activation id for the fused-epilogue path; only the two combinations that have a fused epilogue are accepted
    (SiLU-GLU and sigmoid-SwiGLU), everything else runs the activation as its own kernel."""
    if glu_type == GLUType.GLU and act_fn == ACTFunc.SILU:
        return ACTFunc.SILU.value
    if glu_type == GLUType.SWIGLU and act_fn == ACTFunc.SIGMOID:
        return ACTFunc.SIGMOID.value
    raise ValueError(f"Unsupported ACTFunc and GLUType combination in the fused kernel flow: {act_fn}, {glu_type}.")


DEFAULT_SELECTIVE_LOADING_THRESHOLD = 1.0     # decode: gather only the selected experts when T·k/E is below this
DEFAULT_BLOCK_SIZE = 512
DEFAULT_SKIP_MODE = (False, False)
DEFAULT_LNC_SIZE = 1                          # a H100 GPU is one logical core (the two dies share L2/HBM coherently)
DEFAULT_PADDING_VALUE = -1
DEFAULT_HIDDEN_ACT_SCALING_FACTOR = 1.702


def create_spmd_ranks(model_state_dict: Dict[str, Any], prefix: str, world_size: int) -> None:
    """Add the ``spmd_rank.rank`` entry (``arange(world)``; the sharder hands rank r its own id) to a full checkpoint."""
    model_state_dict[f"{prefix}spmd_rank.rank"] = torch.arange(0, world_size, dtype=torch.int32)
