"""Packing / unpacking of microscaling (MX) weights (role of reference
``quantization/microscaling/transform_weights.py:27-416``).

Checkpoint formats handled:

* ``fp4_x2`` — two e2m1 codes per ``uint8`` (low nibble first), blocks of 16 bytes + one E8M0 scale: the layout MXFP4
  checkpoints ship in (gpt-oss style ``[..., G, 16]`` blocks, ``[..., G]`` scales);
* ``fp4_x4`` — four codes per 16-bit word (``QuantizedDtype.F4E2M1FN_X4``), ``[..., G, 8]``;
* ``fp8_x4`` — four e4m3 / e5m2 bytes per ``uint32`` (``QuantizedDtype.F8E4M3FN_X4``), ``[..., G, 8]``.

All of them are little-endian views of the same byte stream, so every routine here is a ``view`` plus a 16-entry table
look-up and an ``ldexp`` — no element loops.  The tcgen05 ``kind::mxf4`` / ``mxf8f6f4`` operand layout is exactly the
``x2`` / byte stream with K contiguous, so these tensors can be handed to a block-scaled GEMM as they are; the scale
factors need the 128×4 tile interleave from ``experimental.quantization.microscaling.swizzle``.
"""
from __future__ import annotations

from typing import Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F

from ..quantization_config import QuantizedDtype

FP4_VALUES = [
    +0.0, +0.5, +1.0, +1.5, +2.0, +3.0, +4.0, +6.0,
    -0.0, -0.5, -1.0, -1.5, -2.0, -3.0, -4.0, -6.0,
]
E8M0_BIAS = 127
MX_BLOCK = 32


def _lut(dtype: torch.dtype, device) -> torch.Tensor:
    return torch.tensor(FP4_VALUES, dtype=dtype, device=device)


def _apply_scale(vals: torch.Tensor, scales_e8m0: torch.Tensor) -> torch.Tensor:
    """``vals [..., G, B] · 2^(scale-127)`` with the scale broadcast over the block."""
    exp = scales_e8m0.to(torch.int32) - E8M0_BIAS
    return torch.ldexp(vals, exp.unsqueeze(-1))


def split_byte_4bit_tensor(tensor: torch.Tensor, **_unused) -> torch.Tensor:
    """``[..., P]`` bytes holding two 4-bit codes each → ``[..., 2P]`` uint8 codes (low nibble first)."""
    b = tensor.contiguous().view(torch.uint8)
    return torch.stack((b & 0x0F, b >> 4), dim=-1).reshape(*b.shape[:-1], b.shape[-1] * 2)


def pack_byte_4bit_tensor(tensor: torch.Tensor, **_unused) -> torch.Tensor:
    """Inverse of :func:`split_byte_4bit_tensor`."""
    assert tensor.dtype == torch.uint8, f"{tensor.dtype=} must be uint8"
    assert tensor.shape[-1] >= 2 and tensor.shape[-1] % 2 == 0, f"last dim {tensor.shape[-1]} must be even"
    pairs = tensor.reshape(*tensor.shape[:-1], -1, 2)
    return (pairs[..., 0] | (pairs[..., 1] << 4)).contiguous()


def apply_lut_byte_4bit_tensor(blocks: torch.Tensor, *, dtype: torch.dtype = torch.float32, **_unused) -> torch.Tensor:
    """uint8 e2m1 codes ``[..., G, B]`` → values ``[..., G·B]`` (no scale)."""
    out = _lut(dtype, blocks.device)[blocks.long()]
    return out.reshape(*blocks.shape[:-2], blocks.shape[-2] * blocks.shape[-1])


def dequant_byte_4bit_tensor(blocks: torch.Tensor, scales: torch.Tensor, **_unused) -> torch.Tensor:
    """Unpacked codes ``[..., G, B]`` + E8M0 scales ``[..., G]`` → bf16 ``[..., G·B]``."""
    vals = _apply_scale(_lut(torch.float32, blocks.device)[blocks.long()], scales)
    return vals.to(torch.bfloat16).reshape(*blocks.shape[:-2], blocks.shape[-2] * blocks.shape[-1])


def get_mxfp4_tensor(blocks: torch.Tensor, scales: torch.Tensor, *, dtype: torch.dtype = torch.bfloat16, **_unused
                     ) -> torch.Tensor:
    """MXFP4 ``fp4_x2`` blocks ``[..., G, 16]`` + scales ``[..., G]`` → ``[..., G·32]`` in ``dtype``."""
    assert blocks.shape[:-1] == scales.shape, f"{blocks.shape=} does not match {scales.shape=}"
    codes = split_byte_4bit_tensor(blocks)                                    # [..., G, 32]
    vals = _apply_scale(_lut(torch.float32, blocks.device)[codes.long()], scales)
    return vals.to(dtype).reshape(*blocks.shape[:-2], -1)


def _quad(out: torch.Tensor, prefix, G: int, B: int, output_quad_row: bool) -> torch.Tensor:
    # ``quad row`` = the four values of one packed word kept as a trailing dim (the reference's partition layout)
    return out.reshape(*prefix, G * B, 4) if output_quad_row else out.reshape(*prefix, G * B * 4)


def get_mxfp4_tensor_from_uint16(blocks: torch.Tensor, scales: torch.Tensor, *, dtype: torch.dtype = torch.bfloat16,
                                 output_quad_row: bool = False, **_unused) -> torch.Tensor:
    """``fp4_x4`` words ``[..., G, 8]`` + scales ``[..., G]`` → ``[..., G·32]`` (or ``[..., G·8, 4]``)."""
    assert blocks.shape[:-1] == scales.shape, f"{blocks.shape=} does not match {scales.shape=}"
    *prefix, G, B = blocks.shape
    codes = split_byte_4bit_tensor(blocks.contiguous().view(torch.uint8))     # little-endian: byte0 = codes 0,1
    vals = _apply_scale(_lut(torch.float32, blocks.device)[codes.long()], scales).to(dtype)
    return _quad(vals, prefix, G, B, output_quad_row)


def get_mxfp8_tensor_from_uint32(blocks: torch.Tensor, scales: torch.Tensor, *, dtype: torch.dtype = torch.bfloat16,
                                 fp8_dtype: torch.dtype = torch.float8_e4m3fn, output_quad_row: bool = False,
                                 replace_nan_with_zeros: bool = False, **_unused) -> torch.Tensor:
    """``fp8_x4`` words ``[..., G, 8]`` + scales ``[..., G]`` → ``[..., G·32]`` (or ``[..., G·8, 4]``)."""
    assert blocks.shape[:-1] == scales.shape, f"{blocks.shape=} does not match {scales.shape=}"
    *prefix, G, B = blocks.shape
    vals = blocks.contiguous().view(torch.uint8).view(fp8_dtype).float()      # [..., G, 32]
    vals = _apply_scale(vals, scales)
    if replace_nan_with_zeros:
        vals = torch.nan_to_num(vals, nan=0.0)
    return _quad(vals.to(dtype), prefix, G, B, output_quad_row)


def pack_fp4_x4_uint16(X: Union[torch.Tensor, np.ndarray]):
    """Re-view ``fp4_x2`` bytes as ``fp4_x4`` 16-bit words (last dim halves)."""
    x = X      # reference parameter names in the signature
    if isinstance(x, torch.Tensor):
        assert x.dtype == torch.uint8, f"expected uint8, got {x.dtype}"
        return x.contiguous().view(QuantizedDtype.F4E2M1FN_X4.value)
    if isinstance(x, np.ndarray):
        assert x.dtype == np.uint8
        return np.ascontiguousarray(x).view(np.uint16)
    raise ValueError("Unsupported input dtype!")


def quantize_to_mxfp4(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """float ``[..., K]`` → (``fp4_x2`` blocks ``[..., K/32, 16]``, E8M0 scales ``[..., K/32]``).  The producer-side
    counterpart of :func:`get_mxfp4_tensor` (the reference only ships the consumer side; used to build test
    checkpoints and to quantise bf16 expert weights offline)."""
    assert w.shape[-1] % MX_BLOCK == 0
    wb = w.float().reshape(*w.shape[:-1], -1, MX_BLOCK)
    amax = wb.abs().amax(-1).clamp(min=2.0 ** -120)
    exp = torch.floor(torch.log2(amax)) - 2                                   # e2m1 max = 1.5·2^2
    scaled = torch.ldexp(wb, -exp.to(torch.int32).unsqueeze(-1)).clamp(-6.0, 6.0)
    mags = torch.tensor(FP4_VALUES[:8], device=w.device)
    idx = (scaled.abs().unsqueeze(-1) - mags).abs().argmin(-1)
    codes = (idx | ((scaled < 0).long() << 3)).to(torch.uint8)
    return pack_byte_4bit_tensor(codes), (exp + E8M0_BIAS).clamp(0, 254).to(torch.uint8)


def split_gate_up(W_gate_up, scale_gate_up, bias_gate_up):
    """De-interleave fused gate/up tensors whose ``2I`` axis (dim 1) alternates gate, up rows
    (``W [E, 2I, H/32, 16]``, ``scale [E, 2I, H/32]``, ``bias [E, 2I]``)."""
    w_gate_up = W_gate_up      # reference parameter names in the signature
    parts = (w_gate_up[:, 0::2], scale_gate_up[:, 0::2], bias_gate_up[:, 0::2],
             w_gate_up[:, 1::2], scale_gate_up[:, 1::2], bias_gate_up[:, 1::2])
    if isinstance(w_gate_up, torch.Tensor):
        return tuple(p.contiguous() for p in parts)
    return parts


def _pad_tensor(x, pad_to, pad_value=0):
    """Right-pad every dim ``i`` of ``x`` to ``pad_to[i]`` with a constant."""
    if isinstance(x, torch.Tensor):
        spec = []
        for i in reversed(range(x.dim())):
            spec += [0, max(0, pad_to[i] - x.shape[i])]
        return F.pad(x, tuple(spec), "constant", pad_value)
    if isinstance(x, np.ndarray):
        return np.pad(x, [(0, max(0, pad_to[i] - x.shape[i])) for i in range(x.ndim)], mode="constant",
                      constant_values=pad_value)
    raise ValueError("Invalid input type!")


def reshape_pad_proj(W, scale, bias, pad_multiple: int = 512):
    """Flatten ``W [E, R, C/32, 8]`` (x4-packed) to ``[E, R, C/4]`` and right-pad rows / columns up to a multiple of
    ``pad_multiple`` elements (scales padded with the E8M0 bias, i.e. 2⁰; weights / bias with zero).

    The reference hard-codes the gpt-oss-120b geometry (128 experts, 2880 → 3072); here the target is derived from the
    tensor so that any expert geometry can be aligned for the 128-row GEMM tiles.
    """
    w = W      # reference parameter names in the signature
    E, R = w.shape[0], w.shape[1]
    C = w.shape[2] * w.shape[3] * 4
    up = lambda n: -(-n // pad_multiple) * pad_multiple  # noqa: E731
    w2 = w.reshape((E, R, C // 4))
    return (_pad_tensor(w2, (E, up(R), up(C) // 4)), _pad_tensor(scale, (E, up(R), up(C) // MX_BLOCK), E8M0_BIAS),
            _pad_tensor(bias, (E, up(R))))
