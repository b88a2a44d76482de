"""PyTorch reference for OCP microscaling formats (role of reference
``experimental/quantization/microscaling/mx_torch.py:65-253``): MXFP8 (e4m3) and MXFP4 (e2m1) with one shared
power-of-two E8M0 scale per block of 32 along the last dim; packing 4 values per word
(mxfp4 → uint16, mxfp8 → uint32) as in ``quantization_config.QuantizedDtype``."""
from __future__ import annotations

from typing import Tuple

import torch

BLOCK = 32
_FP4_VALUES = torch.tensor([0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0])
_FP4_MAX_EXP = 2      # 6 = 1.5·2^2
_FP8_MAX_EXP = 8      # 448 = 1.75·2^8


def float_to_e8m0(scale: torch.Tensor) -> torch.Tensor:
    return (torch.log2(scale.float()).round() + 127).clamp(0, 254).to(torch.uint8)


def e8m0_to_float(e: torch.Tensor) -> torch.Tensor:
    return torch.pow(2.0, e.float() - 127.0)


def _block_scale(x: torch.Tensor, elem_max_exp: int) -> torch.Tensor:
    xb = x.float().reshape(*x.shape[:-1], -1, BLOCK)
    amax = xb.abs().amax(-1).clamp(min=2.0 ** -100)
    return torch.pow(2.0, torch.floor(torch.log2(amax)) - elem_max_exp)     # [..., nblk]


def _to_fp4_code(v: torch.Tensor) -> torch.Tensor:
    """Nearest e2m1 code (sign bit 3, magnitude index 0-7)."""
    mag = v.abs().clamp(max=6.0)
    idx = (mag.unsqueeze(-1) - _FP4_VALUES.to(v.device)).abs().argmin(-1)
    return (idx | ((v < 0).long() << 3)).to(torch.uint8)


def _from_fp4_code(c: torch.Tensor) -> torch.Tensor:
    mag = _FP4_VALUES.to(c.device)[(c & 7).long()]
    return torch.where((c & 8) != 0, -mag, mag)


def quantize_mx(x: torch.Tensor, kind: str = "mxfp8") -> Tuple[torch.Tensor, torch.Tensor]:
    """Return ``(packed, scale_e8m0)``; last dim must be a multiple of 32."""
    assert x.shape[-1] % BLOCK == 0
    scale = _block_scale(x, _FP4_MAX_EXP if kind == "mxfp4" else _FP8_MAX_EXP)
    xs = x.float() / scale.repeat_interleave(BLOCK, dim=-1)
    if kind == "mxfp4":
        codes = _to_fp4_code(xs).reshape(*x.shape[:-1], -1, 4).to(torch.int32)
        packed = (codes[..., 0] | (codes[..., 1] << 4) | (codes[..., 2] << 8) | (codes[..., 3] << 12)).to(torch.uint16)
    else:
        b = xs.clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8).reshape(*x.shape[:-1], -1, 4).to(torch.int64)
        packed = (b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16) | (b[..., 3] << 24)).to(torch.uint32)
    return packed, float_to_e8m0(scale)


def dequantize_mxfp4_packed(packed: torch.Tensor) -> torch.Tensor:
    p = packed.to(torch.int32)
    codes = torch.stack([(p >> s) & 0xF for s in (0, 4, 8, 12)], dim=-1).reshape(*packed.shape[:-1], -1)
    return _from_fp4_code(codes.to(torch.uint8))


def dequantize_mxfp8_packed(packed: torch.Tensor) -> torch.Tensor:
    p = packed.to(torch.int64)
    b = torch.stack([(p >> s) & 0xFF for s in (0, 8, 16, 24)], dim=-1).reshape(*packed.shape[:-1], -1).to(torch.uint8)
    return b.view(torch.float8_e4m3fn).float()


def mx_matmul(a: torch.Tensor, b_packed: torch.Tensor, b_scale: torch.Tensor, kind: str = "mxfp8",
              out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``a [M,K] @ dequant(b)[N,K]ᵀ`` — numerics oracle for the block-scaled tensor-core path."""
    vals = dequantize_mxfp4_packed(b_packed) if kind == "mxfp4" else dequantize_mxfp8_packed(b_packed)
    w = vals * e8m0_to_float(b_scale).repeat_interleave(BLOCK, dim=-1)
    return (a.float() @ w.t()).to(out_dtype)


# ---------------------------------------------------------------------------------------------------------------------
# Reference-named entry points (experimental/quantization/microscaling/mx_torch.py:65-253) in the Blackwell operand
# layout: BOTH operands K-major, blocks of 32 along K (the last dim), x4 packing along K.  The reference's layout
# (K on the partition axis, 8×4 "quad-row" blocks) is a Trainium SBUF artefact with no counterpart here.
# ---------------------------------------------------------------------------------------------------------------------
VALID_MX_TYPES = (torch.uint16, torch.uint32)
VALID_QMX_INPUT_TYPE = (torch.bfloat16, torch.float16, torch.float32)
VALID_QMX_OUTPUT_TYPE = torch.uint32                     # online quantisation produces fp8_x4 words


def quantize_mxfp8(in_tensor: torch.Tensor, out_x4_dtype: torch.dtype = torch.uint32,
                   fp8_dtype: torch.dtype = torch.float8_e4m3fn, use_unbiased_scale: bool = False
                   ) -> Tuple[torch.Tensor, torch.Tensor]:
    """OCP MXFP8 quantisation of ``[..., K]``: returns (``uint32 [..., K/4]``, ``uint8 E8M0 [..., K/32]``).

    Scale = 2^(floor(log2(amax)) − emax) with emax = 8 for e4m3 (15 for e5m2); ``use_unbiased_scale`` lowers emax by one
    (no element saturates, one bit less precision) like the reference's flag."""
    assert in_tensor.dtype in VALID_QMX_INPUT_TYPE, f"expected one of {VALID_QMX_INPUT_TYPE}, got {in_tensor.dtype}"
    assert out_x4_dtype == VALID_QMX_OUTPUT_TYPE, "online quantisation produces fp8_x4 (uint32) only"
    assert in_tensor.shape[-1] % BLOCK == 0
    emax = (8 if fp8_dtype == torch.float8_e4m3fn else 15) - (1 if use_unbiased_scale else 0)
    fmax = torch.finfo(fp8_dtype).max
    # IEEE exponent of the block absmax read from the bit pattern: exact floor(log2(x)), no transcendental rounding
    xb = in_tensor.float().reshape(*in_tensor.shape[:-1], -1, BLOCK)
    amax = xb.abs().amax(-1)
    exp = ((amax.view(torch.int32) >> 23) & 0xFF) - 127
    exp = torch.where(amax == 0, torch.full_like(exp, -126), exp)
    e8m0 = (exp + 127 - emax).clamp(0, 254)
    q = torch.ldexp(xb, -(e8m0 - 127).unsqueeze(-1)).clamp(-fmax, fmax).to(fp8_dtype)
    packed = q.reshape(*in_tensor.shape).contiguous().view(torch.uint8).view(torch.uint32)
    return packed, e8m0.to(torch.uint8)


def dequantize_mx_tensor(tensor: torch.Tensor, scale: torch.Tensor, dtype: torch.dtype = torch.float32,
                         input_is_transposed: bool = False, output_is_transposed: bool = False,
                         fp8_dtype: torch.dtype = torch.float8_e4m3fn) -> torch.Tensor:
    """x4-packed MX tensor (``uint16`` = fp4, ``uint32`` = fp8) ``[..., M, K/4]`` + scales ``[..., M, K/32]`` →
    ``[..., M, K]`` in ``dtype``."""
    from .transform_weights import get_mxfp4_tensor_from_uint16, get_mxfp8_tensor_from_uint32

    if input_is_transposed:
        tensor, scale = tensor.transpose(-2, -1), scale.transpose(-2, -1)
    *shape, m, k4 = tensor.shape
    blocks = tensor.reshape(*shape, m, k4 // 8, 8)
    if tensor.dtype == torch.uint16 or tensor.dtype == torch.float16:
        out = get_mxfp4_tensor_from_uint16(blocks.view(torch.uint16) if tensor.dtype != torch.uint16 else blocks, scale, dtype=dtype)
    elif tensor.dtype == torch.uint32:
        out = get_mxfp8_tensor_from_uint32(blocks, scale, dtype=dtype, fp8_dtype=fp8_dtype)
    else:
        raise ValueError(f"Unsupported dtype: {tensor.dtype}")
    return out.transpose(-2, -1) if output_is_transposed else out


def matmul_mx_single_tile(a_x4: torch.Tensor, b_x4: torch.Tensor, a_scale: torch.Tensor, b_scale: torch.Tensor,
                          output_dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """One UMMA-sized tile (M ≤ 128, N ≤ 256, K ≤ 128 elements... any multiple of 32): ``A [M,K] @ B [N,K]ᵀ`` with the
    block scales applied to the operands and fp32 accumulation — what ``tcgen05.mma…block_scale`` computes."""
    assert a_x4.dtype in VALID_MX_TYPES and b_x4.dtype in VALID_MX_TYPES
    assert a_x4.dim() == 2 and b_x4.dim() == 2
    a = dequantize_mx_tensor(a_x4, a_scale, torch.float32)
    b = dequantize_mx_tensor(b_x4, b_scale, torch.float32)
    assert a.shape[1] == b.shape[1], f"contraction dims differ: {a.shape[1]} vs {b.shape[1]}"
    return (a @ b.t()).to(output_dtype)


def matmul_mx(a_x4: torch.Tensor, b_x4: torch.Tensor, a_scale: torch.Tensor, b_scale: torch.Tensor,
              accumulation_dtype: torch.dtype = torch.float32, output_dtype: torch.dtype = torch.bfloat16,
              tile_k: int = 128) -> torch.Tensor:
    """Tiled MX GEMM oracle: accumulates K in ``tile_k``-element steps in ``accumulation_dtype`` (a tensor core accumulates in
    fp32; pass bf16 to study a lower-precision accumulator)."""
    per_word_a = 4
    k_elems = a_x4.shape[1] * per_word_a
    out = torch.zeros(a_x4.shape[0], b_x4.shape[0], dtype=accumulation_dtype)
    for k0 in range(0, k_elems, tile_k):
        k1 = min(k0 + tile_k, k_elems)
        out += matmul_mx_single_tile(a_x4[:, k0 // 4:k1 // 4], b_x4[:, k0 // 4:k1 // 4], a_scale[:, k0 // BLOCK:k1 // BLOCK],
                                     b_scale[:, k0 // BLOCK:k1 // BLOCK], accumulation_dtype)
    return out.to(output_dtype)
