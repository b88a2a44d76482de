"""Linear layers on microscaling (OCP MX) weights.

Weights are the K-contiguous byte stream the checkpoints ship (``quantization/microscaling``): MXFP4 = e2m1 codes two per
byte (low nibble first; ``uint16`` x4 words are a view of the same bytes), MXFP8 = one e4m3 / e5m2 byte per element
(``uint32`` x4 words likewise); one E8M0 scale per 32 elements of a row.

* ``rows <= 8`` on CUDA (token generation): ``csrc/gemv_mx.cu`` — the codes are decoded in registers, nothing is expanded in
  memory, so a decode step reads 4.25 / 8.25 bits per weight instead of 16;
* ``NXD_GEMM_MX=1`` with MXFP8 e4m3 weights on CUDA (prefill): the activations are quantised to MXFP8 as well (OCP ``mx``
  scale rule, 32-element groups) and the block-scaled FP8 GEMM of ``ops.gemm_fp8`` runs on the codes — W8A8-MX numerics, the
  oracle :func:`matmul_mxfp8_reference` of the quantised activations;
* otherwise: de-quantise to the activation dtype and run the dense GEMM (wgmma bf16 kernel on CUDA) — numerically the
  oracle ``experimental…mx_torch.mx_matmul``.

H100 has no 4-bit tensor-core MMA and the block-scaled GEMM takes e4m3 operands only, so ``NXD_GEMM_F4=1`` and
``NXD_GEMM_MX=1`` with MXFP4 or e5m2 MX weights raise on CUDA tensors; :func:`matmul_f4_reference` keeps the 4-bit numerics."""
from __future__ import annotations

import os
from typing import Optional

import torch

from . import _ext

_FMT = {"mxfp4": 0, "mxfp8": 1, "mxfp8_e4m3": 1, "mxfp8_e5m2": 2}                    # gemv_mx format codes
_MMA_FMT = {"mxfp4": 5, "mxfp8": 0, "mxfp8_e4m3": 0, "mxfp8_e5m2": 1}               # kind::mxf8f6f4 operand formats


def kind_of(weight: torch.Tensor, fp8_dtype: torch.dtype = torch.float8_e4m3fn) -> str:
    if weight.dtype in (torch.uint16, torch.float16, torch.int16):
        return "mxfp4"
    if weight.dtype in (torch.uint32, torch.int32):
        return "mxfp8_e5m2" if fp8_dtype == torch.float8_e5m2 else "mxfp8"
    raise ValueError(f"not an x4-packed MX weight: {weight.dtype}")


def dequantize(weight: torch.Tensor, scale: torch.Tensor, kind: str, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """``[N, K/4]`` x4 words (or the raw byte stream) + ``[N, K/32]`` E8M0 → ``[N, K]``."""
    b = weight.contiguous().view(torch.uint8)
    N = scale.shape[0]
    if _FMT[kind] == 0:
        lut = torch.tensor([0, .5, 1, 1.5, 2, 3, 4, 6, -0., -.5, -1, -1.5, -2, -3, -4, -6], dtype=torch.float32, device=b.device)
        vals = torch.stack((lut[(b & 0xF).long()], lut[(b >> 4).long()]), dim=-1).reshape(N, -1)
    else:
        vals = b.view(torch.float8_e4m3fn if _FMT[kind] == 1 else torch.float8_e5m2).float().reshape(N, -1)
    return torch.ldexp(vals.reshape(N, -1, 32), (scale.to(torch.int32) - 127).unsqueeze(-1)).reshape(N, -1).to(dtype)


def tile_scales(scale: torch.Tensor, pad: int = 127) -> torch.Tensor:
    """E8M0 scales ``[R, K/32]`` → the chunked layout the block-scaled GEMM streams: ``[ceil(R/128), K/128, 512]`` where the
    512-byte chunk of (row tile, 128-wide K block) holds scale (r, j) at byte ``(r % 32) * 16 + (r // 32) * 4 + j`` — what
    a Blackwell ``tcgen05.cp.32x128b.warpx4`` spreads over 4 tensor-memory columns (kept as the layout the CPU test replays).  Rows are padded with ``pad`` (E8M0 127 = 2^0).  The same chunking
    serves the 4-bit kinds: a chunk is always 128 rows × 4 consecutive scales, whatever they span."""
    R, KB = scale.shape
    assert KB % 4 == 0, "the number of scale columns must be a multiple of 4"
    T = (R + 127) // 128
    if T * 128 != R:
        scale = torch.cat([scale, torch.full((T * 128 - R, KB), pad, dtype=scale.dtype, device=scale.device)])
    s = scale.reshape(T, 4, 32, KB // 4, 4)                       # [tile, r // 32, r % 32, k block of 128, j]
    return s.permute(0, 3, 2, 1, 4).contiguous().reshape(T, KB // 4, 512)


def matmul_mxfp8_reference(a_q: torch.Tensor, a_scale: torch.Tensor, b_q: torch.Tensor, b_scale: torch.Tensor,
                           a_kind: str = "mxfp8", b_kind: str = "mxfp8") -> torch.Tensor:
    """fp32 oracle of the block-scaled GEMM: ``dequant(a) @ dequant(b)ᵀ``."""
    return dequantize(a_q, a_scale, a_kind) @ dequantize(b_q, b_scale, b_kind).t()


def _no_block_scaled_mma(flag: str, *tensors: torch.Tensor) -> bool:
    if os.environ.get(flag, "0") != "1" or not all(t.is_cuda for t in tensors):
        return False
    raise RuntimeError(f"{flag}=1: H100 has no FP4 tensor-core MMA; the block-scaled FP8 GEMM takes MXFP8 e4m3 weights only")


def gemm_mx_eligible(x2d: torch.Tensor, weight: torch.Tensor, scale: torch.Tensor, kind: str) -> bool:
    """True when ``NXD_GEMM_MX=1`` routes this CUDA call to the block-scaled FP8 GEMM; raises for MX kinds it cannot take."""
    if os.environ.get("NXD_GEMM_MX", "0") != "1" or not all(t.is_cuda for t in (x2d, weight, scale)):
        return False
    if kind not in ("mxfp8", "mxfp8_e4m3"):
        raise RuntimeError(f"NXD_GEMM_MX=1: the block-scaled FP8 GEMM takes MXFP8 e4m3 weights only, not {kind}")
    return True


def _linear_mx_blockscaled(x2: torch.Tensor, weight: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """W8A8-MX: activations quantised with the OCP MX rule in 32-element groups, then the block-scaled FP8 GEMM."""
    from . import gemm_fp8

    N = scale.shape[0]
    wq = weight.contiguous().view(torch.uint8).reshape(N, -1).view(torch.float8_e4m3fn)
    xq, xs = gemm_fp8.quantize_groups(x2, 32, "mx")
    return gemm_fp8.blockscaled_linear(xq, xs, wq, scale, 32)


# ---- 4-bit quantisers and the W4A4 oracle ------------------------------------------------------------
_E2M1 = (0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0)


def _e2m1_codes(v: torch.Tensor) -> torch.Tensor:
    """Round-to-nearest-even onto the e2m1 grid (|v| ≤ 6 after scaling) → 4-bit codes (bit 3 = sign)."""
    mids = torch.tensor([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0], dtype=torch.float32, device=v.device)
    mag = v.abs().float().clamp(max=6.0)
    lo, hi = torch.bucketize(mag, mids, right=False), torch.bucketize(mag, mids, right=True)      # differ only on exact ties
    idx = torch.where(lo % 2 == 0, lo, hi)
    return (idx | ((v < 0).long() << 3)).to(torch.uint8)


def _pack_nibbles(codes: torch.Tensor) -> torch.Tensor:
    c = codes.reshape(*codes.shape[:-1], -1, 2)
    return (c[..., 0] | (c[..., 1] << 4)).contiguous()


def quantize_mxfp4(x: torch.Tensor) -> "tuple[torch.Tensor, torch.Tensor]":
    """``[R, K]`` → (packed e2m1 bytes ``[R, K/2]``, E8M0 scales ``[R, K/32]``); OCP MXFP4: scale = 2^(⌊log2 amax⌋ − 2)."""
    R, K = x.shape
    xb = x.float().reshape(R, K // 32, 32)
    e = torch.floor(torch.log2(xb.abs().amax(-1).clamp(min=2.0 ** -120))) - 2
    codes = _e2m1_codes(torch.ldexp(xb, -e.to(torch.int32).unsqueeze(-1)).reshape(R, K))
    return _pack_nibbles(codes), (e + 127).clamp(0, 254).to(torch.uint8)


def quantize_nvfp4(x: torch.Tensor) -> "tuple[torch.Tensor, torch.Tensor, torch.Tensor]":
    """``[R, K]`` → (packed e2m1 bytes ``[R, K/2]``, UE4M3 block scales ``[R, K/16]`` as bytes, fp32 per-tensor factor): a block's
    scale is ``amax_block / 6`` expressed in units of the per-tensor factor ``amax_tensor / (6 · 448)`` and rounded to e4m3."""
    R, K = x.shape
    xb = x.float().reshape(R, K // 16, 16)
    g = (xb.abs().amax() / (6.0 * 448.0)).clamp(min=2.0 ** -120)
    sf = (xb.abs().amax(-1) / 6.0 / g).clamp(max=448.0).to(torch.float8_e4m3fn)
    eff = (sf.float() * g).clamp(min=2.0 ** -120).unsqueeze(-1)
    codes = _e2m1_codes((xb / eff).reshape(R, K))
    return _pack_nibbles(codes), sf.view(torch.uint8), g.reshape(())


def dequantize_f4(codes: torch.Tensor, scale: torch.Tensor, vec_size: int, global_scale=1.0) -> torch.Tensor:
    """Packed e2m1 ``[R, K/2]`` + block scales ``[R, K/vec_size]`` (E8M0 for 32, UE4M3 for 16) → fp32 ``[R, K]``."""
    b = codes.contiguous().view(torch.uint8)
    R = scale.shape[0]
    lut = torch.tensor(_E2M1 + tuple(-v for v in _E2M1), dtype=torch.float32, device=b.device)
    vals = torch.stack((lut[(b & 0xF).long()], lut[(b >> 4).long()]), dim=-1).reshape(R, -1, vec_size)
    if vec_size == 32:
        return torch.ldexp(vals, (scale.to(torch.int32) - 127).unsqueeze(-1)).reshape(R, -1)
    return (vals * (scale.view(torch.float8_e4m3fn).float() * global_scale).unsqueeze(-1)).reshape(R, -1)


def matmul_f4_reference(a_q, a_scale, b_q, b_scale, vec_size: int = 32, a_global=1.0, b_global=1.0) -> torch.Tensor:
    """fp32 oracle of the 4-bit block-scaled GEMM: ``dequant(a) @ dequant(b)ᵀ``."""
    return dequantize_f4(a_q, a_scale, vec_size, a_global) @ dequantize_f4(b_q, b_scale, vec_size, b_global).t()


def gemm_f4_eligible(M: int, N: int, K: int, *tensors: torch.Tensor) -> bool:
    return _no_block_scaled_mma("NXD_GEMM_F4", *tensors)


def gemv_eligible(x2d: torch.Tensor, weight: torch.Tensor, scale: torch.Tensor) -> bool:
    """The MX GEMV loads 16-byte vectors of the activations and the codes, so both must start 16-byte aligned."""
    if os.environ.get("NXD_GEMV_MX", "0") != "1":                 # opt-in
        return False
    return (x2d.is_cuda and x2d.dtype == torch.bfloat16 and x2d.dim() == 2 and 1 <= x2d.shape[0] <= 8 and x2d.shape[1] % 32 == 0
            and x2d.is_contiguous() and weight.is_contiguous() and scale.is_contiguous() and scale.dtype == torch.uint8
            and scale.dim() == 2 and x2d.data_ptr() % 16 == 0 and weight.data_ptr() % 16 == 0
            and _ext.use_cuda(x2d, weight, scale) and hasattr(_ext.ext(), "gemv_mx"))


def grouped_gemv_eligible(x: torch.Tensor, weight: torch.Tensor, scale: torch.Tensor) -> bool:
    """As :func:`gemv_eligible` for the per-slot expert GEMV (``x [S, K]``, stacked ``[E, N, K]`` codes), given the
    contiguous tensors the kernel will read."""
    if os.environ.get("NXD_GEMV_MX", "0") != "1":
        return False
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 2 and x.shape[1] % 32 == 0
            and x.data_ptr() % 16 == 0 and weight.data_ptr() % 16 == 0
            and _ext.use_cuda(x, weight, scale) and hasattr(_ext.ext(), "gemv_mx_grouped"))


def grouped_linear_mx(x: torch.Tensor, weight: torch.Tensor, scale: torch.Tensor, expert: torch.Tensor, kind: Optional[str] = None
                      ) -> torch.Tensor:
    """Row ``s`` of ``x [S, K]`` against expert ``expert[s]`` of the stacked MX weights ``[E, N, K]`` (x4 words or bytes) with scales
    ``[E, N, K/32]`` → ``[S, N]``: the selective-loading step of a decode-time MoE block.  CUDA (opt-in ``NXD_GEMV_MX=1``): one
    launch that reads only the chosen experts' codes, ids stay on the device; otherwise gather + de-quantise + batched matmul."""
    kind = kind or kind_of(weight)
    E, N = scale.shape[0], scale.shape[1]
    xc, wc = x.contiguous(), weight.contiguous()
    if grouped_gemv_eligible(xc, wc, scale):
        _ext.count_launch()
        return _ext.ext().gemv_mx_grouped(xc, wc, scale.contiguous(), expert.long().contiguous(), _FMT[kind])
    wb = weight.contiguous().view(torch.uint8).reshape(E, N, -1)[expert.long()]                      # [S, N, bytes]
    w = dequantize(wb.reshape(-1, wb.shape[-1]), scale[expert.long()].reshape(-1, scale.shape[-1]), kind).view(x.shape[0], N, -1)
    return torch.einsum("sk,snk->sn", x.float(), w).to(x.dtype)


def linear_mx(x: torch.Tensor, weight: torch.Tensor, scale: torch.Tensor, kind: Optional[str] = None,
              residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``x [..., K] @ dequant(weight)[N, K]ᵀ (+ residual)`` → ``[..., N]`` in ``x.dtype``."""
    kind = kind or kind_of(weight)
    x2 = x.reshape(-1, x.shape[-1])
    if gemv_eligible(x2.contiguous(), weight, scale):
        _ext.count_launch()
        r2 = None if residual is None else residual.reshape(-1, residual.shape[-1]).contiguous()
        y = _ext.ext().gemv_mx(x2.contiguous(), weight, scale, _FMT[kind], r2)
        return y.view(*x.shape[:-1], y.shape[-1])
    if kind == "mxfp4":
        _no_block_scaled_mma("NXD_GEMM_F4", x2, weight, scale)       # no FP4 tensor-core MMA on H100: raise, never de-quantise
    if gemm_mx_eligible(x2, weight, scale, kind):
        y = _linear_mx_blockscaled(x2, weight, scale).view(*x.shape[:-1], scale.shape[0])
        if residual is not None:
            y = y + residual.to(y.dtype)
        return y.to(x.dtype)
    w = dequantize(weight, scale, kind, x.dtype if x.dtype in (torch.bfloat16, torch.float16) else torch.float32)
    y = torch.nn.functional.linear(x.to(w.dtype), w)
    if residual is not None:
        y = y + residual.to(y.dtype)
    return y.to(x.dtype)
