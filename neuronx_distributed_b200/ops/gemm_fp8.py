"""fp8 × fp8 linear with outer-product scales: ``y = (xq @ wqᵀ) · xs[:, None] · ws[None, :]``.

CUDA: the fp8 instantiation of the wgmma GEMM (``csrc/gemm_sm90.cu``: ``wgmma m64n256k32.e4m3``, e4m3 operands staged by
TMA as 128-byte swizzle rows of 128 elements, fp32 accumulation in registers, scales applied in the epilogue).
CPU: fp32 reference.  Reference: quantization/quantization_layers.py (scaled matmul of the quantised parallel layers)."""
from __future__ import annotations

import torch

from . import _ext


def scaled_linear(xq: torch.Tensor, xs: torch.Tensor, wq: torch.Tensor, ws: torch.Tensor,
                  out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    shape = xq.shape
    x2 = xq.reshape(-1, shape[-1])
    s2 = xs.reshape(-1, 1).float()
    e = _ext.ext() if x2.is_cuda else None
    if (e is not None and hasattr(e, "gemm_fp8") and x2.shape[1] % 16 == 0 and wq.shape[0] % 8 == 0
            and xq.dtype == torch.float8_e4m3fn and wq.dtype == torch.float8_e4m3fn and out_dtype == torch.bfloat16):
        out = torch.empty(x2.shape[0], wq.shape[0], dtype=out_dtype, device=x2.device)
        _ext.count_launch()
        e.gemm_fp8(x2.contiguous(), wq.contiguous(), out, s2.expand(x2.shape[0], 1).contiguous().view(-1),
                   ws.float().reshape(-1).expand(wq.shape[0]).contiguous())
        return out.view(*shape[:-1], wq.shape[0])
    y = (x2.float() @ wq.float().t()) * s2 * ws.float().reshape(1, -1)
    return y.to(out_dtype).view(*shape[:-1], wq.shape[0])
