"""bf16 GEMM on Hopper wgmma tensor cores (kernel: ``csrc/gemm_sm90.cu``).

``matmul(a, b, trans_a, trans_b)`` computes ``op(a) @ op(b)`` for row-major 2-D bf16 tensors with
fp32 accumulation in registers.  The three layouts training needs map to wgmma operand majors without
any transposition copies:

    fwd   : x[M,K] @ W[N,K]^T     → A K-major,  B K-major     ("nt")
    dgrad : g[M,K] @ W[K,N]       → A K-major,  B MN-major    ("nn")
    wgrad : g[K,M]^T @ x[K,N]     → A MN-major, B MN-major    ("tn")
"""
from __future__ import annotations

import os

import torch

from . import _ext

_MIN_DIM = 64

#: activation codes of the decode GEMV epilogue (``csrc/decode.cu`` gemv_act): HF ``hidden_act`` name → code
GEMV_ACT = {"gelu": 1, "gelu_fast": 2, "gelu_new": 2, "gelu_pytorch_tanh": 2}


def _act_torch(y: torch.Tensor, act: int) -> torch.Tensor:
    if act == 0:
        return y
    if act not in (1, 2):
        raise ValueError(f"act must be 0 (none), 1 (exact GELU) or 2 (tanh GELU), got {act}")
    return torch.nn.functional.gelu(y, approximate="none" if act == 1 else "tanh")


def fused_wgrad_enabled() -> bool:
    return os.environ.get("NXD_DISABLE_FUSED_WGRAD", "0") != "1" and os.environ.get("NXD_DISABLE_TCGEN05_GEMM", "0") != "1"


def _eligible(a: torch.Tensor, b: torch.Tensor, M: int, N: int, K: int) -> bool:
    if os.environ.get("NXD_DISABLE_TCGEN05_GEMM", "0") == "1":
        return False
    if not (a.is_cuda and b.is_cuda and a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16):
        return False
    if not (a.is_contiguous() and b.is_contiguous()) or a.data_ptr() % 16 or b.data_ptr() % 16:
        return False
    if not _ext.use_cuda(a, b) or not hasattr(_ext.ext(), "gemm_bf16"):
        return False
    # TMA needs 16-byte aligned rows; kernel handles ragged M/N/K tails via TMA zero fill
    return M >= 1 and N % 8 == 0 and K % 8 == 0 and M % 8 == 0


def _gemv_eligible(a: torch.Tensor, b: torch.Tensor, M: int, K: int, trans_a: bool, trans_b: bool, out, out_dtype) -> bool:
    """``x[M <= 8, K] @ W[N, K]ᵀ`` with a bf16 result goes to the decode GEMV.  It loads 16-byte vectors of both operands,
    so both must start 16-byte aligned: a contiguous view at an element offset that is not a multiple of 8 (a tensor cut
    out of a flat buffer after tensors of odd sizes) is not, and takes the general path."""
    return (M <= 8 and not trans_a and trans_b and out is None and out_dtype == torch.bfloat16 and a.is_cuda
            and a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and K % 8 == 0 and a.is_contiguous() and b.is_contiguous()
            and a.data_ptr() % 16 == 0 and b.data_ptr() % 16 == 0
            and _ext.ext() is not None and hasattr(_ext.ext(), "gemv") and os.environ.get("NXD_DISABLE_TCGEN05_GEMM", "0") != "1")


def matmul(a: torch.Tensor, b: torch.Tensor, trans_a: bool = False, trans_b: bool = False,
           out: torch.Tensor | None = None, accumulate: bool = False, out_dtype=None, bias: torch.Tensor | None = None,
           act: int = 0) -> torch.Tensor:
    """``op(a) @ op(b)`` for 2-D tensors. ``accumulate`` adds into ``out`` (fp32 or bf16).  ``bias [N]`` and ``act`` (a
    :data:`GEMV_ACT` code; 0 none) give ``act(op(a) @ op(b) + bias)``: in the decode GEMV's epilogue when it runs, else as
    separate ops on the result (not with ``out``)."""
    M = a.shape[1] if trans_a else a.shape[0]
    K = a.shape[0] if trans_a else a.shape[1]
    N = b.shape[0] if trans_b else b.shape[1]
    out_dtype = out_dtype or (out.dtype if out is not None else a.dtype)
    if bias is not None or act:
        if out is not None:
            raise ValueError("matmul: bias / act do not combine with out=")
        if (_gemv_eligible(a, b, M, K, trans_a, trans_b, out, out_dtype)
                and (bias is None or (bias.dtype == torch.bfloat16 and bias.is_contiguous() and bias.shape == (N,)))):
            _ext.count_launch()
            return _ext.ext().gemv(a, b, None, bias=bias, act=act)
        y = matmul(a, b, trans_a, trans_b, out_dtype=out_dtype)
        return _act_torch(y if bias is None else y + bias, act)
    if _gemv_eligible(a, b, M, K, trans_a, trans_b, out, out_dtype):
        # decode-time GEMV: a bandwidth problem (every weight byte read once), not a tensor-core one — csrc/decode.cu
        _ext.count_launch()
        return _ext.ext().gemv(a, b, None)
    if _eligible(a, b, M, N, K) and out_dtype in (torch.bfloat16, torch.float32):
        if out is None:
            out = torch.empty(M, N, dtype=out_dtype, device=a.device)
            accumulate = False
        _ext.count_launch()
        _ext.ext().gemm_bf16(a, b, out, bool(trans_a), bool(trans_b), bool(accumulate))
        return out
    if a.is_cuda and a.dtype == torch.bfloat16 and not os.environ.get("NXD_DISABLE_TCGEN05_GEMM") \
            and (not a.is_contiguous() or not b.is_contiguous()):
        # make operands dense once and retry the tensor-core kernel
        return matmul(a.contiguous(), b.contiguous(), trans_a, trans_b, out, accumulate, out_dtype)
    aa = a.t() if trans_a else a
    bb = b.t() if trans_b else b
    res = torch.matmul(aa, bb)
    if out is not None:
        if accumulate:
            out.add_(res.to(out.dtype))
        else:
            out.copy_(res)
        return out
    return res.to(out_dtype)


def linear_nt(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, act: int = 0) -> torch.Tensor:
    """``act(x[..., K] @ w[N, K]^T + bias)`` (see :func:`matmul`)."""
    x2 = x.reshape(-1, x.shape[-1])
    return matmul(x2, w, False, True, bias=bias, act=act).view(*x.shape[:-1], w.shape[0])


# ---------------------------------------------------------------------------------------------------------------------
# Grouped (MoE blockwise) GEMM: rows of ``x`` come in ``block_size``-row blocks, block i is multiplied by the weights of
# expert ``block_to_expert[i]``.  CUDA: MODE 3/4 of ``csrc/gemm_sm90.cu`` (the per-block expert only shifts the TMA
# coordinate of the weight tile — no per-block weight copies, no host sync); CPU / odd shapes: plain loop.
# Role of the reference's blockwise NKI kernels (modules/moe/blockwise.py:180-468, 1037-1127).
def _grouped_ok(x: torch.Tensor, w: torch.Tensor, block_size: int) -> bool:
    e = _ext.ext()
    return (x.is_cuda and e is not None and hasattr(e, "grouped_gemm") and x.dtype == torch.bfloat16
            and w.dtype == torch.bfloat16 and block_size % 128 == 0 and w.shape[1] % 64 == 0 and w.shape[2] % 64 == 0
            and os.environ.get("NXD_DISABLE_GROUPED_GEMM", "0") != "1")


def _grouped_ref(x, w, b2e, block_size):
    nb = b2e.numel()
    xb = x.view(nb, block_size, x.shape[-1])
    return torch.einsum("bth,bhi->bti", xb, w[b2e.long()]).reshape(nb * block_size, w.shape[-1])


class _GroupedMatmul(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b2e, seg_first_block, block_size):
        ctx.save_for_backward(x, w, b2e, seg_first_block)
        ctx.block_size = block_size
        _ext.count_launch()
        return _ext.ext().grouped_gemm(x.contiguous(), w.contiguous(), b2e, block_size, False)

    @staticmethod
    def backward(ctx, gy):
        x, w, b2e, seg = ctx.saved_tensors
        gy = gy.contiguous()
        gx = gw = None
        if ctx.needs_input_grad[0]:
            _ext.count_launch()
            gx = _ext.ext().grouped_gemm(gy, w.contiguous(), b2e, ctx.block_size, True)       # dy · W[e]ᵀ
        if ctx.needs_input_grad[1]:
            _ext.count_launch()
            mg = getattr(w, "main_grad", None)
            if mg is not None and fused_wgrad_enabled() and mg.dtype == torch.float32 and mg.is_contiguous():
                fresh = getattr(w, "main_grad_fresh", False)
                _ext.ext().grouped_wgrad(x.contiguous(), gy, mg.view_as(w), seg, ctx.block_size, not fresh)
                w.main_grad_fresh = False
                cb = getattr(w, "_nxd_grad_ready", None)
                if cb is not None:
                    cb(w)
            else:
                gw = torch.empty_like(w)
                _ext.ext().grouped_wgrad(x.contiguous(), gy, gw, seg, ctx.block_size, False)
        return gx, gw, None, None, None


def grouped_matmul(x: torch.Tensor, w: torch.Tensor, block_to_expert: torch.Tensor, seg_first_block: torch.Tensor,
                   block_size: int) -> torch.Tensor:
    """``y[i·B:(i+1)·B] = x[i·B:(i+1)·B] @ w[block_to_expert[i]]`` with ``x [nb·B, K]``, ``w [E, K, N]``."""
    if _grouped_ok(x, w, block_size):
        return _GroupedMatmul.apply(x, w, block_to_expert.int(), seg_first_block.int(), block_size)
    return _grouped_ref(x, w, block_to_expert, block_size)
