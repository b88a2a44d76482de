"""RMSNorm forward/backward (kernels: ``csrc/elementwise.cu`` rmsnorm_fwd / rmsnorm_bwd).

fp32 statistics regardless of I/O dtype (reference ``modules/rms_norm.py:10-33``).  The backward
kernel emits dX and per-CTA partial dW rows that a tiny second kernel reduces.  Rows whose width is not a
multiple of 16 bytes (or that do not start 16-byte aligned) take the torch composition.
"""
from __future__ import annotations

import torch

from . import _ext


def _vec_rows(*ts) -> bool:
    """The norm kernels move rows as 16-byte packets: every row of every operand must start 16-byte aligned."""
    return all(t.shape[-1] * t.element_size() % 16 == 0 and t.data_ptr() % 16 == 0 for t in ts)


def _aligned(t: torch.Tensor) -> torch.Tensor:
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _rms_ref(x, w, eps):
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (xf * rstd * w.float()).to(x.dtype), rstd


class _RMSNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        ctx.eps = eps
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        if _ext.use_cuda(x2, weight) and x2.dtype in (torch.bfloat16, torch.float32, torch.float16) \
                and _vec_rows(x2 := x2.contiguous(), weight := weight.contiguous()):
            _ext.count_launch()
            y, rstd = _ext.ext().rmsnorm_fwd(x2, weight, float(eps))
            ctx.cuda = True
        else:
            y, rstd = _rms_ref(x2, weight, eps)
            ctx.cuda = False
        ctx.save_for_backward(x2, weight, rstd)
        return y.view(shape)

    @staticmethod
    def backward(ctx, gy):
        x2, weight, rstd = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1])
        if ctx.cuda:
            _ext.count_launch(2)
            gx, gw = _ext.ext().rmsnorm_bwd(_aligned(g2), x2.contiguous(), weight.contiguous(), rstd)
            return gx.view(gy.shape), gw.to(weight.dtype), None
        xf, gf, wf = x2.float(), g2.float(), weight.float()
        xhat = xf * rstd
        gw = (gf * xhat).sum(0)
        gxh = gf * wf
        gx = rstd * (gxh - xhat * (gxh * xhat).mean(-1, keepdim=True))
        return gx.to(x2.dtype).view(gy.shape), gw.to(weight.dtype), None


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    return _RMSNorm.apply(x, weight, eps)


class _AddRMSNorm(torch.autograd.Function):
    """``h = x + residual``; ``y = rmsnorm(h) * w`` → ``(y, h)`` in one pass (kernels: ``csrc/fused_norm.cu``).  Backward takes
    the gradients of both outputs (``gh`` = what arrives on the residual path) and returns ONE tensor used for ``x`` and
    ``residual``: ``dh = gh + rmsnorm_bwd(gy)``."""

    @staticmethod
    def forward(ctx, x, residual, weight, eps):
        shape = x.shape
        x2, r2 = x.reshape(-1, shape[-1]), residual.reshape(-1, shape[-1])
        if _ext.use_cuda(x2, weight) and x2.dtype in (torch.bfloat16, torch.float32, torch.float16) and r2.dtype == x2.dtype \
                and _vec_rows(x2 := x2.contiguous(), r2 := r2.contiguous(), weight := weight.contiguous()):
            _ext.count_launch()
            y, h, rstd = _ext.ext().add_rmsnorm_fwd(x2, r2, weight, float(eps))
            ctx.cuda = True
        else:
            h = x2 + r2
            y, rstd = _rms_ref(h, weight, eps)
            ctx.cuda = False
        ctx.save_for_backward(h, weight, rstd)
        return y.view(shape), h.view(shape)

    @staticmethod
    def backward(ctx, gy, gh):
        h, weight, rstd = ctx.saved_tensors
        g2, r2 = gy.reshape(-1, gy.shape[-1]), gh.reshape(-1, gh.shape[-1])
        if ctx.cuda:
            _ext.count_launch(2)
            dh, gw = _ext.ext().add_rmsnorm_bwd(_aligned(g2), _aligned(r2), h, weight.contiguous(), rstd)
        else:
            hf, gf, wf = h.float(), g2.float(), weight.float()
            hhat = hf * rstd
            gw = (gf * hhat).sum(0)
            gxh = gf * wf
            dh = (r2.float() + rstd * (gxh - hhat * (gxh * hhat).mean(-1, keepdim=True))).to(h.dtype)
        dh = dh.view(gy.shape)
        return dh, dh, gw.to(weight.dtype), None


def add_rms_norm(x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6):
    """Returns ``(rmsnorm(x + residual) * weight, x + residual)``."""
    return _AddRMSNorm.apply(x, residual, weight, eps)
