"""Dispatch of TP linear layers onto the fused GEMM+collective kernels.

``dispatch(x, weight, in_mode, out_mode, seq_dim, group)`` returns an object with
``forward``/``backward`` when the sm_90a fused path applies, else ``None`` (the caller then
runs collectives + matmul through the library path).  Filled in by ``_fused_impl`` once the
extension exposes the kernels; selection can be forced off with ``NXD_TP_BACKEND=nccl``.
"""
from __future__ import annotations

import os

import torch


_BACKEND = os.environ.get("NXD_TP_BACKEND", "fused")


def set_backend(name: str) -> None:
    """``"fused"`` (hand-written kernels; default on CUDA), ``"nccl"`` (library baseline) or ``"nocomm"`` (measurement only: the same
    GEMM shapes with the collectives replaced by local copies — numerically meaningless, used by ``bench.py`` to report the
    exposed tensor-parallel communication time as ``t(fused) − t(nocomm)``)."""
    global _BACKEND
    assert name in ("fused", "nccl", "nocomm")
    _BACKEND = name


def get_backend() -> str:
    return _BACKEND


class _NoComm:
    """Column+SP / Row+SP linear with the collective replaced by a local copy of the right shape (timing experiments only)."""

    def __init__(self, world: int, column: bool):
        self.world, self.column = world, column
        self.gathered = None

    @staticmethod
    def _flat(t):
        return t.reshape(-1, t.shape[-1])

    def forward(self, x, weight):
        from . import gemm

        x2 = self._flat(x).contiguous()
        if self.column:
            xg = x2.repeat(self.world, 1)                      # stands in for the all-gather (one local copy)
            self.gathered = xg
            out = gemm.matmul(xg, weight, False, True)
            return out.view(x.shape[0] * self.world, *x.shape[1:-1], weight.shape[0])
        out = gemm.matmul(x2, weight, False, True)
        ms = out.shape[0] // self.world
        return out[:ms].contiguous().view(x.shape[0] // self.world, *x.shape[1:-1], weight.shape[0])

    def backward(self, x, weight, gy, has_bias, need_gx, need_gw, gathered=None, gy_dgrad=None):
        from . import gemm
        from ..parallel_layers.layers import wgrad

        g2 = self._flat(gy).contiguous()
        gbias = g2.float().sum(0).to(gy.dtype) if has_bias else None
        gx = gw = None
        if self.column:
            if need_gx:
                gx = gemm.matmul(g2, weight, False, False)[: g2.shape[0] // self.world].contiguous().view(x.shape)
            if need_gw:
                gw = wgrad(g2, gathered if gathered is not None else self.gathered, weight)
        else:
            gf = g2.repeat(self.world, 1)
            if need_gx:
                gx = gemm.matmul(gf, weight, False, False).view(x.shape)
            if need_gw:
                gw = wgrad(gf, self._flat(x), weight)
        return gx, gw, gbias


def dispatch(x: torch.Tensor, weight: torch.Tensor, in_mode: str, out_mode: str, seq_dim: int, group):
    if _BACKEND == "nocomm" and x.is_cuda and seq_dim == 0:
        import torch.distributed as dist

        world = dist.get_world_size(group)
        if world > 1 and in_mode == "gather" and out_mode == "none":
            return _NoComm(world, True)
        if world > 1 and in_mode == "none" and out_mode == "scatter":
            return _NoComm(world, False)
        return None
    if _BACKEND != "fused" or not x.is_cuda:
        return None
    try:
        from . import _fused_impl
    except ImportError:
        return None
    return _fused_impl.select(x, weight, in_mode, out_mode, seq_dim, group)
