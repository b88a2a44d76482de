"""Runtime-mode helpers.

The reference has one global switch, ``NXD_CPU_MODE`` (reference
``src/neuronx_distributed/utils/__init__.py:6-26``), that swaps XLA collectives for gloo.
Here the split is *device kind*: CUDA (NCCL process groups + sm_90a kernels) or CPU
(gloo process groups + plain PyTorch math).  CPU mode is chosen automatically when no GPU
is visible, or forced with ``NXD_CPU_MODE=1`` so the whole library is testable with
``torchrun --nproc-per-node N`` on a laptop.
"""
from __future__ import annotations

import os

import torch

_FORCED_CPU = None  # type: ignore[var-annotated]


def set_cpu_mode(flag: bool | None) -> None:
    """Force (True/False) or un-force (None) CPU mode from python (tests use this)."""
    global _FORCED_CPU
    _FORCED_CPU = flag


def cpu_mode() -> bool:
    if _FORCED_CPU is not None:
        return _FORCED_CPU
    if os.environ.get("NXD_CPU_MODE", "0") == "1":
        return True
    return not torch.cuda.is_available()


def get_device() -> torch.device:
    """Device this rank computes on (reference ``utils/__init__.py:16-21``)."""
    if cpu_mode():
        return torch.device("cpu")
    return torch.device("cuda", torch.cuda.current_device())


def default_backend() -> str:
    return "gloo" if cpu_mode() else "nccl"


def mark_step() -> None:
    """Graph cut on lazy XLA; CUDA is eager so this is intentionally a no-op
    (reference ``utils/__init__.py:23-26``)."""
    return None


def master_print(*args, **kwargs) -> None:
    import torch.distributed as dist

    if not dist.is_available() or not dist.is_initialized() or dist.get_rank() == 0:
        print(*args, **kwargs, flush=True)


def synchronize() -> None:
    if not cpu_mode():
        torch.cuda.synchronize()


from .logger import get_logger  # noqa: E402

__all__ = [
    "cpu_mode",
    "set_cpu_mode",
    "get_device",
    "default_backend",
    "mark_step",
    "master_print",
    "synchronize",
    "get_logger",
]
