"""Loader for the in-tree sm_90a (H100) extension ``nxd_b200_C``.

The extension is built IN-TREE (``neuronx_distributed_b200/_build/nxd_b200_C.so``) by
``__graft_entry__.build()`` / ``python -m neuronx_distributed_b200.ops.build`` so that it travels
with the source snapshot to GPU boxes.  On a machine with a GPU the CUDA path is the one that
runs: if the extension cannot be loaded there, ops raise instead of silently falling back
(set ``NXD_ALLOW_EAGER_FALLBACK=1`` to override, e.g. for debugging).
"""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os
import sys
from pathlib import Path
from typing import Optional

import torch

PKG_DIR = Path(__file__).resolve().parent.parent
BUILD_DIR = PKG_DIR / "_build"
EXT_NAME = "nxd_b200_C"

_C = None
_PLAN_PROXY = None          # set by inference.launch_plan.record(): kernel calls are recorded through it
_LOAD_ERROR: Optional[BaseException] = None
_TRIED = False


def _load():
    global _C, _LOAD_ERROR, _TRIED
    if _TRIED:
        return _C
    _TRIED = True
    so = BUILD_DIR / f"{EXT_NAME}.so"
    if not so.exists():
        _LOAD_ERROR = FileNotFoundError(f"{so} not built; run `python -m neuronx_distributed_b200.ops.build`")
        return None
    try:
        loader = importlib.machinery.ExtensionFileLoader(EXT_NAME, str(so))
        spec = importlib.util.spec_from_loader(EXT_NAME, loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        sys.modules[EXT_NAME] = mod
        _C = mod
    except BaseException as e:  # pragma: no cover - depends on box
        _LOAD_ERROR = e
        _C = None
    return _C


def ext():
    """The extension module or ``None``."""
    if _PLAN_PROXY is not None:
        return _PLAN_PROXY
    return _load()


def load_error() -> Optional[BaseException]:
    _load()
    return _LOAD_ERROR


def use_cuda(*tensors: torch.Tensor) -> bool:
    """True when the hand-written kernels must handle these tensors.

    CPU tensors → False (reference math).  CUDA tensors → True if the extension loaded; if
    it did not, raise loudly unless the eager fallback is explicitly allowed."""
    if not tensors or not all(isinstance(t, torch.Tensor) and t.is_cuda for t in tensors):
        return False
    if os.environ.get("NXD_FORCE_EAGER", "0") == "1":
        return False
    if _load() is not None:
        return True
    if os.environ.get("NXD_ALLOW_EAGER_FALLBACK", "0") == "1":
        return False
    raise RuntimeError(
        f"CUDA tensors given but the sm_90a extension is not loaded ({_LOAD_ERROR!r}). "
        "Build it with `python -m neuronx_distributed_b200.ops.build` or set NXD_ALLOW_EAGER_FALLBACK=1."
    )


# launch accounting — bench.py reports how many of OUR kernels ran in the timed region
_LAUNCHES = 0


def count_launch(n: int = 1) -> None:
    global _LAUNCHES
    _LAUNCHES += n


def launches() -> int:
    return _LAUNCHES


def reset_launches() -> None:
    global _LAUNCHES
    _LAUNCHES = 0
