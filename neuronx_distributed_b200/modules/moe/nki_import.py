"""Kernel resolution with fallbacks — the role of reference ``modules/moe/nki_import.py`` (``NKIImport`` / ``import_nki`` /
``import_nki_beta2``: look a kernel up by name in a list of candidate modules and return ``(kernel, None)`` or
``(None, reason)`` instead of raising, so callers can degrade to their torch path and say why).

Here the candidates are, in order: the sm_90a extension (``ops._ext.ext()``, entry points of ``csrc/*.cu``), the ``ops``
package (Python front ends that pick the kernel or its CPU oracle), and ``modules.moe.blockwise``.  The reference's names are
kept as aliases so code written against them imports unchanged."""
from __future__ import annotations

import importlib
from dataclasses import dataclass
from typing import Any, Optional, Tuple


@dataclass
class KernelImport:
    """What to resolve: ``name`` inside ``module_name`` (``None``: search the default places).  ``is_kernel``: the name must be a
    device entry point — resolution fails when the extension is not loaded.  ``nki_jit_type`` is accepted for signature
    compatibility (there is nothing to JIT: the kernels are compiled ahead of time)."""
    name: str
    module_name: Optional[str] = None
    nki_jit_type: Optional[str] = None
    is_kernel: Optional[bool] = None


NKIImport = KernelImport

_PKG = __name__.rsplit(".", 3)[0]                       # neuronx_distributed_b200


def _candidates(cfg: KernelImport):
    if cfg.module_name:
        yield f"{_PKG}.{cfg.module_name}"
        yield f"{_PKG}.ops.{cfg.module_name}"
        yield f"{_PKG}.modules.moe.{cfg.module_name}"
        yield cfg.module_name
    else:
        yield f"{_PKG}.ops"
        yield f"{_PKG}.modules.moe.blockwise"


def import_kernel(import_config: KernelImport) -> Tuple[Optional[Any], Optional[str]]:
    """``(object, None)`` or ``(None, reason)``; never raises for a missing module / attribute / extension."""
    from ...ops import _ext

    last = None
    e = _ext.ext()
    if e is not None and not import_config.module_name and hasattr(e, import_config.name):
        return getattr(e, import_config.name), None
    if import_config.is_kernel and e is None:
        return None, f"Failed to import {import_config.name}: the sm_90a extension is not loaded ({_ext.load_error()!r})"
    for path in _candidates(import_config):
        try:
            module = importlib.import_module(path)
        except ImportError as err:
            last = str(err)
            continue
        if hasattr(module, import_config.name):
            return getattr(module, import_config.name), None
        last = f"Attribute {import_config.name} not found in {path}"
    return None, f"Failed to import {import_config.name}: {last}"


import_nki = import_kernel
import_nki_beta2 = import_kernel
