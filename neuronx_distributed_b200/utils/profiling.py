"""Profiling / debugging helpers (SURVEY §5.1, §5.2).

* ``nvtx_range(name)`` — NVTX range when ``NXD_NVTX=1`` (no-op otherwise): pipeline tasks, decoder layers and optimizer phases
  are bracketed so Nsight timelines show the schedule.  The reference's only timeline is a host-clock Chrome trace that is
  force-disabled (``pipeline/model.py:336-339``).
* ``device_timer()`` — CUDA-event stopwatch (device time, not host time) for step / phase timing.
"""
from __future__ import annotations

import contextlib
import os
from typing import Iterator, Optional

import torch

_NVTX = os.environ.get("NXD_NVTX", "0") == "1"


@contextlib.contextmanager
def nvtx_range(name: str) -> Iterator[None]:
    if _NVTX and torch.cuda.is_available():
        torch.cuda.nvtx.range_push(name)
        try:
            yield
        finally:
            torch.cuda.nvtx.range_pop()
    else:
        yield


class device_timer:
    """``with device_timer() as t: ...; t.ms`` — elapsed device time between two CUDA events on the current stream
    (falls back to the host clock on CPU)."""

    def __init__(self) -> None:
        self.ms: Optional[float] = None

    def __enter__(self):
        if torch.cuda.is_available():
            self._e0, self._e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self._e0.record()
        else:
            import time
            self._t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        if torch.cuda.is_available():
            self._e1.record()
            self._e1.synchronize()
            self.ms = self._e0.elapsed_time(self._e1)
        else:
            import time
            self.ms = (time.perf_counter() - self._t0) * 1e3
        return False
