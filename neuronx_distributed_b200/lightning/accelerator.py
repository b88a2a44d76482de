"""Lightning accelerator for H100 GPUs (role of reference ``lightning/accelerator.py:17-82`` — ``NeuronXLAAccelerator``).

One process drives one GPU (``torchrun`` / Lightning's subprocess launcher), so ``get_parallel_devices(n)`` is the list of
local CUDA devices and ``auto_device_count`` is what the driver reports.  Derives from Lightning's ``CUDAAccelerator`` when
Lightning is importable; otherwise a stand-in with the same static interface, so strategy code and tests can use it."""
from __future__ import annotations

from typing import Any, Dict, List, Union

import torch

try:  # pragma: no cover - lightning is not installed in the offline image
    from lightning.pytorch.accelerators import CUDAAccelerator as _Base
except Exception:  # noqa: BLE001
    class _Base:  # type: ignore[no-redef]
        def setup_device(self, device: torch.device) -> None:
            pass

        def teardown(self) -> None:
            pass


def _parse_devices(devices: Union[int, str, List[int]]) -> Union[int, List[int]]:
    if isinstance(devices, str):
        devices = devices.strip()
        if devices in ("auto", "-1"):
            return max(1, torch.cuda.device_count())
        devices = [int(d) for d in devices.split(",") if d.strip()] if "," in devices else int(devices)
    if isinstance(devices, int):
        if devices == -1:
            return max(1, torch.cuda.device_count())
        if devices < 1:
            raise ValueError(f"devices must be a positive count or a list of indices, got {devices}")
        return devices
    if not devices or any((not isinstance(d, int)) or d < 0 for d in devices):
        raise ValueError(f"invalid device list {devices}")
    return list(devices)


class NeuronXLAAccelerator(_Base):
    """Name kept from the reference so ``Trainer(accelerator=NeuronXLAAccelerator())`` ports unchanged."""

    def setup_device(self, device: torch.device) -> None:
        if device.type == "cuda":
            torch.cuda.set_device(device)

    def get_device_stats(self, device) -> Dict[str, Any]:
        if torch.cuda.is_available():
            return torch.cuda.memory_stats(device)
        return {}

    @staticmethod
    def parse_devices(devices: Union[int, str, List[int]]) -> Union[int, List[int]]:
        return _parse_devices(devices)

    @staticmethod
    def get_parallel_devices(devices: Union[int, str, List[int]]) -> List[torch.device]:
        parsed = _parse_devices(devices)
        idx = list(range(parsed)) if isinstance(parsed, int) else parsed
        kind = "cuda" if torch.cuda.is_available() else "cpu"
        return [torch.device(kind, i) if kind == "cuda" else torch.device("cpu") for i in idx]

    @staticmethod
    def auto_device_count() -> int:
        return torch.cuda.device_count()

    @staticmethod
    def is_available() -> bool:
        return torch.cuda.is_available()

    @classmethod
    def register_accelerators(cls, accelerator_registry) -> None:
        accelerator_registry.register("b200", cls, description=cls.__name__)


B200Accelerator = NeuronXLAAccelerator
