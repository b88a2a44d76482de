"""Small shared enums / helpers (reference ``utils/utils.py:6-70``)."""
from __future__ import annotations

import json
import os
from enum import Enum
from typing import Any, Dict, Union


class hardware(Enum):  # noqa: N801  (reference spelling)
    """Target platform.  This framework targets exactly one GPU (H100; the member keeps its name ``B200``); the Trainium names of the reference resolve to it
    so that scripts passing ``hardware_type="trn2"`` keep working."""

    B200 = "b200"
    CUSTOM = "custom"

    @classmethod
    def _missing_(cls, value):
        if isinstance(value, str) and value.lower() in ("trn1", "trn1n", "inf2", "trn2", "trn3", "b200", "sm_100a", "sm100"):
            return cls.B200
        if value == os.environ.get("NEURON_PLATFORM_TARGET_OVERRIDE"):
            return cls.CUSTOM
        return None


hardware.TRN1 = hardware.TRN2 = hardware.TRN3 = hardware.B200  # type: ignore[attr-defined]


class HloMetadataLevel(Enum):
    """Verbosity of the per-program debug metadata the inference builder records (NVTX ranges + source locations of
    captured graphs here; HLO metadata in the reference)."""

    DEBUG = "debug"
    INFO = "info"
    NONE = "none"

    @classmethod
    def _missing_(cls, value):
        if value is True:
            return cls.DEBUG
        if value is False:
            return cls.INFO
        return None


def get_dict_from_json(json_file: Union[str, os.PathLike]) -> Dict[Any, Any]:
    """Parse a JSON file into a dict; ``ValueError`` with the path when it is not valid JSON."""
    try:
        with open(json_file, "r") as f:
            return json.load(f)
    except json.JSONDecodeError as e:
        raise ValueError(f"Failed to parse {json_file} as JSON: {e}") from e
