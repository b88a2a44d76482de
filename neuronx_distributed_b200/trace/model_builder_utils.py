"""Artifacts passed between ``trace`` → ``compile`` → ``NxDModel.add`` (reference ``trace/model_builder_utils.py:8-179``).

The reference's artifacts are protobufs on their way through a compiler (HLO, metaneff, NEFF).  Here there is no
compiler: a *trace* is the validated call signature + example inputs of one bucket (and the structure of its outputs,
recorded by one eager run), a *compilation* is the same bucket with a captured CUDA graph and persistent input/output
buffers.  The class names and the way they are threaded through the API are the reference's."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch


class ModelBuilderConstants:
    DEFAULT_WORLD_SIZE = 1
    LAYOUT_TRANSFORMER_KEY = "layout_transformer"        # kept for API parity; weights need no re-layout between buckets
    DEFAULT_KEY_PREFIX = "model"
    DEFAULT_COMPILER_WORKDIR = "/tmp/nxd_b200_workdir/"
    LOG_FILE_DEFAULT_NAME = "log-capture.txt"
    GRAPH_HLO_FILE = "program.txt"                        # per-bucket description written by ``compile`` (no HLO here)
    NEFF_FILE = "program.txt"
    WRAPPED_NEFF_FILE = "program.txt"
    METANEFF_FILE = "metadata.txt"


@dataclass
class ModelParamInfo:
    """One parameter of the model's ``forward`` signature; positional = no default value."""
    param_name: str
    is_positional: bool


@dataclass
class ProvidedArgInfo:
    """One example input, bound to the signature parameter it feeds."""
    param_name: str
    is_positional: bool
    tensor: torch.Tensor


@dataclass
class TraceArtifacts:
    model: Any                                             # nn.Module or callable
    provided_args: List[ProvidedArgInfo]
    model_params: List[ModelParamInfo]
    output_spec: Any = None                                # nested structure with tensors replaced by (shape, dtype)
    weight_name_to_idx: Dict[str, int] = field(default_factory=dict)
    weight_names_to_skip: set = field(default_factory=set)
    state_names: List[str] = field(default_factory=list)   # buffers the call mutates (KV cache …)
    _plan: Any = field(default=None, repr=False)           # LaunchPlan of the bucket, recorded on demand

    def record_plan(self):
        """The bucket's :class:`~.launch_plan.LaunchPlan` (recorded by one more eager run of the example inputs — state
        buffers are written once more, like in the tracing run)."""
        if self._plan is None:
            from ..inference.launch_plan import LaunchPlan, record

            if isinstance(self.model, LaunchPlan):
                self._plan = self.model
            else:
                self._plan = record(self.model, [a.tensor for a in self.provided_args],
                                    [a.param_name for a in self.provided_args], call_with_kwargs=True)
        return self._plan

    # reference field names, so that generic code written against them keeps working
    @property
    def hlo(self) -> Dict[str, Any]:
        """The reference's traced program is an HLO module; here: the call description, plus the bucket's launch plan (JSON
        form, key ``"plan"``) once one was recorded."""
        d = self.describe()
        if self._plan is not None:
            d["plan"] = self._plan.to_json()
        return d

    @property
    def metaneff(self) -> Dict[str, Any]:
        return {"input_names": [a.param_name for a in self.provided_args], "weights": list(self.weight_name_to_idx),
                "states": list(self.state_names)}

    def input_signature(self) -> Tuple[Tuple[str, Tuple[int, ...], str], ...]:
        return tuple((a.param_name, tuple(a.tensor.shape), str(a.tensor.dtype)) for a in self.provided_args)

    def describe(self) -> Dict[str, Any]:
        name = type(self.model).__name__ if not callable(self.model) or hasattr(self.model, "forward") else \
            getattr(self.model, "__name__", "callable")
        return {"model": name, "inputs": self.input_signature(), "outputs": self.output_spec}

    def flattener(self, inputs):
        """Ordered tensor list → the same list (inputs are already flat tensors; kept as the reference's hook point)."""
        return list(inputs)

    def packer(self, outputs):
        return outputs


@dataclass
class CompilationArtifacts:
    """A runnable bucket: ``program(*ordered_inputs)``; ``graph`` is the captured CUDA graph (None → eager)."""
    program: Callable
    key: str = ""
    compiler_workdir: Optional[str] = None
    compiler_args: Optional[str] = None
    captured: bool = False
    plan: Any = None                                       # LaunchPlan the program interprets (None: the module itself runs)

    def get_neff_bytes(self) -> bytes:
        """The reference returns the NEFF file; the nearest H100 artefact is a description of the captured program."""
        return repr({"key": self.key, "captured_cuda_graph": self.captured, "args": self.compiler_args}).encode()


@dataclass
class WLOArtifacts(CompilationArtifacts):
    """Weight-layout-optimised compilation of the priority bucket (reference :92-104).  The reference lets the compiler
    pick weight layouts and extracts a transformer program from the HLO; here the bucket's launch plan is split by
    :meth:`LaunchPlan.hoist_weight_only`: everything that depends only on frozen weights (casts, transposes,
    de-quantisation, input-independent masks / tables) moves into ``transformer`` — run once per weight load — and
    ``plan`` (what the program interprets / what is captured into the CUDA graph) consumes its results."""
    transformer: Any = None
    layout_transform_map: Dict[str, List[str]] = field(default_factory=dict)


@dataclass
class LayoutTransformerArtifacts:
    """The weight → derived-weight programs of the compiled buckets (reference :127-157), keyed by bucket."""
    key: str = ModelBuilderConstants.LAYOUT_TRANSFORMER_KEY
    transformers: Dict[str, Any] = field(default_factory=dict)          # bucket key → (transformer plan, consumer plan)

    def construct_layout_transformer_object(self, local_ranks_size: int = 1):
        """Callable that re-derives the hoisted constants from the (already updated, in place) weights of every bucket."""
        pairs = list(self.transformers.values())

        def transform(weights=None):
            for transformer, main in pairs:
                main.apply_transformer(transformer)
            return weights

        return transform


def generate_key(trace_artifacts: TraceArtifacts, key: Optional[str] = None) -> str:
    """``key`` if given, else ``model_<hash of the bucket's input signature>`` (the reference hashes the HLO)."""
    if key is not None:
        return key
    h = hashlib.sha256(repr(trace_artifacts.input_signature()).encode()).hexdigest()[:8]
    return f"{ModelBuilderConstants.DEFAULT_KEY_PREFIX}_{h}"
