"""``ModelBuilder`` — register per-bucket step functions and "compile" them.

Reference (``trace/model_builder.py:441-1369``, ``model_builder_v2.py:33-319``): XLA-trace each bucket (context
encoding / token generation / speculation) to HLO → neuronx-cc → NEFF, optimise weight layout across buckets, build
a state (KV cache) initialiser, write per-rank sharded safetensors.  On H100 "compile" means: run every bucket's step
once to warm up allocators/NCCL, then capture it into a CUDA graph with persistent input/output/state buffers;
weights are shared by all buckets by construction (same parameter tensors), so no layout pass is needed.
``shard_checkpoint`` keeps the reference's output format: ``tp{rank}_sharded_checkpoint.safetensors``."""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

from ..inference.sharding import shard_state_dict_for_rank
from .functions import append_default_compiler_flags, compile, compile_layout_transformer, compile_wlo, trace  # noqa: F401,A004
from .nxd_model import BucketProgram, NxDModel


@dataclass
class BaseModelInstance:
    """Factory + aliasing info for one traced key (reference model_builder.py:46-64)."""
    module_cls: Callable[[], nn.Module]
    input_output_aliases: Dict[Any, Any] = field(default_factory=dict)
    module: Optional[nn.Module] = None

    def load_module(self) -> None:
        if self.module is None:
            self.module = self.module_cls()

    def get(self, bucket_rank: int = 0, **kwargs) -> Tuple[nn.Module, Dict]:
        self.load_module()
        return self.module, self.input_output_aliases


class ModelBuilder:
    def __init__(self, router: Any = None, tp_degree: int = 1, checkpoint_loader: Optional[Callable[[], Dict[str, torch.Tensor]]] = None,
                 start_rank_id: int = 0, pp_degree: int = 1, ep_degree: int = 1, local_ranks_size: Optional[int] = None,
                 world_size: Optional[int] = None, compiler_workdir: Optional[str] = None, master_proc_env_vars: Optional[Dict] = None,
                 debug: bool = False, num_cores_per_group: int = 1, init_custom_process_group_fn: Optional[Callable] = None,
                 logical_nc_config: int = 1, weights_to_skip_layout_optimization=None, compiler_flag_hook: Optional[Callable] = None,
                 model: Optional[nn.Module] = None, use_cuda_graphs: Optional[bool] = None):
        """Positional order of reference model_builder.py:230-249.  ``master_proc_env_vars`` (environment of the reference's
        per-rank compile workers), ``init_custom_process_group_fn`` (called once here, right away: this process IS the rank) and
        ``compiler_flag_hook`` (there is no compiler command line) are accepted for source compatibility."""
        if master_proc_env_vars:
            os.environ.update({str(k): str(v) for k, v in master_proc_env_vars.items()})
        if init_custom_process_group_fn is not None:
            init_custom_process_group_fn()
        self.compiler_flag_hook = compiler_flag_hook
        self.router, self.tp_degree, self.checkpoint_loader = router, tp_degree, checkpoint_loader
        self.world_size = world_size or tp_degree * pp_degree
        self.start_rank_id, self.local_ranks_size = start_rank_id, local_ranks_size
        self.model = model
        self.entries: Dict[str, Dict[str, Any]] = {}
        self.use_cuda_graphs = torch.cuda.is_available() if use_cuda_graphs is None else use_cuda_graphs

    def add(self, key: str, model_instance: Any, example_inputs: Sequence[Tuple[torch.Tensor, ...]],
            compiler_args: Any = None, bucket_config: Any = None, priority_model_idx: Optional[int] = None,
            step_fn: Optional[Callable] = None) -> "ModelBuilder":
        """``example_inputs``: one tuple of tensors per bucket.  ``model_instance``: a module, a ``BaseModelInstance`` or
        any callable; ``step_fn(module, *inputs)`` overrides how the bucket is executed."""
        self.entries[key] = {"instance": model_instance, "examples": list(example_inputs), "step_fn": step_fn,
                             "priority": priority_model_idx}
        return self

    def trace(self, initialize_model_weights: bool = True, dry_run: bool = False, disable_fail_fast: bool = False,
              tag: Optional[str] = None) -> NxDModel:
        """Positional order of reference model_builder.py:394.  ``dry_run``: build every bucket program (validates that the
        entries are callable on their example shapes' metadata) but load no weights; ``disable_fail_fast`` concerned the
        reference's parallel compile workers."""
        if isinstance(initialize_model_weights, str):                       # earlier form of this package: trace(tag)
            initialize_model_weights, tag = True, initialize_model_weights
        if dry_run:
            initialize_model_weights = False
        nxd = NxDModel(world_size=self.world_size, router=self.router)
        for key, e in self.entries.items():
            inst = e["instance"]
            if isinstance(inst, BaseModelInstance):
                module, _ = inst.get()
            else:
                module = inst
            fn = e["step_fn"] or (lambda m, *a: m(*a))
            for ex in e["examples"]:
                prog = BucketProgram(key, module, fn, tuple(ex), use_cuda_graph=self.use_cuda_graphs)
                nxd.add_program(prog)
        if initialize_model_weights and self.checkpoint_loader is not None and self.model is not None:
            from ..parallel_layers import parallel_state as ps

            sd = shard_state_dict_for_rank(self.model, self.checkpoint_loader(), ps.get_tensor_model_parallel_rank(),
                                           ps.get_tensor_model_parallel_size())
            self.model.load_state_dict(sd, strict=False)
        return nxd

    compile = trace

    # ---- pieces of the v1 build exposed by the reference (model_builder.py:700-1369) -------------------------------------
    def build_nxd_model(self) -> NxDModel:
        return self.trace()

    def build_state_initializer(self):
        """State (KV-cache) buffers = the registered buffers of the bucket modules; returns an initialiser that re-creates
        them zero-filled (shapes / dtypes are taken from the live buffers)."""
        from .nxd_model import StateInitializer

        shapes, dtypes = {}, {}
        for e in self.entries.values():
            inst = e["instance"]
            module = inst.get()[0] if isinstance(inst, BaseModelInstance) else inst
            if isinstance(module, nn.Module):
                for n, b in module.named_buffers():
                    shapes[n], dtypes[n] = list(b.shape), b.dtype
        return StateInitializer(shapes, dtypes, 1) if shapes else None

    def build_flattener_map(self) -> Dict[str, Callable]:
        return {f"{k}_{i}": (lambda inputs: list(inputs)) for k, e in self.entries.items() for i in range(len(e["examples"]))}

    def build_packer(self) -> Callable:
        return lambda outputs: outputs

    def shard_weights(self, rank: int, model_container: Any = None, serialize_path: Optional[str] = None) -> Dict[str, torch.Tensor]:
        """Rank ``rank``'s shard of the checkpoint returned by ``checkpoint_loader`` (preshard hooks applied)."""
        assert self.checkpoint_loader is not None, "a checkpoint_loader is required"
        model = self.model
        if model is None and model_container is not None:
            inst = getattr(model_container, "model_instance", model_container)
            model = inst.get()[0] if isinstance(inst, BaseModelInstance) else inst
        assert model is not None, "no model to take the parallel attributes from"
        return shard_checkpoint(self.checkpoint_loader(), model, self.tp_degree, start_rank=rank, end_rank=rank,
                                serialize_path=serialize_path)[0]

    def shard_weights_with_cache(self, rank: int, model_container: Any = None, serialize_path: Optional[str] = None):
        """Same as :meth:`shard_weights` but pre-processes (hooks, key clean-up) the full checkpoint only once."""
        if not hasattr(self, "_ckpt_cache"):
            self._ckpt_cache = self.checkpoint_loader()
        loader, self.checkpoint_loader = self.checkpoint_loader, (lambda: dict(self._ckpt_cache))
        try:
            return self.shard_weights(rank, model_container, serialize_path)
        finally:
            self.checkpoint_loader = loader

    @staticmethod
    def cast_weights(checkpoint: Dict[str, torch.Tensor], model: nn.Module) -> Dict[str, torch.Tensor]:
        """Cast floating checkpoint tensors to the dtype of the parameter they load into (bf16 models from fp32 files)."""
        params = dict(model.named_parameters())
        for k, v in list(checkpoint.items()):
            p = params.get(k)
            if p is not None and isinstance(v, torch.Tensor) and v.is_floating_point() and p.is_floating_point() \
                    and v.dtype != p.dtype and v.element_size() > 1 and p.element_size() > 1:
                checkpoint[k] = v.to(p.dtype)
        return checkpoint

    def write_neff_to_file(self, nxd_model: NxDModel, path: str) -> None:
        """The reference dumps the compiled NEFFs; the analogue here is the bucket description of the runtime model."""
        os.makedirs(path, exist_ok=True)
        with open(os.path.join(path, "programs.txt"), "w") as f:
            for k, progs in nxd_model.programs.items():
                for p in progs:
                    f.write(f"{k}: shapes={p.shapes} dtypes={p.dtypes} cuda_graph={p.graph is not None}\n")

    def transform_weight_layout_with_overriden_option(self, sharded_checkpoint_dir: str, transformer: Any = None,
                                                      option: Optional[str] = None) -> Optional[Dict[int, Dict[str, torch.Tensor]]]:
        """Run the layout transformer of a WLO build (``compile_wlo`` → ``WLOArtifacts.transformer``, a plan object or its path)
        over the rank shards in ``sharded_checkpoint_dir`` AHEAD of time and serialise the derived tensors
        (``tp<r>_derived.safetensors``) so that loading does not recompute them (reference model_builder.py:1330-1369).
        ``option`` / ``$NXD_LAYOUT_TRANSFORMATION_OPTIONS``: ``NXD_LAYOUT_ON_CPU_AND_SERIALIZE`` or
        ``NXD_LAYOUT_ON_DEVICE_AND_SERIALIZE``; unset → nothing is done (transform at load, the default flow)."""
        from . import hlo_utils

        option = option or os.environ.get(hlo_utils.NXD_LAYOUT_TRANSFORMATION_OPTIONS)
        if option is None:
            return None
        if transformer is None:
            raise ValueError("a layout transformer (WLOArtifacts.transformer or its file) is required")
        start, n = getattr(self, "start_rank_id", 0), getattr(self, "local_ranks_size", None) or self.tp_degree
        if option == hlo_utils.NXD_LAYOUT_ON_CPU_AND_SERIALIZE:
            return hlo_utils.transform_weight_layout_on_cpu(transformer, None, start, n, sharded_checkpoint_dir)
        if option == hlo_utils.NXD_LAYOUT_ON_DEVICE_AND_SERIALIZE:
            hlo_utils.transform_weight_layout_on_device_and_save_to_disk(None, start, n, transformer, sharded_checkpoint_dir)
            return None
        raise ValueError(f"Unknown layout option: {option}")

    def shard_checkpoint(self, serialize_path: Optional[str] = None) -> List[Dict[str, torch.Tensor]]:
        assert self.model is not None and self.checkpoint_loader is not None
        return shard_checkpoint(self.checkpoint_loader(), self.model, self.tp_degree, serialize_path=serialize_path)


def shard_checkpoint(checkpoint: Dict[str, torch.Tensor], model: nn.Module, tp_degree: Optional[int] = None,
                     start_rank: int = 0, end_rank: Optional[int] = None, load_on_device: bool = False,
                     serialize_path: Optional[str] = None) -> List[Dict[str, torch.Tensor]]:
    """Shard a full checkpoint for ranks ``[start_rank, end_rank]`` using the model's parallel attributes; optionally
    write ``tp{rank}_sharded_checkpoint.safetensors`` (reference trace/functions.py:880-908)."""
    from ..parallel_layers import parallel_state as ps
    from ..utils.safetensors_utils import save_state_dict_safetensors

    tp = tp_degree or ps.get_tensor_model_parallel_size()
    end_rank = tp - 1 if end_rank is None else end_rank
    out = []
    for r in range(start_rank, end_rank + 1):
        sd = shard_state_dict_for_rank(model, checkpoint, r, tp)
        sd = {k: v.contiguous() for k, v in sd.items() if isinstance(v, torch.Tensor)}
        if serialize_path is not None:
            os.makedirs(serialize_path, exist_ok=True)
            save_state_dict_safetensors(sd, os.path.join(serialize_path, f"tp{r}_sharded_checkpoint.safetensors"))
        out.append(sd)
    return out


class ModelContainer:
    """One registered key of the v1 builder: the model instance, its example inputs (one tuple per bucket) and the per-key
    options (reference :66-83)."""

    def __init__(self, model_instance, example_inputs, compiler_args=None, bucket_config=None, priority_model_idx=None):
        self.model_instance, self.example_inputs = model_instance, example_inputs
        self.compiler_args, self.bucket_config, self.priority_model_idx = compiler_args, bucket_config, priority_model_idx
        self.traced = None


class JITWrapper:
    """Reference :85-95 wraps a Python callable for TorchScript; callables need no wrapping to be captured here."""

    def __init__(self, func, is_torchscript: bool = False):
        self.func = func

    def __call__(self, inputs):
        return self.func(inputs)


def get_hash_module(module_description) -> str:
    import hashlib

    return hashlib.sha256(repr(module_description).encode()).hexdigest()


def init_process_wrapper(*args, **kwargs):
    """The reference spawns one worker process per rank for tracing; ranks are ``torchrun`` processes here."""
    raise RuntimeError("launch one process per GPU with torchrun; the builder does not spawn workers")
