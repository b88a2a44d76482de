"""v0 inference API + checkpoint-sharding helpers (reference ``trace/trace.py:62-825``).

``parallel_model_trace(func, example_inputs, tp_degree=…)`` returns a :class:`ParallelModel`; on H100 each rank is its own
``torchrun`` process, so the returned wrapper holds THIS rank's captured program (the reference's wrapper holds one traced
model per rank inside a single process)."""
from __future__ import annotations

import os
import warnings
from typing import Any, Callable, Dict, List, Optional, Sequence

import torch
from torch import nn

from ..inference.sharding import shard_tensor
from ..parallel_layers.utils import create_local_weight as _create_local_weight
from ..parallel_layers.utils import divide
from ..utils.safetensors_utils import check_for_duplicate_tensors


class ParallelModel(nn.Module):
    """Base class of the traced-model wrappers."""

    def __init__(self):
        super().__init__()
        self.load = False


class TensorParallelNeuronModel(ParallelModel):
    """Wrapper over per-rank traced models (reference :67-123).  ``models`` holds the local rank's program(s); calling the
    wrapper runs the first one (all ranks of a TP group return identical outputs after the final gather/reduce)."""

    def __init__(self, models: Sequence[Callable]):
        super().__init__()
        self.models = list(models)
        self.load = True

    def forward(self, *tensors):
        return self.models[0](*tensors)


def collect_tp_neuron_models(models, mp_q=None, bucket_config=None, tp_degree: int = 1) -> TensorParallelNeuronModel:
    return TensorParallelNeuronModel(models)


collect_tp_bucket_neuron_models = collect_tp_neuron_models


def generate_ranked_folder(tp_rank: int, bucket_rank: int, bucket_degree: int) -> str:
    """Sub-directory name of one (tp rank, bucket) traced artefact."""
    return f"tp_{tp_rank}" if bucket_degree <= 1 else f"tp_{tp_rank}_bk_{bucket_rank}"


def find_unique_dtypes(model: nn.Module) -> Dict[torch.dtype, int]:
    """``{dtype: parameter count}`` — used to sanity-check that a model was cast before tracing."""
    out: Dict[torch.dtype, int] = {}
    for p in model.parameters():
        out[p.dtype] = out.get(p.dtype, 0) + 1
    return out


# ---------------------------------------------------------------------------------------------------------------------
# checkpoint sharding (reference :628-825)
# ---------------------------------------------------------------------------------------------------------------------
def invoke_preshard_hook(module: Optional[nn.Module], checkpoint: Dict[str, Any], prefix: str) -> None:
    """Depth-first: the first module on a path that defines ``preshard_hook`` handles its whole subtree (GQA K/V
    replication, QKV fusion, padding, SPMD-rank entries …)."""
    if module is None:
        return
    hook = getattr(module, "preshard_hook", None)
    if hook is not None:
        for leaf in ("weight", "bias") if getattr(module, "add_bias", False) or getattr(module, "bias", None) is not None else ("weight",):
            try:
                hook(checkpoint, prefix + leaf)
            except KeyError:
                pass
        return
    for name, child in module._modules.items():
        if child is not None:
            invoke_preshard_hook(child, checkpoint, prefix + name + ".")


def preprocess_checkpoint(model: nn.Module, checkpoint: Dict[str, Any]) -> None:
    """In place: warn about shared tensors, run preshard hooks, fold LoRA updates, drop keys the model does not have."""
    check_for_duplicate_tensors(checkpoint, False)
    invoke_preshard_hook(model, checkpoint, "")
    if hasattr(model, "lora_wrapped_model") and hasattr(model, "update_weights_for_lora"):
        updated = model.update_weights_for_lora(checkpoint)
        if updated is not None and updated is not checkpoint:
            checkpoint.clear()
            checkpoint.update(updated)
    known = set(model.state_dict().keys())
    hooked = {n[: n.rfind(".") + 1] for n, p in model.named_parameters() if hasattr(p, "get_tensor_from_state_dict")}
    extra = [k for k in checkpoint if k not in known and not any(k.startswith(h) for h in hooked)]
    if extra:
        warnings.warn(f"Removing redundant keys from checkpoint: {extra}")
    for k in extra:
        checkpoint.pop(k, None)


def create_local_weight(rank: int, world_size: int, full_weight: torch.Tensor, partition_dim: int, per_partition_size: int,
                        stride: int, out_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Reference argument order (rank first); see ``parallel_layers.utils.create_local_weight``."""
    return _create_local_weight(full_weight, partition_dim, per_partition_size, stride, out_weight, rank=rank, world_size=world_size)


def create_local_weight_qkv(rank: int, world_size: int, full_weight: torch.Tensor, partition_dim: int, q_len: int, kv_len: int,
                            out_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Shard a ``[Q; K; V]``-concatenated tensor section by section so rank r gets ``[Q_r; K_r; V_r]``."""
    q, k, v = torch.split(full_weight, [q_len, kv_len, kv_len], dim=partition_dim)
    parts = [t.narrow(partition_dim, rank * divide(n, world_size), divide(n, world_size)) for t, n in ((q, q_len), (k, kv_len), (v, kv_len))]
    with torch.no_grad():
        res = torch.cat(parts, dim=partition_dim)
        if out_weight is not None:
            out_weight.copy_(res)
            return out_weight
        return res


def create_local_weight_with_expert_parallel(rank: int, world_size: int, full_weight: torch.Tensor, partition_dim: int,
                                             per_partition_size: int, stride: int, local_expert_indices, tensor_dtype=None,
                                             out_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    local = create_local_weight(rank, world_size, full_weight, partition_dim, per_partition_size, stride, out_weight)
    if local_expert_indices is None:
        return local
    idx = torch.as_tensor(list(local_expert_indices), dtype=torch.long)
    if local.dtype in (torch.float8_e4m3fn, torch.float8_e5m2):
        return local.view(torch.int8)[idx].view(local.dtype)
    if local.dtype == torch.uint16:
        return local.view(torch.int16)[idx].view(local.dtype)
    return local[idx]


def shard_children(module: Optional[nn.Module], checkpoint: Dict[str, Any], prefix: str, dtype: Optional[torch.dtype], rank: int,
                   tp_degree: int, is_lora_cpu_shard: bool = False) -> None:
    """In place: replace every entry of ``checkpoint`` that belongs to a parameter under ``module`` by rank ``rank``'s
    shard, according to the parameter's parallel attributes (TP partition dim / stride / rank ordering, expert
    parallelism, ``get_tensor_from_state_dict`` hooks).  Raises if a shard's shape differs from the parameter's."""
    if module is None:
        return
    for name, p in module.named_parameters():
        key = prefix + name
        getter = getattr(p, "get_tensor_from_state_dict", None)
        if getter is not None and not is_lora_cpu_shard:
            try:
                tensor = getter(prefix=key[: key.rfind(".") + 1], state_dict=checkpoint)
            except (RuntimeError, KeyError):
                tensor = checkpoint.get(key)
        else:
            tensor = checkpoint.get(key)
        if tensor is None:
            continue
        local = shard_tensor(tensor, p, rank, tp_degree)
        if dtype is not None and local.is_floating_point() and p.is_floating_point() and local.dtype != p.dtype \
                and local.element_size() > 1 and p.element_size() > 1:
            local = local.to(dtype)
        if tuple(local.shape) != tuple(p.shape) and not is_lora_cpu_shard:
            raise RuntimeError(f"expected shape {tuple(p.shape)} for {key} but found {tuple(local.shape)}")
        checkpoint[key] = local


def get_sharded_checkpoint(checkpoint: Dict[str, Any], model: nn.Module, rank: int, tp_degree: int, is_cached: bool = False) -> None:
    """In place: turn a full checkpoint into rank ``rank``'s shard (reference :646-656).  ``is_cached`` skips the
    preprocessing when the same (already pre-processed) checkpoint is sharded for several ranks in a row — note that the
    dict is overwritten with shards, so pass a copy per rank."""
    if not is_cached:
        preprocess_checkpoint(model, checkpoint)
    dtype = getattr(getattr(model, "config", None), "torch_dtype", None)
    shard_children(model, checkpoint, "", dtype, rank, tp_degree)


# ---- v0 entry points (reference :242-371).  A "traced parallel model" is the per-rank module plus its captured bucket programs;
# every rank is its own process (torchrun) instead of being spawned by the library. ---------------------------------------------
def parallel_model_trace(func: Callable[[], Any], example_inputs: Any, tp_degree: int = 1, **kwargs):
    from .model_builder import ModelBuilder

    module, _aliases = func()
    ex = example_inputs if isinstance(example_inputs, (tuple, list)) else (example_inputs,)
    return ModelBuilder(tp_degree=tp_degree).add("main", module, [tuple(ex)]).trace()


def parallel_model_save(model, save_dir: str) -> None:
    model.save(save_dir, save_weights=True)


def parallel_model_load(model_dir: str) -> Any:
    load_dir = model_dir      # reference parameter names in the signature
    return torch.load(os.path.join(load_dir, "nxd_model_meta.pt"), weights_only=False)
