"""Program surgery for weight-layout optimisation (role of reference ``trace/hlo_utils.py``).

The reference rewrites HLO protobufs: it marks the priority bucket's weights as transposable, lets the compiler choose
layouts, extracts a "weight layout transformation" (WLT) program, re-points every other bucket at the transformed weights
and transforms the sharded checkpoint on CPU or on device.  The program representation here is the :class:`LaunchPlan`
(``inference/launch_plan.py``) — the recorded launch list of a bucket — and the same steps become plan passes:

=======================================  ================================================================================
reference (HLO)                          here (launch plan)
=======================================  ================================================================================
``read_hlo`` / ``write_hlo``             JSON load / save of a plan
``mark_weights_for_wlo``                 record the plan, store the skip set on the trace artifacts
``extract_weight_layout_transform_hlo``  ``LaunchPlan.hoist_weight_only`` → (transformer plan, per-call plan)
``get_layout_transform_map`` / ``get_wlt_map``  weight name → chain of hoisted ops / a callable applying the chain
``apply_layout_transformation``          hoist the same weight-only launches out of a non-priority bucket
``transform_weight_layout_on_cpu``       run the transformer over ``tp<r>_sharded_checkpoint.safetensors`` files
``prepare_parameter_usage_map`` …        ``LaunchPlan.weight_usage`` / ``kernel_weight_names`` (views are looked through)
=======================================  ================================================================================

What gets hoisted on H100 is not a compiler-chosen tiling (the wgmma GEMMs read K-major weights through TMA in every
bucket) but everything a bucket recomputes from frozen weights on each call: dtype casts, transposes that end in a copy,
de-quantisation of int8 / fp8 / MX weights, input-independent masks and rotary tables."""
from __future__ import annotations

import os
from typing import Any, Callable, Dict, List, Optional, Sequence, Set, Tuple

import torch

from ..inference.launch_plan import LaunchPlan, PlanError

TRANSPOSABLE_WEIGHT_IDX = "transposable_weight_idx"          # meta key (the reference's HLO frontend attribute)
# Where the layout transformer of a WLO build runs when its results are serialised ahead of time instead of being recomputed
# at every load (reference hlo_utils.py:36-38, read by ``ModelBuilder.transform_weight_layout_with_overriden_option``)
NXD_LAYOUT_TRANSFORMATION_OPTIONS = "NXD_LAYOUT_TRANSFORMATION_OPTIONS"           # environment variable
NXD_LAYOUT_ON_CPU_AND_SERIALIZE = "NXD_LAYOUT_ON_CPU_AND_SERIALIZE"
NXD_LAYOUT_ON_DEVICE_AND_SERIALIZE = "NXD_LAYOUT_ON_DEVICE_AND_SERIALIZE"


# ---- plans on disk ---------------------------------------------------------------------------------------------------------
def read_hlo(hlo_path: str) -> LaunchPlan:
    return LaunchPlan.load(hlo_path)


def write_hlo(hlo_path: str, hlo_module: LaunchPlan) -> None:
    os.makedirs(os.path.dirname(os.path.abspath(hlo_path)), exist_ok=True)
    hlo_module.save(hlo_path)


def _plan_of(obj: Any) -> LaunchPlan:
    if isinstance(obj, LaunchPlan):
        return obj
    if hasattr(obj, "record_plan"):
        return obj.record_plan()
    if getattr(obj, "plan", None) is not None:
        return obj.plan
    raise PlanError(f"no launch plan in {type(obj).__name__}")


# ---- marking ---------------------------------------------------------------------------------------------------------------
def add_weight_idx_attr_to_hlo(hlo: LaunchPlan, weight_name_to_idx: Dict[str, int], weight_names_to_skip: Optional[Set[str]] = None
                               ) -> LaunchPlan:
    """Store the indices of the weights that may be re-laid-out in the plan's metadata (skip list removed)."""
    idx = sorted(i for n, i in weight_name_to_idx.items() if n not in (weight_names_to_skip or ()))
    hlo.meta[TRANSPOSABLE_WEIGHT_IDX] = idx
    return hlo


def mark_weights_for_wlo(trace_artifacts: Any, weights_to_skip_layout_optimization: Optional[Set[str]] = None, **_) -> None:
    """Record the priority bucket's plan and note which weights the layout pass may touch."""
    skip = set(weights_to_skip_layout_optimization or ())
    invalid = skip - set(trace_artifacts.weight_name_to_idx)
    if invalid:
        raise RuntimeError(f"Weight layout optimization marking failed: Invalid weights in skip set: {invalid}")
    trace_artifacts.weight_names_to_skip = set(trace_artifacts.weight_names_to_skip) | skip
    add_weight_idx_attr_to_hlo(_plan_of(trace_artifacts), trace_artifacts.weight_name_to_idx, trace_artifacts.weight_names_to_skip)


# ---- extraction / application ---------------------------------------------------------------------------------------------
def extract_weight_layout_transform_hlo(hlo_stub: Any, weight_name_to_idx: Optional[Dict[str, int]] = None,
                                        weights_to_skip: Optional[Set[str]] = None, **_) -> Tuple[LaunchPlan, LaunchPlan]:
    """(transformer plan, per-call plan) of a bucket."""
    plan = _plan_of(hlo_stub)
    skip = set(weights_to_skip or ()) | set(getattr(hlo_stub, "weight_names_to_skip", ()) or ())
    transformer, main, tmap = plan.hoist_weight_only(skip)
    transformer.meta["layout_transform_map"] = tmap
    return transformer, main


def get_layout_transform_map(hlo_stub: Any, weight_name_to_idx: Optional[Dict[str, int]] = None) -> Dict[Any, List[str]]:
    """Weight → names of the hoisted ops that start from it.  Keys are weight indices when ``weight_name_to_idx`` is given
    (the reference keys by parameter number), else weight names."""
    if isinstance(hlo_stub, LaunchPlan) and "layout_transform_map" in hlo_stub.meta:
        tmap = hlo_stub.meta["layout_transform_map"]
    elif getattr(hlo_stub, "layout_transform_map", None):
        tmap = hlo_stub.layout_transform_map
    else:
        tmap = _plan_of(hlo_stub).hoist_weight_only(getattr(hlo_stub, "weight_names_to_skip", ()) or ())[2]
    if weight_name_to_idx:
        return {weight_name_to_idx[n]: ops for n, ops in tmap.items() if n in weight_name_to_idx}
    return dict(tmap)


def get_wlt(transformer: LaunchPlan, weight_name: str) -> Optional[Callable[[torch.Tensor], List[torch.Tensor]]]:
    """Callable ``weight → [derived tensors]`` for the hoisted launches that depend on ``weight_name`` ONLY (None when the
    weight is not transformed, or only together with other constants)."""
    wid = next((i for i, c in transformer.constants.items() if c.name == weight_name), None)
    if wid is None:
        return None
    reach: Set[int] = {wid}
    nodes = []
    for n in transformer.nodes:
        ins = set(n.inputs())
        if ins and ins <= reach:
            nodes.append(n)
            reach.update(o for o in n.outs if o is not None)
    wanted = [v for v in transformer.meta.get("derived_ids", []) if v in reach and v != wid]
    if not wanted:
        return None

    def apply(weight: torch.Tensor) -> List[torch.Tensor]:
        sub = LaunchPlan(nodes, [{"id": wid, "name": weight_name, "shape": list(weight.shape), "dtype": str(weight.dtype)}],
                         {"l": [{"t": v} for v in wanted]}, {}, weight.device.type, dict(transformer.meta))
        sub.device = weight.device
        return sub.run(weight)

    return apply


def get_wlt_map(hlo: LaunchPlan) -> Dict[str, Callable]:
    out = {}
    for c in hlo.constants.values():
        f = get_wlt(hlo, c.name)
        if f is not None:
            out[c.name] = f
    return out


def apply_layout_transformation(trace_artifacts: Any, priority_model_trace_artifacts: Any = None, wlo_artifacts: Any = None,
                                key: Optional[str] = None, **_) -> Tuple[LaunchPlan, LaunchPlan]:
    """Non-priority bucket: hoist its weight-only launches too, honouring the priority bucket's skip set.  Returns
    (transformer, per-call plan) and stores the per-call plan on the trace artifacts, so that a following ``compile`` captures
    the reduced launch list."""
    skip = set(getattr(trace_artifacts, "weight_names_to_skip", ()) or ())
    if priority_model_trace_artifacts is not None:
        skip |= set(getattr(priority_model_trace_artifacts, "weight_names_to_skip", ()) or ())
    transformer, main, tmap = _plan_of(trace_artifacts).hoist_weight_only(skip)
    main.apply_transformer(transformer)
    transformer.meta["layout_transform_map"] = tmap
    if hasattr(trace_artifacts, "_plan"):
        trace_artifacts._plan = main
    return transformer, main


def append_layout_computation_to_hlo(hlo: LaunchPlan, transformer: LaunchPlan) -> LaunchPlan:
    """Inverse of the extraction: one plan that runs the transformer's launches and then the per-call ones."""
    derived = set(transformer.meta.get("derived_ids", []))
    consts = {i: c for i, c in hlo.constants.items() if i not in derived}
    consts.update(transformer.constants)
    merged = LaunchPlan(list(transformer.nodes) + list(hlo.nodes), list(hlo.inputs), hlo.outputs, consts, hlo.device_type,
                        {k: v for k, v in hlo.meta.items() if k != "derived_ids"})
    merged.tensors = {i: t for i, t in {**hlo.tensors, **transformer.tensors}.items() if i in consts}
    merged.device = hlo.device
    return merged


def update_computation_id_and_name(*args, **kwargs):
    raise NotImplementedError("launch plans have one value-id space per bucket; there are no computations to renumber")


def prepare_metaneff_for_wlt_hlo(wlt_hlo: LaunchPlan, *args, **kwargs) -> Dict[str, Any]:
    """Input / output description of a transformer plan (the reference builds a metaneff proto for it)."""
    return {"inputs": [(c.name, tuple(c.shape), c.dtype) for c in wlt_hlo.constants.values()],
            "outputs": [f"_derived_{v}" for v in wlt_hlo.meta.get("derived_ids", [])]}


def read_metaneff(metaneff_path: str) -> Dict[str, Any]:
    import json

    with open(metaneff_path) as f:
        return json.load(f)


def get_input_order(metaneff: Any) -> Any:
    """Trace artifacts → input names in call order; a plan → (constant names, shapes), the reference's return shape."""
    if isinstance(metaneff, LaunchPlan):
        return [c.name for c in metaneff.constants.values()], [tuple(c.shape) for c in metaneff.constants.values()]
    return [a.param_name for a in metaneff.provided_args]


# ---- transforming checkpoints ------------------------------------------------------------------------------------------------
def update_weight(weights: Dict[str, torch.Tensor], transformer: Optional[LaunchPlan] = None, **_) -> Dict[str, torch.Tensor]:
    """``weights`` plus the transformer's derived tensors (``_derived_<id>``), computed from ``weights``."""
    if transformer is None:
        return weights
    t = LaunchPlan(transformer.nodes, [], transformer.outputs, transformer.constants, transformer.device_type, dict(transformer.meta))
    t.tensors = dict(transformer.tensors)
    t.bind({k: v for k, v in weights.items()}, strict=False)
    t.device = next(iter(weights.values())).device if weights else transformer.device
    out = dict(weights)
    for vid, val in zip(t.meta.get("derived_ids", []), t.run()):
        out[f"_derived_{vid}"] = val
    return out


def transform_weight_layout_on_cpu(hlo_filename: Any, metaneff_filename: Any = None, start_rank_id: int = 0, local_ranks_size: int = 1,
                                   sharded_checkpoint_dir: Optional[str] = None, device: Optional[torch.device] = None
                                   ) -> Dict[int, Dict[str, torch.Tensor]]:
    """Run a transformer plan (path or object) over ``tp<r>_sharded_checkpoint.safetensors`` of the given ranks and write the
    derived tensors next to the weights (``tp<r>_derived.safetensors``), so that loading does not have to recompute them."""
    from ..utils.safetensors_utils import load_state_dict_safetensors, save_state_dict_safetensors

    transformer = hlo_filename if isinstance(hlo_filename, LaunchPlan) else read_hlo(hlo_filename)
    done: Dict[int, Dict[str, torch.Tensor]] = {}
    for rank in range(start_rank_id, start_rank_id + local_ranks_size):
        ckpt = load_state_dict_safetensors(os.path.join(sharded_checkpoint_dir, f"tp{rank}_sharded_checkpoint.safetensors"))
        if device is not None:
            ckpt = {k: v.to(device) for k, v in ckpt.items()}
        full = update_weight(ckpt, transformer)
        derived = {k: v.cpu().contiguous() for k, v in full.items() if k.startswith("_derived_")}
        save_state_dict_safetensors(derived, os.path.join(sharded_checkpoint_dir, f"tp{rank}_derived.safetensors"))
        done[rank] = derived
    return done


def transform_weight_layout_on_device_and_save_to_disk(metaneff_filename: Any, start_rank_id: int, local_ranks_size: int,
                                                       wlt_neff_path: Any, sharded_checkpoint_dir: str) -> None:
    """Same transformation with the shard moved to this process's GPU for the run (de-quantisation / casts of a large shard are
    bandwidth-bound: HBM instead of host memory); results are brought back and written next to the shard."""
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None
    transform_weight_layout_on_cpu(wlt_neff_path, metaneff_filename, start_rank_id, local_ranks_size, sharded_checkpoint_dir, device=dev)


def convert_inputs_to_optimal_shape(inputs, *args, **kwargs):
    return inputs                                              # buckets take their inputs in the traced shapes


def cleanup_after_layout_transformation(trace_artifacts: Any = None, *args, **kwargs) -> None:
    if trace_artifacts is not None and isinstance(getattr(trace_artifacts, "_plan", None), LaunchPlan):
        trace_artifacts._plan.meta.pop(TRANSPOSABLE_WEIGHT_IDX, None)


# ---- toolchain ----------------------------------------------------------------------------------------------------------------
def get_compiler_package_dir() -> str:
    return os.environ.get("CUDA_HOME", "/usr/local/cuda")


def get_executable_full_qualified_path(executable: str = "nvcc") -> Optional[str]:
    import shutil

    return shutil.which(executable) or (os.path.join(get_compiler_package_dir(), "bin", executable)
                                        if os.path.exists(os.path.join(get_compiler_package_dir(), "bin", executable)) else None)


# ---- usage analysis ------------------------------------------------------------------------------------------------------------
def is_nki_kernel_called(plan: Any, node_index: Optional[int] = None) -> bool:
    """Does the plan (or its node ``node_index``) launch a hand-written extension kernel / fused framework op?"""
    p = _plan_of(plan)
    if node_index is not None:
        return p.nodes[node_index].kind != "op"
    return any(n.kind != "op" for n in p.nodes)


def prepare_parameter_usage_map(plan: Any, parameters_list: Optional[Sequence[str]] = None) -> Dict[str, List[int]]:
    """Constant name → indices of the nodes that consume it (through views)."""
    use = _plan_of(plan).weight_usage()
    return {k: [i for i, _ in v] for k, v in use.items() if parameters_list is None or k in parameters_list}


def traceback_instruction_to_parameter(plan: Any, value_id: int, traced: Optional[Set[int]] = None) -> Optional[str]:
    """Follow a value back through view ops to the constant it aliases; its name, or None."""
    p = _plan_of(plan)
    root = p._roots().get(value_id, value_id)
    return p.constants[root].name if root in p.constants else None


def get_nki_kernel_weight_names(plan: Any, *args, **kwargs) -> Set[str]:
    """Weights that feed extension kernels / fused ops directly (the reference keeps those out of the layout pass because the
    kernel fixes their layout; hoisting is value-preserving here, so this is informational)."""
    return set(_plan_of(plan).kernel_weight_names())

