"""Model construction helpers: meta-device init, staggered materialisation, attribute
preservation (reference ``utils/model_utils.py:147-386``)."""
from __future__ import annotations

import contextlib
import math
from typing import Callable, Dict, Optional

import torch
import torch.distributed as dist
from torch import nn

from ..utils import cpu_mode, get_device
from ..utils.logger import get_logger


logger = get_logger()


def move_model_to_device(model: nn.Module, device: Optional[torch.device] = None) -> nn.Module:
    """Reference ``utils/model_utils.py`` re-exports this helper; the implementation lives with the TP utilities."""
    from ..parallel_layers.utils import move_model_to_device as _move

    return _move(model, device)

_PARALLEL_ATTRS = ("tensor_model_parallel", "partition_dim", "partition_stride", "num_partitions", "rank_ordering",
                   "sequence_parallel_enabled", "shared", "expert_model_parallel", "fused_qkv", "qkv_sections")


def is_hf_pretrained_model(model) -> bool:
    try:
        from transformers import PreTrainedModel

        return isinstance(model, PreTrainedModel)
    except Exception:
        return False


def is_nxd_pipeline_model(model) -> bool:
    try:
        from ..pipeline.model import NxDPPModel

        return isinstance(model, NxDPPModel)
    except Exception:
        return False


@contextlib.contextmanager
def init_on_device(device: torch.device, include_buffers: bool = False, force_custom_init_on_device: bool = False):
    """Create parameters (and optionally buffers) directly on ``device`` (typically ``meta``) while
    keeping the parallel attributes set by the TP layers (reference :147-213).  This is always the "custom" implementation of
    the reference (it keeps ``requires_grad=False`` and the parallel attributes, which the accelerate one loses), so
    ``force_custom_init_on_device`` changes nothing."""
    old_register_parameter = nn.Module.register_parameter
    old_register_buffer = nn.Module.register_buffer

    def register_parameter(module, name, param):
        old_register_parameter(module, name, param)
        if param is not None:
            cur = module._parameters[name]
            attrs = dict(cur.__dict__)
            new = nn.Parameter(cur.to(device), requires_grad=cur.requires_grad)
            new.__dict__.update(attrs)
            module._parameters[name] = new

    def register_buffer(module, name, buf, persistent=True):
        old_register_buffer(module, name, buf, persistent=persistent)
        if buf is not None:
            module._buffers[name] = module._buffers[name].to(device)

    try:
        nn.Module.register_parameter = register_parameter
        if include_buffers:
            nn.Module.register_buffer = register_buffer
        yield
    finally:
        nn.Module.register_parameter = old_register_parameter
        nn.Module.register_buffer = old_register_buffer


class _SavedParallelAttributes(dict):
    """``{param_name: {attr: value}}`` that can also be used as ``with preserve_parallel_attributes(model): …`` — the
    attributes are written back on exit (operations such as ``to_empty`` / re-materialisation create new Parameter
    objects and drop custom attributes; reference :164-202 is a context manager)."""

    def __init__(self, model: nn.Module, data: Dict[str, Dict]):
        super().__init__(data)
        self._model = model

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        restore_parallel_attributes(self._model, self)
        return False


def preserve_parallel_attributes(model: nn.Module) -> _SavedParallelAttributes:
    return _SavedParallelAttributes(
        model, {n: {k: v for k, v in p.__dict__.items() if k in _PARALLEL_ATTRS} for n, p in model.named_parameters()})


def restore_parallel_attributes(model: nn.Module, saved: Dict[str, Dict]) -> None:
    for n, p in model.named_parameters():
        for k, v in saved.get(n, {}).items():
            setattr(p, k, v)


def get_tied_parameters(model: nn.Module):
    seen: Dict[int, str] = {}
    tied = []
    for name, p in model.named_parameters(remove_duplicate=False):
        if id(p) in seen:
            tied.append((seen[id(p)], name))
        else:
            seen[id(p)] = name
    return tied


def reinit_model(model: nn.Module, device: torch.device, param_init_fn: Optional[Callable]) -> None:
    """Materialise a meta-device model on ``device`` and (re-)initialise every module with
    ``param_init_fn(module, device)``; tied parameters stay tied (reference :276-332)."""
    saved = preserve_parallel_attributes(model)
    tied = get_tied_parameters(model)
    for module in model.modules():
        has_meta = any(p.device.type == "meta" for p in module.parameters(recurse=False)) or any(
            b.device.type == "meta" for b in module.buffers(recurse=False))
        if not has_meta:
            continue
        module.to_empty(device=device, recurse=False)
        if param_init_fn is not None:
            param_init_fn(module, device)
        elif hasattr(module, "reset_parameters"):
            module.reset_parameters()
    restore_parallel_attributes(model, saved)
    mods = dict(model.named_modules())
    for a, b in tied:
        pa, na = a.rsplit(".", 1) if "." in a else ("", a)
        pb, nb = b.rsplit(".", 1) if "." in b else ("", b)
        setattr(mods[pb], nb, getattr(mods[pa], na))


def get_model_sequential(model, device=None, sequential_move_factor: int = 11, param_init_fn: Optional[Callable] = None,
                         move_to_device: bool = True) -> nn.Module:
    """Bring a model onto the device ``sequential_move_factor`` local ranks at a time, so host memory holds at most that many
    full CPU copies at once (reference :335-356).  Two forms:

    * ``get_model_sequential(model, device, sequential_move_factor=11, param_init_fn=None)`` — the reference's: ``model`` exists
      (possibly on the meta device): materialise it, re-initialise with ``param_init_fn(module, device)`` if given, move it
      (a pipeline model moves its local stages);
    * ``get_model_sequential(model_fn, sequential_move_factor, move_to_device=…)`` — build it inside the wave as well."""
    build = None
    if not isinstance(model, nn.Module):
        build, model = model, None
        if isinstance(device, int):                                       # (model_fn, sequential_move_factor)
            sequential_move_factor, device = device, None
    device = device if device is not None else get_device()

    def bring_up():
        m = build() if build is not None else model
        if build is None or move_to_device:
            if hasattr(m, "maybe_materialize_local_module") and hasattr(m, "move_model_to_device"):   # NxDPPModel
                m.maybe_materialize_local_module()
                m.move_model_to_device()
            elif build is None:
                maybe_materalize_model(m)
                if param_init_fn is not None:
                    reinit_model(m, torch.device("cpu"), param_init_fn)
                m.to(device)
            else:
                m.to(device)
        return m

    if not dist.is_initialized() or dist.get_world_size() == 1:
        return bring_up()
    local_world = torch.cuda.device_count() if not cpu_mode() else dist.get_world_size()
    local_rank = dist.get_rank() % max(1, local_world)
    waves = max(1, math.ceil(local_world / max(1, sequential_move_factor)))
    out = None
    for w in range(waves):
        if local_rank % waves == w:
            out = bring_up()
        if waves > 1:
            dist.barrier()
    return out


def maybe_materalize_model(model: nn.Module) -> None:
    """Reference name (sic). Materialise any remaining meta tensors as empty storage."""
    for module in model.modules():
        if any(p.device.type == "meta" for p in module.parameters(recurse=False)):
            module.to_empty(device=get_device(), recurse=False)


def get_delay_tracing(arg):
    """The delayed-tracing flag of a pipeline model (``_delay_tracing``) or of an nxd_config (``pipeline_config._delay_tracing``);
    ``None`` when the argument carries none (reference model_utils.py:285-296)."""
    if type(arg).__name__ == "NxDPPModel" or hasattr(arg, "original_torch_module"):
        return bool(getattr(arg, "_delay_tracing", False))
    if isinstance(arg, dict):
        return (arg.get("pipeline_config") or {}).get("_delay_tracing")
    return None


def check_delay_tracing(nxd_config) -> bool:
    """Delayed tracing applies when the pipeline model is built by the model wrapper and the user gave no ``input_names``: the
    first batch then names the traced inputs (reference model_utils.py:299-309)."""
    pc = (nxd_config or {}).get("pipeline_config") or {}
    return bool(pc.get("use_model_wrapper", False)) and not pc.get("input_names")


# ---------------------------------------------------------------------------------------------------------------------
# shared (tied) weights, availability probes, structure filters (reference utils/model_utils.py:48-161, 244-253, 370-386)
# ---------------------------------------------------------------------------------------------------------------------
def analyze_shared_parameters(module: nn.Module, shared_parameters=None, prefix: str = ""):
    """Groups of parameter names that refer to the same Parameter object (``[["embed.weight", "lm_head.weight"], …]``)."""
    groups: Dict[int, list] = {}
    for name, p in module.named_parameters(prefix=prefix, remove_duplicate=False):
        groups.setdefault(id(p), []).append(name)
    return [names for names in groups.values() if len(names) > 1]


def _resolve(module: nn.Module, path: str):
    parent_path, _, leaf = path.rpartition(".")
    parent = module.get_submodule(parent_path) if parent_path else module
    return parent, leaf


def retie_shared_weights(module: nn.Module, shared_weight_names) -> None:
    """Make every name of a group point at the first name's Parameter again (after ``to_empty`` / load / device moves)."""
    for names in shared_weight_names:
        parent, leaf = _resolve(module, names[0])
        ref = getattr(parent, leaf)
        for other in names[1:]:
            p2, l2 = _resolve(module, other)
            setattr(p2, l2, ref)


@contextlib.contextmanager
def preserve_shared_weights(model: nn.Module, ignore_hf: bool = False):
    """Record the tied-parameter groups on entry and re-tie them on exit (HF models re-tie through ``tie_weights``)."""
    use_hf = is_hf_pretrained_model(model) and not ignore_hf
    names = None if use_hf else analyze_shared_parameters(model)
    try:
        yield
    finally:
        if use_hf:
            model.tie_weights()
        else:
            retie_shared_weights(model, names)


def is_hf_transformers_available() -> bool:
    import importlib.util

    return importlib.util.find_spec("transformers") is not None


def is_hf_accelerate_available() -> bool:
    import importlib.util

    return importlib.util.find_spec("accelerate") is not None


def is_nxdt_available() -> bool:
    import importlib.util

    return importlib.util.find_spec("neuronx_distributed_training") is not None


def is_nxdt_pretrained_model(model: nn.Module) -> bool:
    if not is_nxdt_available():
        return False
    from neuronx_distributed_training.models.megatron.module import MegatronModule  # type: ignore

    return isinstance(model, MegatronModule)


def recursive_filter(item, predicate):
    """Copy of a nested dict / list / tuple / set keeping only the tensors for which ``predicate(tensor)`` holds
    (non-tensor leaves are always kept) — e.g. ``recursive_filter(state, lambda t: not t.is_meta)``."""
    def keep(obj) -> bool:
        return predicate(obj) if isinstance(obj, torch.Tensor) else True

    if isinstance(item, dict):
        return {k: recursive_filter(v, predicate) for k, v in item.items() if keep(v)}
    if isinstance(item, (list, tuple, set)):
        return type(item)(recursive_filter(v, predicate) for v in item if keep(v))
    return item if keep(item) else None


def has_fake_tensors(model: nn.Module, ignored_params=None) -> bool:
    """True if any (non-ignored) parameter has no storage yet (meta device / FakeTensor) and must be materialised."""
    from torch._subclasses.fake_tensor import FakeTensor

    ignored = {id(p) for p in (ignored_params or ())}
    return any((p.device.type == "meta" or isinstance(p, FakeTensor)) and id(p) not in ignored for p in model.parameters())


import enum as _enum  # noqa: E402


class LogicalNCConfig(_enum.IntEnum):
    """Logical cores per device.  A H100 is ONE logical device (its two dies share L2/HBM coherently and are scheduled
    as one grid over all its SMs), so only ``LNC_1`` is ever returned; ``LNC_2`` exists for configs ported from Trn2."""

    LNC_1 = 1
    LNC_2 = 2


def get_platform_lnc() -> LogicalNCConfig:
    return LogicalNCConfig.LNC_1
