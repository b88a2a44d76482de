"""``NxDModel`` — runtime holding the compiled bucket programs (reference ``trace/nxd_model/nxd_model.py:41-969``).

* a **shape-based router** selects the program whose example input shapes match (per key, first fit by total size);
* each :class:`BucketProgram` owns persistent input buffers and, on CUDA, a captured graph: ``forward`` copies the
  inputs into the static buffers, replays the graph and returns the static outputs;
* state (KV cache) lives in the wrapped module and is shared by all programs;
* ``save``/``load`` persist weights as per-rank safetensors; ``save(portable=True)`` (= the reference's
  ``convert_nxd_model_to_torchscript_model`` + ``torch.jit.save``) writes every bucket as a launch plan
  (``launch_plan.py``) so that ``load`` needs no model code;
* buckets compiled with ``compile_wlo`` come with a layout-transformer plan that re-derives the hoisted constants after
  every ``set_weights`` / ``replace_weights``.

Two ways to fill it: ``add_program`` (v1 ``ModelBuilder.add(key, …)`` buckets) and ``add(key, trace_artifacts,
compilation_artifacts)`` (v2 ``trace`` → ``compile`` units, reference :87-194), after which ``forward`` accepts positional
and keyword tensors, orders the keyword ones by the traced signature and routes by (argument names, shapes)."""
from __future__ import annotations

import os
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn


from .base_nxd_model import BaseNxDModel, StateInitializer  # noqa: F401


class JITWrapper(nn.Module):
    """A Python callable (the input flattener / output packer of a bucket) as a module, so it sits in the model's module tree
    and is scripted / saved with it (reference ``nxd_model.py:29-39``)."""

    def __init__(self, func):
        super().__init__()
        self.func = func

    def forward(self, inputs):
        return self.func(inputs)


class BucketProgram:
    def __init__(self, key: str, module: nn.Module, fn: Callable, example: Tuple[torch.Tensor, ...],
                 use_cuda_graph: bool = True, warmup: int = 2):
        self.key, self.module, self.fn = key, module, fn
        self.shapes = tuple(tuple(t.shape) for t in example)
        self.dtypes = tuple(t.dtype for t in example)
        self.static_in = [t.clone() for t in example]
        self.graph = None
        self.static_out = None
        cuda = all(t.is_cuda for t in example) and torch.cuda.is_available()
        if use_cuda_graph and cuda:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s), torch.no_grad():
                for _ in range(warmup):
                    self.fn(self.module, *self.static_in)
            torch.cuda.current_stream().wait_stream(s)
            self.graph = torch.cuda.CUDAGraph()
            with torch.no_grad(), torch.cuda.graph(self.graph):
                self.static_out = self.fn(self.module, *self.static_in)

    def matches(self, inputs: Sequence[torch.Tensor]) -> bool:
        return len(inputs) == len(self.shapes) and all(tuple(t.shape) == s for t, s in zip(inputs, self.shapes))

    def __call__(self, *inputs: torch.Tensor):
        if self.graph is None:
            with torch.no_grad():
                return self.fn(self.module, *inputs)
        for dst, src in zip(self.static_in, inputs):
            dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_out


SUPPORTED_FORWARD_MODES = {"default", "ranked", "ranked_to_cpu", "async"}


class NxDModel(BaseNxDModel):
    def __init__(self, world_size: int = 1, router: Any = None, start_rank: Optional[int] = None,
                 local_ranks_size: Optional[int] = None, state_initializer: Optional[StateInitializer] = None,
                 layout_transformer: Any = None):
        super().__init__()
        self.world_size, self.custom_router = world_size, router
        if start_rank is None:
            assert local_ranks_size is None or local_ranks_size == world_size, \
                f"{local_ranks_size=} but start_rank is not defined. If local_ranks_size is set, the start rank must also be set."
            self.start_rank, self.local_ranks_size = 0, world_size
        else:
            assert local_ranks_size is not None, \
                f"{start_rank=} but found local_ranks_size to be unset. If setting start_rank, local_ranks_size must also be set."
            self.start_rank, self.local_ranks_size = start_rank, local_ranks_size
        self.programs: Dict[str, List[BucketProgram]] = {}
        # v2 units: key → (trace artifacts, compilation artifacts)
        self.units: Dict[str, Tuple[Any, Any]] = {}
        self.model_params: List[Any] = []
        self.input_shape_map: Dict[str, List[str]] = {}
        self.state_initializer = state_initializer
        self.states: List[Dict[str, torch.Tensor]] = []
        self.layout_transformer = layout_transformer
        self._layout_pairs: Dict[str, Tuple[Any, Any]] = dict(getattr(layout_transformer, "transformers", None) or {})
        self.loaded_on_device = False

    @property
    def loaded_on_neuron(self) -> bool:               # reference attribute name
        return self.loaded_on_device

    # ---- construction ------------------------------------------------------------------
    def add_program(self, prog: BucketProgram) -> None:
        self.programs.setdefault(prog.key, []).append(prog)
        self.programs[prog.key].sort(key=lambda p: sum(int(torch.tensor(s).prod()) for s in p.shapes))

    def add(self, key: str, trace_artifacts: Any, compilation_artifacts: Any) -> "NxDModel":
        """Register one traced + compiled bucket (reference :87-194).  All buckets of one NxDModel must come from the same
        ``forward`` signature; two buckets may not share (argument names, shapes, dtypes)."""
        if key in self.units:
            raise KeyError(f"key {key!r} is already registered")
        params = [(p.param_name, p.is_positional) for p in trace_artifacts.model_params]
        if self.model_params and params != self.model_params:
            raise ValueError(f"bucket {key!r} was traced from a different signature: {params} vs {self.model_params}")
        sig = self._route_key([a.param_name for a in trace_artifacts.provided_args], [a.tensor for a in trace_artifacts.provided_args])
        # two buckets with the same route are legal (e.g. prefill vs speculation programs of one shape): forward() then
        # requires ``model_name``
        self.model_params = params
        self.input_shape_map.setdefault(sig, []).append(key)
        self.units[key] = (trace_artifacts, compilation_artifacts)
        if getattr(compilation_artifacts, "transformer", None) is not None:
            self._layout_pairs[key] = (compilation_artifacts.transformer, compilation_artifacts.plan)
        return self

    @staticmethod
    def _route_key(names: Sequence[str], tensors: Sequence[torch.Tensor]) -> str:
        return ";".join(f"{n}:{tuple(t.shape)}:{t.dtype}" for n, t in zip(names, tensors))

    def get_available_keys(self) -> List[str]:
        return list(self.programs) + list(self.units)

    def _unit(self, key: str):
        if key not in self.units:
            raise KeyError(f"{key!r} is not a registered bucket; available: {self.get_available_keys()}")
        return self.units[key]

    def get_hlo(self, key: str):
        """The reference returns the HLO proto of a bucket; the H100 analogue is the bucket's call description."""
        return self._unit(key)[0].hlo

    def get_metaneff(self, key: str):
        return self._unit(key)[0].metaneff

    def get_neff(self, key: str) -> bytes:
        return self._unit(key)[1].get_neff_bytes()

    # ---- routing / execution -------------------------------------------------------------
    def convert_dict_to_ordered_list(self, inputs: Dict[str, Any], num_pos_args: int) -> Tuple[List[Any], List[str]]:
        """Keyword inputs → list ordered by the traced signature; returns it with the names of ALL supplied arguments
        (positional ones first)."""
        names = [n for n, _ in self.model_params]
        pos = names[:num_pos_args]
        unknown = set(inputs) - set(names)
        if unknown:
            raise KeyError(f"unexpected keyword inputs {sorted(unknown)}; the traced signature has {names}")
        dup = set(inputs) & set(pos)
        if dup:
            raise KeyError(f"{sorted(dup)} given both positionally and by keyword")
        ordered = [n for n in names[num_pos_args:] if n in inputs]
        return [inputs[n] for n in ordered], pos + ordered

    def router(self, inputs: Sequence[torch.Tensor], arg_names: Optional[Sequence[str]] = None, key: Optional[str] = None):
        """v2 (``arg_names`` given): list of bucket keys whose traced (names, shapes, dtypes) equal the call's.
        v1: the matching :class:`BucketProgram`."""
        if arg_names is not None:
            sig = self._route_key(arg_names, inputs)
            if sig not in self.input_shape_map:
                raise KeyError(f"no bucket was traced for inputs {sig}; known routes: {list(self.input_shape_map)}")
            return list(self.input_shape_map[sig])
        if self.custom_router is not None:
            r = self.custom_router(inputs)
            if isinstance(r, BucketProgram):
                return r
            key = r if isinstance(r, str) else key
        keys = [key] if key is not None else list(self.programs)
        for k in keys:
            for p in self.programs.get(k, []):
                if p.matches(inputs):
                    return p
        raise ValueError(f"no compiled bucket for input shapes {[tuple(t.shape) for t in inputs]} (keys {keys})")

    def _my_rank_index(self, n: int) -> int:
        if n == 1:
            return 0
        import torch.distributed as dist

        r = dist.get_rank() if dist.is_initialized() else 0
        return (r - self.start_rank) if n == self.local_ranks_size else r

    def forward(self, *args, model_name: Optional[str] = None, forward_mode: str = "default", **kwargs):
        """``default``: tensors in, this bucket's outputs out.  ``ranked`` / ``ranked_to_cpu`` / ``async``: every input is a
        list with one tensor per rank (this process uses its own entry) and every output comes back as a one-per-local-rank
        list — ``async`` returns without synchronising (CUDA launches are asynchronous anyway; call ``.cpu()`` to block),
        ``ranked_to_cpu`` copies the outputs to host."""
        assert forward_mode in SUPPORTED_FORWARD_MODES, f"{forward_mode=} is not supported. It must be one of {SUPPORTED_FORWARD_MODES}"
        if not self.units:                                   # v1 programs
            return self.router(args, key=model_name)(*args)
        if not self.loaded_on_device:
            raise RuntimeError("Model not initialized. Call set_weights() followed by to_neuron()")
        kw, names = self.convert_dict_to_ordered_list(kwargs, len(args))
        inputs = list(args) + kw
        if forward_mode != "default":
            inputs = [x[self._my_rank_index(len(x))] if isinstance(x, (list, tuple)) else x for x in inputs]
        routes = self.router(inputs, names)
        if len(routes) > 1:
            assert model_name is not None, (f"Got {len(routes)} possible routes but model_name wasn't provided. The Model "
                                            "Name must be provided if input routing is ambiguous.")
            assert model_name in routes, f"{model_name=} is not among the routes for these inputs: {routes}"
        else:
            assert model_name is None or model_name == routes[0], \
                f"Provided model_name does not match model name found by the shape router. Found {routes[0]} but got {model_name}"
            model_name = routes[0]
        ta, ca = self.units[model_name]
        out = ta.packer(ca.program(*ta.flattener(inputs)))
        if forward_mode == "default":
            return out
        flat = list(out) if isinstance(out, (list, tuple)) else [out]
        if forward_mode == "ranked_to_cpu":
            flat = [t.cpu() if isinstance(t, torch.Tensor) else t for t in flat]
        return [[t] for t in flat]                           # [output][local rank]

    # ---- weights / state -----------------------------------------------------------------
    def _unique_modules(self) -> List[nn.Module]:
        seen: Dict[int, nn.Module] = {}
        for progs in self.programs.values():
            for p in progs:
                if isinstance(p.module, nn.Module):
                    seen[id(p.module)] = p.module
        for ta, _ in self.units.values():
            if isinstance(ta.model, nn.Module):
                seen[id(ta.model)] = ta.model
        return list(seen.values())

    def _my_shard(self, sharded_checkpoint: Sequence[Dict[str, torch.Tensor]]) -> Dict[str, torch.Tensor]:
        from ...parallel_layers import parallel_state as ps

        r = ps.get_tensor_model_parallel_rank() if ps.model_parallel_is_initialized() else 0
        if len(sharded_checkpoint) == self.world_size and self.world_size > r:
            return sharded_checkpoint[r]
        return sharded_checkpoint[min(r - self.start_rank, len(sharded_checkpoint) - 1)] if len(sharded_checkpoint) > 1 \
            else sharded_checkpoint[0]

    def _named_state(self) -> List[Dict[str, torch.Tensor]]:
        """Name → tensor maps of everything that holds weights / state: the wrapped modules and the constants of plan-backed
        buckets (several buckets bind the same tensors)."""
        from ...inference.launch_plan import LaunchPlan

        maps: List[Dict[str, torch.Tensor]] = []
        for m in self._unique_modules():
            own = dict(m.named_parameters())
            own.update(dict(m.named_buffers()))
            maps.append(own)
        seen = set()
        for ta, ca in self.units.values():
            for plan in (ta.model, getattr(ca, "plan", None)):
                if isinstance(plan, LaunchPlan) and id(plan) not in seen:
                    seen.add(id(plan))
                    maps.append({n: t for n, t in plan.named_constants().items() if not n.startswith(("_const_", "_derived_"))})
        return maps

    def _run_layout_transformers(self) -> None:
        for transformer, main in self._layout_pairs.values():
            main.apply_transformer(transformer)

    def set_weights(self, sharded_checkpoint: Sequence[Dict[str, torch.Tensor]]) -> None:
        """Copy this rank's shard INTO the existing parameter tensors (their addresses are baked into captured graphs), then
        re-derive the constants the layout transformers computed from them."""
        sd = self._my_shard(sharded_checkpoint)
        with torch.no_grad():
            for own in self._named_state():
                for k, v in sd.items():
                    if k in own and tuple(own[k].shape) == tuple(v.shape):
                        own[k].copy_(v)
        self._run_layout_transformers()
        self._weights_set = True

    def replace_weights(self, sharded_checkpoint: Sequence[Dict[str, torch.Tensor]]) -> None:
        """Swap in new weights after the model is live (LoRA merge, checkpoint hot-swap): same in-place copy, graphs stay
        valid."""
        self.set_weights(sharded_checkpoint)

    def to_neuron(self) -> None:     # reference name
        """Mark the model ready: weights already live on the device (``set_weights`` copied in place, or the module was built
        with real weights); create the state buffers if a :class:`StateInitializer` was given."""
        if self.state_initializer is not None and not self.states:
            self.states = self.state_initializer()
        self.loaded_on_device = True

    to_device = to_neuron

    # ---- v1 runtime names (reference trace/spmd.py:180-291) ------------------------------------------------------------
    def initialize(self, checkpoint: Sequence[Dict[str, torch.Tensor]], start_rank_tensor: Any = None) -> None:
        """Load the sharded checkpoint and create the state buffers (v1: one call; v2: ``set_weights`` + ``to_neuron``)."""
        if start_rank_tensor is not None:
            self.start_rank = int(start_rank_tensor)
        self.set_weights(checkpoint)
        self.to_neuron()

    def initialize_with_saved_weights(self, start_rank_tensor: Any = None) -> None:
        """The modules already hold their weights (built with real weights or restored by :meth:`load`)."""
        if start_rank_tensor is not None:
            self.start_rank = int(start_rank_tensor)
        self._weights_set = True
        self.to_neuron()

    def initialize_spmd_models(self, states, weights, start_rank_id: int = 0) -> None:
        self.states = list(states) if states else self.states
        self.initialize(weights, start_rank_id)

    def mock_initialization(self, mock: bool = True) -> None:
        """Mark the model initialised without weights (shape-only dry runs)."""
        self.loaded_on_device = bool(mock)

    def forward_ranked(self, *args, model_name: Optional[str] = None, **kwargs):
        return self.forward(*args, model_name=model_name, forward_mode="ranked", **kwargs)

    def forward_async(self, *args, model_name: Optional[str] = None, **kwargs):
        return self.forward(*args, model_name=model_name, forward_mode="async", **kwargs)

    @property
    def dtype(self) -> Optional[torch.dtype]:
        for m in self._unique_modules():
            for p in m.parameters():
                return p.dtype
        for own in self._named_state():
            for t in own.values():
                if t.is_floating_point():
                    return t.dtype
        return None

    @property
    def config(self):
        for m in self._unique_modules():
            if hasattr(m, "config"):
                return m.config
        return None

    def _find_buffer(self, buffer_key: str) -> torch.Tensor:
        for st in self.states:
            if buffer_key in st:
                return st[buffer_key]
        for own in self._named_state():
            if buffer_key in own:
                return own[buffer_key]
        raise KeyError(f"no state / weight buffer named {buffer_key!r}")

    def read_from_neuron_buffer(self, buffer_key: str, rank: int = 0) -> torch.Tensor:
        """Host copy of a state (KV cache) or weight buffer of this process's rank."""
        return self._find_buffer(buffer_key).detach().cpu()

    def write_to_neuron_buffer(self, tensor: torch.Tensor, buffer_key: str, rank: int = 0) -> None:
        dst = self._find_buffer(buffer_key)
        assert tuple(dst.shape) == tuple(tensor.shape), f"shape mismatch for {buffer_key}: {tuple(tensor.shape)} vs {tuple(dst.shape)}"
        with torch.no_grad():
            dst.copy_(tensor.to(dst.dtype))

    # ---- persistence ---------------------------------------------------------------------
    def _rank(self) -> int:
        import torch.distributed as dist

        return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0

    def portable_plans(self) -> Dict[str, Any]:
        """Bucket key → launch plan (recorded now for buckets that were compiled straight from the module), plus
        ``__lt__<key>`` → layout transformer for WLO buckets."""
        plans: Dict[str, Any] = {}
        for key, (ta, ca) in self.units.items():
            plans[key] = getattr(ca, "plan", None) or ta.record_plan()
        for key, (transformer, _main) in self._layout_pairs.items():
            plans[f"__lt__{key}"] = transformer
        return plans

    def save(self, path_to_save: str, save_weights: bool = False, portable: bool = False) -> None:
        """Directory with ``nxd_model_meta.pt`` (bucket keys, signatures, example input shapes; the module object itself when
        it pickles, so ``load`` can re-capture without user code) and optionally ``weights_<i>_tp<rank>.safetensors``.

        ``portable=True`` writes the model-code-free artefact instead: one launch plan per bucket
        (``plans_rank<r>.json``) and the constants they bind (``constants_rank<r>.safetensors``: state buffers and
        captured tables always, checkpoint weights when ``save_weights``)."""
        from ...parallel_layers import parallel_state as ps
        from ...utils.safetensors_utils import save_state_dict_safetensors

        os.makedirs(path_to_save, exist_ok=True)
        meta: Dict[str, Any] = {
            "world_size": self.world_size, "model_params": self.model_params,
            "programs": {k: [{"shapes": p.shapes, "dtypes": [str(d) for d in p.dtypes]} for p in v] for k, v in self.programs.items()},
            "units": {k: {"inputs": ta.input_signature(), "outputs": ta.output_spec, "flags": ca.compiler_args}
                      for k, (ta, ca) in self.units.items()},
        }
        if portable:
            if not self.units:
                raise ValueError("portable save needs buckets registered with add(key, trace_artifacts, compilation_artifacts)")
            from ...inference.launch_plan import save_plans

            extra = {"world_size": self.world_size, "model_params": [list(p) for p in self.model_params],
                     "units": {k: {"inputs": [list(i[:1]) + [list(i[1]), i[2]] for i in u["inputs"]], "flags": u["flags"],
                                   "state": list(self.units[k][0].state_names)} for k, u in meta["units"].items()}}
            save_plans(path_to_save, self.portable_plans(), self._rank(), extra, save_weights=save_weights)
            return
        mods = self._unique_modules()
        if self.units and len(mods) == 1:
            try:
                import io
                import pickle

                buf = io.BytesIO()
                pickle.dump(mods[0], buf)
                meta["module_pickle"] = buf.getvalue()
            except Exception:  # noqa: BLE001  (process groups, lambdas … → load() then needs ``model=``)
                meta["module_pickle"] = None
        torch.save(meta, os.path.join(path_to_save, "nxd_model_meta.pt"))
        if save_weights:
            r = ps.get_tensor_model_parallel_rank() if ps.model_parallel_is_initialized() else 0
            for i, m in enumerate(mods):
                save_state_dict_safetensors(m.state_dict(), os.path.join(path_to_save, f"weights_{i}_tp{r}.safetensors"))

    @classmethod
    def _load_portable(cls, path_to_model: str, start_rank: Optional[int], local_ranks_size: Optional[int],
                       device: Optional[torch.device]) -> "NxDModel":
        from ..functions import compile as _compile
        from ...inference.launch_plan import load_plans
        from ..model_builder_utils import ModelParamInfo, ProvidedArgInfo, TraceArtifacts

        import torch.distributed as dist

        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        plans, _tensors, extra = load_plans(path_to_model, rank, device)
        nxd = cls(world_size=extra.get("world_size", 1), start_rank=start_rank, local_ranks_size=local_ranks_size)
        params = [ModelParamInfo(n, bool(p)) for n, p in extra.get("model_params", [])]
        positional = {p.param_name: p.is_positional for p in params}
        complete = True
        for key, plan in plans.items():
            if key.startswith("__lt__"):
                continue
            lt = plans.get(f"__lt__{key}")
            missing = [c.name for i, c in plan.constants.items() if i not in plan.tensors and not c.name.startswith("_derived_")]
            if lt is not None:
                missing += [c.name for i, c in lt.constants.items() if i not in lt.tensors]
            if missing:                                          # saved without weights: allocate, set_weights() fills them
                complete = False
                for p in (plan, lt):
                    if p is None:
                        continue
                    for i, c in p.constants.items():
                        if i not in p.tensors and not c.name.startswith("_derived_"):
                            shared = next((q.named_constants()[c.name] for q in plans.values() if c.name in q.named_constants()), None)
                            p.tensors[i] = shared if shared is not None else \
                                torch.zeros(c.shape, dtype=getattr(torch, c.dtype), device=plan.device)
            if lt is not None:
                plan.apply_transformer(lt)
            u = extra["units"][key]
            provided = [ProvidedArgInfo(n, positional.get(n, True), torch.zeros(shape, dtype=getattr(torch, dt.replace("torch.", "")),
                                                                              device=plan.device))
                        for n, shape, dt in u["inputs"]]
            ta = TraceArtifacts(model=plan, provided_args=provided, model_params=params, state_names=list(u.get("state", [])))
            ta._plan = plan
            ca = _compile(ta, None, None, u.get("flags"), key)
            nxd.add(key, ta, ca)
            if lt is not None:
                nxd._layout_pairs[key] = (lt, plan)
        nxd._weights_set = complete
        return nxd

    @classmethod
    def load(cls, path_to_model: str, start_rank: Optional[int] = None, local_ranks_size: Optional[int] = None,
             model: Optional[nn.Module] = None, device: Optional[torch.device] = None) -> "NxDModel":
        """Rebuild a saved v2 model.  A portable artefact (``save(portable=True)``) is re-captured from its launch plans —
        no model code needed.  Otherwise every bucket is re-traced from the recorded input signatures; ``model`` is then
        needed when the module could not be pickled at save time."""
        import pickle

        from ...parallel_layers import parallel_state as ps
        from ...utils.safetensors_utils import load_state_dict_safetensors
        from ..functions import compile as _compile
        from ..functions import trace as _trace

        if model is None and not os.path.exists(os.path.join(path_to_model, "nxd_model_meta.pt")):
            return cls._load_portable(path_to_model, start_rank, local_ranks_size, device)
        meta = torch.load(os.path.join(path_to_model, "nxd_model_meta.pt"), weights_only=False)
        if model is None:
            if not meta.get("module_pickle"):
                raise ValueError("the saved model does not embed its module; pass model=<the nn.Module>")
            model = pickle.loads(meta["module_pickle"])
        dev = device or (torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu"))
        model = model.to(dev)
        r = ps.get_tensor_model_parallel_rank() if ps.model_parallel_is_initialized() else 0
        wpath = os.path.join(path_to_model, f"weights_0_tp{r}.safetensors")
        if os.path.exists(wpath):
            model.load_state_dict(load_state_dict_safetensors(wpath), strict=False)
        nxd = cls(world_size=meta["world_size"], start_rank=start_rank, local_ranks_size=local_ranks_size)
        for key, u in meta["units"].items():
            tensors = {n: torch.zeros(shape, dtype=getattr(torch, dt.replace("torch.", "")), device=dev) for n, shape, dt in u["inputs"]}
            ta = _trace(model, None, tensors)
            nxd.add(key, ta, _compile(ta, None, None, u.get("flags"), key))
        nxd._weights_set = os.path.exists(wpath)
        return nxd


class TorchScriptNxDModel(NxDModel):
    """An ``NxDModel`` whose buckets interpret launch plans: it carries no reference to the model's Python code, and
    ``save`` / ``load`` default to the portable artefact (reference ``nxd_model.py:709-969``)."""

    def save(self, path_to_save: str, save_weights: bool = True, portable: bool = True) -> None:  # noqa: D102
        super().save(path_to_save, save_weights=save_weights, portable=portable)


def convert_nxd_model_to_torchscript_model(nxd_model: NxDModel, save_weights: bool = False) -> TorchScriptNxDModel:
    """Model-code-free copy of ``nxd_model`` (reference ``nxd_model.py:924-969``): every bucket is recorded into a launch
    plan and re-compiled from it.  The copy SHARES weights and state tensors with ``nxd_model``.  ``save_weights`` is the
    default of the copy's ``save``."""
    from ..functions import compile as _compile
    from ..model_builder_utils import TraceArtifacts

    out = TorchScriptNxDModel(world_size=nxd_model.world_size, start_rank=nxd_model.start_rank if nxd_model.start_rank else None,
                              local_ranks_size=nxd_model.local_ranks_size if nxd_model.start_rank else None)
    if not nxd_model.units:
        raise ValueError("only models built from trace → compile units can be converted")
    for key, (ta, ca) in nxd_model.units.items():
        plan = getattr(ca, "plan", None) or ta.record_plan()
        pta = TraceArtifacts(model=plan, provided_args=ta.provided_args, model_params=ta.model_params, output_spec=ta.output_spec,
                             weight_name_to_idx=dict(ta.weight_name_to_idx), weight_names_to_skip=set(ta.weight_names_to_skip),
                             state_names=list(ta.state_names))
        pta._plan = plan
        out.add(key, pta, _compile(pta, None, None, ca.compiler_args, key))
        if key in nxd_model._layout_pairs:
            out._layout_pairs[key] = nxd_model._layout_pairs[key]
    out.loaded_on_device = nxd_model.loaded_on_device
    out._default_save_weights = save_weights
    return out
