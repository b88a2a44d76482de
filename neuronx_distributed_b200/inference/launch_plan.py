"""Launch plans — the model-code-free inference artefact (role of the reference's TorchScript / HLO+NEFF artefacts:
``trace/nxd_model/nxd_model.py:709-969`` ``TorchScriptNxDModel``, ``trace/hlo_utils.py`` graph surgery).

A CUDA graph cannot be serialised and there is no tracing compiler on this stack, so the portable form of a bucket is the
ordered list of *launches* one call performs — recorded once, replayed by a ~100-line interpreter, and re-captured into a
CUDA graph at load time:

* **recording** runs the bucket under a ``TorchDispatchMode``: every dispatcher op (``aten::…`` after composite ops are
  decomposed) becomes a node; calls into the sm_90a extension are seen through a proxy of ``ops._ext.ext()`` and become
  ``ext`` nodes (kernel name + tensor / scalar arguments); framework functions that own process-local resources —
  collectives, symmetric-memory kernels, fused GEMM+collective ops — are decorated with :func:`plan_op` and become ``py``
  nodes that re-resolve their groups / workspaces when replayed (process groups are stored by registry name);
* tensors that enter the recording from outside (weights, KV caches, tables) are **constants**: named after the module's
  parameters / buffers when they are one, so ``set_weights`` / ``replace_weights`` keep working on a loaded artefact, and
  shared between the buckets of one model (the prefill and decode plans mutate the same KV cache);
* the IR supports the passes the reference performs on HLO: dead-code elimination, weight usage maps, and hoisting of
  weight-only sub-graphs into a *layout transformer* plan that runs once per weight load (dtype casts, transposes,
  de-quantisation, input-independent masks and tables) — see :meth:`LaunchPlan.hoist_weight_only`.

Replay needs ``torch`` + this package, not the model's Python code.  Python scalars read from tensors during recording
(``.item()``) are baked into the plan, exactly like TorchScript tracing; ``meta['baked_scalars']`` counts them.
"""
from __future__ import annotations

import enum
import importlib
import json
import os
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, Iterable, List, Optional, Sequence, Set, Tuple

import torch
from torch.utils._python_dispatch import TorchDispatchMode


class PlanError(RuntimeError):
    pass


# ---------------------------------------------------------------------------------------------------------------------
# registry of replayable framework functions
# ---------------------------------------------------------------------------------------------------------------------
from ..utils.plan_registry import PY_OPS as _PY_OPS
from ..utils.plan_registry import active_recorder, plan_op, recording, set_recorder  # noqa: F401


# extension entry points that take raw peer pointers / epochs: only legal inside a plan_op
_EXT_RESOURCE_PREFIXES = ("vmm_", "symm_", "tp_gemm", "nvls_", "gemv_allreduce", "zero1_", "oneshot_", "allreduce_")
# Extension entry points that allocate their results and write to none of their arguments.  Everything else (``gemm_bf16`` /
# ``grouped_gemm`` with an ``out`` argument, ``decode_rope_kv`` appending to the cache, optimizer kernels …) is treated as
# writing to EVERY tensor argument: conservative — such tensors count as state, are never hoisted or dropped — but safe.
_EXT_PURE = frozenset({"rmsnorm_fwd", "rmsnorm_bwd", "add_rmsnorm_fwd", "add_rmsnorm_bwd", "swiglu_fwd", "swiglu_bwd", "rope_apply",
                       "ce_stats", "ce_backward", "decode_attention", "decode_attention_partial", "gemv", "gemv_mx",
                       "moe_block_tkg", "moe_block_metadata", "row_argmax", "row_topk", "flash_attn_fwd",
                       "flash_attn_bwd", "moe_block_tkg_supported", "row_topk_supported", "grouped_gemm",
                       "gemm_fp8_block", "quantize_fp8_groups", "grouped_gemm_fp8_block"})
# … and the ones that write exactly these positional arguments (everything else they take is read-only)
_EXT_WRITES = {"gemm_bf16": (2,), "gemm_fp8": (2,), "grouped_wgrad": (2,), "decode_rope_kv": (6, 7),
               "multi_tensor_sq_norm": (1,)}


# ---------------------------------------------------------------------------------------------------------------------
# value encoding (JSON)
# ---------------------------------------------------------------------------------------------------------------------
def _pg_name(pg) -> str:
    from ..parallel_layers import parallel_state as ps

    name = ps.group_name(pg)
    if name is None:
        raise PlanError("a process group that is not registered in parallel_state cannot be stored in a launch plan")
    return name


def _encode(x: Any, ref: Callable[[torch.Tensor], int]) -> Any:
    if isinstance(x, torch.Tensor):
        return {"t": ref(x)}
    if x is None or isinstance(x, (bool, str)):
        return x
    if isinstance(x, (torch.SymInt, torch.SymFloat, torch.SymBool)):
        raise PlanError("symbolic shapes cannot be recorded")
    if isinstance(x, int) and not isinstance(x, enum.Enum):
        return int(x)
    if isinstance(x, float):
        return float(x)
    if isinstance(x, torch.dtype):
        return {"dtype": str(x).split(".", 1)[1]}
    if isinstance(x, torch.device):
        return {"device": str(x)}
    if isinstance(x, torch.layout):
        return {"layout": str(x).split(".", 1)[1]}
    if isinstance(x, torch.memory_format):
        return {"mf": str(x).split(".", 1)[1]}
    if isinstance(x, (tuple, torch.Size)):
        return {"tu": [_encode(v, ref) for v in x]}
    if isinstance(x, list):
        return {"l": [_encode(v, ref) for v in x]}
    if isinstance(x, dict):
        return {"d": {str(k): _encode(v, ref) for k, v in x.items()}}
    if isinstance(x, slice):
        return {"slice": [_encode(x.start, ref), _encode(x.stop, ref), _encode(x.step, ref)]}
    if x is Ellipsis:
        return {"ellipsis": 1}
    try:
        import torch.distributed as dist

        if isinstance(x, dist.ProcessGroup):
            return {"pg": _pg_name(x)}
        if isinstance(x, (dist.ReduceOp, dist.ReduceOp.RedOpType)):
            return {"redop": str(x).split(".")[-1]}
    except (ImportError, AttributeError):
        pass
    if isinstance(x, enum.Enum):
        return {"enum": [type(x).__module__, type(x).__qualname__, x.name]}
    raise PlanError(f"a value of type {type(x).__name__} cannot be stored in a launch plan")


def _decode(x: Any, env: Dict[int, torch.Tensor], device: Optional[torch.device], recorded_type: str) -> Any:
    if not isinstance(x, dict):
        return x
    (tag, v), = x.items()
    if tag == "t":
        return env[v]
    if tag == "dtype":
        return getattr(torch, v)
    if tag == "device":
        d = torch.device(v)
        return device if (device is not None and d.type == recorded_type) else d
    if tag == "layout":
        return getattr(torch, v)
    if tag == "mf":
        return getattr(torch, v)
    if tag == "tu":
        return tuple(_decode(i, env, device, recorded_type) for i in v)
    if tag == "l":
        return [_decode(i, env, device, recorded_type) for i in v]
    if tag == "d":
        return {k: _decode(i, env, device, recorded_type) for k, i in v.items()}
    if tag == "slice":
        return slice(*[_decode(i, env, device, recorded_type) for i in v])
    if tag == "ellipsis":
        return Ellipsis
    if tag == "pg":
        from ..parallel_layers import parallel_state as ps

        return ps.group_by_name(v)
    if tag == "redop":
        import torch.distributed as dist

        return getattr(dist.ReduceOp, v)
    if tag == "enum":
        mod, qual, name = v
        obj: Any = importlib.import_module(mod)
        for part in qual.split("."):
            obj = getattr(obj, part)
        return obj[name]
    raise PlanError(f"unknown tag {tag!r} in a launch plan")


def _refs(x: Any, out: List[int]) -> List[int]:
    """All value ids referenced by an encoded argument tree."""
    if isinstance(x, dict):
        (tag, v), = x.items()
        if tag == "t":
            out.append(v)
        elif tag in ("tu", "l", "slice"):
            for i in v:
                _refs(i, out)
        elif tag == "d":
            for i in v.values():
                _refs(i, out)
    return out


def _flat_tensors(x: Any, out: List[Any]) -> List[Any]:
    """Leaves of an op result in a fixed order: tensors and placeholders (``None``) for everything else."""
    if isinstance(x, torch.Tensor):
        out.append(x)
    elif isinstance(x, (list, tuple)):
        for i in x:
            _flat_tensors(i, out)
    elif isinstance(x, dict):
        for k in x:
            _flat_tensors(x[k], out)
    else:
        out.append(None)
    return out


def _storage_ptr(t: torch.Tensor) -> int:
    try:
        return t.untyped_storage().data_ptr() if t.device.type != "meta" else 0
    except (RuntimeError, NotImplementedError):
        return 0


# ---------------------------------------------------------------------------------------------------------------------
# IR
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Node:
    kind: str                       # "op" (dispatcher op) | "ext" (extension kernel) | "py" (plan_op)
    target: str
    args: Any
    kwargs: Any
    outs: List[Optional[int]]       # value ids of the flattened result (None: not a tensor)
    mutates: List[int] = field(default_factory=list)
    pure: bool = True               # no effect besides ``outs`` / ``mutates``
    alias_of: Dict[int, int] = field(default_factory=dict)    # out id → the input id whose storage it shares

    def inputs(self) -> List[int]:
        return _refs(self.kwargs, _refs(self.args, []))

    def to_json(self) -> Dict[str, Any]:
        return {"k": self.kind, "f": self.target, "a": self.args, "kw": self.kwargs, "o": self.outs, "m": self.mutates,
                "p": self.pure, "al": {str(k): v for k, v in self.alias_of.items()}}

    @staticmethod
    def from_json(d: Dict[str, Any]) -> "Node":
        return Node(d["k"], d["f"], d["a"], d["kw"], d["o"], d.get("m", []), d.get("p", True),
                    {int(k): v for k, v in d.get("al", {}).items()})


@dataclass
class ConstInfo:
    name: str
    shape: Tuple[int, ...]
    dtype: str
    named: bool                     # a module parameter / buffer (survives under its own name) vs an anonymous capture
    device_type: str = ""           # where the recorded tensor lived ("" = the plan's device type)
    in_checkpoint: bool = True      # a key of the module's ``state_dict`` (non-persistent buffers and captures are not)


def _resolve_op(target: str) -> Callable:
    qual, _, overload = target.partition(".")
    ns, _, op = qual.partition("::")
    return getattr(getattr(getattr(torch.ops, ns), op), overload or "default")


class LaunchPlan:
    """See the module docstring.  Callable: ``plan(*tensors)`` or ``plan(**{input_name: tensor})``."""

    FORMAT = 1

    def __init__(self, nodes: List[Node], inputs: List[Dict[str, Any]], outputs: Any, constants: Dict[int, ConstInfo],
                 device_type: str, meta: Optional[Dict[str, Any]] = None):
        self.nodes, self.inputs, self.outputs, self.constants = nodes, inputs, outputs, constants
        self.device_type = device_type
        self.meta: Dict[str, Any] = meta or {}
        self.tensors: Dict[int, torch.Tensor] = {}             # constant id → bound tensor
        self.device: Optional[torch.device] = None
        self._schedule: Optional[List[List[int]]] = None
        self._fns: Optional[List[Callable]] = None

    # ---- constants -------------------------------------------------------------------------------------------------
    def named_constants(self) -> Dict[str, torch.Tensor]:
        return {c.name: self.tensors[i] for i, c in self.constants.items() if i in self.tensors}

    def bind(self, tensors: Dict[str, torch.Tensor], strict: bool = True) -> "LaunchPlan":
        """Attach constant tensors by name (the SAME tensor objects may be bound to several plans — shared state)."""
        for i, c in self.constants.items():
            if c.name in tensors:
                t = tensors[c.name]
                if tuple(t.shape) != tuple(c.shape):
                    raise PlanError(f"constant {c.name}: shape {tuple(t.shape)} does not match the recorded {tuple(c.shape)}")
                self.tensors[i] = t
            elif strict and i not in self.tensors:
                raise PlanError(f"no tensor for constant {c.name!r}")
        for t in self.tensors.values():
            if t.device.type == self.device_type:
                self.device = t.device
                break
        return self

    def state_names(self) -> List[str]:
        """Constants some node writes to (KV caches …)."""
        roots = self._mutated_roots()
        return [c.name for i, c in self.constants.items() if i in roots]

    # ---- execution -------------------------------------------------------------------------------------------------
    def _prepare(self) -> None:
        for m in self.meta.get("py_modules", []):
            importlib.import_module(m)
        fns: List[Callable] = []
        for n in self.nodes:
            if n.kind == "op":
                fns.append(_resolve_op(n.target))
            elif n.kind == "ext":
                from ..ops import _ext

                mod = _ext._load()
                if mod is None:
                    raise PlanError(f"the plan launches the extension kernel {n.target!r} but the extension is not loaded: "
                                    f"{_ext.load_error()!r}")
                fns.append(getattr(mod, n.target))
            elif n.kind == "py":
                if n.target not in _PY_OPS:
                    raise PlanError(f"plan op {n.target!r} is not registered (modules imported: {self.meta.get('py_modules')})")
                fns.append(_PY_OPS[n.target][0])
            else:
                raise PlanError(f"unknown node kind {n.kind!r}")
        keep = set(_refs(self.outputs, [])) | set(self.constants) | {i["id"] for i in self.inputs}
        last: Dict[int, int] = {}
        for idx, n in enumerate(self.nodes):
            for v in n.inputs():
                last[v] = idx
        sched: List[List[int]] = [[] for _ in self.nodes]
        for v, idx in last.items():
            if v not in keep:
                sched[idx].append(v)
        for idx, n in enumerate(self.nodes):                       # results nobody reads
            for o in n.outs:
                if o is not None and o not in last and o not in keep:
                    sched[idx].append(o)
        self._fns, self._schedule = fns, sched

    def run(self, *inputs: torch.Tensor) -> Any:
        if self._fns is None:
            self._prepare()
        if len(inputs) != len(self.inputs):
            raise PlanError(f"the plan takes {len(self.inputs)} tensors ({[i['name'] for i in self.inputs]}), got {len(inputs)}")
        env: Dict[int, torch.Tensor] = dict(self.tensors)
        missing = [c.name for i, c in self.constants.items() if i not in env]
        if missing:
            raise PlanError(f"constants without a tensor: {missing[:5]}{' …' if len(missing) > 5 else ''}")
        for spec, t in zip(self.inputs, inputs):
            if tuple(t.shape) != tuple(spec["shape"]):
                raise PlanError(f"input {spec['name']}: shape {tuple(t.shape)} does not match the recorded {tuple(spec['shape'])}")
            env[spec["id"]] = t
        dev, rtype = self.device, self.device_type
        with torch.no_grad():
            for n, fn, dead in zip(self.nodes, self._fns, self._schedule):
                out = fn(*_decode(n.args, env, dev, rtype), **_decode(n.kwargs, env, dev, rtype))
                if len(n.outs) == 1 and isinstance(out, torch.Tensor):
                    env[n.outs[0]] = out
                else:
                    for vid, t in zip(n.outs, _flat_tensors(out, [])):
                        if vid is not None:
                            env[vid] = t
                for v in dead:
                    env.pop(v, None)
        return _decode(self.outputs, env, dev, rtype)

    def __call__(self, *args: torch.Tensor, **kwargs: torch.Tensor) -> Any:
        if kwargs:
            names = [i["name"] for i in self.inputs]
            by_name = dict(zip(names[:len(args)], args))
            by_name.update(kwargs)
            args = tuple(by_name[n] for n in names)
        return self.run(*args)

    # ---- analysis / passes (the roles of reference trace/hlo_utils.py) ----------------------------------------------
    def _roots(self) -> Dict[int, int]:
        """Value id → id of the value whose storage it (transitively) aliases."""
        root: Dict[int, int] = {}
        for n in self.nodes:
            for o, base in n.alias_of.items():
                root[o] = root.get(base, base)
        return root

    def _mutated_roots(self) -> Set[int]:
        root = self._roots()
        return {root.get(v, v) for n in self.nodes for v in n.mutates}

    def weight_usage(self) -> Dict[str, List[Tuple[int, str]]]:
        """Constant name → [(node index, target)] of the nodes that read it directly or through views (reference
        ``prepare_parameter_usage_map``)."""
        root = self._roots()
        use: Dict[str, List[Tuple[int, str]]] = {c.name: [] for c in self.constants.values()}
        for idx, n in enumerate(self.nodes):
            if n.alias_of and n.pure and not n.mutates and all(o in n.alias_of for o in n.outs if o is not None):
                continue                                           # a pure view: its consumers are the real users
            for v in set(n.inputs()):
                r = root.get(v, v)
                if r in self.constants:
                    use[self.constants[r].name].append((idx, n.target))
        return use

    def kernel_weight_names(self) -> List[str]:
        """Weights consumed by extension kernels (reference ``get_nki_kernel_weight_names``)."""
        kinds = {idx: n.kind for idx, n in enumerate(self.nodes)}
        return sorted(name for name, users in self.weight_usage().items() if any(kinds[i] != "op" for i, _ in users))

    def calls_extension(self) -> bool:
        return any(n.kind == "ext" for n in self.nodes)

    def dce(self) -> int:
        """Drop pure nodes whose results are never read and whose writes land in dead intermediates.  Returns the number
        of nodes removed."""
        root = self._roots()
        external = set(self.constants) | {i["id"] for i in self.inputs}
        live = set(_refs(self.outputs, []))
        live_roots = {root.get(v, v) for v in live}
        keep: List[Node] = []
        removed = 0
        for n in reversed(self.nodes):
            outs = [o for o in n.outs if o is not None]
            writes = {root.get(v, v) for v in n.mutates}
            needed = (not n.pure) or any(o in live for o in outs) or any(w in external or w in live_roots for w in writes)
            if needed:
                keep.append(n)
                for v in n.inputs():
                    live.add(v)
                    live_roots.add(root.get(v, v))
            else:
                removed += 1
        self.nodes = keep[::-1]
        self._fns = None
        return removed

    def hoist_weight_only(self, skip: Iterable[str] = ()) -> Tuple["LaunchPlan", "LaunchPlan", Dict[str, List[str]]]:
        """Split the plan into a *layout transformer* (everything that depends only on frozen constants: casts,
        transposes, de-quantisation, input-independent masks / tables) and the remaining per-call plan, which consumes
        the transformer's results as new constants ``_derived_<id>``.  Returns ``(transformer, main, transform_map)``;
        ``transform_map`` names, per weight, the chain of hoisted ops that start from it.  Constants named in ``skip``
        and everything written to in place (state) stay untouched."""
        skip = set(skip)
        mut, root = self._mutated_roots(), self._roots()
        frozen: Set[int] = {i for i, c in self.constants.items() if i not in mut and c.name not in skip}
        hoisted: List[Node] = []
        rest: List[Node] = []
        origin: Dict[int, Set[int]] = {i: {i} for i in frozen}
        for n in self.nodes:
            ins = n.inputs()
            outs = [o for o in n.outs if o is not None]
            ok = n.pure and not n.mutates and n.kind == "op" and outs and all(v in frozen for v in ins) and \
                not any(root.get(o, o) in mut for o in outs)
            if ok:
                hoisted.append(n)
                src: Set[int] = set()
                for v in ins:
                    src |= origin.get(v, set())
                for o in outs:
                    frozen.add(o)
                    origin[o] = src
            else:
                rest.append(n)
        produced = {o for n in hoisted for o in n.outs if o is not None}
        needed = set(_refs(self.outputs, []))
        for n in rest:
            needed.update(n.inputs())
        derived = sorted(produced & needed)
        hoisted_in: Set[int] = set()
        for n in hoisted:
            hoisted_in.update(n.inputs())
        t_consts = {i: c for i, c in self.constants.items() if i in hoisted_in}
        transformer = LaunchPlan(hoisted, [], {"l": [{"t": v} for v in derived]}, t_consts, self.device_type,
                                 {"py_modules": self.meta.get("py_modules", []), "derived_ids": derived, "is_transformer": True})
        shapes = self.meta.get("value_specs", {})
        m_consts = {i: c for i, c in self.constants.items() if i in needed}
        for v in derived:
            shp, dt = shapes.get(str(v), ((), "float32"))
            m_consts[v] = ConstInfo(f"_derived_{v}", tuple(shp), dt, named=False, in_checkpoint=False)
        main = LaunchPlan(rest, list(self.inputs), self.outputs, m_consts, self.device_type,
                          dict(self.meta, derived_ids=derived))
        tmap: Dict[str, List[str]] = {}
        for n in hoisted:
            srcs: Set[int] = set()
            for v in n.inputs():
                srcs |= origin.get(v, set())
            if len(srcs) == 1:
                (s,) = srcs
                if s in self.constants:
                    tmap.setdefault(self.constants[s].name, []).append(n.target)
        transformer.tensors = {i: t for i, t in self.tensors.items() if i in t_consts}
        main.tensors = {i: t for i, t in self.tensors.items() if i in m_consts}
        transformer.device = main.device = self.device
        return transformer, main, tmap

    def apply_transformer(self, transformer: "LaunchPlan") -> None:
        """Run ``transformer`` (on its bound weights) and bind its results as this plan's derived constants.  Constants
        that are already bound are overwritten IN PLACE: their addresses may be baked into a captured CUDA graph (a
        derived view of a weight aliases the weight, and the copy is then a no-op)."""
        outs = transformer.run()
        for vid, t in zip(transformer.meta["derived_ids"], outs):
            if vid not in self.constants:
                continue
            old = self.tensors.get(vid)
            if old is not None and old.shape == t.shape and old.dtype == t.dtype and old.device == t.device:
                if old.data_ptr() != t.data_ptr() or old.stride() != t.stride():
                    old.copy_(t)
            else:
                self.tensors[vid] = t

    # ---- description / persistence ---------------------------------------------------------------------------------
    def summary(self) -> Dict[str, Any]:
        by: Dict[str, int] = {}
        for n in self.nodes:
            by[n.target] = by.get(n.target, 0) + 1
        return {"nodes": len(self.nodes), "ext_kernels": sum(n.kind == "ext" for n in self.nodes),
                "py_ops": sum(n.kind == "py" for n in self.nodes), "constants": len(self.constants),
                "inputs": [(i["name"], tuple(i["shape"]), i["dtype"]) for i in self.inputs],
                "top_targets": sorted(by.items(), key=lambda kv: -kv[1])[:8], "baked_scalars": self.meta.get("baked_scalars", 0)}

    def to_json(self) -> Dict[str, Any]:
        return {"format": self.FORMAT, "device_type": self.device_type, "meta": self.meta,
                "inputs": self.inputs, "outputs": self.outputs,
                "constants": {str(i): [c.name, list(c.shape), c.dtype, c.named, c.device_type, c.in_checkpoint]
                              for i, c in self.constants.items()},
                "nodes": [n.to_json() for n in self.nodes]}

    @staticmethod
    def from_json(d: Dict[str, Any]) -> "LaunchPlan":
        if d.get("format") != LaunchPlan.FORMAT:
            raise PlanError(f"launch plan format {d.get('format')} is not supported (expected {LaunchPlan.FORMAT})")
        consts = {int(i): ConstInfo(v[0], tuple(v[1]), v[2], bool(v[3]), v[4] if len(v) > 4 else "",
                                   bool(v[5]) if len(v) > 5 else bool(v[3])) for i, v in d["constants"].items()}
        return LaunchPlan([Node.from_json(n) for n in d["nodes"]], d["inputs"], d["outputs"], consts, d["device_type"], d.get("meta"))

    def save(self, path: str) -> None:
        with open(path, "w") as f:
            json.dump(self.to_json(), f)

    @staticmethod
    def load(path: str) -> "LaunchPlan":
        with open(path) as f:
            return LaunchPlan.from_json(json.load(f))


# ---------------------------------------------------------------------------------------------------------------------
# recording
# ---------------------------------------------------------------------------------------------------------------------
class _ExtProxy:
    """Stands in for the extension module while a recording is active."""

    def __init__(self, real: Any, rec: "_Recorder"):
        self._real, self._rec = real, rec

    def __getattr__(self, name: str):
        fn = getattr(self._real, name)
        if not callable(fn):
            return fn
        rec = self._rec

        def call(*args, **kwargs):
            if rec.paused:
                return fn(*args, **kwargs)
            if name.startswith(_EXT_RESOURCE_PREFIXES):
                raise PlanError(f"extension entry point {name!r} takes process-local resources (peer pointers, epochs); "
                                "call it from a function decorated with @plan_op")
            return rec.record_call("ext", name, fn, args, kwargs)

        return call


class _Recorder(TorchDispatchMode):
    def __init__(self, names: Dict[int, str], by_mem: Dict[Tuple, str], checkpoint_keys: Optional[Set[str]] = None):
        super().__init__()
        self.names, self.mem_names = names, by_mem
        self.checkpoint_keys = checkpoint_keys
        self.nodes: List[Node] = []
        self.by_pyid: Dict[int, int] = {}
        self.by_mem: Dict[Tuple, int] = {}
        self.keep: List[torch.Tensor] = []
        self.constants: Dict[int, Tuple[ConstInfo, torch.Tensor]] = {}
        self.specs: Dict[str, Tuple[Tuple[int, ...], str]] = {}
        self.produced_storage: Set[int] = set()
        self.py_modules: Set[str] = set()
        self.paused = 0
        self.baked = 0
        self.warnings: List[str] = []
        self._next = 0

    # value numbering
    def _new(self, t: torch.Tensor) -> int:
        vid = self._next
        self._next += 1
        self.by_pyid[id(t)] = vid
        self.keep.append(t)
        self.specs[str(vid)] = (tuple(t.shape), str(t.dtype).split(".", 1)[1])
        return vid

    @staticmethod
    def _mem_key(t: torch.Tensor) -> Tuple:
        return (_storage_ptr(t), t.storage_offset(), tuple(t.shape), tuple(t.stride()), t.dtype)

    def ref(self, t: torch.Tensor) -> int:
        vid = self.by_pyid.get(id(t))
        if vid is not None:
            return vid
        key = self._mem_key(t)
        vid = self.by_mem.get(key) if key[0] else None
        if vid is not None:                                        # another Python object over the same memory (``.data``)
            self.by_pyid[id(t)] = vid
            self.keep.append(t)
            return vid
        if key[0] and key[0] in self.produced_storage:
            self.warnings.append(f"a tensor of shape {tuple(t.shape)} aliases memory produced inside the recording but was "
                                 "created outside the dispatcher; it is frozen as a constant")
        vid = self._new(t)
        name = self.names.get(id(t)) or self.mem_names.get(key)
        named = name is not None
        if name is None:
            name = f"_const_{vid}"
        in_ckpt = named and (self.checkpoint_keys is None or name in self.checkpoint_keys)
        self.constants[vid] = (ConstInfo(name, tuple(t.shape), str(t.dtype).split(".", 1)[1], named, t.device.type, in_ckpt), t)
        if key[0]:
            self.by_mem[key] = vid
        return vid

    def bind_input(self, t: torch.Tensor) -> int:
        if id(t) in self.by_pyid:
            raise PlanError("the same tensor object was passed for two inputs")
        return self._new(t)

    def _bind_outputs(self, out: Any, in_tensors: Sequence[torch.Tensor]) -> Tuple[List[Optional[int]], Dict[int, int]]:
        flat = _flat_tensors(out, [])
        outs: List[Optional[int]] = []
        alias: Dict[int, int] = {}
        in_ptrs = {}
        for t in in_tensors:
            p = _storage_ptr(t)
            if p:
                in_ptrs.setdefault(p, self.by_pyid[id(t)])
        for t in flat:
            if t is None:
                outs.append(None)
                continue
            vid = self.by_pyid.get(id(t))
            if vid is None:
                vid = self._new(t)
                p = _storage_ptr(t)
                if p in in_ptrs:
                    alias[vid] = in_ptrs[p]
                elif p:
                    self.produced_storage.add(p)
            outs.append(vid)
        return outs, alias

    # dispatcher ops
    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if self.paused:
            return func(*args, **kwargs)
        if func.namespace in ("c10d", "_c10d_functional", "c10d_functional"):
            raise PlanError(f"{func} was issued directly through torch.distributed while a launch plan was being recorded; "
                            "route collectives through parallel_layers.comm (or a @plan_op function) so that the plan can "
                            "store the process group by name")
        in_tensors: List[torch.Tensor] = []

        def ref(t):
            in_tensors.append(t)
            return self.ref(t)

        enc_a, enc_k = _encode(list(args), ref)["l"], _encode(dict(kwargs), ref)["d"]
        out = func(*args, **kwargs)
        flat = _flat_tensors(out, [])
        if not any(t is not None for t in flat):
            schema = func._schema
            if not any(a.alias_info is not None and a.alias_info.is_write for a in schema.arguments):
                self.baked += 1                                    # ``.item()``, ``equal`` …: the Python value is baked in
                return out
        mutates: List[int] = []
        schema = func._schema
        for i, a in enumerate(schema.arguments):
            if a.alias_info is not None and a.alias_info.is_write:
                val = args[i] if i < len(args) else kwargs.get(a.name)
                for t in _flat_tensors(val, []):
                    if t is not None:
                        mutates.append(self.by_pyid[id(t)])
        outs, alias = self._bind_outputs(out, in_tensors)
        name = f"{schema.name}.{func._overloadname}" if func._overloadname else schema.name
        pure = torch.Tag.nondeterministic_seeded not in func.tags
        self.nodes.append(Node("op", name, {"l": enc_a}, {"d": enc_k}, outs, mutates, pure, alias))
        return out

    # extension kernels and plan ops
    def record_call(self, kind: str, name: str, fn: Callable, args, kwargs) -> Any:
        in_tensors: List[torch.Tensor] = []

        def ref(t):
            in_tensors.append(t)
            return self.ref(t)

        enc_a, enc_k = _encode(list(args), ref)["l"], _encode(dict(kwargs), ref)["d"]
        self.paused += 1
        try:
            out = fn(*args, **kwargs)
        finally:
            self.paused -= 1
        outs, alias = self._bind_outputs(out, in_tensors)
        if kind == "py":
            pure = _PY_OPS[name][1]
            self.py_modules.add(fn.__module__)
        else:
            pure = name in _EXT_PURE
        if kind == "ext" and name in _EXT_WRITES:
            pure = True                                            # no effect besides the listed arguments and the results
            mutates = sorted({self.by_pyid[id(t)] for i in _EXT_WRITES[name] if i < len(args)
                              for t in _flat_tensors(args[i], []) if t is not None})
        else:
            # anything not declared pure may write into any tensor argument
            mutates = [] if pure else sorted({self.by_pyid[id(t)] for t in in_tensors})
        self.nodes.append(Node(kind, name, {"l": enc_a}, {"d": enc_k}, outs, mutates, pure, alias))
        return out


def _named_tensors(model: Any) -> Tuple[Dict[int, str], Dict[Tuple, str], Dict[str, torch.Tensor]]:
    ids: Dict[int, str] = {}
    mem: Dict[Tuple, str] = {}
    by_name: Dict[str, torch.Tensor] = {}
    if isinstance(model, torch.nn.Module):
        for n, t in list(model.named_parameters(remove_duplicate=False)) + list(model.named_buffers(remove_duplicate=False)):
            if id(t) in ids:
                continue                                           # tied weights keep their first name
            ids[id(t)] = n
            by_name[n] = t
            key = _Recorder._mem_key(t)
            if key[0]:
                mem.setdefault(key, n)
    return ids, mem, by_name


def record(model: Callable, example_inputs: Sequence[torch.Tensor], input_names: Optional[Sequence[str]] = None,
           call_with_kwargs: bool = False) -> LaunchPlan:
    """Run ``model(*example_inputs)`` once (under ``no_grad``) and return its :class:`LaunchPlan`, with the constants bound
    to the live tensors of ``model`` (weights, buffers, captured tables)."""
    from ..ops import _ext

    if active_recorder() is not None:
        raise PlanError("a recording is already active")
    names = list(input_names) if input_names is not None else [f"arg{i}" for i in range(len(example_inputs))]
    ids, mem, _ = _named_tensors(model)
    ckpt_keys = set(model.state_dict().keys()) if isinstance(model, torch.nn.Module) else None
    rec = _Recorder(ids, mem, ckpt_keys)
    inputs = [{"id": rec.bind_input(t), "name": n, "shape": list(t.shape), "dtype": str(t.dtype).split(".", 1)[1]}
              for n, t in zip(names, example_inputs)]
    real = _ext._load()
    set_recorder(rec)
    _ext._PLAN_PROXY = _ExtProxy(real, rec) if real is not None else None
    try:
        with torch.no_grad(), rec:
            out = model(**dict(zip(names, example_inputs))) if call_with_kwargs else model(*example_inputs)
    finally:
        set_recorder(None)
        _ext._PLAN_PROXY = None
    outputs = _encode(out, rec.ref)
    dev_types = [t.device.type for t in example_inputs]
    device_type = "cuda" if "cuda" in dev_types else (dev_types[0] if dev_types else "cpu")
    consts = {vid: info for vid, (info, _) in rec.constants.items()}
    taken: Dict[str, int] = {}
    for vid, info in consts.items():                               # names must be unique inside one plan
        if info.name in taken:
            info.name = f"{info.name}#{vid}"
        taken[info.name] = vid
    plan = LaunchPlan(rec.nodes, inputs, outputs, consts, device_type,
                      {"py_modules": sorted(rec.py_modules), "baked_scalars": rec.baked, "warnings": rec.warnings,
                       "value_specs": {k: [list(s), d] for k, (s, d) in rec.specs.items()}})
    plan.tensors = {vid: t for vid, (_, t) in rec.constants.items()}
    for t in plan.tensors.values():
        if t.device.type == device_type:
            plan.device = t.device
            break
    if plan.device is None and example_inputs:
        plan.device = example_inputs[0].device
    return plan


# ---------------------------------------------------------------------------------------------------------------------
# multi-bucket artefact on disk
# ---------------------------------------------------------------------------------------------------------------------
def save_plans(path: str, plans: Dict[str, LaunchPlan], rank: int = 0, extra: Optional[Dict[str, Any]] = None,
               save_weights: bool = True) -> None:
    """``<path>/plans_rank<r>.json`` (all buckets) + ``<path>/constants_rank<r>.safetensors`` (one copy of every named
    constant — buckets share them — and each bucket's anonymous captures under ``<key>::<name>``).  Derived constants
    (outputs of a layout transformer) are not stored: they are recomputed at load.  ``save_weights=False`` leaves out the
    ``state_dict`` entries that no bucket writes to (the checkpoint weights: supply them with ``set_weights`` after loading);
    non-persistent buffers and captured tables are always stored."""
    from ..utils.safetensors_utils import save_state_dict_safetensors

    os.makedirs(path, exist_ok=True)
    tensors: Dict[str, torch.Tensor] = {}
    state: Set[str] = set()
    for plan in plans.values():
        state.update(plan.state_names())
    for key, plan in plans.items():
        derived = set(plan.meta.get("derived_ids", [])) if not plan.meta.get("is_transformer") else set()
        for vid, c in plan.constants.items():
            if vid in derived and c.name.startswith("_derived_"):
                continue
            if not save_weights and c.named and c.in_checkpoint and c.name not in state:
                continue
            if vid not in plan.tensors:
                raise PlanError(f"bucket {key}: constant {c.name} has no tensor to save")
            name = c.name if c.named else f"{key}::{c.name}"
            t = plan.tensors[vid]
            if name in tensors and tensors[name].data_ptr() != t.data_ptr():
                raise PlanError(f"two different tensors are named {name!r}")
            tensors[name] = t
    save_state_dict_safetensors({k: v.detach().contiguous() for k, v in tensors.items()},
                                os.path.join(path, f"constants_rank{rank}.safetensors"))
    with open(os.path.join(path, f"plans_rank{rank}.json"), "w") as f:
        json.dump({"plans": {k: p.to_json() for k, p in plans.items()}, "extra": extra or {}}, f)


def load_plans(path: str, rank: int = 0, device: Optional[torch.device] = None
               ) -> Tuple[Dict[str, LaunchPlan], Dict[str, torch.Tensor], Dict[str, Any]]:
    from ..utils.safetensors_utils import load_state_dict_safetensors

    with open(os.path.join(path, f"plans_rank{rank}.json")) as f:
        blob = json.load(f)
    dev = device or (torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu"))
    raw = load_state_dict_safetensors(os.path.join(path, f"constants_rank{rank}.safetensors"))
    plans = {k: LaunchPlan.from_json(p) for k, p in blob["plans"].items()}
    host: Set[str] = set()                                         # constants that lived on the host in a device plan
    for key, plan in plans.items():
        for c in plan.constants.values():
            if c.device_type and c.device_type != plan.device_type:
                host.add(c.name if c.named else f"{key}::{c.name}")
    tensors: Dict[str, torch.Tensor] = {name: (t if name in host else t.to(dev)) for name, t in raw.items()}
    for key, plan in plans.items():
        mine = {}
        for c in plan.constants.values():
            n = c.name if c.named else f"{key}::{c.name}"
            if n in tensors:
                mine[c.name] = tensors[n]
        plan.bind(mine, strict=False)
        plan.device = dev
    return plans, tensors, blob.get("extra", {})
