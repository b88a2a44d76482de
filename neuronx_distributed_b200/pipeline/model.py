"""Pipeline-parallel engine.

Capability parity with reference ``pipeline/model.py`` (``NxDPPModel`` :74-2038): FX-trace (or
manual) partition into stages, 1F1B / interleaved / inference schedules, micro-batching, p2p of
stage IO, tied-weight handling, loss extraction, ``local_*`` accessors with original parameter
names, ``_debug_mode`` for partition-only tests.

H100 design (differs from the XLA engine):
* eager CUDA — no graph breaks / mark_step; every task is ordinary stream-ordered work;
* stage IO goes over NCCL ``batch_isend_irecv`` (one group per schedule step) on NCCL's stream and is
  awaited just-in-time, so activation/gradient transfers overlap the neighbouring compute;
* tensor metadata is exchanged lazily, once per (direction, chunk), over the gloo PP group;
* inputs may be device tensors (the reference requires CPU tensors, model.py:1113-1120).
"""
from __future__ import annotations

import contextlib
from typing import Any, Callable, Dict, List, Optional, Tuple, Type

import torch
import torch.distributed as dist
from torch import nn

from ..utils.profiling import nvtx_range
from ..parallel_layers import comm as pl_comm
from ..parallel_layers import grads as pl_grads
from ..parallel_layers import parallel_state as ps
from ..utils import get_device
from ..utils.logger import get_logger
from ..utils.serialization import SerializationManager, find_loss_from_output_and_spec
from . import partition as part
from .comm import P2PBatch, TensorMeta, recv_python_object, send_python_object
from .scheduler import (
    BackwardPostprocessTask,
    BackwardPreprocessTask,
    BackwardStepTask,
    ForwardPostprocessTask,
    ForwardPreprocessTask,
    ForwardStepTask,
    InferenceSchedule,
    ReduceGradsTask,
    Train1F1BSchedule,
    TrainInterleavedSchedule,
)
from .timeline import PPTimeline

logger = get_logger()


class _Stage:
    """One pipeline stage (model chunk) held by this rank."""

    def __init__(self, index: int, module: nn.Module, io: part.StageIO):
        self.index, self.module, self.io = index, module, io


@contextlib.contextmanager
def mark_timeline(timeline, msg: str):
    """``with mark_timeline(tl, "fwd mb3"): …`` brackets an event (reference pipeline/model.py:61-67)."""
    timeline.mark_event_start(msg)
    try:
        yield
    finally:
        timeline.mark_event_end(msg)


# keyword names of the two batch entries a manually partitioned model is driven with (reference model.py:70-71; the
# misspelling is the reference's public name)
INPUTS_ARG_NAME = "inputs"
LABLES_ARG_NAME = "labels"


class NxDPPModel(nn.Module):
    def __init__(
        self,
        module: nn.Module,
        transformer_layer_cls: Optional[Type] = None,
        num_microbatches: int = 1,
        virtual_pipeline_size: int = 1,
        output_loss_value_spec: Any = None,
        return_mb_loss: bool = False,
        broadcast_and_average_loss: bool = False,
        pipeline_cuts: Optional[List[str]] = None,
        input_names: Optional[List[str]] = None,
        leaf_module_cls: Optional[List[Any]] = None,
        autowrap_functions: Optional[Tuple[Callable, ...]] = None,
        autowrap_modules: Optional[Tuple[Any, ...]] = None,
        autowrap_obj_methods: Optional[Dict[Any, List[Callable]]] = None,
        tracer_cls: Any = None,
        param_init_fn: Optional[Callable] = None,
        trace_file_path: Optional[str] = None,
        use_zero1_optimizer: bool = False,
        auto_partition: bool = False,
        deallocate_pipeline_outputs: bool = False,
        use_model_wrapper: bool = False,
        use_optimizer_wrapper: bool = False,
        return_loss_on_cpu: bool = False,
        fuse_microbatches: bool = False,
        manual_pp_partition: bool = False,
        manual_pp_stage_partition_fn: Optional[Callable] = None,
        manual_pp_loss_fn: Optional[Callable] = None,
        _turn_off_odd_even_scheduler: bool = False,
        _all_reduce_send_recv: bool = False,
        _fused_send_recv: bool = False,
        _fused_fwd_bwd: bool = False,
        _mark_step_before_pp_runtime: bool = True,
        _mark_step_after_pp_runtime: bool = True,
        _deallocate_send_tensors: bool = True,
        _use_gloo_for_metadata_comm: bool = False,
        _debug_mode: bool = False,
        _debug_pp_size: int = 8,
        _debug_pp_rank: int = 0,
        _delay_tracing: bool = False,
    ):
        super().__init__()
        self.original_torch_module = module
        self.transformer_layer_cls = transformer_layer_cls
        self.num_microbatches = num_microbatches
        self.virtual_pipeline_size = virtual_pipeline_size
        self.output_loss_value_spec = output_loss_value_spec
        self.return_mb_loss, self.broadcast_and_average_loss = return_mb_loss, broadcast_and_average_loss
        self.pipeline_cuts = list(pipeline_cuts) if pipeline_cuts else []
        self.input_names = input_names
        self.leaf_module_cls = list(leaf_module_cls or [])
        self.autowrap_functions, self.autowrap_modules = tuple(autowrap_functions or ()), tuple(autowrap_modules or ())
        self.tracer_cls, self.param_init_fn = tracer_cls, param_init_fn
        self.use_zero1_optimizer, self.auto_partition = use_zero1_optimizer, auto_partition
        self.use_model_wrapper, self.use_optimizer_wrapper = use_model_wrapper, use_optimizer_wrapper
        self.return_loss_on_cpu, self.deallocate_pipeline_outputs = return_loss_on_cpu, deallocate_pipeline_outputs
        self.manual_pp_partition = manual_pp_partition
        self.manual_pp_stage_partition_fn, self.manual_pp_loss_fn = manual_pp_stage_partition_fn, manual_pp_loss_fn
        self._debug_mode = _debug_mode
        # delayed tracing (reference model.py:210-232): with no ``input_names`` the traced inputs are taken from the keyword
        # arguments of the FIRST run_train / run_eval call — partitioning waits for that batch
        self._delay_tracing = bool(_delay_tracing) and input_names is None and not manual_pp_partition
        self.pp_size = _debug_pp_size if _debug_mode else ps.get_pipeline_model_parallel_size()
        self.pp_rank = _debug_pp_rank if _debug_mode else ps.get_pipeline_model_parallel_rank()
        self.num_stages = self.pp_size * virtual_pipeline_size
        self.serializer = SerializationManager()
        self.timeline = PPTimeline(trace_file_path, self.pp_rank)
        self.partitioned = False
        self.model_moved_to_device = False
        self.shape_meta: Dict[Tuple[str, int], Any] = {}
        self.local_name_to_original_name: Dict[str, str] = {}
        self.original_name_to_local_name: Dict[str, str] = {}
        self.shared_weight_groups: List[Dict[str, Any]] = []
        self.stages: List[_Stage] = []
        self.local_stage_modules = nn.ModuleList()
        self._losses: List[torch.Tensor] = []
        self.training_mode = True
        if auto_partition and transformer_layer_cls is None and not manual_pp_partition:
            raise ValueError("auto_partition needs transformer_layer_cls (the block class whose instances are distributed over the stages)")
        if manual_pp_partition:
            self._manual_partition()
        elif self._delay_tracing:
            pass                                                    # first batch decides the input names
        elif transformer_layer_cls is not None or self.pipeline_cuts:
            self.trace_and_partition()

    # =================================================================== partition
    def _layer_names(self) -> List[str]:
        return [n for n, m in self.original_torch_module.named_modules()
                if self.transformer_layer_cls is not None and isinstance(m, self.transformer_layer_cls)]

    def trace_and_partition(self) -> None:
        model = self.original_torch_module
        layers = self._layer_names()
        if self.auto_partition or not self.pipeline_cuts:
            cuts_idx = part.create_partitions(len(layers), self.num_stages)
            self.pipeline_cuts = [layers[i] for i in cuts_idx]
        assert len(self.pipeline_cuts) == self.num_stages - 1, (
            f"need {self.num_stages - 1} pipeline cuts for {self.num_stages} stages, got {self.pipeline_cuts}")
        leaf = list(self.leaf_module_cls) + ([self.transformer_layer_cls] if self.transformer_layer_cls else [])
        traced = part.trace_model(model, self.input_names, leaf, self.autowrap_functions, self.autowrap_modules,
                                  self.tracer_cls)
        self.traced_model = traced
        split = part.partition_traced_model(traced, self.pipeline_cuts, self.num_stages)
        ios, final_outputs = part.analyze_pipeline_module(split)
        # parameters/buffers touched directly by the root forward (not through a leaf module) are re-homed onto the
        # stage that uses them so they are owned, moved and optimised with that stage
        import operator

        for s_idx, io in enumerate(ios):
            sub = getattr(split, f"submod_{s_idx}")
            for arg_name, target in io.attr_args.items():
                val = operator.attrgetter(target)(split)
                holder = "_pp_attr_" + arg_name
                if isinstance(val, nn.Parameter):
                    sub.register_parameter(holder, val)
                else:
                    sub.register_buffer(holder, val)
        self.final_output_names = final_outputs
        self._output_spec = self._capture_output_spec(split)
        self.model_input_names = [n.name for n in split.graph.nodes if n.op == "placeholder"]
        stage_modules = [getattr(split, f"submod_{i}") for i in range(self.num_stages)]
        shared = part.analyze_shared_weights_across_stages(split, stage_modules)
        self._register_stages(stage_modules, ios, shared)

    @staticmethod
    def _capture_output_spec(split) -> Any:
        for node in split.graph.nodes:
            if node.op == "output":
                return torch.fx.node.map_arg(node.args[0], lambda n: n.name)
        return None

    def _manual_partition(self) -> None:
        from .manual_pipe_stage import PipelineStageModule

        model = self.original_torch_module
        assert isinstance(model, PipelineStageModule) or self.manual_pp_stage_partition_fn is not None, (
            "manual_pp_partition needs a PipelineStageModule or manual_pp_stage_partition_fn")
        stage_modules, ios = [], []
        for s in range(self.num_stages):
            if part.stage_to_pipeline_parallel_rank(s, self.pp_size) == self.pp_rank:
                m = (self.manual_pp_stage_partition_fn(model, self.num_stages, s) if self.manual_pp_stage_partition_fn
                     else model.build_stage(self.num_stages, s))
            else:
                m = None
            stage_modules.append(m)
            io = part.StageIO()
            io.inputs_from_prev = ["hidden"] if s > 0 else []
            io.outputs_to_next = ["hidden"] if s < self.num_stages - 1 else []
            io.produces = ["hidden"]
            io.call_args = ["hidden"] if s > 0 else []
            ios.append(io)
        self.model_input_names = list(self.input_names or [])
        self.final_output_names = ["hidden"]
        self._output_spec = "hidden"
        self._manual = True
        shared = model.shared_across_stages(self.num_stages) if isinstance(model, PipelineStageModule) \
            and not self.manual_pp_stage_partition_fn else []
        self._register_stages(stage_modules, ios, shared)

    def _register_stages(self, stage_modules: List[Optional[nn.Module]], ios: List[part.StageIO], shared) -> None:
        self.stage_ios = ios
        names_of: Dict[int, List[str]] = {}
        for n, p in self.original_torch_module.named_parameters(remove_duplicate=False):
            names_of.setdefault(id(p), []).append(n)

        def _orig_name(p, local_leaf: str) -> str:
            cands = names_of.get(id(p), [])
            for c in cands:  # a tied parameter keeps the name it has inside *this* stage's module
                if c.endswith(local_leaf) or local_leaf.endswith(c):
                    return c
            return cands[0] if cands else local_leaf

        name_of_buf = {id(b): n for n, b in self.original_torch_module.named_buffers(remove_duplicate=False)}
        for s, m in enumerate(stage_modules):
            if part.stage_to_pipeline_parallel_rank(s, self.pp_size) != self.pp_rank or m is None:
                continue
            chunk = len(self.stages)
            self.stages.append(_Stage(s, m, ios[s]))
            self.local_stage_modules.append(m)
            for ln, p in m.named_parameters(remove_duplicate=False):
                local = f"local_stage_modules.{chunk}.{ln}"
                orig = _orig_name(p, ln)
                self.local_name_to_original_name[local] = orig
                self.original_name_to_local_name[orig] = local
            for ln, b in m.named_buffers(remove_duplicate=False):
                local = f"local_stage_modules.{chunk}.{ln}"
                self.local_name_to_original_name[local] = name_of_buf.get(id(b), ln)
        # tied weights living on several stages → process groups + `shared` flag on all but the first
        for group in shared:
            stages = sorted({s for s, _ in group})
            ranks_pp = sorted({part.stage_to_pipeline_parallel_rank(s, self.pp_size) for s in stages})
            if len(ranks_pp) < 2:
                continue
            entry = {"stages": stages, "pp_ranks": ranks_pp, "param": None, "pg": None}
            for s, lname in group:
                if part.stage_to_pipeline_parallel_rank(s, self.pp_size) == self.pp_rank:
                    mod = stage_modules[s]
                    p = dict(mod.named_parameters(remove_duplicate=False))[lname]
                    entry["param"] = p
                    if s != stages[0]:
                        p.shared = True
            self.shared_weight_groups.append(entry)
        if not self._debug_mode and self.shared_weight_groups:
            self._create_shared_weight_groups()
        self.partitioned = True
        # drop the reference to non-local stage modules so their parameters can be freed
        self.num_local_chunks = len(self.stages)

    def _create_shared_weight_groups(self) -> None:
        pp_groups = ps.get_pipeline_model_parallel_replica_groups()
        for entry in self.shared_weight_groups:
            mine = None
            for ranks in pp_groups:  # every rank creates every group, in the same order
                sub = [ranks[r] for r in entry["pp_ranks"]]
                pg = ps.create_pg_with_ranks(sub)
                if dist.get_rank() in sub:
                    mine = pg
            entry["pg"] = mine

    # =================================================================== device / weights
    def move_model_to_device(self) -> None:
        if self.model_moved_to_device:
            return
        from ..parallel_layers.utils import move_model_to_device

        dev = get_device()
        for st in self.stages:
            if any(p.device.type == "meta" for p in st.module.parameters()):
                from ..utils.model_utils import reinit_model

                reinit_model(st.module, dev, self.param_init_fn)
            else:
                move_model_to_device(st.module, dev)
        self.model_moved_to_device = True
        self._nxd_on_device = True
        self._sync_shared_weights()

    def _sync_shared_weights(self) -> None:
        for e in self.shared_weight_groups:
            if e["param"] is None or e["pg"] is None:
                continue
            p = e["param"]
            with torch.no_grad():
                if not getattr(p, "shared", False):
                    pass
                else:
                    p.zero_()
                dist.all_reduce(p.data, group=e["pg"])

    def _reduce_shared_weight_grads(self) -> None:
        for e in self.shared_weight_groups:
            p = e["param"]
            if p is None or e["pg"] is None:
                continue
            g = p.grad if p.grad is not None else getattr(p, "main_grad", None)
            if g is None:
                g = torch.zeros_like(p)
                p.grad = g
            dist.all_reduce(g, group=e["pg"])

    # =================================================================== public run API
    def forward(self, *args, **kwargs):
        raise RuntimeError("NxDPPModel: call run_train(**batch) or run_eval(**batch), not forward()")

    def train(self, mode: bool = True):
        self.training_mode = mode
        return super().train(mode)

    def run_train(self, **kwargs):
        self.train(True)
        return self._run(kwargs, train=True)

    def run_eval(self, **kwargs):
        self.train(False)
        with torch.no_grad():
            return self._run(kwargs, train=False)

    def _make_schedule(self, train: bool):
        n = self.num_microbatches
        if not train:
            return InferenceSchedule(n, self.pp_size, self.pp_rank, self.virtual_pipeline_size)
        if self.virtual_pipeline_size > 1:
            return TrainInterleavedSchedule(n, self.virtual_pipeline_size, self.pp_size, self.pp_rank)
        return Train1F1BSchedule(n, self.pp_size, self.pp_rank)

    def _split_microbatches(self, kwargs: Dict[str, Any]) -> List[Dict[str, Any]]:
        n = self.num_microbatches
        mbs: List[Dict[str, Any]] = [dict() for _ in range(n)]
        for k, v in kwargs.items():
            if isinstance(v, torch.Tensor) and v.dim() > 0:
                assert v.shape[0] % n == 0, f"batch dim {v.shape[0]} of {k} not divisible by {n} microbatches"
                for i, piece in enumerate(v.chunk(n, dim=0)):
                    mbs[i][k] = piece.to(get_device(), non_blocking=True)
            else:
                for i in range(n):
                    mbs[i][k] = v
        return mbs

    def _run(self, kwargs: Dict[str, Any], train: bool):
        if not self.partitioned and self._delay_tracing:
            self.perform_delayed_tracing_and_partition(**kwargs)
            self.move_model_to_device()
        assert self.partitioned, "model is not partitioned"
        self.move_model_to_device()
        self._mbs = self._split_microbatches(kwargs)
        self._act: Dict[Tuple[int, int], Dict[str, torch.Tensor]] = {}     # (mb, chunk) → named stage inputs
        self._out: Dict[Tuple[int, int], Dict[str, torch.Tensor]] = {}     # (mb, chunk) → named outputs (sent fwd)
        self._inp_leaves: Dict[Tuple[int, int], Dict[str, torch.Tensor]] = {}
        self._grad_in: Dict[Tuple[int, int], Dict[str, torch.Tensor]] = {}
        self._pending: List[Any] = []
        self._pending_sends: List[Any] = []
        self._losses = []
        self._train = train
        group = None if self._debug_mode else ps.get_pipeline_model_parallel_group()
        for step in self._make_schedule(train):
            batch = P2PBatch(group)
            for task in step:
                self._dispatch(task, batch)
            self._flush(batch)
        self._wait_all()
        self._drain_sends()
        self.timeline.mark_step_end()               # one trace dump per run_train / run_eval call (no-op without trace_file_path)
        return self._process_loss()

    # ------------------------------------------------------------------ task dispatch
    def _dispatch(self, task, batch: P2PBatch) -> None:
        if isinstance(task, ReduceGradsTask):
            self._flush(batch)
            return self._reduce_grads()
        name = type(task).__name__
        label = f"{name}_mb{task.mb}_c{task.model_chunk}"
        self.timeline.mark_event_start(label)
        with nvtx_range(label):
            self._dispatch_task(task, batch)
        self.timeline.mark_event_end(label)

    def _dispatch_task(self, task, batch: P2PBatch) -> None:
        if isinstance(task, ForwardPreprocessTask):
            self._fwd_pre(task, batch)
        elif isinstance(task, ForwardStepTask):
            self._flush(batch)
            self._fwd_step(task)
        elif isinstance(task, ForwardPostprocessTask):
            self._fwd_post(task, batch)
        elif isinstance(task, BackwardPreprocessTask):
            self._bwd_pre(task, batch)
        elif isinstance(task, BackwardStepTask):
            self._flush(batch)
            self._bwd_step(task)
        elif isinstance(task, BackwardPostprocessTask):
            self._bwd_post(task, batch)

    def _flush(self, batch: P2PBatch) -> None:
        recv_works, send_works = batch.launch()
        self._pending.extend(recv_works)
        if send_works or batch.keep:
            self._pending_sends.append((send_works, list(batch.keep)))   # keeps sent tensors alive
            batch.keep.clear()

    def _wait_all(self) -> None:
        """Block only on *received* data; sends complete in the background (waiting on a send here could
        deadlock two neighbours that each wait for the other to post its receive)."""
        for w in self._pending:
            w.wait()
        self._pending.clear()

    def _drain_sends(self) -> None:
        for works, _keep in self._pending_sends:
            for w in works:
                w.wait()
        self._pending_sends.clear()

    # ------------------------------------------------------------------ helpers
    def _stage(self, chunk: int) -> _Stage:
        return self.stages[chunk]

    def _global_stage(self, chunk: int) -> int:
        return self.stages[chunk].index

    def _prev_rank(self) -> int:
        return ps.get_pipeline_model_parallel_prev_rank()

    def _next_rank(self) -> int:
        return ps.get_pipeline_model_parallel_next_rank()

    def _meta_exchange_send(self, key: Tuple[str, int], tensors: Dict[str, torch.Tensor], dst: int) -> None:
        if key in self.shape_meta:
            return
        metas = {n: TensorMeta(i, t.dtype, t.shape, t.requires_grad) for i, (n, t) in enumerate(tensors.items())}
        send_python_object(metas, dst)
        self.shape_meta[key] = metas

    def _meta_exchange_recv(self, key: Tuple[str, int], src: int) -> Dict[str, TensorMeta]:
        if key not in self.shape_meta:
            self.shape_meta[key] = recv_python_object(src)
        return self.shape_meta[key]

    # ------------------------------------------------------------------ forward
    def _fwd_pre(self, task, batch: P2PBatch) -> None:
        st = self._stage(task.model_chunk)
        if st.index == 0 or not st.io.inputs_from_prev:
            return
        self._flush(batch)  # metadata handshake must not sit behind an unlaunched group
        metas = self._meta_exchange_recv(("fwd", st.index), self._prev_rank())
        bufs = {n: batch.recv(m, self._prev_rank()) for n, m in metas.items()}
        self._act[(task.mb, task.model_chunk)] = bufs
        self._recv_req = {n: m.requires_grad for n, m in metas.items()}

    def _fwd_step(self, task) -> None:
        self._wait_all()
        st = self._stage(task.model_chunk)
        key = (task.mb, task.model_chunk)
        recvd = self._act.pop(key, {})
        metas = self.shape_meta.get(("fwd", st.index), {})
        leaves = {}
        for n, t in recvd.items():
            if self._train and t.is_floating_point() and getattr(metas.get(n), "requires_grad", True):
                t.requires_grad_(True)
            leaves[n] = t
        self._inp_leaves[key] = leaves
        mb = self._mbs[task.mb]
        if getattr(self, "_manual", False):
            if st.index == 0:
                out = st.module(**{k: mb[k] for k in self.model_input_names if k in mb}) if self.model_input_names \
                    else st.module(**mb)
            else:
                out = st.module(leaves["hidden"])
            named = {"hidden": out}
            if st.index == self.num_stages - 1 and self.manual_pp_loss_fn is not None:
                labels = mb.get(LABLES_ARG_NAME)
                named = {"hidden": self.manual_pp_loss_fn(out, labels)}
        else:
            args = [leaves[a] if a in leaves else
                    (getattr(st.module, "_pp_attr_" + a) if a in st.io.attr_args else mb.get(a)) for a in st.io.call_args]
            out = st.module(*args)
            named = {n: (out if idx is None else out[idx]) for n, idx in st.io.produces}
        # forward everything the next stage needs: own products + pass-along values
        outgoing = {}
        for n in st.io.outputs_to_next:
            if n in named and named[n] is not None:
                outgoing[n] = named[n]
            elif n in leaves:
                outgoing[n] = leaves[n]
        self._out[key] = {"named": named, "outgoing": outgoing}
        if st.index == self.num_stages - 1:
            loss = self._extract_loss(named)
            if loss is not None:
                self._losses.append(loss if self._train else loss.detach())
                self._out[key]["loss"] = loss

    def _extract_loss(self, named: Dict[str, Any]) -> Optional[torch.Tensor]:
        if getattr(self, "_manual", False):
            out = named["hidden"]
        else:
            def build(spec):
                if isinstance(spec, str):
                    return named.get(spec)
                if isinstance(spec, (tuple, list)):
                    return type(spec)(build(s) for s in spec)
                if isinstance(spec, dict):
                    return {k: build(v) for k, v in spec.items()}
                return spec
            out = build(self._output_spec)
        self._last_output = out
        if not self._train and self.output_loss_value_spec is None and not isinstance(out, torch.Tensor):
            return None
        try:
            return find_loss_from_output_and_spec(out, self.output_loss_value_spec)
        except Exception:
            return None

    def _fwd_post(self, task, batch: P2PBatch) -> None:
        st = self._stage(task.model_chunk)
        if st.index == self.num_stages - 1:
            return
        rec = self._out.get((task.mb, task.model_chunk))
        if rec is None:
            return
        outgoing = rec["outgoing"]
        self._flush(batch)
        self._meta_exchange_send(("fwd", st.index + 1), outgoing, self._next_rank())
        for n, t in outgoing.items():
            batch.send(t.detach(), self._next_rank())

    # ------------------------------------------------------------------ backward
    def _bwd_pre(self, task, batch: P2PBatch) -> None:
        st = self._stage(task.model_chunk)
        if st.index == self.num_stages - 1:
            return
        self._flush(batch)
        metas = self._meta_exchange_recv(("bwd", st.index), self._next_rank())
        self._grad_in[(task.mb, task.model_chunk)] = {n: batch.recv(m, self._next_rank()) for n, m in metas.items()}

    def _bwd_step(self, task) -> None:
        self._wait_all()
        st = self._stage(task.model_chunk)
        key = (task.mb, task.model_chunk)
        rec = self._out.pop(key)
        if st.index == self.num_stages - 1:
            loss = rec["loss"]
            (loss / self.num_microbatches).backward()
        else:
            grads = self._grad_in.pop(key)
            outs, gs = [], []
            for n, g in grads.items():
                t = rec["outgoing"][n]
                if t.requires_grad:
                    outs.append(t)
                    gs.append(g)
            if outs:
                torch.autograd.backward(outs, gs)
        self._bwd_ready = self._inp_leaves.pop(key, {})

    def _bwd_post(self, task, batch: P2PBatch) -> None:
        st = self._stage(task.model_chunk)
        if st.index == 0:
            return
        leaves = self._bwd_ready
        grads = {n: (t.grad if t.grad is not None else torch.zeros_like(t)) for n, t in leaves.items()
                 if t.is_floating_point() and t.requires_grad}
        self._flush(batch)
        self._meta_exchange_send(("bwd", st.index - 1), grads, self._prev_rank())
        for n, g in grads.items():
            batch.send(g, self._prev_rank())

    # ------------------------------------------------------------------ post
    def _reduce_grads(self) -> None:
        self._wait_all()
        if not self.use_zero1_optimizer and not self.use_optimizer_wrapper and ps.get_data_parallel_size() > 1:
            gl = [p.grad for p in self.local_parameters() if p.grad is not None]
            pl_grads.bucket_allreduce_gradients(gl)
        self._reduce_shared_weight_grads()

    def _process_loss(self):
        is_last = self.pp_rank == self.pp_size - 1
        if not self._losses:
            loss = None
        elif self.return_mb_loss:
            loss = [l.detach() for l in self._losses]
        else:
            loss = torch.stack([l.detach().float() for l in self._losses]).mean()
        if self.broadcast_and_average_loss and not self._debug_mode:
            t = loss if (is_last and isinstance(loss, torch.Tensor)) else torch.zeros((), device=get_device())
            t = t.clone()
            if ps.get_context_model_parallel_size() > 1:
                pl_comm.all_reduce(t, op="avg", group=ps.get_context_model_parallel_group())
            if ps.get_data_parallel_size() > 1:
                pl_comm.all_reduce(t, op="avg", group=ps.get_data_parallel_group())
            if not is_last:
                t.zero_()
            pl_comm.all_reduce(t, group=ps.get_pipeline_model_parallel_group())
            loss = t
        if self.return_loss_on_cpu and isinstance(loss, torch.Tensor):
            loss = loss.cpu()
        if not self._train and loss is None and is_last:
            return getattr(self, "_last_output", None)
        return loss

    # =================================================================== local accessors
    def local_named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True):
        seen = set()
        for name, p in self.local_stage_modules.named_parameters(prefix="local_stage_modules", recurse=recurse):
            if remove_duplicate and id(p) in seen:
                continue
            seen.add(id(p))
            yield prefix + self.local_name_to_original_name.get(name, name), p

    def local_parameters(self, recurse: bool = True):
        for _, p in self.local_named_parameters(recurse=recurse):
            yield p

    def parameters(self, recurse: bool = True):
        return self.local_parameters(recurse)

    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True):
        return self.local_named_parameters(prefix, recurse, remove_duplicate)

    def local_named_buffers(self, prefix: str = "", recurse: bool = True):
        for name, b in self.local_stage_modules.named_buffers(prefix="local_stage_modules", recurse=recurse):
            yield prefix + self.local_name_to_original_name.get(name, name), b

    def local_modules(self):
        return self.local_stage_modules.modules()

    def local_named_modules(self, *a, **k):
        return self.local_stage_modules.named_modules(*a, **k)

    def local_children(self):
        return self.local_stage_modules.children()

    def local_state_dict(self, *args, **kwargs) -> Dict[str, Any]:
        sd = self.local_stage_modules.state_dict(prefix="local_stage_modules.")
        return {self.local_name_to_original_name.get(k, k): v for k, v in sd.items()}

    def state_dict(self, *args, **kwargs):
        return self.local_state_dict()

    def load_state_dict(self, state_dict: Dict[str, Any], strict: bool = True):
        local = {}
        for k, v in state_dict.items():
            lk = self.original_name_to_local_name.get(k)
            if lk is not None:
                local[lk[len("local_stage_modules."):]] = v
        return self.local_stage_modules.load_state_dict(local, strict=False if not strict else strict and
                                                        len(local) == len(self.local_stage_modules.state_dict()))

    def get_model_layers(self) -> List[str]:
        return self._layer_names()

    # =================================================================== reference-named entry points
    # (reference pipeline/model.py: trace :353, partition :383, cut_pipeline_stage :718, register_shared_weights :486, …)
    def trace(self, args=None, kwargs=None, input_names: Optional[List[str]] = None, leaf_modules: Optional[List[Any]] = None,
              autowrap_functions=None, autowrap_modules=None, autowrap_obj_methods=None, tracer_cls=None) -> None:
        """Record the tracing options; the FX trace itself runs together with the cut in :meth:`partition` (the graph is
        only ever needed to be split)."""
        assert not self.partitioned, "the model is already partitioned"
        if input_names is None and (args is not None or kwargs is not None):
            import inspect

            sig = list(inspect.signature(self.original_torch_module.forward).parameters)
            input_names = sig[: len(args or [])] + list((kwargs or {}).keys())
        if input_names is not None:
            self.input_names = list(input_names)
        if leaf_modules:
            self.leaf_module_cls = list(self.leaf_module_cls) + [m for m in leaf_modules if isinstance(m, type)]
        self.autowrap_functions = tuple(autowrap_functions or self.autowrap_functions)
        self.autowrap_modules = tuple(autowrap_modules or self.autowrap_modules)
        self.tracer_cls = tracer_cls or self.tracer_cls
        self._traced_requested = True

    def cut_pipeline_stage(self, cut_point: str) -> None:
        """Add a cut AFTER the module named ``cut_point`` (must be called before :meth:`partition`)."""
        assert not self.partitioned, "cut_pipeline_stage must be called before the model is partitioned"
        names = {n for n, _ in self.original_torch_module.named_modules()}
        assert cut_point in names, f"{cut_point} is not a module of the model"
        if cut_point not in self.pipeline_cuts:
            self.pipeline_cuts.append(cut_point)

    def partition(self) -> None:
        """Trace + split at the registered cuts and keep this rank's stage(s)."""
        if self.partitioned:
            return
        if self.manual_pp_partition:
            return self._manual_partition()
        order = {n: i for i, (n, _) in enumerate(self.original_torch_module.named_modules())}
        self.pipeline_cuts.sort(key=lambda c: order.get(c, 0))
        self.trace_and_partition()

    def perform_delayed_tracing_and_partition(self, *args, **kwargs) -> None:
        """Trace and partition now.  With delayed tracing the input names come from this call's keyword arguments (the first
        batch): FX does not need tensor shapes, only which ``forward`` parameters are tensors and which stay at their defaults."""
        if self.partitioned:
            return
        if self._delay_tracing and self.input_names is None and kwargs:
            self.input_names = [k for k, v in kwargs.items() if v is not None]
        self._delay_tracing = False
        self.partition()

    def maybe_materialize_local_module(self) -> None:
        """Give storage to this rank's stage(s) if the model was built on the meta device (and only to them)."""
        self.move_model_to_device()

    def register_shared_weights(self, weight_pairs: Optional[List[Any]] = None) -> None:
        """Tied weights are discovered from parameter identity during partitioning (``analyze_shared_weights_across_stages``);
        extra groups can be declared as lists of original parameter names, e.g. ``[["embed.weight", "lm_head.weight"]]``."""
        for names in weight_pairs or []:
            mine = [self.original_name_to_local_name[n] for n in names if n in self.original_name_to_local_name]
            params = dict(self.local_stage_modules.named_parameters(prefix="local_stage_modules", remove_duplicate=False))
            p = params[mine[0]] if mine else None
            stages = sorted({st.index for st in self.stages} if mine else set())
            self.shared_weight_groups.append({"stages": stages, "pp_ranks": list(range(self.pp_size)), "param": p, "pg": None,
                                              "names": list(names)})
        if weight_pairs and not self._debug_mode:
            self._create_shared_weight_groups()

    def create_schedule(self, train: bool = True):
        return self._make_schedule(train)

    def clear_minibatch_state(self) -> None:
        """Drop every per-step buffer (activations kept for backward, received gradients, pending handles, losses)."""
        for name in ("_act", "_out", "_inp_leaves", "_grad_in"):
            getattr(self, name, {}).clear()
        for name in ("_pending", "_pending_sends", "_losses"):
            lst = getattr(self, name, None)
            if lst is not None:
                lst.clear()
        self._mbs = []

    def get_current_stage(self, model_chunk_id: int = 0) -> int:
        """Global stage index of local chunk ``model_chunk_id`` (``chunk · pp_size + pp_rank``)."""
        return self.stages[model_chunk_id].index if self.stages else model_chunk_id * self.pp_size + self.pp_rank

    def is_last_stage(self, model_chunk_id: Optional[int] = None) -> bool:
        chunk = len(self.stages) - 1 if model_chunk_id is None else model_chunk_id
        return self.get_current_stage(chunk) == self.num_stages - 1

    def is_last_pp_rank_last_model_chunk(self, model_chunk_id: int) -> bool:
        return self.pp_rank == self.pp_size - 1 and model_chunk_id == self.virtual_pipeline_size - 1

    def get_batch_iterator(self, batch: Dict[str, Any]):
        """Iterator over the micro-batches of ``batch`` (dim 0 split into ``num_microbatches`` equal parts)."""
        return iter(self._split_microbatches(batch))

    @staticmethod
    def custom_backward(outputs: torch.Tensor, grad_outputs: Optional[torch.Tensor]) -> None:
        """Backward through ``output`` even after its storage was released by :meth:`maybe_deallocate_output_tensor` — the
        autograd engine only needs the graph, not the values (reference :890-925, after Megatron-LM)."""
        output, grad_output = outputs, grad_outputs      # reference parameter names in the signature
        assert output.numel() == 1 or grad_output is not None or output.numel() > 0
        if grad_output is None:
            assert output.numel() == 1, "implicit grad requires scalar output."
            grad_output = torch.ones_like(output, memory_format=torch.preserve_format)
        torch.autograd.backward((output,), (grad_output,))

    def maybe_deallocate_output_tensor(self, model_chunk: int = 0) -> None:
        """After a stage's outputs were sent downstream, free their storage (only the autograd graph is needed for the
        backward of this stage): enabled by ``deallocate_pipeline_outputs``."""
        model_chunk_id = model_chunk      # reference parameter names in the signature
        if not self.deallocate_pipeline_outputs:
            return
        for (mb, chunk), outs in list(getattr(self, "_out", {}).items()):
            if chunk != model_chunk_id:
                continue
            for t in outs.values():
                if isinstance(t, torch.Tensor) and t._base is None and t.requires_grad:
                    t.data = torch.empty((1,), device=t.device, dtype=t.dtype)

    # ---- full-module style accessors (a pipeline rank sees its local stage modules) ----------------------------------
    def named_buffers(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True):
        return self.local_named_buffers(prefix, recurse)

    def buffers(self, recurse: bool = True):
        for _, b in self.local_named_buffers(recurse=recurse):
            yield b

    def local_buffers(self, recurse: bool = True):
        return self.buffers(recurse)

    def local_named_children(self):
        return self.local_stage_modules.named_children()

    def translate_origin_state_dict_to_local_state_dict(self, origin_state_dict: Dict[str, Any]) -> Dict[str, Any]:
        """Keys of the un-partitioned model → keys of ``local_stage_modules`` (entries of other stages are dropped)."""
        out = {}
        for k, v in origin_state_dict.items():
            lk = self.original_name_to_local_name.get(k)
            if lk is None:
                lk = next((loc for loc, orig in self.local_name_to_original_name.items() if orig == k), None)
            if lk is not None:
                out[lk] = v
        return out

    def translate_local_state_dict_to_origin_state_dict(self, local_state_dict: Dict[str, Any]) -> Dict[str, Any]:
        return {self.local_name_to_original_name.get(k, k): v for k, v in local_state_dict.items()}

    def construct_state_dict_per_model_chunk(self, origin_state_dict_all_model_chunks: Dict[str, Any], strict: bool = True) -> List[Dict[str, Any]]:
        """Split an original-key state dict into one dict per local model chunk (keys relative to the chunk's module)."""
        state_dict = origin_state_dict_all_model_chunks      # reference parameter names in the signature
        per_chunk: List[Dict[str, Any]] = [dict() for _ in self.stages]
        local = self.translate_origin_state_dict_to_local_state_dict(state_dict)
        for k, v in local.items():
            _, chunk, rest = k.split(".", 2)
            per_chunk[int(chunk)][rest] = v
        if strict:
            for i, st in enumerate(self.stages):
                missing = set(st.module.state_dict().keys()) - set(per_chunk[i])
                if missing:
                    raise RuntimeError(f"missing keys for model chunk {i}: {sorted(missing)[:5]}…")
        return per_chunk
