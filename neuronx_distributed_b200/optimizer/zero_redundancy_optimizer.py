"""ZeRO-1: optimizer state and fp32 master weights sharded over the data-parallel group.

Role parity with reference ``optimizer/zero_redundancy_optimizer.py`` (``NeuronZero1Optimizer``
:30, ``NeuronEPZero1Optimizer`` :163) whose base class lives in torch_xla (external, K13 in
SURVEY §2.9) — this is a from-scratch implementation designed for H100:

* **Flat contiguous buffers.**  Per (param-group, dtype) the model parameters are re-pointed
  into one flat ``param_flat`` buffer and gradients accumulate into one flat fp32 (or bf16)
  ``grad_flat`` buffer; rank r of the sharding group owns the contiguous range
  ``[r·L/n, (r+1)·L/n)``.  Reduce-scatter / all-gather are therefore single contiguous
  collectives (or single fused kernels), not per-parameter ones, and the AdamW update of the
  whole shard is ONE multi-tensor launch that also writes the bf16 parameters.
* **fp32 gradient accumulation** (``use_grad_acc_hook``): a post-accumulate hook adds each
  bf16 ``p.grad`` into the fp32 flat buffer and frees it (reference trainer.py:284-285).
* **Grad clipping on shards**: squared norms are taken on this rank's shard slices, with
  TP-duplicated parameters counted 1/tp (same rule as ``grads.get_grad_norm``), then summed over
  the sharding group and the TP (+PP, EP) groups; the clip coefficient stays on device and is
  folded into the AdamW kernel (reference zero_redundancy_optimizer.py:71-104).
* On CUDA with dp>1 the reduce-scatter(+cast+scale) and all-gather(+cast) run through the
  peer-memory kernels in ``ops/zero1_comm.py`` when available, else NCCL.

State-dict schema keeps the reference's keys — ``state``, ``base_state``, ``shape_info``,
``param_groups``, ``sharded_master_weights`` (reference :299-320; trainer/checkpoint.py:644-649);
``shape_info`` additionally records the flat ranges so shards can be re-assembled/re-sharded
offline (``optimizer/convert_zero_checkpoints.py``).
"""
from __future__ import annotations

import os

from dataclasses import dataclass
from typing import Any, Callable, Dict, Iterable, List, Optional, Tuple, Type

import torch
import torch.distributed as dist

from .. import ops
from ..parallel_layers import comm
from ..parallel_layers import parallel_state as ps
from ..utils.logger import get_logger

logger = get_logger()

_ALIGN = 128  # elements; keeps every shard boundary 256-byte aligned for vectorised kernels


@dataclass
class _ParamSlot:
    param: torch.nn.Parameter
    offset: int           # start in the flat buffer (elements)
    numel: int
    group_idx: int


class _FlatGroup:
    """Flat storage for one optimizer param-group (single model dtype)."""

    def __init__(self, params: List[torch.nn.Parameter], group_idx: int, world: int, rank: int,
                 grad_dtype: torch.dtype, master_dtype: torch.dtype, use_master: bool, arena=None):
        self.world, self.rank = world, rank
        self.slots: List[_ParamSlot] = []
        off = 0
        for p in params:
            self.slots.append(_ParamSlot(p, off, p.numel(), group_idx))
            off += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        per = (off + world - 1) // world
        per = (per + _ALIGN - 1) // _ALIGN * _ALIGN
        self.shard_numel = per
        self.total = per * world
        p0 = params[0]
        self.model_dtype, self.device = p0.dtype, p0.device
        self.group_idx, self.arena = group_idx, arena
        if arena is not None:   # peer-visible buffers for the NVLink reduce-scatter / all-gather kernels
            self.param_flat, self.param_off = arena.alloc(self.total, self.model_dtype)
            self.grad_flat, self.grad_off = arena.alloc(self.total, grad_dtype)
            self.rs_out = torch.zeros(per, dtype=torch.float32, device=self.device)
        else:
            self.param_flat = torch.zeros(self.total, dtype=self.model_dtype, device=self.device)
            self.grad_flat = torch.zeros(self.total, dtype=grad_dtype, device=self.device)
        for s in self.slots:
            view = self.param_flat[s.offset : s.offset + s.numel].view_as(s.param)
            view.copy_(s.param.data)
            s.param.data = view
            s.param.main_grad = self.grad_flat[s.offset : s.offset + s.numel].view_as(s.param)
        lo, hi = self.shard_range
        self.use_master = use_master
        if use_master:
            self.master_shard = self.param_flat[lo:hi].to(master_dtype).clone()
        else:
            self.master_shard = self.param_flat[lo:hi]
        self.grad_shard: Optional[torch.Tensor] = None  # set by reduce step

    @property
    def shard_range(self) -> Tuple[int, int]:
        return self.rank * self.shard_numel, (self.rank + 1) * self.shard_numel

    def shard_slices(self) -> List[Tuple[_ParamSlot, int, int, int]]:
        """(slot, start_in_shard, start_in_param, length) for params overlapping my shard."""
        lo, hi = self.shard_range
        out = []
        for s in self.slots:
            a, b = max(lo, s.offset), min(hi, s.offset + s.numel)
            if a < b:
                out.append((s, a - lo, a - s.offset, b - a))
        return out


class Zero1Optimizer(torch.optim.Optimizer):
    def __init__(
        self,
        params: Iterable,
        optimizer_class: Type[torch.optim.Optimizer],
        optimizer_dtype: Optional[torch.dtype] = None,
        grad_clipping: bool = True,
        max_norm: Optional[float] = None,
        pin_layout: bool = False,
        sharding_groups: Any = None,
        grad_norm_groups: Any = None,
        lazy_init: bool = False,
        coalesce_cc: bool = True,
        bucket_cap_mb_all_gather: int = 130,
        bucket_cap_mb_reduce_scatter: int = 130,
        use_grad_acc_hook: bool = False,
        higher_cc_precision: bool = False,
        save_master_weights: bool = False,
        use_master_weights: bool = True,
        process_group=None,
        grad_scale_divisor: Optional[float] = None,
        overlap_grad_reduce: Optional[bool] = None,
        overlap_ctas: int = 16,
        **defaults: Any,
    ):
        del pin_layout, grad_norm_groups, lazy_init, coalesce_cc  # XLA-only knobs
        self.base_cls = optimizer_class
        self.grad_clipping = grad_clipping
        self.max_norm = max_norm if max_norm is not None else 1.0
        self.use_grad_acc_hook = use_grad_acc_hook
        self.higher_cc_precision = higher_cc_precision
        self.save_master_weights = save_master_weights
        self.use_master_weights = use_master_weights
        self.optimizer_dtype = optimizer_dtype or torch.float32
        self.bucket_cap_rs = bucket_cap_mb_reduce_scatter * 1024 * 1024
        self.bucket_cap_ag = bucket_cap_mb_all_gather * 1024 * 1024
        self.pg = process_group if process_group is not None else (
            ps.get_zero1_sharding_group() if ps.model_parallel_is_initialized() else dist.group.WORLD)
        self.sharding_groups = sharding_groups
        self.world = dist.get_world_size(self.pg)
        self.rank = dist.get_rank(self.pg)
        self.grad_scale_divisor = float(grad_scale_divisor) if grad_scale_divisor else float(self.world)
        super().__init__(params, dict(defaults))
        self._grad_norm: Optional[torch.Tensor] = None
        self._hooks = []
        # Overlap of the gradient reduce-scatter with the backward pass (reference: bucketed reduce-scatter of the XLA
        # ZeRO optimizer, trainer.py:258-285): the flat gradient buffer is cut into contiguous buckets; when the last
        # gradient of a bucket has been produced (post-accumulate hook or the fused wgrad epilogue) its pull
        # reduce-scatter is launched on a side stream with a handful of CTAs, so it runs under the remaining backward.
        if overlap_grad_reduce is None:
            overlap_grad_reduce = os.environ.get("NXD_ZERO1_OVERLAP", "0") == "1"
        self.overlap_grad_reduce = bool(overlap_grad_reduce)
        self.overlap_ctas = int(overlap_ctas)
        self._sync_enabled = True
        self._comm_stream = None
        self._build()

    # ------------------------------------------------------------------ setup
    def _build(self) -> None:
        self.flat_groups: List[_FlatGroup] = []
        base_groups = []
        arena = None
        first = next(p for g in self.param_groups for p in g["params"])
        if first.is_cuda and ops.zero1_comm.available(self.pg):
            total = 0
            for group in self.param_groups:
                ps_ = [p for p in group["params"] if p.requires_grad]
                n = sum((p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN for p in ps_)
                per = ((n + self.world - 1) // self.world + _ALIGN - 1) // _ALIGN * _ALIGN
                gbytes = 4 if (self.use_grad_acc_hook or ps_[0].dtype == torch.float32) else ps_[0].element_size()
                total += per * self.world * (ps_[0].element_size() + gbytes) + 1024
            arena = ops.zero1_comm.Zero1Symm(self.pg, total)
        self.arena = arena
        for gi, group in enumerate(self.param_groups):
            params = [p for p in group["params"] if p.requires_grad]
            assert params, "empty param group"
            assert len({p.dtype for p in params}) == 1, "one dtype per param group"
            grad_dtype = torch.float32 if (self.use_grad_acc_hook or params[0].dtype == torch.float32) else params[0].dtype
            fg = _FlatGroup(params, gi, self.world, self.rank, grad_dtype, self.optimizer_dtype,
                            self.use_master_weights and params[0].dtype != self.optimizer_dtype, arena)
            self.flat_groups.append(fg)
            shard_param = torch.nn.Parameter(fg.master_shard, requires_grad=True)
            if fg.use_master:
                lo, hi = fg.shard_range
                shard_param._lowp_view = fg.param_flat[lo:hi]  # fused AdamW refreshes the bf16 copy
            fg.base_param = shard_param
            base_groups.append({**{k: v for k, v in group.items() if k != "params"}, "params": [shard_param]})
            for s in fg.slots:
                self._install_hook(s.param)
        self.base_optimizer = self.base_cls(base_groups, **{k: v for k, v in self.defaults.items()})
        self.base = self.base_optimizer
        self._build_buckets()

    # ------------------------------------------------------------------ overlapped (bucketed) reduce-scatter
    def _build_buckets(self) -> None:
        self._buckets = []          # (fg, begin, end, n_slots)
        self._slot_buckets = {}     # id(param) -> [bucket index]
        self._overlap_active = (self.overlap_grad_reduce and self.world > 1
                                and all(fg.arena is not None for fg in self.flat_groups))
        tp = 1
        if self._overlap_active and ps.model_parallel_is_initialized():
            tp = ps.get_tensor_model_parallel_size()
            # context parallel averages EVERY gradient over the CP group at step() (grads.allreduce_context_parallel_gradients)
            # and the pipeline engine back-propagates several micro-batches per step without a no_sync() bracket: in both
            # cases a bucket reduced during backward would miss contributions → fall back to the reduce-scatter at step()
            if ps.get_context_model_parallel_size() > 1 or ps.get_pipeline_model_parallel_size() > 1:
                from ..utils.logger import get_logger

                get_logger("zero1").warning("overlap_grad_reduce disabled: context/pipeline parallelism finalise gradients at step()")
                self._overlap_active = False
        if not self._overlap_active:
            return
        for fg in self.flat_groups:
            per = max(_ALIGN, (self.bucket_cap_rs // fg.grad_flat.element_size()) // _ALIGN * _ALIGN)
            for begin in range(0, fg.total, per):
                end = min(fg.total, begin + per)
                members = [s for s in fg.slots if s.offset < end and s.offset + s.numel > begin]
                if not members:
                    continue       # padding-only tail: nothing to reduce, stays zero
                bi = len(self._buckets)
                # a weight used more than once per backward (tied embeddings: `shared`) signals once per use through
                # the fused wgrad epilogue, so its buckets are never launched early (count + 1 is never reached)
                # ... and so are weights with more than one use per backward that are not PP-`shared`
                # (tie_word_embeddings without PP: the fused lm_head wgrad signals before the embedding gradient arrives).
                # Sequence-parallel-tagged parameters (norm / bias / router weights, TP all-reduce of their gradient at
                # step() in the reference, grads.py:330-346) get that all-reduce in the gradient hook instead, see
                # `_grad_ready`, so their buckets can still go early.
                tied = any(getattr(s.param, "shared", False) or getattr(s.param, "_nxd_multi_use", False) for s in members)
                self._buckets.append((fg, begin, end, len(members) + (1 if tied else 0)))
                for s in members:
                    self._slot_buckets.setdefault(id(s.param), []).append(bi)
        for fg in self.flat_groups:
            for s in fg.slots:
                s.param._nxd_grad_ready = self._grad_ready
        self._comm_stream = torch.cuda.Stream()
        self._sp_eager_tp = tp > 1
        self._reset_buckets()

    def _reset_buckets(self) -> None:
        self._bucket_remaining = [b[3] for b in self._buckets]
        self._bucket_launched = [False] * len(self._buckets)

    def set_grad_sync(self, enabled: bool) -> None:
        """``False`` while accumulating non-final micro-batches (DDP ``no_sync`` semantics)."""
        self._sync_enabled = bool(enabled)

    def no_sync(self):
        import contextlib

        @contextlib.contextmanager
        def ctx():
            old = self._sync_enabled
            self._sync_enabled = False
            try:
                yield
            finally:
                self._sync_enabled = old
        return ctx()

    def _grad_ready(self, param) -> None:
        if not (self._overlap_active and self._sync_enabled):
            return
        if getattr(self, "_sp_eager_tp", False) and getattr(param, "sequence_parallel_enabled", False) \
                and not getattr(param, "_nxd_sp_reduced", False):
            # this rank saw S/tp of the tokens: the gradient is final only after the TP sum.  Done here (a few KB, one-shot
            # all-reduce) so the bucket can be reduce-scattered under the backward; NxDOptimizer.step skips it later.
            comm.all_reduce(param.main_grad, group=ps.get_tensor_model_parallel_group())
            param._nxd_sp_reduced = True
        for bi in self._slot_buckets.get(id(param), ()):
            self._bucket_remaining[bi] -= 1
            if self._bucket_remaining[bi] == 0 and not self._bucket_launched[bi]:
                self._launch_bucket(bi)

    def _launch_bucket(self, bi: int) -> None:
        fg, begin, end, _ = self._buckets[bi]
        lo, hi = fg.shard_range
        a, b = max(begin, lo), min(end, hi)
        cur = torch.cuda.current_stream()
        self._comm_stream.wait_stream(cur)
        with torch.cuda.stream(self._comm_stream):
            fg.arena.reduce_scatter(fg.grad_off, fg.grad_flat.dtype, fg.shard_numel, 1.0 / self.grad_scale_divisor, fg.rs_out,
                                    fg.group_idx, sub_begin=max(a - lo, 0) if a < b else 0, sub_len=max(b - a, 0),
                                    max_ctas=self.overlap_ctas)
        self._bucket_launched[bi] = True

    def _install_hook(self, p: torch.nn.Parameter) -> None:
        def hook(param):
            if param.grad is None:
                return
            if getattr(param, "main_grad_fresh", False):   # first contribution since zero_grad: overwrite
                param.main_grad.copy_(param.grad)
                param.main_grad_fresh = False
            else:
                param.main_grad.add_(param.grad)
            param.grad = None
            cb = getattr(param, "_nxd_grad_ready", None)
            if cb is not None:
                cb(param)

        self._hooks.append(p.register_post_accumulate_grad_hook(hook))

    # ------------------------------------------------------------------ grads
    def zero_grad(self, set_to_none: bool = True) -> None:
        """No memset of the (multi-GB) flat gradient buffer: parameters are marked *fresh* and the first
        gradient contribution of the step overwrites instead of accumulating."""
        for fg in self.flat_groups:
            for s in fg.slots:
                s.param.grad = None
                s.param.main_grad_fresh = True
                if getattr(s.param, "_nxd_sp_reduced", False):
                    s.param._nxd_sp_reduced = False
        if getattr(self, "_overlap_active", False):
            self._reset_buckets()

    def _zero_untouched(self) -> None:
        for fg in self.flat_groups:
            for s in fg.slots:
                if getattr(s.param, "main_grad_fresh", False):   # received no gradient this step
                    s.param.main_grad.zero_()
                    s.param.main_grad_fresh = False

    def _reduce_scatter_grads(self) -> None:
        """grad_flat (summed over microbatches) → this rank's averaged shard."""
        for fg in self.flat_groups:
            lo, hi = fg.shard_range
            if self.world == 1:
                fg.grad_shard = fg.grad_flat[lo:hi]
                continue
            if fg.arena is not None and self._overlap_active:
                continue           # handled bucket-wise below
            if fg.arena is not None:
                fg.grad_shard = fg.arena.reduce_scatter(fg.grad_off, fg.grad_flat.dtype, fg.shard_numel,
                                                        1.0 / self.grad_scale_divisor, fg.rs_out, fg.group_idx)
                continue
            gf = fg.grad_flat
            if self.higher_cc_precision and gf.dtype != torch.float32:
                gf = gf.float()
            gf.div_(self.grad_scale_divisor)
            out = torch.empty(fg.shard_numel, dtype=gf.dtype, device=gf.device)
            if dist.get_backend(self.pg) == "gloo":
                dist.all_reduce(gf, group=self.pg)
                out.copy_(gf[lo:hi])
            else:
                # bucketed: contiguous column blocks of the [world, shard] view
                view = gf.view(self.world, fg.shard_numel)
                cols = max(_ALIGN, self.bucket_cap_rs // (gf.element_size() * self.world))
                for c0 in range(0, fg.shard_numel, cols):
                    c1 = min(fg.shard_numel, c0 + cols)
                    if c0 == 0 and c1 == fg.shard_numel:
                        dist.reduce_scatter_tensor(out, gf, group=self.pg)
                    else:
                        blk = view[:, c0:c1].contiguous()
                        dist.reduce_scatter_tensor(out[c0:c1], blk.view(-1), group=self.pg)
            fg.grad_shard = out
        if self._overlap_active:
            # buckets whose last gradient never signalled (unused parameters, sync disabled during backward): now, in
            # index order — identical on every rank, which the epoch handshake of the kernels relies on
            for bi in range(len(self._buckets)):
                if not self._bucket_launched[bi]:
                    self._launch_bucket(bi)
            torch.cuda.current_stream().wait_stream(self._comm_stream)
            for fg in self.flat_groups:
                fg.grad_shard = fg.rs_out
            self._reset_buckets()

    def _all_gather_params(self) -> None:
        if self.world == 1:
            return
        for fg in self.flat_groups:
            lo, hi = fg.shard_range
            if fg.arena is not None and fg.master_shard.dtype == torch.float32:
                fg.arena.all_gather(fg.master_shard, fg.param_off, fg.model_dtype, fg.shard_numel, fg.group_idx)
                continue
            if dist.get_backend(self.pg) == "gloo":
                parts = [torch.empty(fg.shard_numel, dtype=fg.model_dtype, device=fg.device) for _ in range(self.world)]
                dist.all_gather(parts, fg.param_flat[lo:hi].clone(), group=self.pg)
                fg.param_flat.copy_(torch.cat(parts))
            else:
                dist.all_gather_into_tensor(fg.param_flat, fg.param_flat[lo:hi].clone(), group=self.pg)

    def _shard_sq_norm(self) -> torch.Tensor:
        """Σ‖g‖² over my shards, TP-duplicates weighted 1/tp, tied (``shared``) params skipped."""
        tp = ps.get_tensor_model_parallel_size() if ps.model_parallel_is_initialized() else 1
        dev = self.flat_groups[0].device
        sharded, dup = [], []
        for fg in self.flat_groups:
            for slot, s0, _p0, n in fg.shard_slices():
                if getattr(slot.param, "shared", False):
                    continue
                piece = fg.grad_shard[s0 : s0 + n]
                (sharded if getattr(slot.param, "tensor_model_parallel", False) else dup).append(piece)
        total = ops.optim.multi_tensor_sq_norm(sharded).to(dev) if sharded else torch.zeros((), device=dev)
        if dup:
            total = total + ops.optim.multi_tensor_sq_norm(dup).to(dev) / tp
        return total.float()

    def _global_grad_norm(self) -> torch.Tensor:
        sq = self._shard_sq_norm()
        if self.world > 1:
            comm.all_reduce(sq, group=self.pg)
        if ps.model_parallel_is_initialized():
            if ps.get_tensor_model_parallel_size() > 1:
                comm.all_reduce(sq, group=ps.get_tensor_model_parallel_group())
            if ps.get_pipeline_model_parallel_size() > 1:
                comm.all_reduce(sq, group=ps.get_pipeline_model_parallel_group())
        return sq.sqrt()

    @property
    def grad_norm(self) -> Optional[torch.Tensor]:
        return self._grad_norm

    # ------------------------------------------------------------------- step
    @torch.no_grad()
    def step(self, closure: Optional[Callable] = None, **kwargs):
        loss = closure() if closure is not None else None
        self._zero_untouched()
        self._reduce_scatter_grads()
        coeff = None
        if self.grad_clipping:
            self._grad_norm = self._global_grad_norm()
            coeff = torch.clamp(self.max_norm / (self._grad_norm + 1e-6), max=1.0)
        for fg in self.flat_groups:
            fg.base_param.grad = fg.grad_shard if fg.grad_shard.dtype == fg.base_param.dtype else fg.grad_shard.to(fg.base_param.dtype)
        self._sync_hparams()
        fused_ok = hasattr(self.base_optimizer, "grad_scale")
        if fused_ok:
            self.base_optimizer.grad_scale = coeff
        elif coeff is not None:
            for fg in self.flat_groups:
                fg.base_param.grad.mul_(coeff)
        self.base_optimizer.step()
        writes_lowp = getattr(self.base_optimizer, "supports_lowp_view", False)
        for fg in self.flat_groups:
            if fg.use_master and not writes_lowp:
                lo, hi = fg.shard_range
                fg.param_flat[lo:hi].copy_(fg.master_shard)
            fg.base_param.grad = None
        self._all_gather_params()
        # keep user-visible hyper-parameters in sync (lr schedulers mutate self.param_groups)
        return loss

    def _sync_hparams(self) -> None:
        for g, bg in zip(self.param_groups, self.base_optimizer.param_groups):
            for k, v in g.items():
                if k != "params":
                    bg[k] = v

    # -------------------------------------------------------------- state dict
    def state_dict(self) -> Dict[str, Any]:
        base = self.base_optimizer.state_dict()
        shape_info = {}
        idx = 0
        for gi, fg in enumerate(self.flat_groups):
            for s in fg.slots:
                shape_info[idx] = {"shape": tuple(s.param.shape), "group": gi, "flat_offset": s.offset, "numel": s.numel}
                idx += 1
        out = {
            "state": base["state"],
            "base_state": base["state"],
            "param_groups": [{k: v for k, v in g.items() if k != "params"} | {"params": list(range(len(g["params"])))}
                             for g in self.param_groups],
            "shape_info": shape_info,
            "flat_layout": [{"shard_numel": fg.shard_numel, "total": fg.total, "world": self.world, "rank": self.rank}
                            for fg in self.flat_groups],
        }
        if self.save_master_weights or self.use_master_weights:
            out["sharded_master_weights"] = {gi: fg.master_shard.detach().clone() for gi, fg in enumerate(self.flat_groups)}
        return out

    def load_state_dict(self, state_dict: Dict[str, Any]) -> None:
        base_sd = self.base_optimizer.state_dict()
        base_sd["state"] = state_dict.get("base_state", state_dict["state"])
        self.base_optimizer.load_state_dict(base_sd)
        for g, sg in zip(self.param_groups, state_dict["param_groups"]):
            for k, v in sg.items():
                if k != "params":
                    g[k] = v
        self._sync_hparams()
        smw = state_dict.get("sharded_master_weights")
        if smw is not None:
            for gi, fg in enumerate(self.flat_groups):
                w = smw[gi] if gi in smw else smw[str(gi)]
                fg.master_shard.copy_(w.to(fg.master_shard.device))
                lo, hi = fg.shard_range
                fg.param_flat[lo:hi].copy_(fg.master_shard)
            self._all_gather_params()

    def add_param_group(self, param_group: Dict[str, Any]) -> None:
        super().add_param_group(param_group)

    # ---- per-rank shard files (reference :107-160; superseded by ``nxd.save_checkpoint`` there and here) ----------------
    @staticmethod
    def _shard_path(output_dir: str) -> str:
        return os.path.join(output_dir, "optim.dp_rank_{:02d}.tp_rank_{:02d}".format(ps.get_data_parallel_rank(),
                                                                                      ps.get_tensor_model_parallel_rank()))

    def save_sharded_state_dict(self, output_dir: str, num_workers_per_step: int = 8) -> None:
        """Write this rank's optimizer shard to ``<output_dir>/optim.dp_rank_XX.tp_rank_YY``.  At most
        ``num_workers_per_step`` local ranks write at the same time (bounds host memory / file-system pressure)."""
        from ..parallel_layers.utils import get_local_world_size, move_all_tensor_to_cpu

        os.makedirs(output_dir, exist_ok=True)
        sd = self.state_dict()
        sd["dp_rank"], sd["tp_rank"] = ps.get_data_parallel_rank(), ps.get_tensor_model_parallel_rank()
        local_rank = int(os.environ.get("LOCAL_RANK", dist.get_rank() if dist.is_initialized() else 0))
        waves = max(1, -(-get_local_world_size() // max(1, num_workers_per_step)))
        for wave in range(waves):
            if local_rank // max(1, num_workers_per_step) == wave:
                torch.save(move_all_tensor_to_cpu(sd), self._shard_path(output_dir))
            if dist.is_initialized() and waves > 1:
                dist.barrier()
        if dist.is_initialized():
            dist.barrier()

    def load_sharded_state_dict(self, output_dir: str, num_workers_per_step: int = 8) -> None:
        from ..parallel_layers.utils import get_local_world_size

        local_rank = int(os.environ.get("LOCAL_RANK", dist.get_rank() if dist.is_initialized() else 0))
        waves = max(1, -(-get_local_world_size() // max(1, num_workers_per_step)))
        for wave in range(waves):
            if local_rank // max(1, num_workers_per_step) == wave:
                sd = torch.load(self._shard_path(output_dir), map_location="cpu", weights_only=False)
                sd.pop("dp_rank", None), sd.pop("tp_rank", None)
                self.load_state_dict(sd)
            if dist.is_initialized() and waves > 1:
                dist.barrier()


class NeuronZero1Optimizer(Zero1Optimizer):
    """Reference-named entry point."""


class NeuronEPZero1Optimizer(torch.optim.Optimizer):
    """Expert-parallel aware ZeRO-1 (reference :163-287): non-expert params shard over the full DP
    group, expert params (``param.expert_model_parallel``) shard over the expert-DP group with
    their gradients pre-scaled by 1/ep."""

    def __init__(self, params: Iterable, optimizer_class, **kw):
        groups = list(params)
        if groups and not isinstance(groups[0], dict):
            groups = [{"params": groups}]
        ep_groups, nonep_groups = [], []
        for g in groups:
            rest = {k: v for k, v in g.items() if k != "params"}
            e = [p for p in g["params"] if getattr(p, "expert_model_parallel", False)]
            n = [p for p in g["params"] if not getattr(p, "expert_model_parallel", False)]
            if e:
                ep_groups.append({**rest, "params": e})
            if n:
                nonep_groups.append({**rest, "params": n})
        kw.pop("sharding_groups", None)
        self.non_ep = Zero1Optimizer(nonep_groups, optimizer_class, process_group=ps.get_data_parallel_group(), **kw) \
            if nonep_groups else None
        ep_kw = dict(kw)
        self.ep = Zero1Optimizer(ep_groups, optimizer_class, process_group=ps.get_expert_data_parallel_group(),
                                 grad_scale_divisor=ps.get_data_parallel_size(), **ep_kw) if ep_groups else None
        self._opts = [o for o in (self.non_ep, self.ep) if o is not None]
        super().__init__([g for o in self._opts for g in o.param_groups], {})
        self.grad_clipping = kw.get("grad_clipping", True)
        self.max_norm = kw.get("max_norm", 1.0) or 1.0
        self._grad_norm = None

    @property
    def grad_norm(self):
        return self._grad_norm

    def zero_grad(self, set_to_none: bool = True) -> None:
        for o in self._opts:
            o.zero_grad(set_to_none)

    @torch.no_grad()
    def step(self, closure=None, **kw):
        for o in self._opts:
            o._zero_untouched()
            o._reduce_scatter_grads()
        coeff = None
        if self.grad_clipping:
            dev = self._opts[0].flat_groups[0].device
            sq = torch.zeros((), device=dev)
            for o in self._opts:
                part = o._shard_sq_norm()
                if o.world > 1:
                    comm.all_reduce(part, group=o.pg)
                if o is self.ep and ps.get_expert_model_parallel_size() > 1:
                    comm.all_reduce(part, group=ps.get_expert_model_parallel_group())
                sq = sq + part
            if ps.get_tensor_model_parallel_size() > 1:
                comm.all_reduce(sq, group=ps.get_tensor_model_parallel_group())
            if ps.get_pipeline_model_parallel_size() > 1:
                comm.all_reduce(sq, group=ps.get_pipeline_model_parallel_group())
            self._grad_norm = sq.sqrt()
            coeff = torch.clamp(self.max_norm / (self._grad_norm + 1e-6), max=1.0)
        for o in self._opts:
            for fg in o.flat_groups:
                fg.base_param.grad = fg.grad_shard.to(fg.base_param.dtype)
            if hasattr(o.base_optimizer, "grad_scale"):
                o.base_optimizer.grad_scale = coeff
            elif coeff is not None:
                for fg in o.flat_groups:
                    fg.base_param.grad.mul_(coeff)
            o._sync_hparams()
            o.base_optimizer.step()
            for fg in o.flat_groups:
                if fg.use_master:
                    lo, hi = fg.shard_range
                    fg.param_flat[lo:hi].copy_(fg.master_shard)
                fg.base_param.grad = None
            o._all_gather_params()

    @property
    def sharding_groups(self):
        """``(dp groups for the dense parameters, expert-dp groups for the expert parameters)`` as rank lists."""
        return ps.get_data_parallel_replica_groups(), ps.get_expert_data_parallel_replica_groups()

    def save_sharded_state_dict(self, output_dir: str, num_workers_per_step: int = 8) -> None:
        os.makedirs(output_dir, exist_ok=True)
        path = os.path.join(output_dir, "optim.dp_rank_{:02d}.tp_rank_{:02d}".format(ps.get_data_parallel_rank(),
                                                                                      ps.get_tensor_model_parallel_rank()))
        from ..parallel_layers.utils import move_all_tensor_to_cpu

        torch.save(move_all_tensor_to_cpu(self.state_dict()), path)
        if dist.is_initialized():
            dist.barrier()

    def load_sharded_state_dict(self, output_dir: str, num_workers_per_step: int = 8) -> None:
        path = os.path.join(output_dir, "optim.dp_rank_{:02d}.tp_rank_{:02d}".format(ps.get_data_parallel_rank(),
                                                                                      ps.get_tensor_model_parallel_rank()))
        self.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))

    def state_dict(self):
        return {"non_ep": self.non_ep.state_dict() if self.non_ep else None,
                "ep": self.ep.state_dict() if self.ep else None}

    def load_state_dict(self, state_dict):
        sd = state_dict      # reference parameter names in the signature
        if self.non_ep and sd.get("non_ep") is not None:
            self.non_ep.load_state_dict(sd["non_ep"])
        if self.ep and sd.get("ep") is not None:
            self.ep.load_state_dict(sd["ep"])
