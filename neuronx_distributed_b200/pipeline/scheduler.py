"""Pipeline schedules as pure data.

Capability parity with reference ``pipeline/scheduler.py`` (task types :4-71, ``InferenceSchedule``
:144-154, ``Train1F1BSchedule`` :157-253, ``TrainInterleavedSchedule`` :256-541): a schedule is an
iterable of *steps*; each step is a list of tasks (recv / compute / send for one micro-batch and
model chunk); the last step is ``[ReduceGradsTask()]``.

Construction here is two-phase instead of the reference's step-id arithmetic:

1. :meth:`compute_order` — the per-stage sequence of (is_forward, microbatch, chunk) compute slots
   (warm-up forwards, 1F1B pairs, cool-down backwards);
2. :meth:`steps` — decorates every slot with the p2p tasks it needs.  Ordering rule that keeps
   blocking p2p deadlock-free (reference :226-233): in the steady state a stage first *receives the
   gradient* for the backward it is about to run, and only then *sends the activation* of the
   forward it just ran.

The engine executes sends asynchronously on an NCCL side stream, so the rule is conservative on
H100 but is kept so CPU/gloo (blocking p2p) runs the same schedules.
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from typing import Iterator, List, Tuple, Union


class PipelineTask:
    def __init__(self, mb: int, model_chunk: int = 0, graph_break: bool = True):
        self.mb, self.model_chunk, self.graph_break = mb, model_chunk, graph_break

    def __eq__(self, other) -> bool:
        return (type(self) is type(other) and self.mb == other.mb and self.model_chunk == other.model_chunk
                and self.graph_break == other.graph_break)

    def __hash__(self):
        return hash((type(self).__name__, self.mb, self.model_chunk, self.graph_break))

    def __repr__(self) -> str:
        return (f"{type(self).__name__}_microbatch_{self.mb}_modelchunk_{self.model_chunk}"
                f"_graphbreak_{self.graph_break}")


class ForwardPreprocessTask(PipelineTask):
    """receive the stage input of (mb, chunk) from the previous stage"""


class ForwardStepTask(PipelineTask):
    """run the stage module forward"""


class ForwardPostprocessTask(PipelineTask):
    """send the stage output to the next stage"""


class BackwardPreprocessTask(PipelineTask):
    """receive the output gradient from the next stage"""


class BackwardStepTask(PipelineTask):
    """run backward through the stage"""


class BackwardPostprocessTask(PipelineTask):
    """send the input gradient to the previous stage"""


class PostProcessTask:
    def __init__(self, graph_break: bool = True):
        self.mb, self.model_chunk, self.graph_break = -1, -1, graph_break


class ReduceGradsTask(PostProcessTask):
    def __repr__(self) -> str:
        return "ReduceGradsTask"

    def __eq__(self, other) -> bool:
        return type(self) is type(other)

    def __hash__(self):
        return hash("ReduceGradsTask")


Task = Union[PipelineTask, ReduceGradsTask]
Slot = Tuple[bool, int, int]  # (is_forward, microbatch, chunk)


class PipeSchedule(ABC):
    def __init__(self, num_microbatches: int, stages: int, stage_id: int):
        self.num_microbatches, self.stages, self.stage_id = num_microbatches, stages, stage_id
        self.prev_stage, self.next_stage = stage_id - 1, stage_id + 1

    @abstractmethod
    def steps(self) -> Iterator[List[Task]]:
        ...

    def _valid_micro_batch(self, mb: int) -> bool:
        return 0 <= mb < self.num_microbatches

    def _valid_stage(self, s: int) -> bool:
        return 0 <= s < self.stages

    @property
    def stage(self) -> int:
        return self.stage_id

    @property
    def num_stages(self) -> int:
        return self.stages

    @property
    def is_first_stage(self) -> bool:
        return self.stage_id == 0

    @property
    def is_last_stage(self) -> bool:
        return self.stage_id == self.stages - 1

    def __iter__(self):
        self._it = None
        return self

    def __next__(self):
        if self._it is None:
            self._it = self.steps()
        return next(self._it)


class InferenceSchedule(PipeSchedule):
    """Forward-only: all micro-batches through chunk 0, then chunk 1, … (one chunk without virtual pipeline)."""

    def __init__(self, num_microbatches: int, stages: int, stage_id: int, num_model_chunks: int = 1):
        super().__init__(num_microbatches, stages, stage_id)
        self.num_model_chunks = num_model_chunks

    def steps(self):
        for c in range(self.num_model_chunks):
            for mb in range(self.num_microbatches):
                yield [ForwardPreprocessTask(mb, c), ForwardStepTask(mb, c), ForwardPostprocessTask(mb, c)]


class Train1F1BSchedule(PipeSchedule):
    """Non-interleaved 1F1B: ``stages - stage_id - 1`` warm-up forwards, then forward/backward pairs,
    then the remaining backwards."""

    def __init__(self, num_microbatches: int, stages: int, stage_id: int):
        super().__init__(num_microbatches, stages, stage_id)
        self.get_microbatche_schedule()

    def get_microbatche_schedule(self) -> None:     # (sic) reference spelling, scheduler.py:179
        """Phase lengths of this stage: warm-up forwards, steady 1F1B pairs, cool-down backwards."""
        self.num_warmup_steps = min(self.stages - self.stage_id - 1, self.num_microbatches)
        self.num_steady_state_microbatches = self.num_microbatches - self.num_warmup_steps
        self.num_remaining_microbatches = self.num_warmup_steps

    def compute_order(self) -> List[Slot]:
        w, n = self.num_warmup_steps, self.num_microbatches
        order: List[Slot] = [(True, mb, 0) for mb in range(w)]
        for i in range(n - w):
            order += [(True, w + i, 0), (False, i, 0)]
        order += [(False, mb, 0) for mb in range(n - w, n)]
        return order

    def steps(self):
        has_next, has_prev = self._valid_stage(self.next_stage), self._valid_stage(self.prev_stage)
        w, steady = self.num_warmup_steps, self.num_steady_state_microbatches
        last_fwd = -1
        for is_fwd, mb, _ in self.compute_order():
            cmds: List[Task] = []
            if is_fwd:
                cmds += [ForwardPreprocessTask(mb), ForwardStepTask(mb)]
                if mb < w and has_next:          # warm-up: ship the activation right away
                    cmds.append(ForwardPostprocessTask(mb))
                last_fwd = mb
            else:
                if has_next:
                    cmds.append(BackwardPreprocessTask(mb))          # recv grad first …
                    if mb < steady:
                        cmds.append(ForwardPostprocessTask(last_fwd))  # … then send the pending activation
                cmds.append(BackwardStepTask(mb))
                if has_prev:
                    cmds.append(BackwardPostprocessTask(mb))
            yield cmds
        yield [ReduceGradsTask()]


class TrainInterleavedSchedule(PipeSchedule):
    """Interleaved (virtual-pipeline) 1F1B: each rank owns ``num_model_chunks`` model chunks; slots
    advance in groups of ``stages`` micro-batches per chunk (Megatron ordering).  ``recv`` tasks are
    always issued one slot ahead of their compute, ``send`` tasks right after it."""

    def __init__(self, num_microbatches: int, num_model_chunks: int, stages: int, stage_id: int,
                 fused_send_recv: bool = False, fused_fwd_bwd: bool = False, use_odd_even_scheduler: bool = False):
        super().__init__(num_microbatches, stages, stage_id)
        if num_microbatches % stages != 0:
            raise ValueError(
                "Interleaved pipeline requires num_microbatches % pipeline_parallel_size == 0, current "
                f"num_microbatches {num_microbatches} and pipeline_parallel_size {stages}")
        if num_microbatches <= stages:
            fused_send_recv = fused_fwd_bwd = False
        self.num_model_chunks = num_model_chunks
        self.fused_send_recv, self.fused_fwd_bwd = fused_send_recv, fused_fwd_bwd
        self.use_odd_even_scheduler = use_odd_even_scheduler
        self.get_step_schedule()

    def get_step_schedule(self) -> None:
        """Phase lengths in (micro-batch × chunk) steps: all-forward-then-all-backward when ``num_microbatches == stages``,
        otherwise ``2·(stages − stage − 1) + (chunks − 1)·stages`` warm-up forwards (reference scheduler.py:296-317)."""
        self.num_microbatches_steps = self.num_microbatches * self.num_model_chunks
        if self.num_microbatches == self.stages:
            self.num_warmup_steps = self.num_microbatches_steps
        else:
            self.num_warmup_steps = min((self.stages - self.stage_id - 1) * 2 + (self.num_model_chunks - 1) * self.stages,
                                        self.num_microbatches_steps)
        self.num_steady_state_steps = self.num_microbatches_steps - self.num_warmup_steps
        self.num_remaining_steps = self.num_warmup_steps

    # slot index (k-th forward / k-th backward on this rank) → (microbatch, chunk)
    def _slot(self, k: int, forward: bool) -> Tuple[int, int]:
        group = self.stages * self.num_model_chunks
        g, r = divmod(k, group)
        chunk = r // self.stages
        if not forward:
            chunk = self.num_model_chunks - 1 - chunk
        return g * self.stages + r % self.stages, chunk

    def get_model_chunk_id(self, step_id: int, is_forward: bool = True) -> int:
        return self._slot(step_id if is_forward else step_id - self.num_warmup_steps, is_forward)[1]

    def get_microbatch_id(self, step_id: int, is_forward: bool = True) -> int:
        return self._slot(step_id if is_forward else step_id - self.num_warmup_steps, is_forward)[0]

    def compute_order(self) -> List[Slot]:
        n, w = self.num_microbatches_steps, self.num_warmup_steps
        order: List[Slot] = [(True, *self._slot(k, True)) for k in range(w)]
        for i in range(n - w):
            order += [(True, *self._slot(w + i, True)), (False, *self._slot(i, False))]
        order += [(False, *self._slot(k, False)) for k in range(n - w, n)]
        return order

    # whether a forward slot must send to / a backward slot must receive from the next stage
    def _fwd_has_consumer(self, chunk: int) -> bool:
        return not (self.is_last_stage and chunk == self.num_model_chunks - 1)

    def _fwd_has_producer(self, chunk: int) -> bool:
        return not (self.is_first_stage and chunk == 0)

    def _comm(self, cmds: List[Task], k_fwd, k_bwd, recv_fwd, send_fwd, recv_bwd, send_bwd) -> None:
        """Append the p2p tasks around the compute of forward slot ``k_fwd`` / backward slot ``k_bwd``.
        recv tasks refer to the *next* slot, send tasks to the current one."""
        def f_pre(gb=True):
            mb, c = self._slot(k_fwd + 1, True)
            return ForwardPreprocessTask(mb, c, gb)

        def f_post(gb=True):
            mb, c = self._slot(k_fwd, True)
            return ForwardPostprocessTask(mb, c, gb)

        def b_pre():
            mb, c = self._slot(k_bwd + 1, False)
            return BackwardPreprocessTask(mb, c)

        def b_post():
            mb, c = self._slot(k_bwd, False)
            return BackwardPostprocessTask(mb, c)

        fsr = self.fused_send_recv
        if self.use_odd_even_scheduler:
            seq = ([("rf", recv_fwd), ("sf", send_fwd), ("sb", send_bwd), ("rb", recv_bwd)] if self.stage_id % 2 == 0
                   else [("sf", send_fwd), ("rf", recv_fwd), ("rb", recv_bwd), ("sb", send_bwd)])
            for kind, on in seq:
                if on:
                    cmds.append({"rf": f_pre, "sf": f_post, "sb": b_post, "rb": b_pre}[kind]())
            return
        if not self.is_last_stage:
            if recv_fwd:
                cmds.append(f_pre(not fsr or not send_bwd))
            if send_bwd:
                cmds.append(b_post())
            if send_fwd:
                cmds.append(f_post(not fsr or not recv_bwd))
            if recv_bwd:
                cmds.append(b_pre())
        else:  # last stage sends before it receives so the ring of blocking p2p calls cannot deadlock
            if send_fwd:
                cmds.append(f_post(not fsr or not recv_bwd))
            if recv_bwd:
                cmds.append(b_pre())
            if recv_fwd:
                cmds.append(f_pre(not fsr or not send_bwd))
            if send_bwd:
                cmds.append(b_post())

    def steps(self):
        n, w = self.num_microbatches_steps, self.num_warmup_steps
        total = w + self.num_steady_state_steps + self.num_remaining_steps
        for step in range(total):
            cmds: List[Task] = []
            if step < w:                                   # ---- warm-up: forward only
                if step == 0:
                    mb, c = self._slot(0, True)
                    cmds.append(ForwardPreprocessTask(mb, c))
                mb, c = self._slot(step, True)
                cmds.append(ForwardStepTask(mb, c))
                recv_fwd = step != n - 1
                send_fwd = self._fwd_has_consumer(c)
                recv_bwd = step == w - 1 and self._fwd_has_consumer(self._slot(0, False)[1])
                self._comm(cmds, step, -1, recv_fwd, send_fwd, recv_bwd, False)
            elif step < w + self.num_steady_state_steps:   # ---- steady: one forward + one backward
                kf, kb = step, step - w
                mbf, cf = self._slot(kf, True)
                mbb, cb = self._slot(kb, False)
                cmds.append(ForwardStepTask(mbf, cf, not self.fused_fwd_bwd))
                cmds.append(BackwardStepTask(mbb, cb))
                recv_fwd = step != w + self.num_steady_state_steps - 1
                send_fwd = self._fwd_has_consumer(cf)
                recv_bwd = self._fwd_has_consumer(self._slot(kb + 1, False)[1])
                send_bwd = self._fwd_has_producer(cb)
                self._comm(cmds, kf, kb, recv_fwd, send_fwd, recv_bwd, send_bwd)
            else:                                          # ---- cool-down: backward only
                kb = step - w
                mbb, cb = self._slot(kb, False)
                cmds.append(BackwardStepTask(mbb, cb))
                recv_bwd = step != total - 1 and self._fwd_has_consumer(self._slot(kb + 1, False)[1])
                send_bwd = self._fwd_has_producer(cb)
                self._comm(cmds, -1, kb, False, False, recv_bwd, send_bwd)
            yield cmds
        yield [ReduceGradsTask()]


class TrainSchedule(Train1F1BSchedule):
    """Deprecated name kept for source compatibility (reference :544-685 kept a lock-step variant; its
    compute order per stage equals :class:`Train1F1BSchedule`)."""
