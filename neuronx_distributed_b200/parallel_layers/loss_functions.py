"""Vocab-parallel cross entropy and log-prob extraction.

Capability parity with reference ``parallel_layers/loss_functions.py`` (``parallel_cross_entropy``
:217, ``_ParallelCrossEntropy`` :10-129, ``DistributedLogprob`` / ``from_parallel_logits_to_logprobs``
:131-215).

H100 design: one pass over the local ``[T, V/tp]`` logits produces three per-row statistics
(local max, local sum-exp relative to that max, target logit if owned); the three reference
all-reduces (MAX, SUM, SUM) collapse into ONE all-gather of a ``[T, 3]`` fp32 tensor followed by
a log-sum-exp merge, and the softmax is *recomputed* in backward from the saved logits and the
row log-normaliser instead of being stored in fp32 (saves T·V/tp·4 bytes).  On CUDA the two
passes are the hand-written kernels ``ops.cross_entropy.ce_stats / ce_backward``.

Deviation (documented): label smoothing averages log-probs over the *global* vocabulary; the
reference averages over the local partition only (its ``vocab_size`` is the shard size), which
coincides with this for tp=1.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from . import comm
from . import parallel_state as ps
from .utils import EmbeddingUtility


def _row_stats(logits2d: torch.Tensor, target1d: torch.Tensor, vocab_start: int):
    """(local max, local sumexp wrt local max, owned target logit or 0, owned mask, sum of logits) per row, fp32."""
    from .. import ops

    return ops.cross_entropy.ce_stats(logits2d, target1d, vocab_start)


class _ParallelCrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vocab_parallel_logits, target, label_smoothing=0.0, group=None):
        from .. import ops

        group = group if group is not None else ps.get_tensor_model_parallel_group()
        n, r = dist.get_world_size(group), dist.get_rank(group)
        vp = vocab_parallel_logits.shape[-1]
        start, _ = EmbeddingUtility.range_from_per_partition_vocab_size(vp, r, n)
        logits2d = vocab_parallel_logits.reshape(-1, vp)
        tgt = target.reshape(-1)
        # stats: [T, 4] = (max, sumexp, target_logit, sum_logits)
        stats = ops.cross_entropy.ce_stats(logits2d, tgt, start)
        if n > 1:
            allstats = comm.all_gather(stats.unsqueeze(0), dim=0, group=group)  # [n, T, 4]
            gmax = allstats[..., 0].max(dim=0).values
            sumexp = (allstats[..., 1] * torch.exp(allstats[..., 0] - gmax)).sum(0)
            pred = allstats[..., 2].sum(0)
            sum_logits = allstats[..., 3].sum(0)
        else:
            gmax, sumexp, pred, sum_logits = stats[:, 0], stats[:, 1], stats[:, 2], stats[:, 3]
        lse = gmax + torch.log(sumexp)  # log normaliser per row
        loss = lse - pred
        vocab = vp * n
        if label_smoothing > 0:
            assert 1.0 > label_smoothing > 0.0
            smoothing = label_smoothing * vocab / (vocab - 1)
            mean_log_probs = sum_logits / vocab - lse
            loss = (1.0 - smoothing) * loss - smoothing * mean_log_probs
        ctx.label_smoothing, ctx.vocab, ctx.start = label_smoothing, vocab, start
        ctx.save_for_backward(logits2d, tgt, lse)
        ctx.shape = vocab_parallel_logits.shape
        return loss.view(target.shape)

    @staticmethod
    def backward(ctx, grad_output):
        from .. import ops

        logits2d, tgt, lse = ctx.saved_tensors
        if ctx.label_smoothing > 0:
            smoothing = ctx.label_smoothing * ctx.vocab / (ctx.vocab - 1)
        else:
            smoothing = 0.0
        g = ops.cross_entropy.ce_backward(
            logits2d, tgt, lse, grad_output.reshape(-1).float(), ctx.start, smoothing, ctx.vocab
        )
        return g.view(ctx.shape), None, None, None


def parallel_cross_entropy(vocab_parallel_logits, target, label_smoothing: float = 0.0, process_group=None):
    """Per-token cross-entropy for logits sharded along the vocab (last) dim across TP."""
    return _ParallelCrossEntropy.apply(vocab_parallel_logits, target, label_smoothing, process_group)


class DistributedLogprob(torch.autograd.Function):
    """log p(target) from vocab-parallel logits (DPO/ORPO-style objectives; reference :131-204)."""

    @staticmethod
    def forward(ctx, vocab_parallel_logits, target, inference_only=False, group=None):
        from .. import ops

        group = group if group is not None else ps.get_tensor_model_parallel_group()
        n, r = dist.get_world_size(group), dist.get_rank(group)
        vp = vocab_parallel_logits.shape[-1]
        start, _ = EmbeddingUtility.range_from_per_partition_vocab_size(vp, r, n)
        logits2d = vocab_parallel_logits.reshape(-1, vp)
        tgt = target.reshape(-1)
        stats = ops.cross_entropy.ce_stats(logits2d, tgt, start)
        if n > 1:
            allstats = comm.all_gather(stats.unsqueeze(0), dim=0, group=group)
            gmax = allstats[..., 0].max(dim=0).values
            sumexp = (allstats[..., 1] * torch.exp(allstats[..., 0] - gmax)).sum(0)
            pred = allstats[..., 2].sum(0)
        else:
            gmax, sumexp, pred = stats[:, 0], stats[:, 1], stats[:, 2]
        lse = gmax + torch.log(sumexp)
        ctx.inference_only = bool(inference_only)
        if not inference_only:
            ctx.save_for_backward(logits2d, tgt, lse)
            ctx.start, ctx.shape, ctx.vocab = start, vocab_parallel_logits.shape, vp * n
        return (pred - lse).view(target.shape)

    @staticmethod
    def backward(ctx, grad_output):
        from .. import ops

        if ctx.inference_only:
            raise RuntimeError("log-probs computed with inference=True keep no state for backward; pass inference=False")
        logits2d, tgt, lse = ctx.saved_tensors
        # d(logp)/dlogits = onehot - softmax = -(softmax - onehot)
        g = ops.cross_entropy.ce_backward(
            logits2d, tgt, lse, (-grad_output).reshape(-1).float(), ctx.start, 0.0, ctx.vocab
        )
        return g.view(ctx.shape), None, None, None


def from_parallel_logits_to_logprobs(vocab_parallel_logits, target, inference: bool = True, process_group=None,
                                     inference_only: Optional[bool] = None):
    """Log-probabilities of ``target[:, 1:]`` under ``logits[:, :-1]`` (next-token shift as in the reference :206-215;
    pass the UNSHIFTED targets).  ``inference=True`` (the reference's default) keeps nothing for a backward pass; pass
    ``inference=False`` when the log-probs feed a training objective (DPO / ORPO).  ``inference_only`` is this package's
    earlier name of the same flag."""
    if inference_only is not None:
        inference = inference_only
    target = target.roll(shifts=-1, dims=-1)
    probs = DistributedLogprob.apply(vocab_parallel_logits, target, inference, process_group)
    return probs[:, :-1].contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# lm_head + cross entropy without materialising the logits (SURVEY §7.4 ``lmhead_ce_fused``)
# ---------------------------------------------------------------------------------------------------------------------
class _FusedLinearCrossEntropy(torch.autograd.Function):
    """``mean_over_unmasked( CE( gather(h) @ Wᵀ , target) )`` in row chunks: per chunk the vocab-parallel logits
    ``[chunk, V/tp]`` are produced by the tensor-core GEMM, reduced to row statistics (``ce_stats`` + ONE all-gather of
    ``[chunk, 4]`` floats across TP), turned into their gradient in place (``ce_backward``) and consumed at once by the
    dgrad GEMM (``dX_chunk = g @ W``) and the wgrad GEMM (``dW += gᵀ @ x_chunk``, fp32 accumulation).  The full
    ``[S·B, V/tp]`` logits (bf16: 1 GB for Llama-2-7B at 16k tokens, plus the same again for their gradient) never exist;
    the chunk buffer stays L2-sized.  The reference materialises the logits (``ColumnParallelLinear`` →
    ``parallel_cross_entropy``, loss_functions.py:12-100).

    The loss is a scalar, so the backward only scales the gradients computed during the forward by the incoming scalar
    gradient (the Liger-kernel arrangement): no recomputation of the lm_head GEMM."""

    @staticmethod
    def forward(ctx, h, weight, target, label_smoothing, group, sequence_parallel, chunk_rows, ignore_index):
        from .. import ops

        group = group if group is not None else ps.get_tensor_model_parallel_group()
        n, r = dist.get_world_size(group), dist.get_rank(group)
        vp, H = weight.shape
        start, _ = EmbeddingUtility.range_from_per_partition_vocab_size(vp, r, n)
        x = h.reshape(-1, H) if not (sequence_parallel and n > 1) else \
            comm.all_gather(h.contiguous(), dim=0, group=group).reshape(-1, H)
        x = x.contiguous()
        tgt = target.reshape(-1)
        T = x.shape[0]
        assert tgt.numel() == T, f"target has {tgt.numel()} entries for {T} rows of hidden states"
        mask = tgt != ignore_index
        safe = torch.where(mask, tgt, torch.zeros_like(tgt))
        row_scale = mask.float() / mask.sum().clamp(min=1).float()       # d(mean loss)/d(per-row loss)
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dx = torch.empty_like(x) if need_x else None
        dw = torch.empty(vp, H, dtype=torch.float32, device=x.device) if need_w else None
        vocab = vp * n
        smoothing = label_smoothing * vocab / (vocab - 1) if label_smoothing > 0 else 0.0
        loss = torch.zeros((), dtype=torch.float32, device=x.device)
        step = max(1, int(chunk_rows))
        for i, lo in enumerate(range(0, T, step)):
            hi = min(T, lo + step)
            xc, tc, sc = x[lo:hi], safe[lo:hi], row_scale[lo:hi]
            logits = ops.gemm.matmul(xc, weight, False, True)                                     # [c, V/tp]
            stats = ops.cross_entropy.ce_stats(logits, tc, start)
            if n > 1:
                alls = comm.all_gather(stats.unsqueeze(0), dim=0, group=group)                    # [n, c, 4]
                gmax = alls[..., 0].max(dim=0).values
                sumexp = (alls[..., 1] * torch.exp(alls[..., 0] - gmax)).sum(0)
                pred, sum_logits = alls[..., 2].sum(0), alls[..., 3].sum(0)
            else:
                gmax, sumexp, pred, sum_logits = stats[:, 0], stats[:, 1], stats[:, 2], stats[:, 3]
            lse = gmax + torch.log(sumexp)
            per_row = lse - pred
            if smoothing > 0:
                per_row = (1.0 - smoothing) * per_row - smoothing * (sum_logits / vocab - lse)
            loss += (per_row * sc).sum()
            if need_x or need_w:
                g = ops.cross_entropy.ce_backward(logits, tc, lse, sc, start, smoothing, vocab)   # [c, V/tp], logits dtype
                del logits
                if need_x:
                    ops.gemm.matmul(g, weight, False, False, out=dx[lo:hi])                       # partial over vocab shards
                if need_w:
                    ops.gemm.matmul(g, xc, True, False, out=dw, accumulate=i > 0)
        ctx.group, ctx.n, ctx.sp, ctx.h_shape = group, n, bool(sequence_parallel), h.shape
        ctx.weight = weight
        ctx.save_for_backward(*(t for t in (dx, dw) if t is not None))
        ctx.have = (dx is not None, dw is not None)
        return loss

    @staticmethod
    def backward(ctx, gloss):
        saved = list(ctx.saved_tensors)
        dx = saved.pop(0) if ctx.have[0] else None
        dw = saved.pop(0) if ctx.have[1] else None
        gh = gw = None
        if dx is not None:
            dx = dx * gloss.to(dx.dtype)
            if ctx.n > 1:
                dx = comm.reduce_scatter(dx, dim=0, group=ctx.group) if ctx.sp else comm.all_reduce(dx, group=ctx.group)
            gh = dx.view(ctx.h_shape)
        if dw is not None:
            weight = ctx.weight
            mg = getattr(weight, "main_grad", None)
            if mg is not None and mg.dtype == torch.float32 and mg.shape == dw.shape:
                # ZeRO-1 fp32 gradient accumulation: add straight into the flat buffer (same contract as layers.wgrad)
                if getattr(weight, "main_grad_fresh", False):
                    torch.mul(dw, gloss.float(), out=mg)
                else:
                    mg.addcmul_(dw, gloss.float().expand_as(dw))
                weight.main_grad_fresh = False
                cb = getattr(weight, "_nxd_grad_ready", None)
                if cb is not None:
                    cb(weight)
            else:
                gw = (dw * gloss.float()).to(weight.dtype)
        return gh, gw, None, None, None, None, None, None


def fused_linear_cross_entropy(hidden: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, label_smoothing: float = 0.0,
                               process_group=None, sequence_parallel: bool = False, chunk_rows: int = 2048,
                               ignore_index: int = -100) -> torch.Tensor:
    """Mean cross entropy of ``lm_head(hidden)`` against ``target`` over the entries ``!= ignore_index`` — a scalar — with
    the vocab-parallel ``weight [V/tp, H]``, never holding more than ``chunk_rows`` rows of logits.  ``hidden`` is
    ``[S, B, H]`` (``[S/tp, B, H]`` with ``sequence_parallel``: gathered along dim 0 inside, its gradient reduce-scattered);
    ``target`` has the shape of the gathered leading dims."""
    return _FusedLinearCrossEntropy.apply(hidden, weight, target, float(label_smoothing), process_group, bool(sequence_parallel),
                                          int(chunk_rows), int(ignore_index))
