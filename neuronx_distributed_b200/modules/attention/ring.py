"""Context-parallel ring attention.

Role of the reference's NKI ring kernels (``kernels/ring_attention_kernel.py:44-167``, K3/K4): each CP rank holds a
contiguous ``S/cp`` slice of Q, K, V; K/V blocks travel around the CP ring and every rank merges the partial
attention of each visiting block into its output with a log-sum-exp update.  With contiguous slices and a causal
mask, a block that originated on a *later* rank is skipped, the local block is causal, earlier blocks are dense
(same — load-imbalanced — split as the reference: no zig-zag).

H100 design: the ring transfer is an NCCL p2p exchange issued *before* the block's attention so it overlaps the
compute; the exchange is itself an autograd node (its backward moves dK/dV the opposite way round the ring), so
backward is the exact transpose of forward without a hand-written second pass.  Per-block attention is the own
flash kernel with a differentiable LSE output (``ops.attention.flash_attention_with_lse``; head_dim 64/80/96/128, bf16), the SDPA
flash op for other shapes on CUDA, and an fp32 reference on CPU.

Sliding window W (Mistral / Mixtral): a block whose queries sit ``off`` positions after its keys is computed by the windowed
kernels with that query offset, and is empty once off ≥ W + c − 1 (c = chunk length).  So with the contiguous split a rank
needs K/V only from the previous ceil((W − 1)/c) ranks, and the ring stops after that many hops.  ``_visible_pairs`` is the one
block plan both the ring and the pull implementation iterate.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.distributed as dist

from ...parallel_layers import parallel_state as ps


def _block_visibility(sq: int, sk: int, window: Optional[int], q_offset: int, device) -> torch.Tensor:
    """``[sq, sk]`` visibility of a causal block.  CP blocks have equal lengths; a shorter query block aligns its last row with
    the last key, as SDPA's flash op does."""
    from ... import ops

    return ops.attention.window_visibility(sq, sk, window, device, q_offset + sk - sq)


def block_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool, scale: float,
                    window: Optional[int] = None, q_offset: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """q [B,Sq,H,D], k/v [B,Sk,Hkv,D] → (out [B,Sq,H,D], lse [B,H,Sq] fp32).

    A causal block sees keys j ≤ i + q_offset, and with a sliding ``window`` W only j > i + q_offset − W (``q_offset``: global
    position of query row 0 minus that of key row 0).  A dense block (``causal=False``) sees every key, so ``window`` and
    ``q_offset`` apply to causal blocks only.  A row that sees no key gets O = 0 and LSE = −inf."""
    if not causal:
        window, q_offset = None, 0
    if q.is_cuda:
        from ... import ops

        own = ops.attention.flash_attention_with_lse(q, k, v, causal, scale, window, q_offset)   # own kernels, LSE differentiable
        if own is not None:
            return own
    hq, hkv = q.shape[2], k.shape[2]
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    if hq != hkv:
        kt, vt = kt.repeat_interleave(hq // hkv, 1), vt.repeat_interleave(hq // hkv, 1)
    # the SDPA flash op takes no mask, so a windowed block it would get goes to the masked fp32 path below
    if q.is_cuda and q.dtype in (torch.bfloat16, torch.float16) and window is None and q_offset == 0:
        out, lse = torch.ops.aten._scaled_dot_product_flash_attention(qt, kt, vt, 0.0, causal, False, scale=scale)[:2]
        return out.transpose(1, 2), lse.float()
    s = torch.matmul(qt.float(), kt.float().transpose(-1, -2)) * scale
    if causal:
        vis = _block_visibility(s.shape[-2], s.shape[-1], window, q_offset, s.device)
        s = s.masked_fill(~vis, float("-inf"))
        # a row with no visible key (possible with an offset window): logsumexp over zeros keeps its gradient finite, its
        # P is exp(−inf) = 0, and its LSE is set to −inf afterwards
        empty = ~vis.any(-1)
        lse = torch.logsumexp(s.masked_fill(empty[:, None], 0.0), dim=-1)
        p = torch.exp(s - lse.unsqueeze(-1))
        lse = lse.masked_fill(empty, float("-inf"))
    else:
        lse = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - lse.unsqueeze(-1))
    out = torch.matmul(p, vt.float()).to(q.dtype)
    return out.transpose(1, 2), lse


def _merge_block(out: Optional[torch.Tensor], lse: Optional[torch.Tensor], o_b: torch.Tensor, lse_b: torch.Tensor):
    """Fold one block's ``(o_b [B,S,H,D], lse_b [B,H,S])`` into the running ``(out fp32, lse)`` by log-sum-exp weights;
    ``out is None`` starts the merge.  A row for which both LSEs are −inf (no key seen yet, e.g. an offset window) keeps O = 0
    and LSE = −inf, with no NaN in the forward or the backward, whatever the block order."""
    if out is None:
        return o_b.float(), lse_b.float()
    empty = torch.isneginf(lse) & torch.isneginf(lse_b)
    lse, lse_b = lse.masked_fill(empty, 0.0), lse_b.masked_fill(empty, 0.0)      # both O are 0 there: any finite weights do
    new = torch.logaddexp(lse, lse_b)
    w_old = torch.exp(lse - new).transpose(1, 2).unsqueeze(-1)     # [B,S,H,1]
    w_new = torch.exp(lse_b - new).transpose(1, 2).unsqueeze(-1)
    return out * w_old + o_b.float() * w_new, new.masked_fill(empty, float("-inf"))


def _window_arg(sliding_window: Optional[int], causal: bool) -> Optional[int]:
    from ... import ops

    if sliding_window is not None and not causal:
        raise ValueError("sliding_window needs causal=True")
    return ops.attention.check_window(sliding_window) or None


class _RingShift(torch.autograd.Function):
    """send ``x`` to the next rank of the ring, receive the previous rank's; backward shifts the other way."""

    @staticmethod
    def forward(ctx, x, group, nxt, prv):
        ctx.group, ctx.nxt, ctx.prv = group, nxt, prv
        return _exchange(x, group, nxt, prv)

    @staticmethod
    def backward(ctx, g):
        return _exchange(g.contiguous(), ctx.group, ctx.prv, ctx.nxt), None, None, None


def _exchange(x: torch.Tensor, group, send_to: int, recv_from: int) -> torch.Tensor:
    buf = torch.empty_like(x)
    ops = [dist.P2POp(dist.isend, x.contiguous(), send_to, group), dist.P2POp(dist.irecv, buf, recv_from, group)]
    for w in dist.batch_isend_irecv(ops):
        w.wait()
    return buf


def ring_hops(cp: int, chunk: int, window: Optional[int]) -> int:
    """Ring shifts per pass: cp − 1, or with a sliding window only as far back as a block can still be visible,
    min(cp − 1, ceil((W − 1) / chunk)).  It depends on shapes only, so every rank derives the same count."""
    return cp - 1 if window is None else min(cp - 1, -(-(window - 1) // chunk))


def ring_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True,
                   scale: Optional[float] = None, group=None, sliding_window: Optional[int] = None) -> torch.Tensor:
    """q/k/v: this rank's ``[B, S/cp, H, D]`` slices (contiguous split) → attention output for the local queries.

    ``sliding_window`` W (causal only): query i sees keys i − W < j ≤ i in global positions; the ring then stops after
    :func:`ring_hops` shifts, so a rank receives K/V only from the ranks its window reaches."""
    group = group if group is not None else ps.get_context_model_parallel_group()
    cp = dist.get_world_size(group)
    scale = scale if scale is not None else 1.0 / math.sqrt(q.shape[-1])
    window = _window_arg(sliding_window, causal)
    if cp == 1:
        return block_attention(q, k, v, causal, scale, window)[0]
    r = dist.get_rank(group)
    ranks = dist.get_process_group_ranks(group)
    nxt, prv = ranks[(r + 1) % cp], ranks[(r - 1) % cp]
    hops = ring_hops(cp, q.shape[1], window)
    plan = _visible_pairs(r, cp, "contiguous", causal, window, q.shape[1])
    blocks = {src: (blk_causal, off) for _, src, _, blk_causal, off in plan}           # one block per source rank
    out: Optional[torch.Tensor] = None
    lse: Optional[torch.Tensor] = None
    kv = torch.stack([k, v])  # travel together: one message per hop
    for step in range(hops + 1):
        src = (r - step) % cp                       # origin rank of the block currently held
        nxt_kv = _RingShift.apply(kv, group, nxt, prv) if step < hops else None   # start next hop early
        if src in blocks:
            o_b, lse_b = block_attention(q, kv[0], kv[1], blocks[src][0], scale, window, blocks[src][1])
            out, lse = _merge_block(out, lse, o_b, lse_b)
        if nxt_kv is None:
            last_kv = kv
        kv = nxt_kv
    # tie the last visiting block into the graph with zero weight: a rank that skipped it (causal) must still run
    # every ring-shift backward, otherwise its neighbours would wait forever for the matching exchange
    out = out + 0.0 * last_kv.float().sum()
    return out.to(q.dtype)


# ---------------------------------------------------------------------------------------------------------------------
# Context-parallel attention WITHOUT a ring: every rank publishes its K/V slice in NVSwitch-visible symmetric memory and
# the attention kernels read the other ranks' slices where they are (cp.async tile loads over NVLink inside the kernel) — the
# K/V "rotation" of the reference's ring kernels (K3/K4, kernels/ring_attention_kernel.py:118-167) happens inside the
# attention kernel, and there are no ring steps to serialise on.  Backward re-publishes K/V, computes every block's
# (dQ, dK, dV) from the GLOBAL softmax statistics (so no per-block LSE gradients are needed) and returns the dK/dV
# contributions to their owners with ONE reduce-scatter (in-switch sum on NVLS).
# ---------------------------------------------------------------------------------------------------------------------
def _block_backward(q, k, v, out, lse, dout, causal: bool, scale: float, window: Optional[int] = None, q_offset: int = 0):
    """Gradients of one K/V block given the GLOBAL output ``out`` / log-normaliser ``lse`` of the rows:
    P = exp(S − lse), dV = Pᵀ dO, dS = P ∘ (dO Vᵀ − rowsum(dO ∘ out)), dQ = dS K · scale, dK = dSᵀ Q · scale.
    ``window`` / ``q_offset``: the visibility of a causal block, as in :func:`block_attention`."""
    if not causal:
        window, q_offset = None, 0
    if q.is_cuda:
        from ... import ops

        if ops.attention.flash_kernels_apply(q, k, v, causal):
            return ops.attention._flash_backward(dout, q, k, v, out, lse, causal, scale, None, window or 0, q_offset)
    hq, hkv = q.shape[2], k.shape[2]
    g = hq // hkv
    qt, dot, ot = q.transpose(1, 2).float(), dout.transpose(1, 2).float(), out.transpose(1, 2).float()     # [B,H,S,D]
    kt, vt = k.transpose(1, 2).float().repeat_interleave(g, 1), v.transpose(1, 2).float().repeat_interleave(g, 1)
    s = torch.matmul(qt, kt.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(~_block_visibility(s.shape[-2], s.shape[-1], window, q_offset, s.device), float("-inf"))
    p = torch.exp(s - lse.unsqueeze(-1))
    dv = torch.matmul(p.transpose(-1, -2), dot)
    ds = p * (torch.matmul(dot, vt.transpose(-1, -2)) - (dot * ot).sum(-1, keepdim=True))
    dq = torch.matmul(ds, kt) * scale
    dk = torch.matmul(ds.transpose(-1, -2), qt) * scale
    B, _, Sk, D = dk.shape
    dk, dv = dk.view(B, hkv, g, Sk, D).sum(2), dv.view(B, hkv, g, Sk, D).sum(2)
    return dq.transpose(1, 2).to(q.dtype), dk.transpose(1, 2).to(k.dtype), dv.transpose(1, 2).to(v.dtype)


def _chunk_ids(rank: int, cp: int, layout: str):
    """Global sequence-chunk ids held by ``rank``, in local order.  ``contiguous``: one chunk per rank.  ``zigzag``: the sequence
    is cut into 2·cp chunks and rank r holds chunks r and 2·cp−1−r — with a causal mask every rank then owns the same number of
    visible (query chunk, key chunk) pairs (2·cp + 1), instead of r + 1 for the contiguous split."""
    if layout == "contiguous":
        return [rank]
    if layout == "zigzag":
        return [rank, 2 * cp - 1 - rank]
    raise ValueError(f"unknown context-parallel layout {layout!r}")


def _visible_pairs(rank: int, cp: int, layout: str, causal: bool, window: Optional[int] = None, chunk: int = 1):
    """The block plan of one rank: ``(local query chunk, source rank, source chunk, causal, q_offset)`` for every non-empty
    block it computes, own rank first, then the ranks before it round the ring.

    ``chunk``: positions per sequence chunk; ``q_offset`` is the global position of the block's query row 0 minus that of its
    key row 0, (gq − gk)·chunk.  ``causal`` says whether the block needs the causal rule (with ``window`` W, the windowed rule
    at that offset); a block with ``causal=False`` sees every key.  Without a window only the diagonal is causal.  With one,
    a block is empty, and left out, iff q_offset ≥ W + chunk − 1, and fully visible iff q_offset > 0 and
    W ≥ q_offset + chunk."""
    mine = _chunk_ids(rank, cp, layout)
    pairs = []
    for step in range(cp):
        src = (rank - step) % cp
        theirs = _chunk_ids(src, cp, layout)
        for qi, gq in enumerate(mine):
            for kj, gk in enumerate(theirs):
                off = (gq - gk) * chunk
                if not causal:
                    pairs.append((qi, src, kj, False, off))
                elif gk <= gq:
                    if window is None:
                        pairs.append((qi, src, kj, gk == gq, off))
                    elif off < window + chunk - 1:
                        pairs.append((qi, src, kj, gk == gq or window < off + chunk, off))
    return pairs


class _PullAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, causal, scale, group, layout, window):
        from ... import ops

        cp, r = dist.get_world_size(group), dist.get_rank(group)
        nq = len(_chunk_ids(r, cp, layout))
        assert q.shape[1] % nq == 0 and k.shape[1] % nq == 0, "the local sequence must split into the layout's chunks"
        kv = torch.stack([k, v]).contiguous()                        # one slot per rank: [2, B, S/cp, Hkv, D]
        views = ops.nvls.publish(kv, group)
        qs = q.chunk(nq, dim=1)
        outs = [None] * nq
        lses = [None] * nq
        with torch.no_grad():
            for qi, src, kj, blk_causal, off in _visible_pairs(r, cp, layout, causal, window, q.shape[1] // nq):
                kb, vb = views[src][0].chunk(nq, dim=1)[kj], views[src][1].chunk(nq, dim=1)[kj]
                o_b, lse_b = block_attention(qs[qi], kb, vb, blk_causal, scale, window, off)
                outs[qi], lses[qi] = _merge_block(outs[qi], lses[qi], o_b, lse_b)
        out = torch.cat(outs, dim=1).to(q.dtype)
        lse = torch.cat(lses, dim=2)                                 # [B, H, S/cp]
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.causal, ctx.scale, ctx.group, ctx.layout, ctx.window = causal, scale, group, layout, window
        return out

    @staticmethod
    def backward(ctx, dout):
        from ... import ops
        from ...parallel_layers import comm

        q, k, v, out, lse = ctx.saved_tensors
        group, causal, scale, layout, window = ctx.group, ctx.causal, ctx.scale, ctx.layout, ctx.window
        cp, r = dist.get_world_size(group), dist.get_rank(group)
        nq = len(_chunk_ids(r, cp, layout))
        views = ops.nvls.publish(torch.stack([k, v]).contiguous(), group)          # peers' K/V again (the slot was reused since)
        dqs = [torch.zeros_like(c, dtype=torch.float32) for c in q.chunk(nq, dim=1)]
        dkv = torch.zeros((cp,) + tuple(views[r].shape), dtype=torch.float32, device=q.device)      # [cp, 2, B, S/cp, Hkv, D]
        qs, os_, ds = q.chunk(nq, dim=1), out.chunk(nq, dim=1), dout.contiguous().chunk(nq, dim=1)
        ls = lse.chunk(nq, dim=2)
        c = k.shape[1] // nq
        for qi, src, kj, blk_causal, off in _visible_pairs(r, cp, layout, causal, window, c):
            kb, vb = views[src][0].chunk(nq, dim=1)[kj], views[src][1].chunk(nq, dim=1)[kj]
            dq_b, dk_b, dv_b = _block_backward(qs[qi].contiguous(), kb.contiguous(), vb.contiguous(), os_[qi].contiguous(),
                                               ls[qi].contiguous(), ds[qi].contiguous(), blk_causal, scale, window, off)
            dqs[qi] += dq_b.float()
            dkv[src, 0, :, kj * c:(kj + 1) * c] += dk_b.float()
            dkv[src, 1, :, kj * c:(kj + 1) * c] += dv_b.float()
        # every rank holds its contributions to ALL blocks; each owner needs the sum over ranks of its own block
        flat = dkv.reshape(cp * dkv[0].numel() // dkv.shape[-1], dkv.shape[-1])
        if flat.is_cuda and ops.nvls.available(group) and ops.nvls.has_multicast(group):
            mine = ops.nvls.reduce_scatter_sum(flat, group)
        else:
            mine = comm.reduce_scatter(flat, dim=0, group=group)
        mine = mine.view(dkv.shape[1:])
        return torch.cat(dqs, dim=1).to(q.dtype), mine[0].to(k.dtype), mine[1].to(v.dtype), None, None, None, None, None


def pull_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True, scale: Optional[float] = None,
                   group=None, layout: str = "contiguous", sliding_window: Optional[int] = None) -> torch.Tensor:
    """Same contract as :func:`ring_attention` (``[B, S/cp, H, D]`` slices in, local output out), no ring: see the section
    comment above.  ``layout="zigzag"``: the local slice is chunks (r, 2·cp−1−r) of the sequence (``utils.batch_utils`` cuts
    batches that way) — causal work is then balanced over the ranks.  Opt-in from the models with ``NXD_CP_PULL=1`` until the
    symmetric-memory path has run on hardware.  ``sliding_window``: as in :func:`ring_attention`; blocks wholly outside the window
    are neither read nor computed."""
    group = group if group is not None else ps.get_context_model_parallel_group()
    scale = scale if scale is not None else 1.0 / math.sqrt(q.shape[-1])
    window = _window_arg(sliding_window, causal)
    if dist.get_world_size(group) == 1:
        return block_attention(q, k, v, causal, scale, window)[0]
    return _PullAttention.apply(q, k, v, causal, scale, group, layout, window)
