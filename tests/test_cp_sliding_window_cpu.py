"""Context parallelism with a sliding window (Mistral / Mixtral ``sliding_window``) on the CPU paths: the block plan covers the
windowed-causal mask exactly once, ring and pull attention equal dense windowed attention in forward and all gradients, the ring
stops after ceil((W − 1)/c) hops, rows that see no key in a block produce no NaN, and a windowed Llama gives the same logits
at CP = 2 (ring, pull, zigzag) as at CP = 1 once ``NXD_CP_WINDOW=1`` opts in."""
import math

import pytest
import torch

from dist_utils import run_distributed


def _windows(c, S):
    """W = 1, c − 1, c, c + 1, 2c + 3 and ≥ S (deduplicated, ≥ 1)."""
    return sorted({w for w in (1, c - 1, c, c + 1, 2 * c + 3, S) if w >= 1})


def _dense(q, k, v, window):
    """Dense causal attention over the full sequence, limited to the window when one is given; fp32 autograd reference."""
    from neuronx_distributed_b200.ops.attention import window_visibility

    S, H, Hkv, D = q.shape[1], q.shape[2], k.shape[2], q.shape[3]
    s = torch.einsum("bqhd,bkhd->bhqk", q, k.repeat_interleave(H // Hkv, 2)) / math.sqrt(D)
    s = s.masked_fill(~window_visibility(S, S, window), float("-inf"))
    return torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v.repeat_interleave(H // Hkv, 2))


@pytest.mark.parametrize("layout", ["contiguous", "zigzag"])
@pytest.mark.parametrize("cp", [1, 2, 3, 4])
def test_plan_covers_windowed_mask_exactly_once(cp, layout):
    from neuronx_distributed_b200.modules.attention.ring import _chunk_ids, _visible_pairs
    from neuronx_distributed_b200.ops.attention import window_visibility

    c = 5
    n_chunks = cp * (2 if layout == "zigzag" else 1)
    S = n_chunks * c
    for W in _windows(c, S) + [None]:
        covered = torch.zeros(S, S, dtype=torch.int64)
        for r in range(cp):
            for qi, src, kj, causal, off in _visible_pairs(r, cp, layout, True, W, c):
                gq, gk = _chunk_ids(r, cp, layout)[qi], _chunk_ids(src, cp, layout)[kj]
                assert off == (gq - gk) * c
                vis = window_visibility(c, c, W, q_offset=off) if causal else torch.ones(c, c, dtype=torch.bool)
                assert vis.any(), (r, qi, src, kj, W)
                if not causal:          # a block marked dense must be fully visible under the windowed rule
                    assert window_visibility(c, c, W, q_offset=off).all()
                covered[gq * c:(gq + 1) * c, gk * c:(gk + 1) * c] += vis.long()
        assert torch.equal(covered, window_visibility(S, S, W).long()), (cp, layout, W)


def test_ring_hops():
    from neuronx_distributed_b200.modules.attention.ring import ring_hops

    assert ring_hops(8, 8192, None) == 7
    assert ring_hops(8, 8192, 4096) == 1            # Mistral-7B at 64k, cp = 8: one neighbour
    assert ring_hops(8, 8192, 1) == 0
    assert ring_hops(8, 8192, 8193) == 1 and ring_hops(8, 8192, 8194) == 2
    assert ring_hops(4, 16, 10 ** 6) == 3


def _ring_window(rank, world):
    import torch.distributed as dist

    from neuronx_distributed_b200.modules.attention import ring
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=1, context_parallel_size=world)
    calls = [0]
    exchange = ring._exchange

    def counting(*a):
        calls[0] += 1
        return exchange(*a)

    ring._exchange = counting
    B, S, H, Hkv, D = 2, 16, 4, 2, 8
    c = S // world
    gen = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn(B, S, h, D, generator=gen) for h in (H, Hkv, Hkv))
    go = torch.randn(B, S, H, D, generator=gen)
    sl = slice(rank * c, (rank + 1) * c)
    for W in _windows(c, S) + [None]:
        ql, kl, vl = (t[:, sl].clone().requires_grad_(True) for t in (q, k, v))
        calls[0] = 0
        out = ring.ring_attention(ql, kl, vl, causal=True, sliding_window=W)
        fwd_calls = calls[0]
        out.backward(go[:, sl])
        bwd_calls = calls[0] - fwd_calls
        hops = world - 1 if W is None else min(world - 1, math.ceil((W - 1) / c))
        assert fwd_calls == hops and bwd_calls == hops, (W, fwd_calls, bwd_calls)
        qf, kf, vf = (t.clone().requires_grad_(True) for t in (q, k, v))
        ref = _dense(qf, kf, vf, W)
        ref.backward(go)
        for got, want in ((out, ref[:, sl]), (ql.grad, qf.grad[:, sl]), (kl.grad, kf.grad[:, sl]), (vl.grad, vf.grad[:, sl])):
            assert torch.isfinite(got).all(), W
            torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
        if W is not None and W >= S:        # a window that covers the sequence is the plain causal ring
            q2, k2, v2 = (t[:, sl].clone() for t in (q, k, v))
            torch.testing.assert_close(out.detach(), ring.ring_attention(q2, k2, v2, causal=True), rtol=0, atol=0)
    with pytest.raises(ValueError):
        ring.ring_attention(q[:, sl], k[:, sl], v[:, sl], causal=False, sliding_window=4)
    dist.barrier()


@pytest.mark.parametrize("world", [2, 4])
def test_ring_attention_window_matches_dense(world):
    run_distributed(_ring_window, world, timeout=180)


def _pull_window(rank, world, layout):
    import torch.distributed as dist

    from neuronx_distributed_b200.modules.attention.ring import pull_attention
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.utils.batch_utils import context_parallel_slice

    ps.initialize_model_parallel(tensor_model_parallel_size=1, context_parallel_size=world)
    B, S, H, Hkv, D = 2, 32, 4, 2, 8
    c = S // (world * (2 if layout == "zigzag" else 1))
    gen = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn(B, S, h, D, generator=gen) for h in (H, Hkv, Hkv))
    go = torch.randn(B, S, H, D, generator=gen)

    def cut(t):
        return context_parallel_slice(t, rank, world, 1, layout)

    for W in _windows(c, S):
        ql, kl, vl = (cut(t).clone().requires_grad_(True) for t in (q, k, v))
        out = pull_attention(ql, kl, vl, causal=True, layout=layout, sliding_window=W)
        out.backward(cut(go))
        qf, kf, vf = (t.clone().requires_grad_(True) for t in (q, k, v))
        ref = _dense(qf, kf, vf, W)
        ref.backward(go)
        for got, want in ((out, cut(ref)), (ql.grad, cut(qf.grad)), (kl.grad, cut(kf.grad)), (vl.grad, cut(vf.grad))):
            assert torch.isfinite(got).all(), W
            torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
    dist.barrier()


@pytest.mark.parametrize("layout", ["contiguous", "zigzag"])
@pytest.mark.parametrize("world", [2, 4])
def test_pull_attention_window_matches_dense(world, layout):
    run_distributed(_pull_window, world, layout, timeout=180)


def test_offset_block_with_empty_rows_and_merge_have_no_nan():
    """An off-diagonal block whose window leaves rows empty gives O = 0 and LSE = −inf there, merging two such rows keeps them so
    in either order, and the gradients through both stay finite."""
    from neuronx_distributed_b200.modules.attention.ring import _merge_block, block_attention

    gen = torch.Generator().manual_seed(1)
    B, c, H, Hkv, D = 1, 8, 4, 2, 8
    q, k, v = (torch.randn(B, c, h, D, generator=gen).requires_grad_(True) for h in (H, Hkv, Hkv))
    W = 3                                   # q_offset = c: row i sees keys i + c − 3 < j ≤ c − 1, so rows ≥ 2 see none
    o, lse = block_attention(q, k, v, True, D ** -0.5, W, c)
    assert torch.equal(o[:, 2:], torch.zeros_like(o[:, 2:]))
    assert torch.isneginf(lse[..., 2:]).all() and torch.isfinite(lse[..., :2]).all()
    o2, lse2 = block_attention(q, k, v, True, D ** -0.5, 1, c)          # W = 1 at offset c: every row empty
    assert torch.equal(o2, torch.zeros_like(o2)) and torch.isneginf(lse2).all()
    for a, b in (((o, lse), (o2, lse2)), ((o2, lse2), (o, lse))):
        out, m = _merge_block(*_merge_block(None, None, *a), *b)
        torch.testing.assert_close(out, o.float(), rtol=0, atol=0)
        torch.testing.assert_close(m, lse, rtol=0, atol=0)
        (out.sum() + m[..., :2].sum()).backward(retain_graph=True)
        for t in (q, k, v):
            assert torch.isfinite(t.grad).all()
            t.grad = None


def _llama_logits(rank, world, mode):
    import os

    os.environ["NXD_CP_PULL"] = "1" if mode == "pull" else "0"     # read when models.llama is imported (fresh worker process)
    os.environ["NXD_CP_WINDOW"] = "1"
    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.utils.batch_utils import context_parallel_slice

    ps.initialize_model_parallel(tensor_model_parallel_size=1, context_parallel_size=world)
    layout = "zigzag" if mode == "zigzag" else "contiguous"
    S, W = 32, 6                            # chunk 16 (8 for zigzag): the window reaches into the previous chunk only

    def logits(cp, window):
        cfg = LlamaConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                          num_key_value_heads=2, dtype=torch.float32, max_position_embeddings=S, context_parallel=cp,
                          cp_layout=layout, sliding_window=window)
        torch.manual_seed(7)
        model = LlamaForCausalLM(cfg)
        ids = torch.randint(0, 64, (2, S), generator=torch.Generator().manual_seed(100))
        with torch.no_grad():
            if cp:
                return model(context_parallel_slice(ids, rank, world, 1, layout))[1]
            return context_parallel_slice(model(ids)[1], rank, world, 0, layout)     # [S, B, V] → this rank's rows

    got, ref, no_window = logits(True, W), logits(False, W), logits(False, None)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)
    assert (ref - no_window).abs().max() > 1e-2          # control: the window changes the logits


@pytest.mark.parametrize("mode", ["ring", "pull", "zigzag"])
def test_llama_context_parallel_window_matches_single(mode):
    run_distributed(_llama_logits, 2, mode, timeout=180)
