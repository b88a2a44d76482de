"""Context-parallel sliding-window attention on the H100 (sm_90a).

- The windowed flash kernels with a query offset (one off-diagonal CP block: query i sees keys i + off − W < j ≤ i + off)
  against float64 references from the same bf16 inputs, with and without an LSE gradient, for blocks that are fully visible,
  partly visible and partly empty.  Empty rows give O = 0, LSE = −inf and dQ = 0; keys no row sees give dK = dV = 0.
- off = 0 is bit-identical to ``flash_attention(…, sliding_window=W)``, and the offset backward is bit-reproducible.
- A one-process emulation of CP (the block plan, ``block_attention`` and the LSE merge, exactly as ring and pull attention
  run them) equals windowed flash attention on the full sequence at the Mistral-7B per-GPU shape, forward and backward.
- With at least 2 GPUs, a real NCCL ``ring_attention`` does too.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DIMS = (64, 80, 96, 128)


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _rel(a, b):
    return ((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _relf(a, b):
    """Frobenius-norm relative difference."""
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


# CP against one full-sequence kernel call: both sides round to bf16 (the CP side every block's O and gradients before they
# are merged or summed), and one bf16 rounding alone is ≈ 1.6·10⁻³ relative RMS, so two independent roundings differ by
# ≈ 2.3·10⁻³.  Measured on an H100: O 0.9–1.7·10⁻³, gradients 1.4–2.9·10⁻³ for cp 2 / 4 / 8 and both layouts.  A lost or
# repeated block changes the softmax weights of whole rows, far beyond rounding.
CP_TOL = 4e-3


def _vis(c, W, off, device="cuda"):
    i = torch.arange(c, device=device)[:, None] + off
    j = torch.arange(c, device=device)[None, :]
    return (j <= i) & (j > i - W)


def _ref64(q, k, v, go, glse, scale, vis):
    """float64 (O, LSE, dQ, dK, dV) with an LSE gradient ``glse`` [B, H, S] (or None); a row that sees no key gets O = 0,
    LSE = −inf and zero gradients."""
    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    g = H // Hkv
    qd, kd, vd, gd = (t.double() for t in (q, k, v, go))
    kk, vv = kd.repeat_interleave(g, 2), vd.repeat_interleave(g, 2)
    s = (torch.einsum("bqhd,bkhd->bhqk", qd, kk) * scale).masked_fill(~vis, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.where(vis, torch.exp(s - lse.unsqueeze(-1).clamp_min(-1e300)), torch.zeros((), dtype=s.dtype, device=s.device))
    o = torch.einsum("bhqk,bkhd->bqhd", p, vv)
    dp = torch.einsum("bqhd,bkhd->bhqk", gd, vv)
    delta = (gd * o).sum(-1).transpose(1, 2)
    if glse is not None:
        delta = delta - glse.double()
    ds = p * (dp - delta.unsqueeze(-1))
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kk) * scale
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, qd).view(B, Sk, Hkv, g, D).sum(3) * scale
    dv = torch.einsum("bhqk,bqhd->bkhd", p, gd).view(B, Sk, Hkv, g, D).sum(3)
    return o, lse, dq, dk, dv


def _make(B, S, H, Hkv, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()   # noqa: E731
    return rn(B, S, H, D), rn(B, S, Hkv, D), rn(B, S, Hkv, D), rn(B, S, H, D), torch.randn(B, H, S, device="cuda", generator=g)


def _run(q, k, v, go, glse, scale, window, off):
    from neuronx_distributed_b200.ops import _ext

    e = _ext.ext()
    o, lse = e.flash_attn_fwd(q, k, v, True, scale, False, None, window, off)
    dq, dk, dv = e.flash_attn_bwd(go, q, k, v, o, lse, True, scale, False, glse, None, window, off)
    return o, lse, dq, dk, dv


def _offset_cases(c):
    """(q_offset, W): offsets c and 2c with a window that keeps the block fully visible, partly visible, partly empty (rows
    ≥ W − off + c − 1 see no key), and W = 1 at offset c (every row empty)."""
    return ((c, 2 * c), (c, c + c // 2), (c, c // 2), (c, 1), (2 * c, 3 * c), (2 * c, 2 * c + c // 3), (2 * c, c + c // 2))


@pytest.mark.parametrize("c", (64, 200, 1024))
@pytest.mark.parametrize("D", DIMS)
def test_offset_window_vs_float64(D, c):
    scale = 1.0 / math.sqrt(D)
    for G in (1, 4):
        H, Hkv = 8, 8 // G
        for off, W in _offset_cases(c):
            q, k, v, go, glse = _make(1, c, H, Hkv, D, seed=D * 7919 + c * 31 + off + W + G)
            vis = _vis(c, W, off)
            for g_lse in (None, glse.contiguous()):
                what = (D, c, G, off, W, g_lse is not None)
                got = _run(q, k, v, go, g_lse, scale, W, off)
                ref = _ref64(q, k, v, go, g_lse, scale, vis[None, None])
                o, lse, dq, dk, dv = got
                ro, rl, rdq, rdk, rdv = ref
                for t in got:
                    assert not torch.isnan(t).any(), what
                fin = torch.isfinite(rl)
                assert torch.equal(torch.isfinite(lse), fin), what
                if fin.any():
                    assert (lse[fin].double() - rl[fin]).abs().max().item() < 2e-2, what
                for name, a, b in (("o", o, ro), ("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
                    assert _rel(a, b) < 3e-2 if b.abs().max() > 0 else not a.any(), (what, name, _rel(a, b))
                empty_rows = ~vis.any(1)
                unseen_keys = ~vis.any(0)
                assert not o[:, empty_rows].any() and not dq[:, empty_rows].any(), what
                assert bool(torch.isneginf(lse[..., empty_rows]).all()), what
                assert not dk[:, unseen_keys].any() and not dv[:, unseen_keys].any(), what


@pytest.mark.parametrize("D", DIMS)
def test_zero_offset_is_the_diagonal_rule_and_offset_backward_reproducible(D):
    from neuronx_distributed_b200.ops import attention

    S, scale = 1000, 1.0 / math.sqrt(D)
    q, k, v, go, glse = _make(2, S, 8, 2, D, seed=97 + D)
    for W in (1, 65, 200, S):
        qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
        ref = attention.flash_attention(qa, ka, va, causal=True, sliding_window=W)
        ref.backward(go)
        qb, kb, vb = (t.clone().requires_grad_(True) for t in (q, k, v))
        out, _ = attention.flash_attention_with_lse(qb, kb, vb, True, scale, W, 0)
        out.backward(go)
        assert torch.equal(out, ref) and torch.equal(qb.grad, qa.grad) and torch.equal(kb.grad, ka.grad), (D, W)
        assert torch.equal(vb.grad, va.grad), (D, W)
    c = S // 2
    qc, kc, vc, gc = (t[:, :c].contiguous() for t in (q, k, v, go))
    for off, W in ((c, c), (2 * c, 2 * c + 7)):
        a = _run(qc, kc, vc, gc, glse[..., :c].contiguous(), scale, W, off)
        b = _run(qc, kc, vc, gc, glse[..., :c].contiguous(), scale, W, off)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), (D, off, W)


def test_offset_arguments_are_checked():
    from neuronx_distributed_b200.ops import _ext, attention

    e = _ext.ext()
    q, k, v, go, _ = _make(1, 128, 4, 4, 128, seed=1)
    with pytest.raises(RuntimeError, match="q_offset"):
        e.flash_attn_fwd(q, k, v, True, 0.1, True, None, 16, -1)
    with pytest.raises(RuntimeError, match="q_offset needs a sliding window"):
        e.flash_attn_fwd(q, k, v, True, 0.1, True, None, 0, 64)
    with pytest.raises(RuntimeError, match="causal"):
        e.flash_attn_fwd(q, k, v, False, 0.1, True, None, 16, 64)
    o, lse = e.flash_attn_fwd(q, k, v, True, 0.1, True)
    with pytest.raises(RuntimeError, match="q_offset needs a sliding window"):
        e.flash_attn_bwd(go, q, k, v, o, lse, True, 0.1, True, None, None, 0, 64)
    with pytest.raises(RuntimeError, match="q_offset"):
        e.flash_attn_bwd(go, q, k, v, o, lse, True, 0.1, True, None, None, 16, -1)
    with pytest.raises(ValueError):
        attention.flash_attention_with_lse(q, k, v, True, 0.1, None, 64)
    with pytest.raises(ValueError):
        attention.flash_attention_with_lse(q, k, v, False, 0.1, 16, 0)


def _emulate_cp(q, k, v, cp, layout, W, scale):
    """CP attention of every rank in one process, as ring / pull attention compute it: the block plan, ``block_attention`` per
    block and the LSE merge.  q/k/v are fp32 leaves cast to bf16 per block, so gradients of the blocks add in fp32.  Returns
    the output in global order."""
    from neuronx_distributed_b200.modules.attention.ring import _chunk_ids, _merge_block, _visible_pairs, block_attention

    n = len(_chunk_ids(0, cp, layout))
    c = q.shape[1] // (cp * n)
    chunk = lambda t, g: t[:, g * c:(g + 1) * c].bfloat16()     # noqa: E731
    outs = [None] * (cp * n)
    for r in range(cp):
        mine = _chunk_ids(r, cp, layout)
        acc = [(None, None)] * n
        for qi, src, kj, causal, off in _visible_pairs(r, cp, layout, True, W, c):
            gk = _chunk_ids(src, cp, layout)[kj]
            o_b, lse_b = block_attention(chunk(q, mine[qi]), chunk(k, gk), chunk(v, gk), causal, scale, W, off)
            acc[qi] = _merge_block(*acc[qi], o_b, lse_b)
        for qi, g in enumerate(mine):
            outs[g] = acc[qi][0]
    return torch.cat(outs, dim=1)


@pytest.mark.parametrize("layout", ("contiguous", "zigzag"))
@pytest.mark.parametrize("cp", (2, 4, 8))
def test_cp_emulation_matches_full_window_attention(cp, layout):
    from neuronx_distributed_b200.ops import attention

    B, S, H, Hkv, D, W = 1, 8192, 32, 8, 128, 4096
    scale = 1.0 / math.sqrt(D)
    q, k, v, go, _ = _make(B, S, H, Hkv, D, seed=cp * 10 + (layout == "zigzag"))
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    ref = attention.flash_attention(qa, ka, va, causal=True, sliding_window=W)
    ref.backward(go)
    qb, kb, vb = (t.float().requires_grad_(True) for t in (q, k, v))
    out = _emulate_cp(qb, kb, vb, cp, layout, W, scale)
    out.backward(go.float())
    errs = {name: _relf(a, b) for name, a, b in
            (("o", out, ref), ("dq", qb.grad, qa.grad), ("dk", kb.grad, ka.grad), ("dv", vb.grad, va.grad))}
    assert all(e < CP_TOL for e in errs.values()), (cp, layout, errs)


def _nccl_ring(rank, world):
    import torch.distributed as dist

    from neuronx_distributed_b200.modules.attention.ring import ring_attention
    from neuronx_distributed_b200.ops import attention
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=1, context_parallel_size=world)
    B, S, H, Hkv, D, W = 1, 8192, 32, 8, 128, 4096
    q, k, v, go, _ = _make(B, S, H, Hkv, D, seed=5)            # same seed on every rank: the same global tensors
    c = S // world
    sl = slice(rank * c, (rank + 1) * c)
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    ref = attention.flash_attention(qa, ka, va, causal=True, sliding_window=W)
    ref.backward(go)
    ql, kl, vl = (t[:, sl].clone().requires_grad_(True) for t in (q, k, v))
    out = ring_attention(ql, kl, vl, causal=True, sliding_window=W)
    out.backward(go[:, sl])
    for name, a, b in (("o", out, ref[:, sl]), ("dq", ql.grad, qa.grad[:, sl]), ("dk", kl.grad, ka.grad[:, sl]),
                       ("dv", vl.grad, va.grad[:, sl])):
        assert _relf(a, b) < CP_TOL, (rank, name, _relf(a, b))
    dist.barrier()


@pytest.mark.multigpu
def test_nccl_ring_attention_window_matches_full():
    """NCCL refuses two ranks on one device, so this needs one GPU per rank."""
    from dist_utils import run_distributed

    run_distributed(_nccl_ring, torch.cuda.device_count(), use_cuda=True, timeout=600)
