"""Attention dropout in the flash kernels (H100, sm_90a) at head_dim 64, 80, 96 and 128.

The reference for every check is the host rule ``ops.attention.attention_dropout_keep``:
- O, dQ, dK and dV against float64 attention that applies the host mask, with GQA, a key-padding mask, causal attention
  and a sliding window, and the LSE bit-identical to the p = 0 run (it uses the undropped probabilities);
- exact checks that each of the forward, dK/dV and dQ kernels drops exactly the elements the rule drops, over several
  query and key tiles;
- the same mask for every memory layout, the same result for the same seed, and no host sync on the way.
"""
import math
import os

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


def _seed(s):
    return torch.tensor([s], dtype=torch.int64, device="cuda")


def _keep(seed, B, H, Sq, Sk, p, head_offset=0):
    from neuronx_distributed_b200.ops import attention

    return attention.attention_dropout_keep(seed, B, H, Sq, Sk, p, head_offset).cuda()


def _ref64(q, k, v, go, causal, scale, mask, window, keep, p):
    """float64 (O, LSE, dQ, dK, dV) of attention whose probabilities are multiplied by keep / (1 − p)."""
    from neuronx_distributed_b200.ops import attention

    B, Sq, H, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    g = H // Hkv
    qd, kd, vd, gd = (t.double() for t in (q, k, v, go))
    kk, vv = kd.repeat_interleave(g, 2), vd.repeat_interleave(g, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", qd, kk) * scale
    vis = torch.ones(B, 1, Sq, Sk, dtype=torch.bool, device=q.device)
    if causal:
        vis = vis & attention.window_visibility(Sq, Sk, window, q.device)
    if mask is not None:
        vis = vis & mask.bool()[:, None, None, :]
    s = s.masked_fill(~vis, float("-inf"))
    lse = torch.logsumexp(s, -1)
    pr = torch.where(vis, torch.exp(s - lse.unsqueeze(-1).clamp_min(-1e300)), torch.zeros((), dtype=s.dtype, device=s.device))
    z = keep.double() / (1 - p)
    o = torch.einsum("bhqk,bkhd->bqhd", pr * z, vv)
    dp = torch.einsum("bqhd,bkhd->bhqk", gd, vv)
    delta = (gd * o).sum(-1).transpose(1, 2).unsqueeze(-1)
    ds = pr * (dp * z - delta)
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kk) * scale
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, qd).view(B, Sk, Hkv, g, D).sum(3) * scale
    dv = torch.einsum("bhqk,bqhd->bkhd", pr * z, gd).view(B, Sk, Hkv, g, D).sum(3)
    return o, lse, dq, dk, dv


def _run(q, k, v, go, causal, scale, mask=None, window=0, p=0.0, seed=None, head_offset=0):
    """(O, LSE, dQ, dK, dV) from the extension."""
    from neuronx_distributed_b200.ops import _ext, attention

    e = _ext.ext()
    tv = attention._tma_view
    q, k, v, go = tv(q), tv(k), tv(v), tv(go)
    o, lse = e.flash_attn_fwd(q, k, v, causal, scale, True, mask, window, 0, p, seed, head_offset)
    dq, dk, dv = e.flash_attn_bwd(go, q, k, v, o, lse, causal, scale, True, None, mask, window, 0, p, seed, head_offset)
    return o, lse, dq, dk, dv


def _rand(B, Sq, Sk, H, Hkv, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()   # noqa: E731
    return rn(B, Sq, H, D), rn(B, Sk, Hkv, D), rn(B, Sk, Hkv, D), rn(B, Sq, H, D)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("kind", ["plain", "masked", "causal", "window"])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_vs_float64(_ext, D, kind, p):
    """GQA H = 4 / Hkv = 2, S = 200 (ragged last tiles), head offset 2, against float64 with the host mask."""
    B, S, H, Hkv = 2, 200, 4, 2
    q, k, v, go = _rand(B, S, S, H, Hkv, D, seed=D + int(p * 10))
    scale = 1.0 / math.sqrt(D)
    causal = kind in ("causal", "window")
    window = 37 if kind == "window" else 0
    mask = None
    if kind == "masked":
        mask = torch.arange(S, device="cuda")[None, :] < torch.tensor([S, 111], device="cuda")[:, None]
    seed = 0x5EED0000 + D
    got = _run(q, k, v, go, causal, scale, mask, window, p, _seed(seed), 2)
    keep = _keep(seed, B, H, S, S, p, head_offset=2)
    ref = _ref64(q, k, v, go, causal, scale, mask, window or None, keep, p)
    o, lse, dq, dk, dv = got
    assert _rel(o, ref[0]) < 2e-2, (D, kind, p)
    for name, a, b in (("dq", dq, ref[2]), ("dk", dk, ref[3]), ("dv", dv, ref[4])):
        assert _rel(a, b) < 3e-2, (D, kind, p, name, _rel(a, b))
    lse0 = _run(q, k, v, go, causal, scale, mask, window)[1]
    assert torch.equal(lse, lse0)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_each_kernel_applies_exactly_the_host_mask(_ext, D, p):
    """q = k = 0 makes P uniform.  With V (forward), dO (dK/dV) or K (dQ) one-hot over a chunk of D keys or queries, each
    output column reads one element of the mask: O[i, d] ≠ 0 iff (i, c·D + d) is kept; dV[j, d] ≠ 0 iff (c·D + d, j) is
    kept (dO on one head of each GQA pair at a time); dQ[i, d] > 0 iff (i, c·D + d) is kept (constant V and dO: a kept
    element gives P·(dP/(1 − p) − δ) > 0, a dropped one −P·δ < 0).  S = 200: four 64-key tiles, two 128-row tiles."""
    B, S, H, Hkv = 2, 200, 4, 2
    scale = 1.0 / math.sqrt(D)
    seed = 777 + D
    keep = _keep(seed, B, H, S, S, p)
    z = torch.zeros(B, S, H, D, device="cuda", dtype=torch.bfloat16)
    zk = torch.zeros(B, S, Hkv, D, device="cuda", dtype=torch.bfloat16)
    for c in range((S + D - 1) // D):
        cols = torch.arange(c * D, min(S, (c + 1) * D), device="cuda")
        n = len(cols)
        onehot = torch.zeros(B, S, Hkv, D, device="cuda", dtype=torch.bfloat16)
        onehot[:, cols, :, torch.arange(n, device="cuda")] = 1
        # forward: V one-hot over keys c·D + d
        o, *_ = _run(z, zk, onehot, z, False, scale, p=p, seed=_seed(seed))
        want = keep[:, :, :, cols].permute(0, 2, 1, 3)                               # [B, S_q, H, n]
        assert torch.equal(o[..., :n] != 0, want), (D, p, c, "forward")
        # dK/dV: dO one-hot over queries c·D + d on heads h ≡ r (mod 2), so dV of kv head hk reads head 2·hk + r
        for r in range(2):
            go = torch.zeros(B, S, H, D, device="cuda", dtype=torch.bfloat16)
            go[:, cols, r::2, torch.arange(n, device="cuda")] = 1
            dv = _run(z, zk, zk, go, False, scale, p=p, seed=_seed(seed))[4]
            want = keep[:, r::2][:, :, cols, :].permute(0, 3, 1, 2)                 # [B, S_kv, Hkv, n]
            assert torch.equal(dv[..., :n] != 0, want), (D, p, c, r, "dkdv")
        # dQ: K one-hot over keys c·D + d, V = dO = 1/2
        half = torch.full((B, S, Hkv, D), 0.5, device="cuda", dtype=torch.bfloat16)
        dq = _run(z, onehot, half, torch.full_like(z, 0.5), False, scale, p=p, seed=_seed(seed))[2]
        want = keep[:, :, :, cols].permute(0, 2, 1, 3)
        assert torch.equal(dq[..., :n] > 0, want), (D, p, c, "dq")
        assert (dq[..., :n] != 0).all()


def _layouts(q, k, v):
    """The same values as [B,S,H,D], [S,B,H,D] memory and slices of a fused [S, B, (H + 2·Hkv)·D] projection."""
    B, S, H, D = q.shape
    Hkv = k.shape[2]
    sb = lambda t: t.transpose(0, 1).contiguous().transpose(0, 1)               # noqa: E731
    f = torch.cat([t.transpose(0, 1).reshape(S, B, -1) for t in (q, k, v)], -1).contiguous()
    fused = (f[..., : H * D].view(S, B, H, D).transpose(0, 1), f[..., H * D:(H + Hkv) * D].view(S, B, Hkv, D).transpose(0, 1),
             f[..., (H + Hkv) * D:].view(S, B, Hkv, D).transpose(0, 1))
    return {"bshd": (q, k, v), "sbhd": (sb(q), sb(k), sb(v)), "fused": fused}


@pytest.mark.parametrize("D", DIMS)
def test_layouts_seeds_and_reproducibility(_ext, D):
    """One seed: the same O and gradients bit for bit for every layout and for a repeated call; another seed differs."""
    from neuronx_distributed_b200.ops import attention

    q, k, v, go = _rand(2, 200, 200, 4, 2, D, seed=5 * D)
    results = {}
    for name, (a, b, c) in _layouts(q, k, v).items():
        for rep in range(2):
            qg, kg, vg = (t.detach().requires_grad_(True) for t in (a, b, c))
            o = attention.flash_attention(qg, kg, vg, causal=True, dropout_p=0.2, dropout_seed=_seed(99))
            o.backward(go)
            results[name, rep] = [t.contiguous() for t in (o, qg.grad, kg.grad, vg.grad)]
    ref = results["bshd", 0]
    for key, got in results.items():
        for a, b in zip(got, ref):
            assert torch.equal(a, b), (D, key)
    other = attention.flash_attention(q, k, v, causal=True, dropout_p=0.2, dropout_seed=_seed(100))
    assert not torch.equal(other, ref[0])


def test_reference_entry_points_take_dropout(_ext):
    """``nki_flash_attn_func`` / ``NKIAttnFunc.apply`` with ``dropout_p`` are ``flash_attention`` with the same seed on the
    kernels (both layouts), draw a seed when given none, and refuse dropout on inputs the kernels do not take."""
    from neuronx_distributed_b200.kernels import NKIAttnFunc, nki_flash_attn_func
    from neuronx_distributed_b200.kernels.kernel_utils import permute
    from neuronx_distributed_b200.ops import attention

    q, k, v, go = (t.transpose(1, 2) for t in _rand(2, 256, 256, 4, 4, 64, seed=11))      # [B, H, S, D]
    seed = torch.tensor([4321], dtype=torch.int32, device="cuda")
    want = attention.flash_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), causal=True, dropout_p=0.1,
                                     dropout_seed=seed).transpose(1, 2)
    assert torch.equal(nki_flash_attn_func(q, k, v, dropout_p=0.1, seed=seed, transpose_nki_inputs=False), want)
    qt, kt, _ = permute(q, k, v)
    assert torch.equal(NKIAttnFunc.apply(qt, kt, v, None, True, True, seed, 0.1), want)
    assert not torch.equal(nki_flash_attn_func(q, k, v, dropout_p=0.0, transpose_nki_inputs=False), want)
    qg = q.detach().requires_grad_(True)
    torch.manual_seed(3)
    o = nki_flash_attn_func(qg, k, v, dropout_p=0.1, transpose_nki_inputs=False)
    o.backward(go)
    torch.manual_seed(3)
    assert torch.equal(nki_flash_attn_func(q, k, v, dropout_p=0.1, transpose_nki_inputs=False), o)
    assert qg.grad is not None and torch.isfinite(qg.grad).all()
    with pytest.raises(AssertionError):
        nki_flash_attn_func(q.float(), k.float(), v.float(), dropout_p=0.1, transpose_nki_inputs=False)


def test_no_host_sync(_ext):
    """The seed is drawn and read on the device: forward and backward never synchronise with the host."""
    from neuronx_distributed_b200.ops import attention

    q, k, v, go = _rand(2, 256, 256, 4, 4, 64, seed=1)
    qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        o = attention.flash_attention(qg, kg, vg, causal=True, dropout_p=0.1)
        o.backward(go)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert qg.grad is not None and torch.isfinite(o).all()


# ---- models in train mode: kernels vs the host-rule fallback (NXD_DISABLE_OWN_ATTENTION=1) ---------------------------------
def _one_rank_model_parallel():
    import torch.distributed as dist

    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29546")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    if not ps.model_parallel_is_initialized():
        ps.initialize_model_parallel(1)


def _bert(p, kw):
    from neuronx_distributed_b200.models import bert

    m = bert.BertModel(bert.BertConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                                       num_attention_heads=4, max_position_embeddings=256, hidden_dropout_prob=0.0,
                                       attention_probs_dropout_prob=p, **kw))
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, 512, (3, 160), device="cuda", generator=g)
    am = (torch.arange(160, device="cuda")[None, :] < torch.tensor([160, 97, 33], device="cuda")[:, None]).long()
    return m, lambda: m(ids, torch.zeros_like(ids), am)[0]


def _neox(p, kw):
    from neuronx_distributed_b200.models import gpt_neox

    m = gpt_neox.GPTNeoXForCausalLM(gpt_neox.GPTNeoXConfig(vocab_size=512, hidden_size=256, intermediate_size=1024,
                                                           num_hidden_layers=2, num_attention_heads=4,
                                                           max_position_embeddings=256, attention_dropout=p, **kw))
    ids = torch.randint(0, 512, (2, 150), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    return m, lambda: m(ids)[1]


@pytest.mark.parametrize("name,make", [("bert_d64", _bert), ("neox_d64", _neox)])
def test_models_train_with_attention_dropout(_ext, monkeypatch, name, make):
    """Train mode, attention dropout 0.1: loss and gradients on the kernels match the host-rule fallback; eval mode equals
    the model without dropout bit for bit."""
    _one_rank_model_parallel()
    kw = dict(dtype=torch.bfloat16, device=torch.device("cuda", 0))
    results = []
    for disable in ("0", "1"):
        monkeypatch.setenv("NXD_DISABLE_OWN_ATTENTION", disable)
        torch.manual_seed(0)
        m, fwd = make(0.1, kw)
        m.train()
        n0 = _ext.launches()
        torch.manual_seed(5)
        out = fwd().float()
        w = torch.randn(out.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
        loss = (out * w).sum() / out.numel() ** 0.5
        loss.backward()
        torch.cuda.synchronize()
        results.append((float(loss), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None},
                        _ext.launches() - n0))
    (l_own, g_own, n_own), (l_ref, g_ref, n_ref) = results
    assert n_own >= n_ref + 2 * 4, "own attention kernels did not run"
    assert abs(l_own - l_ref) <= 2e-2 * max(1.0, abs(l_ref)), (name, l_own, l_ref)
    gmax = max(g.abs().max().item() for g in g_ref.values())
    for n in g_ref:
        if n.endswith("attention.key.bias"):                  # exact gradient 0: both hold rounding noise only
            assert max(g_own[n].abs().max().item(), g_ref[n].abs().max().item()) < 1e-3 * gmax, (name, n)
            continue
        assert _rel(g_own[n].float(), g_ref[n].double()) < 5e-2, (name, n, _rel(g_own[n].float(), g_ref[n].double()))
    monkeypatch.setenv("NXD_DISABLE_OWN_ATTENTION", "0")
    outs = []
    for p in (0.1, 0.0):
        torch.manual_seed(0)
        m, fwd = make(p, kw)
        m.eval()
        with torch.no_grad():
            outs.append(fwd())
    assert torch.equal(outs[0], outs[1])
