"""Sliding-window attention on the H100 (sm_90a): the flash kernels (forward, dK/dV, dQ) and the decode kernels with a
window W (query i sees keys i − W < j ≤ i), against float64 references computed from the same bf16 inputs.

Besides the float64 bounds (those of ``test_attention_head_dims_gpu``), three properties are checked exactly:
- W ≥ S visits the same key and query tiles in the same order as the causal kernels, so it is bit-identical to them;
- every gradient element is written by one thread, so the windowed backward is reproducible;
- the decode kernel reads only the cache rows inside the window: NaN in every other row changes nothing.
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


def _vis(S, W, mask=None, device="cuda"):
    """[B or 1, 1, S, S] bool: i − W < j ≤ i (W = None: causal) and the key-padding mask."""
    i = torch.arange(S, device=device)[:, None]
    j = torch.arange(S, device=device)[None, :]
    vis = (j <= i) if W is None else (j <= i) & (j > i - W)
    vis = vis[None, None]
    return vis if mask is None else vis & mask.bool()[:, None, None, :]


def _ref64(q, k, v, go, scale, vis):
    """float64 (O, LSE, dQ, dK, dV); a query row that sees no key gets O = 0, LSE = −inf and zero gradients."""
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
    ds = p * (dp - (gd * o).sum(-1).transpose(1, 2).unsqueeze(-1))
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kk) * scale
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, qd).view(B, Sk, Hkv, g, D).sum(3) * scale
    dv = torch.einsum("bhqk,bqhd->bkhd", p, gd).view(B, Sk, Hkv, g, D).sum(3)
    return o, lse, dq, dk, dv


def _make(layout, B, S, H, Hkv, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()   # noqa: E731
    if layout == "bshd":
        q, k, v = rn(B, S, H, D), rn(B, S, Hkv, D), rn(B, S, Hkv, D)
    elif layout == "sbhd":
        q, k, v = rn(S, B, H, D).transpose(0, 1), rn(S, B, Hkv, D).transpose(0, 1), rn(S, B, Hkv, D).transpose(0, 1)
    else:                                                                             # slices of a fused QKV projection
        f = rn(S, B, (H + 2 * Hkv) * D)
        q = f[..., : H * D].view(S, B, H, D).transpose(0, 1)
        k = f[..., H * D:(H + Hkv) * D].view(S, B, Hkv, D).transpose(0, 1)
        v = f[..., (H + Hkv) * D:].view(S, B, Hkv, D).transpose(0, 1)
    return q, k, v, rn(B, S, H, D)


def _run(q, k, v, go, scale, window, mask=None):
    """(O, LSE, dQ, dK, dV) from the extension, causal, through the calls the autograd front-end makes."""
    from neuronx_distributed_b200.ops import _ext, attention

    e = _ext.ext()
    tv = attention._tma_view
    q, k, v, go = tv(q), tv(k), tv(v), tv(go)
    o, lse = e.flash_attn_fwd(q, k, v, True, scale, True, mask, window)
    dq, dk, dv = e.flash_attn_bwd(go, q, k, v, o, lse, True, scale, True, None, mask, window)
    return o, lse, dq, dk, dv


def _check64(got, ref, what, single_key=False):
    """``single_key`` (W = 1): every row attends to itself alone, P = 1 and O = v_i exactly, so the exact dS = dO·(v_i − O)
    and with it dQ and dK are 0.  The kernels return the fp32 rounding of dP − δ there (about 1e-6 measured), which has no
    relative bound against 0; it is bounded absolutely instead, far below the O(1) gradients of any wider window."""
    o, lse, dq, dk, dv = got
    ro, rl, rdq, rdk, rdv = ref
    assert _rel(o, ro) < 2e-2, what
    fin = torch.isfinite(rl)
    assert torch.equal(torch.isfinite(lse), fin), what
    assert (lse[fin].double() - rl[fin]).abs().max().item() < 2e-2, what
    for name, a, b in (("dq", dq, rdq), ("dk", dk, rdk), ("dv", dv, rdv)):
        if single_key and name != "dv":
            assert b.abs().max().item() < 1e-12 and a.abs().max().item() < 1e-4, (what, name, a.abs().max().item())
            continue
        assert _rel(a, b) < 3e-2, (what, name, _rel(a, b))
    for t in got:
        assert not torch.isnan(t).any(), what


# (layout, S, H, Hkv, masked): GQA 1 / 4 / 8, the three memory layouts, S not a multiple of 64, with and without a mask
CASES = (("bshd", 333, 4, 4, False), ("sbhd", 1000, 8, 2, True), ("fused", 333, 8, 1, True))


@pytest.mark.parametrize("W", (1, 63, 64, 65, 200))
@pytest.mark.parametrize("D", DIMS)
def test_window_vs_float64(_ext, D, W):
    from neuronx_distributed_b200.ops import attention

    for layout, S, H, Hkv, masked in CASES:
        what = (D, W, layout, S, H // Hkv, masked)
        B = 2
        q, k, v, go = _make(layout, B, S, H, Hkv, D, seed=D * 1000 + W + S)
        mask = None
        if masked:
            mask = torch.rand(B, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(W)) < 0.75
            mask[1, 100:100 + min(W, 40)] = False          # at W ≤ 40 query 100 + W − 1 of batch 1 sees no key at all
        scale = 1.0 / math.sqrt(D)
        vis = _vis(S, W, mask)
        got = _run(q, k, v, go, scale, W, mask)
        ref = _ref64(q, k, v, go, scale, vis)
        _check64(got, ref, what, single_key=W == 1)
        o, lse, dq, dk, dv = got
        empty = ~vis.any(-1)[:, 0]                                                # [B, S] rows that see no key
        if masked:
            assert not dk[~mask].any() and not dv[~mask].any(), what
            if W <= 40:
                assert bool(empty[1, 100 + W - 1]), what
        if empty.any():
            assert not o[empty].any() and not dq[empty].any(), what
            assert bool((lse.transpose(1, 2)[empty] == float("-inf")).all()), what
        # the autograd front-end gives the same result and runs the kernels
        qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))
        n0 = _ext.launches()
        fo = attention.flash_attention(qg, kg, vg, causal=True, key_padding_mask=mask, sliding_window=W)
        fo.backward(go)
        assert _ext.launches() >= n0 + 4, what
        assert torch.equal(fo, o) and torch.equal(qg.grad, dq) and torch.equal(kg.grad, dk) and torch.equal(vg.grad, dv), what


@pytest.mark.parametrize("D", DIMS)
def test_window_at_least_s_is_bit_identical_to_causal(_ext, D):
    S = 333
    q, k, v, go = _make("sbhd", 2, S, 8, 2, D, seed=41 + D)
    mask = torch.rand(2, S, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)) < 0.8
    scale = 1.0 / math.sqrt(D)
    for m in (None, mask):
        causal = _run(q, k, v, go, scale, 0, m)
        for W in (S, S + 1, 1 << 30):
            got = _run(q, k, v, go, scale, W, m)
            assert all(torch.equal(a, b) for a, b in zip(got, causal)), (D, W, m is not None)


@pytest.mark.parametrize("D", DIMS)
def test_window_backward_is_bit_reproducible(_ext, D):
    q, k, v, go = _make("bshd", 2, 1000, 8, 2, D, seed=53 + D)
    mask = torch.rand(2, 1000, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) < 0.8
    scale = 1.0 / math.sqrt(D)
    for W, m in ((65, None), (200, mask), (1, mask)):
        a, b = _run(q, k, v, go, scale, W, m), _run(q, k, v, go, scale, W, m)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), (D, W, m is not None)


def test_window_arguments_are_checked(_ext):
    from neuronx_distributed_b200.ops import attention

    q, k, v, go = _make("bshd", 1, 128, 4, 4, 128, seed=1)
    e = _ext.ext()
    with pytest.raises(RuntimeError, match="causal"):
        e.flash_attn_fwd(q, k, v, False, 0.1, True, None, 16)
    with pytest.raises(RuntimeError, match="window"):
        e.flash_attn_fwd(q, k, v, True, 0.1, True, None, -1)
    with pytest.raises(ValueError):
        attention.flash_attention(q, k, v, causal=False, sliding_window=16)


# ---- decode ---------------------------------------------------------------------------------------------------------
def _decode_ref64(q, kc, vc, pos, W):
    """float64 decode attention of q [B,1,H,D] over caches [B,L,Hkv,D], keys pos − W < j ≤ pos."""
    B, _, H, D = q.shape
    L, Hkv = kc.shape[1], kc.shape[2]
    kk, vv = (t.double().repeat_interleave(H // Hkv, 2) for t in (kc, vc))
    s = torch.einsum("bhd,blhd->bhl", q[:, 0].double(), kk) / math.sqrt(D)
    j = torch.arange(L, device=q.device)[None, :]
    vis = (j <= pos[:, None]) & (j > pos[:, None] - W)
    s = s.masked_fill(~vis[:, None], float("-inf"))
    return torch.einsum("bhl,blhd->bhd", s.softmax(-1), vv).unsqueeze(1), vis


@pytest.mark.parametrize("G", (1, 2, 4, 8))
def test_decode_window_vs_float64_and_reads_only_the_window(_ext, G):
    from neuronx_distributed_b200.ops import attention

    W, L, H, D = 300, 4096, 8, 128
    pos = torch.tensor([17, W - 1, W, 3999], device="cuda")                      # pos < W, W − 1, W, pos ≫ W
    B, Hkv = pos.numel(), H // G
    g = torch.Generator(device="cuda").manual_seed(G)
    q = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    # strided caches: [L, B, Hkv, D] memory, and a [B, L, Hkv, 2D] buffer whose first half is the cache
    kc = torch.randn(L, B, Hkv, D, device="cuda", generator=g).bfloat16().transpose(0, 1)
    vc = torch.randn(B, L, Hkv, 2 * D, device="cuda", generator=g).bfloat16()[..., :D]
    n0 = _ext.launches()
    got = attention.decode_attention(q, kc, vc, pos, sliding_window=W)
    assert _ext.launches() > n0
    ref, vis = _decode_ref64(q, kc, vc, pos, W)
    assert _rel(got, ref) < 2e-2, G
    # NaN in every cache row outside each sequence's window: the kernel never reads them
    kn, vn = kc.clone(), vc.clone()
    kn[~vis], vn[~vis] = float("nan"), float("nan")
    got_nan = attention.decode_attention(q, kn, vn, pos, sliding_window=W)
    assert torch.isfinite(got_nan).all() and torch.equal(got_nan, got), G
    # no window: unchanged kernel, full causal prefix
    full, _ = _decode_ref64(q, kc, vc, pos, L + 1)
    assert _rel(attention.decode_attention(q, kc, vc, pos), full) < 2e-2


@pytest.mark.parametrize("G", (1, 4))
def test_decode_partial_window_matches_torch(_ext, G):
    """Flash-decoding's local partial on the kernel vs the torch path, local positions before, inside and past the shard."""
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial

    W, L, H, D = 100, 512, 8, 128
    local = torch.tensor([-40, -1, 0, 63, 99, 100, 400, 511, 530, 700], device="cuda")
    B, Hkv = local.numel(), H // G
    g = torch.Generator(device="cuda").manual_seed(7 + G)
    q = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = (torch.randn(B, L, Hkv, D, device="cuda", generator=g).bfloat16() for _ in range(2))
    n0 = _ext.launches()
    o, m, l = _local_partial(q, kc, vc, local, 1.0 / math.sqrt(D), sliding_window=W)
    assert _ext.launches() > n0
    ro, rm, rl = _local_partial(q.cpu(), kc.cpu(), vc.cpu(), local.cpu(), 1.0 / math.sqrt(D), sliding_window=W)
    ro, rm, rl = ro.cuda(), rm.cuda(), rl.cuda()
    none = torch.isinf(rm)
    assert torch.equal(torch.isinf(m), none) and bool(none[0].all()) and bool(none[-1].all())
    assert not o[none].any() and not l[none].any()
    assert (m[~none] - rm[~none]).abs().max().item() < 1e-3
    assert _rel(l[~none], rl[~none].double()) < 1e-2 and _rel(o[~none], ro[~none].double()) < 1e-2


# ---- models on CUDA in bf16 -------------------------------------------------------------------------------------------
def _one_rank_model_parallel():
    import torch.distributed as dist

    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29544")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    if not ps.model_parallel_is_initialized():
        ps.initialize_model_parallel(1)


def _mistral_cfg(**kw):
    from neuronx_distributed_b200.models.llama import LlamaConfig

    return LlamaConfig(vocab_size=1024, hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                       num_key_value_heads=2, max_position_embeddings=512, dtype=torch.bfloat16, device=torch.device("cuda", 0),
                       **kw)


def test_mistral_shaped_training_matches_sdpa(_ext, monkeypatch):
    """Loss and parameter gradients of a windowed Llama (W = 100 < S = 300) on the own kernels vs SDPA with the window mask."""
    from neuronx_distributed_b200.models.llama import LlamaForCausalLM

    _one_rank_model_parallel()
    ids = torch.randint(0, 1024, (2, 300), device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    results = []
    for disable in ("0", "1"):
        monkeypatch.setenv("NXD_DISABLE_OWN_ATTENTION", disable)
        torch.manual_seed(0)
        m = LlamaForCausalLM(_mistral_cfg(sliding_window=100))
        n0 = _ext.launches()
        loss, _ = m(ids, labels=ids)
        loss.backward()
        torch.cuda.synchronize()
        results.append((loss.item(), {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None},
                        _ext.launches() - n0))
    (l_own, g_own, n_own), (l_ref, g_ref, n_ref) = results
    assert n_own >= n_ref + 2 * 4, "own attention kernels did not run"
    assert abs(l_own - l_ref) <= 2e-2 * max(1.0, abs(l_ref)), (l_own, l_ref)
    assert g_own.keys() == g_ref.keys() and g_own
    for n in g_ref:
        assert _rel(g_own[n].float(), g_ref[n].double()) < 5e-2, (n, _rel(g_own[n].float(), g_ref[n].double()))


def test_mistral_shaped_inference_graph_and_sdpa(_ext, monkeypatch):
    """Prefill past the window and decode steps past it: the CUDA-graph replay of a decode step gives the eager logits bit for
    bit, and a run with attention on SDPA (teacher-forced on the same tokens) agrees on every confident greedy token."""
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.ops import attention

    _one_rank_model_parallel()
    W, P, N = 64, 160, 24
    torch.manual_seed(0)
    m = LlamaForInference(_mistral_cfg(sliding_window=W), batch_size=2, max_seq_len=512, on_device_sampling=False).eval()
    ids = torch.randint(0, 1024, (2, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    last = torch.tensor([P - 1, 120], device="cuda")

    def run(step):
        logits = [m.context_encoding(ids, last)]
        toks, pos = [logits[0].argmax(-1)], last + 1
        for _ in range(N):
            logits.append(step(toks[-1].view(2, 1), pos).clone())
            toks.append(logits[-1].argmax(-1))
            pos = pos + 1
        return torch.stack(toks, 1), logits

    eager_toks, eager_logits = run(m.token_generation)

    # CUDA graph of one decode step, replayed with each step's token and positions copied into its static inputs
    st_tok, st_pos = eager_toks[:, 0].view(2, 1).clone(), last + 1
    m.context_encoding(ids, last)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.token_generation(st_tok, st_pos)               # warm-up writes the same cache row the first replay writes
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_out = m.token_generation(st_tok, st_pos)

    def replay(tok, pos):
        st_tok.copy_(tok)
        st_pos.copy_(pos)
        graph.replay()
        return st_out

    graph_toks, graph_logits = run(replay)
    assert torch.equal(graph_toks, eager_toks)
    assert all(torch.equal(a, b) for a, b in zip(graph_logits, eager_logits))

    # SDPA run on the eager tokens: prefill through NXD_DISABLE_OWN_ATTENTION, decode through the fp32 SDPA branch
    monkeypatch.setenv("NXD_DISABLE_OWN_ATTENTION", "1")
    orig = attention.decode_attention
    monkeypatch.setattr(attention, "decode_attention", lambda q, k, v, p, sliding_window: orig(
        q.float(), k.float(), v.float(), p, sliding_window=sliding_window).to(q.dtype))
    ref_logits = [m.context_encoding(ids, last)]
    pos = last + 1
    for i in range(N):
        ref_logits.append(m.token_generation(eager_toks[:, i].view(2, 1), pos).clone())
        pos = pos + 1
    for i, (a, r) in enumerate(zip(eager_logits, ref_logits)):
        assert _rel(a.float(), r.double()) < 5e-2, (i, _rel(a.float(), r.double()))
        top2 = r.float().topk(2, -1).values
        sure = (top2[:, 0] - top2[:, 1]) > 0.05 * r.float().std()
        assert torch.equal(a.argmax(-1)[sure], r.argmax(-1)[sure]), i
