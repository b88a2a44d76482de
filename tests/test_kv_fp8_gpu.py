"""fp8 (e4m3) KV cache on the H100 (sm_90a): the decode kernel reading e4m3 caches, the fused RoPE + append kernel writing
them, and a Mistral-shaped model served from an fp8 cache.

- Decode attention is compared with float64 attention over the *de-quantised* cache, so the bound is the bf16 kernel's.
- The append must produce the bytes ``KVCacheManager._q`` makes of the rows the bf16 kernel writes, including torch's
  non-saturating overflow rule and its reciprocal-multiply division.
"""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _rel(a, b):
    return ((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _deq(t, s):
    return t.double() * s


def _decode_ref64(q, kd, vd, pos, W):
    """float64 decode attention of q [B,1,H,D] over de-quantised caches [B,L,Hkv,D], keys pos − W < j ≤ pos."""
    B, _, H, D = q.shape
    L, Hkv = kd.shape[1], kd.shape[2]
    kk, vv = (t.repeat_interleave(H // Hkv, 2) for t in (kd, vd))
    s = torch.einsum("bhd,blhd->bhl", q[:, 0].double(), kk) / math.sqrt(D)
    j = torch.arange(L, device=q.device)[None, :]
    vis = (j <= pos[:, None]) & (j > pos[:, None] - W)
    s = s.masked_fill(~vis[:, None], float("-inf"))
    return torch.einsum("bhl,blhd->bhd", s.softmax(-1), vv).unsqueeze(1), vis


@pytest.mark.parametrize("G", (1, 2, 4, 8))
@pytest.mark.parametrize("W", (None, 300))
def test_decode_e4m3_vs_float64_on_dequantised_cache(_ext, G, W):
    from neuronx_distributed_b200.ops import attention

    L, H, D, ks, vs = 4096, 8, 128, 0.3, 0.7
    pos = torch.tensor([17, 299, 300, 3999], device="cuda")                  # below, at and past the window
    B, Hkv = pos.numel(), H // G
    g = torch.Generator(device="cuda").manual_seed(G)
    q = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    # strided caches: [L, B, Hkv, D] memory, and a [B, L, Hkv, 2D] buffer whose first half is the cache
    kc = (torch.randn(L, B, Hkv, D, device="cuda", generator=g) / ks).to(E4M3).transpose(0, 1)
    vc = (torch.randn(B, L, Hkv, 2 * D, device="cuda", generator=g) / vs).to(E4M3)[..., :D]
    n0 = _ext.launches()
    got = attention.decode_attention(q, kc, vc, pos, sliding_window=W, k_scale=ks, v_scale=vs)
    assert _ext.launches() > n0
    ref, vis = _decode_ref64(q, _deq(kc, ks), _deq(vc, vs), pos, W or L + 1)
    assert _rel(got, ref) < 2e-2, (G, W, _rel(got, ref))
    if W is not None:
        # NaN bytes in every row outside each sequence's window: the kernel never reads them
        kn, vn = kc.clone(), vc.clone()
        kn.view(torch.uint8)[~vis] = 0x7F
        vn.view(torch.uint8)[~vis] = 0x7F
        got_nan = attention.decode_attention(q, kn, vn, pos, sliding_window=W, k_scale=ks, v_scale=vs)
        assert torch.isfinite(got_nan).all() and torch.equal(got_nan, got), G


def test_decode_e4m3_argument_checks(_ext):
    e = _ext.ext()
    q = torch.randn(1, 1, 8, 128, device="cuda").bfloat16()
    kb = torch.randn(1, 64, 8, 128, device="cuda").bfloat16()
    k8 = kb.to(E4M3)
    pos = torch.tensor([10], device="cuda")
    with pytest.raises(RuntimeError, match="fp8 cache only"):
        e.decode_attention(q, kb, kb, pos, 0.1, 0, k_scale=2.0)
    with pytest.raises(RuntimeError, match="same dtype"):
        e.decode_attention(q, k8, kb, pos, 0.1)
    buf = torch.zeros(1 * 64 * 8 * 128 + 4, dtype=E4M3, device="cuda")
    odd = buf[4:].view(1, 64, 8, 128)                                         # 4-byte aligned base
    with pytest.raises(RuntimeError, match="8 bytes at a time"):
        e.decode_attention(q, odd, odd, pos, 0.1)
    with pytest.raises(RuntimeError, match="fp8 cache only"):
        e.decode_rope_kv(q, kb[:, :1], kb[:, :1], pos, torch.ones(64, 64, device="cuda"), torch.zeros(64, 64, device="cuda"),
                         kb, kb, v_scale=0.5)


@pytest.mark.parametrize("G", (1, 4))
def test_decode_partial_e4m3_matches_torch(_ext, G):
    """Flash-decoding's local partial on the kernel vs the torch path, local positions before, inside and past the shard."""
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial

    W, L, H, D, ks, vs = 100, 512, 8, 128, 0.3, 0.7
    local = torch.tensor([-40, -1, 0, 63, 99, 100, 400, 511, 530, 700], device="cuda")
    B, Hkv = local.numel(), H // G
    g = torch.Generator(device="cuda").manual_seed(7 + G)
    q = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    kc = (torch.randn(B, L, Hkv, D, device="cuda", generator=g) / ks).to(E4M3)
    vc = (torch.randn(B, L, Hkv, D, device="cuda", generator=g) / vs).to(E4M3)
    for window in (None, W):
        n0 = _ext.launches()
        o, m, l = _local_partial(q, kc, vc, local, 1.0 / math.sqrt(D), window, ks, vs)
        assert _ext.launches() > n0
        ro, rm, rl = _local_partial(q.cpu(), kc.cpu(), vc.cpu(), local.cpu(), 1.0 / math.sqrt(D), window, ks, vs)
        ro, rm, rl = ro.cuda(), rm.cuda(), rl.cuda()
        none = torch.isinf(rm)
        assert torch.equal(torch.isinf(m), none) and bool(none[0].all()) and bool(none[1].all())
        assert not o[none].any() and not l[none].any()
        assert (m[~none] - rm[~none]).abs().max().item() < 1e-3
        assert _rel(l[~none], rl[~none].double()) < 1e-2 and _rel(o[~none], ro[~none].double()) < 1e-2


@pytest.mark.parametrize("scale", (1.0, 0.3))
def test_decode_rope_kv_e4m3_bytes_equal_cache_rule(_ext, scale):
    """The e4m3 append writes ``KVCacheManager._q`` of the rows the bf16 append writes from the same inputs."""
    from neuronx_distributed_b200.inference.kv_cache import KVCacheManager
    from neuronx_distributed_b200.ops import rope
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    e = _ext.ext()
    B, H, Hkv, D, L = 3, 8, 2, 128, 64
    g = torch.Generator(device="cuda").manual_seed(11)
    f = torch.randn(B, 1, (H + 2 * Hkv) * D, device="cuda", generator=g).bfloat16() * 3
    if scale == 1.0:                                                          # the overflow rule: saturating vs NaN bytes
        special = torch.tensor([448, 464, 466, -466, float("inf"), float("-inf"), float("nan"), -0.0, 1e-4, -1e-4])
    else:
        # the division rule: at scale 0.3 these are the only finite bf16 values whose e4m3 byte differs between x · (1/scale)
        # and a true x / scale (found by enumerating every finite bf16 value)
        special = torch.tensor([0.00439453125, -0.00439453125])
    f[0, 0, H * D:H * D + special.numel()] = special.to(f.dtype)             # k head 0 of sequence 0 (position 0: no rotation)
    f[0, 0, (H + Hkv) * D + 7:(H + Hkv) * D + 7 + special.numel()] = special.to(f.dtype)       # v head 0
    q = f[..., :H * D].view(B, 1, H, D)
    k = f[..., H * D:(H + Hkv) * D].view(B, 1, Hkv, D)
    v = f[..., (H + Hkv) * D:].view(B, 1, Hkv, D)
    pos = torch.tensor([0, 5, 63], device="cuda")
    cos, sin = rope.rope_tables(L, D, 10000.0, torch.device("cuda"), 0, 1.0)
    kb = torch.zeros(B, L, Hkv, D, device="cuda", dtype=torch.bfloat16)
    vb = torch.zeros_like(kb)
    k8 = torch.zeros(B, L, Hkv, D, device="cuda", dtype=E4M3)
    v8 = torch.zeros_like(k8)
    qb = e.decode_rope_kv(q, k, v, pos, cos, sin, kb, vb)
    q8 = e.decode_rope_kv(q, k, v, pos, cos, sin, k8, v8, k_scale=scale, v_scale=scale)
    assert torch.equal(q8, qb)
    mgr = KVCacheManager(1, 1, 1, 1, 1, device="cuda", kv_quant=KVQuantizationConfig(scale=scale))
    b = torch.arange(B, device="cuda")
    for name, c8, cb in (("k", k8, kb), ("v", v8, vb)):
        want = mgr._q(cb[b, pos]).view(torch.uint8)
        got = c8[b, pos].view(torch.uint8)
        bad = (got != want).nonzero()
        assert bad.numel() == 0, (name, bad[:5].tolist(), got[tuple(bad[:5].t())].tolist(), want[tuple(bad[:5].t())].tolist())
        rest = torch.ones(B, L, dtype=torch.bool, device="cuda")
        rest[b, pos] = False
        assert not c8.view(torch.uint8)[rest].any(), name                     # no other row was written
    if scale == 1.0:
        for c8, off in ((k8, 0), (v8, 7)):                                   # 448, 464, 466, −466, inf, −inf, NaN
            assert c8[0, 0, 0, off:off + 7].view(torch.uint8).tolist() == [0x7E, 0x7E, 0x7F, 0xFF, 0x7F, 0xFF, 0x7F]
    else:
        # the planted values went through unrotated, and true division (float64 quotient of the fp32 operands, rounded once
        # to fp32) would have written other bytes
        x = special.to(torch.bfloat16).double()
        s32 = float(torch.tensor(scale, dtype=torch.float32))
        true_div = (x / s32).float().to(E4M3).view(torch.uint8).tolist()
        for c8, cb, off in ((k8, kb, 0), (v8, vb, 7)):
            assert torch.equal(cb[0, 0, 0, off:off + 2].cpu().double(), x)
            got = c8[0, 0, 0, off:off + 2].view(torch.uint8).tolist()
            assert got == mgr._q(cb[0, 0, 0, off:off + 2]).view(torch.uint8).tolist(), got
            assert all(a != t for a, t in zip(got, true_div)), (got, true_div)


# ---- a Mistral-shaped model on an fp8 cache ---------------------------------------------------------------------------
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


def test_mistral_shaped_fp8_cache_graph_torch_path_and_bf16_cache(_ext, monkeypatch):
    """GQA with a window (64) shorter than prompt + generation, KV cache in e4m3 at scale 0.3:
    - the CUDA-graph replay of a decode step gives the eager logits bit for bit;
    - attention forced through fp32 torch math on the same quantised cache agrees (rel. error < 5e-2, confident tokens);
    - the bf16-cache model agrees within a bound set by e4m3's relative step (below)."""
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.ops import attention
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    _one_rank_model_parallel()
    W, P, N = 64, 160, 24
    torch.manual_seed(0)
    m = LlamaForInference(_mistral_cfg(sliding_window=W), batch_size=2, max_seq_len=512, on_device_sampling=False,
                          kv_quant=KVQuantizationConfig(scale=0.3)).eval()
    assert m.kv.k[0].dtype == E4M3 and m.kv.kernel_scales() == (0.3, 0.3)
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

    # every decode step appends with the fused kernel and attends with the decode kernel, both on the e4m3 cache
    e, calls = _ext.ext(), []
    for name in ("decode_rope_kv", "decode_attention"):
        fn = getattr(e, name)
        monkeypatch.setattr(e, name, lambda *a, _fn=fn, _n=name, **kw: calls.append((_n, a[6 if _n == "decode_rope_kv" else 1].dtype,
                                                                                     kw.get("k_scale"))) or _fn(*a, **kw))
    eager_toks, eager_logits = run(m.token_generation)
    monkeypatch.undo()
    assert sorted(set(calls)) == [("decode_attention", E4M3, 0.3), ("decode_rope_kv", E4M3, 0.3)]
    assert len(calls) == 2 * N * 2

    st_tok, st_pos = eager_toks[:, 0].view(2, 1).clone(), last + 1
    m.context_encoding(ids, last)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.token_generation(st_tok, st_pos)
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

    def teacher_forced(model):
        out = [model.context_encoding(ids, last)]
        pos = last + 1
        for i in range(N):
            out.append(model.token_generation(eager_toks[:, i].view(2, 1), pos).clone())
            pos = pos + 1
        return out

    # fp32 torch attention over the same quantised cache (prefill through SDPA, decode through the de-quantising fallback)
    with monkeypatch.context() as mp:
        mp.setenv("NXD_DISABLE_OWN_ATTENTION", "1")
        orig = attention.decode_attention
        mp.setattr(attention, "decode_attention",
                   lambda q, k, v, p, sliding_window, k_scale=1.0, v_scale=1.0: orig(
                       q.float(), k, v, p, sliding_window=sliding_window, k_scale=k_scale, v_scale=v_scale).to(q.dtype))
        ref_logits = teacher_forced(m)
    for i, (a, r) in enumerate(zip(eager_logits, ref_logits)):
        assert _rel(a.float(), r.double()) < 5e-2, (i, _rel(a.float(), r.double()))
        top2 = r.float().topk(2, -1).values
        sure = (top2[:, 0] - top2[:, 1]) > 0.05 * r.float().std()
        assert torch.equal(a.argmax(-1)[sure], r.argmax(-1)[sure]), i

    # bf16 cache, same weights.  Every cached element is within e4m3's relative step 2⁻⁴ of its bf16 value.  The attention
    # output is a convex combination of V rows (one 2⁻⁴), and the K error moves the softmax weights by at most as much
    # again at these logit scales (a second 2⁻⁴); nothing downstream amplifies a relative error of the residual stream.
    # Bound: 2 · 2⁻⁴ = 0.125 on the relative logit error.
    bound = 2 * 2 ** -4
    torch.manual_seed(0)
    m16 = LlamaForInference(_mistral_cfg(sliding_window=W), batch_size=2, max_seq_len=512, on_device_sampling=False).eval()
    m16.load_state_dict(m.state_dict())
    bf16_logits = teacher_forced(m16)
    for i, (a, r) in enumerate(zip(eager_logits, bf16_logits)):
        assert _rel(a.float(), r.double()) < bound, (i, _rel(a.float(), r.double()))
