"""Token generation at head_dim 64, 80 and 96 on the H100 (sm_90a): the decode kernel (``csrc/decode.cu``), flash-decoding's
local partial, the verification kernel (``csrc/attention_sm90.cu`` ``spec_attn_kernel``) and the rolling-cache variants of
both, against float64 attention on the de-quantised cache; the extension's head-size check; and ``LlamaForInference`` at
D = 64 / 80 / 96 generating on the kernels (eager, CUDA graph, speculation chain, Medusa tree) against the torch path."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_speculation_attention_cpu import medusa_tree, random_tree, visible  # noqa: E402

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
DIMS = (64, 80, 96)


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _rel(a, b):
    return ((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _vis(pos, W, L, mask, depth, sw):
    """[B, W, L] bool on the GPU, built row by row from the rule."""
    return torch.stack([torch.stack([visible(int(p), w, W, L, mask, depth, sw) for w in range(W)]) for p in pos.tolist()]).cuda()


def _ref64(q, kd, vd, vis):
    """float64 attention of q [B,W,H,D] over de-quantised caches [B,L,Hkv,D] under ``vis`` [B,W,L]; 0 where nothing is seen."""
    B, W, H, D = q.shape
    G = H // kd.shape[2]
    kk, vv = kd.repeat_interleave(G, 2), vd.repeat_interleave(G, 2)
    s = torch.einsum("bwhd,blhd->bwhl", q.double(), kk) / math.sqrt(D)
    s = s.masked_fill(~vis[:, :, None], float("-inf"))
    p = torch.nan_to_num(s.softmax(-1), nan=0.0)
    return torch.einsum("bwhl,blhd->bwhd", p, vv)


def _caches(B, L, Hkv, D, dtype, g, ks=1.0, vs=1.0):
    """Strided caches: [L, B, Hkv, D] memory for k, and the first half of a [B, L, Hkv, 2D] buffer for v."""
    k = (torch.randn(L, B, Hkv, D, device="cuda", generator=g) / ks).to(dtype).transpose(0, 1)
    v = (torch.randn(B, L, Hkv, 2 * D, device="cuda", generator=g) / vs).to(dtype)[..., :D]
    return k, v


def _nan_(t, rows):
    """NaN bytes into ``t[rows]`` (bf16 or e4m3)."""
    if t.dtype == E4M3:
        t.view(torch.uint8)[rows] = 0x7F
    else:
        t.view(torch.int16)[rows] = 0x7FC0


def _scales(cache):
    return ((0.3, 0.7), {"k_scale": 0.3, "v_scale": 0.7}) if cache == "e4m3" else ((1.0, 1.0), {})


# ---- one-token decode ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("sw", (None, 300))
@pytest.mark.parametrize("G", (1, 2, 4, 8))
@pytest.mark.parametrize("D", DIMS)
def test_decode_vs_float64_and_unread_rows(_ext, D, G, sw, cache):
    """``decode_attention`` on the kernel against float64; NaN bytes in every row the token cannot see leave the output
    bit-identical.  Positions: 0, inside the cache, one where the window starts past row 0, and L − 1."""
    from neuronx_distributed_b200.ops import attention

    L, H = 1024, 8
    pos = torch.tensor([0, 150, 700, L - 1], device="cuda")
    B, Hkv = pos.numel(), H // G
    (ks, vs), kw = _scales(cache)
    g = torch.Generator(device="cuda").manual_seed(1000 * D + 10 * G + (sw or 0))
    q = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = _caches(B, L, Hkv, D, E4M3 if cache == "e4m3" else torch.bfloat16, g, ks, vs)
    n0 = _ext.launches()
    got = attention.decode_attention(q, kc, vc, pos, sliding_window=sw, **kw)
    assert _ext.launches() == n0 + 2                                          # the kernel and the combine ran
    vis = _vis(pos, 1, L, None, None, sw)
    ref = _ref64(q, kc.double() * ks, vc.double() * vs, vis)
    assert got.shape == (B, 1, H, D) and got.dtype == torch.bfloat16
    assert _rel(got, ref) < 2e-2, _rel(got, ref)
    kn, vn = kc.clone(), vc.clone()
    for t in (kn, vn):
        _nan_(t, ~vis[:, 0])
    got_nan = attention.decode_attention(q, kn, vn, pos, sliding_window=sw, **kw)
    assert torch.isfinite(got_nan).all() and torch.equal(got_nan, got)


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("G", (1, 4, 8))
@pytest.mark.parametrize("D", DIMS)
def test_decode_partial_matches_torch(_ext, D, G, cache):
    """Flash-decoding's local partial on the kernel vs its torch path, local positions before, inside and past the shard."""
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial

    W, L, H = 100, 512, 8
    (ks, vs), kw = _scales(cache)
    local = torch.tensor([-40, -1, 0, 63, 99, 100, 400, 511, 530, 700], device="cuda")
    B, Hkv = local.numel(), H // G
    g = torch.Generator(device="cuda").manual_seed(7 + G + D)
    q = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = _caches(B, L, Hkv, D, E4M3 if cache == "e4m3" else torch.bfloat16, g, ks, vs)
    for window in (None, W):
        n0 = _ext.launches()
        o, m, l = _local_partial(q, kc, vc, local, 1.0 / math.sqrt(D), window, ks, vs)
        assert _ext.launches() == n0 + 2
        assert o.shape == (B, H, D)
        ro, rm, rl = _local_partial(q.cpu(), kc.cpu(), vc.cpu(), local.cpu(), 1.0 / math.sqrt(D), window, ks, vs)
        ro, rm, rl = ro.cuda(), rm.cuda(), rl.cuda()
        none = torch.isinf(rm)
        assert torch.equal(torch.isinf(m), none) and bool(none[0].all()) and bool(none[1].all())
        assert not o[none].any() and not l[none].any()
        assert (m[~none] - rm[~none]).abs().max().item() < 1e-3
        assert _rel(l[~none], rl[~none].double()) < 1e-2 and _rel(o[~none], ro[~none].double()) < 1e-2


# ---- verification windows --------------------------------------------------------------------------------------------------
def _window(kind, W):
    if kind == "chain":
        return None, None
    mask, depth = medusa_tree() if kind == "medusa" else random_tree(W, W)
    return mask.cuda(), depth.cuda()


WINDOWS = (("chain", 5), ("chain", 64), ("medusa", 10), ("random", 64))


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("sw", (None, 300))
@pytest.mark.parametrize("kind,W", WINDOWS)
@pytest.mark.parametrize("G", (1, 4, 8))
@pytest.mark.parametrize("D", DIMS)
def test_speculation_vs_float64(_ext, D, G, kind, W, sw, cache):
    from neuronx_distributed_b200.ops import attention

    L, H = 1024, 8
    pos = torch.tensor([0, 150, 299, 700, L - W], device="cuda")            # 0, inside and past the window, p + W = L
    B, Hkv = pos.numel(), H // G
    (ks, vs), kw = _scales(cache)
    g = torch.Generator(device="cuda").manual_seed(1000 * D + 100 * G + W)
    q = torch.randn(B, W, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = _caches(B, L, Hkv, D, E4M3 if cache == "e4m3" else torch.bfloat16, g, ks, vs)
    mask, depth = _window(kind, W)
    n0 = _ext.launches()
    got = attention.speculation_attention(q, kc, vc, pos, mask, depth, sliding_window=sw, **kw)
    assert _ext.launches() == n0 + 2
    ref = _ref64(q, kc.double() * ks, vc.double() * vs, _vis(pos, W, L, mask, depth, sw))
    assert got.shape == (B, W, H, D) and got.dtype == torch.bfloat16
    assert _rel(got, ref) < 2e-2, _rel(got, ref)


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("sw", (None, 300))
@pytest.mark.parametrize("G", (1, 4))
@pytest.mark.parametrize("D", DIMS)
def test_speculation_unseen_nan_slots_do_not_reach_output(_ext, D, G, sw, cache):
    """NaN bytes in every slot no token sees, including a window column the tree hides from every node (its V row is
    zeroed in shared memory), leave the output finite and bit-identical."""
    from neuronx_distributed_b200.ops import attention

    L, H, W = 1024, 8, 10
    pos = torch.tensor([0, 150, 700, L - W], device="cuda")
    B, Hkv = pos.numel(), H // G
    (ks, vs), kw = _scales(cache)
    g = torch.Generator(device="cuda").manual_seed(G + D)
    q = torch.randn(B, W, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = _caches(B, L, Hkv, D, E4M3 if cache == "e4m3" else torch.bfloat16, g, ks, vs)
    mask, depth = medusa_tree("cuda")
    mask = mask.clone()
    mask[:, 4] = False                                                       # window column 4: seen by no node
    got = attention.speculation_attention(q, kc, vc, pos, mask, depth, sliding_window=sw, **kw)
    unseen = ~_vis(pos, W, L, mask, depth, sw).any(1)                        # [B, L]
    assert bool(unseen[torch.arange(B, device="cuda"), pos + 4].all())
    kn, vn = kc.clone(), vc.clone()
    for t in (kn, vn):
        _nan_(t, unseen)
    n0 = _ext.launches()
    got_nan = attention.speculation_attention(q, kn, vn, pos, mask, depth, sliding_window=sw, **kw)
    assert _ext.launches() == n0 + 2
    assert torch.isfinite(got_nan).all() and torch.equal(got_nan, got)


# ---- rolling cache ---------------------------------------------------------------------------------------------------------
SW = 300
R = SW + 64


def _ring(hist, pos, W):
    """Ring [B, R, Hkv, D] of the linear history [B, T, Hkv, D] after positions < pos[b] + W were written; rows no token at
    pos can see hold NaN."""
    B = hist.shape[0]
    j = torch.arange(R, device=hist.device)[None, :]
    end = (pos + W)[:, None]
    t = end - 1 - (end - 1 - j) % R                                          # newest position of row j
    ring = hist.gather(1, t.clamp(min=0)[:, :, None, None].expand(B, R, *hist.shape[2:])).clone()
    _nan_(ring, (t < 0) | (t <= pos[:, None] - SW))
    return ring


def _history(B, T, Hkv, D, cache, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    k, v = (torch.randn(B, T, Hkv, D, device="cuda", generator=g) for _ in range(2))
    if cache == "e4m3":
        return (k / 0.3).to(E4M3), (v / 0.7).to(E4M3), {"k_scale": 0.3, "v_scale": 0.7}
    return k.bfloat16(), v.bfloat16(), {}


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("G", (1, 4))
@pytest.mark.parametrize("D", DIMS)
def test_ring_equals_linear(_ext, D, G, cache):
    """Decode and verification (chain, Medusa tree, random 64-node tree) on a ring give bit for bit what the linear kernels
    give on the same history."""
    from neuronx_distributed_b200.ops import attention

    H = 8
    pos = torch.tensor([5, SW + 7, R - 1, R, 3 * R + 17, 11 * R + 250], device="cuda")
    B, T = pos.numel(), int(pos.max()) + 64
    kc, vc, kw = _history(B, T, H // G, D, cache, D + G)
    g = torch.Generator(device="cuda").manual_seed(9)
    q = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    want = attention.decode_attention(q, kc, vc, pos, sliding_window=SW, **kw)
    n0 = _ext.launches()
    got = attention.decode_attention(q, _ring(kc, pos, 1), _ring(vc, pos, 1), pos, sliding_window=SW, rolling=True, **kw)
    assert _ext.launches() == n0 + 2
    assert torch.isfinite(got).all() and torch.equal(got, want)
    for kind, W in (("chain", 5), ("medusa", 10), ("random", 64)):
        mask, depth = (None, None) if kind == "chain" else (medusa_tree("cuda") if kind == "medusa" else random_tree(W, 5, "cuda"))
        q = torch.randn(B, W, H, D, device="cuda", generator=g).bfloat16()
        want = attention.speculation_attention(q, kc, vc, pos, mask, depth, SW, **kw)
        n0 = _ext.launches()
        got = attention.speculation_attention(q, _ring(kc, pos, W), _ring(vc, pos, W), pos, mask, depth, SW, rolling=True, **kw)
        assert _ext.launches() == n0 + 2
        assert torch.isfinite(got).all() and torch.equal(got, want), kind


# ---- head sizes the kernels do not take --------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", (32, 256))
def test_other_head_dims_raise_in_extension_and_run_on_torch(_ext, D):
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial
    from neuronx_distributed_b200.ops import attention

    e = _ext.ext()
    L, H, Hkv, W = 256, 8, 2, 5
    pos = torch.tensor([0, 100, L - W], device="cuda")
    B = pos.numel()
    g = torch.Generator(device="cuda").manual_seed(D)
    q1 = torch.randn(B, 1, H, D, device="cuda", generator=g).bfloat16()
    qw = torch.randn(B, W, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = _caches(B, L, Hkv, D, torch.bfloat16, g)
    with pytest.raises(RuntimeError, match="D in \\{64, 80, 96, 128\\}"):
        e.decode_attention(q1, kc, vc, pos, 1.0 / math.sqrt(D))
    with pytest.raises(RuntimeError, match="D in \\{64, 80, 96, 128\\}"):
        e.decode_attention_partial(q1, kc, vc, pos, 1.0 / math.sqrt(D))
    with pytest.raises(RuntimeError, match="D in \\{64, 80, 96, 128\\}"):
        e.speculation_attention(qw, kc, vc, pos, scale=1.0 / math.sqrt(D))
    n0 = _ext.launches()
    got1 = attention.decode_attention(q1, kc, vc, pos)
    gotw = attention.speculation_attention(qw, kc, vc, pos)
    o, m, l = _local_partial(q1, kc, vc, pos, 1.0 / math.sqrt(D))
    assert _ext.launches() == n0                                              # all three took the torch path
    kd, vd = kc.double(), vc.double()
    assert _rel(got1, _ref64(q1, kd, vd, _vis(pos, 1, L, None, None, None))) < 2e-2
    assert _rel(gotw, _ref64(qw, kd, vd, _vis(pos, W, L, None, None, None))) < 2e-2
    ref1 = _ref64(q1, kd, vd, _vis(pos, 1, L, None, None, None))[:, 0]
    assert _rel(o / l[..., None], ref1) < 2e-2


# ---- the model -------------------------------------------------------------------------------------------------------------
def _model(D, G, kv_fp8):
    from test_kv_fp8_gpu import _one_rank_model_parallel

    from neuronx_distributed_b200.models.llama import LlamaConfig
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    _one_rank_model_parallel()
    H = 8
    cfg = LlamaConfig(vocab_size=1024, hidden_size=H * D, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=H,
                      num_key_value_heads=H // G, max_position_embeddings=512, dtype=torch.bfloat16,
                      device=torch.device("cuda", 0))
    torch.manual_seed(0)
    return LlamaForInference(cfg, batch_size=2, max_seq_len=512, on_device_sampling=False,
                             kv_quant=KVQuantizationConfig(scale=0.3) if kv_fp8 else None).eval()


def _close(a, r, what):
    a, r = a.float(), r.float()
    assert _rel(a, r.double()) < 5e-2, (what, _rel(a, r.double()))
    top2 = r.topk(2, -1).values
    sure = (top2[..., 0] - top2[..., 1]) > 0.05 * r.std()
    assert torch.equal(a.argmax(-1)[sure], r.argmax(-1)[sure]), what


@pytest.mark.parametrize("kv_fp8", (False, True))
@pytest.mark.parametrize("D,G", ((64, 4), (80, 2), (96, 1)))
def test_model_generates_on_the_kernels(_ext, monkeypatch, D, G, kv_fp8):
    """``LlamaForInference`` at D = 64 / 80 / 96: decode steps on the kernel, a CUDA-graph replay equal to eager, logits close
    to fp32 torch attention, a speculation chain equal to step-by-step decode, a Medusa tree close to the torch path."""
    from neuronx_distributed_b200.ops import attention

    m = _model(D, G, kv_fp8)
    P, N = 160, 8
    ids = torch.randint(0, 1024, (2, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    last = torch.tensor([P - 1, 120], device="cuda")

    def run(step, toks=None):
        logits = [m.context_encoding(ids, last)]
        out, pos = [logits[0].argmax(-1)], last + 1
        for i in range(N):
            tok = out[-1] if toks is None else toks[:, i]
            logits.append(step(tok.view(2, 1), pos).clone())
            out.append(logits[-1].argmax(-1))
            pos = pos + 1
        return torch.stack(out, 1), logits

    e, calls = _ext.ext(), []
    fn = e.decode_attention
    monkeypatch.setattr(e, "decode_attention", lambda *a, **kw: calls.append((a[0].shape[-1], a[1].dtype)) or fn(*a, **kw))
    eager_toks, eager_logits = run(m.token_generation)
    monkeypatch.undo()
    assert calls == [(D, E4M3 if kv_fp8 else torch.bfloat16)] * (2 * N)      # every layer of every step on the kernel

    # CUDA-graph replay of a decode step: the eager logits bit for bit
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

    # fp32 torch attention over the same cache (prefill through SDPA, decode through the torch path; an e4m3 cache is
    # de-quantised to q's dtype there, a bf16 one is widened here)
    def fp32(t):
        return t.float() if t.dtype == torch.bfloat16 else t

    with monkeypatch.context() as mp:
        mp.setenv("NXD_DISABLE_OWN_ATTENTION", "1")
        orig = attention.decode_attention
        mp.setattr(attention, "decode_attention",
                   lambda q, k, v, p, sliding_window, k_scale=1.0, v_scale=1.0: orig(
                       q.float(), fp32(k), fp32(v), p, sliding_window=sliding_window, k_scale=k_scale,
                       v_scale=v_scale).to(q.dtype))
        _, ref_logits = run(m.token_generation, eager_toks)
    for i, (a, r) in enumerate(zip(eager_logits, ref_logits)):
        _close(a, r, f"step {i}")

    # a speculation chain on the kernel verifies what step-by-step decode computes
    pos = last + 1
    window = eager_toks[:, :5]
    e, spec_calls = _ext.ext(), []
    fn = e.speculation_attention
    monkeypatch.setattr(e, "speculation_attention", lambda *a, **kw: spec_calls.append(a[0].shape[-1]) or fn(*a, **kw))
    m.context_encoding(ids, last)
    spec = m.speculation_forward(window, pos).clone()
    monkeypatch.undo()
    assert spec_calls == [D] * 2
    steps = torch.stack(eager_logits[1:6], 1)
    _close(spec, steps, "chain")

    # a Medusa tree on the kernel vs the forced torch path (no kernel scales: RoPE, append and attention in torch)
    mask, depth = medusa_tree("cuda")
    tree_ids = torch.randint(0, 1024, (2, depth.numel()), device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    m.context_encoding(ids, last)
    tree = m.speculation_forward(tree_ids, pos, tree_mask=mask, tree_depth=depth).clone()
    with monkeypatch.context() as mp:
        mp.setattr(m.kv, "kernel_scales", lambda: None)
        m.context_encoding(ids, last)
        tree_ref = m.speculation_forward(tree_ids, pos, tree_mask=mask, tree_depth=depth).clone()
    _close(tree, tree_ref, "tree")
