"""Verification of W new tokens per sequence on the H100 (sm_90a): the ``spec_attn`` kernel of ``csrc/attention_sm90.cu``
against float64 attention on the de-quantised cache, the W-token RoPE + cache append of ``decode_rope_kv``, and a
Mistral-shaped model verifying speculation chains and Medusa trees on bf16 and e4m3 caches."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_speculation_attention_cpu import medusa_tree, random_tree, visible  # noqa: E402

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn


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


def _tree(kind, W):
    if kind == "chain":
        return None, None
    mask, depth = medusa_tree() if W == 10 else random_tree(W, W)
    return mask.cuda(), depth.cuda()


def _caches(B, L, Hkv, D, dtype, g, ks=1.0, vs=1.0):
    """Strided caches: [L, B, Hkv, D] memory for k, and the first half of a [B, L, Hkv, 2D] buffer for v."""
    k = (torch.randn(L, B, Hkv, D, device="cuda", generator=g) / ks).to(dtype).transpose(0, 1)
    v = (torch.randn(B, L, Hkv, 2 * D, device="cuda", generator=g) / vs).to(dtype)[..., :D]
    return k, v


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("sw", (None, 300))
@pytest.mark.parametrize("kind", ("chain", "tree"))
@pytest.mark.parametrize("W", (2, 5, 10, 64))
@pytest.mark.parametrize("G", (1, 2, 4, 8))
def test_kernel_vs_float64(_ext, G, W, kind, sw, cache):
    from neuronx_distributed_b200.ops import attention

    L, H, D = 1024, 8, 128
    pos = torch.tensor([0, 150, 299, 700, L - W], device="cuda")            # 0, inside and past the window, p + W = L
    B, Hkv = pos.numel(), H // G
    ks, vs = (0.3, 0.7) if cache == "e4m3" else (1.0, 1.0)
    g = torch.Generator(device="cuda").manual_seed(100 * G + W)
    q = torch.randn(B, W, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = _caches(B, L, Hkv, D, E4M3 if cache == "e4m3" else torch.bfloat16, g, ks, vs)
    mask, depth = _tree(kind, W)
    kw = {"k_scale": ks, "v_scale": vs} if cache == "e4m3" else {}
    n0 = _ext.launches()
    got = attention.speculation_attention(q, kc, vc, pos, mask, depth, sliding_window=sw, **kw)
    assert _ext.launches() == n0 + 2                                          # the kernel and the combine ran
    vis = _vis(pos, W, L, mask, depth, sw)
    ref = _ref64(q, kc.double() * ks, vc.double() * vs, vis)
    assert got.shape == (B, W, H, D) and got.dtype == torch.bfloat16
    assert _rel(got, ref) < 2e-2, _rel(got, ref)


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("sw", (None, 300))
@pytest.mark.parametrize("G", (1, 4))
def test_unseen_nan_slots_do_not_reach_output(_ext, G, sw, cache):
    """NaN bytes in every slot no token of the sequence sees (past the window, before the sliding window, and window
    columns the tree hides from every node) leave the output finite and bit-identical."""
    from neuronx_distributed_b200.ops import attention

    L, H, D, W = 1024, 8, 128, 10
    pos = torch.tensor([0, 150, 700, L - W], device="cuda")
    B, Hkv = pos.numel(), H // G
    dt = E4M3 if cache == "e4m3" else torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(G)
    q = torch.randn(B, W, H, D, device="cuda", generator=g).bfloat16()
    kc, vc = _caches(B, L, Hkv, D, dt, g)
    mask, depth = medusa_tree("cuda")
    mask = mask.clone()
    mask[:, 4] = False                                                       # window column 4: seen by no node
    got = attention.speculation_attention(q, kc, vc, pos, mask, depth, sliding_window=sw)
    unseen = ~_vis(pos, W, L, mask, depth, sw).any(1)                        # [B, L]
    assert bool(unseen[torch.arange(B, device="cuda"), pos + 4].all())
    kn, vn = kc.clone(), vc.clone()
    for t in (kn, vn):
        if dt == E4M3:
            t.view(torch.uint8)[unseen] = 0x7F
        else:
            t.view(torch.int16)[unseen] = 0x7FC0
    got_nan = attention.speculation_attention(q, kn, vn, pos, mask, depth, sliding_window=sw)
    assert torch.isfinite(got_nan).all() and torch.equal(got_nan, got)


# ---- W-token RoPE + cache append -----------------------------------------------------------------------------------------
def _append_inputs(B, W, H, Hkv, D, L, seed):
    from neuronx_distributed_b200.ops import rope

    g = torch.Generator(device="cuda").manual_seed(seed)
    f = torch.randn(B, W, (H + 2 * Hkv) * D, device="cuda", generator=g).bfloat16() * 3     # a fused QKV projection output
    q = f[..., :H * D].view(B, W, H, D)
    k = f[..., H * D:(H + Hkv) * D].view(B, W, Hkv, D)
    v = f[..., (H + Hkv) * D:].view(B, W, Hkv, D)
    cos, sin = rope.rope_tables(L, D, 10000.0, torch.device("cuda"), 0, 1.0)
    return q, k, v, cos, sin


def _ulp(x):
    """bf16 ulp of each element (of the smallest normal for zeros)."""
    a = x.float().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def test_append_chain_equals_one_token_calls(_ext):
    e = _ext.ext()
    B, W, H, Hkv, D, L = 3, 6, 8, 2, 128, 64
    q, k, v, cos, sin = _append_inputs(B, W, H, Hkv, D, L, 1)
    pos = torch.tensor([0, 5, L - W], device="cuda")
    kc, vc = (torch.zeros(B, L, Hkv, D, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    k1, v1 = kc.clone(), vc.clone()
    qw = e.decode_rope_kv(q, k, v, pos, cos, sin, kc, vc)
    q1 = torch.cat([e.decode_rope_kv(q[:, w:w + 1], k[:, w:w + 1], v[:, w:w + 1], pos + w, cos, sin, k1, v1) for w in range(W)], 1)
    assert torch.equal(qw, q1) and torch.equal(kc, k1) and torch.equal(vc, v1)
    written = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    written[torch.arange(B, device="cuda")[:, None], pos[:, None] + torch.arange(W, device="cuda")] = True
    assert not kc[~written].any() and not vc[~written].any()                 # no other slot was written


@pytest.mark.parametrize("scale", (1.0, 0.3))
def test_append_tree_matches_torch_path_and_e4m3_rule(_ext, scale):
    """Tree depths: token w is rotated at p + depth[w] and written to slot p + w.  Slots as the torch path writes them,
    rows within one bf16 ulp of its fp32 rotation, and the e4m3 bytes are ``KVCacheManager._q`` of the bf16 rows."""
    from neuronx_distributed_b200.inference.kv_cache import KVCacheManager
    from neuronx_distributed_b200.ops.rope import rotate
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    e = _ext.ext()
    B, H, Hkv, D, L = 2, 8, 2, 128, 64
    _, depth = medusa_tree("cuda")
    W = depth.numel()
    q, k, v, cos, sin = _append_inputs(B, W, H, Hkv, D, L, 2)
    pos = torch.tensor([3, L - W], device="cuda")
    kb, vb = (torch.zeros(B, L, Hkv, D, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    k8, v8 = (torch.zeros(B, L, Hkv, D, device="cuda", dtype=E4M3) for _ in range(2))
    qb = e.decode_rope_kv(q, k, v, pos, cos, sin, kb, vb, depth=depth)
    q8 = e.decode_rope_kv(q, k, v, pos, cos, sin, k8, v8, k_scale=scale, v_scale=scale, depth=depth)
    assert torch.equal(qb, q8)
    idx = pos[:, None] + depth[None, :]
    qt, kt = rotate(q, cos[idx], sin[idx]), rotate(k, cos[idx], sin[idx])
    slots = pos[:, None] + torch.arange(W, device="cuda")
    b = torch.arange(B, device="cuda")[:, None]
    assert ((qb.float() - qt.float()).abs() <= _ulp(qt)).all()
    assert ((kb[b, slots].float() - kt.float()).abs() <= _ulp(kt)).all()
    assert torch.equal(vb[b, slots], v)
    rest = torch.ones(B, L, dtype=torch.bool, device="cuda")
    rest[b, slots] = False
    assert not kb[rest].any() and not vb[rest].any() and not k8.view(torch.uint8)[rest].any() and not v8.view(torch.uint8)[rest].any()
    mgr = KVCacheManager(1, 1, 1, 1, 1, device="cuda", kv_quant=KVQuantizationConfig(scale=scale))
    assert torch.equal(k8.view(torch.uint8), mgr._q(kb).view(torch.uint8))
    assert torch.equal(v8.view(torch.uint8), mgr._q(vb).view(torch.uint8))


# ---- a Mistral-shaped model verifying windows -----------------------------------------------------------------------------
def _model(kv_fp8):
    from test_kv_fp8_gpu import _mistral_cfg, _one_rank_model_parallel

    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    _one_rank_model_parallel()
    torch.manual_seed(0)
    return LlamaForInference(_mistral_cfg(sliding_window=64), batch_size=2, max_seq_len=512, on_device_sampling=False,
                             kv_quant=KVQuantizationConfig(scale=0.3) if kv_fp8 else None).eval()


def _close(a, r, what):
    a, r = a.float(), r.float()
    assert _rel(a, r.double()) < 5e-2, (what, _rel(a, r.double()))
    top2 = r.topk(2, -1).values
    sure = (top2[..., 0] - top2[..., 1]) > 0.05 * r.std()
    assert torch.equal(a.argmax(-1)[sure], r.argmax(-1)[sure]), what


@pytest.mark.parametrize("kv_fp8", (False, True))
def test_mistral_speculation_chain_tree_and_graph(_ext, monkeypatch, kv_fp8):
    m = _model(kv_fp8)
    P = 160
    ids = torch.randint(0, 1024, (2, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    last = torch.tensor([P - 1, 120], device="cuda")
    pos = last + 1
    window = torch.randint(0, 1024, (2, 5), device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))

    e, calls = _ext.ext(), []
    fn = e.speculation_attention
    monkeypatch.setattr(e, "speculation_attention", lambda *a, **kw: calls.append(a[1].dtype) or fn(*a, **kw))
    monkeypatch.setattr(m.kv, "get", lambda *a, **kw: pytest.fail("kv.get called on the kernel path"))
    m.context_encoding(ids, last)
    spec = m.speculation_forward(window, pos).clone()                        # [2, 5, V]
    monkeypatch.undo()
    assert calls == [E4M3 if kv_fp8 else torch.bfloat16] * 2                  # one call per layer, on the cache as stored

    # a chain verifies exactly what 5 token-generation steps compute
    m.context_encoding(ids, last)
    steps = [m.token_generation(window[:, i:i + 1], pos + i).clone() for i in range(5)]
    _close(spec, torch.stack(steps, 1), "chain")

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

    # CUDA-graph replay of the tree verification gives the eager logits bit for bit
    st_ids, st_pos = tree_ids.clone(), pos.clone()
    m.context_encoding(ids, last)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.speculation_forward(st_ids, st_pos, tree_mask=mask, tree_depth=depth)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_out = m.speculation_forward(st_ids, st_pos, tree_mask=mask, tree_depth=depth)
    m.context_encoding(ids, last)
    graph.replay()
    assert torch.equal(st_out, tree)


def test_speculative_and_medusa_generate_on_gpu(_ext):
    from test_kv_fp8_gpu import _one_rank_model_parallel

    from neuronx_distributed_b200.models.llama import LlamaConfig
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.utils.medusa import MedusaHeads, medusa_generate
    from neuronx_distributed_b200.utils.speculative import speculative_generate
    from test_speculation_attention_cpu import MEDUSA_CHOICES

    _one_rank_model_parallel()
    N, L = 24, 96

    def cfg(layers):
        return LlamaConfig(vocab_size=4096, hidden_size=256, intermediate_size=704, num_hidden_layers=layers,
                           num_attention_heads=8, dtype=torch.bfloat16, device=torch.device("cuda", 0), max_position_embeddings=L)

    torch.manual_seed(0)
    target = LlamaForInference(cfg(4), batch_size=1, max_seq_len=L).eval()
    torch.manual_seed(0)
    draft = LlamaForInference(cfg(1), batch_size=1, max_seq_len=L).eval()
    prompt = torch.randint(0, 4096, (1, 32), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    n0 = _ext.launches()
    out, _ = speculative_generate(target, draft, prompt, N, 4)
    assert out.shape == (1, N) and _ext.launches() > n0
    target.kv.reset()
    heads = MedusaHeads(256, 4096, 3, dtype=torch.bfloat16, device="cuda").eval()
    for proj in heads.proj:
        proj.weight.data.copy_(target.lm.lm_head.weight.data)
    out, _ = medusa_generate(target, heads, prompt, N, MEDUSA_CHOICES, topk=10)
    assert out.shape == (1, N)
