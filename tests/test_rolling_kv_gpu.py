"""Rolling KV cache on the H100 (sm_90a): the decode, verification and RoPE + append kernels read and write a ring of
R = SW + 64 rows and give bit for bit what they give on a linear cache holding the same history, and a Mistral-shaped
model serving from a ring (prefill, decode across several wraps, CUDA-graph replay, a speculation chain and a Medusa tree
with compaction) computes the linear model's logits exactly, on bf16 and e4m3 caches."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_speculation_attention_cpu import medusa_tree, random_tree  # noqa: E402

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
SW = 300
R = SW + 64


@pytest.fixture(scope="module")
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _nan_(t, rows):
    """NaN bytes into ``t[rows]`` (bf16 or e4m3)."""
    if t.dtype == E4M3:
        t.view(torch.uint8)[rows] = 0x7F
    else:
        t.view(torch.int16)[rows] = 0x7FC0


def _ring(hist, pos, W):
    """Ring [B, R, Hkv, D] of the linear history [B, T, Hkv, D] after positions < pos[b] + W were written.  Rows whose
    position no token at pos can see (before pos − SW, or never written) hold NaN."""
    B = hist.shape[0]
    j = torch.arange(R, device=hist.device)[None, :]
    end = (pos + W)[:, None]
    t = end - 1 - (end - 1 - j) % R                                          # newest position of row j
    ring = hist.gather(1, t.clamp(min=0)[:, :, None, None].expand(B, R, *hist.shape[2:])).clone()
    _nan_(ring, (t < 0) | (t <= pos[:, None] - SW))
    return ring


def _history(B, T, Hkv, cache, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    k, v = (torch.randn(B, T, Hkv, 128, device="cuda", generator=g) for _ in range(2))
    if cache == "e4m3":
        return (k / 0.3).to(E4M3), (v / 0.7).to(E4M3), {"k_scale": 0.3, "v_scale": 0.7}
    return k.bfloat16(), v.bfloat16(), {}


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("G", (1, 2, 4, 8))
def test_decode_ring_equals_linear(_ext, G, cache):
    from neuronx_distributed_b200.ops import attention

    H = 8
    pos = torch.tensor([5, SW + 7, R - 1, R, 3 * R + 17, 11 * R + 250], device="cuda")
    B, T = pos.numel(), int(pos.max()) + 1
    kc, vc, kw = _history(B, T, H // G, cache, G)
    q = torch.randn(B, 1, H, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9)).bfloat16()
    kr, vr = _ring(kc, pos, 1), _ring(vc, pos, 1)
    want = attention.decode_attention(q, kc, vc, pos, sliding_window=SW, **kw)
    n0 = _ext.launches()
    got = attention.decode_attention(q, kr, vr, pos, sliding_window=SW, rolling=True, **kw)
    assert _ext.launches() == n0 + 2
    assert torch.isfinite(got).all() and torch.equal(got, want)


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("kind,W", (("chain", 5), ("chain", 64), ("medusa", 10), ("random", 64)))
@pytest.mark.parametrize("G", (1, 4, 8))
def test_verification_ring_equals_linear(_ext, G, kind, W, cache):
    from neuronx_distributed_b200.ops import attention

    H = 8
    mask, depth = (None, None) if kind == "chain" else (medusa_tree("cuda") if kind == "medusa" else random_tree(W, 5, "cuda"))
    # inside the first lap, windows that wrap inside a 64-row tile, committed rows that wrap, far laps
    pos = torch.tensor([0, 40, R - 3, R - W // 2, 2 * R + 30, 7 * R - 20], device="cuda")
    B, T = pos.numel(), int(pos.max()) + W
    kc, vc, kw = _history(B, T, H // G, cache, 10 * G + W)
    q = torch.randn(B, W, H, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(W)).bfloat16()
    kr, vr = _ring(kc, pos, W), _ring(vc, pos, W)
    want = attention.speculation_attention(q, kc, vc, pos, mask, depth, SW, **kw)
    n0 = _ext.launches()
    got = attention.speculation_attention(q, kr, vr, pos, mask, depth, SW, rolling=True, **kw)
    assert _ext.launches() == n0 + 2
    assert torch.isfinite(got).all() and torch.equal(got, want)


@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
@pytest.mark.parametrize("tree", (False, True))
def test_append_ring_rows(_ext, tree, cache):
    """Token w lands in ring row (p + w) mod R with the bytes the linear kernel writes to row p + w; no other row changes."""
    from neuronx_distributed_b200.ops import rope

    e = _ext.ext()
    Rr, B, H, Hkv, D = 70, 3, 8, 2, 128
    depth = medusa_tree("cuda")[1] if tree else None
    W = 10 if tree else 6
    T = 8 * Rr
    pos = torch.tensor([3, Rr - 2, 6 * Rr + 1], device="cuda")
    g = torch.Generator(device="cuda").manual_seed(3)
    f = torch.randn(B, W, (H + 2 * Hkv) * D, device="cuda", generator=g).bfloat16() * 3
    q, k, v = f[..., :H * D].view(B, W, H, D), f[..., H * D:(H + Hkv) * D].view(B, W, Hkv, D), f[..., (H + Hkv) * D:].view(B, W, Hkv, D)
    cos, sin = rope.rope_tables(T, D, 10000.0, torch.device("cuda"), 0, 1.0)
    dt = E4M3 if cache == "e4m3" else torch.bfloat16
    kw = {"k_scale": 0.3, "v_scale": 0.3} if cache == "e4m3" else {}
    kl, vl = (torch.zeros(B, T, Hkv, D, device="cuda", dtype=dt) for _ in range(2))
    kr, vr = (torch.zeros(B, Rr, Hkv, D, device="cuda", dtype=dt) for _ in range(2))
    ql = e.decode_rope_kv(q, k, v, pos, cos, sin, kl, vl, depth=depth, **kw)
    qr = e.decode_rope_kv(q, k, v, pos, cos, sin, kr, vr, depth=depth, rolling=True, **kw)
    assert torch.equal(ql, qr)
    b = torch.arange(B, device="cuda")[:, None]
    slots = pos[:, None] + torch.arange(W, device="cuda")
    for lin, ring in ((kl, kr), (vl, vr)):
        assert torch.equal(ring[b, slots % Rr].view(torch.uint8), lin[b, slots].view(torch.uint8))
        rest = torch.ones(B, Rr, dtype=torch.bool, device="cuda")
        rest[b, slots % Rr] = False
        assert not ring.view(torch.uint8)[rest].any()


# ---- a Mistral-shaped model -----------------------------------------------------------------------------------------------
def _models(kv_fp8):
    from test_kv_fp8_gpu import _mistral_cfg, _one_rank_model_parallel

    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    _one_rank_model_parallel()
    out = []
    for rolling in (False, True):
        torch.manual_seed(0)
        out.append(LlamaForInference(_mistral_cfg(sliding_window=64), batch_size=2, max_seq_len=512, on_device_sampling=False,
                                     kv_quant=KVQuantizationConfig(scale=0.3) if kv_fp8 else None,
                                     rolling_kv_cache=rolling).eval())
    lin, ring = out
    assert ring.kv.rolling and ring.kv.rows == 128 and ring.kv.k[0].shape[1] == 128 and lin.kv.k[0].shape[1] == 512
    return lin, ring


@pytest.mark.parametrize("kv_fp8", (False, True))
def test_mistral_ring_equals_linear_bit_for_bit(_ext, monkeypatch, kv_fp8):
    lin, ring = _models(kv_fp8)
    P = 256
    ids = torch.randint(0, 1024, (2, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    last = torch.tensor([200, 40], device="cuda")                           # past the ring; a short prompt in a long bucket
    steps = 2 * 128 + 4                                                     # both sequences wrap the ring at least twice

    def run(m, step):
        logits = [m.context_encoding(ids, last).clone()]
        toks, pos = [logits[0].argmax(-1)], last + 1
        for _ in range(steps):
            logits.append(step(toks[-1].view(2, 1), pos).clone())
            toks.append(logits[-1].argmax(-1))
            pos = pos + 1
        return logits, pos

    e, calls = _ext.ext(), []
    for name in ("decode_rope_kv", "decode_attention"):
        fn = getattr(e, name)
        monkeypatch.setattr(e, name, lambda *a, _fn=fn, _n=name, **kw: calls.append((_n, kw.get("rolling"))) or _fn(*a, **kw))
    ring_logits, pos = run(ring, ring.token_generation)
    monkeypatch.undo()
    assert sorted(set(calls)) == [("decode_attention", True), ("decode_rope_kv", True)]
    lin_logits, _ = run(lin, lin.token_generation)
    for i, (a, b) in enumerate(zip(ring_logits, lin_logits)):
        assert torch.equal(a, b), i

    # CUDA-graph replay of the ring's decode step
    st_tok, st_pos = torch.zeros(2, 1, dtype=torch.long, device="cuda"), last + 1
    ring.context_encoding(ids, last)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ring.token_generation(st_tok, st_pos)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_out = ring.token_generation(st_tok, st_pos)

    def replay(tok, p):
        st_tok.copy_(tok)
        st_pos.copy_(p)
        graph.replay()
        return st_out

    graph_logits, _ = run(ring, replay)
    for i, (a, b) in enumerate(zip(graph_logits, lin_logits)):
        assert torch.equal(a, b), i

    # after the decode run (both caches hold the same history): a chain, then a Medusa tree, its compaction and one more step
    run(ring, ring.token_generation)
    run(lin, lin.token_generation)
    chain = torch.randint(0, 1024, (2, 5), device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
    assert torch.equal(ring.speculation_forward(chain, pos), lin.speculation_forward(chain, pos))
    mask, depth = medusa_tree("cuda")
    tree_ids = torch.randint(0, 1024, (2, depth.numel()), device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    assert torch.equal(ring.speculation_forward(tree_ids, pos, tree_mask=mask, tree_depth=depth),
                       lin.speculation_forward(tree_ids, pos, tree_mask=mask, tree_depth=depth))
    nodes = torch.tensor([[0, 1, 4, 7], [0, 2, 6, 9]], device="cuda")
    nxt = torch.tensor([[3], [5]], device="cuda")
    outs = []
    for m in (ring, lin):
        m.kv.compact_window(pos, nodes)
        outs.append(m.token_generation(nxt, pos + 4))
    assert torch.equal(outs[0], outs[1])
