"""Rolling KV cache without a GPU: the ring rules of ``KVCacheManager`` (row count, prefill from per-sequence prompt
lengths, decode / window writes and ``compact_window`` across the wrap), the rolling visibility rules against the linear
rule on the unrolled history, the torch decode and verification paths on a ring against float64 on the linear history,
a tiny Mistral-shaped model generating from a ring as it does from the full cache, and the argument errors."""
import pytest
import torch

from dist_utils import run_distributed
from test_speculation_attention_cpu import MEDUSA_CHOICES, medusa_tree, random_tree, ref64, rel

from neuronx_distributed_b200.inference.kv_cache import KVCacheManager
from neuronx_distributed_b200.ops import attention

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2


def _pair(B, max_len, sw, Hkv=2, D=4, dtype=torch.float32, kv_quant=None):
    """(rolling, linear) managers of one layer holding the same positions."""
    ring = KVCacheManager(1, B, max_len, Hkv, D, dtype=dtype, kv_quant=kv_quant, rolling_window=sw)
    lin = KVCacheManager(1, B, max_len, Hkv, D, dtype=dtype, kv_quant=kv_quant)
    return ring, lin


def _same_history(ring, lin, ends, n=None):
    """Ring row t mod R of sequence b equals linear row t for the last n (default R) positions before ends[b]."""
    R = ring.rows
    for b, end in enumerate(ends):
        for t in range(max(0, end - (n or R)), end):
            for a, c in ((ring.k[0], lin.k[0]), (ring.v[0], lin.v[0])):
                assert torch.equal(a[b, t % R].view(torch.uint8), c[b, t].view(torch.uint8)), (b, t)


def test_row_count_and_mode():
    ring = KVCacheManager(2, 3, 1000, 2, 8, dtype=torch.float32, rolling_window=100)
    assert ring.rolling and ring.rows == 100 + attention.SPEC_MAX_TOKENS and ring.k[1].shape == (3, 164, 2, 8)
    short = KVCacheManager(1, 1, 150, 2, 8, dtype=torch.float32, rolling_window=100)   # SW + 64 ≥ max_seq_len: linear
    assert not short.rolling and short.rows == 150 and short.k[0].shape[1] == 150
    assert KVCacheManager(1, 1, 150, 2, 8).rows == 150 and not KVCacheManager(1, 1, 150, 2, 8).rolling


@pytest.mark.parametrize("dtype", (torch.float32, torch.bfloat16, E4M3))
def test_prefill_lengths_below_at_and_past_the_ring(dtype):
    """Prompt lengths < R, = R, > R and with right-padding past R in one batch: every ring row holds the newest prompt position
    of its residue class, rows with none keep their bytes, and padding never lands."""
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    kvq = KVQuantizationConfig(scale=0.5, dequant_dtype=torch.float32) if dtype == E4M3 else None
    sw, B, S = 10, 5, 200
    ring, lin = _pair(B, 400, sw, dtype=torch.float32 if kvq else dtype, kv_quant=kvq)
    R = ring.rows
    assert R == 74
    lens = torch.tensor([30, R, R + 1, 190, 50])                           # the last one is padded far past R
    g = torch.Generator().manual_seed(0)
    k, v = (torch.randn(B, S, 2, 4, generator=g).to(torch.float32 if kvq else dtype) for _ in range(2))
    for t in ring.k + ring.v:
        t.view(torch.uint8).fill_(0x5A)                                     # stale content
    sentinel = ring.k[0].clone()
    ring.write_prefill(0, k, v, lengths=lens)
    lin.write_prefill(0, k, v)
    _same_history(ring, lin, lens.tolist())
    for b, n in enumerate(lens.tolist()):
        if n < R:
            assert torch.equal(ring.k[0][b, n:].view(torch.uint8), sentinel[b, n:].view(torch.uint8))
    # no lengths: the whole bucket is the prompt
    ring.write_prefill(0, k, v)
    _same_history(ring, lin, [S] * B)


def test_prefill_seq_ids():
    ring, lin = _pair(4, 300, 8)
    k, v = torch.randn(2, 100, 2, 4), torch.randn(2, 100, 2, 4)
    ids = torch.tensor([3, 1])
    ring.write_prefill(0, k, v, seq_ids=ids, lengths=torch.tensor([100, 40]))
    lin.write_prefill(0, k, v, seq_ids=ids)
    R = ring.rows
    for b, n in ((3, 100), (1, 40)):
        for t in range(max(0, n - R), n):
            assert torch.equal(ring.k[0][b, t % R], lin.k[0][b, t]) and torch.equal(ring.v[0][b, t % R], lin.v[0][b, t])
    assert not ring.k[0][0].any() and not ring.k[0][2].any()


def test_decode_window_and_compact_wrap():
    """Decode and window writes past the end of the ring, and compact_window whose source and destination straddle the
    wrap, keep the ring equal to the linear cache on the last R positions."""
    B, sw = 2, 6
    ring, lin = _pair(B, 1000, sw)
    R = ring.rows
    g = torch.Generator().manual_seed(1)
    pos = torch.tensor([R - 3, 2 * R - 1])
    k, v = torch.randn(B, 40, 2, 4, generator=g), torch.randn(B, 40, 2, 4, generator=g)
    for m in (ring, lin):
        m.write_prefill(0, k, v, lengths=torch.tensor([40, 40]))
    steps = 2 * R - 1                                                       # decode across the wrap, more than once
    for step in range(steps):
        kd, vd = torch.randn(B, 1, 2, 4, generator=g), torch.randn(B, 1, 2, 4, generator=g)
        for m in (ring, lin):
            m.write_window(0, kd, vd, pos + step)
    p = pos + steps
    _same_history(ring, lin, p.tolist())
    W = 10
    assert ((p % R) + W > R).all()                                          # both windows straddle the end of the ring
    kw, vw = torch.randn(B, W, 2, 4, generator=g), torch.randn(B, W, 2, 4, generator=g)
    for m in (ring, lin):
        m.write_window(0, kw, vw, p)
    _same_history(ring, lin, (p + W).tolist())
    offsets = torch.tensor([[0, 3, 7, 9], [0, 1, 5, 8]])
    for m in (ring, lin):
        m.compact_window(p, offsets)
    _same_history(ring, lin, (p + 4).tolist(), n=R - W + 4)                 # the window overwrote the oldest W positions
    with pytest.raises(ValueError, match="prefix"):
        ring.stored(0, 10)


def test_decode_visibility_matches_linear_rule_on_unrolled_history():
    """One decode token is the W = 1 chain of the verification rule: ``speculation_visibility(…, 1, …)[:, 0]``."""
    for L, sw in ((20, 7), (20, 19), (33, 1)):
        pos = torch.tensor([0, 5, L - 1, L, L + 3, 3 * L + 11])
        vr = attention.speculation_visibility(pos, L, 1, window=sw, rolling=True)[:, 0]
        T = int(pos.max()) + 1
        vl = attention.speculation_visibility(pos, T, 1, window=sw)[:, 0]
        t = torch.arange(T)[None, :]
        assert torch.equal(vl, (t <= pos[:, None]) & (t > pos[:, None] - sw))   # the plain decode rule
        j = torch.arange(L)
        for b, p in enumerate(pos.tolist()):
            c = p - (p - j) % L                                             # logical position of row j
            want = torch.where(c >= 0, vl[b, c.clamp(min=0)], torch.zeros_like(vr[b]))
            assert torch.equal(vr[b], want)
            assert int(vr[b].sum()) == int(vl[b].sum())                     # nothing the linear rule sees is lost


@pytest.mark.parametrize("kind", ("chain", "medusa", "random"))
def test_speculation_visibility_matches_linear_rule_on_unrolled_history(kind):
    W = 10
    mask, depth = (None, None) if kind == "chain" else (medusa_tree() if kind == "medusa" else random_tree(W, 4))
    for sw in (4, 12):
        L = sw + W - 1 + (kind == "random")
        pos = torch.tensor([0, 3, L - W, L - 2, L + 5, 4 * L + 1])
        vr = attention.speculation_visibility(pos, L, W, mask, depth, sw, rolling=True)
        T = int(pos.max()) + W
        vl = attention.speculation_visibility(pos, T, W, mask, depth, sw)
        j = torch.arange(L)
        for b, p in enumerate(pos.tolist()):
            u = (j - p) % L
            c = torch.where(u < W, p + u, p - 1 - (p - 1 - j) % L)
            want = torch.where(c >= 0, vl[b][:, c.clamp(min=0)], torch.zeros_like(vr[b]))
            assert torch.equal(vr[b], want), (sw, p)
            assert torch.equal(vr[b].sum(1), vl[b].sum(1))


def _ring_from(hist, L, end):
    """[B, L, ...] ring holding positions < end[b] of hist [B, T, ...] (row t mod L: the newest such t)."""
    ring = torch.zeros((hist.shape[0], L) + hist.shape[2:], dtype=hist.dtype)
    for b, e in enumerate(end):
        for t in range(max(0, e - L), e):
            ring[b, t % L] = hist[b, t]
    return ring


def _hist(B, T, Hkv, D, cache, g):
    k, v = torch.randn(B, T, Hkv, D, generator=g), torch.randn(B, T, Hkv, D, generator=g)
    if cache in (E4M3, E5M2):
        k8, v8 = (k / 0.5).to(cache), (v / 0.25).to(cache)
        return k8, v8, k8.double() * 0.5, v8.double() * 0.25, {"k_scale": 0.5, "v_scale": 0.25}
    k, v = k.to(cache), v.to(cache)
    return k, v, k.double(), v.double(), {}


@pytest.mark.parametrize("cache", (torch.float32, torch.bfloat16, E4M3, E5M2))
def test_torch_decode_on_ring_vs_float64_linear(cache):
    B, H, Hkv, D, sw = 6, 8, 2, 16, 9
    L = sw + 5
    g = torch.Generator().manual_seed(2)
    pos = torch.tensor([0, 4, L - 1, L, 2 * L + 3, 4 * L + 7])               # several wraps
    T = int(pos.max()) + 1
    kc, vc, kd, vd, kw = _hist(B, T, Hkv, D, cache, g)
    q = torch.randn(B, 1, H, D, generator=g).to(torch.float32 if cache == torch.float32 else torch.bfloat16)
    kr, vr = _ring_from(kc, L, (pos + 1).tolist()), _ring_from(vc, L, (pos + 1).tolist())
    got = attention.decode_attention(q, kr, vr, pos, sliding_window=sw, rolling=True, **kw)
    want = ref64(q, kd, vd, pos, sw=sw)
    assert rel(got, want) < (1e-5 if cache == torch.float32 else 2e-2)


@pytest.mark.parametrize("kind", ("chain", "medusa"))
@pytest.mark.parametrize("cache", (torch.float32, torch.bfloat16, E4M3, E5M2))
def test_torch_verification_on_ring_vs_float64_linear(cache, kind):
    B, H, Hkv, D, sw = 6, 4, 2, 16, 7
    W = 5 if kind == "chain" else 10
    mask, depth = (None, None) if kind == "chain" else medusa_tree()
    L = sw + W - 1                                                          # the smallest ring the rule allows
    g = torch.Generator().manual_seed(3)
    pos = torch.tensor([0, 3, L - W, L - 1, 2 * L + 3, 5 * L + 2])
    T = int(pos.max()) + W
    kc, vc, kd, vd, kw = _hist(B, T, Hkv, D, cache, g)
    q = torch.randn(B, W, H, D, generator=g).to(torch.float32 if cache == torch.float32 else torch.bfloat16)
    end = (pos + W).tolist()
    kr, vr = _ring_from(kc, L, end), _ring_from(vc, L, end)
    got = attention.speculation_attention(q, kr, vr, pos, mask, depth, sw, rolling=True, **kw)
    want = ref64(q, kd, vd, pos, mask, depth, sw)
    assert rel(got, want) < (1e-5 if cache == torch.float32 else 2e-2)


def test_argument_errors():
    q = torch.randn(1, 1, 4, 16)
    k = torch.zeros(1, 12, 2, 16)
    pos = torch.tensor([30])
    for sw in (None, 12, 20):
        with pytest.raises(ValueError, match="rolling"):
            attention.decode_attention(q, k, k, pos, sliding_window=sw, rolling=True)
    attention.decode_attention(q, k, k, pos, sliding_window=11, rolling=True)
    qw = torch.randn(1, 4, 4, 16)
    for sw in (None, 10):                                                   # 10 + 4 − 1 > 12
        with pytest.raises(ValueError, match="rolling"):
            attention.speculation_attention(qw, k, k, pos, sliding_window=sw, rolling=True)
        with pytest.raises(ValueError, match="rolling"):
            attention.speculation_attention_torch(qw, k, k, pos, sliding_window=sw, rolling=True)
    attention.speculation_attention(qw, k, k, pos, sliding_window=9, rolling=True)
    ring = KVCacheManager(1, 1, 500, 2, 4, dtype=torch.float32, rolling_window=8)
    for fn in (lambda: ring.write_prefill_sharded(0, k, k, 0), lambda: ring.write_decode_sharded(0, k[:, :1], k[:, :1], pos, 0)):
        with pytest.raises(ValueError, match="rolling"):
            fn()
    with pytest.raises(ValueError, match="rolling_window"):
        KVCacheManager(1, 1, 500, 2, 4, rolling_window=0)


# ---- a tiny Mistral-shaped model ------------------------------------------------------------------------------------------
def _cfg(sw=8):
    from neuronx_distributed_b200.models.llama import LlamaConfig

    return LlamaConfig(vocab_size=64, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=8,
                       num_key_value_heads=2, dtype=torch.float32, max_position_embeddings=256, sliding_window=sw)


def _pair_models(B, max_len, **kw):
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference

    torch.manual_seed(0)
    lin = LlamaForInference(_cfg(), batch_size=B, max_seq_len=max_len, **kw).eval()
    ring = LlamaForInference(_cfg(), batch_size=B, max_seq_len=max_len, rolling_kv_cache=True, **kw).eval()
    ring.load_state_dict(lin.state_dict())
    assert ring.kv.rolling and ring.kv.rows == 8 + 64 and not lin.kv.rolling
    return ring, lin


def _model_rolling_vs_linear(rank, world):
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.utils.medusa import MedusaHeads, medusa_generate
    from neuronx_distributed_b200.utils.speculative import speculative_generate

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    ring, lin = _pair_models(2, 256, on_device_sampling=False)
    R = ring.kv.rows
    ids = torch.randint(0, 64, (2, 128), generator=torch.Generator().manual_seed(1))
    last = torch.tensor([R + 20, 30])                                       # past the ring; a short prompt in a long bucket
    outs = {}
    for name, m in (("ring", ring), ("lin", lin)):
        logits = [m.context_encoding(ids, last)]
        pos, toks = last + 1, [logits[0].argmax(-1)]
        while int(pos.min()) < 2 * R + 40:                                  # the ring wraps at least twice for both
            logits.append(m.token_generation(toks[-1].view(2, 1), pos))
            toks.append(logits[-1].argmax(-1))
            pos = pos + 1
        outs[name] = (torch.stack(toks, 1), logits)
    assert torch.equal(outs["ring"][0], outs["lin"][0])
    for a, b in zip(outs["ring"][1], outs["lin"][1]):
        assert rel(a, b.double()) < 1e-4

    # speculation chain and Medusa tree windows past the wrap
    window = torch.randint(0, 64, (2, 5), generator=torch.Generator().manual_seed(2))
    mask, depth = medusa_tree()
    tree_ids = torch.randint(0, 64, (2, depth.numel()), generator=torch.Generator().manual_seed(3))
    p = pos
    for a, b in ((ring.speculation_forward(window, p), lin.speculation_forward(window, p)),
                 (ring.speculation_forward(tree_ids, p, tree_mask=mask, tree_depth=depth),
                  lin.speculation_forward(tree_ids, p, tree_mask=mask, tree_depth=depth))):
        assert rel(a, b.double()) < 1e-4 and torch.equal(a.argmax(-1), b.argmax(-1))

    with pytest.raises(ValueError, match="kv_len"):
        ring.token_generation(window[:, :1], p, kv_len=100)
    with pytest.raises(ValueError, match="sliding window"):
        LlamaForInference(_cfg(None), batch_size=1, max_seq_len=256, rolling_kv_cache=True)
    with pytest.raises(ValueError, match="flash_decoding"):
        LlamaForInference(_cfg(), batch_size=1, max_seq_len=256, rolling_kv_cache=True, flash_decoding=True)

    # greedy, speculative and Medusa generation from a prompt longer than the ring give the same tokens
    ring1, lin1 = _pair_models(1, 256)
    torch.manual_seed(1)
    draft_r = LlamaForInference(_cfg(), batch_size=1, max_seq_len=256, rolling_kv_cache=True).eval()
    draft_l = LlamaForInference(_cfg(), batch_size=1, max_seq_len=256).eval()
    draft_l.load_state_dict(draft_r.state_dict())
    prompt = torch.randint(0, 64, (1, R + 9), generator=torch.Generator().manual_seed(4))
    assert torch.equal(ring1.generate(prompt, 100), lin1.generate(prompt, 100))
    got, _ = speculative_generate(ring1, draft_r, prompt, 100, 4)
    want, _ = speculative_generate(lin1, draft_l, prompt, 100, 4)
    assert torch.equal(got, want)
    heads = MedusaHeads(64, 64, 3).eval()
    for proj in heads.proj:
        proj.weight.data.copy_(lin1.lm.lm_head.weight.data)
    got, _ = medusa_generate(ring1, heads, prompt, 100, MEDUSA_CHOICES, topk=10)
    want, _ = medusa_generate(lin1, heads, prompt, 100, MEDUSA_CHOICES, topk=10)
    assert torch.equal(got, want)


def test_mistral_shaped_model_rolling_equals_linear():
    run_distributed(_model_rolling_vs_linear, 1, timeout=300)
