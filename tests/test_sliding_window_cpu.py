"""Sliding-window attention (Mistral / Mixtral ``sliding_window``) on the CPU paths: ``flash_attention`` and
``decode_attention`` against a float64 masked softmax, flash decoding's local partial, HF config loading, and tiny Mistral /
Mixtral models against ``transformers`` past the window, in training-style forward, prefill, decode and speculation."""
import dataclasses

import pytest
import torch

from dist_utils import run_distributed


def _vis(s_q, s_kv, window, kpm=None):
    """[B or 1, S_q, S_kv] bool: causal, i − W < j ≤ i, and the key-padding mask."""
    i, j = torch.arange(s_q)[:, None], torch.arange(s_kv)[None, :]
    vis = (j <= i) & (j > i - window) if window is not None else j <= i
    vis = vis[None]
    return vis & kpm[:, None, :].bool() if kpm is not None else vis


def _ref(q, k, v, vis, scale):
    """float64 softmax(q·kᵀ·scale, masked)·v for [B, S, H, D] tensors (K/V repeated for GQA); empty rows give NaN."""
    g = q.shape[2] // k.shape[2]
    qd = q.double().transpose(1, 2)
    kd, vd = (t.double().transpose(1, 2).repeat_interleave(g, 1) for t in (k, v))
    s = (qd @ kd.transpose(-1, -2) * scale).masked_fill(~vis[:, None], float("-inf"))
    return (torch.softmax(s, -1) @ vd).transpose(1, 2)


@pytest.mark.parametrize("window", [1, 5, 16])
@pytest.mark.parametrize("hkv", [4, 1])
def test_flash_attention_window_vs_float64(window, hkv):
    from neuronx_distributed_b200.ops import attention

    g = torch.Generator().manual_seed(0)
    B, S, H, D = 2, 37, 4, 16
    q = torch.randn(B, S, H, D, generator=g)
    k, v = (torch.randn(B, S, hkv, D, generator=g) for _ in range(2))
    got = attention.flash_attention(q, k, v, causal=True, sliding_window=window)
    want = _ref(q, k, v, _vis(S, S, window), D ** -0.5)
    torch.testing.assert_close(got.double(), want, rtol=0, atol=2e-6)
    # the window matters: rows past it differ from full causal attention
    if window < S:
        assert not torch.allclose(got[:, window:], attention.flash_attention(q, k, v, causal=True)[:, window:])


def test_flash_attention_window_with_padding_mask():
    from neuronx_distributed_b200.ops import attention

    g = torch.Generator().manual_seed(1)
    B, S, H, D, W = 3, 29, 4, 16, 6
    q = torch.randn(B, S, H, D, generator=g)
    k, v = (torch.randn(B, S, 2, D, generator=g) for _ in range(2))
    kpm = torch.rand(B, S, generator=g) < 0.7
    kpm[0, :4] = False                                      # left padding
    kpm[1, 10:16] = False                                   # query 15 of batch 1 sees keys 10..15: all masked → empty row
    got = attention.flash_attention(q, k, v, causal=True, key_padding_mask=kpm, sliding_window=W)
    vis = _vis(S, S, W, kpm)
    assert not bool(vis[1, 15].any())
    want = _ref(q, k, v, vis, D ** -0.5)
    live = vis.any(-1)                                      # [B, S] rows that see at least one key
    torch.testing.assert_close(got.double()[live], want[live], rtol=0, atol=2e-6)
    # an emptied row follows the SDPA fallback's rule for rows without a visible key, as without a window
    empty = attention.flash_attention(q, k, v, causal=True, key_padding_mask=vis[:, 15].clone())[:, 15]
    torch.testing.assert_close(got[:, 15][~live[:, 15]], empty[~live[:, 15]], rtol=0, atol=0, equal_nan=True)


def test_window_at_least_s_is_causal_and_invalid_arguments_raise():
    from neuronx_distributed_b200.ops import attention

    g = torch.Generator().manual_seed(2)
    q, k, v = (torch.randn(2, 20, 4, 16, generator=g) for _ in range(3))
    full = attention.flash_attention(q, k, v, causal=True)
    for w in (20, 21, 1 << 20):
        torch.testing.assert_close(attention.flash_attention(q, k, v, causal=True, sliding_window=w), full, rtol=0, atol=1e-6)
    with pytest.raises(ValueError):
        attention.flash_attention(q, k, v, causal=False, sliding_window=4)
    for bad in (0, -3):
        with pytest.raises(ValueError):
            attention.flash_attention(q, k, v, causal=True, sliding_window=bad)
        with pytest.raises(ValueError):
            attention.decode_attention(q[:, :1], k, v, torch.tensor([3, 5]), sliding_window=bad)


@pytest.mark.parametrize("window", [1, 4, 9, 64])
def test_decode_attention_window_vs_float64(window):
    from neuronx_distributed_b200.ops import attention

    g = torch.Generator().manual_seed(3)
    B, L, H, Hkv, D = 4, 24, 8, 2, 16
    q = torch.randn(B, 1, H, D, generator=g)
    k, v = (torch.randn(B, L, Hkv, D, generator=g) for _ in range(2))
    pos = torch.tensor([0, window - 1 if window <= L else 5, min(window, L - 1), L - 1])
    got = attention.decode_attention(q, k, v, pos, sliding_window=window)
    j = torch.arange(L)[None, :]
    vis = ((j <= pos[:, None]) & (j > pos[:, None] - window))[:, None, :]       # [B, 1, L]
    torch.testing.assert_close(got.double(), _ref(q, k, v, vis, D ** -0.5), rtol=0, atol=2e-6)
    if window >= L:
        torch.testing.assert_close(got, attention.decode_attention(q, k, v, pos), rtol=0, atol=0)


def test_local_partial_window():
    """Flash decoding's per-shard partial with local positions before, inside and past the shard."""
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial

    g = torch.Generator().manual_seed(4)
    B, L, H, Hkv, D, W = 6, 16, 4, 2, 16, 5
    q = torch.randn(B, 1, H, D, generator=g)
    k, v = (torch.randn(B, L, Hkv, D, generator=g) for _ in range(2))
    local = torch.tensor([-3, 2, 9, 15, 18, 40])            # 18: rows 14, 15 visible; 40: window past the shard
    o, m, l = _local_partial(q, k, v, local, 0.25, sliding_window=W)
    j = torch.arange(L)[None, :]
    vis = (j <= local[:, None]) & (j > local[:, None] - W)
    s = torch.einsum("bhd,blhd->bhl", q[:, 0].double(), k.double().repeat_interleave(2, 2)) * 0.25
    s = s.masked_fill(~vis[:, None], float("-inf"))
    m_ref = s.max(-1).values
    p = torch.exp(s - torch.where(torch.isinf(m_ref), torch.zeros_like(m_ref), m_ref)[..., None])
    for b in range(B):
        if vis[b].any():
            torch.testing.assert_close(m[b].double(), m_ref[b], rtol=0, atol=1e-5)
            torch.testing.assert_close(l[b].double(), p[b].sum(-1), rtol=1e-5, atol=0)
            torch.testing.assert_close(o[b].double(), torch.einsum("hl,lhd->hd", p[b], v[b].double().repeat_interleave(2, 1)),
                                       rtol=0, atol=1e-5)
        else:                                               # nothing of this shard is in the window
            assert bool(torch.isinf(m[b]).all()) and float(l[b].abs().max()) == 0.0 and float(o[b].abs().max()) == 0.0
    assert not vis[0].any() and not vis[5].any() and vis[4].sum() == 2


def test_config_from_hf_reads_window_for_mistral_and_mixtral_only():
    from neuronx_distributed_b200.models import hf_compat

    base = dict(vocab_size=128, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=8,
                num_key_value_heads=2, sliding_window=4096)
    assert hf_compat.config_from_hf(dict(base, model_type="mistral")).sliding_window == 4096
    assert hf_compat.config_from_hf(dict(base, model_type="mistral", sliding_window=None)).sliding_window is None
    mx = hf_compat.config_from_hf(dict(base, model_type="mixtral", num_local_experts=4, num_experts_per_tok=2))
    assert mx.sliding_window == 4096
    # Qwen2 carries the field but gates it with use_sliding_window (and per-layer limits): loaded exactly as before
    q2 = hf_compat.config_from_hf(dict(base, model_type="qwen2", use_sliding_window=False, max_window_layers=28))
    assert q2.sliding_window is None
    assert hf_compat.config_from_hf(dict(base, model_type="llama")).sliding_window is None
    no_field = dict(base)
    del no_field["sliding_window"]
    assert hf_compat.config_from_hf(dict(no_field, model_type="qwen2")) == q2


def _hf(fam: str, window: int, kvh: int = 2):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(0)
    common = dict(vocab_size=128, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=8,
                  num_key_value_heads=kvh, max_position_embeddings=64, attn_implementation="eager", sliding_window=window)
    if fam == "mistral":
        hc = transformers.MistralConfig(**common)
        return hc, transformers.MistralForCausalLM(hc).eval()
    hc = transformers.MixtralConfig(num_local_experts=4, num_experts_per_tok=2, **common)
    return hc, transformers.MixtralForCausalLM(hc).eval()


def _model_cls(fam):
    if fam == "mistral":
        from neuronx_distributed_b200.models.llama import LlamaForCausalLM
        return LlamaForCausalLM
    from neuronx_distributed_b200.models.mixtral import MixtralForCausalLM
    return MixtralForCausalLM


def _logits_parity(rank, world, fam):
    from neuronx_distributed_b200.models import hf_compat
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.mappings import gather_from_tensor_model_parallel_region as gather

    ps.initialize_model_parallel(world)
    hc, hf = _hf(fam, 8)
    cfg = hf_compat.config_from_hf(hc, dtype=torch.float32)
    assert cfg.sliding_window == 8
    model = _model_cls(fam)(cfg).eval()
    res = hf_compat.load_hf_checkpoint(model, hf.state_dict())
    assert not res.missing_keys and not res.unexpected_keys
    ids = torch.randint(0, 128, (2, 32), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        ref = hf(ids).logits
        lg = gather(model(ids)[1]).transpose(0, 1)
    assert float((lg - ref).abs().max()) < 2e-5
    # without the window the same weights give other logits past position 8
    full = _model_cls(fam)(dataclasses.replace(cfg, sliding_window=None)).eval()
    hf_compat.load_hf_checkpoint(full, hf.state_dict())
    with torch.no_grad():
        lg_full = gather(full(ids)[1]).transpose(0, 1)
    assert float((lg_full[:, :8] - lg[:, :8]).abs().max()) < 1e-5 and float((lg_full[:, 8:] - ref[:, 8:]).abs().max()) > 1e-3


@pytest.mark.parametrize("fam", ["mistral", "mixtral"])
@pytest.mark.parametrize("world", [1, 2])
def test_hf_window_logits_parity(fam, world):
    pytest.importorskip("transformers")
    run_distributed(_logits_parity, world, fam, timeout=300)


def _generation(rank, world, fam):
    from neuronx_distributed_b200.models import hf_compat
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(world)
    W, P, N = 8, 12, 14                                     # window, prompt (longer than the window), new tokens
    hc, hf = _hf(fam, W)
    cfg = hf_compat.config_from_hf(hc, dtype=torch.float32)
    srv = LlamaForInference(cfg, batch_size=1, max_seq_len=64, lm_cls=_model_cls(fam)).eval()
    res = hf_compat.load_hf_checkpoint(srv, hf.state_dict())
    assert not res.missing_keys and not res.unexpected_keys
    prompt = torch.randint(1, 128, (1, P), generator=torch.Generator().manual_seed(2))
    want = hf.generate(prompt, max_new_tokens=N, do_sample=False, pad_token_id=0)[0, P:].tolist()
    tok = srv.context_encoding(prompt, torch.tensor([P - 1]))
    got = [int(tok[0])]
    for i in range(N - 1):
        tok = srv.token_generation(tok.view(1, 1), torch.tensor([P + i]))
        got.append(int(tok[0]))
    assert got == want, (got, want)
    # speculation chain past the window: re-encode the prompt, decode 2 tokens, then verify the next 5 known tokens at once
    srv.context_encoding(prompt, torch.tensor([P - 1]))
    for i in range(2):
        srv.token_generation(torch.tensor([[want[i]]]), torch.tensor([P + i]))
    chain = torch.tensor([want[2:7]])
    spec = srv.speculation_forward(chain, torch.tensor([P + 2]))
    assert spec[0].tolist() == want[3:8], (spec[0].tolist(), want[3:8])
    # the same chain written as a Medusa tree (each node's parent is the node before it, depth = index)
    tree = srv.speculation_forward(chain, torch.tensor([P + 2]), tree_mask=torch.ones(5, 5, dtype=torch.bool).tril(),
                                   tree_depth=torch.arange(5))
    assert tree[0].tolist() == want[3:8], (tree[0].tolist(), want[3:8])


@pytest.mark.parametrize("fam", ["mistral", "mixtral"])
def test_hf_window_generation_matches_transformers(fam):
    pytest.importorskip("transformers")
    run_distributed(_generation, 2, fam, timeout=300)


def _cp_raises(rank, world):
    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=1, context_parallel_size=world)
    cfg = LlamaConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=1, num_attention_heads=4,
                      dtype=torch.float32, max_position_embeddings=32, context_parallel=True, sliding_window=4)
    model = LlamaForCausalLM(cfg)
    with pytest.raises(NotImplementedError, match="sliding_window"):
        model(torch.randint(0, 64, (1, 8)))


def test_context_parallel_with_window_raises():
    run_distributed(_cp_raises, 2, timeout=120)
