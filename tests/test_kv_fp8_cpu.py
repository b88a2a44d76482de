"""fp8 (e4m3) KV cache without a GPU: ``LlamaForInference(kv_quant=…)`` stores and generates from a quantised cache, flash
decoding and speculation windows read it, and ``ops.attention.decode_attention`` de-quantises it on its torch path."""
import math

import pytest
import torch

from dist_utils import run_distributed


def _cfg(dtype=torch.float32, **kw):
    from neuronx_distributed_b200.models.llama import LlamaConfig

    return LlamaConfig(vocab_size=64, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=8,
                       num_key_value_heads=2, dtype=dtype, max_position_embeddings=32, **kw)


def _kvq(scale, dequant=torch.float32):
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    return KVQuantizationConfig(scale=scale, dequant_dtype=dequant)


def _model_storage(rank, world):
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    plain = LlamaForInference(_cfg(torch.bfloat16), batch_size=2, max_seq_len=32).eval()
    torch.manual_seed(0)
    fp8 = LlamaForInference(_cfg(torch.bfloat16), batch_size=2, max_seq_len=32, kv_quant=KVQuantizationConfig(scale=0.5)).eval()
    fp8.load_state_dict(plain.state_dict())
    assert fp8.kv.k[0].dtype == torch.float8_e4m3fn and fp8.kv.v[0].dtype == torch.float8_e4m3fn
    assert fp8.kv.k[0].nbytes * 2 == plain.kv.k[0].nbytes and fp8.kv.v[1].nbytes * 2 == plain.kv.v[1].nbytes
    assert fp8.kv.kernel_scales() is None                          # on the CPU no kernel reads it
    ids = torch.randint(0, 64, (2, 12), generator=torch.Generator().manual_seed(1))
    got = fp8.generate(ids, 6)
    assert got.shape == (2, 6) and int(got.min()) >= 0 and int(got.max()) < 64
    # prompt rows hold the manager's rule applied to the bf16 rows the plain model stores
    plain.generate(ids, 6)
    for t in ("k", "v"):
        want = fp8.kv._q(getattr(plain.kv, t)[1][:, :12])
        assert torch.equal(getattr(fp8.kv, t)[1][:, :12].view(torch.uint8), want.view(torch.uint8)), t
    for bad in (dict(k_quant_method="per_key_symmetric"), dict(v_quant_method="per_channel_symmetric"), dict(per_key=True)):
        with pytest.raises(ValueError, match="per-key"):
            LlamaForInference(_cfg(torch.bfloat16), batch_size=2, max_seq_len=32, kv_quant=KVQuantizationConfig(direct_cast=False, **bad))
    with pytest.raises(ValueError, match="dequant_dtype"):          # an fp32 model with the default bf16 de-quantisation
        LlamaForInference(_cfg(), batch_size=2, max_seq_len=32, kv_quant=KVQuantizationConfig(scale=0.5))


def test_llama_inference_fp8_cache_storage_generation_and_per_key_rejection():
    run_distributed(_model_storage, 1, timeout=120)


def _flash_decode_fp8(rank, world):
    """TP = 4 over 2 KV heads: each KV head's fp8 cache is sharded along the sequence over 2 ranks; generation equals the
    replicated fp8-cache model token for token."""
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    plain = LlamaForInference(_cfg(), batch_size=2, max_seq_len=32, kv_quant=_kvq(0.3)).eval()
    torch.manual_seed(0)
    fd = LlamaForInference(_cfg(), batch_size=2, max_seq_len=32, flash_decoding=True, kv_quant=_kvq(0.3)).eval()
    fd.load_state_dict(plain.state_dict())
    assert fd.kv.k[0].shape[1] == 16 and fd.kv.k[0].dtype == torch.float8_e4m3fn
    ids = torch.randint(0, 64, (2, 20), generator=torch.Generator().manual_seed(1))   # prompt crosses the shard boundary (16)
    lens = torch.tensor([20, 13])
    want = plain.generate(ids, 8, prompt_lens=lens)
    got = fd.generate(ids, 8, prompt_lens=lens)
    assert torch.equal(got, want), (got, want)


def test_llama_inference_flash_decoding_tp4_fp8_cache():
    run_distributed(_flash_decode_fp8, 4, timeout=240)


def _speculation_fp8(rank, world):
    """A speculation window verified in one pass over the fp8 cache gives the logits of W single-token decode steps over the
    same fp8 cache."""
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    m = LlamaForInference(_cfg(), batch_size=2, max_seq_len=32, on_device_sampling=False, kv_quant=_kvq(0.3)).eval()
    ids = torch.randint(0, 64, (2, 10), generator=torch.Generator().manual_seed(2))
    chain = torch.randint(0, 64, (2, 4), generator=torch.Generator().manual_seed(3))
    pos0 = torch.tensor([10, 7])
    m.kv.reset()
    m.context_encoding(ids, pos0 - 1)
    steps = [m.token_generation(chain[:, i:i + 1], pos0 + i) for i in range(chain.shape[1])]
    step_logits = torch.stack(steps, 1)                                 # [B, W, V]
    m.kv.reset()
    m.context_encoding(ids, pos0 - 1)
    win_logits = m.speculation_forward(chain, pos0)                     # [B, W, V]
    err = (win_logits - step_logits).abs().max() / step_logits.abs().max()
    assert err < 1e-5, err


def test_speculation_window_on_fp8_cache_matches_step_decode():
    run_distributed(_speculation_fp8, 1, timeout=120)


def _ref64(q, k, v, pos, W, ks, vs):
    """float64 decode attention over the de-quantised caches."""
    B, _, H, D = q.shape
    L, Hkv = k.shape[1], k.shape[2]
    kk = (k.double() * ks).repeat_interleave(H // Hkv, 2)
    vv = (v.double() * vs).repeat_interleave(H // Hkv, 2)
    s = torch.einsum("bhd,blhd->bhl", q[:, 0].double(), kk) / math.sqrt(D)
    j = torch.arange(L)[None, :]
    vis = (j <= pos[:, None]) & (j > pos[:, None] - W)
    s = s.masked_fill(~vis[:, None], float("-inf"))
    return torch.einsum("bhl,blhd->bhd", s.softmax(-1), vv).unsqueeze(1)


@pytest.mark.parametrize("dtype", (torch.float8_e4m3fn, torch.float8_e5m2))
@pytest.mark.parametrize("window", (None, 5))
def test_decode_attention_fp8_cache_torch_path_vs_float64(dtype, window):
    from neuronx_distributed_b200.ops import attention

    g = torch.Generator().manual_seed(0)
    B, L, H, Hkv, D = 3, 24, 8, 2, 64
    q = torch.randn(B, 1, H, D, generator=g)
    k = (torch.randn(B, L, Hkv, D, generator=g) / 0.3).to(dtype)
    v = (torch.randn(B, L, Hkv, D, generator=g) / 0.7).to(dtype)
    pos = torch.tensor([0, 11, 23])
    got = attention.decode_attention(q, k, v, pos, sliding_window=window, k_scale=0.3, v_scale=0.7)
    ref = _ref64(q, k, v, pos, window or L + 1, 0.3, 0.7)
    assert got.dtype == torch.float32
    assert (got.double() - ref).abs().max() <= 1e-5 * ref.abs().max(), (got.double() - ref).abs().max()


def test_decode_attention_rejects_scales_on_a_bf16_cache():
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial
    from neuronx_distributed_b200.ops import attention

    q = torch.randn(1, 1, 2, 64).bfloat16()
    k = v = torch.randn(1, 8, 2, 64).bfloat16()
    pos = torch.tensor([5])
    with pytest.raises(ValueError, match="fp8 caches only"):
        attention.decode_attention(q, k, v, pos, k_scale=0.5)
    with pytest.raises(ValueError, match="fp8 caches only"):
        _local_partial(q, k, v, pos, 0.125, v_scale=2.0)
    with pytest.raises(ValueError, match="same dtype"):
        attention.decode_attention(q, k.to(torch.float8_e4m3fn), v, pos)
    # scales of 1.0 are the defaults: the bf16 call is unchanged
    assert torch.equal(attention.decode_attention(q, k, v, pos, k_scale=1.0, v_scale=1.0), attention.decode_attention(q, k, v, pos))


def test_write_decode_sharded_fp8_copies_bytes_on_the_owner_only():
    from neuronx_distributed_b200.modules.attention.flash_decode import write_decode_sharded

    g = torch.Generator().manual_seed(4)
    kc = torch.randn(3, 8, 2, 16, generator=g).to(torch.float8_e4m3fn)
    vc = torch.randn(3, 8, 2, 16, generator=g).to(torch.float8_e4m3fn)
    k0, v0 = kc.clone(), vc.clone()
    kn = torch.randn(3, 1, 2, 16, generator=g).to(torch.float8_e4m3fn)
    vn = torch.randn(3, 1, 2, 16, generator=g).to(torch.float8_e4m3fn)
    pos = torch.tensor([3, 12, 8])                   # rank 1 (positions 8..15) owns sequences 1 and 2
    write_decode_sharded(kc, vc, kn, vn, pos, 1)
    want_k, want_v = k0.clone(), v0.clone()
    want_k[1, 4], want_v[1, 4] = kn[1, 0], vn[1, 0]
    want_k[2, 0], want_v[2, 0] = kn[2, 0], vn[2, 0]
    assert torch.equal(kc.view(torch.uint8), want_k.view(torch.uint8))
    assert torch.equal(vc.view(torch.uint8), want_v.view(torch.uint8))
