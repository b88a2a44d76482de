"""Key-padding mask of ``ops.attention.flash_attention`` on the SDPA path (CPU), and BERT with padded batches vs
``transformers`` at TP=1 and TP=2."""
import pytest
import torch
import torch.nn.functional as F

from dist_utils import run_distributed


def _sdpa_bool(q, k, v, causal, mask):
    """SDPA with the equivalent boolean mask, on [B, H, S, D] tensors with K/V repeated for GQA."""
    g = q.shape[2] // k.shape[2]
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2).repeat_interleave(g, 1), v.transpose(1, 2).repeat_interleave(g, 1)
    vis = mask[:, None, None, :]
    if causal:
        vis = vis & torch.ones(q.shape[1], k.shape[1], dtype=torch.bool).tril()
    return F.scaled_dot_product_attention(qt, kt, vt, attn_mask=vis).transpose(1, 2)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("hkv", [4, 2])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_key_padding_mask_matches_sdpa(causal, hkv, dtype):
    from neuronx_distributed_b200.ops import attention

    g = torch.Generator().manual_seed(0)
    B, S, H, D = 3, 37, 4, 16
    q = torch.randn(B, S, H, D, generator=g).to(dtype)
    k, v = (torch.randn(B, S, hkv, D, generator=g).to(dtype) for _ in range(2))
    mask = torch.rand(B, S, generator=g) < 0.6
    mask[0, :5] = False                                     # left padding on row 0
    mask[2] = False                                         # every key of row 2 masked
    got = attention.flash_attention(q, k, v, causal=causal, key_padding_mask=mask)
    want = _sdpa_bool(q, k, v, causal, mask)
    assert got.shape == (B, S, H, D) and got.dtype == dtype
    torch.testing.assert_close(got, want, rtol=0, atol=0, equal_nan=True)
    # integer masks (nonzero = visible) are accepted as well
    torch.testing.assert_close(attention.flash_attention(q, k, v, causal=causal, key_padding_mask=mask.long()), got,
                               rtol=0, atol=0, equal_nan=True)


def test_no_mask_is_unchanged():
    from neuronx_distributed_b200.ops import attention

    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(2, 20, 4, 16, generator=g) for _ in range(3))
    for causal in (False, True):
        want = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=causal)
        assert torch.equal(attention.flash_attention(q, k, v, causal=causal), want.transpose(1, 2))


def test_flash_kernels_apply_predicate():
    from neuronx_distributed_b200.ops import attention

    q = torch.zeros(1, 8, 2, 64, dtype=torch.bfloat16)
    assert not attention.flash_kernels_apply(q, q, q)      # CPU tensors never take the kernels
    assert attention.FLASH_HEAD_DIMS == (64, 80, 96, 128)


def _bert_padded(rank, world):
    from neuronx_distributed_b200.models import bert, hf_compat
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.mappings import gather_from_tensor_model_parallel_region as gather

    transformers = pytest.importorskip("transformers")
    ps.initialize_model_parallel(world)
    torch.manual_seed(0)
    kw = dict(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
              max_position_embeddings=32)
    hf = transformers.BertForPreTraining(transformers.BertConfig(**kw, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                                                                 attn_implementation="eager")).eval()
    m = bert.BertForPreTraining(bert.BertConfig(**kw, hidden_dropout_prob=0.0, dtype=torch.float32)).eval()
    res = hf_compat.load_hf_checkpoint(m, hf.state_dict())
    assert not res.missing_keys and not res.unexpected_keys, res
    ids = torch.randint(0, 64, (3, 16), generator=torch.Generator().manual_seed(1))
    tt = torch.zeros_like(ids)
    right = torch.ones(3, 16, dtype=torch.long)
    right[1, 11:] = 0
    right[2, 3:] = 0
    left = right.flip(1)
    for am in (right, left):
        with torch.no_grad():
            ref = hf(input_ids=ids, token_type_ids=tt, attention_mask=am)
            seq, _ = m.bert(ids, tt, am)
            _, (mlm, nsp) = m(ids, tt, am)
            hidden = hf.bert(input_ids=ids, token_type_ids=tt, attention_mask=am).last_hidden_state
        assert float((seq - hidden).abs().max()) < 2e-5
        assert float((gather(mlm) - ref.prediction_logits).abs().max()) < 2e-5
        assert float((nsp - ref.seq_relationship_logits).abs().max()) < 2e-5


@pytest.mark.parametrize("world", [1, 2])
def test_bert_padded_batch_matches_transformers(world):
    pytest.importorskip("transformers")
    run_distributed(_bert_padded, world, timeout=300)
