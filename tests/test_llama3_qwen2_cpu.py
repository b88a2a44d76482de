"""Llama-3.1 / 3.2 and Qwen2 / Qwen2.5 checkpoints against ``transformers``: Llama-3 ("llama3") RoPE frequency rescaling
and q / k / v projection biases, loaded TP-sharded (with KV replication where the kv heads do not cover the ranks),
served through ``LlamaForInference`` and trained one step under sequence parallelism."""
import pytest
import torch

from dist_utils import run_distributed

transformers = pytest.importorskip("transformers")

# original_max_position_embeddings = 32 puts the 16 frequencies of head_dim 32 in all three bands: wavelength 2π < 8
# (kept), 2π·10^¼ and 2π·10^½ between 8 and 32 (smoothed), the rest > 32 (divided by the factor)
LLAMA3_SCALING = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                  "original_max_position_embeddings": 32}


def _hf_llama3():
    torch.manual_seed(0)
    hc = transformers.LlamaConfig(vocab_size=128, hidden_size=128, intermediate_size=96, num_hidden_layers=2,
                                  num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=64,
                                  rope_scaling=dict(LLAMA3_SCALING), attn_implementation="eager")
    return hc, transformers.LlamaForCausalLM(hc).eval()


def _hf_qwen2(heads: int, kv_heads: int, head_dim: int = 16):
    torch.manual_seed(0)
    hc = transformers.Qwen2Config(vocab_size=128, hidden_size=heads * head_dim, intermediate_size=96, num_hidden_layers=2,
                                  num_attention_heads=heads, num_key_value_heads=kv_heads, max_position_embeddings=64,
                                  attn_implementation="eager")
    hf = transformers.Qwen2ForCausalLM(hc).eval()
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():                     # transformers initialises the biases to zero: make them matter
        for n, p in hf.named_parameters():
            if n.endswith(("q_proj.bias", "k_proj.bias", "v_proj.bias")):
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
    return hc, hf


def test_rope_tables_llama3_match_transformers():
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS

    from neuronx_distributed_b200.models import hf_compat
    from neuronx_distributed_b200.ops.rope import rope_tables

    hc, _ = _hf_llama3()
    cfg = hf_compat.config_from_hf(hc)
    assert cfg.rope_scaling == {k: v for k, v in LLAMA3_SCALING.items() if k != "rope_type"} and cfg.rope_scaling_factor == 1.0
    inv, attention_factor = ROPE_INIT_FUNCTIONS["llama3"](hc, "cpu")
    assert attention_factor == 1.0
    t = torch.arange(40, 104, dtype=torch.float32)
    cos, sin = rope_tables(64, cfg.head_dim, cfg.rope_theta, offset=40, rope_scaling=cfg.rope_scaling)
    assert torch.equal(cos, torch.outer(t, inv).cos()) and torch.equal(sin, torch.outer(t, inv).sin())
    # without rope_scaling the tables are the plain ones, bit for bit (also with a linear factor)
    for scaling in (1.0, 2.0):
        inv0 = 1.0 / (1e4 ** (torch.arange(0, 32, 2, dtype=torch.float32) / 32))
        fr = torch.outer(torch.arange(0, 64, dtype=torch.float32) / scaling, inv0)
        c0, s0 = rope_tables(64, 32, 1e4, scaling=scaling, rope_scaling=None)
        assert torch.equal(c0, fr.cos()) and torch.equal(s0, fr.sin())
    # other rope types keep plain RoPE, as before
    for other in ({"rope_type": "yarn", "factor": 4.0}, {"rope_type": "dynamic", "factor": 2.0}):
        c = hf_compat.config_from_hf({**hc.to_dict(), "rope_parameters": None, "rope_scaling": other})
        assert c.rope_scaling is None and c.rope_scaling_factor == 1.0


def _parity(rank, world, fam, heads, kv_heads, tmp):
    import os

    from neuronx_distributed_b200.models import hf_compat
    from neuronx_distributed_b200.models.llama import LlamaForCausalLM
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.mappings import gather_from_tensor_model_parallel_region

    ps.initialize_model_parallel(world)
    hc, hf = _hf_llama3() if fam == "llama3" else _hf_qwen2(heads, kv_heads)
    sd = hf.state_dict()
    cfg = hf_compat.config_from_hf(hc, dtype=torch.float32)
    assert cfg.qkv_bias == (fam == "qwen2") and (cfg.rope_scaling is not None) == (fam == "llama3")
    model = LlamaForCausalLM(cfg).eval()
    res = hf_compat.load_hf_checkpoint(model, sd)
    assert not res.missing_keys and not res.unexpected_keys, res
    ids = torch.randint(0, 128, (2, 40), generator=torch.Generator().manual_seed(1))      # past original_max_position_embeddings
    with torch.no_grad():
        ref = hf(ids).logits
        _, lg = model(ids)
    lg = gather_from_tensor_model_parallel_region(lg).transpose(0, 1)
    err = float((lg - ref).abs().max())
    assert err < 2e-5, err

    # sharded model → HF names, bit for bit (biases included, KV replicas dropped); and through files
    back = hf_compat.nxd_to_hf_state_dict(hf_compat.gather_full_state_dict(model), cfg, **hf_compat._kv_args(model))
    assert set(back) == set(sd) and all(torch.equal(back[k], sd[k]) for k in sd)
    out = os.path.join(tmp, "hf_out")
    hf_compat.save_hf_checkpoint(model, out, hf_config=hc)
    cfg2 = hf_compat.config_from_hf(out, dtype=torch.float32)
    assert cfg2.qkv_bias == cfg.qkv_bias and cfg2.rope_scaling == cfg.rope_scaling
    model2 = LlamaForCausalLM(cfg2).eval()
    hf_compat.load_hf_checkpoint(model2, out)
    with torch.no_grad():
        _, lg2 = model2(ids)
    assert torch.equal(gather_from_tensor_model_parallel_region(lg2).transpose(0, 1), lg)

    # serving: greedy tokens equal transformers' generate (prefill, then one token at a time, then a 4-token window)
    srv = LlamaForInference(hf_compat.config_from_hf(hc, dtype=torch.float32), batch_size=1, max_seq_len=64).eval()
    res = hf_compat.load_hf_checkpoint(srv, sd)
    assert not res.missing_keys and not res.unexpected_keys, res
    prompt = torch.randint(0, 128, (1, 30), generator=torch.Generator().manual_seed(2))
    want = hf.generate(prompt, max_new_tokens=12, do_sample=False, pad_token_id=0)[0, 30:].tolist()
    got = srv.generate(prompt, 8)[0].tolist()
    assert got == want[:8], (got, want)
    # verify the next 4 tokens HF chose as one window at positions 38..41: each predicts the token after it
    nxt = srv.speculation_forward(torch.tensor([want[7:11]]), torch.tensor([38]))
    assert nxt[0].tolist() == want[8:12], (nxt, want)


@pytest.mark.parametrize("world", [1, 2, 4])
def test_llama3_rope_scaling_parity(tmp_path, world):
    """4 heads / 2 kv heads: TP 4 replicates each kv head twice."""
    run_distributed(_parity, world, "llama3", 4, 2, str(tmp_path), timeout=300)


@pytest.mark.parametrize("world,heads,kv_heads", [(1, 14, 2), (2, 14, 2), (4, 8, 2)])
def test_qwen2_qkv_bias_parity(tmp_path, world, heads, kv_heads):
    """14 / 2 heads: GQA group 7 (Qwen2.5-0.5B's); 8 / 2 heads at TP 4 replicates each kv head twice."""
    run_distributed(_parity, world, "qwen2", heads, kv_heads, str(tmp_path), timeout=300)


def _train_step(rank, world, fuse_qkv):
    from neuronx_distributed_b200.models import hf_compat
    from neuronx_distributed_b200.models.llama import LlamaForCausalLM
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.grads import allreduce_sequence_parallel_gradients

    ps.initialize_model_parallel(world)
    hc, hf = _hf_qwen2(8, 1)                  # one kv head: replicated over both ranks at TP 2
    ids = torch.randint(0, 128, (2, 16), generator=torch.Generator().manual_seed(3))
    hf.train()
    hf(ids, labels=ids).loss.backward()
    cfg = hf_compat.config_from_hf(hc, dtype=torch.float32, sequence_parallel_enabled=world > 1, fuse_qkv=fuse_qkv)
    model = LlamaForCausalLM(cfg).train()
    hf_compat.load_hf_checkpoint(model, hf.state_dict())
    loss, _ = model(ids, labels=ids)
    loss.backward()
    allreduce_sequence_parallel_gradients(torch.optim.SGD(model.parameters(), lr=0.0))   # the norms saw S / tp tokens
    # the gradients, gathered and renamed as the weights are (KV replicas dropped: every replica holds the group's sum)
    kv = hf_compat._kv_args(model)
    assert kv["kv_size_multiplier"] == world
    for layer in model.model.layers:          # every replica of the kv head carries the same (summed) bias gradient
        qkv = layer.self_attn.qkv_proj
        g = qkv.bias_qkv.grad[qkv.q_output_size_per_partition:] if fuse_qkv else torch.cat([qkv.bias_k.grad, qkv.bias_v.grad])
        reps = [torch.empty_like(g) for _ in range(world)]
        torch.distributed.all_gather(reps, g.contiguous())
        assert all(torch.equal(r, reps[0]) for r in reps)
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(p.grad)
    grads = hf_compat.nxd_to_hf_state_dict(hf_compat.gather_full_state_dict(model), cfg, **kv)
    want = {n: p.grad for n, p in hf.named_parameters()}
    assert set(grads) == set(want)
    for n, g in want.items():
        err = float((grads[n] - g).abs().max())
        assert err <= 1e-5 * max(1.0, float(g.abs().max())), (n, err)


@pytest.mark.parametrize("fuse_qkv", [True, False])
@pytest.mark.parametrize("world", [1, 2])
def test_qwen2_training_step_grads(world, fuse_qkv):
    """TP 2 + SP with the kv head replicated on both ranks: q / k / v weight and bias gradients (and every other one)
    equal transformers' fp32 gradients, as the TP 1 model's do."""
    run_distributed(_train_step, world, fuse_qkv, timeout=300)
