"""GPT-NeoX / Pythia serving (``models.gpt_neox_inference``) on CPU against ``transformers.GPTNeoXForCausalLM`` with the same
random weights: greedy tokens and logits over prefill + 16 decode steps at TP = 1 and 2, speculation chains and Medusa trees
against step-by-step decode, the HF config spellings, and the ``run_hf.py --family gpt_neox`` demo."""
import os
import subprocess
import sys

import pytest
import torch

from dist_utils import run_distributed

transformers = pytest.importorskip("transformers")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S, STEPS, B = 7, 16, 2

# (use_parallel_residual, rotary_pct, head_dim, hidden_act): partial and full rotary, D = 80 with R = 20, both GELU forms
CASES = [(True, 0.25, 32, "gelu"), (False, 1.0, 32, "gelu_fast"), (True, 0.25, 80, "gelu_fast"), (False, 0.25, 80, "gelu")]


def _hf(par, pct, D, act, seed=0):
    torch.manual_seed(seed)
    H = 4
    hc = transformers.GPTNeoXConfig(vocab_size=96, hidden_size=H * D, intermediate_size=2 * H * D, num_hidden_layers=2,
                                    num_attention_heads=H, rotary_pct=pct, hidden_act=act, use_parallel_residual=par,
                                    max_position_embeddings=64, attn_implementation="eager", initializer_range=0.2)
    return hc, transformers.GPTNeoXForCausalLM(hc).eval()


def _serve(hc, hf, **kw):
    from neuronx_distributed_b200.models import hf_compat
    from neuronx_distributed_b200.models.gpt_neox_inference import GPTNeoXForInference

    cfg = hf_compat.config_from_hf(hc, dtype=torch.float32)
    srv = GPTNeoXForInference(cfg, batch_size=B, max_seq_len=48, on_device_sampling=False, **kw).eval()
    res = hf_compat.load_hf_checkpoint(srv, hf.state_dict())
    assert not res.missing_keys and not res.unexpected_keys, res
    return srv


def _parity(rank, world):
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.mappings import gather_from_tensor_model_parallel_region as gather

    ps.initialize_model_parallel(world)
    for case in CASES:
        hc, hf = _hf(*case)
        prompt = torch.randint(0, 96, (B, S), generator=torch.Generator().manual_seed(1))
        full = prompt
        with torch.no_grad():                                   # HF greedy decode, full forward per step (no EOS / padding)
            for _ in range(STEPS + 1):
                full = torch.cat([full, hf(full).logits[:, -1].argmax(-1, keepdim=True)], 1)       # [B, S + 17]
            want = hf(full).logits                                                                  # [B, S + 17, V]
        srv = _serve(hc, hf)
        lg = gather(srv.context_encoding(prompt, torch.full((B,), S - 1)))
        got = [lg]
        for i in range(STEPS):
            got.append(gather(srv.token_generation(full[:, S + i].view(B, 1), torch.full((B,), S + i))))
        got = torch.stack(got, 1)                                                                   # [B, 17, V]
        err = float((got - want[:, S - 1: S + STEPS]).abs().max())
        assert err < 1e-4, (case, world, err)
        assert torch.equal(got.argmax(-1), full[:, S:]), (case, world)


def test_neox_matches_hf_tp1():
    run_distributed(_parity, 1, timeout=300)


def test_neox_matches_hf_tp2():
    run_distributed(_parity, 2, timeout=300)


def _speculation(rank, world):
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(world)
    hc, hf = _hf(True, 0.25, 80, "gelu_fast")
    srv = _serve(hc, hf)
    g = torch.Generator().manual_seed(3)
    prompt, nxt = torch.randint(0, 96, (B, S), generator=g), torch.randint(0, 96, (B, 4), generator=g)
    pos = torch.full((B,), S)
    # a chain of 4 equals 4 decode steps
    srv.context_encoding(prompt, torch.full((B,), S - 1))
    step = torch.stack([srv.token_generation(nxt[:, w: w + 1], pos + w) for w in range(4)], 1)
    srv.context_encoding(prompt, torch.full((B,), S - 1))
    chain = srv.speculation_forward(nxt, pos)
    assert float((chain - step).abs().max()) < 1e-5
    # a Medusa tree: root 0, children 1 and 2, grandchild 3 under 1 — each node equals the chain of its ancestors
    mask = torch.tensor([[1, 0, 0, 0], [1, 1, 0, 0], [1, 0, 1, 0], [1, 1, 0, 1]], dtype=torch.bool)
    depth = torch.tensor([0, 1, 1, 2])
    srv.context_encoding(prompt, torch.full((B,), S - 1))
    tree, hidden = srv.speculation_forward(nxt, pos, tree_mask=mask, tree_depth=depth, return_hidden=True)
    assert hidden.shape == (B, 4, hc.hidden_size)
    for node, path in enumerate(([0], [0, 1], [0, 2], [0, 1, 3])):
        srv.context_encoding(prompt, torch.full((B,), S - 1))
        ref = srv.speculation_forward(nxt[:, path], pos)[:, -1]
        assert float((tree[:, node] - ref).abs().max()) < 1e-5, node


def test_neox_speculation_chain_and_medusa_tree():
    run_distributed(_speculation, 1, timeout=300)


def _options(rank, world):
    from neuronx_distributed_b200.models import hf_compat
    from neuronx_distributed_b200.models.gpt_neox import GPTNeoXConfig
    from neuronx_distributed_b200.models.gpt_neox_inference import GPTNeoXForInference
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(world)
    cfg = GPTNeoXConfig(vocab_size=64, hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=4,
                        dtype=torch.float32)
    for kw in ({"rolling_kv_cache": True}, {"flash_decoding": True}):
        with pytest.raises(ValueError):
            GPTNeoXForInference(cfg, max_seq_len=32, **kw)
    # legacy Pythia config.json spelling and a transformers-5 config object give the same config
    legacy = {"model_type": "gpt_neox", "vocab_size": 50304, "hidden_size": 2560, "intermediate_size": 10240, "num_hidden_layers": 32,
              "num_attention_heads": 32, "rotary_pct": 0.25, "rotary_emb_base": 10000, "max_position_embeddings": 2048,
              "layer_norm_eps": 1e-5, "use_parallel_residual": True, "hidden_act": "gelu", "tie_word_embeddings": False,
              "torch_dtype": "float16"}
    a = hf_compat.config_from_hf(legacy)
    b = hf_compat.config_from_hf(transformers.GPTNeoXConfig(**{k: v for k, v in legacy.items() if k != "model_type"}))
    assert isinstance(a, GPTNeoXConfig) and a.head_dim == 80 and a.rotary_pct == 0.25 and a.rotary_emb_base == 10000.0
    for f in ("vocab_size", "hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "rotary_pct",
              "rotary_emb_base", "max_position_embeddings", "layer_norm_eps", "use_parallel_residual", "hidden_act"):
        assert getattr(a, f) == getattr(b, f), f
    c = hf_compat.config_from_hf(dict(legacy, rotary_pct=None, rotary_emb_base=None, hidden_act="gelu_fast", use_parallel_residual=False,
                                      rope_parameters={"partial_rotary_factor": 0.5, "rope_theta": 5e5}))
    assert (c.rotary_pct, c.rotary_emb_base, c.hidden_act, c.use_parallel_residual) == (0.5, 5e5, "gelu_fast", False)
    with pytest.raises(ValueError):
        hf_compat.config_from_hf(dict(legacy, tie_word_embeddings=True))


def test_neox_options_and_hf_config():
    run_distributed(_options, 1, timeout=300)


def test_run_hf_gpt_neox_demo():
    env = dict(os.environ, PYTHONPATH=ROOT, MASTER_PORT="29731", NXD_LOG_LEVEL="WARNING", NXD_CPU_MODE="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "inference", "run_hf.py"), "--family", "gpt_neox", "--seq_len", "64"],
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]
    assert "accuracy check vs transformers (greedy, matching prefix): 32/32 tokens" in p.stdout, p.stdout[-3000:]
