"""Attention dropout off the GPU: the host Philox4x32-10 and the keep rule of ``ops.attention.attention_dropout_keep``, the
explicit-softmax path that applies it, and the BERT / GPT-NeoX
wiring (tensor-parallel head offsets, activation checkpointing, the pre-training example)."""
import math
import os
import subprocess
import sys

import pytest
import torch

from dist_utils import run_distributed

from neuronx_distributed_b200.ops import attention

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32-10."""
    cases = [((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
              "d16cfe09 94fdcceb 5001e420 24126ea1")]
    for counter, key, want in cases:
        assert " ".join(f"{int(w):08x}" for w in attention.philox4x32_10(counter, key)) == want


def test_keep_rule_is_the_documented_function_of_the_coordinates():
    seed, p = 0x123456789ABCDEF, 0.3
    keep = attention.attention_dropout_keep(seed, 2, 3, 40, 50, p)
    t = attention.dropout_keep_threshold(p)
    for b, h, i, j in [(0, 0, 0, 0), (1, 2, 39, 49), (0, 1, 8, 9), (1, 0, 17, 30), (0, 2, 24, 8)]:
        words = attention.philox4x32_10((j & ~8, i & ~8, h, b), (seed & 0xFFFFFFFF, seed >> 32))
        assert bool(keep[b, h, i, j]) == (int(words[2 * ((i >> 3) & 1) + ((j >> 3) & 1)]) < t)
    # independent of the shape asked for, and head h of a call at head_offset o is global head o + h
    assert torch.equal(attention.attention_dropout_keep(seed, 2, 3, 23, 17, p), keep[:, :, :23, :17])
    assert torch.equal(attention.attention_dropout_keep(seed, 2, 2, 40, 50, p, head_offset=1), keep[:, 1:])
    assert torch.equal(attention.attention_dropout_keep(torch.tensor([seed]), 2, 3, 40, 50, p), keep)
    assert attention.dropout_keep_threshold(0.0) == 2 ** 32 - 1 and attention.dropout_keep_threshold(0.5) == 2 ** 31


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_kept_fraction_within_binomial_bounds(p):
    keep = attention.attention_dropout_keep(20240601, 2, 4, 256, 256, p)
    n = keep.numel()
    frac = keep.float().mean().item()
    assert abs(frac - (1 - p)) < 6 * math.sqrt(p * (1 - p) / n), frac
    # every one of the four words of a block is used: each quarter of the 16 × 16 pattern keeps about 1 − p
    for di in (0, 8):
        for dj in (0, 8):
            sub = keep.view(2, 4, 16, 16, 16, 16)[:, :, :, di:di + 8, :, dj:dj + 8]
            assert abs(sub.float().mean().item() - (1 - p)) < 6 * math.sqrt(p * (1 - p) / sub.numel())


def _reference(q, k, v, causal, scale, mask, window, p, seed, head_offset=0):
    """float64 attention with the host rule's dropout mask; a row that sees no key gives 0."""
    B, S, H, D = q.shape
    Skv, Hkv = k.shape[1], k.shape[2]
    qt, kt, vt = (t.double().transpose(1, 2) for t in (q, k, v))
    kt, vt = kt.repeat_interleave(H // Hkv, 1), vt.repeat_interleave(H // Hkv, 1)
    vis = torch.ones(B, 1, S, Skv, dtype=torch.bool)
    if mask is not None:
        vis = vis & mask[:, None, None, :]
    if causal:
        vis = vis & attention.window_visibility(S, Skv, window)
    s = (qt @ kt.transpose(-1, -2) * scale).masked_fill(~vis, float("-inf"))
    probs = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
    probs = probs * attention.attention_dropout_keep(seed, B, H, S, Skv, p, head_offset).double() / (1 - p)
    return (probs @ vt).transpose(1, 2)


@pytest.mark.parametrize("case", ["plain", "masked", "causal", "window"])
def test_fallback_matches_float64_reference(case):
    torch.manual_seed(0)
    B, S, H, Hkv, D, p, seed = 2, 40, 4, 2, 16, 0.3, 987654321
    q, k, v = (torch.randn(B, S, h, D, requires_grad=True) for h in (H, Hkv, Hkv))
    mask = None
    if case == "masked":
        mask = torch.ones(B, S, dtype=torch.bool)
        mask[0, 30:] = False
        mask[1, :] = False                                 # a batch that sees no key at all: O = 0, gradients 0
    causal = case in ("causal", "window")
    window = 9 if case == "window" else None
    scale = 1 / math.sqrt(D)
    out = attention.flash_attention(q, k, v, causal=causal, key_padding_mask=mask, sliding_window=window, dropout_p=p,
                                    dropout_seed=seed, head_offset=3)
    q64, k64, v64 = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref = _reference(q64, k64, v64, causal, scale, mask, window, p, seed, head_offset=3)
    torch.testing.assert_close(out.double(), ref, rtol=1e-5, atol=1e-5)
    go = torch.randn_like(out)
    g = torch.autograd.grad(out, (q, k, v), go)
    g_ref = torch.autograd.grad(ref, (q64, k64, v64), go.double())
    for a, r in zip(g, g_ref):
        torch.testing.assert_close(a.double(), r, rtol=1e-4, atol=1e-5)
    if case == "masked":
        assert out[1].abs().max() == 0 and g[0][1].abs().max() == 0
    # a different seed drops differently; p = 0.5 with one seed is not the result of p = 0.3
    assert not torch.allclose(out, attention.flash_attention(q, k, v, causal=causal, key_padding_mask=mask,
                                                             sliding_window=window, dropout_p=p, dropout_seed=seed + 1,
                                                             head_offset=3))


def test_zero_dropout_is_todays_path_and_arguments_are_checked():
    torch.manual_seed(1)
    q, k, v = (torch.randn(2, 24, 4, 32) for _ in range(3))
    mask = torch.rand(2, 24) > 0.2
    for causal, m in ((True, None), (False, mask)):
        want = attention._sdpa(q, k, v, causal, 1 / math.sqrt(32), m)
        assert torch.equal(attention.flash_attention(q, k, v, causal=causal, key_padding_mask=m, dropout_p=0.0), want)
        assert torch.equal(attention.flash_attention(q, k, v, causal=causal, key_padding_mask=m, dropout_p=0.0,
                                                     dropout_seed=5, head_offset=2), want)
    for bad in (-0.1, 1.0, 1.5):
        with pytest.raises(ValueError):
            attention.flash_attention(q, k, v, dropout_p=bad)
    # without a seed one is drawn from the default generator: the same generator state gives the same output
    torch.manual_seed(7)
    a = attention.flash_attention(q, k, v, dropout_p=0.2)
    torch.manual_seed(7)
    assert torch.equal(attention.flash_attention(q, k, v, dropout_p=0.2), a)


def _bert_tp(rank, world, out_path):
    """BERT-tiny (4 heads) in train mode with attention dropout 0.1 and no hidden dropout: loss and gradients."""
    from neuronx_distributed_b200.models import bert, hf_compat
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.mappings import gather_from_tensor_model_parallel_region as gather

    transformers = pytest.importorskip("transformers")
    ps.initialize_model_parallel(world)
    torch.manual_seed(0)
    kw = dict(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
              max_position_embeddings=32)
    hf = transformers.BertForPreTraining(transformers.BertConfig(**kw, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0))
    m = bert.BertForPreTraining(bert.BertConfig(**kw, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.1,
                                                dtype=torch.float32))
    hf_compat.load_hf_checkpoint(m, hf.state_dict())
    gen = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 64, (3, 20), generator=gen)
    am = torch.ones(3, 20, dtype=torch.long)
    am[1, 15:] = 0
    labels = torch.where(torch.rand(3, 20, generator=gen) < 0.3, ids, torch.full_like(ids, -100))
    nsp = torch.tensor([0, 1, 1])
    res = {}
    for mode in ("train", "eval"):
        m.train(mode == "train")
        m.zero_grad()
        torch.manual_seed(42)                              # the same seed draw on every rank, as parallel_state seeds TP groups
        loss, _ = m(ids, torch.zeros_like(ids), am, labels, nsp)
        loss.backward()
        res[mode] = dict(loss=loss.detach(), pos=m.bert.embeddings.position_embeddings.weight.grad.clone(),
                         query=gather(m.bert.layers[0].attention.query.weight.grad.t().contiguous()).t().contiguous(),
                         value=gather(m.bert.layers[1].attention.value.weight.grad.t().contiguous()).t().contiguous())
    if rank == 0:
        torch.save(res, out_path)


def test_bert_attention_dropout_tp2_equals_tp1(tmp_path):
    pytest.importorskip("transformers")
    run_distributed(_bert_tp, 1, str(tmp_path / "tp1.pt"))
    run_distributed(_bert_tp, 2, str(tmp_path / "tp2.pt"))
    one, two = torch.load(tmp_path / "tp1.pt"), torch.load(tmp_path / "tp2.pt")
    for mode in ("train", "eval"):
        for key in one[mode]:
            torch.testing.assert_close(two[mode][key], one[mode][key], rtol=1e-5, atol=1e-6, msg=f"{mode} {key}")
    assert not torch.allclose(one["train"]["loss"], one["eval"]["loss"])     # the dropout is on in train mode only


def _neox_checkpointing(rank, world, out_path):
    from neuronx_distributed_b200.models.gpt_neox import GPTNeoXConfig, GPTNeoXForCausalLM
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(world)
    res = {}
    for ac in ("none", "full"):
        torch.manual_seed(0)
        cfg = GPTNeoXConfig(vocab_size=64, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128,
                            max_position_embeddings=32, attention_dropout=0.2, activation_checkpointing=ac, dtype=torch.float32)
        m = GPTNeoXForCausalLM(cfg).train()
        ids = torch.randint(0, 64, (2, 24), generator=torch.Generator().manual_seed(3))
        torch.manual_seed(11)
        loss, _ = m(ids, labels=ids)
        loss.backward()
        res[ac] = (loss.detach(), {n: p.grad.clone() for n, p in m.named_parameters()})
        m.eval()
        with torch.no_grad():
            _, logits = m(ids)
        res[ac + "_eval"] = logits
    if rank == 0:
        torch.save(res, out_path)


def test_gpt_neox_attention_dropout_under_activation_checkpointing(tmp_path):
    """``activation_checkpointing="full"`` recomputes each layer with the default generator restored, so the recomputed
    attention draws the same seed and drops the same elements: the gradients equal those without checkpointing."""
    run_distributed(_neox_checkpointing, 1, str(tmp_path / "neox.pt"))
    res = torch.load(tmp_path / "neox.pt")
    (l0, g0), (l1, g1) = res["none"], res["full"]
    assert torch.equal(l0, l1)
    for n in g0:
        torch.testing.assert_close(g1[n], g0[n], rtol=1e-6, atol=1e-7, msg=n)
    assert torch.equal(res["none_eval"], res["full_eval"])


def test_bert_example_runs_with_dropout():
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29761", os.path.join(ROOT, "examples", "training", "bert", "tp_dp_bert_pretrain.py"),
                        "--model", "tiny", "--tensor_parallel_size", "2", "--batch_size", "4", "--seq_len", "32",
                        "--max_steps", "2", "--dropout", "0.1"], env=env, text=True, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "step 2 loss" in r.stdout
