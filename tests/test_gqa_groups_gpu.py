"""Token generation at GQA groups 3, 5, 6 and 7 on the H100 (sm_90a): ``decode_attention``, flash-decoding's local partial
and ``speculation_attention`` run their kernels (``decode_attn_kernel``, ``spec_attn_kernel``) at the geometries of
Llama-3.2-3B (24 / 8 heads), Qwen2.5-14B / 32B (40 / 8), Qwen2.5-1.5B (12 / 2), Qwen2.5-7B (28 / 4, and its TP 4 shard 7 / 1)
and Qwen2.5-0.5B (14 / 2, head_dim 64), checked slot by slot with the probes of ``test_decode_probes_cpu.py``.  When G does
not divide 64, a token's G query rows can straddle two 64-row tiles of the verification kernel; the W = 10 and W = 64
windows at G = 7 put tokens across every tile boundary.  Then a Llama model with G = 7, q / k / v bias and Llama-3 RoPE
serves prefill, 16 decode steps and a speculation round on the kernels, against the torch attention path."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_decode_probes_cpu as probes  # noqa: E402
from test_decode_probes_cpu import (TILE, Case, check_planted, check_random, check_visibility,  # noqa: E402
                                    check_visibility_partial, decode_run, partial_run, spec_run)

pytestmark = pytest.mark.gpu

CACHES = ("bf16", "e4m3")
DIMS = (64, 80, 96, 128)
GROUPS = (3, 5, 6, 7)


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def spec_ranges(p, L, W, G, depth, window, splits, rolling, rt):
    """``spec_attn_kernel``'s split ranges of row tile ``rt`` when G need not divide 64: a token counts in every tile that
    holds one of its rows, so the tile's last token is rounded up."""
    w_lo, w_hi = rt * TILE // G, min((rt * TILE + TILE + G - 1) // G, W)
    dmin = min(int(depth[w]) for w in range(w_lo, w_hi))
    lo_l = min(p, p + dmin - window + 1) if window > 0 else 0
    lo = max(lo_l, 0) if rolling else min(max(lo_l, 0), L)
    hi = max(p + W, lo) if rolling else max(min(p + W, L), lo)
    per = ((hi - lo + splits - 1) // splits + TILE - 1) // TILE * TILE
    return [(lo + s * per, min(hi, lo + s * per + per)) for s in range(splits)]


@pytest.fixture(autouse=True)
def _tile_rule(monkeypatch):
    monkeypatch.setattr(probes, "spec_ranges", spec_ranges)       # the probes plant at the kernel's split edges


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def counted(_ext, run, per_call=2):
    """``run`` that asserts each call went through the extension's kernels (the attention kernel and a combine)."""
    def wrapped(*a):
        n0 = _ext.launches()
        out = run(*a)
        assert _ext.launches() == n0 + per_call, "fell back to the torch path"
        return out
    return wrapped


def _id(c):
    return c.name


# ---- one-token decode -----------------------------------------------------------------------------------------------------
DECODE = [
    Case("llama3.2-3b-8k", H=24, Hkv=8, D=128, L=8192, pos=(4999, 8191)),
    Case("llama3.2-3b-32k", H=24, Hkv=8, D=128, L=32768, pos=(32767,)),
    Case("qwen2.5-14b-32k", H=40, Hkv=8, D=128, L=32768, pos=(20000, 32767)),
    Case("qwen2.5-14b-sw4096", H=40, Hkv=8, D=128, L=32768, pos=(30000,), window=4096),
    Case("qwen2.5-1.5b", H=12, Hkv=2, D=128, L=4096, pos=(0, 2047, 4095)),
    Case("qwen2.5-7b", H=28, Hkv=4, D=128, L=4096, pos=(1, 3000)),
    Case("qwen2.5-7b-sw300", H=28, Hkv=4, D=128, L=4096, pos=(299, 4095), window=300),
    Case("qwen2.5-7b-rolling", H=28, Hkv=4, D=128, L=4160, pos=(9000,), window=4096, rolling=True),
    Case("qwen2.5-7b-tp4", H=7, Hkv=1, D=128, L=32768, pos=(1024, 32767)),
    Case("qwen2.5-7b-tp4-rolling", H=7, Hkv=1, D=128, L=512, pos=(100, 1535), window=300, rolling=True),
    Case("qwen2.5-0.5b", H=14, Hkv=2, D=64, L=4096, pos=(5, 4095)),
    Case("qwen2.5-0.5b-sw300", H=14, Hkv=2, D=64, L=4096, pos=(300, 4095), window=300),
]
DECODE += [Case(f"grid-d{D}-g{G}" + ("-sw300" if sw else ""), H=2 * G, Hkv=2, D=D, L=1024, pos=(0, 150, 700, 1023),
                window=sw) for D in DIMS for G in GROUPS for sw in (0, 300)]
DECODE += [Case(f"grid-rolling-d{D}-g{G}", H=2 * G, Hkv=2, D=D, L=512, pos=(100, 600, 1535), window=300, rolling=True)
           for D in DIMS for G in (3, 7)]
# flash-decoding's local positions: before the shard, inside it and past its end
PARTIAL = [Case(f"local-d{D}-g{G}", H=2 * G, Hkv=2, D=D, L=512, pos=(-40, -1, 0, 63, 511, 512, 700), window=sw)
           for D in DIMS for G in GROUPS for sw in (0, 100)]


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", DECODE, ids=_id)
def test_decode_probes(_ext, case, cache):
    """Visibility sums (bf16 output and the exact fp32 partial), planted slots and float64 with per-element bounds."""
    run = counted(_ext, decode_run(case))
    check_visibility(case, cache, run, "cuda")
    if not case.rolling:
        check_visibility_partial(case, cache, counted(_ext, partial_run(case)), "cuda")
    check_planted(case, cache, run, "cuda", sms(), spec=False)
    check_random(case, cache, run, "cuda", sms(), spec=False)


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", PARTIAL, ids=_id)
def test_partial_probes_at_local_positions(_ext, case, cache):
    check_visibility_partial(case, cache, counted(_ext, partial_run(case)), "cuda")
    check_planted(case, cache, counted(_ext, partial_run(case)), "cuda", sms(), spec=False, partial=True)


# ---- verification of W tokens ---------------------------------------------------------------------------------------------
SPEC = [
    Case("llama3.2-3b-chain5", H=24, Hkv=8, D=128, L=8192, pos=(3000, 8187), W=5),
    Case("llama3.2-3b-medusa-sw", H=24, Hkv=8, D=128, L=8192, pos=(300, 8182), W=10, window=300, tree="medusa"),
    Case("qwen2.5-14b-medusa", H=40, Hkv=8, D=128, L=4096, pos=(1024,), W=10, tree="medusa"),
    Case("qwen2.5-14b-w64", H=40, Hkv=8, D=128, L=4096, pos=(4032,), W=64),           # W·G = 320: 5 row tiles
    Case("qwen2.5-1.5b-random64", H=12, Hkv=2, D=128, L=2048, pos=(0, 1500), W=64, tree="random"),
    Case("qwen2.5-1.5b-chain5-sw", H=12, Hkv=2, D=128, L=32768, pos=(20000,), W=5, window=4096),
    # G = 7: tokens 9, 18, 27, 36, 45 and 54 straddle the tile boundaries
    Case("qwen2.5-7b-chain10", H=28, Hkv=4, D=128, L=4096, pos=(1000, 4086), W=10),
    Case("qwen2.5-7b-chain10-sw10", H=28, Hkv=4, D=128, L=4096, pos=(9, 3000), W=10, window=10),
    Case("qwen2.5-7b-w64", H=28, Hkv=4, D=128, L=8192, pos=(8128,), W=64),             # W·G = 448: 7 row tiles
    Case("qwen2.5-7b-w64-sw64", H=28, Hkv=4, D=128, L=8192, pos=(63, 5000), W=64, window=64),
    Case("qwen2.5-7b-random64-sw64", H=28, Hkv=4, D=128, L=4096, pos=(2000,), W=64, window=64, tree="random"),
    Case("qwen2.5-7b-medusa-sw10", H=28, Hkv=4, D=128, L=4096, pos=(1, 2000), W=10, window=10, tree="medusa"),
    Case("qwen2.5-7b-tp4-w64", H=7, Hkv=1, D=128, L=2048, pos=(500, 1984), W=64),
    Case("qwen2.5-7b-tp4-random64", H=7, Hkv=1, D=128, L=2048, pos=(700,), W=64, window=200, tree="random"),
    Case("qwen2.5-7b-tp4-rolling-w63", H=7, Hkv=1, D=128, L=4158, pos=(3 * 4158 + 100,), W=63, window=4096, rolling=True),
    Case("qwen2.5-7b-rolling-medusa", H=28, Hkv=4, D=128, L=4105, pos=(5000, 9000), W=10, window=4096, rolling=True,
         tree="medusa"),
    Case("qwen2.5-0.5b-medusa-sw", H=14, Hkv=2, D=64, L=4096, pos=(300, 4086), W=10, window=300, tree="medusa"),
    Case("qwen2.5-0.5b-random64", H=14, Hkv=2, D=64, L=1024, pos=(700,), W=64, window=200, tree="random"),
]
SPEC += [Case(f"grid-d{D}-g{G}-" + (tree or "chain") + ("-sw200" if sw else ""), H=2 * G, Hkv=2, D=D, L=1024,
              pos=(0, 500, 1019), W=5 if tree is None else (10 if tree == "medusa" else 12), window=sw, tree=tree)
         for D in DIMS for G in GROUPS for tree, sw in ((None, 0), ("medusa", 200), ("random", 0))]
SPEC += [Case(f"grid-w64-d{D}-g{G}-sw64", H=2 * G, Hkv=2, D=D, L=1024, pos=(63, 960), W=64, window=64)
         for D in DIMS for G in GROUPS]
SPEC += [Case(f"grid-rolling-d{D}-g{G}", H=2 * G, Hkv=2, D=D, L=512, pos=(100, 1400), W=5, window=508, rolling=True)
         for D in DIMS for G in (3, 7)]


@pytest.mark.parametrize("cache", CACHES)
@pytest.mark.parametrize("case", SPEC, ids=_id)
def test_spec_probes(_ext, case, cache):
    run = counted(_ext, spec_run(case))
    check_visibility(case, cache, run, "cuda")
    check_planted(case, cache, run, "cuda", sms(), spec=True)
    check_random(case, cache, run, "cuda", sms(), spec=True)


def test_groups_past_8_stay_on_the_torch_path(_ext):
    """G = 16 (Llama-3.1-405B at TP 8): no kernel is compiled for it; the torch path serves it."""
    from neuronx_distributed_b200.ops import attention

    q = torch.randn(1, 1, 16, 128, device="cuda", dtype=torch.bfloat16)
    kc = torch.randn(1, 256, 1, 128, device="cuda", dtype=torch.bfloat16)
    pos = torch.tensor([200], device="cuda")
    n0 = _ext.launches()
    got = attention.decode_attention(q, kc, kc, pos, scale=0.125)
    assert _ext.launches() == n0
    assert torch.equal(got, attention.speculation_attention_torch(q, kc, kc, pos, scale=0.125))


# ---- a model ------------------------------------------------------------------------------------------------------------
def test_model_g7_qkv_bias_llama3_rope_on_the_kernels(_ext, monkeypatch):
    """14 / 2 heads of head_dim 64 (Qwen2.5-0.5B's attention), q / k / v bias and Llama-3 RoPE, bf16: prefill, 16 greedy
    decode steps and a 10-node Medusa verification on the kernels, against the same model with token-generation attention
    on ``speculation_attention_torch``, fed the same tokens.  Both read one bf16 cache and differ in the order of fp32 sums
    and in where P is rounded to bf16, so the logits agree to 2 % of their largest magnitude and the confident argmaxes
    agree."""
    from test_kv_fp8_gpu import _one_rank_model_parallel
    from test_speculation_attention_cpu import medusa_tree

    from neuronx_distributed_b200.models.llama import LlamaConfig
    from neuronx_distributed_b200.models.llama_inference import LlamaForInference
    from neuronx_distributed_b200.ops import attention

    _one_rank_model_parallel()
    cfg = LlamaConfig(vocab_size=1024, hidden_size=896, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=14,
                      num_key_value_heads=2, max_position_embeddings=512, rope_theta=1e6, qkv_bias=True,
                      rope_scaling={"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                    "original_max_position_embeddings": 64},
                      dtype=torch.bfloat16, device=torch.device("cuda", 0))
    torch.manual_seed(0)
    m = LlamaForInference(cfg, batch_size=2, max_seq_len=512, on_device_sampling=False).eval()
    with torch.no_grad():
        for layer in m.lm.model.layers:
            layer.self_attn.qkv_proj.bias_qkv.normal_(0.0, 0.5)
    P, N = 200, 16
    g = torch.Generator(device="cuda").manual_seed(6)
    ids = torch.randint(0, 1024, (2, P), device="cuda", generator=g)
    last = torch.tensor([P - 1, 150], device="cuda")
    mask, depth = (t.cuda() for t in medusa_tree())
    tree_ids = torch.randint(0, 1024, (2, mask.shape[0]), device="cuda", generator=g)

    def run(toks=None):
        logits = [m.context_encoding(ids, last)]
        out, pos = [logits[0].argmax(-1)], last + 1
        for i in range(N):
            tok = out[-1] if toks is None else toks[:, i]
            logits.append(m.token_generation(tok.view(2, 1), pos).clone())
            out.append(logits[-1].argmax(-1))
            pos = pos + 1
        logits.append(m.speculation_forward(tree_ids, pos, tree_mask=mask, tree_depth=depth).float())
        return torch.stack(out, 1), logits

    n0 = _ext.launches()
    e, calls = _ext.ext(), []
    for name in ("decode_attention", "speculation_attention"):
        fn = getattr(e, name)
        monkeypatch.setattr(e, name, lambda *a, _fn=fn, _n=name, **kw: calls.append(_n) or _fn(*a, **kw))
    toks, kern = run()
    monkeypatch.undo()
    assert calls == ["decode_attention"] * (2 * N) + ["speculation_attention"] * 2     # every layer on the kernels
    assert _ext.launches() > n0

    torch_path = attention.speculation_attention_torch
    monkeypatch.setattr(attention, "decode_attention", lambda q, kc, vc, pos, scale=None, sliding_window=None, **kw:
                        torch_path(q, kc, vc, pos, sliding_window=sliding_window, scale=scale, **kw))
    monkeypatch.setattr(attention, "speculation_attention", torch_path)
    _, ref = run(toks[:, :N])
    for i, (a, r) in enumerate(zip(kern, ref)):
        a, r = a.float(), r.float()
        err = float((a - r).abs().max() / r.abs().max())
        assert err < 2e-2, (i, err)
        top2 = r.topk(2, -1).values
        sure = (top2[..., 0] - top2[..., 1]) > 0.05 * r.std()
        assert torch.equal(a.argmax(-1)[sure], r.argmax(-1)[sure]), i
