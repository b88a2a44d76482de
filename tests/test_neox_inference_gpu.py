"""GPT-NeoX / Pythia serving on the H100 kernels: ``decode_rope_kv`` at a rotary width R < head_dim (partial rotary), the
decode GEMV's bias / GELU / residual epilogue against float64, and ``GPTNeoXForInference`` generating on the kernels at
head_dim 64 / 80 / 96 / 128 (D = 256 on the torch attention path) with bf16 and e4m3 caches."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_speculation_attention_cpu import medusa_tree  # noqa: E402

pytestmark = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert torch.cuda.is_available() and ops.extension_available(), ops._ext.load_error()
    return ops._ext


# ---- decode_rope_kv at R < D -----------------------------------------------------------------------------------------------
def _windows():
    mask, depth = medusa_tree("cuda")
    return (("decode", None), ("chain", None), ("tree", (mask, depth)))


@pytest.mark.parametrize("rolling", (False, True))
@pytest.mark.parametrize("kv", ("bf16", "e4m3"))
@pytest.mark.parametrize("D", (64, 80, 96, 128, 256))
def test_decode_rope_kv_partial_rotary(_ext, D, kv, rolling):
    """Dims [0, R) of q_out and of the cache rows: ``ops.rope.rotate`` of the first R dims; dims [R, D): the input bit for bit
    (bf16) or ``KVCacheManager``'s quantisation of it (e4m3); v as before.  q / k / v are strided views of [B, W, H, 3D]."""
    from neuronx_distributed_b200 import ops
    from neuronx_distributed_b200.inference.kv_cache import KVCacheManager
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    e, dev = _ext.ext(), torch.device("cuda")
    B, H, L, n_pos = 3, 4, 48, 160
    scale = 0.05
    kvm = KVCacheManager(1, B, L, H, D, dtype=torch.bfloat16, device=dev,
                         kv_quant=KVQuantizationConfig(scale=scale) if kv == "e4m3" else None)
    g = torch.Generator(device="cuda").manual_seed(D)
    for R in sorted({16, 20, 24, 32, D} & set(range(2, D + 1, 2))):
        cos, sin = ops.rope.rope_tables(n_pos, R, 10000.0, dev)
        for name, tree in _windows():
            W = 1 if name == "decode" else (tree[1].numel() if tree is not None else 5)
            depth = tree[1] if tree is not None else None
            pos = torch.tensor([40, 3, 100], device=dev) if rolling else torch.tensor([0, L - W - 7, L - W], device=dev)
            qkv = torch.randn(B, W, H, 3 * D, device=dev, generator=g).to(torch.bfloat16)
            q, k, v = qkv.split(D, dim=-1)
            kc, vc = torch.zeros_like(kvm.k[0]), torch.zeros_like(kvm.v[0])
            kw = {"k_scale": scale, "v_scale": scale} if kv == "e4m3" else {}
            q_out = e.decode_rope_kv(q, k, v, pos, cos, sin, kc, vc, depth=depth, rolling=rolling, **kw)
            d = torch.arange(W, device=dev) if depth is None else depth
            rp = (pos[:, None] + d[None]).clamp(max=(n_pos if rolling else L) - 1)
            c, s = cos[rp], sin[rp]                                                     # [B, W, R/2]
            slot = pos[:, None] + torch.arange(W, device=dev)[None]
            slot = slot % L if rolling else slot.clamp(max=L - 1)
            b = torch.arange(B, device=dev)[:, None]
            krow, vrow = kc[b, slot], vc[b, slot]                                       # [B, W, H, D] as stored
            what = (D, R, kv, name, rolling)
            # q: bf16 rows
            torch.testing.assert_close(q_out[..., :R].float(), ops.rope.rotate(q[..., :R], c, s).float(), atol=2e-2, rtol=2e-2,
                                       msg=str(what))
            assert torch.equal(q_out[..., R:], q[..., R:]), what
            k_rot = ops.rope.rotate(k[..., :R], c, s)
            if kv == "bf16":
                torch.testing.assert_close(krow[..., :R].float(), k_rot.float(), atol=2e-2, rtol=2e-2, msg=str(what))
                assert torch.equal(krow[..., R:], k[..., R:]), what
                assert torch.equal(vrow, v), what
            else:
                torch.testing.assert_close(krow[..., :R].float() * scale, k_rot.float(), atol=2e-2, rtol=7e-2, msg=str(what))
                assert torch.equal(krow[..., R:].view(torch.uint8), kvm._q(k[..., R:]).view(torch.uint8)), what
                assert torch.equal(vrow.view(torch.uint8), kvm._q(v).view(torch.uint8)), what


def test_decode_rope_kv_rejects_bad_tables(_ext):
    """A table wider than D / 2 and cos / sin of different widths raise."""
    e, dev, D = _ext.ext(), torch.device("cuda"), 80
    q, k, v = torch.randn(2, 1, 4, 3 * D, device=dev).to(torch.bfloat16).split(D, dim=-1)
    kc = torch.zeros(2, 32, 4, D, device=dev, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    pos = torch.zeros(2, dtype=torch.long, device=dev)
    for cw, sw in ((D // 2 + 1, D // 2 + 1), (8, 6)):
        cos, sin = torch.ones(64, cw, device=dev), torch.ones(64, sw, device=dev)
        with pytest.raises(RuntimeError):
            e.decode_rope_kv(q, k, v, pos, cos, sin, kc, vc)


# ---- the GEMV epilogue -----------------------------------------------------------------------------------------------------
def _gelu64(h, act):
    if act == 0:
        return h
    if act == 1:
        return 0.5 * h * (1 + torch.erf(h / 2 ** 0.5))
    return 0.5 * h * (1 + torch.tanh(0.7978845608028654 * (h + 0.044715 * h ** 3)))


@pytest.mark.parametrize("N,K", ((7680, 2560), (2560, 2560), (10240, 2560), (2560, 10240), (2304, 6144), (3072, 6144)))
def test_gemv_bias_act_epilogue_vs_float64(_ext, N, K):
    """y = act(x·Wᵀ + b) + r with one bf16 rounding, against float64: per element, the fp32 accumulation bound
    K·2⁻²⁴·Σ|x||w| carried through the activation (slope ≤ 1.13), the activation's own error (the hardware tanh: 2⁻¹⁰·|h|) and
    the final bf16 rounding (2⁻⁸ of the result)."""
    e = _ext.ext()
    g = torch.Generator(device="cuda").manual_seed(N + K)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    b = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    for M in range(1, 9):
        x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        r = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
        h = x.double() @ w.double().t() + b.double()
        acc = K * 2.0 ** -24 * (x.double().abs() @ w.double().abs().t() + b.double().abs())
        for act in (1, 2):
            for res in (None, r):
                y = e.gemv(x, w, res, bias=b, act=act)
                want = _gelu64(h, act) + (0 if res is None else r.double())
                bound = 1.13 * acc + (2.0 ** -10 * h.abs() if act == 2 else 1e-6 * h.abs()) + 2.0 ** -8 * want.abs() + 1e-30
                err = (y.double() - want).abs()
                assert bool((err <= bound).all()), (M, N, K, act, res is None, float((err / bound).max()))
        # the plain kernel is unchanged by the new arguments' defaults
        assert torch.equal(e.gemv(x, w, r), e.gemv(x, w, r, bias=None, act=0))


def test_gemv_epilogue_through_ops_gemm(_ext):
    from neuronx_distributed_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(3, 512, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(1024, 512, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    b = torch.randn(1024, device="cuda", generator=g).to(torch.bfloat16)
    _ext.reset_launches()
    y = ops.gemm.linear_nt(x.view(3, 1, 512), w, b, ops.gemm.GEMV_ACT["gelu_fast"])
    assert _ext.launches() == 1 and y.shape == (3, 1, 1024)
    assert torch.equal(y.view(3, 1024), _ext.ext().gemv(x, w, None, bias=b, act=2))
    with pytest.raises(RuntimeError):
        _ext.ext().gemv(x, w, None, bias=b, act=3)


# ---- the model -------------------------------------------------------------------------------------------------------------
def _model(D, kv_fp8, layers=2, H=8):
    from test_kv_fp8_gpu import _one_rank_model_parallel

    from neuronx_distributed_b200.models.gpt_neox import GPTNeoXConfig
    from neuronx_distributed_b200.models.gpt_neox_inference import GPTNeoXForInference
    from neuronx_distributed_b200.quantization import KVQuantizationConfig

    _one_rank_model_parallel()
    cfg = GPTNeoXConfig(vocab_size=1024, hidden_size=H * D, intermediate_size=4 * H * D, num_hidden_layers=layers,
                        num_attention_heads=H, rotary_pct=0.25, max_position_embeddings=512, hidden_act="gelu_fast",
                        initializer_range=0.05, dtype=torch.bfloat16, device=torch.device("cuda", 0))
    torch.manual_seed(0)
    m = GPTNeoXForInference(cfg, batch_size=2, max_seq_len=512, on_device_sampling=False,
                            kv_quant=KVQuantizationConfig(scale=0.3) if kv_fp8 else None).eval()
    with torch.no_grad():                                        # non-zero biases and LayerNorm affines
        for n, p in m.lm.named_parameters():
            if n.endswith("bias") or "layernorm" in n or "layer_norm" in n:
                p.add_(torch.randn_like(p) * 0.05)
    return m


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def _close(a, r, what):
    a, r = a.float(), r.float()
    assert _rel(a, r) < 5e-2, (what, _rel(a, r))
    top2 = r.topk(2, -1).values
    sure = (top2[..., 0] - top2[..., 1]) > 0.05 * r.std()
    assert torch.equal(a.argmax(-1)[sure], r.argmax(-1)[sure]), what


@pytest.mark.parametrize("kv_fp8", (False, True))
@pytest.mark.parametrize("D", (64, 80, 96, 128))
def test_neox_generates_on_the_kernels(_ext, monkeypatch, D, kv_fp8):
    """Every layer of every decode step on ``decode_rope_kv`` + ``decode_attention`` with the expected launches and none of
    the torch RoPE / cache-write / attention paths; a CUDA-graph replay equal to eager; logits close to fp32 torch attention;
    a speculation chain equal to step-by-step decode; a Medusa tree close to the forced torch path."""
    from neuronx_distributed_b200 import ops
    from neuronx_distributed_b200.ops import attention

    layers = 2
    m = _model(D, kv_fp8, layers)
    P, N = 160, 8
    ids = torch.randint(0, 1024, (2, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    last = torch.tensor([P - 1, 120], device="cuda")

    def run(step, toks=None):
        logits = [m.context_encoding(ids, last)]
        out, pos = [logits[0].argmax(-1)], last + 1
        for i in range(N):
            tok = out[-1] if toks is None else toks[:, i]
            logits.append(step(tok.view(2, 1), pos).clone())
            out.append(logits[-1].argmax(-1))
            pos = pos + 1
        return torch.stack(out, 1), logits

    e, calls, launches = _ext.ext(), [], []
    fa, fr = e.decode_attention, e.decode_rope_kv

    def step(tok, pos):
        _ext.reset_launches()
        out = m.token_generation(tok, pos)
        launches.append(_ext.launches())
        return out

    def forbidden(*a, **kw):
        raise AssertionError("a torch path ran at decode")

    monkeypatch.setattr(e, "decode_attention", lambda *a, **kw: calls.append(("attn", a[0].shape[-1], a[1].dtype)) or fa(*a, **kw))
    monkeypatch.setattr(e, "decode_rope_kv", lambda *a, **kw: calls.append(("rope", a[4].shape[-1])) or fr(*a, **kw))
    monkeypatch.setattr(ops.rope, "rotate", forbidden)
    monkeypatch.setattr(m.kv, "write_window", forbidden)
    monkeypatch.setattr(attention, "speculation_attention_torch", forbidden)
    eager_toks, eager_logits = run(step)
    monkeypatch.undo()
    dt = E4M3 if kv_fp8 else torch.bfloat16
    assert calls == [("rope", D * 25 // 200), ("attn", D, dt)] * (layers * N), calls[:4]
    # per layer: QKV, dense, h→4h and 4h→h GEMVs (bias / GELU / residual in their epilogues), the RoPE + append launch and the
    # two-kernel decode attention; per step: the embed_out GEMV
    assert launches == [7 * layers + 1] * N, launches

    # CUDA-graph replay of a decode step: the eager logits bit for bit
    st_tok, st_pos = eager_toks[:, 0].view(2, 1).clone(), last + 1
    m.context_encoding(ids, last)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.token_generation(st_tok, st_pos)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_out = m.token_generation(st_tok, st_pos)

    def replay(tok, pos):
        st_tok.copy_(tok)
        st_pos.copy_(pos)
        graph.replay()
        return st_out

    graph_toks, graph_logits = run(replay)
    assert torch.equal(graph_toks, eager_toks)
    assert all(torch.equal(a, b) for a, b in zip(graph_logits, eager_logits))

    # fp32 torch attention over the same cache
    def fp32(t):
        return t.float() if t.dtype == torch.bfloat16 else t

    with monkeypatch.context() as mp:
        mp.setenv("NXD_DISABLE_OWN_ATTENTION", "1")
        orig = attention.decode_attention
        mp.setattr(attention, "decode_attention",
                   lambda q, k, v, p, sliding_window, k_scale=1.0, v_scale=1.0: orig(
                       q.float(), fp32(k), fp32(v), p, sliding_window=sliding_window, k_scale=k_scale,
                       v_scale=v_scale).to(q.dtype))
        _, ref_logits = run(m.token_generation, eager_toks)
    for i, (a, r) in enumerate(zip(eager_logits, ref_logits)):
        _close(a, r, f"step {i}")

    # a speculation chain on the kernels verifies what step-by-step decode computes
    pos = last + 1
    m.context_encoding(ids, last)
    spec = m.speculation_forward(eager_toks[:, :5], pos).clone()
    _close(spec, torch.stack(eager_logits[1:6], 1), "chain")

    # a Medusa tree on the kernels vs the forced torch path (no kernel scales: RoPE, append and attention in torch)
    mask, depth = medusa_tree("cuda")
    tree_ids = torch.randint(0, 1024, (2, depth.numel()), device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    m.context_encoding(ids, last)
    tree = m.speculation_forward(tree_ids, pos, tree_mask=mask, tree_depth=depth).clone()
    with monkeypatch.context() as mp:
        mp.setattr(m.kv, "kernel_scales", lambda: None)
        m.context_encoding(ids, last)
        tree_ref = m.speculation_forward(tree_ids, pos, tree_mask=mask, tree_depth=depth).clone()
    _close(tree, tree_ref, "tree")


@pytest.mark.parametrize("kv_fp8", (False, True))
def test_neox_head_dim_256_generates_on_torch_attention(_ext, monkeypatch, kv_fp8):
    """Pythia-1b's head size: attention off the kernels (torch path), the GEMVs still on the kernel; agrees with the fully
    torch path (no kernel scales)."""
    from neuronx_distributed_b200.ops import attention

    m = _model(256, kv_fp8, layers=2, H=4)
    P, N = 64, 6
    ids = torch.randint(0, 1024, (2, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    last = torch.tensor([P - 1, 40], device="cuda")

    def run():
        logits = [m.context_encoding(ids, last)]
        pos = last + 1
        for _ in range(N):
            logits.append(m.token_generation(logits[-1].argmax(-1).view(2, 1), pos).clone())
            pos = pos + 1
        return logits

    torch_calls = []
    orig = attention.speculation_attention_torch
    monkeypatch.setattr(attention, "speculation_attention_torch", lambda *a, **kw: torch_calls.append(1) or orig(*a, **kw))
    got = run()
    assert len(torch_calls) == 2 * N
    with monkeypatch.context() as mp:
        mp.setattr(m.kv, "kernel_scales", lambda: None)
        ref = run()
    for i, (a, r) in enumerate(zip(got, ref)):
        _close(a, r, f"step {i}")
