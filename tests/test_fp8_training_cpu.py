"""Row-wise scaled FP8 training on CPU: the three products of ``ops.gemm_fp8`` on their emulation path against the float64
definition, and the autograd wiring of ``tp_linear(fp8=True)`` (input, weight and bias gradients, the GQA input-gradient
scale, the ZeRO-1 ``main_grad`` protocol, TP = 2 with sequence parallelism), and which layers ``LlamaConfig.fp8_training``
turns on.  ``test_fp8_training_gpu.py`` checks the kernels against the same rule.

The rule, for a bf16 ``t [R, C]``: ``rows(t)`` = one absmax scale per row (``s_r = max(amax_r / 448, 1e-12)``, codes
``RNE(clamp(t / s, ±448))``), ``cols_t(t) = rows(tᵀ)``.  A linear ``y = x·Wᵀ`` with ``g = dL/dy`` runs

    y  = rows(x) · rows(W)ᵀ         dx = rows(g) · cols_t(W)ᵀ         dW = cols_t(g) · cols_t(x)ᵀ
"""
import pytest
import torch

from dist_utils import run_distributed

from neuronx_distributed_b200.ops import gemm_fp8

BF16 = torch.bfloat16


def _rows64(t):
    """float64 of the dequantised rows(t), by the oracle quantiser."""
    q, s = gemm_fp8._quantize_groups_reference(t, t.shape[1], "absmax", None)
    return q.double() * s.double()


def _cols_t64(t):
    return _rows64(t.t())


def _probe(R, C, e, gen):
    """Integers in [-16, 16] (exact e4m3 codes) with one ±448 in every row and every column, times 2^e: every row and column
    amax is 448·2^e, so every scale is the power of two 2^e, the quantisation is lossless and an fp32 sum of up to 64 products
    is exact."""
    t = torch.randint(-16, 17, (R, C), generator=gen).double()
    sign = torch.where(torch.rand(max(R, C), generator=gen) < 0.5, -1.0, 1.0)
    for i in range(max(R, C)):
        t[i % R, i % C] = 448.0 * sign[i]
    return (t * 2.0 ** e).to(BF16)


def test_products_exact_on_probes():
    gen = torch.Generator().manual_seed(0)
    M, N, K = 48, 32, 64
    x, w, g = _probe(M, K, -3, gen), _probe(N, K, -9, gen), _probe(M, N, 2, gen)
    x64, w64, g64 = x.double(), w.double(), g.double()
    assert torch.equal(_rows64(x), x64) and torch.equal(_cols_t64(w), w64.t())        # lossless by construction
    assert torch.equal(gemm_fp8.fp8_forward(x, w), (x64 @ w64.t()).to(BF16))
    assert torch.equal(gemm_fp8.fp8_dgrad(g, w), (g64 @ w64).to(BF16))
    dw = gemm_fp8.fp8_wgrad(g, x)
    assert dw.dtype == torch.float32 and torch.equal(dw, (g64.t() @ x64).float())
    old = torch.randint(-64, 65, (N, K), generator=gen).float()
    acc = gemm_fp8.fp8_wgrad(g, x, out=old.clone(), accumulate=True)
    assert torch.equal(acc, old + (g64.t() @ x64).float())


def _bound(a64, b64, K):
    """Per-element bound of an fp32 dot product of length K over dequantised operands: the fp32 rounding of each operand
    (2^-24 relative each) and of the K-term sum (K·2^-24 relative to Σ|a||b|)."""
    return (K + 2) * 2.0 ** -24 * (a64.abs() @ b64.abs().t())


@pytest.mark.parametrize("M,N,K", [(40, 24, 72), (17, 9, 33)])
def test_products_follow_the_table(M, N, K):
    """Random operands with rows and columns of very different magnitudes: each product equals the float64 product of the
    operands the table names, within the fp32 accumulation bound (bf16 outputs: plus one bf16 rounding).  Quantising by rows
    where the table says columns (or the reverse) misses by orders of magnitude more."""
    gen = torch.Generator().manual_seed(M)

    def rnd(r, c):
        return (torch.randn(r, c, generator=gen) * torch.pow(2.0, torch.randint(-6, 7, (r, 1), generator=gen).float())
                * torch.pow(2.0, torch.randint(-6, 7, (1, c), generator=gen).float())).to(BF16)

    x, w, g = rnd(M, K), rnd(N, K), rnd(M, N)
    cases = [
        (gemm_fp8.fp8_forward(x, w), _rows64(x), _rows64(w), K, True),
        (gemm_fp8.fp8_dgrad(g, w), _rows64(g), _cols_t64(w), N, True),
        (gemm_fp8.fp8_wgrad(g, x), _cols_t64(g), _cols_t64(x), M, False),
    ]
    for y, a64, b64, k, bf16_out in cases:
        ref = a64 @ b64.t()
        bound = _bound(a64, b64, k)
        if bf16_out:
            bound = bound + ref.abs() * 2.0 ** -8
        assert ((y.double() - ref).abs() <= bound).all()


def _fallback_state():
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_fallback_parallel_state()
    return ps


def _rule_grads(x, w, b, gy, col_scale=None):
    """float64 of the table's three products on the emulation path's operands, plus the bias gradient."""
    x2, gy2 = x.reshape(-1, x.shape[-1]), gy.reshape(-1, gy.shape[-1])
    gd = gy2
    if col_scale is not None:
        gd = gy2.clone()
        gd[:, col_scale[0]:] *= col_scale[1]
    y = (_rows64(x2) @ _rows64(w).t()).to(BF16) + b
    dx = (_rows64(gd) @ _cols_t64(w).t()).to(BF16)
    dw = (_cols_t64(gy2) @ _cols_t64(x2).t()).float()
    return y, dx, dw, gy2.sum(0)


@pytest.mark.parametrize("col_scale", [None, (24, 0.5)])
def test_tp_linear_fp8_gradients(col_scale):
    """Forward, input, weight and bias gradients of one fp8 tp_linear; with ``dgrad_col_scale`` the input gradient reads the
    scaled output gradient and the weight gradient the unscaled one.  Probe operands: every product is exact, so the
    comparison is bit for bit."""
    from neuronx_distributed_b200.parallel_layers.layers import tp_linear

    _fallback_state()
    gen = torch.Generator().manual_seed(3)
    S, B, K, N = 16, 2, 64, 32
    x = _probe(S * B, K, -2, gen).view(S, B, K).requires_grad_(True)
    w = _probe(N, K, -7, gen).requires_grad_(True)
    b = (torch.randint(-8, 9, (N,), generator=gen) * 0.25).to(BF16).requires_grad_(True)
    gy = _probe(S * B, N, 1, gen).view(S, B, N)
    y = tp_linear(x, w, b, "none", "none", dgrad_col_scale=col_scale, fp8=True)
    y.backward(gy)
    y_r, dx_r, dw_r, db_r = _rule_grads(x.detach(), w.detach(), b.detach(), gy, col_scale)
    assert torch.equal(y.detach().view(-1, N), y_r)
    assert torch.equal(x.grad.view(-1, K), dx_r)
    assert w.grad.dtype == BF16 and torch.equal(w.grad, dw_r.to(BF16))
    assert torch.equal(b.grad, db_r.to(BF16))


def test_tp_linear_fp8_matches_rule_on_random_data():
    """Random operands: the node's outputs are the emulation products of exactly the table's operands (same code path,
    bit for bit), so a wrong operand (x instead of the gathered x, g instead of gᵀ) cannot hide behind a tolerance."""
    from neuronx_distributed_b200.parallel_layers.layers import tp_linear

    _fallback_state()
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(24, 48, generator=gen).to(BF16).requires_grad_(True)
    w = torch.randn(40, 48, generator=gen).to(BF16).requires_grad_(True)
    gy = torch.randn(24, 40, generator=gen).to(BF16)
    y = tp_linear(x, w, None, "none", "none", fp8=True)
    y.backward(gy)
    assert torch.equal(y, gemm_fp8.fp8_forward(x.detach(), w.detach()))
    assert torch.equal(x.grad, gemm_fp8.fp8_dgrad(gy, w.detach()))
    assert torch.equal(w.grad, gemm_fp8.fp8_wgrad(gy, x.detach()).to(BF16))


def test_tp_linear_fp8_main_grad_protocol():
    """ZeRO-1 fp32 gradient accumulation: the first backward after zero_grad overwrites ``main_grad`` (NaN before), later
    ones add in fp32; no ``.grad`` is produced and ``_nxd_grad_ready`` fires once per backward."""
    from neuronx_distributed_b200.parallel_layers.layers import tp_linear

    _fallback_state()
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(32, 64, generator=gen).to(BF16)
    w = torch.randn(16, 64, generator=gen).to(BF16).requires_grad_(True)
    w.main_grad = torch.full((16, 64), float("nan"))
    w.main_grad_fresh = True
    ready = []
    w._nxd_grad_ready = ready.append
    expect = None
    for step in range(3):
        gy = torch.randn(32, 16, generator=gen).to(BF16)
        tp_linear(x, w, None, "none", "none", fp8=True).backward(gy)
        fresh = gemm_fp8.fp8_wgrad(gy, x)
        expect = fresh if expect is None else expect + fresh
        assert torch.equal(w.main_grad, expect)
        assert len(ready) == step + 1 and ready[-1] is w
        assert w.main_grad_fresh is False and w.grad is None


def _tp2_sp(rank, world):
    """Column (gather → none) and Row (none → scatter) fp8 linears at TP = 2 with SP: each rank's outputs and gradients equal
    the emulation products of that rank's own operands (the gathered x / g, its weight shard)."""
    import torch.distributed as dist

    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.layers import tp_linear

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    gen = torch.Generator().manual_seed(7)
    S, H, I = 32, 48, 64
    x_full = torch.randn(S, H, generator=gen).to(BF16)
    w1 = torch.randn(I, H, generator=gen).to(BF16).chunk(world, 0)[rank].contiguous().requires_grad_(True)
    w2 = torch.randn(H, I, generator=gen).to(BF16).chunk(world, 1)[rank].contiguous().requires_grad_(True)
    g_full = torch.randn(S, H, generator=gen).to(BF16)
    x = x_full.chunk(world, 0)[rank].clone().requires_grad_(True)
    h = tp_linear(x, w1, None, "gather", "none", reduce_dtype=torch.float32, fp8=True)
    hd = h.detach().requires_grad_(True)
    y = tp_linear(hd, w2, None, "none", "scatter", reduce_dtype=torch.float32, fp8=True)
    g = g_full.chunk(world, 0)[rank]
    y.backward(g)
    gh = hd.grad
    h.backward(gh)

    # column: forward on the gathered x, input gradient reduce-scattered from this rank's partial
    assert torch.equal(h.detach(), gemm_fp8.fp8_forward(x_full, w1.detach()))
    part = gemm_fp8.fp8_dgrad(gh, w1.detach()).float()
    dist.all_reduce(part)
    assert torch.equal(x.grad, part.to(BF16).chunk(world, 0)[rank])
    assert torch.equal(w1.grad, gemm_fp8.fp8_wgrad(gh, x_full).to(BF16))
    # row: forward partial reduce-scattered in fp32, gradients from the all-gathered g
    part = gemm_fp8.fp8_forward(hd.detach(), w2.detach()).float()
    dist.all_reduce(part)
    assert torch.equal(y.detach(), part.to(BF16).chunk(world, 0)[rank])
    assert torch.equal(hd.grad, gemm_fp8.fp8_dgrad(g_full, w2.detach()))
    assert torch.equal(w2.grad, gemm_fp8.fp8_wgrad(g_full, hd.detach()).to(BF16))


def test_tp2_sequence_parallel_fp8():
    run_distributed(_tp2_sp, 2)


def test_llama_fp8_training_marks_decoder_linears_only():
    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    from neuronx_distributed_b200.modules.qkv_linear import GQAQKVColumnParallelLinear
    from neuronx_distributed_b200.parallel_layers.layers import BaseParallelLinear

    _fallback_state()
    kw = dict(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
              num_key_value_heads=2)
    torch.manual_seed(0)
    ref = LlamaForCausalLM(LlamaConfig(**kw))
    torch.manual_seed(0)
    m = LlamaForCausalLM(LlamaConfig(fp8_training=True, **kw))
    on = {n for n, mod in m.named_modules()
          if isinstance(mod, (BaseParallelLinear, GQAQKVColumnParallelLinear)) and mod.fp8_training}
    expect = {f"model.layers.{i}.{p}" for i in range(2)
              for p in ("self_attn.qkv_proj", "self_attn.o_proj", "mlp.gate_up_proj", "mlp.down_proj")}
    assert on == expect
    assert not any(getattr(mod, "fp8_training", False) for _, mod in ref.named_modules())
    sd, sd_ref = m.state_dict(), ref.state_dict()
    assert list(sd) == list(sd_ref)
    for k in sd:
        assert sd[k].shape == sd_ref[k].shape and sd[k].dtype == sd_ref[k].dtype, k
