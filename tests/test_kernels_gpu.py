"""Numerics of every hand-written CUDA kernel vs a plain PyTorch fp32 reference (H100, sm_90a)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gc():
    import gpu_check

    assert gpu_check.ops.extension_available(), gpu_check.ops._ext.load_error()
    return gpu_check


def _assert_all(gc, start):
    bad = [r for r in gc.RESULTS[start:] if not r["ok"]]
    assert not bad, bad


def test_extension_is_loaded_and_native():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    e = ops._ext.ext()
    for name in ("gemm_bf16", "ag_gemm_bf16", "gemm_rs_bf16", "rmsnorm_fwd", "fused_adamw", "ce_stats", "symm_alloc"):
        assert hasattr(e, name)


def test_elementwise_kernels(gc):
    n = len(gc.RESULTS)
    gc.check_elementwise()
    _assert_all(gc, n)


def test_tcgen05_gemm_all_layouts(gc):
    n = len(gc.RESULTS)
    gc.check_gemm()
    _assert_all(gc, n)


def test_decode_attention_and_gemv(gc):
    n = len(gc.RESULTS)
    gc.check_decode()
    _assert_all(gc, n)


def test_fp8_gemm(gc):
    n = len(gc.RESULTS)
    gc.check_fp8()
    _assert_all(gc, n)


def test_grouped_moe_gemm_fwd_dgrad_wgrad(gc):
    n = len(gc.RESULTS)
    gc.check_grouped()
    _assert_all(gc, n)


def test_gemm_python_frontend():
    from neuronx_distributed_b200.ops import gemm

    a = torch.randn(512, 256, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(384, 256, device="cuda", dtype=torch.bfloat16)
    y = gemm.linear_nt(a, w)
    ref = a.float() @ w.float().t()
    assert (y.float() - ref).abs().max() / ref.abs().max() < 1e-2


def test_tiny_llama_trains_on_cuda_kernels():
    import __graft_entry__ as ge

    ge.smoke()


@pytest.mark.parametrize("layout", ["bshd", "sbhd", "fused"])
@pytest.mark.parametrize("causal", [True, False])
def test_flash_attention_fwd_bwd_vs_fp32_reference(layout, causal):
    """Flash attention (fwd + dK/dV and dQ bwd kernels) through the autograd front-end vs plain fp32 softmax(QKᵀ)V."""
    import math

    from neuronx_distributed_b200.ops import _ext, attention

    assert hasattr(_ext.ext(), "flash_attn_fwd") and hasattr(_ext.ext(), "flash_attn_bwd")
    torch.manual_seed(1)
    B, S, H, Hkv, D = 2, 384, 4, 2, 128
    dev = "cuda"
    if layout == "bshd":
        q, k, v = (torch.randn(B, S, h, D, device=dev).bfloat16() for h in (H, Hkv, Hkv))
    elif layout == "sbhd":
        q, k, v = (torch.randn(S, B, h, D, device=dev).bfloat16().transpose(0, 1) for h in (H, Hkv, Hkv))
    else:
        f = torch.randn(S, B, (H + 2 * Hkv) * D, device=dev).bfloat16()
        q = f[..., : H * D].view(S, B, H, D).transpose(0, 1)
        k = f[..., H * D:(H + Hkv) * D].view(S, B, Hkv, D).transpose(0, 1)
        v = f[..., (H + Hkv) * D:].view(S, B, Hkv, D).transpose(0, 1)
    q, k, v = (t.detach().requires_grad_(True) for t in (q, k, v))
    n0 = _ext.launches()
    o = attention.flash_attention(q, k, v, causal=causal)
    go = torch.randn(B, S, H, D, device=dev).bfloat16()
    o.backward(go)
    assert _ext.launches() > n0, "own attention kernels did not run"
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    kk, vv = kf.repeat_interleave(H // Hkv, 2), vf.repeat_interleave(H // Hkv, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kk) / math.sqrt(D)
    if causal:
        s = s.masked_fill(~torch.ones(S, S, device=dev, dtype=torch.bool).tril(), float("-inf"))
    ro = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), vv)
    ro.backward(go.float())

    def rel(a, b):
        return ((a.float() - b).abs().max() / b.abs().max()).item()

    assert rel(o, ro) < 2e-2
    assert rel(q.grad, qf.grad) < 3e-2 and rel(k.grad, kf.grad) < 3e-2 and rel(v.grad, vf.grad) < 3e-2


@pytest.mark.parametrize("causal,S_q,S_kv", [(True, 200, 200), (False, 200, 328), (False, 130, 70)])
def test_flash_attention_ragged_lengths_vs_fp32_reference(causal, S_q, S_kv):
    """Lengths that are not multiples of the 64-row tiles (zero-filled tails, masked keys, unwritten rows), and non-causal
    attention with S_q != S_kv."""
    import math

    from neuronx_distributed_b200.ops import _ext, attention

    torch.manual_seed(2)
    B, H, Hkv, D = 2, 4, 2, 128
    q = torch.randn(B, S_q, H, D, device="cuda").bfloat16().requires_grad_(True)
    k, v = (torch.randn(B, S_kv, Hkv, D, device="cuda").bfloat16().requires_grad_(True) for _ in range(2))
    n0 = _ext.launches()
    o = attention.flash_attention(q, k, v, causal=causal)
    go = torch.randn(B, S_q, H, D, device="cuda").bfloat16()
    o.backward(go)
    assert _ext.launches() > n0, "own attention kernels did not run"
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    kk, vv = kf.repeat_interleave(H // Hkv, 2), vf.repeat_interleave(H // Hkv, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kk) / math.sqrt(D)
    if causal:
        s = s.masked_fill(~torch.ones(S_q, S_kv, device="cuda", dtype=torch.bool).tril(), float("-inf"))
    ro = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), vv)
    ro.backward(go.float())

    def rel(a, b):
        return ((a.float() - b).abs().max() / b.abs().max()).item()

    assert rel(o, ro) < 2e-2
    assert rel(q.grad, qf.grad) < 3e-2 and rel(k.grad, kf.grad) < 3e-2 and rel(v.grad, vf.grad) < 3e-2


def test_flash_attention_lse_is_differentiable():
    """Ring attention merges blocks through their LSEs: gradients must flow through the LSE output of the own kernels."""
    import math

    from neuronx_distributed_b200.ops import attention

    torch.manual_seed(3)
    B, S, Sk, H, D = 2, 256, 256, 4, 128      # equal block lengths, as ring attention produces
    q = torch.randn(B, S, H, D, device="cuda").bfloat16().requires_grad_(True)
    k = torch.randn(B, Sk, H, D, device="cuda").bfloat16().requires_grad_(True)
    v = torch.randn(B, Sk, H, D, device="cuda").bfloat16().requires_grad_(True)
    res = attention.flash_attention_with_lse(q, k, v, False, 1.0 / math.sqrt(D))
    assert res is not None
    o, lse = res
    w_o = torch.randn_like(o); w_l = torch.randn_like(lse)
    ((o.float() * w_o.float()).sum() + (lse * w_l).sum()).backward()
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) / math.sqrt(D)
    ro = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), vf)
    rl = torch.logsumexp(s, -1)
    ((ro * w_o.float()).sum() + (rl * w_l).sum()).backward()
    rel = lambda a, b: ((a.float() - b).abs().max() / b.abs().max()).item()
    assert rel(o, ro) < 2e-2 and (lse - rl).abs().max() < 2e-2
    assert rel(q.grad, qf.grad) < 3e-2 and rel(k.grad, kf.grad) < 3e-2 and rel(v.grad, vf.grad) < 3e-2


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fused_add_rmsnorm_vs_fp32_reference(dtype):
    """``csrc/fused_norm.cu``: h = x + r, y = rmsnorm(h)·w and the fused backward, against plain fp32 PyTorch."""
    from neuronx_distributed_b200.ops import _ext, norm

    assert _ext.ext() is not None and hasattr(_ext.ext(), "add_rmsnorm_fwd"), _ext.load_error()
    torch.manual_seed(0)
    rows, H = 1000, 4096
    x = torch.randn(rows, H, device="cuda", dtype=dtype, requires_grad=True)
    r = torch.randn(rows, H, device="cuda", dtype=dtype, requires_grad=True)
    w = (1 + 0.1 * torch.randn(H, device="cuda")).to(dtype).requires_grad_(True)
    cy, ch = torch.randn(rows, H, device="cuda", dtype=dtype), torch.randn(rows, H, device="cuda", dtype=dtype)
    before = _ext.launches()
    y, h = norm.add_rms_norm(x, r, w, 1e-5)
    ((y * cy).sum() + (h * ch).sum()).backward()
    assert _ext.launches() - before == 3                       # forward + backward (row kernel + dW reduction)
    xf, rf, wf = (t.detach().float().requires_grad_(True) for t in (x, r, w))
    hf = (xf + rf).to(dtype).float() if dtype != torch.float32 else xf + rf     # the kernel normalises the STORED sum
    hr = xf + rf
    yr = hf * torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    tol = 2e-2 if dtype == torch.bfloat16 else 1e-4
    assert (h.float() - hr).abs().max() <= (1e-6 if dtype == torch.float32 else 6e-2)
    assert (y.float() - yr).abs().max() / yr.abs().max() < tol
    # gradients against autograd of the fp32 composition
    h2 = xf + rf
    y2 = h2 * torch.rsqrt(h2.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    ((y2 * cy.float()).sum() + (h2 * ch.float()).sum()).backward()
    for got, want in ((x.grad, xf.grad), (r.grad, rf.grad), (w.grad, wf.grad)):
        assert (got.float() - want).abs().max() / want.abs().max() < tol
    assert torch.equal(x.grad, r.grad)


@pytest.mark.gpu
def test_decode_rope_kv_fused_vs_separate_ops():
    """RoPE of q/k at per-sequence positions + KV-cache append in one launch vs the eager composition."""
    from neuronx_distributed_b200 import ops

    e = ops._ext.ext()
    dev = torch.device("cuda")
    B, H, Hkv, D, L = 3, 8, 4, 128, 64
    torch.manual_seed(0)
    qkv = torch.randn(1, B, (H + 2 * Hkv) * D, device=dev, dtype=torch.bfloat16)
    q, k, v = torch.split(qkv, [H * D, Hkv * D, Hkv * D], dim=-1)
    q = q.reshape(1, B, H, D).transpose(0, 1)
    k = k.reshape(1, B, Hkv, D).transpose(0, 1)
    v = v.reshape(1, B, Hkv, D).transpose(0, 1).contiguous()
    cos, sin = ops.rope.rope_tables(L, D, 10000.0, dev)
    pos = torch.tensor([5, 0, 63], device=dev)
    kc = torch.zeros(B, L, Hkv, D, device=dev, dtype=torch.bfloat16)
    vc = torch.zeros_like(kc)
    q_out = e.decode_rope_kv(q, k, v, pos, cos, sin, kc, vc)
    q_ref = ops.rope.rotate(q, cos[pos].unsqueeze(1), sin[pos].unsqueeze(1))
    k_ref = ops.rope.rotate(k, cos[pos].unsqueeze(1), sin[pos].unsqueeze(1))
    torch.testing.assert_close(q_out.float(), q_ref.float(), atol=2e-2, rtol=2e-2)
    b = torch.arange(B, device=dev)
    torch.testing.assert_close(kc[b, pos].float(), k_ref[:, 0].float(), atol=2e-2, rtol=2e-2)
    assert torch.equal(vc[b, pos], v[:, 0])
    assert int((kc != 0).any(dim=-1).any(dim=-1).sum()) == B          # exactly one cache row per sequence was written


@pytest.mark.gpu
def test_moe_block_metadata_kernel_matches_sort_based_build():
    import os

    from neuronx_distributed_b200.modules.moe import blockwise

    dev = torch.device("cuda")
    torch.manual_seed(3)
    for T, k, E, B in ((4096, 2, 8, 512), (1000, 2, 16, 128), (300, 4, 64, 128), (8192, 1, 4, 256)):
        idx = torch.stack([torch.randperm(E, device=dev)[:k] for _ in range(T)])
        got = blockwise.build_block_metadata(idx, E, B)                       # CUDA kernel
        want = blockwise.build_block_metadata(idx.cpu(), E, B)                # sort + cumsum path
        for a, b, name in zip(got, want, ("block_to_expert", "token_position_to_id", "tokens_per_expert")):
            assert torch.equal(a.cpu(), b), (name, T, k, E, B)
