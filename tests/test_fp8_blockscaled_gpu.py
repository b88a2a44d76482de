"""Block-scaled FP8 GEMM and group quantiser on the H100 (``csrc/gemm_fp8_block_sm90.cu``) against float64, element by
element; the block-wise W8A8 layers and MXFP8 ``linear_mx`` under ``NXD_GEMM_MX=1`` with per-element bounds.

The rule, the probe builders and their exactness arguments are in ``test_fp8_blockscaled_cpu.py``:

* the quantiser is compared bit for bit with ``quantize_spec`` (float64 definition, NaN policy included), reading the
  group-major scale buffer ``[K/G, round_up(M, 4)]`` the kernel writes;
* the GEMM runs on operands whose exact result is known and representable (probes, planted scales, dense small-integer
  codes with power-of-two scales), so it must equal float64 rounded once to bf16, bit for bit;
* on full-range codes and wide fp32 scales the error is bounded by a stated model of the fp8 MMA accumulation.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_fp8_blockscaled_cpu import (F64, assert_quantised_as, check_dense, check_planted,  # noqa: E402
                                      check_probes, dense_operands, exact_bf16, quantiser_input, quantize_spec,
                                      reference64, to_e4m3)

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def launched(_ext, fn, n=1):
    """Run ``fn`` and assert that it made exactly ``n`` launches of the extension's kernels (0: the fallback)."""
    n0 = _ext.launches()
    out = fn()
    assert _ext.launches() - n0 == n, ("fell back to eager PyTorch" if n else "launched a kernel")
    return out


def _round4(m):
    return (m + 3) // 4 * 4


def _sa_view(sa, ld=None, fill=0.0):
    """fp32 [K/G, M] as the kernel reads it: a view of a [K/G, ld] buffer (ld a multiple of 4), ``fill`` in [M, ld)."""
    ng, M = sa.shape
    buf = torch.full((ng, ld or _round4(M)), fill, dtype=torch.float32, device=sa.device)
    buf[:, :M] = sa
    return buf[:, :M]


def kernel_gemm(_ext):
    def gemm(a8, b8, sa, sb, G):
        return _ext.ext().gemm_fp8_block(a8, b8, _sa_view(sa), sb.contiguous(), G)
    return gemm


# =====================================================================================================================
# 2. the group quantiser, bit for bit against the float64 rule
# =====================================================================================================================
Q_M = (1, 3, 5, 129, 4097)                  # M % 4 != 0: the scale buffer's row stride is padded
Q_K = (None, 320, 384, 1376, 1792, 2368, 14336)   # None: K = G.  K < 256 and K % 256 != 0 leave a warp segment partly live;
                                                   # 1376 / 1792 / 2368: Llama-2-7B / Mixtral / Qwen2.5-7B down at TP 8


@pytest.mark.parametrize("G", [32, 64, 128])
def test_quantiser_matches_the_rule(_ext, G):
    """Every M, K (K % G == 0), rule and clamp: codes and the raw group-major scale buffer equal ``quantize_spec`` bit for
    bit, NaN and ±inf groups included; the torch oracle on the same CUDA tensor equals it too."""
    from neuronx_distributed_b200.ops import gemm_fp8

    e = _ext.ext()
    for M in Q_M:
        for K in Q_K:
            K = K or G
            if K % G:
                continue
            x = quantiser_input(M, K, G, seed=M * 7 + K).cuda()
            for rule in ("absmax", "mx"):
                for clamp in (None, 24.0):
                    what = f"M={M} K={K} G={G} {rule} clamp={clamp}"
                    q, sbuf = e.quantize_fp8_groups(x, G, rule == "mx", float("inf") if clamp is None else clamp)
                    assert sbuf.shape == (K // G, _round4(M)) and sbuf.stride() == (_round4(M), 1), what
                    qw, sw = quantize_spec(x, G, rule, clamp)
                    assert_quantised_as(q, sbuf[:, :M].t(), qw, sw, what)
                    qo, so = gemm_fp8._quantize_groups_reference(x, G, rule, clamp)
                    assert_quantised_as(qo, so, qw, sw, "torch oracle on CUDA: " + what)
    x = quantiser_input(2 * 3, 1792, G, seed=1).cuda().view(2, 3, 1792)
    q, s = launched(_ext, lambda: gemm_fp8.quantize_groups(x, G, "mx"))
    assert_quantised_as(q.view(6, -1), s.reshape(6, -1), *quantize_spec(x.view(6, -1), G, "mx"), "quantize_groups")


# =====================================================================================================================
# 3. the GEMM, exact by construction
# =====================================================================================================================
SHAPES = {  # name: (N, K)
    "n136-k128": (136, 128),                     # one k-block; an 8-column tail
    "n1288-k768": (1288, 768),
    "n1288-k896": (1288, 896),                   # 7 k-blocks: num_kb % 6 != 0
    "n2056-k896": (2056, 896),                   # at M = 1100: 9 x 17 = 153 tiles > 132 SMs, so a CTA's second tile
                                                 # starts the 6-stage ring out of phase; tiles_m % 8 = 1
    "llama3-8b-qkv": (6144, 4096),
    "llama3-8b-gate_up": (28672, 4096),
    "llama3-8b-down": (4096, 14336),
    "llama3-70b-tp8-qkv": (1280, 8192),
    "llama3-70b-tp8-gate_up": (7168, 8192),
    "llama3-70b-tp8-down": (8192, 3584),
}
GEMM_M = (1, 2, 3, 5, 8, 129, 1000, 1100)    # decode; one row past a tile; tiles_m = 8; tiles_m = 9


@pytest.mark.parametrize("G", [32, 64, 128])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_gemm_exact_probes_planted_scales_and_dense(_ext, shape, G):
    N, K = SHAPES[shape]
    gemm = kernel_gemm(_ext)
    for M in GEMM_M:
        check_probes(gemm, M, N, K, G, "cuda")
        check_dense(gemm, M, N, K, G, "cuda", seed=M)
        if M in (1, 5, 129, 1100):
            check_planted(gemm, M, N, K, G, "cuda")


# =====================================================================================================================
# 4. the GEMM on full-range codes and wide fp32 scales
# =====================================================================================================================
# Error model.  An output is Σ_g part_g · fl(sa · sb), part_g = Σ_{k in g} a_k b_k computed by G/32 chained fp8 wgmma.
# NVIDIA does not document the fp8 MMA's accumulation; published reports (DeepSeek-V3 technical report, §3.3.2) put it
# near 14 bits.  The model here, not measured on this project, is: every addition inside one group's chain loses at most a
# relative 2^-13 (a 14-bit significand, truncated), so |part_g − exact| <= γ(G, 2^-13) · Σ_{k in g} |a_k b_k|.  The
# promotion rounds sa · sb and each fma once in fp32 (u = 2^-24), over K/G groups: γ(K/G + 1, 2^-24) · Σ_g |part_g| sa sb.
# The bf16 store adds at most 2^-8 · |acc|.  With T = Σ_k |a_k b_k| sa sb:
#   |y − ref| <= E + 2^-8 (|ref| + E),   E = γ(G, 2^-13) · T + γ(K/G + 1, 2^-24) · (1 + γ(G, 2^-13)) · T.
def gamma(n, u):
    return n * u / (1 - n * u)


def _random_codes(R, K, g):
    """Uniform over the 254 finite e4m3 codes (±448 included)."""
    c = torch.randint(0, 254, (R, K), generator=g, device="cuda").to(torch.uint8)
    c = torch.where(c >= 0x7F, c + 1, c)                           # skip 0x7F (NaN); 0xFF is never drawn
    return c.view(E4M3)


def _wide(ng, R, g):
    """fp32 scales 2^e · (1 + U[0, 1)), e uniform in [−12, 12]: not powers of two, and a wrong index is off by orders of
    magnitude."""
    e = torch.randint(-12, 13, (ng, R), generator=g, device="cuda").float()
    return torch.exp2(e) * (1 + torch.rand(ng, R, generator=g, device="cuda"))


@pytest.mark.parametrize("G", [32, 64, 128])
@pytest.mark.parametrize("shape,M", [("n1288-k896", 5), ("n2056-k896", 1100), ("llama3-70b-tp8-down", 1100),
                                     ("llama3-8b-down", 8), ("n136-k128", 129)])
def test_gemm_random_codes_within_the_model_bound(_ext, shape, M, G):
    N, K = SHAPES[shape]
    g = torch.Generator(device="cuda").manual_seed(M + K + G)
    a8, b8 = _random_codes(M, K, g), _random_codes(N, K, g)
    sa, sb = _wide(K // G, M, g), _wide(K // G, N, g)
    y = kernel_gemm(_ext)(a8, b8, sa, sb, G)
    a, b = a8.to(F64), b8.to(F64)
    ref = reference64(a, b, sa.to(F64), sb.to(F64), G)
    T = reference64(a.abs(), b.abs(), sa.to(F64), sb.to(F64), G)
    gm = gamma(G, 2.0 ** -13)
    E = gm * T + gamma(K // G + 1, 2.0 ** -24) * (1 + gm) * T
    tol = E + 2.0 ** -8 * (ref.abs() + E)
    _check(y, ref, tol, f"random {shape} M={M} G={G}")


# =====================================================================================================================
# 5. bounds, layouts and the dispatch
# =====================================================================================================================
def test_operand_tails_and_scale_padding_are_not_read(_ext):
    """A and B are views into larger buffers with the e4m3 NaN code in the rows past M and N; scale_a is a view with row
    stride >= M + 4 and NaN in [M, ld).  The outputs are bit-identical to the clean run (and to float64): the tensor maps
    end at M and N, not at the buffers."""
    e = _ext.ext()
    for M, N, K, G in ((5, 1288, 896, 32), (129, 136, 768, 64), (1100, 2056, 896, 128), (3, 6144, 4096, 32)):
        a, b, sa, sb = dense_operands(M, N, K, G, "cuda", seed=M)
        a8, b8 = to_e4m3(a), to_e4m3(b)
        clean = e.gemm_fp8_block(a8, b8, _sa_view(sa.float()), sb.float(), G)
        exact_bf16(clean, reference64(a, b, sa, sb, G), f"clean M={M} N={N} K={K} G={G}")
        abuf = torch.full((M + 200, K), 0x7F, dtype=torch.uint8, device="cuda")
        bbuf = torch.full((N + 200, K), 0x7F, dtype=torch.uint8, device="cuda")
        abuf[:M] = a8.view(torch.uint8)
        bbuf[:N] = b8.view(torch.uint8)
        av, bv = abuf.view(E4M3)[:M], bbuf.view(E4M3)[:N]
        sv = _sa_view(sa.float(), ld=_round4(M + 4) + 4, fill=float("nan"))
        assert av.is_contiguous() and bv.is_contiguous() and sv.stride(0) >= M + 4
        got = e.gemm_fp8_block(av, bv, sv, sb.float(), G)
        assert torch.equal(got, clean), f"NaN past M / N / in the scale padding leaked: M={M} N={N} K={K} G={G}"


def _dense_case(M, N, K, G, seed=0):
    a, b, sa, sb = dense_operands(M, N, K, G, "cuda", seed)
    return to_e4m3(a), to_e4m3(b), a, b, sa, sb


def test_blockscaled_linear_dispatch(_ext):
    """The kernel runs exactly when G, K % 128, N % 8, the e4m3 dtypes and the bf16 output allow it; every fallback is
    the oracle and equals float64 (these operands are exact in fp32, so the fp32 oracle is too)."""
    from neuronx_distributed_b200.ops import gemm_fp8

    def run(M, N, K, G, n, out_dtype=BF16, codes=E4M3):
        a8, b8, a, b, sa, sb = _dense_case(M, N, K, G)
        xq, wq = (a8, b8) if codes == E4M3 else (a.float().to(codes), b.float().to(codes))
        y = launched(_ext, lambda: gemm_fp8.blockscaled_linear(xq, sa.t().float(), wq, sb.t().float(), G,
                                                               out_dtype=out_dtype), n)
        ref = reference64(a, b, sa, sb, G)
        if out_dtype == torch.float32:
            assert torch.equal(y.to(F64), ref)
        else:
            exact_bf16(y, ref, f"M={M} N={N} K={K} G={G} {out_dtype} {codes}")

    run(6, 264, 256, 32, 1)
    run(6, 264, 1376, 32, 0)                    # Llama-2-7B down at TP 8: K % 128 = 96
    run(6, 260, 256, 32, 0)                     # N % 8 != 0
    run(6, 264, 256, 32, 0, out_dtype=torch.float32)
    run(6, 264, 384, 48, 0)                     # group size the kernel does not take
    run(6, 264, 256, 32, 0, codes=torch.float8_e5m2)


@pytest.mark.parametrize("G", [32, 128])
def test_quantiser_scales_need_no_repack(_ext, G):
    """``xs`` straight from ``quantize_groups`` ([B, S, K] leading dimensions, a transposed view of the group-major
    buffer) gives the same bytes as a contiguous ``[M, K/G]`` copy that takes the zero-padded re-pack (M = 6, M % 4 != 0)."""
    from neuronx_distributed_b200.ops import gemm_fp8

    K, N = 1024, 264
    x = (torch.randn(2, 3, K, device="cuda") * 4).to(BF16)
    wq = to_e4m3(torch.randint(-4, 5, (N, K), device="cuda").to(F64))
    ws = torch.exp2(torch.randint(-3, 4, (N, K // G), device="cuda").float())
    xq, xs = launched(_ext, lambda: gemm_fp8.quantize_groups(x, G))
    assert xs.reshape(6, -1).t().stride(1) == 1                  # the view path: no copy
    y = launched(_ext, lambda: gemm_fp8.blockscaled_linear(xq, xs, wq, ws, G))
    y2 = launched(_ext, lambda: gemm_fp8.blockscaled_linear(xq.reshape(6, K), xs.reshape(6, -1).contiguous(), wq, ws, G))
    assert y.shape == (2, 3, N) and torch.equal(y.reshape(6, N), y2)


@pytest.mark.parametrize("two_d", [False, True])
@pytest.mark.parametrize("e8m0", [False, True])
def test_weight_scale_layouts_vs_float64(_ext, two_d, e8m0):
    """Weight scales per (row, group) ``[N, K/G]`` or per 128-row block ``[N/128, K/G]``, fp32 or E8M0, through
    ``blockscaled_linear``: bit-identical to float64 (powers of two 2^0 … 2^3, exact as in ``dense_operands``)."""
    from neuronx_distributed_b200.ops import gemm_fp8

    M, N, K, G = 129, 1280, 896, 32
    a8, b8, a, b, sa, _ = _dense_case(M, N, K, G)
    g = torch.Generator(device="cuda").manual_seed(5)
    rows = N // 128 if two_d else N
    e = torch.randint(0, 4, (rows, K // G), generator=g, device="cuda")
    ws = (e + 127).to(torch.uint8) if e8m0 else torch.exp2(e.float())
    sb = torch.exp2(e.to(F64)).repeat_interleave(N // rows, 0).t()
    y = launched(_ext, lambda: gemm_fp8.blockscaled_linear(a8, sa.t().float(), b8, ws, G))
    exact_bf16(y, reference64(a, b, sa, sb, G), f"two_d={two_d} e8m0={e8m0}")


# =====================================================================================================================
# 6. layers, per element against float64 on their own quantised operands
# =====================================================================================================================
def _layer_bound(xq, xs, wq, ws_kn, G, extra=None):
    """float64 reference and the §4 bound for y = bf16(blockscaled(xq, xs, wq, ws)) (+ ``extra`` in bf16: one more
    rounding of at most 2^-8 of the sum)."""
    a, b = xq.reshape(-1, xq.shape[-1]).to(F64), wq.to(F64)
    sa, sb = xs.reshape(a.shape[0], -1).t().to(F64), ws_kn.to(F64)
    K = a.shape[1]
    ref = reference64(a, b, sa, sb, G)
    T = reference64(a.abs(), b.abs(), sa, sb, G)
    gm = gamma(G, 2.0 ** -13)
    E = gm * T + gamma(K // G + 1, 2.0 ** -24) * (1 + gm) * T
    tol = E + 2.0 ** -8 * (ref.abs() + E)
    if extra is not None:
        ref = ref + extra.to(F64)
        tol = tol + 2.0 ** -8 * (ref.abs() + tol)
    return ref, tol


def _check(y, ref, tol, what):
    err = (y.reshape(ref.shape).to(F64) - ref).abs()
    assert not (err > tol).any(), f"{what}: {int((err > tol).sum())} outside the bound, worst {(err / tol).max():.3f}"
    print(f"RATIO {what}: {(err / tol).max().item():.4f}")


@pytest.mark.parametrize("M", [1, 300])
@pytest.mark.parametrize("block_axis,block_size,scale_dtype", [([1], [128], torch.float32), ([0, 1], [128, 128], torch.float32),
                                                                ([1], [32], torch.uint8)])
def test_blockwise_dynamic_layers_vs_float64(_ext, monkeypatch, M, block_axis, block_size, scale_dtype):
    """QuantizedColumnParallel (with bias) and QuantizedRowParallel at decode (M = 1) and prefill on the kernels, per
    element against float64 on the layer's own quantised activations and weights; then CUDA-graph capture and replay."""
    from neuronx_distributed_b200.ops import gemm_fp8
    from neuronx_distributed_b200.quantization import quantization_layers as ql

    torch.manual_seed(0)
    K, N = 1024, 768
    G = block_size[-1]
    kw = dict(quantization_type="blockwise_symmetric", quantized_dtype=E4M3, block_axis=block_axis, block_size=block_size,
              scale_dtype=scale_dtype, activation_quantization_type="dynamic")
    col = ql.QuantizedColumnParallel(K, N, bias=True, gather_output=False, **kw).eval()
    col.quantize_from_float_weight(torch.randn(N, K) / K ** 0.5)
    col.bias.data.normal_()
    row = ql.QuantizedRowParallel(N, K, bias=False, input_is_parallel=True, **kw).eval()
    row.quantize_from_float_weight(torch.randn(K, N) / N ** 0.5)
    col, row = col.cuda(), row.cuda()

    def no_weight_copy(*a, **k):
        raise AssertionError("block-scaled path de-quantised the weight")

    monkeypatch.setattr(ql, "blockwise_scale_dequantize", no_weight_copy)
    x = (torch.randn(M, K, device="cuda") * 3).to(BF16)
    y = launched(_ext, lambda: col(x), 2)                        # quantiser + block-scaled GEMM
    xq, xs = gemm_fp8.quantize_groups(x, G)                      # the operands the layer used (the kernel is deterministic)
    ws = gemm_fp8.weight_scales_kn(col.scale, N, K, G)
    ref, tol = _layer_bound(xq, xs, col.weight, ws, G, extra=col.bias.to(BF16))
    _check(y, ref, tol, f"column layer M={M} G={G} {block_axis} {scale_dtype}")
    h = y.relu()
    z = launched(_ext, lambda: row._linear_2d(h), 2)
    hq, hs = gemm_fp8.quantize_groups(h, G)
    ref, tol = _layer_bound(hq, hs, row.weight, gemm_fp8.weight_scales_kn(row.scale, K, N, G), G)
    _check(z, ref, tol, f"row layer M={M} G={G} {block_axis} {scale_dtype}")
    # CUDA-graph capture and replay on new data
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        col(static_x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_y = col(static_x)
    x2 = torch.randn_like(x)
    static_x.copy_(x2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_y, col(x2))


def test_linear_mx_under_gemm_mx_flag(_ext, monkeypatch):
    from neuronx_distributed_b200.ops import gemm_fp8, gemm_mx
    from neuronx_distributed_b200.quantization.microscaling.mx_torch import quantize_mx

    torch.manual_seed(1)
    M, N, K = 200, 1024, 2048
    w_packed, w_e8m0 = quantize_mx(torch.randn(N, K, device="cuda"), "mxfp8")
    x = torch.randn(M, K, device="cuda").bfloat16()
    monkeypatch.setenv("NXD_GEMM_MX", "1")
    y = launched(_ext, lambda: gemm_mx.linear_mx(x, w_packed, w_e8m0), 2)
    xq, xs = gemm_fp8.quantize_groups(x, 32, "mx")
    assert_quantised_as(xq, xs, *quantize_spec(x, 32, "mx"), "MX activations")
    wq = w_packed.contiguous().view(torch.uint8).reshape(N, -1).view(E4M3)
    ref, tol = _layer_bound(xq, xs, wq, gemm_fp8.weight_scales_kn(w_e8m0, N, K, 32), 32)
    assert y.dtype == BF16
    _check(y, ref, tol, "linear_mx M=200")
    # the block-scaled GEMM takes e4m3 codes only: 4-bit weights still raise under the flag
    from neuronx_distributed_b200.ops.gemm_mx import quantize_mxfp4

    f4, f4s = quantize_mxfp4(torch.randn(N, K, device="cuda"))
    with pytest.raises(RuntimeError, match="MXFP8 e4m3"):
        gemm_mx.linear_mx(x, f4.view(torch.uint16), f4s)


def test_nonfinite_activations_reach_the_output(_ext):
    """A NaN or ±inf activation (no clamp) makes NaN every output that reads its group, through the kernels, for both
    rules; with a clamp, ±inf is clipped and only NaN propagates."""
    from neuronx_distributed_b200.ops import gemm_fp8

    M, N, K, G = 4, 264, 512, 32
    x = (torch.randn(M, K, device="cuda")).to(BF16)
    x[0, 5], x[1, 100], x[2, K - 1] = float("nan"), float("inf"), -float("inf")
    wq = to_e4m3(torch.randint(-4, 5, (N, K), device="cuda").to(F64))
    ws = torch.ones(N, K // G, device="cuda")
    for rule in ("absmax", "mx"):
        for clamp in (None, 8.0):
            xq, xs = launched(_ext, lambda: gemm_fp8.quantize_groups(x, G, rule, clamp))
            assert_quantised_as(xq, xs, *quantize_spec(x, G, rule, clamp), f"{rule} clamp={clamp}")
            y = launched(_ext, lambda: gemm_fp8.blockscaled_linear(xq, xs, wq, ws, G))
            bad_rows = [0] if clamp else [0, 1, 2]
            assert torch.isnan(y[bad_rows]).all(), (rule, clamp)
            good = [r for r in range(M) if r not in bad_rows]
            assert torch.isfinite(y[good]).all(), (rule, clamp)


# =====================================================================================================================
# 7. refusals, before anything is launched
# =====================================================================================================================
def _unaligned_copy(t):
    """A contiguous copy of ``t`` one element into a fresh buffer: its start is not 16-byte aligned."""
    buf = torch.zeros(t.numel() + 16, dtype=torch.uint8 if t.dtype == E4M3 else t.dtype, device=t.device)
    if t.dtype == E4M3:
        buf = buf.view(E4M3)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


def _raises_before_launch(fn, match):
    """``fn`` must raise RuntimeError.  It runs while a CUDA graph captures the stream, so if a guard were missing the
    kernel would only be recorded into a graph that is never replayed: the test fails on the assertion and nothing runs
    on the bad operand."""
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match=match):
        with torch.cuda.graph(graph):
            fn()


def test_refusals_before_launch(_ext):
    from neuronx_distributed_b200.ops import gemm_fp8

    e = _ext.ext()
    x = (torch.randn(6, 256, device="cuda")).to(BF16)
    xu = _unaligned_copy(x)
    _raises_before_launch(lambda: e.quantize_fp8_groups(xu, 32, False, float("inf")), "16-byte aligned")
    q, s = launched(_ext, lambda: gemm_fp8.quantize_groups(xu, 32), 0)        # the dispatch takes the oracle
    assert_quantised_as(q, s, *quantize_spec(x, 32, "absmax"), "unaligned x through the oracle")

    M, N, K, G = 6, 264, 256, 32
    a8, b8, a, b, sa, sb = _dense_case(M, N, K, G)
    sv, sbf = _sa_view(sa.float()), sb.float().contiguous()
    au, bu = _unaligned_copy(a8), _unaligned_copy(b8)
    _raises_before_launch(lambda: e.gemm_fp8_block(au, b8, sv, sbf, G), "16-byte aligned")
    _raises_before_launch(lambda: e.gemm_fp8_block(a8, bu, sv, sbf, G), "16-byte aligned")
    y = launched(_ext, lambda: gemm_fp8.blockscaled_linear(au, sa.t().float(), b8, sb.t().float(), G), 0)
    exact_bf16(y, reference64(a, b, sa, sb, G), "unaligned a through the oracle")
    # K % 128 (K = 96: K % G == 0 but not a whole k-block)
    a96, b96 = a8[:, :96].contiguous(), b8[:, :96].contiguous()
    _raises_before_launch(lambda: e.gemm_fp8_block(a96, b96, _sa_view(sa[:3].float()), sbf[:3].contiguous(), G), "K % 128")
    # N % 8
    _raises_before_launch(lambda: e.gemm_fp8_block(a8, b8[:260].contiguous(), sv, sbf[:, :260].contiguous(), G), "N % 8")
    # a scale row stride that is not a multiple of 4 (16-byte aligned start)
    buf = torch.zeros(K // G * 7 + 4, device="cuda")
    s7 = buf.as_strided((K // G, M), (7, 1))
    assert s7.data_ptr() % 16 == 0
    _raises_before_launch(lambda: e.gemm_fp8_block(a8, b8, s7, sbf, G), "multiple of 4")
    # G = 48
    a384, b384 = to_e4m3(torch.ones(M, 384, device="cuda", dtype=F64)), to_e4m3(torch.ones(N, 384, device="cuda", dtype=F64))
    _raises_before_launch(lambda: e.gemm_fp8_block(a384, b384, _sa_view(torch.ones(8, M, device="cuda")),
                                                   torch.ones(8, N, device="cuda"), 48), "32, 64 or 128")

