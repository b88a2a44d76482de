"""Grouped (MoE) mode of the block-scaled FP8 GEMM on the H100 (``csrc/gemm_fp8_block_sm90.cu``, GROUPED = true) against
float64, element by element, and W8A8 expert layers on the dropless prefill path.

Block i of the rows is multiplied by expert ``block_to_expert[i]``.  The probe, planted-scale and dense small-integer operands
of ``test_fp8_blockscaled_cpu.py`` are built per expert (a different probe shift and a different power-of-two scale factor
per expert, so a wrong expert or a wrong scale row changes the result), and every output must equal float64 rounded once to
bf16, bit for bit.  Full-range random codes must stay within the fp8-accumulation bound of ``test_fp8_blockscaled_gpu.py``.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_fp8_blockscaled_cpu import (F64, dense_operands, exact_bf16, probe_ks, probe_operands,  # noqa: E402
                                      reference64, to_e4m3)
from test_fp8_blockscaled_gpu import _random_codes, _raises_before_launch, _sa_view  # noqa: E402
from test_fp8_blockscaled_gpu import _unaligned_copy, _wide, gamma, launched  # noqa: E402

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
E4M3 = torch.float8_e4m3fn
NAN_CODE = 0x7F


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _check(y, ref, tol, what):
    """Per element |y − ref| <= tol, and y finite (a NaN would compare false against any bound)."""
    y = y.reshape(ref.shape).to(F64)
    assert torch.isfinite(y).all(), f"{what}: non-finite outputs"
    err = (y - ref).abs()
    assert not (err > tol).any(), f"{what}: {int((err > tol).sum())} outside the bound"
    live = tol > 0
    print(f"RATIO {what}: {(err[live] / tol[live]).max().item():.4f}")


def _kernel(_ext, a, bs, sa, sbs, b2e, B, G):
    """a [M, K], bs [E, N, K] (float64 codes), sa [K/G, M], sbs [E, K/G, N] → the kernel's bf16 [M, N]."""
    w = to_e4m3(torch.nan_to_num(bs, nan=0.0).reshape(-1, bs.shape[-1])).view(bs.shape)
    w.view(torch.uint8)[torch.isnan(bs)] = NAN_CODE
    b2e_t = torch.tensor(b2e, dtype=torch.int32, device="cuda")
    return _ext.ext().grouped_gemm_fp8_block(to_e4m3(a), w, _sa_view(sa.float()), sbs.float().contiguous(), b2e_t, B, G)


def _reference(a, bs, sa, sbs, b2e, B, G):
    out = torch.zeros(a.shape[0], bs.shape[1], dtype=F64, device=a.device)
    for i, e in enumerate(b2e):
        r = slice(i * B, (i + 1) * B)
        out[r] = reference64(a[r], bs[e], sa[:, r], sbs[e], G)
    return out


def _experts(maker, E, N, K, G, used):
    """Per-expert float64 codes [E, N, K] and scales [E, K/G, N] from ``maker(e)``; experts not in ``used`` hold the e4m3
    NaN code and NaN scales, so anything read from them that reached a stored output would show."""
    bs = torch.full((E, N, K), float("nan"), dtype=F64, device="cuda")
    sbs = torch.full((E, K // G, N), float("nan"), dtype=F64, device="cuda")
    for e in used:
        bs[e], sbs[e] = maker(e)
    return bs, sbs


# block layouts: trailing padding blocks (the last used expert repeated, rows of zero codes as the metadata builds them),
# an expert with no block between used ones, and the last expert used (its right-edge over-read is past the map)
LAYOUTS = {"gaps-and-padding": (5, [0, 0, 2, 2, 2, 4, 4, 4], 2), "one-expert": (3, [1, 1], 0),
           "last-expert-first": (4, [3, 0, 0, 2], 0)}
SHAPES = [(256, 128), (136, 256), (200, 896), (1288, 384)]       # (N, K): N % 128 != 0 in three of them


def _zero_padding(a, b2e, B, pad_blocks):
    if pad_blocks:
        a[(len(b2e) - pad_blocks) * B:] = 0
    return a


@pytest.mark.parametrize("G", [32, 64, 128])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_grouped_exact_probes_planted_and_dense(_ext, layout, G):
    E, b2e, pad = LAYOUTS[layout]
    used = sorted(set(b2e))
    B = 128 if layout != "one-expert" else 256
    M = len(b2e) * B
    for N, K in SHAPES:
        P = len(probe_ks(K, G))
        # probes: expert e's column n reads probe k number (n + 7e) mod P, its scales carry an extra 2^(2e - 4)
        a, _, sa, _ = probe_operands(M, N, K, G, "cuda")
        a = _zero_padding(a, b2e, B, pad)

        def probe(e):
            _, b, _, sb = probe_operands(M, N, K, G, "cuda", shift=(7 * e) % P)
            return b, sb * 2.0 ** (2 * e - 4)
        bs, sbs = _experts(probe, E, N, K, G, used)
        ref = _reference(a, bs, sa, sbs, b2e, B, G)
        assert torch.equal(ref.to(BF16).to(F64), ref)
        exact_bf16(_kernel(_ext, a, bs, sa, sbs, b2e, B, G), ref, f"probe {layout} N={N} K={K} G={G}")
        # planted: 2^7 on one (group, column) scale of one used expert moves exactly that expert's blocks at that column
        e0, g0, n0 = used[-1], K // G - 1, N - 1
        sbs2 = sbs.clone()
        sbs2[e0, g0, n0] *= 2.0 ** 7
        got = _kernel(_ext, a, bs, sa, sbs2, b2e, B, G).to(F64)
        base = ref.to(BF16).to(F64)
        moved = torch.zeros_like(base, dtype=torch.bool)
        for i, e in enumerate(b2e):
            if e == e0:
                moved[i * B:(i + 1) * B, n0] = True
        moved &= base != 0
        gk = torch.tensor(probe_ks(K, G), device="cuda")[(n0 + 7 * e0) % P] // G
        if gk == g0:
            assert moved.any()
        else:
            moved[:] = False
        assert torch.equal(got[~moved], base[~moved]), f"planted e{e0} g{g0} n{n0} moved other outputs"
        assert torch.equal(got[moved], base[moved] * 2.0 ** 7)
        # dense small-integer codes with power-of-two scales: exact under any accumulation order
        a, _, sa, _ = dense_operands(M, N, K, G, "cuda", seed=N + K)
        a = _zero_padding(a, b2e, B, pad)

        def dense(e):
            _, b, _, sb = dense_operands(8, N, K, G, "cuda", seed=100 + e)
            return b, sb
        bs, sbs = _experts(dense, E, N, K, G, used)
        exact_bf16(_kernel(_ext, a, bs, sa, sbs, b2e, B, G), _reference(a, bs, sa, sbs, b2e, B, G),
                   f"dense {layout} N={N} K={K} G={G}")


def test_neighbour_rows_do_not_leak_at_ragged_n(_ext):
    """N % 128 != 0: the last column tile of expert e reads the first rows of expert e + 1 through the shared map.  Those
    rows hold ±448 and the NaN code and their scales are NaN or huge; the used experts' outputs stay exact."""
    G, B, K = 128, 128, 512
    for N in (136, 200, 1288):
        b2e = [0, 2, 2]
        a, _, sa, _ = dense_operands(len(b2e) * B, N, K, G, "cuda", seed=N)
        bs, sbs = _experts(lambda e: dense_operands(8, N, K, G, "cuda", seed=e)[1::2], 4, N, K, G, [0, 2])
        for e in (1, 3):
            bs[e] = torch.where(torch.arange(N, device="cuda")[:, None] % 2 == 0, 448.0, -448.0).expand(N, K)
            sbs[e] = 2.0 ** 100
        exact_bf16(_kernel(_ext, a, bs, sa, sbs, b2e, B, G), _reference(a, bs, sa, sbs, b2e, B, G), f"large N={N}")
        w = to_e4m3(torch.nan_to_num(bs).reshape(-1, K)).view(4, N, K)
        w.view(torch.uint8)[1] = NAN_CODE
        w.view(torch.uint8)[3] = NAN_CODE
        sw = sbs.float().clone()
        sw[1] = float("nan")
        sw[3] = float("nan")
        y = _ext.ext().grouped_gemm_fp8_block(to_e4m3(a), w, _sa_view(sa.float()), sw,
                                              torch.tensor(b2e, dtype=torch.int32, device="cuda"), B, G)
        ref = _reference(a, torch.nan_to_num(bs), sa, torch.nan_to_num(sbs), b2e, B, G)
        exact_bf16(y, ref, f"NaN neighbour N={N}")


@pytest.mark.parametrize("G", [32, 64, 128])
def test_grouped_random_codes_within_the_model_bound(_ext, G):
    g = torch.Generator(device="cuda").manual_seed(G)
    E, N, K, B = 6, 1288, 896, 128
    b2e = [0, 0, 0, 3, 5, 5, 1, 1]
    M = len(b2e) * B
    a8 = _random_codes(M, K, g)
    w8 = _random_codes(E * N, K, g).view(E, N, K)
    sa = _wide(K // G, M, g)
    sw = torch.stack([_wide(K // G, N, g) for _ in range(E)])
    y = _ext.ext().grouped_gemm_fp8_block(a8, w8, _sa_view(sa), sw, torch.tensor(b2e, dtype=torch.int32, device="cuda"),
                                          B, G)
    a, w = a8.to(F64), w8.to(F64)
    ref = _reference(a, w, sa.to(F64), sw.to(F64), b2e, B, G)
    T = _reference(a.abs(), w.abs(), sa.to(F64), sw.to(F64), b2e, B, G)
    gm = gamma(G, 2.0 ** -13)
    Eb = gm * T + gamma(K // G + 1, 2.0 ** -24) * (1 + gm) * T
    _check(y, ref, Eb + 2.0 ** -8 * (ref.abs() + Eb), f"grouped random G={G}")


@pytest.mark.parametrize("two_d,e8m0", [(False, False), (False, True), (True, False), (True, True)])
def test_op_scale_layouts_and_k_major_weights(_ext, two_d, e8m0):
    """``grouped_blockscaled_linear`` on ``[E, K, N]`` weights stored K-major: 1-D ``[E, K/G, N]`` and 128 × 128
    ``[E, K/G, N/128]`` scales, fp32 and E8M0, one launch, bit for bit against float64 on dense operands."""
    from neuronx_distributed_b200.ops import gemm_fp8

    E, N, K, G, B = 3, 384, 512, 128, 256
    b2e = [2, 0, 0]
    M = len(b2e) * B
    a, _, sa, _ = dense_operands(M, N, K, G, "cuda", seed=1)
    gen = torch.Generator(device="cuda").manual_seed(2)
    wk = torch.randint(-4, 5, (E, K, N), generator=gen, device="cuda").to(F64)
    cols = N // 128 if two_d else N
    exps = torch.randint(0, 4, (E, K // G, cols), generator=gen, device="cuda")
    ws = (exps + 127).to(torch.uint8) if e8m0 else torch.exp2(exps.to(torch.float32))
    ws64 = torch.exp2(exps.to(F64)).repeat_interleave(N // cols, 2)
    wq = to_e4m3(wk.reshape(-1, N)).view(E, K, N).transpose(1, 2).contiguous().transpose(1, 2)   # K-major storage
    xq, xs = to_e4m3(a), sa.t().float()
    b2e_t = torch.tensor(b2e, device="cuda")
    y = launched(_ext, lambda: gemm_fp8.grouped_blockscaled_linear(xq, xs, wq, ws, b2e_t, B, G), 1)
    exact_bf16(y, _reference(a, wk.transpose(1, 2), sa, ws64, b2e, B, G), f"op two_d={two_d} e8m0={e8m0}")
    # row-major storage is not what the kernel reads: the op takes the fp32 oracle, which agrees to fp32 rounding
    y2 = launched(_ext, lambda: gemm_fp8.grouped_blockscaled_linear(xq, xs, wq.contiguous(), ws, b2e_t, B, G), 0)
    torch.testing.assert_close(y2, y, rtol=2 ** -8, atol=0)


def test_refusals_before_launch(_ext):
    e = _ext.ext()
    E, N, K, G, B = 2, 256, 256, 128, 128
    a = torch.zeros(2 * B, K, device="cuda").to(E4M3)
    w = torch.zeros(E, N, K, device="cuda").to(E4M3)
    sa = _sa_view(torch.ones(K // G, 2 * B, device="cuda"))
    sw = torch.ones(E, K // G, N, device="cuda")
    b2e = torch.zeros(2, dtype=torch.int32, device="cuda")
    e.grouped_gemm_fp8_block(a, w, sa, sw, b2e, B, G)                              # the good call runs
    # every bad operand is built before capture starts
    a_bf, w_bf, a_un, w_un = a.to(BF16), w.to(BF16), _unaligned_copy(a), _unaligned_copy(w)
    a192, w192 = a[:, :192].contiguous(), w[:, :, :192].contiguous()
    sa192, sw192 = _sa_view(torch.ones(3, 2 * B, device="cuda")), torch.ones(E, 3, N, device="cuda")
    w252, sw252 = w[:, :252].contiguous(), sw[:, :, :252].contiguous()
    b2e4, sw128, sw1, b2e_long = torch.zeros(4, dtype=torch.int32, device="cuda"), sw[:, :, :128].contiguous(), \
        sw[:1].contiguous(), b2e.long()
    cases = [
        (lambda: e.grouped_gemm_fp8_block(a_bf, w, sa, sw, b2e, B, G), "e4m3"),
        (lambda: e.grouped_gemm_fp8_block(a, w_bf, sa, sw, b2e, B, G), "e4m3"),
        (lambda: e.grouped_gemm_fp8_block(a_un, w, sa, sw, b2e, B, G), "aligned"),
        (lambda: e.grouped_gemm_fp8_block(a, w_un, sa, sw, b2e, B, G), "aligned"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa, sw, b2e, B, 192), "group size"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa, sw, b2e, B, 16), "group size"),
        (lambda: e.grouped_gemm_fp8_block(a192, w192, sa192, sw192, b2e, B, 64), "K % 128"),
        (lambda: e.grouped_gemm_fp8_block(a, w252, sa, sw252, b2e, B, G), "N % 8"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa, sw, b2e4, 64, G), "block_rows"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa, sw128, b2e, B, G), "scale_b"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa, sw1, b2e, B, G), "scale_b"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa[:, :B], sw, b2e, B, G), "scale_a"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa, sw, b2e[:1], B, G), "block_expert"),
        (lambda: e.grouped_gemm_fp8_block(a, w, sa, sw, b2e_long, B, G), "block_expert"),
    ]
    for fn, match in cases:
        _raises_before_launch(fn, match)


# =====================================================================================================================
# ExpertMLPsV2 prefill with W8A8 experts at real per-rank shapes
# =====================================================================================================================
MODELS = {"mixtral-8x7b-tp8": (4096, 1792, 8, 2, [1], [128]), "qwen3-30b-a3b": (2048, 768, 128, 8, [1], [128]),
          "deepseek-v3-slice": (7168, 2048, 32, 8, [1, 2], [128, 128])}


@pytest.mark.parametrize("model", list(MODELS))
def test_expert_mlps_prefill_vs_float64(_ext, monkeypatch, model):
    """Each projection of the dropless prefill is checked per element against float64 on its own quantised operands with
    the bound above, the combine against float64 of the projections' outputs, and the whole layer makes one metadata launch
    plus a quantiser and a grouped GEMM per projection, with no de-quantised weight."""
    from neuronx_distributed_b200.modules.moe import ExpertMLPsV2, RoutedExpertsMLPOpsConfig
    from neuronx_distributed_b200.ops import gemm_fp8
    from neuronx_distributed_b200.quantization import ActivationQuantizationType, QuantizedDtype, convert
    from neuronx_distributed_b200.quantization import quantization_layers as ql
    from neuronx_distributed_b200.quantization.quantization_config import get_default_blockwise_custom_qconfig_dict

    H, I, E, k, axis, size = MODELS[model]
    T = 512
    torch.manual_seed(0)
    cfg = RoutedExpertsMLPOpsConfig(normalize_top_k_affinities=True, num_experts=E, top_k=k, hidden_size=H,
                                    intermediate_size=I)
    em = ExpertMLPsV2(cfg, dtype=BF16, device=torch.device("cuda")).eval()
    with torch.no_grad():
        for p in em.parameters():
            if p.dim() == 3:
                p.normal_(0, p.shape[1] ** -0.5)
    q = {**get_default_blockwise_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3, "block_axis": axis,
         "block_size": size, "activation_quantization_type": ActivationQuantizationType.DYNAMIC}
    qm = convert(em, q_config=q, inplace=True)
    ex = qm.get_mlp_op()
    assert ex.gate_up_proj.weight.transpose(1, 2).is_contiguous() and ex.down_proj.weight.transpose(1, 2).is_contiguous()
    x = torch.randn(T, H, device="cuda").to(BF16)
    aff = torch.softmax(torch.randn(T, E, device="cuda"), -1)
    idx = aff.topk(k, -1).indices
    calls = []
    real = gemm_fp8.grouped_blockscaled_linear

    def record(*args, **kw):
        y = real(*args, **kw)
        calls.append((args, y))
        return y

    def no_weight_copy(*a, **kw):
        raise AssertionError("W8A8 experts de-quantised a weight")

    monkeypatch.setattr(gemm_fp8, "grouped_blockscaled_linear", record)
    monkeypatch.setattr(ql, "blockwise_scale_dequantize", no_weight_copy)
    out = launched(_ext, lambda: qm(x, aff, idx, seq_len=T), 1 + 2 * 2)
    assert len(calls) == 2
    G = size[0]
    for (xq, xs, wq, ws, b2e, B, Gc), y in calls:
        assert Gc == G and B % 128 == 0
        b2e_l = b2e.tolist()
        Kp, Np = wq.shape[1], wq.shape[2]
        ws64 = gemm_fp8.expert_weight_scales_kn(ws, Np, Kp, G).to(F64)
        a, w = xq.to(F64), wq.to(F64).transpose(1, 2)
        sa = xs.reshape(a.shape[0], -1).t().to(F64)
        ref = _reference(a, w, sa, ws64, b2e_l, B, G)
        Tm = _reference(a.abs(), w.abs(), sa, ws64, b2e_l, B, G)
        gm = gamma(G, 2.0 ** -13)
        Eb = gm * Tm + gamma(Kp // G + 1, 2.0 ** -24) * (1 + gm) * Tm
        _check(y, ref, Eb + 2.0 ** -8 * (ref.abs() + Eb), f"{model} projection K={Kp} N={Np}")
    # combine: out[t] = Σ_j a[t, j] · y_down[slot of (t, j)], k bf16 roundings of the products and the partial sums
    (_, y_down), B = calls[1], calls[1][0][5]
    b2e = calls[1][0][4]
    from neuronx_distributed_b200.modules.moe.blockwise import build_block_metadata

    _, tp2id, _ = build_block_metadata(idx, E, B)
    a = aff.gather(1, idx)
    a = a / a.sum(-1, keepdim=True)
    ref = torch.zeros(T, H, dtype=F64, device="cuda")
    mag = torch.zeros_like(ref)
    valid = tp2id >= 0
    slot_e = b2e.long().repeat_interleave(B)[valid]
    tok = tp2id[valid]
    j = (idx[tok] == slot_e[:, None]).to(torch.int64).argmax(-1)
    w_slot = a.to(F64)[tok, j]
    contrib = y_down[valid].to(F64) * w_slot[:, None]
    ref.index_add_(0, tok, contrib)
    mag.index_add_(0, tok, contrib.abs())
    tol = (k + 2) * 2.0 ** -8 * mag
    _check(out, ref, tol, f"{model} combine")
