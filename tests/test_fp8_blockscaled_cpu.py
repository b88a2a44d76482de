"""Block-scaled FP8 (block-wise e4m3 and MXFP8) on CPU: the group quantiser against the existing torch quantisers, the
fp32 oracle of ``blockscaled_linear`` against float64, and W8A8 block-wise quantised layers at TP=1 and TP=2.

It also holds what ``test_fp8_blockscaled_gpu.py`` checks the kernels of ``csrc/gemm_fp8_block_sm90.cu`` with:

* ``e4m3_rne`` / ``quantize_spec``: the group quantiser's rule, defined in float64 from the e4m3 code table, with its NaN
  policy.  The torch oracle ``_quantize_groups_reference`` is checked against it here, the CUDA quantiser on the GPU.
* ``quantiser_input``: rows whose groups span 2^±30, with edge groups (e4m3 ties, subnormal codes, saturation, zeros, bf16
  subnormals, the largest bf16, powers of two, NaN, ±inf) planted at the first, the last and every third group.
* The GEMM probes (``check_probes``, ``check_planted``, ``check_dense``): operands built so that the exact result is known and
  every output is representable, so a correct kernel is bit-identical to float64.
* ``sim_gemm``: a float64 model of the GEMM kernel's index arithmetic (tile order, stage ring, scale offsets, epilogue
  tail) with one optional fault, and ``sim_quantize`` with the pre-fix NaN-dropping quantiser.  The probes pass on the model
  and reject every fault.
"""
import math

import numpy as np
import pytest
import torch

from dist_utils import run_distributed

from neuronx_distributed_b200.ops import gemm_fp8


def _wide_scales(*shape, gen):
    """Powers of two spread over 2^-12 … 2^12 so that a wrong group / row / column index changes the result by orders of
    magnitude, times a random mantissa so the fp32 scales are not exact powers of two."""
    e = torch.randint(-12, 13, shape, generator=gen).float()
    return torch.pow(2.0, e) * (1 + torch.rand(shape, generator=gen))


def _codes(*shape, gen):
    return (torch.randn(*shape, generator=gen) * 100).clamp(-448, 448).to(torch.float8_e4m3fn)


def _dequant64(q, s, G):
    R, K = q.shape
    return (q.double().reshape(R, K // G, G) * s.double().unsqueeze(-1)).reshape(R, K)


def test_mx_rule_matches_quantize_mx():
    from neuronx_distributed_b200.quantization.microscaling.mx_torch import quantize_mx

    g = torch.Generator().manual_seed(0)
    x = (torch.randn(37, 512, generator=g) * torch.pow(2.0, torch.randint(-20, 20, (37, 16, 1), generator=g).float())
         .repeat_interleave(32, 1).reshape(37, 512)).bfloat16()
    q, s = gemm_fp8.quantize_groups(x, 32, "mx")
    packed, e8m0 = quantize_mx(x, "mxfp8")
    assert torch.equal(q.view(torch.uint8), packed.contiguous().view(torch.uint8).reshape(37, 512))
    assert torch.equal(s, torch.pow(2.0, e8m0.float() - 127.0))


@pytest.mark.parametrize("clamp_bound", [None, 0.75])
def test_absmax_rule_with_one_group_matches_per_row_dynamic(clamp_bound):
    from neuronx_distributed_b200.quantization.quantization_utils import quantize_activation_dynamic

    g = torch.Generator().manual_seed(1)
    x = (torch.randn(3, 11, 256, generator=g) * torch.rand(3, 11, 1, generator=g) * 4).bfloat16()
    q, s = gemm_fp8.quantize_groups(x, 256, "absmax", clamp_bound)
    qr, sr = quantize_activation_dynamic(x, torch.float8_e4m3fn, clamp_bound)
    assert q.shape == x.shape and s.shape == (3, 11, 1)
    assert torch.equal(q.view(torch.uint8), qr.view(torch.uint8)) and torch.equal(s, sr)


@pytest.mark.parametrize("G", [32, 64, 128])
def test_absmax_groups_are_independent(G):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(9, 384, generator=g).bfloat16()
    x[:, :G] *= 1000                                             # a loud first group must not change the others' scales
    q, s = gemm_fp8.quantize_groups(x, G, "absmax")
    amax = x.float().reshape(9, -1, G).abs().amax(-1)
    assert torch.equal(s, (amax / 448.0).clamp(min=1e-12))
    back = (q.float().reshape(9, -1, G) * s.unsqueeze(-1)).reshape(9, 384)
    assert ((back - x.float()).abs() <= x.float().abs() * 2 ** -3 + 1e-30).all()


@pytest.mark.parametrize("G", [32, 64, 128])
@pytest.mark.parametrize("two_d", [False, True])
@pytest.mark.parametrize("e8m0", [False, True])
def test_oracle_matches_float64_with_wide_scales(G, two_d, e8m0):
    g = torch.Generator().manual_seed(3)
    M, N, K = 19, 256, 512
    xq, wq = _codes(M, K, gen=g), _codes(N, K, gen=g)
    xs = _wide_scales(M, K // G, gen=g)
    ws_rows = N // 128 if two_d else N
    if e8m0:
        ws = torch.randint(127 - 12, 127 + 13, (ws_rows, K // G), generator=g, dtype=torch.uint8)
        ws_f = torch.pow(2.0, ws.float() - 127.0)
    else:
        ws = ws_f = _wide_scales(ws_rows, K // G, gen=g)
    ws_full = ws_f.repeat_interleave(N // ws_rows, 0)
    want = _dequant64(xq, xs, G) @ _dequant64(wq, ws_full, G).t()
    got = gemm_fp8.blockscaled_linear(xq, xs, wq, ws, G, out_dtype=torch.float32)
    assert got.shape == (M, N)
    err = ((got.double() - want).norm() / want.norm()).item()
    assert err < 1e-6, err
    # the scales matter per group: a group-shifted weight scale is far off
    shifted = gemm_fp8.blockscaled_linear(xq, xs, wq, torch.roll(ws, 1, dims=1), G, out_dtype=torch.float32)
    assert ((shifted.double() - want).norm() / want.norm()).item() > 0.1


def test_weight_scale_layout_is_group_major():
    ws = torch.arange(6, dtype=torch.float32).reshape(2, 3)           # 2 row blocks of 4 rows, 3 groups
    kn = gemm_fp8.weight_scales_kn(ws, 8, 3 * 32, 32)
    assert kn.shape == (3, 8) and kn.is_contiguous()
    assert torch.equal(kn[:, 5], ws[1]) and torch.equal(kn[:, 0], ws[0])
    e = torch.tensor([[127, 128], [126, 130]], dtype=torch.uint8)
    assert torch.equal(gemm_fp8.weight_scales_kn(e, 2, 64, 32), torch.tensor([[1.0, 0.5], [2.0, 8.0]]))


def _w8a8_oracle(layer, x):
    """Hand-computed W8A8: torch group quantiser on the activations, float64 de-quantised operands."""
    G = layer.block_size[layer.block_axis.index(1)]
    x2 = x.reshape(-1, x.shape[-1])
    xb = x2.float().reshape(x2.shape[0], -1, G)
    xs = (xb.abs().amax(-1) / 448.0).clamp(min=1e-12)
    xq = (xb / xs.unsqueeze(-1)).clamp(-448, 448).to(torch.float8_e4m3fn).reshape(x2.shape)
    ws = layer.scale.float() if layer.scale.dtype != torch.uint8 else torch.pow(2.0, layer.scale.float() - 127.0)
    N = layer.weight.shape[0]
    ws = ws.repeat_interleave(N // ws.shape[0], 0)
    return _dequant64(xq, xs, G) @ _dequant64(layer.weight, ws, G).t()


def _layers(rank, world):
    from neuronx_distributed_b200.parallel_layers import ColumnParallelLinear, RowParallelLinear
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.quantization import ActivationQuantizationType, ScaleDtype, convert
    from neuronx_distributed_b200.quantization import quantization_layers as ql
    from neuronx_distributed_b200.quantization.quantization_config import get_default_blockwise_custom_qconfig_dict

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    H, F = 256, 512
    par = torch.nn.Sequential(ColumnParallelLinear(H, F, bias=True, gather_output=False),
                              RowParallelLinear(F, H, bias=True, input_is_parallel=True)).eval()
    x = torch.randn(2, 5, H)
    pref = par(x)
    dyn = {**get_default_blockwise_custom_qconfig_dict(), "activation_quantization_type": ActivationQuantizationType.DYNAMIC}
    for cfg in ({**dyn, "block_axis": [1], "block_size": [128]},
                {**dyn, "block_axis": [0, 1], "block_size": [128, 128]},
                {**dyn, "block_axis": [1], "block_size": [32], "scale_dtype": ScaleDtype.F8E8M0}):
        q = convert(par, cfg)
        assert all(m._blockscaled_group() == cfg["block_size"][-1] for m in q)
        # each layer against the hand-computed W8A8 oracle of its own shard
        h = torch.relu(q[0](x))
        for layer, inp in ((q[0], x), (q[1], h)):
            want = _w8a8_oracle(layer, inp)
            got = layer._linear_2d(inp).reshape(want.shape)
            err = ((got.double() - want).norm() / want.norm()).item()
            assert err < 1e-6, (cfg["block_size"], err)
        # close to the float model, and no bf16 copy of a weight is made
        orig = ql.blockwise_scale_dequantize
        ql.blockwise_scale_dequantize = None
        try:
            y = q(x)
        finally:
            ql.blockwise_scale_dequantize = orig
        err = float((y - pref).abs().max() / pref.abs().max())
        assert err < 0.08, (cfg["block_size"], err)
        sd = q.state_dict()
        q2 = convert(par, cfg)
        q2.load_state_dict(sd)
        torch.testing.assert_close(q2(x), y)
    # weight-only block-wise layers keep the de-quantise + dense path, bit for bit
    q = convert(par, get_default_blockwise_custom_qconfig_dict())
    assert q[0]._blockscaled_group() == 0
    w = ql.blockwise_scale_dequantize(q[0].weight, q[0].scale, torch.float32)
    assert torch.equal(q[0]._linear_2d(x), torch.nn.functional.linear(x, w))


def test_blockscaled_layers_tp1():
    run_distributed(_layers, 1, timeout=120)


def test_blockscaled_layers_tp2():
    run_distributed(_layers, 2, timeout=150)


# =====================================================================================================================
# 1. The quantiser's rule in float64
# =====================================================================================================================
F64 = torch.float64
E4M3_MAX = 448.0
NAN_CODE = 0x7F


def _e4m3_magnitudes() -> torch.Tensor:
    """Values of the finite non-negative e4m3fn codes 0x00 … 0x7E in code order (which is ascending), decoded from the bits:
    exponent bias 7, subnormals m/8 · 2^-6, 0x7F is NaN."""
    b = torch.arange(127)
    e, m = (b >> 3).to(F64), (b & 7).to(F64)
    return torch.where(e == 0, m / 8 * 2.0 ** -6, (1 + m / 8) * torch.exp2(e - 7))


E4M3_POS = _e4m3_magnitudes()


def e4m3_rne(t: torch.Tensor) -> torch.Tensor:
    """uint8 codes of the e4m3fn values nearest to float64 ``t``: ties go to the even code, |t| > 448 saturates to ±448
    (SATFINITE), the sign bit follows ``t`` (−0 and negative values that round to zero give 0x80), NaN gives 0x7F."""
    pos = E4M3_POS.to(t.device)
    nan = torch.isnan(t)
    a = torch.where(nan, 0.0, t.abs()).clamp(max=E4M3_MAX)
    hi = torch.searchsorted(pos, a.contiguous()).clamp(max=126)      # first magnitude >= a
    lo = (hi - 1).clamp(min=0)
    dlo, dhi = a - pos[lo], pos[hi] - a
    code = torch.where((dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0)), hi, lo)
    code = code | (torch.signbit(t).long() << 7)
    return torch.where(nan, NAN_CODE, code).to(torch.uint8)


def f32(t: torch.Tensor) -> torch.Tensor:
    """float64 → nearest fp32 (ties to even), back in float64."""
    return t.to(torch.float32).to(F64)


def quantize_spec(x: torch.Tensor, G: int, rule: str, clamp=None, absmax_div: str = "reciprocal"):
    """The group quantiser's rule in float64: ``x`` bf16 ``[M, K]`` → (uint8 codes ``[M, K]``, float64 scales ``[M, K/G]``).

    * clamp: ``x`` is clipped to ±fp32(clamp) first;
    * absmax: ``max(fp32(fp32(amax) · fp32(1/448)), fp32(1e-12))``, the product form the kernel and torch on CUDA use.  torch on
      the CPU divides (``absmax_div="true"``: ``fp32(amax / 448)``), which differs in the last bit for about half of all amax;
    * mx: ``2^(⌊log2 amax⌋ − 8)`` with amax floored at 2^-100, the floor taken exactly (frexp).  The kernel and torch round
      log2 to fp32 first; the two agree unless amax lies within about 2^-20 relative below a power of two, which no bf16
      amax does (one bf16 step below 2^e is 2^e · (1 − 2^-8));
    * codes: ``e4m3_rne(clamp(fp32(x / scale), ±448))`` (the float64 quotient rounded to fp32 is the correctly rounded fp32
      division: 53 >= 2·24 + 2 bits make the double rounding innocuous);
    * NaN: a group holding a NaN, or ±inf with no clamp, has no finite amax.  It gets a NaN scale, so all its codes are NaN
      and every output that reads the group is NaN."""
    M, K = x.shape
    xf = x.to(F64)
    if clamp is not None:
        c = float(np.float32(clamp))
        xf = xf.clamp(-c, c)                                      # torch.clamp keeps NaN
    xb = xf.view(M, K // G, G)
    amax = xb.abs().amax(-1)                                      # NaN if the group holds one
    finite = torch.isfinite(amax)
    a = torch.where(finite, amax, 1.0)
    if rule == "mx":
        _, e = torch.frexp(a.clamp(min=2.0 ** -100))              # a = m · 2^e, m in [0.5, 1): ⌊log2 a⌋ = e − 1
        scale = torch.exp2((e - 1 - 8).to(F64))
    else:
        q = f32(a) * f32(torch.tensor(1 / 448, dtype=F64)) if absmax_div == "reciprocal" else a / 448
        scale = torch.maximum(f32(q), f32(torch.tensor(1e-12, dtype=F64)))
    scale = torch.where(finite, scale, float("nan"))
    codes = e4m3_rne(f32(xb / scale.unsqueeze(-1)).clamp(-E4M3_MAX, E4M3_MAX)).view(M, K)
    return codes, scale


def nan_canonical(codes: torch.Tensor) -> torch.Tensor:
    """uint8 e4m3 codes with both NaN codes (0x7F, 0xFF) mapped to 0x7F: the sign of a NaN carries nothing."""
    c = codes.view(torch.uint8)
    return torch.where((c & 0x7F) == 0x7F, NAN_CODE, c)


def assert_quantised_as(codes, scales, want_codes, want_scales, what):
    """Codes bit for bit (NaN sign aside), scales bit for bit with NaN where the spec has NaN."""
    got_c, want_c = nan_canonical(codes).cpu(), nan_canonical(want_codes).cpu()
    bad = got_c != want_c
    assert not bad.any(), (f"{what}: {int(bad.sum())} codes differ, first at {bad.nonzero()[0].tolist()}: "
                           f"{got_c[bad][:4].tolist()} vs {want_c[bad][:4].tolist()}")
    s, w = scales.to(F64).cpu(), want_scales.to(F64).cpu()
    assert torch.equal(torch.isnan(s), torch.isnan(w)), f"{what}: NaN scales differ"
    ok = torch.isnan(w) | (s == w)
    assert ok.all(), f"{what}: {int((~ok).sum())} scales differ: {s[~ok][:4].tolist()} vs {w[~ok][:4].tolist()}"


BF16_MAX = (2 - 2.0 ** -7) * 2.0 ** 127


def edge_groups(G: int, nonfinite: bool = True):
    """[(name, float64 [G] group, may be rescaled)].  The edge values sit at the group's first and last positions (then
    alternately inwards); the rest is filler of at most amax/8.  At amax 448 both rules give the scale 1 exactly
    (fp32(448 · fp32(1/448)) = 1, 2^(8 − 8) = 1), so the codes see the values themselves."""
    t = [
        ("ties", [448, 1.0625, -1.1875, 17, -12.5, 13.5, 272, -304], 1 / 8),     # e4m3 midpoints: even code wins
        ("subnormal codes", [448, 2.0 ** -9, -3 * 2.0 ** -10, 2.0 ** -10, 5 * 2.0 ** -11, 7 * 2.0 ** -10, -2.0 ** -11,
                             2.0 ** -6 - 2.0 ** -10], 2.0 ** -12),
        ("saturation", [464, 448, -464, 456, 472, -480, 496, 504], 1 / 8),        # mx: scale 1, |x| > 448 clips to 448
        ("at 448", [448, -448, 440, 416], 1 / 8),
        ("zeros", [0.0, -0.0], 0.0),
        ("bf16 subnormals", [2.0 ** -127, -2.0 ** -133, 3 * 2.0 ** -130, 2.0 ** -126 - 2.0 ** -133], 0.0),
        ("largest bf16", [BF16_MAX, -1e38, 2.0 ** 100, 1.0], 2.0 ** -20),        # mx scale 2^119
        ("power of two", [2.0 ** 20, -2.0 ** 19, 3.0, 2.0 ** 20 - 2.0 ** 13], 2.0 ** -4),
        ("one bf16 step below", [2.0 ** 20 - 2.0 ** 12, -2.0 ** 19, 2.0 ** 12], 2.0 ** -4),
    ]
    if nonfinite:
        t += [("nan", [float("nan"), 1.0, -2.0], 1 / 8), ("+inf", [float("inf"), 3.0, -1.0], 1 / 8),
              ("-inf", [-float("inf"), 0.5], 1 / 8), ("nan and inf", [float("inf"), float("nan"), 2.0], 1 / 8)]
    out = []
    for i, (name, vals, fill) in enumerate(t):
        g = torch.Generator().manual_seed(100 + i)
        finite = [abs(v) for v in vals if math.isfinite(v)]
        amax = max(finite) if finite else 1.0
        grp = (torch.rand(G, generator=g, dtype=F64) * 2 - 1) * (amax * fill)
        order = [j // 2 if j % 2 == 0 else G - 1 - j // 2 for j in range(G)]   # 0, G−1, 1, G−2, …
        for j, v in enumerate(vals[:G]):
            grp[order[j]] = v
        out.append((name, grp, name not in ("zeros", "bf16 subnormals", "largest bf16")))
    return out


def quantiser_input(M: int, K: int, G: int, seed: int, nonfinite: bool = True) -> torch.Tensor:
    """bf16 [M, K] on the CPU: N(0, 1) groups times 2^e with e uniform in [−30, 30] per group; in every row the first, the
    last (the tail of a row whose K % 256 != 0) and every third group hold an edge group (template (row + group) mod n, times
    a power of two in 2^±30 where the template allows)."""
    g = torch.Generator().manual_seed(seed)
    n_g = K // G
    x = torch.randn(M, n_g, G, generator=g, dtype=F64) * torch.exp2(torch.randint(-30, 31, (M, n_g, 1), generator=g).to(F64))
    edges = edge_groups(G, nonfinite)
    tmpl = torch.stack([grp for _, grp, _ in edges])
    scalable = torch.tensor([sc for _, _, sc in edges])
    cols = torch.tensor(sorted({0, n_g - 1} | set(range(0, n_g, 3))))
    idx = (torch.arange(M)[:, None] + cols[None, :]) % len(edges)
    f = torch.where(scalable[idx], torch.exp2(torch.randint(-30, 31, idx.shape, generator=g).to(F64)), 1.0)
    x[:, cols] = tmpl[idx] * f.unsqueeze(-1)
    return x.view(M, K).to(torch.bfloat16)


def test_e4m3_rne_is_the_torch_conversion_with_saturation():
    """Every fp32 value on a fine grid around each code and each midpoint: the float64 table agrees with torch's RNE
    conversion below 448 and saturates above; the code table decodes like torch's e4m3fn."""
    assert torch.equal(torch.arange(127, dtype=torch.uint8).view(torch.float8_e4m3fn).to(F64), E4M3_POS)
    mids = (E4M3_POS[1:] + E4M3_POS[:-1]) / 2
    pts = torch.cat([E4M3_POS, mids, 464.0 + torch.arange(-4, 5, dtype=F64), torch.tensor([1e30])])
    t32 = torch.cat([pts.float(), torch.nextafter(pts.float(), torch.tensor(0.0)), torch.nextafter(pts.float(),
                                                                                                  torch.tensor(1e38))])
    t32 = torch.cat([t32, -t32])
    mine = e4m3_rne(t32.to(F64))
    theirs = t32.clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
    assert torch.equal(mine, theirs)
    # pinned without torch: ties to even, subnormal ties, saturation, signed zero, NaN
    cases = {1.0625: 0x38, 1.1875: 0x3A, 17.0: 0x58, 12.5: 0x54, 2.0 ** -10: 0x00, 3 * 2.0 ** -10: 0x02, 464.0: 0x7E,
             480.0: 0x7E, 1e300: 0x7E, -0.0: 0x80, -2.0 ** -11: 0x80, float("nan"): 0x7F}
    got = e4m3_rne(torch.tensor(list(cases), dtype=F64)).tolist()
    assert got == list(cases.values()), got


@pytest.mark.parametrize("G", [32, 64, 128])
@pytest.mark.parametrize("rule", ["absmax", "mx"])
@pytest.mark.parametrize("clamp", [None, 24.0])
def test_torch_oracle_matches_the_float64_rule(G, rule, clamp):
    """``_quantize_groups_reference`` on the CPU equals ``quantize_spec`` on every edge group, NaN and ±inf included (torch
    on the CPU divides amax by 448, so the absmax rule is compared in that form here; the CUDA kernel is compared with the
    product form in the GPU file)."""
    x = quantiser_input(13, 6 * G + 2 * 128, G, seed=G)
    q, s = gemm_fp8._quantize_groups_reference(x, G, rule, clamp)
    qw, sw = quantize_spec(x, G, rule, clamp, absmax_div="true")
    assert_quantised_as(q, s, qw, sw, f"G={G} {rule} clamp={clamp}")


def test_the_edges_are_reached():
    """The planted groups produce what they are there for: even-code ties, subnormal codes, saturated codes, the MX scale
    2^119 of the largest bf16, the exponent step at a power of two, NaN scales without a clamp and finite ones with it."""
    G = 32
    edges = {name: grp for name, grp, _ in edge_groups(G)}
    x = torch.stack([edges[n] for n in edges]).to(torch.bfloat16)
    names = list(edges)
    row = {n: i for i, n in enumerate(names)}
    q, s = quantize_spec(x, G, "mx")
    assert s[row["largest bf16"]].item() == 2.0 ** 119
    assert s[row["power of two"]].item() == 2.0 ** 12 and s[row["one bf16 step below"]].item() == 2.0 ** 11
    assert s[row["ties"]].item() == 1.0 and q[row["ties"], G - 1].item() == 0x38                    # 1.0625 → 1.0
    assert q[row["subnormal codes"], G - 1].item() == 0x01                                            # 2^-9
    assert (q[row["saturation"]] & 0x7F == 0x7E).sum() >= 6
    for n in ("nan", "+inf", "-inf", "nan and inf"):
        assert math.isnan(s[row[n]].item()) and (q[row[n]] & 0x7F == 0x7F).all(), n
    qa, sa = quantize_spec(x, G, "absmax")
    assert sa[row["ties"]].item() == 1.0 and sa[row["zeros"]].item() == float(np.float32(1e-12))
    qc, sc = quantize_spec(x, G, "absmax", clamp=24.0)
    assert math.isnan(sc[row["nan"]].item()) and not math.isnan(sc[row["+inf"]].item())


# =====================================================================================================================
# 3. GEMM probes with exactly known results (used by the GPU file on the kernel and below on the model)
# =====================================================================================================================
BM = BN = BK = 128
K_STAGES = 6


def probe_ks(K: int, G: int):
    """k positions the probes read: every group's first and last k in k-blocks 0, 1, 5, 6, 7 (the 6-stage ring wraps from
    stage 5 to stage 0 between k-blocks 5 and 6) and the last two, and the first k of every k-block."""
    nkb = K // BK
    ks = {kb * BK for kb in range(nkb)}
    for kb in {0, 1, 5, 6, 7, nkb - 2, nkb - 1}:
        if 0 <= kb < nkb:
            for g0 in range(kb * BK, (kb + 1) * BK, G):
                ks |= {g0, g0 + G - 1}
    return sorted(ks)


def _scale_exponent(idx, g, mul_i, mul_g):
    """Exponents in [−20, 20] that differ between neighbouring rows (columns), groups, k-blocks and tiles: the map
    (i, g) → (mul_i · i + mul_g · g) mod 41 changes unless the step is a multiple of 41."""
    return ((idx * mul_i + g * mul_g) % 41 - 20).to(F64)


def probe_operands(M, N, K, G, device, shift=0):
    """A row r holds a code in {±1, …, ±4} at every probe k; B column n holds one code at k = ks[(n + shift) mod P].  Each
    output then reads exactly one product: D[r, n] = a · b · sa[r, g] · sb[n, g] for the group g of that k, |a · b| <= 16
    times a power of two in 2^±40, which bf16 holds exactly.  Scales are powers of two keyed on (row, group) and
    (column, group).  Returns float64 codes a [M, K], b [N, K] and scales sa [K/G, M], sb [K/G, N]."""
    ks = torch.tensor(probe_ks(K, G), device=device)
    P = ks.numel()
    r = torch.arange(M, device=device)
    n = torch.arange(N, device=device)
    j = torch.arange(P, device=device)
    a = torch.zeros(M, K, dtype=F64, device=device)
    va = ((r[:, None] * 3 + j[None, :] * 5) % 4 + 1).to(F64) * (1 - 2 * ((r[:, None] + j[None, :]) % 2)).to(F64)
    a[:, ks] = va
    b = torch.zeros(N, K, dtype=F64, device=device)
    kn = ks[(n + shift) % P]
    b[n, kn] = ((n * 7 + 1) % 4 + 1).to(F64) * (1 - 2 * (n // 3 % 2)).to(F64)
    ng = K // G
    gi = torch.arange(ng, device=device)
    sa = torch.exp2(_scale_exponent(r[None, :], gi[:, None], 5, 3))
    sb = torch.exp2(_scale_exponent(n[None, :], gi[:, None], 7, 13))
    return a, b, sa, sb


def reference64(a, b, sa, sb, G):
    """Σ_g (a_g · b_gᵀ) · sa[g] ⊗ sb[g] in float64: the de-quantised operands' product."""
    ad = a * sa.t().repeat_interleave(G, 1)
    bd = b * sb.t().repeat_interleave(G, 1)
    return ad @ bd.t()


def to_e4m3(v: torch.Tensor) -> torch.Tensor:
    q = v.to(torch.float32).to(torch.float8_e4m3fn)
    assert torch.equal(q.to(F64), v), "operand not exact in e4m3"
    return q


def exact_bf16(got, ref, what):
    want = ref.to(torch.bfloat16)
    bad = ~((got == want) | (torch.isnan(got) & torch.isnan(want)))
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {got.numel()} outputs differ, first at "
                           f"{bad.nonzero()[0].tolist()}: {got[bad][:3].tolist()} vs {want[bad][:3].tolist()}")


def _run(gemm, a, b, sa, sb, G):
    return gemm(to_e4m3(a), to_e4m3(b), sa.float(), sb.float(), G)


def check_probes(gemm, M, N, K, G, device):
    """Every (row, probe k) pair, observed through every column that reads that k, bit for bit; enough launches (shifted
    column → k maps) that every probe k meets a column.  Returns the number of (row, k) pairs checked."""
    P = len(probe_ks(K, G))
    for shift in range(0, P, N):
        a, b, sa, sb = probe_operands(M, N, K, G, device, shift)
        ref = reference64(a, b, sa, sb, G)
        assert torch.equal(ref.to(torch.bfloat16).to(F64), ref)           # every output is a bf16 number
        exact_bf16(_run(gemm, a, b, sa, sb, G), ref, f"probe M={M} N={N} K={K} G={G} shift={shift}")
    return M * P


def planted_targets(M, N, K, G):
    """(operand, index, group) planted with 2^7: rows M−1 and min(128, M−1) (the second row tile), columns N−1 and
    min(128, N−1); the last group, group 0, and the first group of k-block 6 where K has one."""
    ng = K // G
    g6 = 6 * BK // G if K > 6 * BK else ng // 2
    return [("a", M - 1, ng - 1), ("a", min(128, M - 1), g6), ("b", N - 1, 0), ("b", min(128, N - 1), ng - 1),
            ("b", min(127, N - 1), g6)]


def check_planted(gemm, M, N, K, G, device):
    """A factor 2^7 on one (row, group) scale of A or (column, group) scale of B moves exactly the outputs that read that
    scale — the row (column) at the columns (rows) whose probe k lies in the group — by exactly 2^7, and nothing else."""
    a, b, sa, sb = probe_operands(M, N, K, G, device)
    base = _run(gemm, a, b, sa, sb, G).to(F64)
    ks = torch.tensor(probe_ks(K, G), device=device)
    gk = ks[torch.arange(N, device=device) % ks.numel()] // G        # the group each column reads
    for op, i, grp in planted_targets(M, N, K, G):
        sa2, sb2 = sa.clone(), sb.clone()
        (sa2 if op == "a" else sb2)[grp, i] *= 2.0 ** 7
        got = _run(gemm, a, b, sa2, sb2, G).to(F64)
        moved = torch.zeros(M, N, dtype=torch.bool, device=device)
        if op == "a":
            moved[i] = gk == grp
        else:
            moved[:, i] = bool(gk[i] == grp)
        moved &= base != 0
        assert torch.equal(got[~moved], base[~moved]), f"planted {op}[{i}, g{grp}] moved other outputs"
        assert torch.equal(got[moved], base[moved] * 2.0 ** 7), f"planted {op}[{i}, g{grp}] not by exactly 2^7"
        assert moved.any() or op == "b", (op, i, grp)


def dense_operands(M, N, K, G, device, seed):
    """Codes uniform in {−4, …, 4}, scale exponents in [−3, 0] (A) and [0, 3] (B).  Every term a · b · sa · sb is an
    integer multiple of 2^emin (emin = the smallest exponent sum) and a group partial is an integer below 16 · G <= 2^11,
    exact under any internal accumulation of the MMA.  Asserted here: Σ_k |a · b · sa · sb| < 2^(24 + emin) for every
    output, so every fp32 partial sum over groups is exact and the bf16 output is float64 rounded once.  (Worst case
    16 · K · 2^6 < 2^24 holds for K <= 14336 anyway.)"""
    g = torch.Generator(device=device).manual_seed(seed)
    ng = K // G
    a = torch.randint(-4, 5, (M, K), generator=g, device=device).to(F64)
    b = torch.randint(-4, 5, (N, K), generator=g, device=device).to(F64)
    sa = torch.exp2(torch.randint(-3, 1, (ng, M), generator=g, device=device).to(F64))
    sb = torch.exp2(torch.randint(0, 4, (ng, N), generator=g, device=device).to(F64))
    emin = math.log2(sa.min().item() * sb.min().item())
    bound = reference64(a.abs(), b.abs(), sa, sb, G)
    assert bound.max().item() < 2.0 ** (24 + emin), "dense operands are not exact in fp32"
    return a, b, sa, sb


def check_dense(gemm, M, N, K, G, device, seed=0):
    a, b, sa, sb = dense_operands(M, N, K, G, device, seed)
    exact_bf16(_run(gemm, a, b, sa, sb, G), reference64(a, b, sa, sb, G), f"dense M={M} N={N} K={K} G={G}")


# =====================================================================================================================
# 8. A float64 model of the kernel's index arithmetic, and the faults the probes must reject
# =====================================================================================================================
def tile_coords(tile: torch.Tensor, tiles_m: int, tiles_n: int, remainder_as_full: bool = False):
    """The kernel's tile order: groups of 8 M-blocks, column-major inside a group, the last group holding tiles_m mod 8.
    ``remainder_as_full``: a fault that maps the remainder group as if it had 8 M-blocks."""
    per_group = 8 * tiles_n
    grp = tile // per_group
    first_m = grp * 8
    gsz = torch.full_like(tile, 8) if remainder_as_full else (tiles_m - first_m).clamp(max=8)
    inn = tile - grp * per_group
    return first_m + inn % gsz, inn // gsz


FAULTS = ("scale_row_off_by_8", "group_without_kb", "last_kb_dropped", "tail_pair_skipped", "remainder_as_full",
          "stale_stage", "nan_dropped")


def _box(t, r0, c0, rows, cols):
    """A TMA box: ``t[r0:r0+rows, c0:c0+cols]`` with zeros outside the tensor."""
    out = torch.zeros(rows, cols, dtype=t.dtype)
    blk = t[r0:r0 + rows, c0:c0 + cols]
    out[:blk.shape[0], :blk.shape[1]] = blk
    return out


def sim_gemm(a8, b8, sa, sb, G, grid=7, fault=None):
    """float64 model of ``gemm_fp8_block_kernel``: e4m3 a [M, K], b [N, K], fp32 sa [K/G, ≥M], sb [K/G, N].  Each CTA walks
    its tiles in ``tile_coords`` order; the producer's loads form one sequence per CTA through a 6-stage ring; a stage holds
    the A / B boxes of one k-block and the scale boxes at group row ``kb · kGroups``; consumers promote each group's
    partial with the scale of their row (rows r_loc and r_loc + 8 of each 16-row slice) and store bf16 pairs of columns
    below N.  Outputs never stored stay NaN."""
    a, b = a8.to(F64), b8.to(F64)
    sa, sb = sa.to(F64), sb.to(F64)
    M, K = a.shape
    N = b.shape[0]
    kG, nkb = BK // G, K // BK
    tiles_m, tiles_n = -(-M // BM), -(-N // BN)
    total = tiles_m * tiles_n
    sa_m = sa[:, :M]                                                 # the A-scale map's inner dimension is M
    out = torch.full((M, N), float("nan"), dtype=F64)
    rows = torch.arange(BM)
    row_src = torch.where(rows % 16 >= 8, rows - 8, rows) if fault == "scale_row_off_by_8" else rows
    for cta in range(min(grid, total)):
        tiles = torch.arange(cta, total, min(grid, total))
        mb, nb = tile_coords(tiles, tiles_m, tiles_n, fault == "remainder_as_full")
        seq = [(t, int(m), int(n), kb) for t, m, n in zip(tiles.tolist(), mb, nb) for kb in range(nkb)]

        def stage(i):
            _, m, n, kb = seq[i]
            g0 = 0 if fault == "group_without_kb" else kb * kG
            return (_box(a, m * BM, kb * BK, BM, BK), _box(b, n * BN, kb * BK, BN, BK),
                    _box(sa_m, g0, m * BM, kG, BM), _box(sb, g0, n * BN, kG, BN))

        acc = None
        for i, (t, m, n, kb) in enumerate(seq):
            if kb == 0:
                acc = torch.zeros(BM, BN, dtype=F64)
            src = i
            if fault == "stale_stage" and i >= K_STAGES and seq[i - K_STAGES][0] != t:
                src = i - K_STAGES                                   # the ring's phase is a tile out of step: old data
            if not (fault == "last_kb_dropped" and kb == nkb - 1):
                A, B, SA, SB = stage(src)
                for g in range(kG):
                    part = A[:, g * G:(g + 1) * G] @ B[:, g * G:(g + 1) * G].t()
                    acc += part * SA[g][row_src][:, None] * SB[g][None, :]
            if kb == nkb - 1 and m < tiles_m:
                r0, c0 = m * BM, n * BN
                rr, cc = min(BM, M - r0), min(BN, N - c0)
                if rr <= 0 or cc <= 0:
                    continue
                if fault == "tail_pair_skipped" and N % BN and c0 + cc == N:
                    cc -= 2
                out[r0:r0 + rr, c0:c0 + cc] = acc[:rr, :cc]
    return out.to(torch.bfloat16)


def sim_quantize(x, G, rule, clamp=None, fault=None):
    """The group quantiser kernel with torch operations.  ``fault="nan_dropped"`` is the kernel before NaN handling: fmaxf /
    fminf (torch.fmax / fmin) drop a NaN operand in the clamp and the amax, and the MX exponent of an infinite amax goes
    through a saturating float → int conversion and a wrapping shift."""
    M, K = x.shape
    cb = torch.tensor(float("inf") if clamp is None else float(np.float32(clamp)), dtype=torch.float32)
    mx_, mn_ = (torch.fmax, torch.fmin) if fault == "nan_dropped" else (torch.maximum, torch.minimum)
    v = mn_(mx_(x.float(), -cb), cb).view(M, K // G, G)
    amax = v.abs().amax(-1) if fault != "nan_dropped" else torch.fmax(v.abs().nan_to_num(nan=0.0).amax(-1),
                                                                        torch.zeros(()))
    if rule == "mx":
        e = torch.floor(torch.log2(torch.fmax(amax, torch.tensor(2.0 ** -100))))
        if fault == "nan_dropped":
            ei = np.clip(np.nan_to_num(e.numpy().astype(np.float64), nan=0.0), -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64)
            bits = (((ei - 8 + 127) << 23) & 0xFFFFFFFF).astype(np.uint32)
            scale = torch.from_numpy(bits.view(np.float32))
        else:
            scale = torch.where(torch.isfinite(amax), torch.exp2(e - 8), float("nan"))
    else:
        scale = torch.fmax(amax * torch.tensor(1 / 448, dtype=torch.float32), torch.tensor(1e-12))
        if fault != "nan_dropped":
            scale = torch.where(torch.isfinite(amax), scale, float("nan"))
    c = mn_(mx_(v / scale.unsqueeze(-1), torch.tensor(-448.0)), torch.tensor(448.0))
    return c.view(M, K).to(torch.float8_e4m3fn).view(torch.uint8), scale


SIM_CASES = ((300, 264, 896, 32, 7), (1100, 136, 256, 64, 7), (129, 1288, 768, 128, 3))


def test_every_tile_is_visited_exactly_once():
    """All tiles_m, tiles_n <= 40 and grids 1, 7, 132: the CTAs' strided tile indices through ``tile_coords`` cover every
    (m_blk, n_blk) once.  The remainder-as-full fault does not whenever tiles_m % 8 != 0 and tiles_m, tiles_n > 1."""
    for tiles_m in range(1, 41):
        for tiles_n in range(1, 41):
            total = tiles_m * tiles_n
            for grid in (1, 7, 132):
                g = min(grid, total)
                tiles = torch.cat([torch.arange(c, total, g) for c in range(g)])
                mb, nb = tile_coords(tiles, tiles_m, tiles_n)
                assert ((mb >= 0) & (mb < tiles_m) & (nb >= 0) & (nb < tiles_n)).all()
                seen = torch.zeros(tiles_m * tiles_n, dtype=torch.long).index_add_(0, mb * tiles_n + nb,
                                                                                  torch.ones_like(mb))
                assert (seen == 1).all(), (tiles_m, tiles_n, grid)
            if tiles_m % 8:
                mb, nb = tile_coords(torch.arange(total), tiles_m, tiles_n, remainder_as_full=True)
                ok = (mb < tiles_m) & (nb < tiles_n)
                assert tiles_m == 1 or tiles_n == 1 or torch.unique(mb[ok] * tiles_n + nb[ok]).numel() < total


def _sim(fault, grid):
    def gemm(a8, b8, sa, sb, G):
        return sim_gemm(a8, b8, sa, sb, G, grid, fault)
    return gemm


@pytest.mark.parametrize("case", SIM_CASES, ids=lambda c: "x".join(map(str, c)))
def test_probes_pass_on_the_model(case):
    M, N, K, G, grid = case
    gemm = _sim(None, grid)
    check_probes(gemm, M, N, K, G, "cpu")
    check_planted(gemm, M, N, K, G, "cpu")
    check_dense(gemm, M, N, K, G, "cpu")


def gemm_caught_by(fault):
    """Names of (case, checker) pairs that reject the model with this fault."""
    names = []
    for M, N, K, G, grid in SIM_CASES:
        gemm = _sim(fault, grid)
        for name, fn in (("probes", check_probes), ("planted", check_planted), ("dense", check_dense)):
            try:
                fn(gemm, M, N, K, G, "cpu")
            except AssertionError:
                names.append(f"{M}x{N}x{K}/{name}")
    return names


@pytest.mark.parametrize("fault", FAULTS)
def test_checks_reject_each_fault(fault):
    """Every simulated fault is rejected: the GEMM faults by the probe checker (and mostly by the others too), the NaN-dropping
    quantiser by the comparison with ``quantize_spec`` on the edge rows."""
    if fault == "nan_dropped":
        failed = []
        for G in (32, 128):
            for rule in ("absmax", "mx"):
                for clamp in (None, 24.0):
                    x = quantiser_input(13, 4 * 128, G, seed=7)
                    q, s = sim_quantize(x, G, rule, clamp, fault)
                    qw, sw = quantize_spec(x, G, rule, clamp)
                    try:
                        assert_quantised_as(q, s, qw, sw, "")
                    except AssertionError:
                        failed.append((G, rule, clamp))
                    # the fault-free model is exact on the same rows: the difference is the NaN handling alone
                    assert_quantised_as(*sim_quantize(x, G, rule, clamp), qw, sw, "fault-free quantiser model")
        assert len(failed) == 8, failed
        return
    got = gemm_caught_by(fault)
    assert any(n.endswith("/probes") for n in got), (fault, got)
