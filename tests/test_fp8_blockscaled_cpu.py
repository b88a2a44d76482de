"""Block-scaled FP8 (block-wise e4m3 and MXFP8) on CPU: the group quantiser against the existing torch quantisers, the
fp32 oracle of ``blockscaled_linear`` against float64, and W8A8 block-wise quantised layers at TP=1 and TP=2."""
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
