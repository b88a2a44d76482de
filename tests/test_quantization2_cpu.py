"""Quantisation subsystem: configs, checkpoint-side utilities, MX packing helpers, quantised parallel layers built empty and
loaded from (plain and torch-packed) quantised checkpoints, static / dynamic activation quantisation, E8M0 and MX weights."""
import warnings

import pytest
import torch

from dist_utils import run_distributed


def test_config_enums_and_bounds():
    from neuronx_distributed_b200.quantization.quantization_config import (
        ActivationQuantizationType, DtypeBound, KVQuantizationConfig, QuantizationType, QuantizedDtype, ScaleDtype,
        get_default_blockwise_custom_qconfig_dict, get_default_custom_qconfig_dict, is_ocp_mx_quantized,
        validate_block_axis_size)

    assert "per_channel_symmetric" in QuantizationType and "nope" not in QuantizationType
    assert torch.int8 in QuantizedDtype and torch.float64 not in QuantizedDtype
    assert QuantizedDtype.get_dtype("f8e4m3") == torch.float8_e4m3fn and QuantizedDtype.F8E4M3FN is QuantizedDtype.F8E4M3
    assert QuantizedDtype.F4E2M1FN_X4.get_packed_count() == 4 and QuantizedDtype.INT8.get_packed_count() == 1
    assert not QuantizedDtype.INT8.is_float() and QuantizedDtype.F8E5M2.is_float()
    assert ScaleDtype.F8E8M0.get_default_scale() == 127 and ScaleDtype.F32.get_default_scale() == 1.0
    assert ScaleDtype.get_dtype("f8e8m0") == torch.uint8
    assert DtypeBound.from_torch_dtype(torch.int8) == (127, -128)
    assert DtypeBound.from_torch_dtype(torch.float8_e4m3fn) == (448.0, -448.0)
    with pytest.raises(ValueError):
        DtypeBound.from_torch_dtype(torch.float64)
    assert ActivationQuantizationType(None) is ActivationQuantizationType.NONE
    assert is_ocp_mx_quantized(QuantizationType.BLOCKWISE_SYMMETRIC, QuantizedDtype.F4E2M1FN_X4, ScaleDtype.F8E8M0)
    assert not is_ocp_mx_quantized(QuantizationType.BLOCKWISE_SYMMETRIC, QuantizedDtype.F8E4M3, ScaleDtype.F32)
    assert validate_block_axis_size([1], [128]) == ([1], [128])
    with pytest.raises(AssertionError):
        validate_block_axis_size([0, 1], [128])
    d = get_default_blockwise_custom_qconfig_dict()
    d["block_size"][0] = 7
    assert get_default_blockwise_custom_qconfig_dict()["block_size"] == [128]           # defaults are not aliased
    assert get_default_custom_qconfig_dict()["quantization_type"] == QuantizationType.PER_TENSOR_SYMMETRIC
    kv = KVQuantizationConfig()
    assert kv.direct_cast and kv.quant_dtype == torch.float8_e4m3fn
    with pytest.raises(AssertionError):
        KVQuantizationConfig(direct_cast=True, k_quant_method="per_key_symmetric")
    with pytest.raises(TypeError):
        KVQuantizationConfig(bogus=1)


def test_checkpoint_side_utils():
    from neuronx_distributed_b200.quantization.dequantize import (blockwise_scale_dequantize,
                                                                  get_broadcastable_shapes_for_blockwise_scale_dequantize,
                                                                  scale_dequantize)
    from neuronx_distributed_b200.quantization.observer import PerChannelAbsMaxObserver
    from neuronx_distributed_b200.quantization.quantization_utils import (
        QuantizedLinear, convert_qint8_to_int8_state_dict, extract_q_scale, quantize_blockwise, quantize_fp8_per_channel,
        quantize_fp8_per_tensor, quantize_per_channel_symmetric, quantize_per_tensor_symmetric,
        quantize_pytorch_model_per_channel_symmetric, quantize_pytorch_model_per_tensor_symmetric,
        quantize_static_quant_activations)
    from neuronx_distributed_b200.quantization.quantize import direct_cast_quantize

    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.ReLU(), torch.nn.Linear(32, 8))
    x = torch.randn(4, 16)
    ref = m(x)
    for fn, shape in ((quantize_pytorch_model_per_tensor_symmetric, (1,)), (quantize_pytorch_model_per_channel_symmetric, (32, 1))):
        for dt, tol in ((torch.qint8, 0.02), (torch.float8_e4m3fn, 0.08)):
            q = fn(m, dtype=dt)
            assert isinstance(q[0], QuantizedLinear) and q[0].scale.shape == shape and isinstance(m[0], torch.nn.Linear)
            assert set(q.state_dict()) == {"0.weight", "0.scale", "0.bias", "2.weight", "2.scale", "2.bias"}
            assert (q(x) - ref).abs().max() / ref.abs().max() < tol
    q = quantize_pytorch_model_per_channel_symmetric(m, modules_to_not_convert=["2"])
    assert isinstance(q[2], torch.nn.Linear) and isinstance(q[0], QuantizedLinear)
    with pytest.raises(ValueError):
        quantize_pytorch_model_per_tensor_symmetric(m, dtype=torch.float16)

    w = m[0].weight.detach()
    qt, qc = quantize_per_tensor_symmetric(w), quantize_per_channel_symmetric(w, 0)
    assert extract_q_scale(qt).shape == (1,) and extract_q_scale(qc).shape == (32, 1)
    assert (qc.dequantize() - w).abs().max() < extract_q_scale(qc).max()
    # torch-packed dynamic-quantisation state dict → plain int8 state dict
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        packed = torch.ao.quantization.quantize_dynamic(m, {torch.nn.Linear}, dtype=torch.qint8).state_dict()
    convert_qint8_to_int8_state_dict(packed)
    assert packed["0.weight"].dtype == torch.int8 and packed["0.scale"].shape == (1,) and packed["0.bias"].shape == (32,)

    obs = PerChannelAbsMaxObserver.with_args(ch_axis=0)()
    obs(w); obs(2 * w)
    s, z = obs.calculate_qparams()
    torch.testing.assert_close(s, 2 * w.abs().amax(1) / 127) and (z == 0).all()

    q8 = quantize_static_quant_activations(torch.tensor([[0.5, -3.0, 100.0]]), torch.tensor([0.5]), torch.int8)
    assert q8.tolist() == [[1, -6, 127]]
    wq, s = quantize_fp8_per_channel(w, torch.float8_e4m3fn, 0)
    assert s.shape == (32, 1) and (wq.float() * s - w).abs().max() / w.abs().max() < 0.07
    wq, s = quantize_fp8_per_tensor(w, torch.float8_e5m2)
    assert wq.dtype == torch.float8_e5m2 and s.dim() == 0
    assert direct_cast_quantize(w, torch.float8_e4m3fn).dtype == torch.float8_e4m3fn

    # blockwise: one scale per (row, 8-column block) and per 2-D (4×8) block
    assert get_broadcastable_shapes_for_blockwise_scale_dequantize((32, 16), (32, 2)) == ((32, 2, 8), (32, 2, 1))
    assert get_broadcastable_shapes_for_blockwise_scale_dequantize((32, 16), (8,)) == ((8, 4, 1, 16), (8, 1, 1, 1))
    for axes, sizes in (([1], [8]), ([0, 1], [4, 8])):
        bq, bs = quantize_blockwise(w, torch.float8_e4m3fn, axes, sizes)
        back = blockwise_scale_dequantize(bq, bs, torch.float32)
        assert (back - w).abs().max() / w.abs().max() < 0.07
    with pytest.raises(AssertionError):
        get_broadcastable_shapes_for_blockwise_scale_dequantize((4, 4), (4, 4))
    y = torch.ones(2, 3, 5)
    assert scale_dequantize(y, torch.arange(5.0).reshape(5, 1), torch.float32)[0, 0].tolist() == [0, 1, 2, 3, 4]


def test_mx_transform_weights_and_experimental_oracles():
    from neuronx_distributed_b200.experimental.quantization.microscaling import expert_mlps_mx as em
    from neuronx_distributed_b200.experimental.quantization.microscaling import swizzle
    from neuronx_distributed_b200.experimental.quantization.microscaling.mx_torch import (dequantize_mx_tensor, matmul_mx,
                                                                                           quantize_mxfp8)
    from neuronx_distributed_b200.quantization.microscaling import transform_weights as tw

    torch.manual_seed(0)
    w = torch.randn(16, 256)
    blocks, scales = tw.quantize_to_mxfp4(w)
    assert blocks.shape == (16, 8, 16) and blocks.dtype == torch.uint8 and scales.shape == (16, 8)
    deq = tw.get_mxfp4_tensor(blocks, scales, dtype=torch.float32)
    assert (deq - w).abs().max() / w.abs().max() < 0.3
    codes = tw.split_byte_4bit_tensor(blocks)
    assert codes.shape == (16, 8, 32) and codes.max() < 16 and torch.equal(tw.pack_byte_4bit_tensor(codes), blocks)
    torch.testing.assert_close(tw.dequant_byte_4bit_tensor(codes, scales).float(), deq.bfloat16().float())
    assert torch.equal(tw.apply_lut_byte_4bit_tensor(codes[..., :1, :]).reshape(-1)[:4],
                       torch.tensor(tw.FP4_VALUES)[codes[0, 0, :4].long()])
    x4 = tw.pack_fp4_x4_uint16(blocks)
    assert x4.dtype == torch.uint16 and x4.shape == (16, 8, 8)
    assert torch.equal(tw.get_mxfp4_tensor_from_uint16(x4, scales, dtype=torch.float32), deq)
    assert tw.get_mxfp4_tensor_from_uint16(x4, scales, output_quad_row=True).shape == (16, 64, 4)
    assert tw.pack_fp4_x4_uint16(blocks.numpy()).dtype.name == "uint16"
    # fp8_x4
    p8, s8 = quantize_mxfp8(w.bfloat16())
    assert p8.dtype == torch.uint32 and p8.shape == (16, 64) and s8.shape == (16, 8)
    d8 = tw.get_mxfp8_tensor_from_uint32(p8.reshape(16, 8, 8), s8, dtype=torch.float32)
    assert (d8 - w).abs().max() / w.abs().max() < 0.13
    assert torch.equal(dequantize_mx_tensor(p8, s8, torch.float32), d8)
    assert torch.equal(dequantize_mx_tensor(p8, s8, torch.float32, output_is_transposed=True), d8.t())
    unb, _ = quantize_mxfp8(w.bfloat16(), use_unbiased_scale=True)       # no saturation: every element within 2^-3 relative
    a = torch.randn(8, 256)
    ap, asc = quantize_mxfp8(a.bfloat16())
    y = matmul_mx(ap, x4.reshape(16, -1), asc, scales, output_dtype=torch.float32)
    assert (y - a @ w.t()).abs().max() / (a @ w.t()).abs().max() < 0.25
    # gate/up de-interleave + padding helper
    W = torch.randint(0, 255, (2, 6, 2, 16), dtype=torch.uint8)
    S = torch.randint(120, 130, (2, 6, 2), dtype=torch.uint8)
    B = torch.randn(2, 6)
    wg, sg, bg, wu, su, bu = tw.split_gate_up(W, S, B)
    assert torch.equal(wg, W[:, 0::2]) and torch.equal(su, S[:, 1::2]) and torch.equal(bu, B[:, 1::2]) and wg.is_contiguous()
    wp, sp, bp = tw.reshape_pad_proj(torch.zeros(2, 96, 3, 8, dtype=torch.uint8), torch.full((2, 96, 3), 126, dtype=torch.uint8),
                                     torch.ones(2, 96), pad_multiple=128)
    assert wp.shape == (2, 128, 32) and sp.shape == (2, 128, 4) and bp.shape == (2, 128)
    assert sp[0, 100, 0] == 127 and sp[0, 0, 3] == 127 and sp[0, 0, 0] == 126 and bp[0, 100] == 0

    # swizzles: data permutation round trip; scale-factor tile interleave matches the byte formula
    t = torch.arange(8 * 3).reshape(8, 3)
    s = swizzle.swizzle_tensor(t)
    assert s[0].tolist() == [0, 3, 6, 9, 1, 4, 7, 10, 2, 5, 8, 11] and torch.equal(swizzle.unswizzle_tensor(s, 8, 3), t)
    assert swizzle.swizzle_tiled_tensor(torch.randn(8, 8, 5)).shape == (8, 2, 20)
    sc = torch.randint(0, 255, (200, 6), dtype=torch.uint8)
    stream = swizzle.swizzle_scale_factors(sc)
    assert stream.numel() == 256 * 8 and torch.equal(swizzle.unswizzle_scale_factors(stream, 200, 6), sc)
    for r, c in ((70, 2), (130, 5), (199, 0)):
        band, rr, kt, cc = r // 128, r % 128, c // 4, c % 4
        assert stream[(band * 2 + kt) * 512 + (rr % 32) * 16 + (rr // 32) * 4 + cc] == sc[r, c]

    # MoE oracles: dense == select; MXFP4-weight/MXFP8-activation tracks the float result
    T, H, I, E = 6, 64, 96, 8
    xn, rl = torch.randn(T, H).bfloat16(), torch.randn(T, E)
    Wg, Wu, Wd = torch.randn(E, I, H) * 0.2, torch.randn(E, I, H) * 0.2, torch.randn(E, H, I) * 0.2
    bg, bu, bd = torch.randn(E, I) * 0.1, torch.randn(E, I) * 0.1, torch.randn(E, H) * 0.1
    ref = em.all_expert_mlps_bf16(xn.float(), rl, Wg, Wu, Wd, bg, bu, bd)
    torch.testing.assert_close(em.select_expert_mlps_bf16(xn.float(), rl, Wg, Wu, Wd, bg, bu, bd), ref, rtol=1e-4, atol=1e-5)

    def q(wt):
        b, s_ = tw.quantize_to_mxfp4(wt)
        return tw.pack_fp4_x4_uint16(b).reshape(*wt.shape[:-1], -1), s_

    (qg, sg_), (qu, su_), (qd, sd_) = q(Wg), q(Wu), q(Wd)
    y = em.all_expert_mlps_act_mxfp8_w_mxfp4(xn, qg, qu, qd, sg_, su_, sd_, bg, bu, bd, router_logits=rl)
    assert y.shape == (T, H) and (y.float() - ref).abs().max() / ref.abs().max() < 0.35


def _layers(rank, world):
    from neuronx_distributed_b200.inference.sharding import shard_state_dict_for_rank
    from neuronx_distributed_b200.parallel_layers import ColumnParallelLinear, RowParallelLinear
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.quantization import ActivationQuantizationType, QuantizationType, QuantizedDtype, ScaleDtype, convert
    from neuronx_distributed_b200.quantization.quantization_config import (get_default_blockwise_custom_qconfig_dict,
                                                                           get_default_custom_qconfig_dict,
                                                                           get_default_per_channel_custom_qconfig_dict)
    from neuronx_distributed_b200.quantization.quantization_layers import (BaseQuantizeParallelLinear, QuantizedColumnParallel,
                                                                           QuantizedRowParallel)
    from neuronx_distributed_b200.quantization.quantization_utils import quantize_pytorch_model_per_channel_symmetric

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    H, F = 64, 128

    class Float(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.up, self.down = torch.nn.Linear(H, F), torch.nn.Linear(F, H)

        def forward(self, x):
            return self.down(torch.relu(self.up(x)))

    class Par(torch.nn.Module):
        def __init__(self, **kw):
            super().__init__()
            self.up = QuantizedColumnParallel(H, F, gather_output=False, **kw)
            self.down = QuantizedRowParallel(F, H, input_is_parallel=True, **kw)

        def forward(self, x):
            return self.down(torch.relu(self.up(x)))

    fm = Float().eval()
    x = torch.randn(5, H)
    ref = fm(x)

    # (1) empty quantised TP model ← plain quantised checkpoint (int8 and fp8), sharded per rank
    for dt, tol in ((torch.qint8, 0.02), (torch.float8_e4m3fn, 0.08)):
        full_sd = quantize_pytorch_model_per_channel_symmetric(fm, dtype=dt).state_dict()
        qd = QuantizedDtype.INT8 if dt == torch.qint8 else QuantizedDtype.F8E4M3
        pm = Par(quantization_type="per_channel_symmetric", quantized_dtype=qd).eval()
        assert isinstance(pm.up, BaseQuantizeParallelLinear) and pm.up.weight.shape == (F // world, H)
        assert pm.up.scale.shape == (F // world, 1) and pm.up.scale.tensor_model_parallel
        assert pm.down.scale.shape == (H, 1) and not pm.down.scale.tensor_model_parallel and not pm.up.weight.requires_grad
        pm.load_state_dict(shard_state_dict_for_rank(pm, full_sd, rank, world))
        err = (pm(x) - ref).abs().max() / ref.abs().max()
        assert err < tol, (dt, float(err))

    # (2) torch dynamic-quantisation (packed qint8, per-tensor) checkpoint through the state-dict adaptor
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        packed_sd = torch.ao.quantization.quantize_dynamic(fm, {torch.nn.Linear}, dtype=torch.qint8).state_dict()
    pm = Par(quantization_type="per_tensor_symmetric", quantized_dtype=torch.int8).eval()
    local = shard_state_dict_for_rank(pm, packed_sd, rank, world)
    assert set(local) == {"up.weight", "up.scale", "up.bias", "down.weight", "down.scale", "down.bias"}, sorted(local)
    pm.load_state_dict(local)
    assert (pm(x) - ref).abs().max() / ref.abs().max() < 0.03

    # (3) convert() from float parallel layers: every scheme; replicated scales agree across ranks
    par = torch.nn.Sequential(ColumnParallelLinear(H, F, bias=True, gather_output=False),
                              RowParallelLinear(F, H, bias=True, input_is_parallel=True)).eval()
    pref = par(x)
    cases = [
        (get_default_custom_qconfig_dict(), 0.03),
        ({**get_default_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3,
          "activation_quantization_type": ActivationQuantizationType.STATIC}, 0.12),
        ({**get_default_per_channel_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3,
          "activation_quantization_type": ActivationQuantizationType.DYNAMIC, "clamp_bound": 50.0}, 0.12),
        ({**get_default_per_channel_custom_qconfig_dict(), "activation_quantization_type": ActivationQuantizationType.DYNAMIC}, 0.12),
        ({**get_default_per_channel_custom_qconfig_dict(), "quantization_per_channel_axis": 1}, 0.03),
        ({**get_default_blockwise_custom_qconfig_dict(), "block_axis": [0, 1], "block_size": [16, 32]}, 0.08),
        ({**get_default_blockwise_custom_qconfig_dict(), "block_axis": [1], "block_size": [32], "scale_dtype": ScaleDtype.F8E8M0}, 0.12),
        ({**get_default_blockwise_custom_qconfig_dict(), "block_axis": [1], "block_size": [32],
          "quantized_dtype": QuantizedDtype.F8E4M3FN_X4, "scale_dtype": ScaleDtype.F8E8M0}, 0.15),
        ({**get_default_blockwise_custom_qconfig_dict(), "block_axis": [1], "block_size": [32],
          "quantized_dtype": QuantizedDtype.F4E2M1FN_X4, "scale_dtype": ScaleDtype.F8E8M0}, 0.45),
    ]
    for cfg, tol in cases:
        q = convert(par, cfg)
        if cfg.get("activation_quantization_type") == ActivationQuantizationType.STATIC:
            assert q[0].input_scale.shape == (1,)
            q[0].input_scale.data.fill_(float(x.abs().max()) / 448.0)
            q[1].input_scale.data.fill_(float(torch.relu(q[0](x)).abs().max()) / 448.0 * 1.5)
        err = float((q(x) - pref).abs().max() / pref.abs().max())
        assert err < tol, (cfg["quantization_type"], cfg["quantized_dtype"], err)
        if cfg["quantization_type"] == QuantizationType.PER_TENSOR_SYMMETRIC and world > 1:
            g = [torch.zeros(1) for _ in range(world)]
            torch.distributed.all_gather(g, q[0].scale.data.float())
            assert all(torch.equal(t, g[0]) for t in g)
        if cfg["quantized_dtype"] == QuantizedDtype.F4E2M1FN_X4:
            assert q[0].weight.dtype == torch.uint16 and q[0].weight.shape == (F // world, H // 4)
            assert q[0].scale.dtype == torch.uint8 and q[0].scale.shape == (F // world, H // 32)
        sd = q.state_dict()                                     # quantised checkpoints round-trip through state_dict
        q2 = convert(par, cfg)
        q2.load_state_dict(sd)
        torch.testing.assert_close(q2(x), q(x))

    # (4) include patterns / deny list / exclusivity
    q = convert(par, get_default_custom_qconfig_dict(), include=["1"])
    assert isinstance(q[0], ColumnParallelLinear) and isinstance(q[1], QuantizedRowParallel)
    q = convert(par, get_default_custom_qconfig_dict(), modules_to_not_convert=["0"])
    assert isinstance(q[0], ColumnParallelLinear) and isinstance(q[1], QuantizedRowParallel)
    try:
        convert(par, None, include=["0"], modules_to_not_convert=["1"])
        raise SystemExit("include + modules_to_not_convert must be rejected")
    except AssertionError:
        pass

    # (5) padded output dim: preshard hook pads weight and per-channel scale of a full checkpoint
    cp = QuantizedColumnParallel(H, 30, bias=False, gather_output=True, pad=True, quantization_type="per_channel_symmetric").eval()
    assert cp.pad_size == (-30) % world and cp.weight.shape[0] == (30 + cp.pad_size) // world
    lin = torch.nn.Linear(H, 30, bias=False)
    full = quantize_pytorch_model_per_channel_symmetric(torch.nn.Sequential(lin)).state_dict()
    full = {k[2:]: v for k, v in full.items() if v is not None}
    cp.load_state_dict(shard_state_dict_for_rank(cp, full, rank, world))
    out = cp(x)
    assert out.shape == (5, 30) and (out - lin(x)).abs().max() / lin(x).abs().max() < 0.02


def test_quantized_layers_checkpoints_tp2():
    run_distributed(_layers, 2, timeout=150)


def _experts(rank, world):
    from neuronx_distributed_b200.modules.moe.moe_parallel_layers import (ExpertFusedColumnParallelLinear,
                                                                          ExpertFusedRowParallelLinear)
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.quantization import QuantizedDtype, ScaleDtype, convert
    from neuronx_distributed_b200.quantization.quantization_config import (
        get_default_blockwise_custom_qconfig_dict, get_default_custom_qconfig_dict,
        get_default_expert_wise_per_channel_custom_qconfig_dict, get_default_per_channel_custom_qconfig_dict)
    from neuronx_distributed_b200.quantization.quantization_layers import (QuantizedExpertFusedColumnParallel,
                                                                           QuantizedExpertFusedRowParallel)

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    torch.manual_seed(0)
    E, H, I, C = 4, 32, 64, 5
    m = torch.nn.Sequential()
    m.add_module("up", ExpertFusedColumnParallelLinear(E, H, I, bias=True))
    m.add_module("down", ExpertFusedRowParallelLinear(E, I, H, bias=True, reduce_output=True))
    with torch.no_grad():
        m.up.bias.normal_(); m.down.bias.normal_()
    x = torch.randn(E, C, H)

    def run(mod, idx=None):
        xx = x if idx is None else x[idx]
        return mod.down(torch.relu(mod.up(xx, idx)), idx)

    # float layer: bias broadcast + autograd function (dgrad all-reduce) sanity
    xr = x.clone().requires_grad_(True)
    m.down(torch.relu(m.up(xr))).sum().backward()
    assert xr.grad is not None and m.up.weight.grad.shape == m.up.weight.shape
    g = [torch.zeros_like(xr.grad) for _ in range(world)]
    torch.distributed.all_gather(g, xr.grad)
    assert all(torch.allclose(t, g[0]) for t in g)                      # input grads identical on every TP rank
    m.zero_grad()
    with torch.no_grad():
        ref, ref_sel = run(m), run(m, torch.tensor([2, 0]))
        for cfg, tol in (
            (get_default_custom_qconfig_dict(), 0.05),
            (get_default_per_channel_custom_qconfig_dict(), 0.03),
            ({**get_default_expert_wise_per_channel_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.INT8}, 0.03),
            (get_default_expert_wise_per_channel_custom_qconfig_dict(), 0.08),
            ({**get_default_blockwise_custom_qconfig_dict(), "block_axis": [1], "block_size": [16]}, 0.08),
            ({**get_default_blockwise_custom_qconfig_dict(), "block_axis": [1, 2], "block_size": [16, 16],
              "scale_dtype": ScaleDtype.F8E8M0}, 0.12),
        ):
            q = convert(m, cfg)
            assert isinstance(q.up, QuantizedExpertFusedColumnParallel) and isinstance(q.down, QuantizedExpertFusedRowParallel)
            assert q.up.weight.shape == (E, H, I // world) and q.down.weight.shape == (E, I // world, H)
            if cfg["quantization_type"].value == "expert_wise_per_channel_symmetric":
                assert q.up.scale.shape == (E, 1, I // world) and q.down.scale.shape == (E, 1, H)
            err = float((run(q) - ref).abs().max() / ref.abs().max())
            assert err < tol, (cfg["quantization_type"], cfg["quantized_dtype"], err)
            err = float((run(q, torch.tensor([2, 0])) - ref_sel).abs().max() / ref_sel.abs().max())
            assert err < tol, ("selected", cfg["quantization_type"], err)
    # built empty with the reference's constructor signature
    e = QuantizedExpertFusedColumnParallel(num_experts=E, input_size=H, output_size=I, quantization_type="per_channel_symmetric",
                                           quantized_dtype=QuantizedDtype.F8E4M3, dtype=torch.bfloat16)
    assert e.weight.dtype == torch.float8_e4m3fn and e.scale.shape == (1, 1, I // world) and e.bias is None
    assert e(x.bfloat16()).shape == (E, C, I // world)


def test_quantized_expert_layers_tp2():
    run_distributed(_experts, 2, timeout=150)


def test_linear_mx_matches_mx_matmul_oracle():
    """``ops.gemm_mx.linear_mx`` (the de-quantise + GEMM path every non-decode call takes) equals the MX oracle for both packings,
    leading dims and a residual; x4 words and raw bytes are the same stream."""
    import torch

    from neuronx_distributed_b200.ops import gemm_mx
    from neuronx_distributed_b200.quantization.microscaling.mx_torch import mx_matmul, quantize_mx

    torch.manual_seed(0)
    w, x, r = torch.randn(24, 96), torch.randn(2, 3, 96), torch.randn(2, 3, 24)
    for kind in ("mxfp4", "mxfp8"):
        p, s = quantize_mx(w, kind)
        assert gemm_mx.kind_of(p) == kind
        want = mx_matmul(x.reshape(-1, 96), p, s, kind, torch.float32).view(2, 3, 24) + r
        torch.testing.assert_close(gemm_mx.linear_mx(x, p, s, residual=r), want)
        torch.testing.assert_close(gemm_mx.linear_mx(x, p.view(torch.uint8), s, kind=kind, residual=r), want)
    assert not gemm_mx.gemv_eligible(x.reshape(-1, 96), p, s)            # CPU / opt-in flag unset


def test_mx_scale_tiling_layout():
    """``tile_scales``: byte (r % 32) * 16 + (r // 32) * 4 + j of chunk (row tile, K block of 128) = scale (r, j); padding = 2^0."""
    import torch

    from neuronx_distributed_b200.ops import gemm_mx

    s = torch.arange(200 * 8, dtype=torch.int32).remainder(251).to(torch.uint8).reshape(200, 8)
    t = gemm_mx.tile_scales(s)
    assert t.shape == (2, 2, 512)
    for r, kb in ((0, 0), (33, 5), (127, 7), (130, 2), (199, 4)):
        rr = r % 128
        assert t[r // 128, kb // 4, (rr % 32) * 16 + (rr // 32) * 4 + kb % 4] == s[r, kb]
    assert (t[1, :, (100 % 32) * 16 + (100 // 32) * 4] == 127).all()      # row 228 does not exist: scale 1.0
    # the oracle of the block-scaled GEMM is the plain product of the de-quantised operands
    from neuronx_distributed_b200.quantization.microscaling.mx_torch import quantize_mxfp8

    a, b = torch.randn(8, 64), torch.randn(5, 64)
    (aq, asc), (bq, bsc) = quantize_mxfp8(a), quantize_mxfp8(b)
    ref = gemm_mx.matmul_mxfp8_reference(aq, asc, bq, bsc)
    assert ((ref - a @ b.t()).norm() / (a @ b.t()).norm()) < 0.08


def test_fp4_gemm_quantisers_oracle_and_scale_addressing():
    """4-bit formats: the MXFP4 / NVFP4 quantisers (round-to-nearest-even on the e2m1 grid),
    the oracle, and a replay of the kernel's scale addressing — which chunk column and which scale bytes each K=64 MMA reads —
    against the un-tiled scale matrix."""
    import torch

    from neuronx_distributed_b200.ops import gemm_mx

    torch.manual_seed(0)
    assert gemm_mx._e2m1_codes(torch.tensor([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, -0.75, 7.0])).tolist() == [0, 2, 2, 4, 4, 6, 6, 10, 7]
    a, b = torch.randn(40, 512) * torch.rand(40, 1) * 3, torch.randn(24, 512)
    want = a @ b.t()
    aq, asc = gemm_mx.quantize_mxfp4(a)
    bq, bsc = gemm_mx.quantize_mxfp4(b)
    assert aq.shape == (40, 256) and asc.shape == (40, 16) and asc.dtype == torch.uint8
    assert torch.equal(gemm_mx.dequantize_f4(aq, asc, 32), gemm_mx.dequantize(aq, asc, "mxfp4"))        # same decode as the MX layers
    assert ((gemm_mx.matmul_f4_reference(aq, asc, bq, bsc, 32) - want).norm() / want.norm()) < 0.2
    aq, asc, ag = gemm_mx.quantize_nvfp4(a)
    bq, bsc, bg = gemm_mx.quantize_nvfp4(b)
    assert asc.shape == (40, 32) and float(ag) > 0
    e_mx = ((gemm_mx.dequantize_f4(*gemm_mx.quantize_mxfp4(a), 32) - a).norm() / a.norm()).item()
    e_nv = ((gemm_mx.dequantize_f4(aq, asc, 16, ag) - a).norm() / a.norm()).item()
    assert e_nv < e_mx < 0.15                                           # finer blocks + e4m3 scales round better than 2^k per 32
    assert ((gemm_mx.matmul_f4_reference(aq, asc, bq, bsc, 16, ag, bg) - want).norm() / want.norm()) < 0.15
    # kernel-side addressing: a k-block is 256 elements; chunk = 128 rows x 4 consecutive scales at byte (r%32)*16 + (r//32)*4 + j;
    # MXFP4: 2 chunks per k-block, MMA k reads bytes {sf_id, sf_id+1} (sf_id = 2·(k&1)) of chunk k>>1;
    # NVFP4: 4 chunks per k-block, MMA k reads bytes 0..3 of chunk k
    R, K = 200, 1024
    for vs, pad in ((32, 127), (16, 0x38)):
        sc = torch.randint(1, 250, (R, K // vs), dtype=torch.uint8)
        t = gemm_mx.tile_scales(sc, pad)
        ch = 256 // (4 * vs)
        assert t.shape == (2, K // 256 * ch, 512)
        for r in (0, 31, 32, 127, 128, 199):
            tile, rr = r // 128, r % 128
            base = (rr % 32) * 16 + (rr // 32) * 4
            for kb in range(K // 256):
                for k in range(4):                                         # the four K=64 MMAs of the k-block
                    chunk, sf_id, nsf = (kb * ch + (k >> 1), 2 * (k & 1), 2) if vs == 32 else (kb * ch + k, 0, 4)
                    got = t[tile, chunk, base + sf_id: base + sf_id + nsf]
                    first = (kb * 256 + k * 64) // vs
                    assert torch.equal(got, sc[r, first: first + nsf]), (vs, r, kb, k)
        assert t[1, 0, (100 % 32) * 16 + (100 // 32) * 4] == pad           # row 228 does not exist
    assert not gemm_mx.gemm_f4_eligible(128, 128, 256, a)                  # CPU / opt-in flag unset


def test_grouped_linear_mx_selects_experts_per_row():
    """``grouped_linear_mx`` (selective loading of a decode MoE block on MX weights): row s uses expert ``expert[s]``."""
    import torch

    from neuronx_distributed_b200.ops import gemm_mx
    from neuronx_distributed_b200.quantization.microscaling.mx_torch import quantize_mx

    torch.manual_seed(0)
    E, N, K, S = 4, 6, 64, 5
    w, x, ex = torch.randn(E, N, K), torch.randn(S, K), torch.tensor([3, 0, 0, 2, 1])
    for kind in ("mxfp4", "mxfp8"):
        p, sc = quantize_mx(w, kind)
        want = torch.stack([x[i] @ gemm_mx.dequantize(p[ex[i]], sc[ex[i]], kind).t() for i in range(S)])
        torch.testing.assert_close(gemm_mx.grouped_linear_mx(x, p, sc, ex), want, rtol=1e-5, atol=1e-5)
