"""Quantised MoE experts on the dropless (blockwise) prefill path, on CPU.

* Weight-only experts (block-wise e4m3, per-channel e4m3 and int8): ``forward_blockwise`` and prefill ``forward`` run and
  match float64 computed from the de-quantised weights.  Before, the grouped projection multiplied the activations by the
  raw e4m3 / int8 weight and raised.
* W8A8 experts (block-wise e4m3, dynamic activations): ``forward_blockwise``, ``forward_all_experts`` and
  ``forward_selective_loading`` all match one float64 reference built from per-token group-quantised activations and
  de-quantised weights, for 1-D and 128 × 128 blocks and fp32 and E8M0 scales.
* The K-major relayout of a W8A8 expert weight changes neither ``state_dict()`` nor the ``_linear_experts`` outputs.
"""
import pytest
import torch

from dist_utils import run_distributed

E, TOP_K, H, I, T = 4, 2, 256, 256, 64
# fp32 model on CPU: the only roundings are fp32 sums and, for W8A8, e4m3 codes of values that reach the quantiser after
# fp32 rather than float64 arithmetic (a code can move by one step where a value sits within ~2^-23 of a rounding midpoint).
# 2^-8 of the largest output (bf16's unit roundoff) bounds both with a wide margin.
BOUND = 2.0 ** -8


def _setup():
    from neuronx_distributed_b200.modules.moe import ExpertMLPsV2, RoutedExpertsMLPOpsConfig
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(1)
    torch.manual_seed(0)
    cfg = RoutedExpertsMLPOpsConfig(normalize_top_k_affinities=True, num_experts=E, top_k=TOP_K, hidden_size=H,
                                    intermediate_size=I)
    em = ExpertMLPsV2(cfg).eval()
    x = torch.randn(T, H)
    aff = torch.softmax(torch.randn(T, E), -1)
    idx = aff.topk(TOP_K, -1).indices
    return em, x, aff, idx


def _dequant64(layer):
    from neuronx_distributed_b200.quantization.quantization_config import QuantizationType

    w = layer.weight.double() if layer.weight.dtype != torch.int8 else layer.weight.to(torch.float64)
    s = layer.scale.double() if layer.scale.dtype != torch.uint8 else torch.pow(2.0, layer.scale.double() - 127)
    if layer.quantization_type == QuantizationType.BLOCKWISE_SYMMETRIC:
        for ax in (1, 2):
            s = s.repeat_interleave(w.shape[ax] // s.shape[ax], ax)
    return w * s


def _quant64(x, G):
    """Per-token group quantisation (absmax / 448, e4m3 round-to-nearest-even) and its float64 de-quantisation."""
    from neuronx_distributed_b200.ops.gemm_fp8 import _quantize_groups_reference

    q, s = _quantize_groups_reference(x.reshape(-1, x.shape[-1]).float(), G, "absmax", None)
    return (q.double().reshape(q.shape[0], -1, G) * s.double().unsqueeze(-1)).reshape(x.shape)


def _reference64(qm, x, aff, idx, G=0):
    """out[t] = Σ_j a[t, e_j] · down_e(silu(gate_e(x)) · up_e(x)) in float64; with G, each projection's input is
    group-quantised per token first (the second from its fp32 value, as the layer computes it)."""
    ex = qm.get_mlp_op()
    w1, w2 = _dequant64(ex.gate_up_proj), _dequant64(ex.down_proj)
    a = aff.double().gather(1, idx)
    a = a / a.sum(-1, keepdim=True)
    out = torch.zeros(T, H, dtype=torch.float64)
    for j in range(TOP_K):
        for e in range(E):
            t = (idx[:, j] == e).nonzero().flatten()
            if t.numel() == 0:
                continue
            xi = _quant64(x[t], G) if G else x[t].double()
            g, u = (xi @ w1[e]).chunk(2, -1)
            hmid = torch.nn.functional.silu(g) * u
            hi = _quant64(hmid.float(), G) if G else hmid
            out[t] += a[t, j:j + 1] * (hi @ w2[e])
    return out


def _close(got, want, what):
    err = (got.double() - want).abs().max().item()
    assert err <= BOUND * want.abs().max().item(), f"{what}: max error {err} vs max |ref| {want.abs().max().item()}"


def _weight_only(rank, world):
    from neuronx_distributed_b200.quantization import QuantizedDtype, convert
    from neuronx_distributed_b200.quantization.quantization_config import (get_default_blockwise_custom_qconfig_dict,
                                                                           get_default_per_channel_custom_qconfig_dict)

    em, x, aff, idx = _setup()
    cfgs = {"blockwise e4m3": {**get_default_blockwise_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3,
                               "block_axis": [1], "block_size": [128]},
            "per-channel e4m3": {**get_default_per_channel_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3},
            "per-channel int8": {**get_default_per_channel_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.INT8}}
    for name, q in cfgs.items():
        qm = convert(em, q_config=q, inplace=False)
        assert qm.get_mlp_op().gate_up_proj._blockscaled_group() == 0
        want = _reference64(qm, x, aff, idx)
        _close(qm.forward_blockwise(x, aff, idx), want, f"{name} forward_blockwise")
        _close(qm(x, aff, idx, seq_len=T), want, f"{name} prefill forward")


def test_weight_only_experts_run_the_dropless_path():
    run_distributed(_weight_only, 1, timeout=180)


def _w8a8(rank, world):
    from neuronx_distributed_b200.quantization import ActivationQuantizationType, QuantizedDtype, ScaleDtype, convert
    from neuronx_distributed_b200.quantization.quantization_config import get_default_blockwise_custom_qconfig_dict

    em, x, aff, idx = _setup()
    base = {**get_default_blockwise_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3,
            "activation_quantization_type": ActivationQuantizationType.DYNAMIC}
    for q in ({**base, "block_axis": [1], "block_size": [128]},
              {**base, "block_axis": [1], "block_size": [32], "scale_dtype": ScaleDtype.F8E8M0},
              {**base, "block_axis": [1, 2], "block_size": [128, 128]},
              {**base, "block_axis": [1, 2], "block_size": [64, 128], "scale_dtype": ScaleDtype.F8E8M0}):
        qm = convert(em, q_config=q, inplace=False)
        G = q["block_size"][0]
        for layer in (qm.get_mlp_op().gate_up_proj, qm.get_mlp_op().down_proj):
            assert layer.activation_quantization_type == ActivationQuantizationType.DYNAMIC
            assert layer._blockscaled_group() == G
            assert layer.weight.transpose(1, 2).is_contiguous()          # relaid out K-major by the constructor
        want = _reference64(qm, x, aff, idx, G)
        what = f"block {q['block_axis']} {q['block_size']} {q.get('scale_dtype')}"
        _close(qm.forward_blockwise(x, aff, idx), want, what + " forward_blockwise")
        _close(qm.forward_all_experts(x, aff, idx), want, what + " forward_all_experts")
        _close(qm.forward_selective_loading(x, aff, idx), want, what + " forward_selective_loading")
        _close(qm(x, aff, idx, seq_len=T), want, what + " prefill forward")
        # activation quantisation matters: the weight-only model of the same weights is measurably different
        wo = _reference64(qm, x, aff, idx)
        assert (wo - want).abs().max() > 2 ** -6 * want.abs().max()


def test_w8a8_experts_agree_in_every_routing_mode():
    run_distributed(_w8a8, 1, timeout=240)


def _relayout(rank, world):
    from neuronx_distributed_b200.quantization import ActivationQuantizationType, QuantizedDtype, convert
    from neuronx_distributed_b200.quantization.quantization_config import get_default_blockwise_custom_qconfig_dict

    em, x, aff, idx = _setup()
    q = {**get_default_blockwise_custom_qconfig_dict(), "quantized_dtype": QuantizedDtype.F8E4M3, "block_axis": [1],
         "block_size": [128]}
    wo = convert(em, q_config=q, inplace=False).get_mlp_op()
    qm = convert(em, q_config={**q, "activation_quantization_type": ActivationQuantizationType.DYNAMIC}, inplace=False)
    ex = qm.get_mlp_op()
    xe = x.unsqueeze(0).expand(E, T, H)
    for name in ("gate_up_proj", "down_proj"):
        layer, plain = getattr(ex, name), getattr(wo, name)
        assert not plain.weight.transpose(1, 2).is_contiguous() and plain.weight.is_contiguous()   # weight-only: untouched
        assert layer.weight.transpose(1, 2).is_contiguous()
        # the same bytes as the weight-only layer quantised from the same float weights
        sd, sd_plain = layer.state_dict(), plain.state_dict()
        assert torch.equal(sd["weight"].view(torch.uint8), sd_plain["weight"].view(torch.uint8))
        assert torch.equal(sd["scale"], sd_plain["scale"])
        # weight-only einsum on the K-major storage: bit for bit the same as on the row-major storage
        layer.activation_quantization_type = ActivationQuantizationType.NONE
        inp = xe if name == "gate_up_proj" else torch.randn(E, T, I)
        assert torch.equal(layer._linear_experts(inp, None), plain._linear_experts(inp, None))
        layer.activation_quantization_type = ActivationQuantizationType.DYNAMIC
        y_k = layer._linear_experts(inp, None)
        # replace the storage with a row-major copy: values, outputs and state_dict bytes do not change, and the next
        # W8A8 use relays it out once
        layer.weight.data = layer.weight.data.contiguous()
        assert torch.equal(layer._linear_experts(inp, None), y_k)
        w = layer._k_major_weight()
        assert w is layer.weight and w.transpose(1, 2).is_contiguous()
        ptr = w.data_ptr()
        assert layer._k_major_weight().data_ptr() == ptr                  # not again
        assert torch.equal(layer._linear_experts(inp, None), y_k)
        assert torch.equal(layer.state_dict()["weight"].view(torch.uint8), sd_plain["weight"].view(torch.uint8))
        # loading a row-major checkpoint copies into the K-major storage
        layer.load_state_dict(sd_plain)
        assert layer.weight.data_ptr() == ptr and layer.weight.transpose(1, 2).is_contiguous()


def test_k_major_relayout_keeps_values_and_state_dict():
    run_distributed(_relayout, 1, timeout=180)


def _scales_and_refusals(rank, world):
    from neuronx_distributed_b200.ops import gemm_fp8
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps
    from neuronx_distributed_b200.quantization import ActivationQuantizationType
    from neuronx_distributed_b200.quantization import quantization_layers as ql

    ps.initialize_model_parallel(1)
    # 2-D blocks and E8M0 expand per expert along N; fp32 [E, K/G, N] passes through untouched
    s = torch.arange(2 * 3 * 2, dtype=torch.float32).reshape(2, 3, 2)
    kn = gemm_fp8.expert_weight_scales_kn(s, 256, 3 * 64, 64)
    assert kn.shape == (2, 3, 256) and torch.equal(kn[1, 2, 128:], s[1, 2, 1].expand(128))
    full = torch.rand(2, 3, 256)
    assert gemm_fp8.expert_weight_scales_kn(full, 256, 192, 64) is full
    e = torch.tensor([[[127, 130]]], dtype=torch.uint8)
    assert torch.equal(gemm_fp8.expert_weight_scales_kn(e, 2, 32, 32), torch.tensor([[[1.0, 8.0]]]))
    # static input scales are per dense layer: expert layers refuse them, and from_float leaves them weight-only
    with pytest.raises(ValueError, match="static"):
        ql.QuantizedExpertFusedColumnParallel(4, 256, 256, quantization_type="blockwise_symmetric",
                                              quantized_dtype=torch.float8_e4m3fn, block_axis=[1], block_size=[128],
                                              activation_quantization_type="static")
    assert ql._expert_activation_quantization({"activation_quantization_type": "static"}) == ActivationQuantizationType.NONE
    assert ql._expert_activation_quantization({}) == ActivationQuantizationType.NONE


def test_expert_scales_and_static_refusal():
    run_distributed(_scales_and_refusals, 1, timeout=120)


def test_grouped_oracle_matches_float64():
    """The fp32 oracle of ``grouped_blockscaled_linear``: block i uses expert ``block_to_expert[i]``; trailing padding
    blocks and an expert with no block included."""
    from neuronx_distributed_b200.ops import gemm_fp8

    g = torch.Generator().manual_seed(5)
    Ex, K, N, B, G = 3, 256, 192, 128, 64
    b2e = torch.tensor([0, 0, 2, 2, 2])                                  # expert 1 has no block, the last two are padding
    xq = (torch.randn(b2e.numel() * B, K, generator=g) * 50).clamp(-448, 448).to(torch.float8_e4m3fn)
    xs = torch.rand(b2e.numel() * B, K // G, generator=g) + 0.5
    wq = (torch.randn(Ex, K, N, generator=g) * 50).clamp(-448, 448).to(torch.float8_e4m3fn)
    ws = torch.rand(Ex, K // G, N, generator=g) + 0.5
    got = gemm_fp8.grouped_blockscaled_linear(xq, xs, wq, ws, b2e, B, G, out_dtype=torch.float32)
    xd = (xq.double().reshape(-1, K // G, G) * xs.double().unsqueeze(-1)).reshape(-1, K)
    wd = (wq.double().reshape(Ex, K // G, G, N) * ws.double().unsqueeze(2)).reshape(Ex, K, N)
    for i, e in enumerate(b2e.tolist()):
        want = xd[i * B:(i + 1) * B] @ wd[e]
        err = ((got[i * B:(i + 1) * B].double() - want).norm() / want.norm()).item()
        assert err < 1e-6, (i, e, err)
