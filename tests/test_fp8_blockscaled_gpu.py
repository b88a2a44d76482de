"""Block-scaled FP8 GEMM and group quantiser on the H100 (csrc/gemm_fp8_block_sm90.cu): kernels vs the torch oracles,
a block-wise W8A8 layer on CUDA vs its CPU result (no bf16 weight copy, CUDA-graph capture), and MXFP8 under NXD_GEMM_MX=1."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

pytestmark = pytest.mark.gpu


def test_fp8_block_quantiser_and_gemm():
    import gpu_check as gc

    assert gc.ops.extension_available(), gc.ops._ext.load_error()
    n = len(gc.RESULTS)
    gc.check_fp8_block()
    bad = [r for r in gc.RESULTS[n:] if not r["ok"]]
    assert not bad, bad


@pytest.mark.parametrize("block_axis,block_size,scale_dtype", [([1], [128], torch.float32), ([0, 1], [128, 128], torch.float32),
                                                                ([1], [32], torch.uint8)])
def test_blockwise_dynamic_layer_on_cuda(monkeypatch, block_axis, block_size, scale_dtype):
    from neuronx_distributed_b200.ops import _ext
    from neuronx_distributed_b200.quantization import quantization_layers as ql

    torch.manual_seed(0)
    K, N = 1024, 768
    layer = ql.QuantizedColumnParallel(K, N, bias=True, gather_output=False, quantization_type="blockwise_symmetric",
                                       quantized_dtype=torch.float8_e4m3fn, block_axis=block_axis, block_size=block_size,
                                       scale_dtype=scale_dtype, activation_quantization_type="dynamic").eval()
    layer.quantize_from_float_weight(torch.randn(N, K) / K ** 0.5)
    layer.bias.data.normal_()
    x = torch.randn(3, 100, K).bfloat16()
    want = layer(x.float())                                          # CPU: fp32 oracle of the same W8A8 numerics
    layer = layer.cuda()

    def no_weight_copy(*a, **k):
        raise AssertionError("block-scaled path de-quantised the weight")

    monkeypatch.setattr(ql, "blockwise_scale_dequantize", no_weight_copy)
    xc = x.cuda()
    n0 = _ext.launches()
    got = layer(xc)
    assert _ext.launches() - n0 == 2                                 # quantiser + block-scaled GEMM
    err = float((got.float().cpu() - want).norm() / want.norm())
    assert err < 1e-2, err
    # CUDA-graph capture and replay on new data
    static_x = xc.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        layer(static_x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_y = layer(static_x)
    x2 = torch.randn_like(xc)
    static_x.copy_(x2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_y, layer(x2))


def test_linear_mx_under_gemm_mx_flag(monkeypatch):
    from neuronx_distributed_b200.ops import _ext, gemm_fp8, gemm_mx
    from neuronx_distributed_b200.quantization.microscaling.mx_torch import quantize_mx

    torch.manual_seed(1)
    M, N, K = 200, 1024, 2048
    w_packed, w_e8m0 = quantize_mx(torch.randn(N, K, device="cuda"), "mxfp8")
    x = torch.randn(M, K, device="cuda").bfloat16()
    monkeypatch.setenv("NXD_GEMM_MX", "1")
    n0 = _ext.launches()
    y = gemm_mx.linear_mx(x, w_packed, w_e8m0)
    assert _ext.launches() - n0 == 2
    xq, xs = gemm_fp8.quantize_groups(x, 32, "mx")
    x_e8m0 = (torch.log2(xs) + 127).to(torch.uint8)
    ref = gemm_mx.matmul_mxfp8_reference(xq.view(torch.uint8), x_e8m0, w_packed, w_e8m0)
    err = float((y.float() - ref).norm() / ref.norm())
    assert y.dtype == torch.bfloat16 and err < 4e-3, err
    # the block-scaled GEMM takes e4m3 codes only: 4-bit weights still raise under the flag
    from neuronx_distributed_b200.ops.gemm_mx import quantize_mxfp4

    f4, f4s = quantize_mxfp4(torch.randn(N, K, device="cuda"))
    with pytest.raises(RuntimeError, match="MXFP8 e4m3"):
        gemm_mx.linear_mx(x, f4.view(torch.uint16), f4s)
