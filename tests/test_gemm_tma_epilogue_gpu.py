"""The bf16 GEMM's TMA epilogue (H100, sm_90a) on persistent multi-tile shapes.

Tiles whose `out` has a 16-byte aligned base and row pitch leave through shared memory: a bulk tensor store, or, to
accumulate into fp32, a bulk tensor reduce-add at L2.  Every CTA here runs many tiles, so a staging buffer rewritten
before its store has read it, or a bulk group still in flight when the kernel ends, shows up as a wrong element.  The
checks are bitwise: accumulating into X equals X + (the stored product) added in fp32 by torch, a bf16 `out` equals the
fp32 `out` rounded to bf16, and on exact-arithmetic inputs the product equals the float64 one.  Inputs are chosen so that
no subnormal arises, where the kernel's flush-to-zero add and torch's add would differ.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

F64 = torch.float64
GUARD = 16          # elements of NaN before `out` (64 bytes for fp32: `out` stays 16-byte aligned) and rows after it


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _grid_bf16(shape, g):
    """Multiples of 1/8 in [-2, 2]: every partial sum of K <= 4096 products is a multiple of 2^-6 below 2^14, so the fp32
    accumulation is exact in any order and no result is subnormal."""
    return (torch.randint(-16, 17, shape, device="cuda", generator=g).float() / 8).bfloat16()


def _operands(layout, M, N, K, g):
    ta, tb = layout[0] == "t", layout[1] == "t"
    a = _grid_bf16((K, M) if ta else (M, K), g)
    b = _grid_bf16((N, K) if tb else (K, N), g)
    return a, b, ta, tb


def _ref64(a, b, ta, tb):
    return (a.to(F64).t() if ta else a.to(F64)) @ (b.to(F64).t() if tb else b.to(F64))


def _x(M, N, g):
    """An fp32 accumulation target with no subnormal and no zero: magnitudes in [1/2, 8)."""
    r = torch.rand(M, N, device="cuda", generator=g) * 7.5 + 0.5
    return torch.where(torch.rand(M, N, device="cuda", generator=g) < 0.5, -r, r)


def _guarded(M, N, dtype, elem_offset=GUARD):
    """`out` [M, N] at `elem_offset` elements into a NaN-filled flat buffer that extends 3 rows past its end."""
    buf = torch.full((elem_offset + (M + 3) * N,), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[elem_offset:elem_offset + M * N].view(M, N)


def _assert_guards(buf, out, what):
    lo = out.storage_offset() - buf.storage_offset()
    hi = lo + out.numel()
    assert torch.isnan(buf[:lo]).all(), f"{what}: written before out"
    assert torch.isnan(buf[hi:]).all(), f"{what}: rows past M written"


def _gemm(_ext, a, b, ta, tb, out, accumulate=False):
    from neuronx_distributed_b200.ops import gemm

    n = _ext.launches()
    gemm.matmul(a, b, ta, tb, out=out, accumulate=accumulate)
    assert _ext.launches() > n, "fell back to eager PyTorch"
    torch.cuda.synchronize()


def _check_epilogue(_ext, a, b, ta, tb, M, N, g, exact):
    """fp32 store, fp32 accumulate into X and bf16 store of one product, each in a guarded buffer."""
    what = f"{'t' if ta else 'n'}{'t' if tb else 'n'} M={M} N={N}"
    buf32, s = _guarded(M, N, torch.float32)
    _gemm(_ext, a, b, ta, tb, s)
    _assert_guards(buf32, s, what + " fp32 store")
    if exact:
        assert torch.equal(s, _ref64(a, b, ta, tb).float()), f"{what}: fp32 store differs from the exact product"

    x = _x(M, N, g)
    bufa, acc = _guarded(M, N, torch.float32)
    acc.copy_(x)
    _gemm(_ext, a, b, ta, tb, acc, accumulate=True)
    _assert_guards(bufa, acc, what + " fp32 accumulate")
    assert torch.equal(_bits(acc), _bits(x + s)), f"{what}: accumulate != X + store"

    buf16, h = _guarded(M, N, torch.bfloat16)
    _gemm(_ext, a, b, ta, tb, h)
    _assert_guards(buf16, h, what + " bf16 store")
    assert torch.equal(_bits(h), _bits(s.bfloat16())), f"{what}: bf16 store != fp32 store rounded to bf16"
    return s


@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
def test_ragged_persistent_tiles(_ext, layout):
    """M = 4096 + 72, N = 32000 + 8: 33 x 126 tiles, about 31 per CTA, with partial tiles along both edges."""
    M, N, K = 4096 + 72, 32000 + 8, 200
    g = torch.Generator(device="cuda").manual_seed(3)
    a, b, ta, tb = _operands(layout, M, N, K, g)
    _check_epilogue(_ext, a, b, ta, tb, M, N, g, exact=True)


@pytest.mark.parametrize("n_out,k_in", [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008)],
                         ids=["qkv", "o", "gate_up", "down"])
def test_wgrad_shapes(_ext, n_out, k_in):
    """The Llama-2-7B weight gradients of one 4096-token micro-batch: gᵀ[n_out, 4096] · x[4096, k_in] into fp32."""
    T = 4096
    g = torch.Generator(device="cuda").manual_seed(n_out + k_in)
    go = _grid_bf16((T, n_out), g)
    x = _grid_bf16((T, k_in), g)
    _check_epilogue(_ext, go, x, True, False, n_out, k_in, g, exact=True)


@pytest.mark.parametrize("accumulate", [False, True], ids=["store", "accumulate"])
def test_misaligned_out_matches_aligned(_ext, accumulate):
    """An fp32 `out` 8 but not 16 bytes into its buffer cannot take a tensor map and is written from registers; the
    result is the aligned (TMA) run's, bit for bit."""
    M, N, K = 4096 + 72, 4096 + 8, 264
    g = torch.Generator(device="cuda").manual_seed(5)
    a, b, ta, tb = _operands("nt", M, N, K, g)
    x = _x(M, N, g)
    runs = []
    for off in (GUARD, GUARD + 2):
        buf, out = _guarded(M, N, torch.float32, off)
        assert (out.data_ptr() % 16 == 0) == (off == GUARD)
        if accumulate:
            out.copy_(x)
        _gemm(_ext, a, b, ta, tb, out, accumulate)
        _assert_guards(buf, out, f"offset {off}")
        runs.append(out.clone())
    assert torch.equal(_bits(runs[0]), _bits(runs[1]))
    if not accumulate:
        assert torch.equal(runs[0], _ref64(a, b, ta, tb).float())


def test_zero1_main_grad_over_micro_batches(_ext):
    """The wgrad of one linear layer into its ZeRO-1 main_grad, a view into the flat fp32 gradient buffer after another
    parameter's slot: the first micro-batch stores, the next two accumulate.  Equal, bit for bit, to the same products
    stored separately and added by torch in fp32; the neighbouring slot and the padding stay untouched."""
    from neuronx_distributed_b200.ops import gemm
    from neuronx_distributed_b200.optimizer.zero_redundancy_optimizer import _FlatGroup
    from neuronx_distributed_b200.parallel_layers.layers import wgrad

    T, n_out, k_in = 4096, 4096, 11008
    g = torch.Generator(device="cuda").manual_seed(7)
    small = torch.nn.Parameter(torch.zeros(1000, device="cuda", dtype=torch.bfloat16))
    w = torch.nn.Parameter(torch.zeros(n_out, k_in, device="cuda", dtype=torch.bfloat16))
    fg = _FlatGroup([small, w], 0, 1, 0, torch.float32, torch.float32, False)
    fg.grad_flat.fill_(float("nan"))
    lo = w.main_grad.storage_offset() - fg.grad_flat.storage_offset()
    assert lo > 0 and w.main_grad.data_ptr() % 16 == 0

    ref = None
    w.main_grad_fresh = True
    for mb in range(3):
        go = (torch.randn(T, n_out, device="cuda", generator=g) * 0.5).bfloat16()
        x = (torch.randn(T, k_in, device="cuda", generator=g) * 0.5).bfloat16()
        n = _ext.launches()
        assert wgrad(go, x, w) is None
        assert _ext.launches() > n
        s = gemm.matmul(go, x, True, False, out_dtype=torch.float32)
        ref = s if ref is None else ref + s
        torch.cuda.synchronize()
        assert torch.equal(_bits(w.main_grad), _bits(ref)), f"micro-batch {mb}"
    assert torch.isnan(fg.grad_flat[:lo]).all(), "neighbouring slot written"
    assert torch.isnan(fg.grad_flat[lo + w.numel():]).all(), "padding past the slot written"
