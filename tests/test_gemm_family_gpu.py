"""The GEMM family besides the dense bf16 GEMM vs float64 at real-model edge shapes (H100, sm_90a): the grouped MoE GEMMs
(MODE 3 forward / dgrad, MODE 4 segmented wgrad of ``csrc/gemm_sm90.cu``), the MoE block metadata, the decode GEMV
(``csrc/decode.cu``), the fp8 GEMM and the MX decode GEMV (``csrc/gemv_mx.cu``).

Every reference is float64, computed from the same low-precision operands the kernel reads.  Wherever the inputs allow it
the accumulation is exact: operands on a grid (multiples of 1/8, small integers, e2m1 codes, power-of-two scales) keep every
partial sum inside fp32's 24-bit significand, so a correct kernel returns the float64 result rounded once and the check is
bit equality.  A dropped or doubled k-block, a wrong expert or scale index, a skipped store or a missed tail then changes
bits.  Where two roundings happen (a residual added in fp32, the MoE layer) the bound is derived beside the check.
"""
import math
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

F64 = torch.float64
BF16 = torch.bfloat16
U_BF16 = 2.0 ** -8                   # bf16 unit roundoff (8 significant bits)


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def ulp(ref: torch.Tensor, dtype=BF16) -> torch.Tensor:
    """Spacing of ``dtype`` numbers at |ref| (bf16 / fp32: 7 / 23 stored bits, normal range from 2^-126)."""
    mant = {BF16: 7, torch.float32: 23}[dtype]
    e = torch.floor(torch.log2(ref.abs().to(F64).clamp_min(2.0 ** -126)))
    return torch.exp2(e - mant)


def within(got, ref, tol, what):
    err = (got.to(F64) - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; worst err "
                           f"{err.max().item():.3e} at bound {tol.flatten()[err.flatten().argmax()].item():.3e}")


def launched(_ext, fn):
    """Run ``fn`` and assert that it went through at least one of the extension's kernels."""
    n = _ext.launches()
    out = fn()
    assert _ext.launches() > n, "fell back to eager PyTorch"
    return out


def _grid(shape, g, amax=2):
    """Multiples of 1/8 in [-amax, amax], exact in bf16.  With amax = 2 a product is a multiple of 2^-6 of magnitude <= 4,
    so a sum of n < 2^16 products stays below 2^18 and needs at most 24 significant bits: exact in fp32 in any order."""
    n = 8 * amax
    return torch.randint(-n, n + 1, shape, device=g.device, generator=g, dtype=torch.int16).to(BF16).mul_(0.125)


def exact(got, ref, what):
    """``got`` is the float64 ``ref`` rounded once to ``got.dtype`` (``ref`` is exact in fp32, so the conversion rounds once)."""
    want = ref.to(got.dtype)
    assert torch.equal(got, want), (f"{what}: {int((got != want).sum())} of {got.numel()} elements differ, max err "
                                    f"{(got.to(F64) - ref).abs().max().item():.3e}")


# =====================================================================================================================
# A. grouped GEMM forward and dgrad (MODE 3)
# =====================================================================================================================
# name: (E, K, N) of the stacked weight [E, K, N].  Forward x[M, K] · W[e] → [M, N] reads W as [E·K, N] (MN-major);
# dgrad dy[M, N] · W[e]ᵀ → [M, K] reads the same bytes as [E·K, N] K-major rows, so its output width is K.
GROUPED = {
    "mixtral-tp8-gate_up": (8, 4096, 3584),
    "mixtral-tp8-down": (8, 1792, 4096),
    "dbrx-tp8-gate_up": (16, 6144, 2688),     # forward N = 2I = 2688: a 128-column tail of the 256-wide tile
    "dbrx-tp8-down": (16, 1344, 6144),        # dgrad N = I = 1344: the last weight tile reads 192 rows of the next expert
    "e64-gate_up": (64, 2048, 2816),
    "e64-down": (64, 1408, 2048),             # dgrad N = 1408: the last weight tile reads 128 rows of the next expert
    "odd-e3": (3, 192, 320),                  # dgrad N = 192 is less than one tile; forward N = 320 = 1¼ tiles
}
BLOCK_SIZES = (128, 256, 512, 1024)


def _block_map(E, B, order, g):
    """A block → expert map that uses expert 0 and expert E−1 (the last expert's weight rows are read): ascending, as
    ``build_block_metadata`` lays blocks out, or randomly permuted, which the forward and dgrad must take as well."""
    nb = max(3, 1024 // B)
    mid = torch.randint(1, max(2, E - 1), (nb - 2,), generator=g).clamp(max=E - 1)
    b2e = torch.cat([torch.tensor([0, E - 1]), mid])
    return b2e.sort().values if order == "sorted" else b2e[torch.randperm(nb, generator=g)]


def grouped_ref64(a, w, b2e, B, dgrad):
    """float64 ``a[block i] · W[b2e[i]]`` (forward) or ``a[block i] · W[b2e[i]]ᵀ`` (dgrad), expert by expert."""
    n_out = w.shape[1] if dgrad else w.shape[2]
    out = torch.empty(b2e.numel(), B, n_out, dtype=F64, device=a.device)
    a64 = a.to(F64).view(b2e.numel(), B, -1)
    for e in b2e.unique().tolist():
        sel = (b2e == e).nonzero()[:, 0].to(a.device)
        we = w[e].to(F64)
        out[sel] = a64[sel] @ (we.t() if dgrad else we)
    return out.view(-1, n_out)


@pytest.mark.parametrize("dgrad", [False, True], ids=["fwd", "dgrad"])
@pytest.mark.parametrize("case", list(GROUPED))
def test_grouped_gemm_vs_float64(_ext, case, dgrad):
    """Through ``ops.gemm.grouped_matmul``: the forward, or its backward with only ``x`` requiring a gradient (the dgrad
    launch alone).  Block sizes 128…1024 (one to eight 128-row tiles per block), sorted and permuted block maps."""
    from neuronx_distributed_b200.ops import gemm

    E, K, N = GROUPED[case]
    g = torch.Generator(device="cuda").manual_seed(E * K + N)
    gc = torch.Generator().manual_seed(E + K)
    w = _grid((E, K, N), g)
    seg = torch.zeros(E + 1, dtype=torch.int32, device="cuda")       # the segments feed the wgrad only
    for B in BLOCK_SIZES:
        for order in ("sorted", "permuted"):
            b2e = _block_map(E, B, order, gc)
            M = b2e.numel() * B
            b2e_d = b2e.cuda()
            what = f"{case} B={B} {order} b2e={b2e.tolist()}"
            if not dgrad:
                a = _grid((M, K), g)
                with torch.no_grad():
                    out = launched(_ext, lambda: gemm.grouped_matmul(a, w, b2e_d, seg, B))
            else:
                a = _grid((M, N), g)                                  # dy
                x = torch.zeros(M, K, dtype=BF16, device="cuda", requires_grad=True)
                y = gemm.grouped_matmul(x, w, b2e_d, seg, B)
                launched(_ext, lambda: y.backward(a))
                out = x.grad
            torch.cuda.synchronize()
            exact(out, grouped_ref64(a, w, b2e, B, dgrad), what)


def test_grouped_gemm_rejects_k_tail_with_kn_weights(_ext):
    """[E, K, N] weights are streamed in 64-row k-blocks of the stacked [E·K, N] tensor: with K % 64 != 0 a block would
    cross into the next expert, so the launch is refused before it is made."""
    w = torch.zeros(3, 104, 192, dtype=BF16, device="cuda")
    a = torch.zeros(128, 104, dtype=BF16, device="cuda")
    b2e = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="K % 64"):
        _ext.ext().grouped_gemm(a, w, b2e, 128, False)


# =====================================================================================================================
# B. grouped wgrad (MODE 4) through the main_grad path of grouped_matmul's backward
# =====================================================================================================================
# name: (E, Mo, No) of the weight gradient [E, Mo, No] = Σ_{rows of e} x[row, Mo]ᵀ · dy[row, No]
WGRAD = {
    "mixtral-tp8-down": (8, 1792, 4096),
    "dbrx-tp8-down": (16, 1344, 6144),        # Mo = 1344: a 64-row tail of the 128-row tile
    "dbrx-tp8-gate_up": (16, 6144, 2688),     # No = 2688: a 128-column tail of the 256-wide tile
    "odd-e3": (3, 192, 320),
}
DISTS = {  # name: block size
    "empty": 128,      # expert 0 and every third expert get no tokens
    "single": 256,     # expert 1 fills exactly one block, expert 0 holds one token
    "skewed": 512,     # one expert holds almost every token, the others one token or none
    "tail": 1024,      # few tokens: most of the static block count is padding, which build_block_metadata gives to E−1
}


def _token_counts(dist, E, B, g):
    if dist == "empty":
        c = torch.randint(1, 2 * B, (E,), generator=g)
        c[::3] = 0
    elif dist == "single":
        c = torch.randint(B + 1, 2 * B, (E,), generator=g)
        c[1], c[0] = B, 1
    elif dist == "skewed":
        c = torch.randint(0, 2, (E,), generator=g)
        c[E // 2] = 6 * B + 5
    else:
        c = torch.zeros(E, dtype=torch.long)
        c[0], c[E - 1] = 5, B + 7
    return c


def _routed_rows(dist, E, B, g):
    """Expert ids of T tokens (top-1) with the given per-expert counts → the CPU-path block metadata, the [E+1] block
    segments (as blockwise_mlp_from_metadata computes them) and the mask of real (non-padding) rows."""
    from neuronx_distributed_b200.modules.moe.blockwise import build_block_metadata

    counts = _token_counts(dist, E, B, g)
    ids = torch.repeat_interleave(torch.arange(E), counts)
    ids = ids[torch.randperm(ids.numel(), generator=g)].view(-1, 1)
    b2e, tp2id, got_counts = build_block_metadata(ids, E, B)
    assert torch.equal(got_counts, counts)
    seg = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(torch.bincount(b2e, minlength=E), 0)])
    return b2e, seg, tp2id >= 0, counts


def wgrad_ref64(x, dy, seg, B):
    """float64 Σ over each expert's row blocks [seg[e]·B, seg[e+1]·B) of xᵀ · dy; an expert without blocks gets 0."""
    E = seg.numel() - 1
    out = torch.zeros(E, x.shape[1], dy.shape[1], dtype=F64, device=x.device)
    for e in range(E):
        lo, hi = int(seg[e]) * B, int(seg[e + 1]) * B
        if hi > lo:
            out[e] = x[lo:hi].to(F64).t() @ dy[lo:hi].to(F64)
    return out


def _nan_guarded(shape, pad=64):
    """A contiguous fp32 view into a NaN-filled buffer with ``pad`` guard elements on both sides."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * pad,), float("nan"), device="cuda")
    return buf, buf[pad:pad + n].view(shape), torch.cat([torch.arange(pad), torch.arange(pad + n, n + 2 * pad)]).cuda()


@pytest.mark.parametrize("accumulate", [False, True], ids=["store", "accumulate"])
@pytest.mark.parametrize("dist", list(DISTS))
@pytest.mark.parametrize("case", list(WGRAD))
def test_grouped_wgrad_vs_float64(_ext, case, dist, accumulate):
    """The fp32 wgrad lands in ``main_grad``: overwritten while ``main_grad_fresh`` is set (every element, NaN before),
    added to its random fp32 contents otherwise.  The accumulation is exact, so the result is float64 (+ out0) rounded
    once to fp32; an expert without tokens gets exactly 0, or keeps out0.  Nothing outside [E, Mo, No] is written."""
    from neuronx_distributed_b200.ops import gemm

    E, Mo, No = WGRAD[case]
    B = DISTS[dist]
    gc = torch.Generator().manual_seed(E * Mo + No + B)
    g = torch.Generator(device="cuda").manual_seed(Mo + No)
    b2e, seg, valid, counts = _routed_rows(dist, E, B, gc)
    if dist == "tail":
        assert int((b2e == E - 1).sum()) > (counts[E - 1].item() + B - 1) // B, "no padding blocks went to E−1"
    rows = b2e.numel() * B
    vd = valid.cuda()[:, None]
    x = _grid((rows, Mo), g) * vd                                   # padding rows are zero, as gathered by the MoE layer
    dy = _grid((rows, No), g) * vd
    buf, mg, guard = _nan_guarded((E, Mo, No))
    if accumulate:
        mg.copy_(torch.randn(E, Mo, No, device="cuda", generator=g) * 16)
    out0 = mg.to(F64)
    w = torch.nn.Parameter(torch.zeros(E, Mo, No, dtype=BF16, device="cuda"))
    w.main_grad, w.main_grad_fresh = mg, not accumulate
    y = gemm.grouped_matmul(x, w, b2e.cuda(), seg.cuda(), B)
    launched(_ext, lambda: y.backward(dy))
    torch.cuda.synchronize()
    assert w.grad is None and w.main_grad_fresh is False
    ref = wgrad_ref64(x, dy, seg, B) + (out0 if accumulate else 0)
    what = f"{case} {dist} B={B} seg={seg.tolist()}"
    exact(mg, ref, what)
    for e in (counts == 0).nonzero()[:, 0].tolist():
        if accumulate:
            assert torch.equal(mg[e], out0[e].float()), f"{what}: expert {e} without tokens changed"
        else:
            assert bool((mg[e] == 0).all()), f"{what}: expert {e} without tokens is not 0"
    assert bool(torch.isnan(buf[guard]).all()), f"{what}: wrote outside [E, Mo, No]"


# =====================================================================================================================
# C. the autograd function: main_grad handshake, grad-ready hook, dx, and the MoE layer
# =====================================================================================================================
def test_grouped_matmul_autograd_main_grad_and_dx(_ext):
    from neuronx_distributed_b200.modules.moe.blockwise import build_block_metadata
    from neuronx_distributed_b200.ops import gemm

    E, K, N, B, T = 8, 1024, 1792, 256, 700
    gc = torch.Generator().manual_seed(21)
    g = torch.Generator(device="cuda").manual_seed(21)
    allowed = torch.tensor([0, 1, 3, 4, 5, 6, 7])                     # expert 2 gets no tokens
    idx = allowed[torch.rand(T, allowed.numel(), generator=gc).argsort(-1)[:, :2]]
    b2e, tp2id, counts = build_block_metadata(idx, E, B)
    assert counts[2] == 0
    seg = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(torch.bincount(b2e, minlength=E), 0)])
    valid = (tp2id >= 0).cuda()[:, None]
    rows = b2e.numel() * B
    x = (_grid((rows, K), g) * valid).requires_grad_(True)
    w = torch.nn.Parameter(_grid((E, K, N), g))
    w.main_grad = torch.randn(E, K, N, device="cuda", generator=g) * 16   # stale contents the first backward overwrites
    w.main_grad_fresh = True
    ready = []
    w._nxd_grad_ready = ready.append
    b2e_d, seg_d = b2e.cuda(), seg.cuda()

    grads = []
    for step in range(2):
        gy = _grid((rows, N), g) * valid                               # padding rows get no gradient from the layer
        y = gemm.grouped_matmul(x, w, b2e_d, seg_d, B)
        n = _ext.launches()
        y.backward(gy)
        torch.cuda.synchronize()
        assert _ext.launches() >= n + 2, "dgrad and wgrad must both run on the extension"
        assert len(ready) == step + 1 and ready[-1] is w, "_nxd_grad_ready fires once per backward"
        assert w.main_grad_fresh is False and w.grad is None
        grads.append(wgrad_ref64(x.detach(), gy, seg, B))
        # step 0 overwrites the stale main_grad; step 1 adds (step 0's fp32 result is exact, so the sum rounds once)
        exact(w.main_grad, sum(grads), f"main_grad after backward {step}")
        exact(x.grad, grouped_ref64(gy, w.detach(), b2e, B, True), f"dx after backward {step}")
        assert bool((x.grad[~valid[:, 0]] == 0).all()), "padding rows of dx must be exactly 0"
        x.grad = None

    # without main_grad the weight gradient is returned as a bf16 tensor: float64 rounded once
    w2 = torch.nn.Parameter(w.detach().clone())
    y = gemm.grouped_matmul(x.detach(), w2, b2e_d, seg_d, B)
    launched(_ext, lambda: y.backward(gy))
    exact(w2.grad, grads[-1], "w.grad without main_grad")


def _glu(h):
    gate, up = h.chunk(2, dim=-1)
    return torch.nn.functional.silu(gate) * up


def _layer_error_bound(hidden, aff, idx, wgu, wdn, bgu, bdn, B):
    """Elementwise bound on |layer_bf16 − layer_f64|, propagated in float64 through the bf16 layer's roundings.
    u = 2^-8 (bf16), γ(n) = n·2^-23/(1 − n·2^-23): fp32 accumulation over n terms in any order, with a whole fp32 ulp
    per addition because the tensor cores may truncate instead of rounding to nearest.
      h = x·W_gu (+ b):  fp32 GEMM (γ(H)·|x|·|W|), one bf16 rounding of the sum, one more of the bias add
      s = silu(gate):    |silu'| <= 1.0998, torch evaluates in fp32 (2^-20 relative) and rounds once
      a = s·up:          both factors' errors (exact product bound, not linearised) + one rounding
      y = a·W_dn (+ b):  the error of a through |W_dn|, then as h with |a'| <= |a| + e_a in place of |x|
      out = Σ_j aff_j·y_j: one rounding per product, index_add_ in bf16 adds k terms (k roundings bound it)."""
    u, k = U_BF16, idx.shape[1]
    H, I = wgu.shape[1], wdn.shape[1]

    def gam(n):
        return n * 2.0 ** -23 / (1 - n * 2.0 ** -23)

    def linear(e_gemm, s, b):
        """Error of bf16(bf16(s̃) + b) where |s̃ − s| <= e_gemm: the GEMM error, then two roundings."""
        e1 = e_gemm + u * (s.abs() + e_gemm)
        if b is None:
            return s, e1
        return s + b, e1 + u * ((s + b).abs() + e1)

    T = hidden.shape[0]
    err = torch.zeros(T, H, dtype=F64, device=hidden.device)
    mag = torch.zeros(T, H, dtype=F64, device=hidden.device)
    for e in idx.unique().tolist():
        tok, _ = (idx == e).nonzero(as_tuple=True)
        x = hidden[tok]
        h, e_h = linear(gam(H) * (x.abs() @ wgu[e].abs()), x @ wgu[e], None if bgu is None else bgu[e])
        gate, up = h.chunk(2, -1)
        eg, eu = e_h.chunk(2, -1)
        s = torch.nn.functional.silu(gate)
        e_s = 1.1 * eg + (u + 2.0 ** -20) * (s.abs() + 1.1 * eg)
        a = s * up
        e_a = e_s * (up.abs() + eu) + s.abs() * eu + u * (s.abs() + e_s) * (up.abs() + eu)
        wd = wdn[e].abs()
        y, e_y = linear(e_a @ wd + gam(I) * ((a.abs() + e_a) @ wd), a @ wdn[e], None if bdn is None else bdn[e])
        w_ = aff[tok, e][:, None]
        err.index_add_(0, tok, w_ * e_y)
        mag.index_add_(0, tok, w_ * (y.abs() + e_y))
    return err + k * 1.02 * u * mag


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
def test_blockwise_expert_mlp_mixtral_tp8_vs_float64_cpu(_ext, bias):
    """A Mixtral-8x7B layer at TP = 8 (H 4096, I 1792, 8 experts, top-2) on the grouped kernels vs the same layer in
    float64 on the CPU path, with the elementwise bound derived in ``_layer_error_bound``."""
    from neuronx_distributed_b200.modules.moe.blockwise import blockwise_expert_mlp

    T, H, I, E, k, B = 64, 4096, 1792, 8, 2, 128
    g = torch.Generator().manual_seed(5)
    hidden = torch.randn(T, H, generator=g).to(BF16)
    idx = torch.rand(T, E, generator=g).argsort(-1)[:, :k]
    aff = torch.rand(T, E, generator=g).to(BF16)
    wgu = (torch.randn(E, H, 2 * I, generator=g) / H ** 0.5).to(BF16)
    wdn = (torch.randn(E, I, H, generator=g) / I ** 0.5).to(BF16)
    bgu = torch.randn(E, 2 * I, generator=g).to(BF16) if bias else None
    bdn = torch.randn(E, H, generator=g).to(BF16) if bias else None

    def experts(dev, dt):
        def cv(t):
            return None if t is None else t.to(device=dev, dtype=dt)

        return SimpleNamespace(glu_mlp=True, activation=_glu, gate_up_proj=SimpleNamespace(weight=cv(wgu), bias=cv(bgu)),
                               down_proj=SimpleNamespace(weight=cv(wdn), bias=cv(bdn), tp=1))

    with torch.no_grad():
        got = launched(_ext, lambda: blockwise_expert_mlp(hidden.cuda(), aff.cuda(), idx.cuda(), experts("cuda", BF16), B))
        ref = blockwise_expert_mlp(hidden.to(F64), aff.to(F64), idx, experts("cpu", F64), B)
        ex = experts("cuda", F64)
        tol = _layer_error_bound(hidden.cuda().to(F64), aff.cuda().to(F64), idx.cuda(), ex.gate_up_proj.weight,
                                 ex.down_proj.weight, ex.gate_up_proj.bias, ex.down_proj.bias, B)
    assert got.dtype == BF16 and got.shape == (T, H)
    within(got, ref.cuda(), tol + 1e-12 * ref.abs().cuda(), f"MoE layer bias={bias}")


# =====================================================================================================================
# D. MoE block metadata (one-launch kernel) vs the CPU sort path, bit for bit
# =====================================================================================================================
META_CASES = [  # (T, k, B)
    (5, 2, 128),        # T·k = 10 < 32: one partly filled warp
    (5, 2, 1024),       # a block larger than T·k
    (333, 3, 128),      # T·k = 999: not a multiple of 32
    (1500, 2, 256),     # T·k = 3000 > 1024: three chunks, the last with a partly filled warp
]


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64], ids=["int32", "int64"])
@pytest.mark.parametrize("E", [1, 2, 60, 256])
@pytest.mark.parametrize("T,k,B", META_CASES, ids=[f"T{t}k{k}B{b}" for t, k, b in META_CASES])
def test_moe_block_metadata_vs_sort_path(_ext, T, k, B, E, idx_dtype):
    from neuronx_distributed_b200.modules.moe.blockwise import build_block_metadata

    g = torch.Generator().manual_seed(T * E + B)
    # from E = 3 on, expert 0 and every fourth expert get no tokens
    allowed = torch.tensor([e for e in range(E) if E < 3 or (e % 4 != 0)])
    kk = min(k, allowed.numel())
    idx = allowed[torch.rand(T, allowed.numel(), generator=g).argsort(-1)[:, :kk]].to(idx_dtype)
    want = build_block_metadata(idx, E, B)                          # sort + cumsum path
    if E >= 3:
        assert bool((want[2] == 0).any())
    got = launched(_ext, lambda: build_block_metadata(idx.cuda(), E, B))
    for a, b, name in zip(got, want, ("block_to_expert", "token_position_to_id", "tokens_per_expert")):
        assert a.dtype == b.dtype and torch.equal(a.cpu(), b), name


# =====================================================================================================================
# E. decode GEMV: y[M <= 8, N] = x · Wᵀ (+ residual)
# =====================================================================================================================
GEMV_N = (8, 16, 4000, 50257, 11008, 12288)      # routers, a 32000/8 vocab shard, GPT-2's vocab, Llama MLP widths
GEMV_K = (8, 264, 4104, 5120, 14336)


@pytest.mark.parametrize("K", GEMV_K)
@pytest.mark.parametrize("N", GEMV_N)
def test_decode_gemv_vs_float64(_ext, N, K):
    """Every template instantiation M = 1…8.  Grid inputs: the fp32 sum is exact (|Σ| <= 4·14336 < 2^16, multiples of
    2^-6), so without a residual y is float64 rounded once.  The residual is added to the fp32 sum and the result rounded
    to bf16: two roundings, within one bf16 ulp of float64."""
    from neuronx_distributed_b200.ops import gemm

    g = torch.Generator(device="cuda").manual_seed(N + K)
    w = _grid((N, K), g)
    w64t = w.to(F64).t()
    for M in range(1, 9):
        x = _grid((M, K), g)
        assert gemm._gemv_eligible(x, w, M, K, False, True, None, BF16)
        y = launched(_ext, lambda: gemm.matmul(x, w, False, True))
        ref = x.to(F64) @ w64t
        exact(y, ref, f"M={M} N={N} K={K}")
        res = (torch.randn(M, N, device="cuda", generator=g) * 64).to(BF16)
        yr = _ext.ext().gemv(x, w, res)
        ref_r = ref + res.to(F64)
        within(yr, ref_r, ulp(ref_r), f"M={M} N={N} K={K} + residual")
    torch.cuda.synchronize()


# =====================================================================================================================
# F. fp8 GEMM (the e4m3 instantiation of gemm_bf16_kernel) with per-row and per-column scales
# =====================================================================================================================
FP8_N = (264, 1000, 4104)


@pytest.mark.parametrize("K", (16, 48, 144, 4096))
@pytest.mark.parametrize("M", (1, 5, 8, 200))
def test_fp8_gemm_vs_float64(_ext, M, K):
    """e4m3 operands are integers in [−8, 8] (exact in e4m3); |Σ| <= 64·4096 = 2^18 is an exact fp32 integer.  Scales
    are powers of two from 2^-8 to 2^8, different for neighbouring rows and neighbouring columns, so their product
    is exact and a wrong scale index changes the result.  K < 128 and K = 144 leave part of the 128-wide k-block to the
    TMA zero fill.  y = float64 rounded once to bf16."""
    from neuronx_distributed_b200.ops import gemm_fp8

    g = torch.Generator(device="cuda").manual_seed(M * K)
    for N in FP8_N:
        a = torch.randint(-8, 9, (M, K), device="cuda", generator=g).float().to(torch.float8_e4m3fn)
        b = torch.randint(-8, 9, (N, K), device="cuda", generator=g).float().to(torch.float8_e4m3fn)
        sa = torch.exp2(((torch.arange(M, device="cuda") * 7 + K) % 17 - 8).float())
        sb = torch.exp2(((torch.arange(N, device="cuda") * 5 + M) % 17 - 8).float())
        y = launched(_ext, lambda: gemm_fp8.scaled_linear(a, sa, b, sb))
        ref = (a.to(F64) @ b.to(F64).t()) * sa.to(F64)[:, None] * sb.to(F64)[None, :]
        assert y.shape == (M, N)
        exact(y, ref, f"M={M} N={N} K={K}")


# =====================================================================================================================
# G. MX decode GEMV (e2m1 / e4m3 / e5m2 codes, E8M0 block scales)
# =====================================================================================================================
MX_KINDS = {"mxfp4": 0, "mxfp8": 1, "mxfp8_e5m2": 2}
E2M1 = torch.tensor([0, .5, 1, 1.5, 2, 3, 4, 6, -0., -.5, -1, -1.5, -2, -3, -4, -6], dtype=F64)
MX_K = (32, 96, 1440, 2080)          # 32·odd blocks per row: 1, 3, 45 and 65 (the last two over two lane rounds)


def mx_weights(kind, R, K, g):
    """(codes as bytes [R, row bytes], E8M0 scales [R, K/32], float64 values [R, K]).  fp4: uniform over the 16 e2m1
    codes; fp8: integers in [−8, 8], exact in e4m3 and e5m2.  Scales 2^-3…2^3 (bytes 124…130)."""
    if MX_KINDS[kind] == 0:
        codes = torch.randint(0, 16, (R, K), generator=g)
        vals = E2M1[codes]
        raw = (codes[:, 0::2] | (codes[:, 1::2] << 4)).to(torch.uint8)
    else:
        vals = torch.randint(-8, 9, (R, K), generator=g).to(F64)
        f8 = torch.float8_e4m3fn if MX_KINDS[kind] == 1 else torch.float8_e5m2
        raw = vals.float().to(f8).view(torch.uint8)
        assert torch.equal(raw.view(f8).to(F64), vals)
    scale = torch.randint(124, 131, (R, K // 32), generator=g).to(torch.uint8)
    vals = (vals.view(R, K // 32, 32) * torch.exp2(scale.to(F64) - 127)[..., None]).view(R, K)
    return raw.cuda(), scale.cuda(), vals.cuda()


def _mx_x(shape, g):
    """Multiples of 1/8 in [−1, 1].  A term x·v·s is a multiple of 2^-7 (fp4) or 2^-6 (fp8) of magnitude <= 48 or 64, so
    Σ over K = 2080 stays below 2^17 resp. 2^18: 24 significant bits, every partial sum exact in fp32."""
    return (torch.randint(-8, 9, shape, generator=g).to(F64) / 8).to(BF16).cuda()


def test_gemv_mx_matches_dequantised_reference(_ext, monkeypatch):
    """``linear_mx`` on the MX GEMV for every format (e2m1, e4m3, e5m2), every M from 1 to 8, K = 32·odd and N = 8 / 1000,
    against float64 on the de-quantised weights: exact without a residual, within one bf16 ulp with one."""
    from neuronx_distributed_b200.ops import gemm_mx

    monkeypatch.setenv("NXD_GEMV_MX", "1")
    for kind in MX_KINDS:
        for K in MX_K:
            g = torch.Generator().manual_seed(K + MX_KINDS[kind])
            for N in (8, 1000):
                w, s, v64 = mx_weights(kind, N, K, g)
                for M in range(1, 9):
                    x = _mx_x((M, K), g)
                    assert gemm_mx.gemv_eligible(x, w, s)
                    y = launched(_ext, lambda: gemm_mx.linear_mx(x, w, s, kind=kind))
                    ref = x.to(F64) @ v64.t()
                    exact(y, ref, f"{kind} M={M} N={N} K={K}")
                    res = (torch.randn(M, N, generator=g) * 64).to(BF16).cuda()
                    yr = launched(_ext, lambda: gemm_mx.linear_mx(x, w, s, kind=kind, residual=res))
                    ref_r = ref + res.to(F64)
                    within(yr, ref_r, ulp(ref_r), f"{kind} M={M} N={N} K={K} + residual")   # fp32 add, then bf16


@pytest.mark.parametrize("kind", list(MX_KINDS))
def test_gemv_mx_grouped_vs_float64(_ext, monkeypatch, kind):
    """Per-slot expert selection: repeated experts, expert 0 and expert E−1, N with a tail of a 8-column CTA."""
    from neuronx_distributed_b200.ops import gemm_mx

    monkeypatch.setenv("NXD_GEMV_MX", "1")
    E, N, K = 8, 1004, 1440
    g = torch.Generator().manual_seed(7 + MX_KINDS[kind])
    w, s, v64 = mx_weights(kind, E * N, K, g)
    w, s, v64 = w.view(E, N, -1), s.view(E, N, -1), v64.view(E, N, K)
    ex = torch.tensor([E - 1, 0, 3, 3, E - 1, 1], device="cuda")
    x = _mx_x((ex.numel(), K), g)
    y = launched(_ext, lambda: gemm_mx.grouped_linear_mx(x, w, s, ex, kind))
    ref = torch.einsum("sk,snk->sn", x.to(F64), v64[ex])
    exact(y, ref, f"{kind} grouped")


# =====================================================================================================================
# H. 16-byte alignment guards of the GEMV paths
# =====================================================================================================================
def _unaligned_copy(t):
    """A contiguous copy of ``t`` one element into a fresh buffer: its start is not 16-byte aligned."""
    buf = torch.zeros(t.numel() + 16, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


def _raises_before_launch(fn, match):
    """``fn`` must raise RuntimeError.  It runs while a CUDA graph captures the stream, so if a guard were missing the
    kernel would only be recorded into a graph that is never replayed: the test fails on the assertion and nothing runs
    on the unaligned pointer."""
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match=match):
        with torch.cuda.graph(graph):
            fn()


def test_gemv_paths_reject_unaligned_operands(_ext, monkeypatch):
    from neuronx_distributed_b200.ops import gemm, gemm_mx

    M, N, K = 4, 64, 64
    g = torch.Generator(device="cuda").manual_seed(1)
    x, w = _grid((M, K), g), _grid((N, K), g)
    xu, wu = _unaligned_copy(x), _unaligned_copy(w)
    ref = x.to(F64) @ w.to(F64).t()
    for a, b in ((xu, w), (x, wu)):
        # the dispatch turns the view away before calling anything, and the general path computes the same product
        assert not gemm._gemv_eligible(a, b, M, K, False, True, None, BF16)
        exact(gemm.matmul(a, b, False, True), ref, "unaligned operand through matmul")
        _raises_before_launch(lambda: _ext.ext().gemv(a, b, None), "16-byte aligned")

    monkeypatch.setenv("NXD_GEMV_MX", "1")
    wq, s, _ = mx_weights("mxfp8", N, K, torch.Generator().manual_seed(2))
    xm = _mx_x((M, K), torch.Generator().manual_seed(3))
    xmu, wqu = _unaligned_copy(xm), _unaligned_copy(wq)
    assert not gemm_mx.gemv_eligible(xmu, wq, s) and not gemm_mx.gemv_eligible(xm, wqu, s)
    assert not gemm_mx.grouped_gemv_eligible(xmu, wq.view(1, N, K), s.view(1, N, -1))
    assert not gemm_mx.grouped_gemv_eligible(xm, wqu.view(1, N, K), s.view(1, N, -1))
    ex = torch.zeros(M, dtype=torch.long, device="cuda")
    for a, b in ((xmu, wq), (xm, wqu)):
        _raises_before_launch(lambda: _ext.ext().gemv_mx(a, b, s, 1, None), "16-byte aligned")
        _raises_before_launch(lambda: _ext.ext().gemv_mx_grouped(a, b.view(1, N, K), s.view(1, N, -1), ex, 1),
                              "16-byte aligned")
