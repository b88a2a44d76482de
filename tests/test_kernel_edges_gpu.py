"""Training-step kernels at real-model edge shapes vs float64 references of the same operation (H100, sm_90a).

Every reference is computed in float64 from the same low-precision inputs the kernel reads.  Each bound follows from
the arithmetic the kernel does and is written beside it; the inputs are chosen so that a wrong index, a dropped or
doubled chunk or a missed tail moves the error far above it.  The extension is built with ``--use_fast_math``:
``__expf``, ``rsqrtf``, ``sqrtf`` and ``/`` are the approximate instructions and fp32 denormals flush to zero.
"""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

F64 = torch.float64
U = 2.0 ** -24                       # fp32 unit roundoff
MANT = {torch.bfloat16: 7, torch.float16: 10, torch.float32: 23}
EMIN = {torch.bfloat16: -126, torch.float16: -14, torch.float32: -126}
VEC = {torch.bfloat16: 8, torch.float16: 8, torch.float32: 4}   # elements per 16-byte packet


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def ulp(ref: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of ``dtype`` numbers at |ref| (subnormal spacing below the normal range)."""
    e = torch.floor(torch.log2(ref.abs().to(F64).clamp_min(2.0 ** EMIN[dtype])))
    return torch.exp2(e - MANT[dtype])


def within(got, ref, tol, what):
    err = (got.to(F64) - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; worst err "
                           f"{err.max().item():.3e} at bound {tol.flatten()[err.flatten().argmax()].item():.3e}")
    return (err / tol).max().item()


def launched(_ext, fn):
    """Run ``fn`` and assert that it went through at least one of the extension's kernels."""
    n = _ext.launches()
    out = fn()
    assert _ext.launches() > n, "fell back to eager PyTorch"
    return out


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# =====================================================================================================================
# A. cross-entropy statistics and backward
# =====================================================================================================================
CE_CASES = [(dt, V) for dt in (torch.bfloat16, torch.float16, torch.float32) for V in (4002, 8004, 30522, 50257, 32000)]
CE_CASES.append((torch.float32, 4001))
PLANT = 12.0                         # planted row maximum; the other logits lie in [-8, 8]


def _ce_inputs(dt, V, offset, rows=8, seed=0):
    """Logits ``[rows, V]`` as a contiguous view at element ``offset`` of a larger buffer.  Each row's unique maximum is
    planted where a kernel goes wrong: the last column (inside the ragged tail when V % vec != 0), column 0, the first
    column of the tail, the middle.  A missed or misread tail loses the maximum, which is compared exactly."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.empty(rows * V + offset + 8, device="cuda", dtype=dt)
    x = buf[offset:offset + rows * V].view(rows, V)
    x.copy_((torch.randn(rows, V, device="cuda", generator=g) * 2).clamp(-8, 8))
    tail0 = V - V % VEC[dt] if V % VEC[dt] else V - 3
    cols = [V - 1, 0, tail0, V // 2, V - 2, 1, tail0 - 1, V // 3][:rows]
    for r, c in enumerate(cols):
        x[r, c] = PLANT
    return x


def _ce_targets(V, start, rows=8):
    # below the shard, its first and last column, above it, the ignore index, two inside, the first global id
    t = [start - 1, start, start + V - 1, start + V, -100, start + V // 2 + 1, start + 3, 0][:rows]
    return torch.tensor(t, device="cuda", dtype=torch.long)


def _sumexp_rel_bound(V, R):
    """Relative bound of the kernel's Σexp(x - max).  n = elements one thread folds (a 256-thread CTA per row).
    __expf(a) is within (2 + 1.173|a|) fp32 ulps: one call per term, the running rescales (at most n calls, their
    arguments telescope to at most the row range R) and the final merge; then a positive sum with an addition chain of
    n + 8 (packet) + 10 (block tree) roundings."""
    n = math.ceil(V / 256)
    return 2.0 ** -23 * ((2 + 1.173 * R) + (2 * n + 1.173 * R) + (2 + 1.173 * R)) + U * (n + 18) * 1.01


@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "offset1"])
@pytest.mark.parametrize("dt,V", CE_CASES, ids=[f"{str(d)[6:]}-V{v}" for d, v in CE_CASES])
def test_ce_stats_vs_float64(_ext, dt, V, offset):
    from neuronx_distributed_b200.ops import cross_entropy as ce

    start = 2 * V                                                  # rank 2 of a vocab-parallel split
    x = _ce_inputs(dt, V, offset)
    assert (x.data_ptr() % 16 != 0) == (offset == 1)
    tgt = _ce_targets(V, start)
    st = launched(_ext, lambda: ce.ce_stats(x, tgt, start))
    torch.cuda.synchronize()
    x64 = x.to(F64)
    mx = x64.max(-1).values
    assert torch.equal(st[:, 0].to(F64), mx), "row max"           # a max of stored values is exact
    local = tgt - start
    owned = (local >= 0) & (local < V)
    tl = torch.where(owned, x64.gather(1, local.clamp(0, V - 1)[:, None])[:, 0], torch.zeros_like(mx))
    assert torch.equal(st[:, 2].to(F64), tl), "target logit"       # a copy of one stored value (0 when not owned)
    se = torch.exp(x64 - mx[:, None]).sum(-1)
    R = (mx - x64.min(-1).values).max().item()
    within(st[:, 1], se, se * _sumexp_rel_bound(V, R), "sum exp")
    # Σx: an fp32 chain of ceil(V/256) + 10 additions per row, bounded by Σ|x|
    sx_tol = U * (math.ceil(V / 256) + 10) * 1.01 * x64.abs().sum(-1)
    within(st[:, 3], x64.sum(-1), sx_tol, "sum x")


@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "offset1"])
@pytest.mark.parametrize("dt,V", CE_CASES, ids=[f"{str(d)[6:]}-V{v}" for d, v in CE_CASES])
def test_ce_backward_vs_float64(_ext, dt, V, offset, smoothing):
    from neuronx_distributed_b200.ops import cross_entropy as ce

    start, vocab = 2 * V, 4 * V
    x = _ce_inputs(dt, V, offset, seed=1)
    tgt = _ce_targets(V, start)
    x64 = x.to(F64)
    lse = torch.logsumexp(x64, -1).float()                          # the kernel's inputs, fp32
    gout = torch.tensor([1.0, -0.75, 0.5, 2.0, 0.0, -1.0, 0.125, 1.5], device="cuda")
    gr = launched(_ext, lambda: ce.ce_backward(x, tgt, lse, gout, start, smoothing, vocab))
    torch.cuda.synchronize()
    assert gr.dtype == dt and gr.shape == x.shape
    s = float(torch.tensor(smoothing, dtype=torch.float32))         # the fp32 smoothing the kernel receives
    a = x64 - lse.to(F64)[:, None]
    p = torch.exp(a)
    local = tgt - start
    owned = ((local >= 0) & (local < V)).to(F64)
    onehot = torch.zeros_like(p).scatter_(1, local.clamp(0, V - 1)[:, None], owned[:, None])
    sm = s / vocab
    g64 = gout.to(F64)[:, None]
    ref = (p - sm - (1.0 - s) * onehot) * g64
    # fp32 work before the final rounding: __expf of an argument that is itself rounded once
    # ((2 + 1.173|a|) ulps + |a|·u relative), s·(1/vocab) (two roundings), the two subtractions and the product by g.
    fp32_err = g64.abs() * (p * (2.0 ** -23 * (2 + 1.173 * a.abs()) + U * a.abs())
                            + 3 * U * (p + sm + onehot)) + U * ref.abs()
    # one ulp of the output dtype covers its rounding (half an ulp) with room for the fp32 work above;
    # 2^-126 is the flush-to-zero of fp32 results
    tol = ulp(ref, dt) + fp32_err + 2.0 ** -126
    within(gr, ref, tol, "ce grad")


def _one_rank_group():
    import torch.distributed as dist

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29544")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    return dist.group.WORLD


def test_parallel_cross_entropy_gpt2_vocab_single_rank(_ext):
    """GPT-2's 50257-wide vocab (not a multiple of the packet width) through the autograd function, with smoothing."""
    from neuronx_distributed_b200.parallel_layers.loss_functions import parallel_cross_entropy

    group = _one_rank_group()
    V, ls = 50257, 0.1
    x = _ce_inputs(torch.bfloat16, V, 0, seed=2).view(2, 4, V).requires_grad_(True)
    tgt = _ce_targets(V, 0).view(2, 4)
    n = _ext.launches()
    loss = parallel_cross_entropy(x, tgt, label_smoothing=ls, process_group=group)
    gl = torch.linspace(-1, 1, 8, device="cuda").view(2, 4)
    loss.backward(gl)
    torch.cuda.synchronize()
    assert _ext.launches() >= n + 2
    x64 = x.detach().to(F64).view(8, V)
    t = tgt.view(-1)
    lse = torch.logsumexp(x64, -1)
    pred = torch.where((t >= 0) & (t < V), x64.gather(1, t.clamp(0, V - 1)[:, None])[:, 0], torch.zeros_like(lse))
    s = ls * V / (V - 1)
    ref = (1 - s) * (lse - pred) - s * (x64.mean(-1) - lse)
    # lse = max + log(sumexp): the sumexp bound (an absolute error in the log), a few fp32 roundings of the O(|lse|)
    # terms, and the smoothed Σx/V (its chain bound over V)
    R = (x64.max(-1).values - x64.min(-1).values).max().item()
    d_lse = _sumexp_rel_bound(V, R) * 1.01 + 4 * U * lse.abs()
    loss_tol = d_lse * (1 + 2 * s) + 8 * U * (lse.abs() + pred.abs()) + s * U * (math.ceil(V / 256) + 10) * x64.abs().mean(-1)
    within(loss.detach().view(-1), ref, loss_tol, "loss")
    p = torch.exp(x64 - lse[:, None])
    onehot = torch.zeros_like(p).scatter_(1, t.clamp(0, V - 1)[:, None], ((t >= 0) & (t < V)).to(F64)[:, None])
    g64 = gl.reshape(-1, 1).to(F64)
    gref = (p - s / V - (1 - s) * onehot) * g64
    # as in test_ce_backward_vs_float64, plus the error of the fp32 lse the backward receives (relative on p)
    a = (x64 - lse[:, None]).abs()
    fp32_err = g64.abs() * (p * (2.0 ** -23 * (2 + 1.173 * a) + U * a + 2 * d_lse[:, None]) + 3 * U * (p + s / V + onehot))
    within(x.grad.view(8, V), gref, ulp(gref, torch.bfloat16) + fp32_err + 2.0 ** -126, "grad")


def test_fused_linear_cross_entropy_unaligned_vocab_shard(_ext):
    """Llama-2-13B's vocab over TP=8 is 4002 columns per rank: the lm-head GEMM output feeds the CE kernels at a width
    that is not a multiple of the packet."""
    from neuronx_distributed_b200.ops import gemm
    from neuronx_distributed_b200.parallel_layers.loss_functions import fused_linear_cross_entropy

    group = _one_rank_group()
    T, H, V, chunk = 96, 256, 4002, 40
    g = torch.Generator(device="cuda").manual_seed(3)
    h = (torch.randn(T, 1, H, device="cuda", generator=g) * 0.5).bfloat16().requires_grad_(True)
    w = (torch.randn(V, H, device="cuda", generator=g) * 0.1).bfloat16().requires_grad_(True)
    tgt = torch.randint(0, V, (T, 1), device="cuda", generator=g)
    tgt[5] = -100
    n = _ext.launches()
    loss = fused_linear_cross_entropy(h, w, tgt, process_group=group, chunk_rows=chunk)
    loss.backward()
    torch.cuda.synchronize()
    assert _ext.launches() >= n + 2 * 3                            # stats + backward for each of the 3 chunks
    # the reference starts from the bf16 logits the chunks' GEMM produces (the same call on the same rows)
    hd = h.detach().view(T, H)
    with torch.no_grad():
        L64 = torch.cat([gemm.matmul(hd[lo:lo + chunk], w.detach(), False, True) for lo in range(0, T, chunk)]).to(F64)
    h64, w64 = hd.to(F64), w.detach().to(F64)
    t = tgt.view(-1)
    keep = t != -100
    ts = torch.where(keep, t, torch.zeros_like(t))
    lse = torch.logsumexp(L64, -1)
    per_row = lse - L64.gather(1, ts[:, None])[:, 0]
    ref = per_row[keep].mean()
    R = (L64.max(-1).values - L64.min(-1).values).max().item()
    d_lse = _sumexp_rel_bound(V, R) * 1.01 + 4 * U * lse.abs().max().item()
    # per row: the lse error and a few fp32 roundings of lse and the target logit; the mean adds a chain over T rows
    loss_tol = d_lse + 8 * U * (lse.abs().max().item() + per_row.abs().max().item()) + U * T * abs(ref.item())
    assert abs(loss.item() - ref.item()) <= loss_tol, (loss.item(), ref.item(), loss_tol)
    p = torch.exp(L64 - lse[:, None])
    gl = (p - torch.zeros_like(p).scatter_(1, ts[:, None], 1.0)) * (keep.to(F64) / keep.sum())[:, None]
    # The softmax carries the lse error (relative, on p), the gradient is stored in bf16 (2^-9), and the dgrad / wgrad
    # products are bf16 GEMMs at widths the tensor-core kernel does not take (cuBLAS may round split-K partials to
    # bf16: 2·2^-9), with a final bf16 rounding of dW (2^-9): relative to the products of magnitudes |g|·|W|, |g|ᵀ·|h|.
    e = 2 * d_lse + 4 * 2.0 ** -9 + 2 * 2.0 ** -8
    dh_err = (h.grad.view(T, H).to(F64) - gl @ w64).norm()
    dw_err = (w.grad.to(F64) - gl.t() @ h64).norm()
    assert dh_err <= e * (gl.abs() @ w64.abs()).norm(), (dh_err.item(), e)
    assert dw_err <= e * (gl.abs().t() @ h64.abs()).norm(), (dw_err.item(), e)


# =====================================================================================================================
# B. RMSNorm and add-RMSNorm
# =====================================================================================================================
NORM_CASES = [(torch.bfloat16, H) for H in (128, 4096, 5120, 8192, 12288, 16384)] + \
             [(torch.float32, H) for H in (4096, 5120, 8192)] + [(torch.bfloat16, 4100)]


def _norm_bounds(x64, w64, g64, rstd, eps, dt, rows, kernel):
    """References and bounds for y, dx, dW.  The sum of squares is a positive fp32 sum whose addition chain is at most
    ceil(H/32) (a thread's columns; >= 32 threads per row) + 10 (block tree) long; ``rsqrtf`` adds 2 ulps and the
    division by H one rounding.  The torch composition (``kernel=False``) is bounded by a chain of H."""
    H = x64.shape[-1]
    chain = (math.ceil(H / 32) + 10) if kernel else H
    r_rstd = 0.5 * U * (chain + 2) * 1.01 + 2 * 2.0 ** -23
    xh = x64 * rstd
    y = xh * w64
    y_tol = ulp(y, dt) + y.abs() * (r_rstd + 3 * U)
    gw = g64 * w64
    dot = (gw * xh).mean(-1, keepdim=True)
    dx = rstd * (gw - xh * dot)
    # dx = rs·(g·w - x̂·mean(g·w·x̂)): every term carries the rstd error (twice through x̂·mean) and a few roundings
    # of its own magnitude; the mean is a chain like the sum of squares
    mag = rstd * (gw.abs() + xh.abs() * (gw * xh).abs().mean(-1, keepdim=True))
    dx_err = mag * (3 * r_rstd + U * (chain + 8))
    # dW = Σ_rows g·x̂: per-CTA partial sums over ceil(rows/grid) rows, then a sum over the grid's partials
    grid = min(rows, 4 * sms())
    dw = (g64 * xh).sum(0)
    dw_tol = ulp(dw, dt) + (g64 * xh).abs().sum(0) * (r_rstd + U * (math.ceil(rows / grid) + grid + 4))
    return y, y_tol, dx, mag, dx_err, dw, dw_tol


@pytest.mark.parametrize("rows", [1, 7, None], ids=["rows1", "rows7", "rows4SMs+5"])
@pytest.mark.parametrize("dt,H", NORM_CASES, ids=[f"{str(d)[6:]}-H{h}" for d, h in NORM_CASES])
def test_rmsnorm_and_add_rmsnorm_vs_float64(_ext, dt, H, rows):
    from neuronx_distributed_b200.ops import norm

    rows = rows or 4 * sms() + 5                                   # more rows than the backward's persistent CTAs
    eps = 1e-6
    kernel = H % VEC[dt] == 0
    g = torch.Generator(device="cuda").manual_seed(H + rows)
    # per-row scales from 2^-3 to 2^3 so a row mixed up with another changes its statistics
    scale = torch.exp2(torch.randint(-3, 4, (rows, 1), device="cuda", generator=g).float())
    x = (torch.randn(rows, H, device="cuda", generator=g) * scale).to(dt)
    r = (torch.randn(rows, H, device="cuda", generator=g) * scale).to(dt)
    w = (torch.rand(H, device="cuda", generator=g) + 0.5).to(dt)
    gy = torch.randn(rows, H, device="cuda", generator=g).to(dt)
    gh = torch.randn(rows, H, device="cuda", generator=g).to(dt)

    # --- plain RMSNorm
    xx, ww = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    n = _ext.launches()
    y = norm.rms_norm(xx, ww, eps)
    y.backward(gy)
    torch.cuda.synchronize()
    assert (_ext.launches() > n) == kernel, "H % vec != 0 must take the torch composition, every other H the kernels"
    x64, w64, g64 = x.to(F64), w.to(F64), gy.to(F64)
    rstd = torch.rsqrt(x64.pow(2).mean(-1, keepdim=True) + eps)
    y_ref, y_tol, dx_ref, _, dx_err, dw_ref, dw_tol = _norm_bounds(x64, w64, g64, rstd, eps, dt, rows, kernel)
    within(y, y_ref, y_tol, "y")
    within(xx.grad, dx_ref, ulp(dx_ref, dt) + dx_err, "dx")
    within(ww.grad, dw_ref, dw_tol, "dW")

    # --- add + RMSNorm
    xa, ra, wa = x.clone().requires_grad_(True), r.clone().requires_grad_(True), w.clone().requires_grad_(True)
    yf, hf = norm.add_rms_norm(xa, ra, wa, eps)
    torch.autograd.backward([yf, hf], [gy, gh])
    torch.cuda.synchronize()
    assert torch.equal(hf, x + r), "h is x + r rounded once to the storage dtype"
    h64 = hf.detach().to(F64)
    rstd_h = torch.rsqrt(h64.pow(2).mean(-1, keepdim=True) + eps)
    y_ref, y_tol, dx_ref, _, dx_err, dw_ref, dw_tol = _norm_bounds(h64, w64, g64, rstd_h, eps, dt, rows, kernel)
    within(yf, y_ref, y_tol, "fused y")
    dh_ref = gh.to(F64) + dx_ref
    dh_tol = ulp(dh_ref, dt) + dx_err + U * (gh.to(F64).abs() + dx_ref.abs())
    within(xa.grad, dh_ref, dh_tol, "dx (= dh)")
    assert torch.equal(xa.grad, ra.grad)
    within(wa.grad, dw_ref, dw_tol, "fused dW")
    if kernel:
        # fused_norm.cu: y is exactly rmsnorm(h_stored), bit for bit, as the unfused sequence computes it
        assert torch.equal(yf, norm.rms_norm(hf.detach(), w, eps)), "fused y differs from rms_norm(h) in some bits"


# =====================================================================================================================
# C. multi-tensor optimizer kernels
# =====================================================================================================================
CHUNK = 65536
SIZES = [1, 3, 65535, 65536, 65537] + [7 + 13 * i for i in range(50)]      # 55 tensors: more than one 48-tensor table


def _flat_views(sizes, dt, fill):
    """Views into one flat buffer.  Even-numbered views start 32-byte aligned (the vector path), odd-numbered ones one
    element later (the scalar path).  Every element outside the views is a guard set to ``fill``."""
    offs, o = [], 0
    for i, n in enumerate(sizes):
        o = (o + 7) // 8 * 8 + 8 + (i % 2)                        # >= 8 guard elements before every view
        offs.append(o)
        o += n
    buf = torch.full((o + 9,), fill, device="cuda", dtype=dt)
    guard = torch.ones(buf.numel(), dtype=torch.bool, device="cuda")
    views = []
    for off, n in zip(offs, sizes):
        views.append(buf[off:off + n])
        guard[off:off + n] = False
    return buf, views, guard


def _bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}[t.dtype])


def _chunk_weighted(views, dt, seed):
    """Fill every 64K-element chunk (and every small tensor) with ±sqrt(c/n) values so that chunk k contributes about
    c_k = 1 + (k mod 7)/4 to Σx²: all chunks count alike and no two neighbours are equal, so a lost, repeated or
    shifted chunk moves the norm by >= 1/(4·Σc) relative."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = 0
    for v in views:
        for lo in range(0, v.numel(), CHUNK):
            n = min(CHUNK, v.numel() - lo)
            c = 1 + (k % 7) / 4
            sign = torch.randint(0, 2, (n,), device="cuda", generator=g).float() * 2 - 1
            mag = math.sqrt(c / n) * (1 + 0.1 * torch.rand(n, device="cuda", generator=g))
            v[lo:lo + n] = (sign * mag).to(dt)
            k += 1
    return k


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16], ids=lambda d: str(d)[6:])
def test_multi_tensor_sq_norm_and_scale_vs_float64(_ext, dt):
    from neuronx_distributed_b200.ops import optim

    sizes = SIZES + [641 * CHUNK + 5]                               # one tensor spans two 640-chunk tables
    buf, views, guard = _flat_views(sizes, dt, 1234.5)
    nchunks = _chunk_weighted(views, dt, 0)
    guard_bits = _bits(buf)[guard].clone()
    ref = sum(float(v.to(F64).pow(2).sum()) for v in views)
    got = launched(_ext, lambda: optim.multi_tensor_sq_norm(views)).item()
    # positive terms: a thread chain of 65536/256 (+ packet) + 10 (block tree) per chunk, then one atomicAdd per chunk
    bound = U * (256 + 8 + 10 + nchunks) * 1.01 * ref
    assert abs(got - ref) <= bound, (got, ref, bound)
    assert bound < ref / (4 * 1.1 * nchunks * 3)                    # a chunk's share stays far above the bound

    sc = torch.tensor(0.7, device="cuda")
    before = [v.clone() for v in views]
    launched(_ext, lambda: optim.multi_tensor_scale_(views, sc))
    torch.cuda.synchronize()
    s64 = float(sc)
    for i, (v, b) in enumerate(zip(views, before)):
        # the product of two fp32 numbers is exact in float64; the kernel rounds it to fp32, then to the storage dtype
        assert torch.equal(v, (b.to(F64) * s64).float().to(dt)), f"tensor {i} (numel {v.numel()})"
    assert torch.equal(_bits(buf)[guard], guard_bits), "multi_tensor_scale_ wrote outside its tensors"


def _adamw_ref(p, g, m, v, gs, lr, b1, b2, eps, wd, step, hf):
    """One float64 step of the kernel's update rule from its fp32 state, and a bound on the kernel's fp32 step.
    The moments use the fp32 betas the kernel receives (1 - beta is exact in fp32 for beta in [0.5, 1]).
    m: g·gs, (1-b1)·gr, b1·m and the sum each rounded once (4u on |m| + |gr|).  v: a sum of non-negative terms;
    gr's rounding counts twice in gr², then (1-b2)·gr, ·gr, b2·v and the sum (6u on v).  The update: the fp32
    step size and decay, sqrt, + eps and the approximate division (16u together) and half v's relative error through
    the sqrt; the final product(s) on p."""
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    b1, b2 = (float(torch.tensor(b, dtype=torch.float32)) for b in (b1, b2))
    gr = g * gs
    m1 = b1 * m + (1 - b1) * gr
    v1 = b2 * v + (1 - b2) * gr * gr
    if hf:
        step_size, denom, pre, post = lr * math.sqrt(bc2) / bc1, v1.sqrt() + eps, 1.0, 1 - lr * wd
    else:
        step_size, denom, pre, post = lr / bc1, (v1 / bc2).sqrt() + eps, 1 - lr * wd, 1.0
    upd = step_size * m1 / denom
    p1 = (p * pre - upd) * post
    m_err = 4 * U * (m.abs() + gr.abs())
    v_err = 6 * U * v1
    u_err = step_size / denom * (m_err + 16 * U * m1.abs()) + upd.abs() * (v_err / (2 * v1.clamp_min(1e-300)))
    p_err = 4 * U * (p.abs() + p1.abs()) + u_err
    return p1, m1, v1, p_err, m_err, v_err


@pytest.mark.parametrize("hf", [True, False], ids=["hf", "torch"])
@pytest.mark.parametrize("with_scale", [True, False], ids=["gscale", "noscale"])
@pytest.mark.parametrize("low", [None, torch.bfloat16, torch.float16, torch.float32], ids=lambda d: str(d)[6:] if d else "nolow")
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16, torch.float16], ids=lambda d: "g" + str(d)[6:])
def test_fused_adamw_vs_float64_replay(_ext, gdt, low, with_scale, hf):
    _adamw_case(_ext, SIZES, gdt, low, with_scale, hf, seed=7)


def test_fused_adamw_2000_chunk_tensor(_ext):
    """Llama-2-7B's embedding is ~2000 chunks of 65536: one tensor over four launches' tables."""
    _adamw_case(_ext, [3, 2000 * CHUNK - 3, 65537], torch.bfloat16, torch.bfloat16, True, True, seed=8)


def _adamw_case(_ext, sizes, gdt, low, with_scale, hf, seed):
    from neuronx_distributed_b200.ops import optim

    lr, b1, b2, eps, wd = 1e-2, 0.9, 0.95, 1e-8, 0.1
    G = torch.Generator(device="cuda").manual_seed(seed)
    pb, ps, pg = _flat_views(sizes, torch.float32, 77.0)
    mb, ms, _ = _flat_views(sizes, torch.float32, 77.0)
    vb, vs, _ = _flat_views(sizes, torch.float32, 77.0)
    gb, gs_, _ = _flat_views(sizes, gdt, 77.0)
    bufs = [pb, mb, vb, gb]
    if low is not None:
        lb, ls, _ = _flat_views(sizes, low, 77.0)
        bufs.append(lb)
    guards = [_bits(b)[pg].clone() for b in bufs]
    for p in ps:
        p.copy_(torch.randn(p.numel(), device="cuda", generator=G))
    for t in ms + vs:
        t.zero_()
    if low is not None:
        for lo, p in zip(ls, ps):
            lo.copy_(p)
    gs = torch.tensor(0.6, device="cuda") if with_scale else None
    gs64 = float(gs) if with_scale else 1.0                          # the fp32 scale the kernel reads
    for step in (1, 2, 3):
        for i, g in enumerate(gs_):
            # magnitudes 2^-6..2^2 varying per tensor and step, signs random: moments cancel across steps
            e = (i + step) % 9 - 6
            g.copy_((torch.randn(g.numel(), device="cuda", generator=G) * 2.0 ** e))
        prev = [(p.to(F64), g.to(F64), m.to(F64), v.to(F64)) for p, g, m, v in zip(ps, gs_, ms, vs)]
        launched(_ext, lambda: optim.fused_adamw_(ps, gs_, ms, vs, lr, b1, b2, eps, wd, step, grad_scale=gs,
                                                  model_params=ls if low is not None else None, hf_form=hf))
        torch.cuda.synchronize()
        for i, (p, m, v) in enumerate(zip(ps, ms, vs)):
            p1, m1, v1, p_err, m_err, v_err = _adamw_ref(*prev[i], gs64, lr, b1, b2, eps, wd, step, hf)
            within(m, m1, m_err, f"step {step} tensor {i} m")
            within(v, v1, v_err, f"step {step} tensor {i} v")
            within(p, p1, p_err, f"step {step} tensor {i} p")
            # an update is ~lr: far above p's bound, so a chunk updated twice, never, or with another chunk's grads fails
            assert p_err.max() < lr * 1e-2
            if low is not None:
                assert torch.equal(ls[i], p.to(low)), f"step {step} tensor {i}: low copy is not p rounded"
        for b, gbits in zip(bufs, guards):
            assert torch.equal(_bits(b)[pg], gbits), "fused_adamw_ wrote outside its tensors"


# =====================================================================================================================
# D. GEMM epilogue: layouts x output dtype x accumulate
# =====================================================================================================================
GEMM_MN = (8, 264, 1000)
GEMM_K = (8, 16, 40, 72, 4096)


def _grid_bf16(shape, g):
    """Multiples of 1/8 in [-2, 2]: every product is a multiple of 2^-6 and every partial sum of K <= 4096 of them is
    below 2^14, so the fp32 accumulation is exact in any order.  What is left is the epilogue's rounding."""
    return (torch.randint(-16, 17, shape, device="cuda", generator=g).float() / 8).bfloat16()


@pytest.mark.parametrize("accumulate", [False, True], ids=["store", "accumulate"])
@pytest.mark.parametrize("out_dt", [torch.float32, torch.bfloat16], ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
def test_gemm_epilogue_vs_float64(_ext, layout, out_dt, accumulate):
    from neuronx_distributed_b200.ops import gemm

    ta, tb = layout[0] == "t", layout[1] == "t"
    g = torch.Generator(device="cuda").manual_seed(11)
    nan_bits = _bits(torch.full((1,), float("nan"), dtype=out_dt))[0].item()
    for M in GEMM_MN:
        for N in GEMM_MN:
            for K in GEMM_K:
                a = _grid_bf16((K, M) if ta else (M, K), g)
                b = _grid_bf16((N, K) if tb else (K, N), g)
                buf = torch.full((M + 24, N), float("nan"), device="cuda", dtype=out_dt)
                out = buf[:M]
                if accumulate:
                    out.copy_(torch.randn(M, N, device="cuda", generator=g) * 16)
                out0 = out.to(F64)
                launched(_ext, lambda: gemm.matmul(a, b, ta, tb, out=out, accumulate=accumulate))
                torch.cuda.synchronize()
                a64 = a.to(F64).t() if ta else a.to(F64)
                b64 = b.to(F64).t() if tb else b.to(F64)
                ref = a64 @ b64 + (out0 if accumulate else 0)
                what = f"{layout} M={M} N={N} K={K}"
                assert torch.equal(_bits(buf[M:]), torch.full_like(_bits(buf[M:]), nan_bits)), f"{what}: rows past M written"
                if not accumulate or out_dt == torch.float32:
                    # the exact sum (plus out0) rounded once: the float64 result rounded to the output dtype
                    assert torch.equal(out, ref.to(out_dt)), f"{what}: max err {(out.to(F64) - ref).abs().max().item()}"
                else:
                    # out0 + acc rounded to fp32, then to bf16: within one bf16 ulp
                    within(out, ref, ulp(ref, torch.bfloat16), what)


# =====================================================================================================================
# E. RoPE
# =====================================================================================================================
def _rope64(x64, cos, sin, sign):
    d2 = x64.shape[-1] // 2
    c = cos.to(F64)[None, :, None, :]
    s = sin.to(F64)[None, :, None, :] * sign
    x1, x2 = x64[..., :d2], x64[..., d2:]
    return (torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1),
            torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], -1))


ROPE_CASES = {
    # GPT-NeoX style: the first 24 of 96 head dims rotate; half = 12 is not a packet multiple → rope_scalar_kernel
    "partial24of96-bf16": (torch.bfloat16, 96, 24, False),
    # [S,B,H,D] storage seen as [B,S,H,D]: strided B/S, packet-aligned → the vector kernel
    "sbhd-view-bf16": (torch.bfloat16, 128, 128, True),
    "fp32": (torch.float32, 64, 64, False),
    "sbhd-view-fp32": (torch.float32, 64, 64, True),
}


@pytest.mark.parametrize("case", list(ROPE_CASES))
def test_rope_fwd_bwd_vs_float64(_ext, case):
    from neuronx_distributed_b200.ops import rope

    dt, Dh, D, sbhd = ROPE_CASES[case]
    B, S, Hh = 3, 37, 5
    g = torch.Generator(device="cuda").manual_seed(13)
    if sbhd:
        base = torch.randn(S, B, Hh, Dh, device="cuda", generator=g).to(dt)
        x = base.transpose(0, 1)
    else:
        base = torch.randn(B, S, Hh, Dh, device="cuda", generator=g).to(dt)
        x = base[..., :D]
    cos, sin = rope.rope_tables(S + 5, D, device="cuda", offset=3)
    cos, sin = cos[:S], sin[:S]
    xx = x.detach().requires_grad_(True)
    n = _ext.launches()
    y = rope.apply_rotary(xx, cos, sin)
    gy = torch.randn(B, S, Hh, D, device="cuda", generator=g).to(dt)
    y.backward(gy)
    torch.cuda.synchronize()
    assert _ext.launches() >= n + 2
    ref, mag = _rope64(x.to(F64), cos, sin, 1.0)
    # a·c ∓ b·s in fp32 (two roundings on the terms' magnitudes), then one rounding to the storage dtype
    within(y, ref, ulp(ref, dt) + 2 * U * mag, "rope forward")
    gref, gmag = _rope64(gy.to(F64), cos, sin, -1.0)                # the inverse rotation
    within(xx.grad, gref, ulp(gref, dt) + 2 * U * gmag, "rope backward")
