"""The one-launch decode MoE block (``csrc/moe_tkg.cu`` through ``ops.moe_tkg``) against a float64 oracle at real-model shapes.

The oracle below follows the rounding points of ``ops.moe_tkg.moe_block_tkg_reference`` (normalised tokens, rounded
logits, affinities, the normalisation sum and the normalised weights are rounded to the activation dtype) and is float64
everywhere else.  Its top-k is a stable descending sort: among equal scores the smaller expert index wins, which is the
kernel's rule (``torch.topk`` leaves that order open, so it is not the oracle).  A CPU test ties the oracle to the module
semantics through ``moe_block_tkg_reference``.

Two input modes:
- exact: no norm, x / router / gate|up weights (and router bias) on power-of-two grids, so router logits and gate|up sums
  are exact in fp32 in any order.  Logits and expert ids (in order) must be bit-equal, routing weights equal or one bf16
  ulp apart (the kernel's affinities use ``__expf``).
- margin: RMSNorm on, a router bias that makes K experts clearly hot.  The kernel may round a normalised element to the
  neighbouring bf16 value wherever the exact value lies within its fp32 error of a rounding midpoint; the bounds allow one
  bf16 ulp in exactly those elements (the generated inputs avoid them, see ``make_inputs``).  Before comparing ids, the
  test asserts that the float64 gap between the chosen and the other experts is larger than the logit bound, so no seed
  can make the routing check flaky.

The output is checked elementwise against the oracle evaluated at the ids and weights the kernel returned (which are
checked first).  The bound, derived in ``out_bound``: one bf16 ulp of the reference (the final rounding) plus fp32
accumulation over the 64-row slices and their partial sums, the activation's evaluation error, and in margin mode the
propagated input ulps and the fp32 error of the gate|up sums.  The sensitivity tests show that the bounds reject a kernel
that drops one 64-row slice of I, moves one routing weight by one bf16 ulp (exact mode), swaps gate and up, or shifts
``e0`` by one.

Out of scope: the non-cooperative launch (``NXD_MOE_TKG_COOP=0``), whose grid is not guaranteed to be co-resident on a
shared GPU.  Every launch here is cooperative and every pointer 16-byte aligned.
"""
import math
import os

import pytest
import torch

F64, BF16 = torch.float64, torch.bfloat16
U32 = 2.0 ** -24                     # fp32 unit roundoff
INF = float("inf")


# =====================================================================================================================
# float64 oracle
# =====================================================================================================================
def rnd(v: torch.Tensor, dt) -> torch.Tensor:
    """Round a float64 value to ``dt`` the way the kernel does (via fp32) and return it as float64."""
    return v.to(torch.float32).to(dt).to(F64)


def ulp_bf16(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |v| (7 stored bits, normal range from 2^-126)."""
    e = torch.floor(torch.log2(v.abs().to(F64).clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def normed(x, gamma, eps):
    """(xn, z): the normalised tokens rounded to x.dtype and their exact value before rounding (None without a norm)."""
    xf = x.to(F64)
    if gamma is None:
        return xf, None
    z = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * gamma.to(F64)
    return rnd(z, x.dtype), z


def router_logits(xn, rw, rb, round_logits, dt):
    L = xn @ rw.to(F64).t()
    if rb is not None:
        L = L + rb.to(F64)
    return rnd(L, dt) if round_logits else L


def route(logits, K, router_act=0, act_over_topk=False, normalize=True, dt=BF16):
    """(idx [T,K] int64, w [T,K] float64): stable top-k, ties to the smaller expert index."""
    actf = (lambda v: torch.softmax(v, -1)) if router_act == 0 else torch.sigmoid
    if act_over_topk:
        idx = torch.sort(logits, dim=-1, descending=True, stable=True).indices[:, :K]
        w = actf(logits.gather(1, idx))
    else:
        aff = actf(logits)
        idx = torch.sort(aff, dim=-1, descending=True, stable=True).indices[:, :K]
        w = aff.gather(1, idx)
    w = rnd(w, dt)
    if normalize:
        w = rnd(w / rnd(w.sum(-1, keepdim=True), dt).clamp(min=1e-9), dt)
    return idx, w


def glu(g, u, act, alpha, beta, clamps):
    g = g.clamp(min=clamps[0], max=clamps[1])
    u = u.clamp(min=clamps[2], max=clamps[3])
    if act == 0:
        return torch.nn.functional.silu(g) * u, u
    if act == 1:
        return torch.nn.functional.gelu(g) * u, u
    if act == 2:
        return torch.nn.functional.gelu(g, approximate="tanh") * u, u
    if act == 3:
        return g * torch.sigmoid(alpha * g) * (u + beta), u + beta
    return torch.relu(g) * u, u


def experts(xn, idx, w, w_gu, w_dn, e0, pre_scale=False, act=0, act_alpha=1.0, act_beta=0.0, clamps=(-INF, INF, -INF, INF),
            xerr=None, exact_gu=True, drop=None, swap=False):
    """The chosen local experts in float64: ``(out [T,H], parts)`` where ``parts`` holds the magnitudes the bound needs.

    ``xerr`` [T,H]: possible error of each normalised input element (margin mode); ``exact_gu``: gate|up sums are exact in
    fp32.  ``drop=(slot, chunk, slice)`` removes one work item of the down GEMV (256 columns of H x 64 rows of I) of the
    slot's expert and ``swap`` exchanges gate and up: both only to show that the bounds see such a kernel."""
    T, H = xn.shape
    El, I = w_gu.shape[0], w_dn.shape[1]
    out = torch.zeros(T, H, dtype=F64, device=xn.device)
    A, B, D = torch.zeros_like(out), torch.zeros_like(out), torch.zeros_like(out)
    le_all = idx - e0
    for le in sorted(set(le_all[(le_all >= 0) & (le_all < El)].tolist())):
        toks, ks = torch.nonzero(le_all == le, as_tuple=True)
        Wg = w_gu[le].to(F64)
        gu = xn[toks] @ Wg
        dgu = torch.zeros_like(gu)
        if xerr is not None:
            dgu += xerr[toks] @ Wg.abs()
        if not exact_gu:                                      # 128 fmaf per lane, then one red.add per 128-row slice
            dgu += (128 + math.ceil(H / 128) + 2) * U32 * (xn[toks].abs() @ Wg.abs())
        del Wg
        wt = w[toks, ks].unsqueeze(1)
        g, u = (gu[:, I:], gu[:, :I]) if swap else (gu[:, :I], gu[:, I:])
        dg, du = dgu[:, :I], dgu[:, I:]
        if pre_scale:
            g, u, dg, du = g * wt, u * wt, dg * wt, du * wt
        a, u_eff = glu(g, u, act, act_alpha, act_beta, clamps)
        ws = torch.ones_like(wt) if pre_scale else wt
        # a(g, u) is 1.2-Lipschitz in g per unit |u|, and |act(g)| <= |g|, for every activation here (clamps only shrink)
        da = 1.2 * dg * (u_eff.abs() + du) + (g.abs() + 1.2 * dg) * du
        Wd = w_dn[le].to(F64)
        if drop is not None and drop[0] in [(int(t), int(k)) for t, k in zip(toks, ks)]:
            row = [(int(t), int(k)) for t, k in zip(toks, ks)].index(drop[0])
            y_drop = (a[row:row + 1] * ws[row:row + 1])[:, drop[2] * 64:(drop[2] + 1) * 64] @ \
                Wd[drop[2] * 64:(drop[2] + 1) * 64, drop[1] * 256:(drop[1] + 1) * 256]
            out[toks[row], drop[1] * 256:(drop[1] + 1) * 256] -= y_drop[0]
        out.index_add_(0, toks, (a * ws) @ Wd)
        Wa = Wd.abs()
        A.index_add_(0, toks, (a.abs() * ws.abs()) @ Wa)
        B.index_add_(0, toks, (g.abs() * u_eff.abs() * ws.abs()) @ Wa)
        D.index_add_(0, toks, (da * ws.abs()) @ Wa)
        del Wd, Wa
    return out, dict(A=A, B=B, D=D, I=I)


def out_bound(ref, parts, K):
    """|kernel - ref| <= ulp_bf16(ref) + 1.01 (u32 (n_acc A + 16 (A + B)) + D) elementwise, where
    A = sum_slots sum_i |w a_i| |W_dn[i,h]| (the fp32 accumulation: 64 fmaf per lane and one red.add per 64-row slice and
    slot, n_acc = 64 + K ceil(I/64) + 2), B = the same with |g_i u_i| (the activation is evaluated to 16 u32 relative to
    |a| + |g u|: __expf, erff, tanhf and the fast division), D = the propagated input ulps (margin mode).  The final bf16
    rounding of the fp32 accumulator adds at most one ulp of the reference."""
    n_acc = 64 + K * math.ceil(parts["I"] / 64) + 2
    return ulp_bf16(ref) + 1.01 * (U32 * (n_acc * parts["A"] + 16 * (parts["A"] + parts["B"])) + parts["D"])


def input_ulps(z, H):
    """Elements of the normalised tokens the kernel may round to the other neighbour: the exact value lies within the fp32
    error of the kernel's RMSNorm (H/32 fmaf per lane + warp sum + rsqrtf + two products, doubled) of a bf16 midpoint.
    Returns one bf16 ulp at those elements and 0 elsewhere."""
    if z is None:
        return None
    eps = 2 * ((H / 32 + 7) / 2 + 6) * U32
    lo, hi = rnd(z * (1 - eps), BF16), rnd(z * (1 + eps), BF16)
    return torch.where(lo != hi, ulp_bf16(z.abs() * (1 + eps)), torch.zeros_like(z))


def logit_bound(xn, xerr, rw, rb, L, round_logits, H):
    """Bound on |kernel logit - oracle logit|: propagated input ulps, H/32 fmaf per lane + warp sum + bias add, then the
    bf16 rounding of both."""
    rwa = rw.to(F64).abs()
    d = (H / 32 + 6) * U32 * (xn.abs() @ rwa.t())
    if xerr is not None:
        d = d + xerr @ rwa.t()
    if rb is not None:
        d = d + U32 * rb.to(F64).abs()
    d = 1.01 * d
    return d + (ulp_bf16(L.abs() + d) if round_logits else U32 * (L.abs() + d))


def oracle(x, gamma, rw, rb, w_gu, w_dn, e0, K, eps=1e-6, router_act=0, act_over_topk=False, normalize=True, pre_scale=False,
           round_logits=True, act=0, act_alpha=1.0, act_beta=0.0, clamps=(-INF, INF, -INF, INF)):
    """(out float64 [T,H], logits float64 [T,E], idx [T,K], w float64 [T,K]) with the reference's rounding points."""
    xn, _ = normed(x, gamma, eps)
    L = router_logits(xn, rw, rb, round_logits, x.dtype)
    idx, w = route(L, K, router_act, act_over_topk, normalize, x.dtype)
    out, _ = experts(xn, idx, w, w_gu, w_dn, e0, pre_scale, act, act_alpha, act_beta, clamps)
    return out, L, idx, w


# =====================================================================================================================
# inputs
# =====================================================================================================================
def _grid_bf16(shape, n, scale, g):
    """Integers in [-n, n] times a power of two ``scale``: exact in bf16 for n <= 256."""
    return torch.randint(-n, n + 1, shape, device=g.device, generator=g, dtype=torch.int16).to(BF16).mul_(scale)


MARGIN_EPS = 1e-5


def make_inputs(mode, T, H, E, I, K, El=None, bias=False, seed=0, dev="cuda"):
    """``exact``: gamma None; x multiples of 1/8 in [-2, 2]; router and gate|up weights multiples of 2^-8 sized for logits
    of std ~1.5 and gate|up of std ~2; bias multiples of 1/16.  Every product is a multiple of 2^-11 and every partial sum
    stays below 2^13 (asserted), so each sum fits fp32's 24 bits in any order.  ``margin``: randn tokens, norm weight in
    [0.5, 1.5], router noise of std ~0.3 and K hot experts (bias +4).  Where a normalised value (eps 1e-5) lies within the
    kernel's RMSNorm error of a bf16 rounding midpoint, that column's norm weight moves by 2^-6: kernel and oracle then
    round every normalised element the same way and the bound's input-ulp term is zero."""
    El = E if El is None else El
    g = torch.Generator(device=dev).manual_seed(seed)
    if mode == "exact":
        r = max(1, min(64, round(580 / math.sqrt(H))))
        q = max(1, min(127, round(770 / math.sqrt(H))))
        x = _grid_bf16((T, H), 16, 0.125, g)
        gamma = None
        rw = _grid_bf16((E, H), r, 2.0 ** -8, g)
        rb = _grid_bf16((E,), 16, 1 / 16, g).float() if bias else None
        w_gu = _grid_bf16((El, H, 2 * I), q, 2.0 ** -8, g)
        assert 2 * r * 2.0 ** -8 * H + 1 < 2 ** 13 and 2 * q * 2.0 ** -8 * H < 2 ** 13
    else:
        x = torch.randn(T, H, device=dev, generator=g).to(BF16)
        gamma = (torch.rand(H, device=dev, generator=g) + 0.5).to(BF16)
        for _ in range(20):                                # move the norm weight off the kernel's rounding ambiguity
            amb = (input_ulps(normed(x, gamma, MARGIN_EPS)[1], H) > 0).any(0)
            if not amb.any():
                break
            gamma = torch.where(amb, (gamma.to(F64) * (1 + 2.0 ** -6)).to(BF16), gamma)
        assert not amb.any()
        rw = (torch.randn(E, H, device=dev, generator=g) * (0.3 / math.sqrt(H))).to(BF16)
        rb = torch.zeros(E, device=dev)
        rb[torch.randperm(E, device=dev, generator=g)[:K]] = 4.0
        w_gu = (torch.randn(El, H, 2 * I, device=dev, generator=g) * (2 / math.sqrt(H))).to(BF16)
    w_dn = (torch.randn(El, I, H, device=dev, generator=g) * I ** -0.5).to(BF16)
    return x, gamma, rw, rb, w_gu, w_dn


# =====================================================================================================================
# CPU: the oracle is the module's semantics, and each bound rejects a wrong kernel
# =====================================================================================================================
ORACLE_VARIANTS = [dict(), dict(router_act=1), dict(act_over_topk=True), dict(act_over_topk=True, router_act=1, normalize=False),
                   dict(pre_scale=True), dict(act=1), dict(act=2, normalize=False), dict(act=4, pre_scale=True),
                   dict(act=3, act_alpha=1.702, act_beta=1.0, clamps=(-0.7, 0.8, -0.6, 0.9)),
                   dict(act=3, act_alpha=1.702, act_beta=1.0, clamps=(-INF, 7.0, -7.0, 7.0), act_over_topk=True),
                   dict(round_logits=False), dict(gamma=False), dict(bias=False), dict(e0=4, El=4)]


@pytest.mark.parametrize("v", ORACLE_VARIANTS, ids=lambda v: "-".join(f"{k}={val}" for k, val in v.items()) or "default")
def test_oracle_matches_the_reference_op_on_fp32(v):
    """On fp32 inputs (rounding points = fp32) the float64 oracle and ``moe_block_tkg_reference`` agree: ids in order
    (random fp32 logits have no ties), logits, weights and the output to fp32 accuracy."""
    from neuronx_distributed_b200.ops import moe_tkg

    v = dict(v)
    use_gamma, use_bias, e0, El = v.pop("gamma", True), v.pop("bias", True), v.pop("e0", 0), v.pop("El", 8)
    torch.manual_seed(0)
    T, H, E, I, K = 5, 48, 8, 40, 3
    x = torch.randn(T, H)
    gamma = torch.rand(H) + 0.5 if use_gamma else None
    rw, rb = torch.randn(E, H) * 0.3, (torch.randn(E) * 0.1 if use_bias else None)
    w_gu, w_dn = torch.randn(El, H, 2 * I) * 0.2, torch.randn(El, I, H) * 0.2
    args = (x, gamma, rw, rb, w_gu, w_dn, e0, K)
    ro, rl, ri, rwt = moe_tkg.moe_block_tkg_reference(*args, eps=1e-5, **v)
    oo, ol, oi, ow = oracle(*args, eps=1e-5, **v)
    assert torch.equal(ri, oi), (ri, oi)
    torch.testing.assert_close(rl.double(), ol, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(rwt.double(), ow, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ro.double(), oo, rtol=1e-4, atol=1e-4)
    assert int(((oi >= e0) & (oi < e0 + El)).sum()) > 0


def _violations(got, ref, bound):
    return int((~((got.to(F64) - ref).abs() <= bound)).sum())


@pytest.mark.parametrize("mode", ["exact", "margin"])
def test_bounds_reject_perturbed_oracles(mode):
    """At the Mixtral TP=8 shape with 8 tokens: the float64 result rounded to bf16 passes the bound, and each perturbation
    of the kind a kernel bug makes (one dropped work item of the down GEMV, one routing weight one bf16 ulp off, gate and up
    swapped, e0 off by one) is rejected by it.  The margin bound covers the worst-case fp32 error of gate|up sums that are
    not exact and is too wide to resolve one ulp of a routing weight; the exact bound resolves it, and in both modes the
    weights themselves are checked to one ulp."""
    T, H, E, I, K = 8, 4096, 8, 1792, 2
    x, gamma, rw, rb, w_gu, w_dn = make_inputs(mode, T, H, E, I, K, seed=3, dev="cpu")
    eps = 1e-5
    xn, z = normed(x, gamma, eps)
    xerr = input_ulps(z, H)
    L = router_logits(xn, rw, rb, True, BF16)
    idx, w = route(L, K)
    kw = dict(xerr=xerr, exact_gu=mode == "exact")
    ref, parts = experts(xn, idx, w, w_gu, w_dn, 0, **kw)
    bound = out_bound(ref, parts, K)
    assert _violations(ref.to(BF16), ref, bound) == 0
    w_up = w.clone()
    w_up[0, 0] = w[0, 0] + ulp_bf16(w[0, 0])
    perturbed = {
        "dropped 64-row slice": experts(xn, idx, w, w_gu, w_dn, 0, drop=((0, 0), 3, 5), **kw)[0],
        "weight one ulp off": experts(xn, idx, w_up, w_gu, w_dn, 0, **kw)[0],
        "gate and up swapped": experts(xn, idx, w, w_gu, w_dn, 0, swap=True, **kw)[0],
        "e0 shifted by one": experts(xn, idx, w, w_gu, w_dn, 1, **kw)[0],
    }
    if mode == "margin":
        del perturbed["weight one ulp off"]
    for name, p in perturbed.items():
        n = _violations(p.to(BF16), ref, bound)
        assert n > 0, f"{mode}: the bound does not see '{name}'"


# =====================================================================================================================
# GPU
# =====================================================================================================================
@pytest.fixture(scope="module")
def _ext():
    from neuronx_distributed_b200 import ops

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


@pytest.fixture
def kernel_on(monkeypatch):
    monkeypatch.setenv("NXD_MOE_TKG_KERNEL", "1")
    monkeypatch.setenv("NXD_MOE_TKG_COOP", "1")


def run_op(_ext, x, gamma, rw, rb, w_gu, w_dn, e0, K, eps=1e-5, **kw):
    """The op on the kernel (exactly one launch)."""
    from neuronx_distributed_b200.ops import moe_tkg

    assert moe_tkg.kernel_eligible(x, rw, w_gu, w_dn, K, gamma)
    n = _ext.launches()
    out, logits, idx, w = moe_tkg.moe_block_tkg(x, gamma, rw, rb, w_gu, w_dn, e0, K, eps, **kw)
    assert _ext.launches() == n + 1, "the op did not launch the kernel"
    torch.cuda.synchronize()
    return out, logits, idx, w


def check(got, inputs, e0, K, mode, eps=1e-5, what="", **kw):
    """Every output of the kernel against the float64 oracle; returns (ref, bound) of the output."""
    x, gamma, rw, rb, w_gu, w_dn = inputs
    out, logits, idx, w = got
    H = x.shape[1]
    route_kw = {k: kw[k] for k in ("router_act", "act_over_topk", "normalize") if k in kw}
    round_logits = kw.get("round_logits", True)
    xn, z = normed(x, gamma, eps)
    xerr = input_ulps(z, H)
    L = router_logits(xn, rw, rb, round_logits, BF16)
    oidx, ow = route(L, K, dt=BF16, **route_kw)
    Lk = logits.to(F64)
    if mode == "exact":
        assert torch.equal(Lk, L), f"{what}: logits differ at {(Lk != L).nonzero().tolist()[:4]}"
        assert torch.equal(idx, oidx), f"{what}: ids {idx.tolist()} want {oidx.tolist()}"
    else:
        tol = logit_bound(xn, xerr, rw, rb, L, round_logits, H)
        assert ((Lk - L).abs() <= tol).all(), f"{what}: logits outside the bound by {((Lk - L).abs() - tol).max().item():.3e}"
        if K < rw.shape[0]:                                   # the choice is clear: no kernel rounding can change it
            chosen = torch.zeros_like(L, dtype=torch.bool).scatter_(1, oidx, True)
            lo = torch.where(chosen, L - tol, torch.full_like(L, INF)).min(-1).values
            hi = torch.where(chosen, torch.full_like(L, -INF), L + tol).max(-1).values
            assert (lo > hi).all(), f"{what}: top-{K} margin {(lo - hi).min().item():.3e} is inside the logit bound"
        assert torch.equal(idx.sort(-1).values, oidx.sort(-1).values), f"{what}: ids {idx.tolist()} want {oidx.tolist()}"
        kidx, ow = route(Lk, K, dt=BF16, **route_kw)         # the order among the chosen follows the kernel's own logits
        assert torch.equal(idx, kidx), f"{what}: ids {idx.tolist()} not in the order of the kernel's logits {kidx.tolist()}"
    wd = (w.to(F64) - ow).abs()
    assert (wd <= ulp_bf16(ow)).all() and torch.equal(rnd(w.to(F64), BF16), w.to(F64)), \
        f"{what}: weights {w.tolist()} want {ow.tolist()}"
    exp_kw = {k: kw[k] for k in ("pre_scale", "act", "act_alpha", "act_beta", "clamps") if k in kw}
    ref, parts = experts(xn, idx, w.to(F64), w_gu, w_dn, e0, xerr=xerr, exact_gu=mode == "exact", **exp_kw)
    bound = out_bound(ref, parts, K)
    err = (out.to(F64) - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; worst {err.max().item():.3e} at bound "
                           f"{bound.flatten()[err.flatten().argmax()].item():.3e}, first {bad.nonzero().tolist()[:4]}")
    return ref, bound


# name: (H, E, K, I, token counts, extra): real-model geometries and the kernel's edges
CASES = {
    "mixtral-8x7b-tp8": (4096, 8, 2, 1792, range(1, 9), {}),
    "mixtral-8x7b-tp1": (4096, 8, 2, 14336, (1,), {}),
    "dbrx-tp8-ep2-e0=0": (6144, 16, 4, 1344, (1, 4), dict(e0=0, El=8)),
    "dbrx-tp8-ep2-e0=8": (6144, 16, 4, 1344, (1, 4), dict(e0=8, El=8)),
    "qwen1.5-moe": (2048, 60, 4, 1408, (1, 5), dict(normalize=False)),            # lanes 32..59: second group partly full
    "qwen3-30b-a3b-tp4": (2048, 128, 8, 192, (1, 8), {}),                          # 2I = 384: a partial 256-column chunk
    "deepseek-v3-tp8": (7168, 256, 8, 256, (8,), dict(router_act=1, bias=True)),   # E at its 256 limit
    "k1-sigmoid-over-topk": (5120, 16, 1, 1024, (1, 3), dict(router_act=1, act_over_topk=True)),
    # H % 128 = 64, H % 256 = 64, I % 64 = 40, 2I % 256 = 208: every tail path
    "ragged-swiglu": (2880, 32, 4, 360, (1, 7), dict(act=3, act_alpha=1.702, act_beta=1.0, clamps=(-INF, 7.0, -7.0, 7.0),
                                                     act_over_topk=True)),
    "minimum": (8, 1, 1, 8, (1, 8), {}),
    "smem-limit": (12800, 8, 2, 512, (8,), {}),                                    # T*H*2 = 200 KiB of dynamic smem
}


def _split(extra):
    extra = dict(extra)
    e0, El, bias = extra.pop("e0", 0), extra.pop("El", None), extra.pop("bias", False)
    return e0, El, bias, extra


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_real_model_shapes_exact(_ext, kernel_on, name):
    H, E, K, I, Ts, extra = CASES[name]
    e0, El, bias, kw = _split(extra)
    for T in Ts:
        inputs = make_inputs("exact", T, H, E, I, K, El=El, bias=bias, seed=T)
        got = run_op(_ext, *inputs, e0, K, **kw)
        check(got, inputs, e0, K, "exact", what=f"{name} T={T}", **kw)


MARGIN_CASES = {"mixtral-8x7b-tp8": (1, 8), "dbrx-tp8-ep2-e0=8": (4,), "qwen3-30b-a3b-tp4": (8,), "deepseek-v3-tp8": (8,),
                "k1-sigmoid-over-topk": (3,), "ragged-swiglu": (7,), "smem-limit": (8,)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MARGIN_CASES))
def test_real_model_shapes_with_norm_margin(_ext, kernel_on, name):
    H, E, K, I, _, extra = CASES[name]
    e0, El, _, kw = _split(extra)
    for T in MARGIN_CASES[name]:
        inputs = make_inputs("margin", T, H, E, I, K, El=El, seed=100 + T)
        if e0:                                             # make the hot experts local to this slice
            inputs[3].zero_()
            inputs[3][e0 + torch.randperm(El, generator=torch.Generator().manual_seed(T))[:K]] = 4.0
        got = run_op(_ext, *inputs, e0, K, **kw)
        check(got, inputs, e0, K, "margin", what=f"{name} T={T}", **kw)


# T, H, E, I, K, e0, El, options: activations 0..4, pre_scale, fp32 logits (the first five were the kernel's first checks)
VARIANTS = [
    (1, 1024, 8, 512, 2, 0, 8, {}),
    (5, 2048, 16, 768, 4, 4, 8, dict(router_act=1, normalize=False)),
    (8, 1024, 64, 256, 8, 0, 64, dict(act_over_topk=True)),
    (3, 1024, 8, 512, 2, 0, 8, dict(pre_scale=True, act=3, act_alpha=1.702, act_beta=1.0, clamps=(-0.7, 0.8, -0.6, 0.9))),
    (2, 4096, 8, 1792, 2, 0, 8, dict(act=2)),
    (4, 1024, 16, 512, 4, 0, 16, dict(act=1)),
    (4, 1024, 16, 512, 4, 0, 16, dict(act=4, pre_scale=True)),
    (6, 1024, 16, 512, 4, 0, 16, dict(round_logits=False, router_act=1, act_over_topk=True)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "margin"])
@pytest.mark.parametrize("case", range(len(VARIANTS)))
def test_activation_and_routing_variants(_ext, kernel_on, case, mode):
    T, H, E, I, K, e0, El, kw = VARIANTS[case]
    inputs = make_inputs(mode, T, H, E, I, K, El=El, bias=True, seed=case)
    if mode == "margin" and e0:
        inputs[3].zero_()
        inputs[3][e0:e0 + K] = 4.0
    got = run_op(_ext, *inputs, e0, K, **kw)
    check(got, inputs, e0, K, mode, what=f"variant {case} {mode} {kw}", **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(router_act=1), dict(act_over_topk=True), dict(act_over_topk=True, router_act=1)],
                         ids=["softmax", "sigmoid", "softmax-over-topk", "sigmoid-over-topk"])
def test_exact_ties_go_to_the_smaller_index(_ext, kernel_on, kw):
    """Router rows duplicated: 16 experts share 4 distinct rows (scattered over the indices), so logits tie bit for bit and
    the smaller expert index must win every tie."""
    T, H, E, I, K = 8, 1024, 16, 256, 3
    x, gamma, rw, rb, w_gu, w_dn = make_inputs("exact", T, H, E, I, K, seed=7)
    group = torch.randperm(E, generator=torch.Generator().manual_seed(1)) % 4
    rw = rw[:4][group.cuda()].contiguous()
    inputs = (x, gamma, rw, rb, w_gu, w_dn)
    got = run_op(_ext, *inputs, 0, K, **kw)
    check(got, inputs, 0, K, "exact", what=f"ties {kw}", **kw)
    assert (got[1][:, :, None] == got[1][:, None, :]).sum() > T * E, "no ties were produced"


@pytest.mark.gpu
def test_expert_parallel_slices_sum_to_the_whole(_ext, kernel_on):
    """DBRX at TP=8 with 4 tokens: the outputs of the e0 = 0 and e0 = 8 slices sum to the El = E result within the sum of
    their bounds; every slice returns the complete logits, ids and weights."""
    H, E, K, I, T = 6144, 16, 4, 1344, 4
    x, gamma, rw, rb, w_gu, w_dn = make_inputs("exact", T, H, E, I, K, seed=11)
    full = run_op(_ext, x, gamma, rw, rb, w_gu, w_dn, 0, K)
    ref, _ = check(full, (x, gamma, rw, rb, w_gu, w_dn), 0, K, "exact", what="EP whole")
    total, tb = torch.zeros_like(ref), torch.zeros_like(ref)
    for e0 in (0, 8):
        sl = (x, gamma, rw, rb, w_gu[e0:e0 + 8].contiguous(), w_dn[e0:e0 + 8].contiguous())
        got = run_op(_ext, *sl, e0, K)
        assert torch.equal(got[1], full[1]) and torch.equal(got[2], full[2]) and torch.equal(got[3], full[3])
        _, b = check(got, sl, e0, K, "exact", what=f"EP slice e0={e0}")
        total += got[0].to(F64)
        tb += b
    assert ((total - ref).abs() <= tb).all(), "the EP slices do not sum to the whole"


@pytest.mark.gpu
def test_expert_parallel_slice_nobody_chose_returns_zeros(_ext, kernel_on):
    H, E, K, I, T = 2048, 16, 2, 512, 8
    x, gamma, rw, rb, w_gu, w_dn = make_inputs("exact", T, H, E, I, K, El=4, seed=12)
    rb = torch.zeros(E, device="cuda")
    rb[12:] = -64.0                                        # experts 12..15 are never chosen
    inputs = (x, gamma, rw, rb, w_gu, w_dn)
    got = run_op(_ext, *inputs, 12, K)
    assert not ((got[2] >= 12).any())
    assert torch.equal(got[0], torch.zeros_like(got[0])), "a slice without chosen experts must return exact zeros"
    check(got, inputs, 12, K, "exact", what="EP slice nobody chose")


@pytest.mark.gpu
def test_tensor_parallel_intermediate_shards_sum_to_full_i(_ext, kernel_on):
    """Mixtral at TP=1 cut into 8 intermediate shards the way TP=8 stores them (gate and up halves each cut per shard): the
    summed partial outputs match the full-I float64 result within the sum of the shard bounds."""
    H, E, K, I, T, n = 4096, 8, 2, 14336, 2, 8
    x, gamma, rw, rb, w_gu, w_dn = make_inputs("exact", T, H, E, I, K, seed=13)
    ref = oracle(x, gamma, rw, rb, w_gu, w_dn, 0, K)[0]
    total, tb = torch.zeros_like(ref), torch.zeros_like(ref)
    s = I // n
    for r in range(n):
        gu_r = torch.cat([w_gu[:, :, r * s:(r + 1) * s], w_gu[:, :, I + r * s:I + (r + 1) * s]], -1).contiguous()
        dn_r = w_dn[:, r * s:(r + 1) * s].contiguous()
        sh = (x, gamma, rw, rb, gu_r, dn_r)
        got = run_op(_ext, *sh, 0, K)
        _, b = check(got, sh, 0, K, "exact", what=f"TP shard {r}")
        total += got[0].to(F64)
        tb += b
    assert ((total - ref).abs() <= tb).all(), f"TP shards: worst {(total - ref).abs().max().item():.3e}"


@pytest.mark.gpu
def test_refusals_fall_back_without_a_launch(_ext, kernel_on):
    """Shapes past the kernel's limits: the support predicate says no, the op returns the reference without a launch, the
    raw binding raises before launching.  An x that is a contiguous view at an 8-byte offset is refused the same way."""
    from neuronx_distributed_b200.ops import moe_tkg

    ext = _ext.ext()
    dev = "cuda"
    cases = {  # name: (T, H, E, I, K)
        "T=9": (9, 64, 8, 16, 2), "K=9": (2, 64, 16, 16, 9), "E=257": (2, 64, 257, 16, 2), "H%8": (2, 60, 8, 16, 2),
        "I%8": (2, 64, 8, 12, 2), "smem > 200 KiB": (8, 12808, 8, 8, 2),
    }
    for name, (T, H, E, I, K) in cases.items():
        assert not ext.moe_block_tkg_supported(T, H, E, I, K), name
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(T, H, device=dev, generator=g).to(BF16)
        rw = (torch.randn(E, H, device=dev, generator=g) * 0.1).to(BF16)
        w_gu = (torch.randn(2, H, 2 * I, device=dev, generator=g) * 0.1).to(BF16)
        w_dn = (torch.randn(2, I, H, device=dev, generator=g) * 0.1).to(BF16)
        _refused(_ext, moe_tkg, ext, (x, None, rw, None, w_gu, w_dn, 0, K), name)
    T, H, E, I, K = 2, 1024, 8, 256, 2
    x, _, rw, _, w_gu, w_dn = make_inputs("exact", T, H, E, I, K, seed=14)
    buf = torch.empty(T * H + 4, dtype=BF16, device=dev)
    xm = buf[4:].view(T, H)
    xm.copy_(x)
    assert xm.is_contiguous() and xm.data_ptr() % 16 == 8
    assert not moe_tkg.kernel_eligible(xm, rw, w_gu, w_dn, K)
    _refused(_ext, moe_tkg, ext, (xm, None, rw, None, w_gu, w_dn, 0, K), "x at an 8-byte offset", "16-byte aligned")


def _refused(_ext, moe_tkg, ext, args, name, msg=None):
    n = _ext.launches()
    got = moe_tkg.moe_block_tkg(*args)
    assert _ext.launches() == n, f"{name}: the op launched the kernel"
    want = moe_tkg.moe_block_tkg_reference(*args)
    for a, b in zip(got, want):
        assert torch.equal(a, b), name
    with pytest.raises(RuntimeError, match=msg):
        ext.moe_block_tkg(*args, 1e-6, 0, False, True, False, True, 0, 1.0, 0.0, -3e38, 3e38, -3e38, 3e38, True)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_graph_replays_and_repeated_calls(_ext, kernel_on):
    """One capture replayed with three different inputs copied into the static input: each replay against its own oracle
    (the barrier memset and the scratch zeroing run inside the graph).  Then eager again, twice: both within the bound.
    Two runs need not be bit-equal: the order of the red.add partial sums differs between runs."""
    from neuronx_distributed_b200.ops import moe_tkg

    H, E, K, I, T = 4096, 8, 2, 1792, 4
    x, gamma, rw, rb, w_gu, w_dn = make_inputs("exact", T, H, E, I, K, seed=20)
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        moe_tkg.moe_block_tkg(static_x, gamma, rw, rb, w_gu, w_dn, 0, K)        # warm-up outside the capture
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cap = moe_tkg.moe_block_tkg(static_x, gamma, rw, rb, w_gu, w_dn, 0, K)
    torch.cuda.current_stream().wait_stream(s)
    for seed in (21, 22, 23):
        xi = make_inputs("exact", T, H, E, I, K, seed=seed)[0]
        static_x.copy_(xi)
        graph.replay()
        torch.cuda.synchronize()
        check([c.clone() for c in cap], (xi, gamma, rw, rb, w_gu, w_dn), 0, K, "exact", what=f"graph replay seed={seed}")
    outs = []
    for _ in range(2):
        got = run_op(_ext, x, gamma, rw, rb, w_gu, w_dn, 0, K)
        _, bound = check(got, (x, gamma, rw, rb, w_gu, w_dn), 0, K, "exact", what="eager after graph")
        outs.append(got)
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1:], outs[1][1:])), "routing is not deterministic"
    assert ((outs[0][0].to(F64) - outs[1][0].to(F64)).abs() <= 2 * bound).all()


# ---- the module -----------------------------------------------------------------------------------------------------
def _one_rank_model_parallel():
    import torch.distributed as dist

    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29544")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    if not ps.model_parallel_is_initialized():
        ps.initialize_model_parallel(1)


MODULES = {  # name: (H, E, K, I, normalize, shared intermediate size or None)
    "mixtral-shaped": (2048, 8, 2, 1024, True, None),
    "qwen-shaped-shared": (1024, 60, 4, 256, False, 1408),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MODULES))
def test_moe_fused_tkg_module_takes_the_kernel(_ext, kernel_on, monkeypatch, name):
    """``MoEFusedTKG`` in bf16 on CUDA with the kernel switched on: the kernel path is taken (one op call per forward, no
    refusal reason), and its output agrees with the float64 oracle and with the flat path on the same device (same chosen
    experts; output within the sum of both bounds).  The flat path rounds every intermediate to bf16, so its bound is
    2^-6 (four bf16 unit roundoffs) of sum_slots |w| (sum_i (|a_i| + 1.2 |g_i u_i|) |W_dn[i,h]| + |y_slot,h|): gate|up,
    activation, down output and the weighted sum each rounded once, and weights normalised in bf16."""
    from neuronx_distributed_b200.modules.moe import ExpertMLPsV2, RoutedExpertsMLPOpsConfig, RouterTopK, SharedExperts
    from neuronx_distributed_b200.modules.moe.moe_fused_tkg import MoEFusedTKG
    from neuronx_distributed_b200.modules.rms_norm import RMSNorm
    from neuronx_distributed_b200.ops import moe_tkg

    _one_rank_model_parallel()
    H, E, K, I, normalize, shared_i = MODULES[name]
    torch.manual_seed(5)
    cfg = RoutedExpertsMLPOpsConfig(num_experts=E, top_k=K, hidden_size=H, intermediate_size=I, hidden_act="silu", glu_mlp=True,
                                    capacity_factor=None, normalize_top_k_affinities=normalize)
    router = RouterTopK(E, K, H, dtype=BF16, bias=True).cuda()
    experts_mod = ExpertMLPsV2(cfg, dtype=BF16).cuda()
    norm = RMSNorm(H, eps=1e-5).to(device="cuda", dtype=BF16)
    shared = SharedExperts(H, shared_i, dtype=BF16).cuda() if shared_i else None
    x_in, gamma, rw, rb, w_gu, w_dn = make_inputs("margin", 4, H, E, I, K, seed=30)
    op = experts_mod.mlp_op
    with torch.no_grad():
        router.linear_router.weight.copy_(rw)
        router.linear_router.bias.copy_(rb.to(BF16))
        norm.weight.copy_(gamma)
        op.gate_up_proj.weight.copy_(w_gu)
        op.down_proj.weight.copy_(w_dn)
    fused = MoEFusedTKG(router, experts_mod, shared, norm, return_router_logits=True, return_expert_index=True).eval()
    x = x_in.view(4, 1, H)
    calls = []
    real = moe_tkg.moe_block_tkg

    def spy(*a, **k):
        r = real(*a, **k)
        calls.append(r)
        return r

    monkeypatch.setattr(moe_tkg, "moe_block_tkg", spy)
    with torch.no_grad():
        assert fused._can_use_kernel(x), fused._why_not
        y, logits, idx = fused(x)
        assert fused._why_not is None and len(calls) == 1, (fused._why_not, len(calls))
        y2 = fused(x)[0]
        assert len(calls) == 2
        sh = shared(norm(x)).to(F64).view(4, H) if shared is not None else 0.0
        monkeypatch.setenv("NXD_MOE_TKG_KERNEL", "0")
        yf, _, idx_f = fused(x)
        assert len(calls) == 2 and fused._why_not is not None                    # the flat path: no call of the op
    torch.cuda.synchronize()
    out, k_logits, k_idx, k_w = calls[0]
    assert torch.equal(k_idx, idx) and torch.equal(k_logits, logits.float())
    # the routed part against the oracle (margin mode), then the shared experts added in bf16
    _, bound = check((out, k_logits, k_idx, k_w), (x_in, gamma, rw, rb.to(BF16).float(), w_gu, w_dn), 0, K, "margin",
                     what=name, normalize=normalize)
    xn, z = normed(x_in, gamma, 1e-5)
    ref, parts = experts(xn, k_idx, k_w.to(F64), w_gu, w_dn, 0, xerr=input_ulps(z, H), exact_gu=False)
    total = ref + sh
    b_kernel = bound + ulp_bf16(total)
    for got in (y, y2):
        assert ((got.view(4, H).to(F64) - total).abs() <= b_kernel).all(), f"{name}: module output outside the bound"
    # the flat path: same chosen experts, output within its own bound of the oracle
    assert torch.equal(idx_f.view(4, K).sort(-1).values, k_idx.sort(-1).values), (idx_f, k_idx)
    Wd_abs_y = torch.zeros_like(ref)
    for t in range(4):
        for s in range(K):
            y1, _ = experts(xn[t:t + 1], k_idx[t:t + 1, s:s + 1], k_w[t:t + 1, s:s + 1].to(F64), w_gu, w_dn, 0)
            Wd_abs_y[t] += y1[0].abs()
    b_flat = ulp_bf16(total) + 2.0 ** -6 * (parts["A"] + 1.2 * parts["B"] + Wd_abs_y) + parts["D"]
    yf64 = yf.view(4, H).to(F64)
    assert ((yf64 - total).abs() <= b_flat).all(), f"{name}: flat path outside its bound"
    assert ((y.view(4, H).to(F64) - yf64).abs() <= b_kernel + b_flat).all()
