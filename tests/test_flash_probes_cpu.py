"""Pair-by-pair probes of the flash attention training kernels, and their checks off the GPU.

The kernels (``csrc/attention_sm90.cu``: ``fa_fwd_kernel``, ``fa_bwd_prep_kernel``, ``fa_bwd_dkdv_kernel``,
``fa_bwd_dq_kernel``) cut the queries and keys into 64-row tiles, run two 64-row warpgroups per 128-row CTA and visit the
union of the tile ranges of the CTA's two halves.  A pair lost, counted twice or moved to its neighbour moves a row by
about 1/n of it, far inside a tolerance relative to max|ref|.  The probes here make every such error exact and large:

A. visibility: with q = 0 (or K = 0) every visible score is exactly 0, ex2.approx(0) = 1 and every rescale is ×1 or ×0,
   so the forward's row sum is the number of visible keys and a one-hot V band names each key; the backward kernels take
   O and LSE as arguments, so O = 0, LSE = 0 and scale = 1 make every visible P = 1 and dS = dP − δ an integer.  Every
   (query, key) pair of the case is observed, exactly, in the forward, the dK/dV kernel and the dQ kernel.
B. planted key: one visible key per row scores ≥ 40 log2-units above every other key the row sees, so O must equal its V
   row bit for bit and the LSE its score.  The planted keys are the rows' first and last visible keys and tile edges.
C. random inputs against float64 with a per-element bound derived from the kernels' arithmetic, which also asserts that
   removing one edge pair from the reference moves some element of O, dQ, dK and dV by at least 10× its bound.

The probes take the kernels as a ``Kernels(fwd, bwd)`` pair of callables, so the same checks run on the CUDA kernels
(``test_flash_probes_gpu.py``), on the float64 simulation here, and on simulated kernels with one deliberate fault each,
which the probes must reject.  Which pairs are visible comes from ``Case.visible``, the rule written at the top of
``attention_sm90.cu``; which tiles a CTA visits from ``key_tiles`` / ``query_tiles`` below, a transcription of the kernels'.
"""
import math
from dataclasses import dataclass
from typing import Callable, NamedTuple, Optional

import numpy as np
import pytest
import torch

from neuronx_distributed_b200.ops import attention

F64 = torch.float64
U = 2.0 ** -24                     # fp32 unit roundoff
BF = 2.0 ** -8                     # bf16 unit roundoff (8 significant bits)
EX2 = 2.0 ** -22                   # exp2f / ex2.approx.ftz.f32 under --use_fast_math: at most 2 fp32 ulp
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
BT = 64                            # rows of a query or key tile; a CTA holds two (one per warpgroup)


# ---- the kernels' tile ranges (attention_sm90.cu key_tiles / query_tiles) -----------------------------------------------
def key_tiles(S_kv: int, causal: bool, window: int, off: int, q0: int):
    """Key tiles [lo, hi) of the 64-row query half starting at q0 (``window`` 0: no window, off must then be 0)."""
    n = (S_kv + BT - 1) // BT
    lo = max(0, q0 + off - window + 1) // BT if window else 0
    hi = min(n, (q0 + BT - 1 + off) // BT + 1) if causal else n
    return lo, hi


def query_tiles(S_q: int, causal: bool, window: int, off: int, k0: int):
    """Query tiles [lo, hi) of the 64-row key half starting at k0."""
    n = (S_q + BT - 1) // BT
    lo = max(0, k0 - off) // BT if causal else 0
    hi = min(n, (k0 + 2 * BT - 2 + window - off) // BT) if window else n
    return lo, hi


def cta_key_range(S_kv, causal, window, off, c, first_half_hi=False):
    """Key tiles the forward / dQ CTA c visits: from its first half's lo to its second half's hi (the union of the two
    monotone ranges).  ``first_half_hi``: a faulty kernel that stops at the first half's hi."""
    lo, hi0 = key_tiles(S_kv, causal, window, off, 2 * BT * c)
    _, hi1 = key_tiles(S_kv, causal, window, off, 2 * BT * c + BT)
    return lo, (hi0 if first_half_hi else hi1)


def cta_query_range(S_q, causal, window, off, c, second_half_lo=False):
    """Query tiles the dK/dV CTA c visits (per query head of its group).  ``second_half_lo``: a faulty kernel that starts
    at the second half's lo."""
    lo0, _ = query_tiles(S_q, causal, window, off, 2 * BT * c)
    lo1, hi = query_tiles(S_q, causal, window, off, 2 * BT * c + BT)
    return (lo1 if second_half_lo else lo0), hi


# ---- cases ----------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    """One launch shape.  The mask (uint8 [B, S_kv]) is built from ``lens`` (right padding: key j < lens[b]), ``left``
    (left padding: key j ≥ left[b]) or ``rand`` (each key kept with that probability); none of them: no mask."""
    name: str
    B: int
    S_q: int
    S_kv: int
    H: int
    Hkv: int
    D: int
    causal: bool = False
    window: int = 0
    q_offset: int = 0
    lens: Optional[tuple] = None
    left: Optional[tuple] = None
    rand: float = 0.0
    dropout: float = 0.0
    layout: str = "bshd"                           # bshd, sbhd or fused (slices of one QKV projection output)
    sbhd_out: bool = False
    head_offset: int = 0
    seed: int = 0x5EED_1234_5678

    @property
    def G(self):
        return self.H // self.Hkv

    @property
    def scale(self):
        return 1.0 / math.sqrt(self.D)

    @property
    def masked(self):
        return self.lens is not None or self.left is not None or self.rand > 0

    @property
    def rscale(self):
        return 1.0 / (1.0 - self.dropout) if self.dropout else 1.0

    def instantiation(self):
        """(HD, MASK, WINDOW, DROPOUT) of the kernels this case launches."""
        return self.D, self.masked, self.window > 0, self.dropout > 0

    def mask(self, device) -> Optional[torch.Tensor]:
        if not self.masked:
            return None
        j = torch.arange(self.S_kv, device=device)[None, :]
        m = torch.ones(self.B, self.S_kv, dtype=torch.bool, device=device)
        if self.lens is not None:
            m &= j < torch.tensor(self.lens, device=device)[:, None]
        if self.left is not None:
            m &= j >= torch.tensor(self.left, device=device)[:, None]
        if self.rand:
            g = torch.Generator().manual_seed(len(self.name) * 7919 + self.S_kv)
            m &= (torch.rand(self.B, self.S_kv, generator=g) < self.rand).to(device)
        return m.to(torch.uint8)

    def visible(self, i, j, b, mask) -> torch.Tensor:
        """The kernels' rule for broadcastable integer tensors (query row i, key j, batch b): i < S_q, 0 ≤ j < S_kv,
        mask[b, j], j ≤ i + off when causal, j > i + off − W when windowed."""
        off = self.q_offset
        v = (i >= 0) & (i < self.S_q) & (j >= 0) & (j < self.S_kv)
        if self.causal:
            v = v & (j <= i + off)
        if self.window:
            v = v & (j > i + off - self.window)
        if mask is not None:
            v = v & (mask.bool()[b, j.clamp(0, self.S_kv - 1)])
        return v

    def keep(self, device) -> Optional[torch.Tensor]:
        """[B, H, S_q, S_kv] bool of ``attention_dropout_keep`` (None without dropout)."""
        if not self.dropout:
            return None
        key = (self.seed, self.B, self.H, self.S_q, self.S_kv, self.dropout, self.head_offset, str(device))
        if key not in _KEEP:
            _KEEP[key] = attention.attention_dropout_keep(self.seed, self.B, self.H, self.S_q, self.S_kv, self.dropout,
                                                          self.head_offset).to(device)
        return _KEEP[key]


_KEEP = {}                         # keep masks by their arguments (the host rule is slow at large shapes)


# A fwd callable is ``fwd(case, q, k, v, mask, scale) → (o [B,S_q,H,D] bf16, lse [B,H,S_q] fp32)``; a bwd callable is
# ``bwd(case, go, q, k, v, o, lse, dlse, mask, scale) → (dq, dk, dv)`` in bf16.  Tensors are logical [B, S, H, D].
class Kernels(NamedTuple):
    fwd: Callable
    bwd: Callable


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(shape, seed, device):
    return torch.randn(*shape, generator=_gen(seed)).to(device)


def _bands(S: int):
    """Band starts a = 64t − 32 for t = 0 … ⌈S/64⌉: 64-row bands that straddle every tile boundary and together hold
    every row 0 … S − 1."""
    return [BT * t - BT // 2 for t in range((S + BT - 1) // BT + 1)]


def band_launches(case: Case, S: int):
    """[n_bands][B·Hkv] band starts: slice s (batch b, kv head h, s = b·Hkv + h) of launch t takes band (t + 7s) mod
    n_bands, so every slice observes every band over the launches, and neighbouring slices observe different bands in
    the same launch (a kernel reading the wrong batch or head shows)."""
    bands = _bands(S)
    n = case.B * case.Hkv
    return [[bands[(t + 7 * s) % len(bands)] for s in range(n)] for t in range(len(bands))]


def _band_index(starts, device):
    """[B, Hkv, 64] row indices a + d of the bands of one launch."""
    return torch.tensor(starts, device=device).view(-1, 1) + torch.arange(BT, device=device)


def _one_hot_band(case: Case, rows: int, idx: torch.Tensor, heads: int, value: torch.Tensor, device):
    """[B, rows, heads, D] with x[b, a + d, h, d] = value[h] for the band a of slice (b, h // (heads / Hkv)), 0 elsewhere."""
    B, D = case.B, case.D
    x = torch.zeros(B, rows, heads, D, dtype=F64, device=device)
    per = heads // case.Hkv
    idx = idx.view(B, case.Hkv, BT)
    for h in range(heads):
        r = idx[:, h // per]                                                        # [B, 64]
        ok = (r >= 0) & (r < rows)
        bb = torch.arange(B, device=device)[:, None].expand_as(r)[ok]
        dd = torch.arange(BT, device=device)[None, :].expand_as(r)[ok]
        x[bb, r[ok], h, dd] = float(value[h])
    return x.to(torch.bfloat16)


def _want(case: Case, i, j, mask, keep) -> torch.Tensor:
    """[B, H, ...] visibility ∧ keep of the pairs (i, j) given as [B, Hkv, ...] index tensors (GQA heads share them)."""
    B, H, G = case.B, case.H, case.G
    i, j = i.repeat_interleave(G, 1), j.repeat_interleave(G, 1)
    b = torch.arange(B, device=i.device).view(B, 1, *([1] * (i.dim() - 2)))
    v = case.visible(i, j, b, mask)
    if keep is not None:
        hh = torch.arange(H, device=i.device).view(1, H, *([1] * (i.dim() - 2)))
        v = v & keep[b, hh, i.clamp(0, case.S_q - 1), j.clamp(0, case.S_kv - 1)]
    return v


# ---- A. visibility probes -------------------------------------------------------------------------------------------------
def check_fwd_visibility(case: Case, k: Kernels, device) -> int:
    """Probe A on the forward.  q = 0: every visible score is 0 and exp2(0 − 0) = 1, every running rescale exp2(0) = 1 (or
    exp2(−inf) = 0 before the row's first visible key), so the fp32 row sum l_i counts the visible keys n_i exactly
    (integers < 2²⁴); dropout zeroes entries of P only after l is summed, so n_i is unchanged.  LSE_i = ln n_i up to
    __log2f (2 ulp of log2 n ≤ 13, i.e. ≤ 2⁻¹⁹) and the approximate division by log2 e (2 ulp): exp(LSE)·(1 ± 3·10⁻⁶)
    = n_i ≤ 8192 rounds to n_i.  V is one-hot over a band of 64 keys, V[a + d, d] = 1, so the fp32 numerator of column d
    is keep·[a + d visible] ∈ {0, 1} exactly (P = 1 is exact in bf16), and O = r·num / n_i (r = 1/(1 − p)) with the
    approximate reciprocal (2 ulp) and the bf16 rounding (2⁻⁸): O·n_i / r = num·(1 ± 2⁻⁷) rounds to num.  Columns ≥ 64
    and rows that see nothing must be exactly 0.  Returns the number of forward launches."""
    mask = case.mask(device)
    keep = case.keep(device)
    q = torch.zeros(case.B, case.S_q, case.H, case.D, dtype=torch.bfloat16, device=device)
    kk = _randn((case.B, case.S_kv, case.Hkv, case.D), 11, device).to(torch.bfloat16)
    i_all = torch.arange(case.S_q, device=device)
    n = case.visible(i_all.view(1, -1, 1), torch.arange(case.S_kv, device=device).view(1, 1, -1),
                     torch.arange(case.B, device=device).view(-1, 1, 1), mask).sum(-1)           # [B, S_q]
    launches = band_launches(case, case.S_kv)
    for t, starts in enumerate(launches):
        idx = _band_index(starts, device)                                           # [B·Hkv, 64]
        v = _one_hot_band(case, case.S_kv, idx, case.Hkv, torch.ones(case.Hkv), device)
        o, lse = k.fwd(case, q, kk, v, mask, case.scale)
        assert o.dtype == torch.bfloat16 and lse.dtype == torch.float32
        jj = idx.view(case.B, case.Hkv, 1, BT)
        ii = i_all.view(1, 1, -1, 1).expand(case.B, case.Hkv, -1, 1)
        want = _want(case, ii, jj, mask, keep)                                      # [B, H, S_q, 64]
        if t == 0:
            fin = torch.isfinite(lse)
            want_fin = (n > 0)[:, None, :].expand_as(lse)
            assert torch.equal(fin, want_fin), f"{case.name}: LSE finite where {(fin != want_fin).nonzero()[:4].tolist()}"
            cnt = torch.where(fin, torch.round(torch.exp(lse.to(F64))), torch.zeros((), dtype=F64, device=device))
            nn = n[:, None, :].expand_as(cnt).to(F64)
            assert torch.equal(cnt, nn), (f"{case.name}: exp(LSE) ≠ visible count at (b, h, i) "
                                          f"{(cnt != nn).nonzero()[:4].tolist()}")
        ob = o.permute(0, 2, 1, 3).to(F64)                                          # [B, H, S_q, D]
        nz = n[:, None, :, None].to(F64)
        got = torch.round(ob[..., :BT] * nz / case.rscale)
        empty = (n == 0)[:, None, :].expand(case.B, case.H, case.S_q)
        assert not ob[empty].any(), f"{case.name}: a row that sees no key is not 0"
        assert not ob[..., BT:].any(), f"{case.name}: columns past the one-hot band are not 0"
        exp = want.to(F64).masked_fill(empty[..., None], 0)
        bad = got != exp
        assert not bad.any(), (f"{case.name} fwd launch {t}: {int(bad.sum())} pairs wrong; first (b, h, i, d) "
                               f"{bad.nonzero()[0].tolist()}")
    return len(launches)


def check_bwd_visibility(case: Case, k: Kernels, device) -> int:
    """Probe A on the dK/dV and dQ kernels, with O = 0, LSE = 0, dlse = None and scale = 1 passed to the backward: δ = 0,
    and with one of q, K zero every score is 0 and every visible P = exp2(0 − 0) = 1 exactly.
    - dK/dV launch: K = 0, V = 1, q[a + d, h, d] = 1 and dO[a + d, h, d] = 2^g for head g of each group, over a band of 64
      query rows.  dP[i, j] = Σ_d dO[i, d] = 2^g on band rows (0 elsewhere), dS = P∘(dP∘Z·r − δ) = 2^g·r on kept visible
      pairs, so dV[j, d] = dK[j, d] = r·Σ_g 2^g·[a + d sees j, kept] — integers ≤ 2·255, each a sum of exact fp32 terms,
      even when above 256, hence exact in bf16; the head bits say which head of the group contributed.  dQ = dS·K = 0.
    - dQ launch: q = 0, V = 1, dO = e₀ (dP = 1), K[a + d, d] = 1 over a band of 64 keys: dQ[i, d] = r·[i sees a + d, kept]
      ∈ {0, 1, 2}; dK = dSᵀ·q = 0.
    Returns the number of backward launches."""
    mask = case.mask(device)
    keep = case.keep(device)
    B, H, G, D = case.B, case.H, case.G, case.D
    zo = torch.zeros(B, case.S_q, H, D, dtype=torch.bfloat16, device=device)
    lse0 = torch.zeros(B, H, case.S_q, dtype=torch.float32, device=device)
    ones_kv = torch.ones(B, case.S_kv, case.Hkv, D, dtype=torch.bfloat16, device=device)
    zeros_kv = torch.zeros_like(ones_kv)
    r = case.rscale
    pow2 = torch.tensor([2.0 ** (h % G) for h in range(H)], dtype=F64)
    j_all = torch.arange(case.S_kv, device=device)
    i_all = torch.arange(case.S_q, device=device)
    n = 0
    for t, starts in enumerate(band_launches(case, case.S_q)):
        idx = _band_index(starts, device)
        q = _one_hot_band(case, case.S_q, idx, H, torch.ones(H), device)
        go = _one_hot_band(case, case.S_q, idx, H, pow2, device)
        dq, dk, dv = k.bwd(case, go, q, zeros_kv, ones_kv, zo, lse0, None, mask, 1.0)
        n += 1
        ii = idx.view(B, case.Hkv, BT, 1)
        want = _want(case, ii, j_all.view(1, 1, 1, -1).expand(B, case.Hkv, 1, -1), mask, keep)   # [B, H, 64, S_kv]
        exp = (want.to(F64) * pow2.to(device).view(1, H, 1, 1)).view(B, case.Hkv, G, BT, -1).sum(2) * r
        exp = exp.permute(0, 3, 1, 2)                                               # [B, S_kv, Hkv, 64]
        assert not dq.to(F64).any(), f"{case.name}: dQ ≠ 0 with K = 0"
        for name, x in (("dV", dv), ("dK", dk)):
            got = x.to(F64)
            assert not got[..., BT:].any(), f"{case.name}: {name} columns past the band are not 0"
            bad = got[..., :BT] != exp
            assert not bad.any(), (f"{case.name} {name} launch {t}: {int(bad.sum())} wrong; first (b, j, hk, d) "
                                   f"{bad.nonzero()[0].tolist()}")
    e0 = torch.zeros(B, case.S_q, H, D, dtype=torch.bfloat16, device=device)
    e0[..., 0] = 1
    zq = torch.zeros(B, case.S_q, H, D, dtype=torch.bfloat16, device=device)
    for t, starts in enumerate(band_launches(case, case.S_kv)):
        idx = _band_index(starts, device)
        kk = _one_hot_band(case, case.S_kv, idx, case.Hkv, torch.ones(case.Hkv), device)
        dq, dk, dv = k.bwd(case, e0, zq, kk, ones_kv, zo, lse0, None, mask, 1.0)
        n += 1
        jj = idx.view(B, case.Hkv, 1, BT)
        want = _want(case, i_all.view(1, 1, -1, 1).expand(B, case.Hkv, -1, 1), jj, mask, keep)    # [B, H, S_q, 64]
        exp = want.to(F64).permute(0, 2, 1, 3) * r                                  # [B, S_q, H, 64]
        got = dq.to(F64)
        assert not dk.to(F64).any(), f"{case.name}: dK ≠ 0 with q = 0"
        assert not got[..., BT:].any(), f"{case.name}: dQ columns past the band are not 0"
        bad = got[..., :BT] != exp
        assert not bad.any(), (f"{case.name} dQ launch {t}: {int(bad.sum())} wrong; first (b, i, h, d) "
                               f"{bad.nonzero()[0].tolist()}")
    return n


def check_dlse(case: Case, k: Kernels, device) -> None:
    """The dS = P∘(dP − δ) plumbing with δ = −dlse: O = 0 and dO = 0 make δ_i = −dlse_i and dP = 0, so dS = P·dlse on
    visible pairs whatever dropout keeps.  LSE = 0 on rows that see a key (P = 1) and −inf on rows that see none, which
    must contribute nothing and give no NaN.  dlse_i = 2^g for head g of a group on the dK launch (K = 0, q one-hot over a
    band of rows: dK[j, d] = Σ_g 2^g·[a + d sees j] ≤ 255, exact) and dlse_i = 1 + (i mod 3) on the dQ launch (q = 0, K
    one-hot over a band of keys: dQ[i, d] = dlse_i·[i sees a + d] ≤ 3).  dV = Σ P·dO = 0."""
    mask = case.mask(device)
    B, H, G, D = case.B, case.H, case.G, case.D
    i_all = torch.arange(case.S_q, device=device)
    j_all = torch.arange(case.S_kv, device=device)
    n = case.visible(i_all.view(1, -1, 1), j_all.view(1, 1, -1), torch.arange(B, device=device).view(-1, 1, 1),
                     mask).sum(-1)                                                  # [B, S_q]
    lse = torch.where(n > 0, 0.0, -math.inf)[:, None, :].expand(B, H, case.S_q).float().contiguous()
    zo = torch.zeros(B, case.S_q, H, D, dtype=torch.bfloat16, device=device)
    ones_kv = torch.ones(B, case.S_kv, case.Hkv, D, dtype=torch.bfloat16, device=device)
    pow2 = torch.tensor([2.0 ** (h % G) for h in range(H)], dtype=torch.float32, device=device)
    starts = band_launches(case, case.S_q)[0]
    idx = _band_index(starts, device)
    q = _one_hot_band(case, case.S_q, idx, H, torch.ones(H), device)
    dlse = pow2.view(1, H, 1).expand(B, H, case.S_q).contiguous()
    dq, dk, dv = k.bwd(case, zo, q, torch.zeros_like(ones_kv), ones_kv, zo, lse, dlse, mask, 1.0)
    for x in (dq, dk, dv):
        assert not torch.isnan(x).any(), f"{case.name}: NaN from the dLSE probe"
    want = _want(case, idx.view(B, case.Hkv, BT, 1), j_all.view(1, 1, 1, -1).expand(B, case.Hkv, 1, -1), mask, None)
    exp = (want.to(F64) * pow2.to(F64).view(1, H, 1, 1)).view(B, case.Hkv, G, BT, -1).sum(2).permute(0, 3, 1, 2)
    assert torch.equal(dk.to(F64)[..., :BT], exp), f"{case.name}: dK of the dLSE probe"
    assert not dv.to(F64).any() and not dq.to(F64).any(), f"{case.name}: dV or dQ ≠ 0 in the dLSE probe"
    starts = band_launches(case, case.S_kv)[0]
    idx = _band_index(starts, device)
    kk = _one_hot_band(case, case.S_kv, idx, case.Hkv, torch.ones(case.Hkv), device)
    dl = (1.0 + (i_all % 3)).float().view(1, 1, -1).expand(B, H, case.S_q).contiguous()
    dq, dk, dv = k.bwd(case, zo, zo, kk, ones_kv, zo, lse, dl, mask, 1.0)
    for x in (dq, dk, dv):
        assert not torch.isnan(x).any(), f"{case.name}: NaN from the dLSE probe"
    want = _want(case, i_all.view(1, 1, -1, 1).expand(B, case.Hkv, -1, 1), idx.view(B, case.Hkv, 1, BT), mask, None)
    exp = (want.to(F64) * dl.to(F64)[..., None]).permute(0, 2, 1, 3)
    assert torch.equal(dq.to(F64)[..., :BT], exp), f"{case.name}: dQ of the dLSE probe"
    assert not dk.to(F64).any(), f"{case.name}: dK ≠ 0 with q = 0 in the dLSE probe"


# ---- B. planted keys ------------------------------------------------------------------------------------------------------
QA = 32.0                          # the planted row's q entries; K entries are 0 / 1
N_CODES = 21 ** 3                  # one hot dimension in each of three groups of 21: 9261 ≥ 8192 distinct key codes


def key_codes(case: Case, device) -> torch.Tensor:
    """[B, S_kv, Hkv, 3] the hot dimensions of each key: code c = (j + 1009·(b·Hkv + h)) mod 9261, distinct over the keys of
    one (batch, kv head) slice and different between slices, so a key read from the wrong slice scores low."""
    j = torch.arange(case.S_kv, device=device).view(1, -1, 1)
    s = torch.arange(case.B * case.Hkv, device=device).view(case.B, 1, case.Hkv)
    c = (j + 1009 * s) % N_CODES
    return torch.stack((c % 21, 21 + (c // 21) % 21, 42 + c // 441), -1)


PLANT_ROUNDS = 4


def plant_targets(case: Case, mask, device, rnd: int) -> torch.Tensor:
    """[B, H, S_q] the planted key of each row in round ``rnd`` (−1: the row sees nothing): round 0 the row's first visible
    key (window start, first key after a masked run, key 0), round 1 its last (diagonal, S_kv − 1, last unmasked key),
    rounds 2 and 3 the first / last key of one of the key tiles the row sees, rotating with the row and head (snapped to
    the next visible key when masked).  Early and late keys of a row's tile sequence both occur."""
    B, H = case.B, case.H
    i = torch.arange(case.S_q, device=device)
    off = case.q_offset
    lo = torch.zeros_like(i)
    hi = torch.full_like(i, case.S_kv - 1)
    if case.causal:
        hi = torch.minimum(hi, i + off)
    if case.window:
        lo = torch.maximum(lo, i + off - case.window + 1)
    m = (mask.bool() if mask is not None else torch.ones(B, case.S_kv, dtype=torch.bool, device=device))
    j = torch.arange(case.S_kv, device=device)
    big = case.S_kv
    # next visible key ≥ j and last visible key ≤ j of every batch
    nxt = torch.where(m, j, big).flip(-1).cummin(-1).values.flip(-1)
    prv = torch.where(m, j, -1).cummax(-1).values
    lo_c, hi_c = lo.clamp(0, case.S_kv - 1), hi.clamp(0, case.S_kv - 1)
    first = nxt[:, lo_c]                                                            # [B, S_q]
    last = prv[:, hi_c]
    ok = (lo <= hi)[None] & (first <= hi[None]) & (last >= lo[None])
    hh = torch.arange(H, device=device).view(1, H, 1)
    if rnd == 0:
        t = first[:, None].expand(B, H, -1)
    elif rnd == 1:
        t = last[:, None].expand(B, H, -1)
    else:
        t_lo, t_hi = lo_c // BT, hi_c // BT
        nt = (t_hi - t_lo + 1).clamp_min(1)
        tile = t_lo[None, None] + (i[None, None] * 7 + hh * 3 + rnd) % nt[None, None]
        e = tile * BT + (0 if rnd == 2 else BT - 1)
        e = torch.maximum(torch.minimum(e, hi_c[None, None]), lo_c[None, None])
        t = torch.gather(nxt[:, None].expand(B, H, -1), 2, e.expand(B, H, -1).contiguous())
        t = torch.where(t <= hi[None, None], t, last[:, None])
    return torch.where(ok[:, None], t, torch.full_like(t, -1))


def check_planted(case: Case, k: Kernels, device) -> int:
    """Probe B.  K holds one 1 in each of three groups of 21 dimensions (``key_codes``); the q row of (b, h, i) is
    QA·code(j*) for its planted key j*, so the planted score is 3·QA = 96 and any other key (which shares at most two hot
    dimensions) scores ≤ 2·QA: with scale = 1 a lead of QA·log2 e ≈ 46 ≥ 40 log2-units, and every score is a small
    integer, exact in bf16 and fp32.  Every other visible key then carries weight < 2⁻⁴⁶ relative to j*, all of them
    together < 8192·2⁻⁴⁶ = 2⁻³³, wherever j* falls in the row's tile sequence (a late j* rescales what came before by
    alpha ≤ 2⁻⁴⁶): P(j*) = exp2(0) = 1 is exact in bf16, l = 1 in fp32, and O = V[j*]·(1 + ε), |ε| < 2⁻³² plus the
    approximate reciprocal (2 ulp), rounds back to V[j*] in bf16 — bit for bit (V uniform in [1, 2) on the bf16 grid).  The
    LSE is (fp32(96·log2 e) + log2 1) / log2 e: 96 up to the product's rounding and the approximate division, 4 ulp.
    Rows that see nothing: O = 0, LSE = −inf.  Returns the number of forward launches."""
    assert QA * LOG2E >= 40
    mask = case.mask(device)
    B, H, G, D = case.B, case.H, case.G, case.D
    assert D >= 63 and case.S_kv <= N_CODES
    codes = key_codes(case, device)
    kk = torch.zeros(B, case.S_kv, case.Hkv, D, dtype=F64, device=device)
    kk.scatter_(3, codes, 1.0)
    kk = kk.to(torch.bfloat16)
    for rnd in range(PLANT_ROUNDS):
        v = (1 + torch.rand(B, case.S_kv, case.Hkv, D, generator=_gen(100 + rnd))).to(device).to(torch.bfloat16)
        tgt = plant_targets(case, mask, device, rnd)                                # [B, H, S_q]
        seen = tgt >= 0
        tj = tgt.clamp_min(0)
        hk = torch.arange(H, device=device).view(1, H, 1) // G
        bb = torch.arange(B, device=device).view(B, 1, 1)
        ii = torch.arange(case.S_q, device=device).view(1, 1, -1)
        assert case.visible(ii, tj, bb, mask)[seen].all()
        c = codes[bb, tj, hk]                                                       # [B, H, S_q, 3]
        q = torch.zeros(B, H, case.S_q, D, dtype=F64, device=device)
        q.scatter_(3, c, QA)
        q = (q * seen[..., None]).permute(0, 2, 1, 3).to(torch.bfloat16)
        o, lse = k.fwd(case, q, kk, v, mask, 1.0)
        want = v[bb, tj, hk].to(F64)                                                # [B, H, S_q, D]
        got = o.permute(0, 2, 1, 3).to(F64)
        bad = seen & (got != want).any(-1)
        assert not bad.any(), (f"{case.name} round {rnd}: {int(bad.sum())} planted rows wrong; first (b, h, i) "
                               f"{bad.nonzero()[0].tolist()} j* = {tgt[bad][0].item()}")
        assert not got[~seen].any(), f"{case.name}: a row that sees nothing is not 0"
        lse64 = lse.to(F64)
        assert bool((lse64[~seen] == -math.inf).all()), f"{case.name}: LSE of an empty row"
        err = (lse64[seen] - 3 * QA).abs()
        assert err.numel() == 0 or err.max().item() <= 4 * 2.0 ** -17, f"{case.name}: planted LSE off by {err.max().item()}"
    return PLANT_ROUNDS


# ---- C. random inputs against float64 -------------------------------------------------------------------------------------
def c_dot(D: int) -> float:
    """Error factor of an fp32 wgmma dot product of length D, in units of u·Σ|aᵢbᵢ|: the bf16 products are exact in fp32,
    and each of the D/16 k-steps adds 16 of them into the accumulator.  Hopper's fp32 tensor-core accumulation is not
    documented as round-to-nearest, so every add is taken to err by a truncation (2u relative to the partial sum, itself
    ≤ Σ|aᵢbᵢ|), and a product passes through at most 15 adds inside its k-step plus D/16 accumulator adds."""
    return 2.0 * (16 + D // 16)


def boost_pair(case: Case, mask, device):
    """(i*, j*): an edge pair each (b, kv head) boosts in head 0 of its group — row 63 (the last row of a CTA's first
    warpgroup) or the first row with a visible key, and its last visible key (its diagonal when causal)."""
    out = []
    m = mask.bool() if mask is not None else None
    for b in range(case.B):
        for i in [63, 64, 127, 0, case.S_q - 1] + list(range(case.S_q)):
            if not 0 <= i < case.S_q:
                continue
            jj = torch.arange(case.S_kv, device=device)
            vis = case.visible(torch.tensor(i, device=device), jj, torch.tensor(b, device=device), m)
            if vis.any():
                out.append((b, i, int(vis.nonzero()[-1, 0])))
                break
    return out


def random_inputs(case: Case, device, seed=3):
    """bf16 q, k, v, dO ~ N(0, 1), and per (b, kv head) one boosted edge pair: k[j*] along q[i*] of head 0 of the group so
    that its score is ln n nats (half the row's weight, where |dS| = P·|dP − δ| peaks), and dO[i*] = 2·v[j*] so that dP of
    the pair stands out: the float64 reference notices in O, dQ, dK and dV when the pair is lost."""
    B, H, G, D = case.B, case.H, case.G, case.D
    q = _randn((B, case.S_q, H, D), seed, device).to(torch.bfloat16)
    kx = _randn((B, case.S_kv, case.Hkv, D), seed + 1, device)
    v = _randn((B, case.S_kv, case.Hkv, D), seed + 2, device).to(torch.bfloat16)
    go = _randn((B, case.S_q, H, D), seed + 3, device).to(torch.bfloat16)
    mask = case.mask(device)
    pairs = boost_pair(case, mask, device)
    for b, i, j in pairs:
        n = int(case.visible(torch.tensor(i, device=device), torch.arange(case.S_kv, device=device),
                             torch.tensor(b, device=device), mask).sum())
        qh = q[b, i, ::G].float()                                                   # [Hkv, D]
        kx[b, j] = qh * (math.log(n) / (case.scale * qh.pow(2).sum(-1, keepdim=True)))
        go[b, i, ::G] = 2 * v[b, j]
    return q, kx.to(torch.bfloat16), v, go, pairs


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().to(F64).clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def ulp32(x: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(x.abs().to(F64).clamp_min(2.0 ** -126)))
    return torch.exp2(e - 23)


def reference(case: Case, q, k, v, go, mask, o_in=None, lse_in=None, drop=()):
    """float64 (O, LSE) and, given the bf16 O and fp32 LSE handed to the backward, (dQ, dK, dV), each with a per-element
    bound on the kernels' error, computed one (batch, head) slice at a time.  ``drop``: (b, h, i, j) pairs removed from the
    visibility (the sensitivity check).  Returns a dict name → (ref, tol), tensors in the outputs' [B, S, H, D] / [B, H, S]
    layouts.

    Forward, per row (x = s·scale·log2 e in log2 units):
    - δx = scale·log2 e·c_dot·u·Σ|q k| + 3u·|x|: the wgmma dot (``c_dot``), scale·log2 e rounded to fp32 and the product;
    - p = exp2(x − m) for the running max m: the max cancels in O = Σ p·v / Σ p, except for the subtraction's u·Δ
      (Δ = max visible x_max − x); exp2f's 2 ulp (EX2) in every p and every rescale; n_steps = 22·n_t + 4 sequential
      steps (n_t key tiles: 16 row-sum adds, 4 P·V k-steps, 2 shuffles and the rescale per tile) of (u + EX2) each;
      ρ = ln 2·(2·max δx + u·Δ) + n_steps·(u + EX2) relative in numerator and l;
    - P is rounded to bf16 before P·V (2⁻⁸ relative on the numerator only; l sums the unrounded P);
    - the approximate reciprocal (2 ulp), the dropout scale, and the bf16 store (half an ulp of |O| + err).
    LSE = (m + log2 l) / log2 e: the weighted δx and u·Δ, l's own chain ρ_l = EX2 + 18u + n_t·(2u + EX2) (each p's exp2
    and ≤ 16 row-sum adds and 2 shuffles, then per later tile one rescale and one add), __log2f's 2 ulp (≤ 2⁻²² + 2 ulp of
    |log2 l|), the add and the approximate division (3 ulp of |LSE|).

    Backward (given O, LSE; L = LSE·log2 e in fp32):
    - P = exp2(x − L): e_P = ln 2·(δx + u·|L| + u·|x − L|) + EX2 relative;
    - dP = dO·Vᵀ: c_dot·u·Σ|dO v|; δ = Σ dO·O (from the bf16 O) − dlse in fp32: 20u·(Σ|dO O| + |dlse|) (each lane's 4
      products, 5 shuffles and the subtraction, truncating);
    - dS = P∘(dP∘Z·r − δ): P·(r·e_dP + e_δ) + (e_P + 2u)·|P (dP Z r − δ)|, then rounded to bf16 (2⁻⁸);
    - dQ = scale·dS·K, dK = scale·Σ_heads dSᵀ·Q, dV = r·Σ_heads (P∘Z)ᵀ·dO (P rounded to bf16): the propagated errors plus
      the fp32 accumulation over all tiles of the row or key, 2u·(15 + 4·n) of Σ|terms| with n the k-steps / 4 in the
      chain (key tiles for dQ; query tiles × G heads for dK, dV), the scale product (u) and the bf16 store (half an ulp)."""
    B, H, G, D = case.B, case.H, case.G, case.D
    dev = q.device
    sc = case.scale
    sl2 = sc * LOG2E
    r = case.rscale
    keep = case.keep(dev)
    i_all = torch.arange(case.S_q, device=dev)[:, None]
    j_all = torch.arange(case.S_kv, device=dev)[None, :]
    n_kt = (case.S_kv + BT - 1) // BT
    n_qt = (case.S_q + BT - 1) // BT
    cd = c_dot(D)
    out = {}
    O = torch.zeros(B, case.S_q, H, D, dtype=F64, device=dev)
    Ot = torch.zeros_like(O)
    LSE = torch.zeros(B, H, case.S_q, dtype=F64, device=dev)
    Lt = torch.zeros_like(LSE)
    bwd = o_in is not None
    if bwd:
        dQ, dQt = torch.zeros_like(O), torch.zeros_like(O)
        dK = torch.zeros(B, case.S_kv, case.Hkv, D, dtype=F64, device=dev)
        dKt, dV, dVt = torch.zeros_like(dK), torch.zeros_like(dK), torch.zeros_like(dK)
    for b in range(B):
        vis_b = case.visible(i_all, j_all, torch.tensor(b, device=dev), mask)      # [S_q, S_kv]
        for h in range(H):
            hk = h // G
            qd, kd, vd, gd = (x.to(F64) for x in (q[b, :, h], k[b, :, hk], v[b, :, hk], go[b, :, h]))
            vis = vis_b.clone()
            for (bb, hh, ii, jj) in drop:
                if bb == b and hh == h:
                    vis[ii, jj] = False
            Z = keep[b, h].to(F64) * r if keep is not None else None
            s = qd @ kd.T
            A = qd.abs() @ kd.abs().T
            x = s * sl2
            dx = sl2 * cd * U * A + 3 * U * x.abs()
            xm = x.masked_fill(~vis, -math.inf)
            m = xm.amax(-1, keepdim=True)
            any_ = torch.isfinite(m)
            m0 = torch.where(any_, m, torch.zeros_like(m))
            p = torch.exp2(xm - m0)
            l = p.sum(-1, keepdim=True)
            lz = l.clamp_min(1e-300)
            pz = p * Z if Z is not None else p
            o = (pz @ vd) / lz
            E = (pz @ vd.abs()) / lz
            delta_x = (m0 - xm).masked_fill(~vis, 0).amax(-1, keepdim=True)
            dxm = dx.masked_fill(~vis, 0).amax(-1, keepdim=True)
            n_t = float(n_kt)
            n_steps = 22 * n_t + 4
            rho_p = n_steps * (U + EX2)
            rho = LN2 * (2 * dxm + U * delta_x) + rho_p
            err = ((2 * rho + BF) / (1 - rho) + 4 * U) * E
            tol = err + bf16_ulp(o.abs() + err) / 2
            O[b, :, h] = torch.where(any_, o, torch.zeros_like(o))
            Ot[b, :, h] = torch.where(any_, tol, torch.zeros_like(tol))
            lse = (m0 + torch.log2(lz)) * LN2
            log2l = torch.log2(lz)
            rho_l = EX2 + 18 * U + n_t * (2 * U + EX2)
            lt = LN2 * (dxm + U * delta_x + 1.5 * rho_l * LOG2E + 2.0 ** -22 + 2 * ulp32(log2l) + U * (m0 + log2l).abs())
            lt = lt + 3 * ulp32(lse)
            LSE[b, h] = torch.where(any_, lse, torch.full_like(lse, -math.inf))[:, 0]
            Lt[b, h] = torch.where(any_, lt, torch.zeros_like(lt))[:, 0]
            if not bwd:
                continue
            od = o_in[b, :, h].to(F64)
            L64 = lse_in[b, h].to(F64)[:, None]
            Lfin = torch.isfinite(L64)
            L2 = torch.where(Lfin, L64 * LOG2E, torch.zeros_like(L64))
            P = torch.where(vis & Lfin, torch.exp2((x - L2).masked_fill(~vis, -math.inf)), torch.zeros((), dtype=F64,
                                                                                                      device=dev))
            eP = LN2 * (dx + U * L2.abs() + U * (x - L2).abs()) + EX2
            dP = gd @ vd.T
            edP = cd * U * (gd.abs() @ vd.abs().T)
            dlt = (gd * od).sum(-1, keepdim=True)
            edl = 20 * U * (gd * od).abs().sum(-1, keepdim=True)
            dPz = dP * Z if Z is not None else dP
            edPz = edP * Z if Z is not None else edP
            dS = P * (dPz - dlt)
            eS0 = P * (edPz + edl) + (eP + 2 * U) * dS.abs()
            eS = eS0 + BF * (dS.abs() + eS0)
            aS = dS.abs() + eS
            dQ[b, :, h] = sc * (dS @ kd)
            gq = 2 * U * (15 + 4 * n_kt)
            dQt[b, :, h] = sc * (eS @ kd.abs() + gq * (aS @ kd.abs())) * (1 + 2 * U)
            dK[b, :, hk] += sc * (dS.T @ qd)
            dKt[b, :, hk] += sc * (eS.T @ qd.abs())
            dKt[b, :, hk] += sc * (2 * U * (15 + 4 * n_qt * G)) * (aS.T @ qd.abs())
            Pz = P * Z if Z is not None else P
            dV[b, :, hk] += Pz.T @ gd
            ePz = (eP + BF * (1 + eP)) * Pz
            dVt[b, :, hk] += ePz.T @ gd.abs() + 2 * U * (15 + 4 * n_qt * G) * ((Pz + ePz).T @ gd.abs())
    out["o"] = (O, Ot)
    out["lse"] = (LSE, Lt)
    if bwd:
        for name, x, t in (("dq", dQ, dQt), ("dk", dK, dKt), ("dv", dV, dVt)):
            t = t * (1 + 4 * U) + U * x.abs()
            out[name] = (x, t + bf16_ulp(x.abs() + t) / 2)
    return out


def _ratio(err, tol):
    return torch.where(tol > 0, err / tol, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))


def check_random(case: Case, k: Kernels, device, seed=3) -> dict:
    """Probe C: O and LSE of the kernels' forward, then dQ, dK, dV of their backward given that O and LSE, each element
    within its bound from ``reference``; and the bounds ≥ 10× tighter than removing the boosted edge pair (head 0 of each
    group) moves some element of O, dQ, dK and dV.  Returns the worst error / bound of each output."""
    mask = case.mask(device)
    q, kk, v, go, pairs = random_inputs(case, device, seed)
    o, lse = k.fwd(case, q, kk, v, mask, case.scale)
    dq, dk, dv = k.bwd(case, go, q, kk, v, o, lse, None, mask, case.scale)
    ref = reference(case, q, kk, v, go, mask, o, lse)
    drop = [(b, hk * case.G, i, j) for b, i, j in pairs for hk in range(case.Hkv)]
    ref_d = reference(case, q, kk, v, go, mask, o, lse, drop=drop)
    worst = {}
    for name, got in (("o", o), ("lse", lse), ("dq", dq), ("dk", dk), ("dv", dv)):
        want, tol = ref[name]
        g64 = got.to(F64)
        if name == "lse":
            fin = torch.isfinite(want)
            assert torch.equal(torch.isfinite(g64), fin), f"{case.name}: LSE finite pattern"
            g64, want, tol = g64[fin], want[fin], tol[fin]
        err = (g64 - want).abs()
        bad = ~(err <= tol)
        assert not bad.any(), (f"{case.name} {name}: {int(bad.sum())} of {bad.numel()} outside the bound; worst err "
                               f"{err.max().item():.3e} at bound {tol.flatten()[err.flatten().argmax()].item():.3e}; "
                               f"first {bad.nonzero()[0].tolist()}")
        worst[name] = _ratio(err, tol).max().item()
        if name != "lse" and not (case.window == 1 and name in ("dq", "dk")):
            # (with W = 1 a row attends to one key, and softmax over one key has dQ = dK = 0 exactly)
            margin = _ratio((ref_d[name][0] - ref[name][0]).abs(), tol).max().item()
            assert margin >= 10, f"{case.name}: removing an edge pair moves {name} only {margin:.1f}× its bound"
    return worst


# ---- the float64 simulation and its faults --------------------------------------------------------------------------------
MUTANTS = ("diagonal_dropped", "window_one_late", "union_first_half_hi", "dkdv_second_half_lo", "mask_other_buffer",
           "gqa_head_skipped", "delta_unrounded_o")


def _visited(case: Case, kernel: str, mutant: Optional[str], device) -> torch.Tensor:
    """[S_q, S_kv] bool: pairs inside a tile the kernel's CTA visits (for the row CTA: its key tiles; for the dK/dV key CTA:
    its query tiles)."""
    win = min(case.window, case.S_kv + case.q_offset) if case.window else 0
    out = torch.zeros(case.S_q, case.S_kv, dtype=torch.bool, device=device)
    if kernel in ("fwd", "dq"):
        for c in range(-(-case.S_q // (2 * BT))):
            lo, hi = cta_key_range(case.S_kv, case.causal, win, case.q_offset, c, mutant == "union_first_half_hi")
            out[2 * BT * c:2 * BT * (c + 1), lo * BT:hi * BT] = True
    else:
        for c in range(-(-case.S_kv // (2 * BT))):
            lo, hi = cta_query_range(case.S_q, case.causal, win, case.q_offset, c, mutant == "dkdv_second_half_lo")
            out[lo * BT:hi * BT, 2 * BT * c:2 * BT * (c + 1)] = True
    return out


def kernel_vis(case: Case, kernel: str, mask, mutant: Optional[str], device) -> torch.Tensor:
    """[B, H, S_q, S_kv] the pairs a (possibly faulty) kernel lets through: the rule, inside visited tiles."""
    i = torch.arange(case.S_q, device=device)[:, None]
    j = torch.arange(case.S_kv, device=device)[None, :]
    b = torch.arange(case.B, device=device)[:, None, None]
    off = case.q_offset
    m = mask
    if mutant == "mask_other_buffer" and mask is not None and kernel in ("fwd", "dq"):
        jj = torch.arange(case.S_kv, device=device) ^ BT                            # the other buffer's tile
        m = torch.where(jj < case.S_kv, mask[:, jj.clamp(max=case.S_kv - 1)], torch.zeros_like(mask))
    v = case.visible(i[None], j[None], b, m)
    if mutant == "diagonal_dropped" and case.causal:
        v = v & (j < i + off)
    if mutant == "window_one_late" and case.window:
        v = v & (j > i + off - case.window + 1)
    v = v & _visited(case, kernel, mutant, device)
    v = v[:, None].expand(case.B, case.H, case.S_q, case.S_kv).clone()
    if mutant == "gqa_head_skipped" and kernel == "dkdv" and case.G > 1:
        v[:, case.G - 1::case.G] = False
    return v


def sim_kernels(mutant: Optional[str] = None) -> Kernels:
    """The kernels' equations in float64 with their output roundings (O, dQ, dK, dV to bf16, LSE to fp32), each kernel on
    its own visibility from ``kernel_vis``; ``mutant`` names one fault (``MUTANTS``)."""
    def fwd(case, q, k, v, mask, scale):
        dev = q.device
        vis = kernel_vis(case, "fwd", mask, mutant, dev)
        o, lse = _sim_fwd(case, q, k, v, vis, scale)
        return o.to(torch.bfloat16), lse.float()

    def bwd(case, go, q, k, v, o, lse, dlse, mask, scale):
        dev = q.device
        G = case.G
        keep = case.keep(dev)
        Z = keep.to(F64) * case.rscale if keep is not None else 1.0
        qd, gd = q.to(F64).transpose(1, 2), go.to(F64).transpose(1, 2)             # [B, H, S, D]
        kd = k.to(F64).transpose(1, 2).repeat_interleave(G, 1)
        vd = v.to(F64).transpose(1, 2).repeat_interleave(G, 1)
        if mutant == "delta_unrounded_o":
            od, _ = _sim_fwd(case, q, k, v, kernel_vis(case, "fwd", mask, None, dev), case.scale if scale != 1.0 else 1.0)
            od = od.transpose(1, 2)
        else:
            od = o.to(F64).transpose(1, 2)
        delta = (gd * od).sum(-1, keepdim=True) - (dlse.to(F64)[..., None] if dlse is not None else 0.0)
        L = lse.to(F64)[..., None]
        s = qd @ kd.transpose(-1, -2) * scale
        dP = gd @ vd.transpose(-1, -2)
        res = []
        for kern in ("dq", "dkdv"):
            vis = kernel_vis(case, kern, mask, mutant, dev)
            P = torch.where(vis, torch.exp((s - L).masked_fill(~vis, -math.inf)), torch.zeros((), dtype=F64, device=dev))
            dS = P * (dP * Z - delta)
            if kern == "dq":
                res.append((dS @ kd * scale).transpose(1, 2))
            else:
                B, H, Sq, Skv = P.shape
                dk = (dS.transpose(-1, -2) @ qd * scale).view(B, case.Hkv, G, Skv, -1).sum(2).transpose(1, 2)
                dv = ((P * Z).transpose(-1, -2) @ gd).view(B, case.Hkv, G, Skv, -1).sum(2).transpose(1, 2)
                res += [dk, dv]
        return tuple(x.to(torch.bfloat16) for x in res)
    return Kernels(fwd, bwd)


def _sim_fwd(case, q, k, v, vis, scale):
    """float64 (O [B, S_q, H, D], LSE [B, H, S_q]) on the pairs ``vis``; an empty row gets O = 0, LSE = −inf."""
    G = case.G
    qd = q.to(F64).transpose(1, 2)
    kd = k.to(F64).transpose(1, 2).repeat_interleave(G, 1)
    vd = v.to(F64).transpose(1, 2).repeat_interleave(G, 1)
    s = (qd @ kd.transpose(-1, -2) * scale).masked_fill(~vis, -math.inf)
    lse = torch.logsumexp(s, -1)
    fin = torch.isfinite(lse)
    p = torch.where(vis, torch.exp(s - torch.where(fin, lse, torch.zeros_like(lse))[..., None]),
                    torch.zeros((), dtype=F64, device=q.device))
    keep = case.keep(q.device)
    if keep is not None:
        p = p * keep.to(F64) * case.rscale
    o = (p @ vd).transpose(1, 2)
    return o, lse


# ---- CPU checks -----------------------------------------------------------------------------------------------------------
def test_tile_ranges_cover_every_visible_pair_exhaustively():
    """For S_q = S_kv = S ≤ 300, every W in 1 … S + off (the launcher clamps larger ones to S + off), off ∈ {0, 1, 63, 64,
    65, 200} and plain causal attention: every visible pair lies in a tile its row CTA visits (forward / dQ: key tiles
    from the first half's lo to the second half's hi) and in one its key CTA visits (dK/dV: query tiles from the first
    half's lo to the second half's hi).  Row i sees keys [i + off − W + 1, i + off] ∩ [0, S); key j is seen by rows
    [j − off, j − off + W − 1] ∩ [0, S).  Non-causal attention visits every tile.  (The launcher requires S_q = S_kv when
    causal, so the causal check runs on square shapes.)"""
    checked = 0
    for off in (0, 1, 63, 64, 65, 200):
        for S in range(1, 301):
            Ws = np.arange(1, S + off + 1)[:, None] if off else np.concatenate([np.arange(1, S + 1), [0]])[:, None]
            W = Ws
            i = np.arange(S)[None, :]
            nolim = W == 0                                                          # plain causal: no window
            vlo = np.where(nolim, 0, np.maximum(0, i + off - W + 1))
            vhi = np.minimum(S - 1, i + off)
            c = i // (2 * BT)
            q0 = 2 * BT * c
            n = (S + BT - 1) // BT
            lo = np.where(nolim, 0, np.maximum(0, q0 + off - W + 1) // BT)
            hi = np.minimum(n, (q0 + 2 * BT - 1 + off) // BT + 1)
            ok = (vlo > vhi) | ((lo * BT <= vlo) & (vhi < hi * BT))
            assert ok.all(), (S, off, int(W[np.nonzero(~ok)[0][0], 0]), int(np.nonzero(~ok)[1][0]))
            j = i
            rlo = np.maximum(0, j - off)
            rhi = np.where(nolim, S - 1, np.minimum(S - 1, j - off + W - 1))
            k0 = 2 * BT * (j // (2 * BT))
            qlo = np.maximum(0, k0 - off) // BT
            qhi = np.where(nolim, n, np.minimum(n, (k0 + BT + 2 * BT - 2 + W - off) // BT))
            ok = (rlo > rhi) | ((qlo * BT <= rlo) & (rhi < qhi * BT))
            assert ok.all(), (S, off, int(W[np.nonzero(~ok)[0][0], 0]), int(np.nonzero(~ok)[1][0]))
            checked += ok.size
    # the vectorised formulas above are the same as the scalar transcriptions the probes use
    for S, W, off in ((300, 65, 63), (129, 1, 0), (200, 264, 64), (64, 0, 0)):
        for c in range(-(-S // (2 * BT))):
            lo, hi = cta_key_range(S, True, W, off, c)
            q0 = 2 * BT * c
            assert lo == (max(0, q0 + off - W + 1) // BT if W else 0)
            assert hi == min((S + BT - 1) // BT, (q0 + 2 * BT - 1 + off) // BT + 1)
            qlo, qhi = cta_query_range(S, True, W, off, c)
            assert qlo == max(0, q0 - off) // BT
            assert qhi == (min((S + BT - 1) // BT, (q0 + 3 * BT - 2 + W - off) // BT) if W else (S + BT - 1) // BT)
    for S_q, S_kv in ((1, 300), (300, 1), (129, 65), (257, 191)):
        assert cta_key_range(S_kv, False, 0, 0, 0) == (0, (S_kv + BT - 1) // BT)
        assert cta_query_range(S_q, False, 0, 0, 0) == (0, (S_q + BT - 1) // BT)
    assert checked > 10 ** 7


CPU = [
    Case("causal-s200-g2", B=2, S_q=200, S_kv=200, H=4, Hkv=2, D=64, causal=True),
    Case("noncausal-129x65-mask", B=2, S_q=129, S_kv=65, H=2, Hkv=1, D=64, rand=0.7),
    Case("window-65-off63", B=1, S_q=193, S_kv=193, H=2, Hkv=2, D=64, causal=True, window=65, q_offset=63),
    Case("window-1-left-pad", B=2, S_q=130, S_kv=130, H=2, Hkv=1, D=64, causal=True, window=1, left=(0, 70)),
    Case("dropout-causal-g2", B=1, S_q=150, S_kv=150, H=4, Hkv=2, D=64, causal=True, dropout=0.5),
    Case("window-129-off200-d96", B=1, S_q=257, S_kv=257, H=2, Hkv=1, D=96, causal=True, window=129, q_offset=200),
]


@pytest.mark.parametrize("case", CPU, ids=lambda c: c.name)
def test_probes_pass_on_the_float64_simulation(case):
    k = sim_kernels()
    check_fwd_visibility(case, k, "cpu")
    check_bwd_visibility(case, k, "cpu")
    check_dlse(case, k, "cpu")
    if not case.dropout:
        check_planted(case, k, "cpu")
    worst = check_random(case, k, "cpu")
    assert all(w <= 1.0 for w in worst.values()), worst


def _probes(case):
    return (("A-fwd", check_fwd_visibility), ("A-bwd", check_bwd_visibility), ("A-dlse", check_dlse),
            ("B-planted", check_planted), ("C-random", check_random))


def caught_by(case: Case, mutant: str):
    """Names of the probes that reject the simulated kernel with this fault."""
    k = sim_kernels(mutant)
    names = []
    for name, fn in _probes(case):
        if name == "B-planted" and case.dropout:
            continue
        try:
            fn(case, k, "cpu")
        except AssertionError:
            names.append(name)
    return names


# each fault on a case where it changes something, and the probes that must reject it
MUTANT_CASES = {
    "diagonal_dropped": (CPU[0], {"A-fwd", "A-bwd", "B-planted", "C-random"}),
    "window_one_late": (CPU[2], {"A-fwd", "A-bwd", "B-planted"}),
    "union_first_half_hi": (CPU[0], {"A-fwd", "A-bwd", "B-planted", "C-random"}),
    "dkdv_second_half_lo": (CPU[0], {"A-bwd"}),
    "mask_other_buffer": (Case("mask-other-buffer", B=2, S_q=200, S_kv=200, H=2, Hkv=1, D=64, lens=(150, 100)),
                          {"A-fwd", "A-bwd", "B-planted", "C-random"}),
    "gqa_head_skipped": (CPU[0], {"A-bwd", "C-random"}),
    "delta_unrounded_o": (CPU[0], {"C-random"}),
}


@pytest.mark.parametrize("mutant", MUTANTS)
def test_probes_reject_each_fault(mutant):
    """Every simulated fault is rejected, and by the probes expected to see it (the caught set is reported)."""
    case, must = MUTANT_CASES[mutant]
    got = set(caught_by(case, mutant))
    assert must <= got, (mutant, sorted(got))


def test_simulated_faults_change_the_visible_pairs():
    """The visibility faults are real on their cases: each removes or adds pairs of the kernel it affects."""
    for mutant in MUTANTS[:6]:
        case, _ = MUTANT_CASES[mutant]
        mask = case.mask("cpu")
        changed = [kern for kern in ("fwd", "dq", "dkdv")
                   if not torch.equal(kernel_vis(case, kern, mask, mutant, "cpu"), kernel_vis(case, kern, mask, None, "cpu"))]
        assert changed, mutant


def test_visibility_probe_observes_every_pair():
    """The bands of the visibility probe hold every key (forward, dQ) and every query row (dK/dV) of the case."""
    for case in CPU:
        for S in (case.S_q, case.S_kv):
            launches = band_launches(case, S)
            for s in range(case.B * case.Hkv):
                rows = {launch[s] + d for launch in launches for d in range(BT) if 0 <= launch[s] + d < S}
                assert rows == set(range(S)), (case.name, s)
