"""Slot-by-slot probes of the token-generation attention kernels, and their checks off the GPU.

The kernels (``csrc/decode.cu`` ``decode_attn_kernel`` + the two combine kernels, ``csrc/attention_sm90.cu``
``spec_attn_kernel``) split a sequence's visible cache slots over CTAs, wrap them around a rolling cache and cut them into
64-slot tiles.  A slot lost, read twice or replaced by its neighbour moves a row's output by only about 1/n of it, far
inside a tolerance relative to max|ref|.  The probes here make every such error exact and large:

A. visibility: q = 0, so every visible score is exactly 0, ex2.approx(0) = 1 and ex2.approx(−inf) = 0, and every
   running rescale and split merge multiplies by exactly 1 or 0.  V holds 0 / 1 entries that encode the slot index, so
   the fp32 sums are exact integers and name the slots that were summed.
B. planted slot: one slot j* per (sequence, token, head) scores ≥ 40 log2-units above every other slot, so the output must
   equal V[j*] bit for bit.  The planted slots are the split edges, tile edges, the ring's wrap rows, the first and last
   visible slots and the window tokens.
C. random inputs against float64 with a per-element bound derived from the kernels' arithmetic, which also asserts that
   dropping one split-edge slot moves the reference by at least 10× the bound somewhere.

The builders and checkers take the attention as a callable, so the same probes run on the CUDA kernels
(``test_decode_probes_gpu.py``), on the torch paths here, and on simulated kernels with deliberately wrong visibility,
which every probe must reject.  Which slots each token sees comes from ``ops.attention.speculation_visibility``.
"""
import math
from dataclasses import dataclass, field
from typing import Callable, Optional

import pytest
import torch

from neuronx_distributed_b200.ops import attention

E4M3 = torch.float8_e4m3fn
F64 = torch.float64
U = 2.0 ** -24                     # fp32 unit roundoff
EX2 = 2.0 ** -22                   # exp2f / ex2.approx.ftz.f32 (what -use_fast_math makes of it): at most 2 fp32 ulp
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
TILE = 64                          # slots of a spec_attn_kernel K/V tile and rows of its query tile


# ---- the launchers' split rules (csrc/binding.cpp) and the kernels' split ranges ----------------------------------------
def decode_splits(B: int, Hkv: int, L: int, window: int, sms: int) -> int:
    """``decode_splits`` of the decode launcher: ~6 CTAs per SM, at most 64 splits, at least 64 rows per split."""
    rows = window if 0 < window < L else L
    s = (6 * sms + B * Hkv - 1) // (B * Hkv)
    return max(1, min(s, 64, (rows + 63) // 64))


def spec_splits(B: int, W: int, G: int, Hkv: int, L: int, window: int, sms: int) -> int:
    """Splits of the ``speculation_attention`` launcher: ~4 CTAs per SM, at most 64, at least 128 slots per split."""
    row_tiles = (W * G + TILE - 1) // TILE
    rows = min(L, min(window, L) + W - 1) if window > 0 else L
    ctas = B * Hkv * row_tiles
    return max(1, min((4 * sms + ctas - 1) // ctas, 64, (rows + 127) // 128))


def decode_ranges(p: int, L: int, window: int, splits: int, rolling: bool):
    """Logical slot range [s0, s1) of every split of ``decode_attn_kernel`` for position p (empty ones included)."""
    hi = p + 1 if rolling else min(p + 1, L)
    if rolling:
        lo = max(p - window + 1, 0)
    else:
        lo = min(max(p - window + 1, 0), L) if window > 0 else 0
    n = max(hi - lo, 0)
    per = (n + splits - 1) // splits
    return [(lo + s * per, min(hi, lo + s * per + per)) for s in range(splits)]


def spec_ranges(p: int, L: int, W: int, G: int, depth, window: int, splits: int, rolling: bool, rt: int):
    """Logical slot range [s0, s1) of every split of row tile ``rt`` of ``spec_attn_kernel`` (whole 64-slot tiles)."""
    w_lo, w_hi = rt * TILE // G, min((rt * TILE + TILE) // G, W)
    dmin = min(int(depth[w]) for w in range(w_lo, w_hi))
    lo_l = min(p, p + dmin - window + 1) if window > 0 else 0
    lo = max(lo_l, 0) if rolling else min(max(lo_l, 0), L)
    hi = max(p + W, lo) if rolling else max(min(p + W, L), lo)
    per = ((hi - lo + splits - 1) // splits + TILE - 1) // TILE * TILE
    return [(lo + s * per, min(hi, lo + s * per + per)) for s in range(splits)]


# ---- cases ----------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    """One launch shape: ``pos`` [B] positions, W tokens per sequence (W = 1: one-token decode), a chain or a tree."""
    name: str
    H: int
    Hkv: int
    D: int
    L: int
    pos: tuple
    W: int = 1
    window: int = 0
    rolling: bool = False
    tree: Optional[str] = None                     # None (a chain), "medusa" or "random"
    mask: Optional[torch.Tensor] = field(default=None, repr=False)
    depth: Optional[torch.Tensor] = field(default=None, repr=False)

    def __post_init__(self):
        if self.tree is not None and self.mask is None:
            from test_speculation_attention_cpu import medusa_tree, random_tree

            self.mask, self.depth = medusa_tree() if self.tree == "medusa" else random_tree(self.W, 11)
            assert self.mask.shape == (self.W, self.W), (self.name, self.mask.shape)

    @property
    def B(self):
        return len(self.pos)

    @property
    def G(self):
        return self.H // self.Hkv

    @property
    def scale(self):
        return 1.0 / math.sqrt(self.D)

    def depths(self):
        return list(range(self.W)) if self.depth is None else [int(d) for d in self.depth]

    def positions(self, device):
        return torch.tensor(self.pos, dtype=torch.long, device=device)

    def vis(self, device) -> torch.Tensor:
        """[B, W, L] bool: the slots (cache rows) each token sees."""
        return attention.speculation_visibility(self.positions(device), self.L, self.W, self.mask, self.depth, self.window,
                                                self.rolling)

    def splits(self, sms: int, spec: bool) -> int:
        if spec:
            return spec_splits(self.B, self.W, self.G, self.Hkv, self.L, self.window, sms)
        return decode_splits(self.B, self.Hkv, self.L, self.window, sms)

    def ranges(self, b: int, sms: int, spec: bool):
        """Every split's logical range of sequence b (spec: over all row tiles)."""
        p, s = self.pos[b], self.splits(sms, spec)
        if not spec:
            return decode_ranges(p, self.L, self.window, s, self.rolling)
        out = []
        for rt in range((self.W * self.G + TILE - 1) // TILE):
            out += spec_ranges(p, self.L, self.W, self.G, self.depths(), self.window, s, self.rolling, rt)
        return out

    def row(self, c: int) -> int:
        return c % self.L if self.rolling else c

    def edges(self, sms: int, spec: bool, vis: torch.Tensor):
        """[B][W] sorted lists of the cache rows to plant: the first and last slot of every split (spec: and of every 64-slot
        tile), the first and last visible slot, the newest slot, the ring's wrap rows and every window token's slot, each
        kept where token w sees it."""
        out = []
        for b in range(self.B):
            cand = set()
            for s0, s1 in self.ranges(b, sms, spec):
                if s1 <= s0:
                    continue
                cand |= {s0, s1 - 1}
                if spec:
                    for t in range(s0, s1, TILE):
                        cand |= {t, min(t + TILE, s1) - 1}
            rows = {self.row(c) for c in cand if c >= 0} | {0, self.L - 1}
            rows |= {self.row(self.pos[b] + u) for u in range(self.W) if self.pos[b] + u >= 0}
            per_w = []
            for w in range(self.W):
                seen = vis[b, w].nonzero()[:, 0].tolist()
                mine = {r for r in rows if 0 <= r < self.L and vis[b, w, r]}
                if seen:
                    mine |= {seen[0], seen[-1]}
                per_w.append(sorted(mine))
            out.append(per_w)
        return out

    def split_len(self, sms: int, spec: bool) -> int:
        """The longest split of sequence 0 (a mutation shifts a slot by it)."""
        return max(s1 - s0 for s0, s1 in self.ranges(0, sms, spec))


# ---- caches ---------------------------------------------------------------------------------------------------------------
def to_cache(x: torch.Tensor, cache: str, scale: float):
    """float values → (cache tensor, its float64 de-quantisation).  An e4m3 cache holds x / scale."""
    if cache == "bf16":
        t = x.to(torch.bfloat16)
        return t, t.to(F64)
    t = (x / scale).to(E4M3)
    return t, t.to(F64) * scale


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |x| (subnormal spacing below the normal range)."""
    e = torch.floor(torch.log2(x.abs().to(F64).clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(seed)


# A run function is ``run(q, kc, vc, positions, k_scale, v_scale) → out [B, W, H, D]`` (the bf16-output paths) or
# ``→ (o [B, H, D], m [B, H], l [B, H])`` (flash-decoding's local partial).
Run = Callable


# ---- A. visibility probe --------------------------------------------------------------------------------------------------
def band_count(case: Case) -> int:
    M = case.D // 2
    return -(-case.L // (M * M))


def band_v(case: Case, t: int, device) -> torch.Tensor:
    """[B, L, Hkv, D] of 0 / 1: slot c carries one-hot(c mod M) in the first M = D/2 columns and one-hot(⌊c/M⌋ mod M) in
    the last M, but only in the M²-slot band that (sequence b, kv head h) owns in launch t: band ⌊c/M²⌋ with
    (⌊c/M²⌋ + b·Hkv + h) mod n_bands = t.  Over the n_bands launches every (b, h, c) is carried once, neighbouring
    sequences and heads carry different bands (a read of the wrong sequence or head shows), and inside a band the two
    one-hots name the slot: a slot lost, doubled or replaced by another slot of the band changes some column sum."""
    M, nb = case.D // 2, band_count(case)
    c = torch.arange(case.L, device=device)
    enc = torch.zeros(case.L, case.D, device=device)
    enc[c, c % M] = 1
    enc[c, M + (c // M) % M] = 1
    own = (c[None, :, None] // (M * M) + torch.arange(case.B, device=device)[:, None, None] * case.Hkv
           + torch.arange(case.Hkv, device=device)[None, None, :]) % nb == t
    return own[..., None].float() * enc[None, :, None, :]


def _expand(x: torch.Tensor, G: int) -> torch.Tensor:
    """[B, L, Hkv, D] → [B, L, H, D] over the GQA group."""
    return x.repeat_interleave(G, 2) if G > 1 else x


def check_visibility(case: Case, cache: str, run: Run, device) -> None:
    """Probe A on a path with a bf16 output: O = S / n with S = Σ_visible V, V the 0 / 1 values (an e4m3 cache stores
    them divided by a power-of-two v_scale, which the kernels multiply back exactly).  Every column sum S is an integer
    of at most M = D/2 ≤ 64 (a band is M² slots, and each one-hot value occurs M times in it).  The kernels compute S / n
    in fp32, exactly up to the division (approximate under --use_fast_math: 2 ulp), and round it to bf16 (8 significant
    bits: at most 2⁻⁸ relative), so O·n = S·(1 + δ) with |δ| ≤ 2⁻⁸ + 2⁻²¹, and |S·δ| ≤ 64·(2⁻⁸ + 2⁻²¹) < 0.26: rounding
    O·n to the nearest integer recovers every S exactly.  A token that sees nothing must get exactly 0."""
    ks, vs = (1.0, 1.0) if cache == "bf16" else (0.5, 2.0)
    g = _gen(device, 5)
    vis = case.vis(device)
    n = vis.sum(-1).to(F64)                                                     # [B, W]
    q = torch.zeros(case.B, case.W, case.H, case.D, dtype=torch.bfloat16, device=device)
    kc, _ = to_cache(torch.rand(case.B, case.L, case.Hkv, case.D, device=device, generator=g) * 2 - 1, cache, ks)
    for t in range(band_count(case)):
        vc, vd = to_cache(band_v(case, t, device), cache, vs)
        out = run(q, kc, vc, case.positions(device), ks, vs)
        assert out.shape == (case.B, case.W, case.H, case.D) and out.dtype == torch.bfloat16
        S = torch.einsum("bwl,blhd->bwhd", vis.to(F64), _expand(vd, case.G))
        assert S.max() <= case.D // 2
        got = torch.round(out.to(F64) * n[:, :, None, None])
        empty = n == 0
        assert torch.equal(out[empty].to(F64), torch.zeros_like(out[empty], dtype=F64)), f"{case.name}: an empty row is not 0"
        bad = (got != S) & ~empty[:, :, None, None]
        assert not bad.any(), (f"{case.name} band {t}: {int(bad.any(-1).sum())} rows (b, w, h) summed the wrong slots; "
                               f"first {bad.nonzero()[0].tolist()}")


def exact_v(case: Case, device) -> torch.Tensor:
    """[B, L, Hkv, D] of 0 / 1 for the exact fp32 partial: column 0 counts the slots, columns 1–16 hold the bits of
    c ⊕ key(b, h) and the rest one-hot((c ⊕ key) mod (D − 17)); key(b, h) differs between sequences and heads."""
    c = torch.arange(case.L, device=device)
    key = (torch.arange(case.B * case.Hkv, device=device).view(case.B, 1, case.Hkv) * 0x9E5 + 0x2B) & 0xFFFF
    x = c[None, :, None] ^ key                                                   # [B, L, Hkv]
    v = torch.zeros(case.B, case.L, case.Hkv, case.D, device=device)
    v[..., 0] = 1
    for i in range(16):
        v[..., 1 + i] = ((x >> i) & 1).float()
    v.scatter_(3, (17 + x % (case.D - 17))[..., None], 1.0)
    return v


def check_visibility_partial(case: Case, cache: str, run: Run, device) -> None:
    """Probe A on flash-decoding's local partial, which returns o = Σ_visible V·v_scale, m (0 or −inf) and l = n in fp32:
    with q = 0 every term is an exact 0 / 1 product, every sum an integer below 2²⁴ and v_scale a power of two, so o, m and l
    must equal the host's sums exactly, whatever order the splits and warps add them in."""
    assert case.W == 1 and not case.rolling
    ks, vs = (1.0, 1.0) if cache == "bf16" else (0.25, 4.0)
    g = _gen(device, 6)
    vis = case.vis(device)[:, 0]                                                  # [B, L]
    q = torch.zeros(case.B, 1, case.H, case.D, dtype=torch.bfloat16, device=device)
    kc, _ = to_cache(torch.rand(case.B, case.L, case.Hkv, case.D, device=device, generator=g) * 2 - 1, cache, ks)
    vc, vd = to_cache(exact_v(case, device), cache, vs)
    o, m, l = run(q, kc, vc, case.positions(device), ks, vs)
    want_o = torch.einsum("bl,blhd->bhd", vis.to(F64), _expand(vd, case.G)).float()
    n = vis.sum(-1).float()[:, None].expand(case.B, case.H)
    want_m = torch.where(n > 0, torch.zeros_like(n), torch.full_like(n, -math.inf))
    for name, got, want in (("o", o, want_o), ("l", l, n), ("m", m, want_m)):
        assert got.dtype == torch.float32 and torch.equal(got, want), (
            f"{case.name}: partial {name} differs at {(got != want).nonzero()[:4].tolist()}")


# ---- B. planted-slot probe ------------------------------------------------------------------------------------------------
QA, KBIG = 64.0, 16.0              # the planted row's q entry and the planted slot's k entry; other k entries are in [−1, 1]


def planted_gap_log2(case: Case) -> float:
    """Score lead of the planted slot over any other slot, in log2 units: QA·(KBIG − 1)·scale·log2 e."""
    return QA * (KBIG - 1) * case.scale * LOG2E


def planted_launches(case: Case, edges):
    """(row group, round) pairs: rows r = w·G + g of a kv head are planted along dimension r mod D, so D rows at a time
    (group ⌊r/D⌋); each round plants a different edge per head."""
    groups = -(-case.W * case.G // case.D)
    rounds = max(-(-len(e) // case.H) for per_w in edges for e in per_w if e)
    return [(grp, rnd) for grp in range(groups) for rnd in range(rounds)]


def planted_inputs(case: Case, cache: str, edges, grp: int, rnd: int, device, seed: int = 7):
    """q, caches and the planted slots of one launch: row (b, w, h = kvh·G + g) of group ``grp`` gets q = QA along
    dimension e = (w·G + g) mod D and plants slot j* = edges[b][w][(h + rnd·H) mod n]; K[b, j*, kvh, e] = KBIG.  No other
    row of that kv head has q along e, so no other plant reaches it.  V is uniform in [1, 2) (on the cache's grid), so two
    slots' V rows practically never agree.  Returns (q, kc, vc, vd, picks [n, 4] = (b, w, h, j*))."""
    ks, vs = (1.0, 1.0) if cache == "bf16" else (2.0, 0.5)
    g = _gen(device, seed + 100 * grp + rnd)
    kx = torch.rand(case.B, case.L, case.Hkv, case.D, device=device, generator=g) * 2 - 1
    vx = torch.rand(case.B, case.L, case.Hkv, case.D, device=device, generator=g) + 1
    q = torch.zeros(case.B, case.W, case.H, case.D, device=device)
    picks = []
    for b in range(case.B):
        for w in range(case.W):
            e_bw = edges[b][w]
            if not e_bw:
                continue
            for h in range(case.H):
                r = w * case.G + h % case.G
                if r // case.D != grp:
                    continue
                j = e_bw[(h + rnd * case.H) % len(e_bw)]
                picks.append((b, w, h, j))
    pk = torch.tensor(picks, dtype=torch.long, device=device).view(-1, 4)
    b, w, h, j = pk.unbind(1)
    e = (w * case.G + h % case.G) % case.D
    q[b, w, h, e] = QA
    kx[b, j, h // case.G, e] = KBIG
    kc, _ = to_cache(kx, cache, ks)
    vc, vd = to_cache(vx, cache, vs)
    return q.to(torch.bfloat16), kc, vc, vd, pk, (ks, vs)


def check_planted(case: Case, cache: str, run: Run, device, sms: int, spec: bool, partial: bool = False) -> int:
    """Probe B.  The planted slot leads by ≥ 40 log2-units (asserted), so every other visible slot carries weight
    < 2⁻⁴⁰ relative to it and all of them together < L·2⁻⁴⁰ ≤ 2⁻²⁵ — below 2⁻¹⁰ of the smallest |V| (V ∈ [1, 2)·v_scale,
    so the others' V is at most twice it).  V[j*] is a bf16 number (an e4m3 one times a power of two); the fp32 output
    is V[j*]·(1 + ε) with |ε| < 2⁻²⁰ (plus the division's 2 ulp), which rounds back to V[j*] in bf16: the output must
    equal V[j*] bit for bit.  The spec kernel rounds P to bf16 before P·V, which leaves P = 1 on j* exact.  The partial
    returns o and l in fp32: o = V[j*]·(1 + ε′) with |ε′| < 2⁻²⁴ rounds to V[j*], and l = 1 + (≤ 2⁻²⁵) rounds to 1.
    Returns the number of launches."""
    assert planted_gap_log2(case) >= 40
    vis = case.vis(device)
    edges = case.edges(sms, spec, vis)
    launches = planted_launches(case, edges)
    for grp, rnd in launches:
        q, kc, vc, vd, pk, (ks, vs) = planted_inputs(case, cache, edges, grp, rnd, device)
        b, w, h, j = pk.unbind(1)
        assert vis[b, w, j].all()
        want = vd[b, j, h // case.G]
        if partial:
            o, m, l = run(q, kc, vc, case.positions(device), ks, vs)
            got_o, got_l = o[b, h], l[b, h]
            bad = (got_o.to(F64) != want).any(-1) | (got_l != 1)
        else:
            out = run(q, kc, vc, case.positions(device), ks, vs)
            bad = (out[b, w, h].to(F64) != want).any(-1)
        assert not bad.any(), (f"{case.name} group {grp} round {rnd}: {int(bad.sum())} of {bad.numel()} planted rows wrong; "
                               f"first (b, w, h, j*) = {pk[bad][0].tolist()}")
    return len(launches)


# ---- C. random inputs against float64 -------------------------------------------------------------------------------------
def random_inputs(case: Case, cache: str, device, sms: int, spec: bool, seed: int = 3):
    """q, K, V ~ N(0, 1) on the cache's grid (e4m3: k_scale 0.3, v_scale 0.7).  In each sequence one split-edge slot
    (the last slot of the first split that has a successor, else the last visible slot) gets K along the q of head 0 of
    each kv head for the first token that sees it, scoring ln n + 2 nats: it carries most of that row's weight, so the
    float64 reference notices when it is lost.  Returns (q, kc, vc, kd, vd, scales, boosted [(b, j)])."""
    ks, vs = (1.0, 1.0) if cache == "bf16" else (0.3, 0.7)
    g = _gen(device, seed)
    q = torch.randn(case.B, case.W, case.H, case.D, device=device, generator=g).to(torch.bfloat16)
    kx = torch.randn(case.B, case.L, case.Hkv, case.D, device=device, generator=g)
    vx = torch.randn(case.B, case.L, case.Hkv, case.D, device=device, generator=g)
    vis = case.vis(device)
    boosted = []
    for b in range(case.B):
        rs = [r for r in case.ranges(b, sms, spec) if r[1] > r[0]]
        cands = [case.row(s1 - 1) for (s0, s1) in rs[:-1]] + [case.row(rs[-1][1] - 1)] if rs else []
        cands = [c for c in cands if vis[b, :, c].any()]
        if not cands:
            continue
        j = cands[0]
        w = int(vis[b, :, j].nonzero()[0, 0])
        n = int(vis[b, w].sum())
        qh = q[b, w, ::case.G].float()                                           # [Hkv, D]: head 0 of each group
        kx[b, j] = qh * ((math.log(n) + 2) / (case.scale * qh.pow(2).sum(-1, keepdim=True)))
        boosted.append((b, j))
    kc, kd = to_cache(kx, cache, ks)
    vc, vd = to_cache(vx, cache, vs)
    return q, kc, vc, kd, vd, (ks, vs), boosted


def ref_and_bound(case: Case, q, kd, vd, vis, spec: bool, n_chain: int, n_merge: int):
    """float64 reference O = Σ p·v / Σ p (p = 2^(d − max), d = q·k·scale·log2 e over the de-quantised cache) and a bound on
    |O_kernel − O| per element:

    - scores: the kernels fold scale·log2 e·k_scale into one fp32 factor (3 roundings) and into q (1); the dot product is
      an fp32 chain (decode: 8 fmas and ≤ 4 shuffle adds; spec: mma.sync over D products, whose internal adds may
      truncate: 2u each), so |d̂ − d| ≤ δd = c·u·S with S = scale·log2 e·Σ|q_i k_i| and c = 24 (decode) or 2D + 16 (spec).
      Subtracting the running max adds u·|d − m|.  A score error δ moves 2^d by ln 2·δ relative; the max cancels in the
      ratio, so each p carries ln 2·(2δd + u·Δ) with Δ = max visible |d − m|.
    - exp2: 2 ulp per ex2.approx (EX2) in every p and in every rescale factor; each of the n_chain sequential steps of a
      lane's running sum (fma o·corr + p·v), the warp / CTA / split merges (n_merge: exp2 factor plus one add each) and the
      v_scale product adds at most (u + EX2) relative to the positive sums Σp|v| and Σp.
    - spec only: P is rounded to bf16 before P·V (8 significant bits: 2⁻⁸ relative per term of the numerator, not of l).

    So with ρ = ln 2·(2δd + u·Δ) + (n_chain + n_merge)·(u + EX2) the fp32 numerator is within (ρ [+ 2⁻⁸])·Σp|v| and the
    row sum within ρ·Σp; the quotient (2 ulp approximate division) is within
    err = ((2ρ [+ 2⁻⁸]) / (1 − ρ) + 4u)·Σp|v| / Σp, and the bf16 rounding adds half an ulp at |O| + err.
    A token that sees nothing must be exactly 0 (bound 0).  Returns (ref, tol) [B, W, H, D]."""
    G = case.G
    q64 = q.to(F64)
    k64, v64 = _expand(kd, G), _expand(vd, G)
    sl2 = case.scale * LOG2E
    d = torch.einsum("bwhd,blhd->bwhl", q64, k64) * sl2
    S = torch.einsum("bwhd,blhd->bwhl", q64.abs(), k64.abs()) * sl2
    vmask = vis[:, :, None, :]
    d = d.masked_fill(~vmask, -math.inf)
    m = d.amax(-1, keepdim=True)
    m0 = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    p = torch.exp2(d - m0)                                                         # 0 where invisible
    l = p.sum(-1)
    lz = l.clamp_min(1e-300)
    ref = torch.einsum("bwhl,blhd->bwhd", p, v64) / lz[..., None]
    E = torch.einsum("bwhl,blhd->bwhd", p, v64.abs()) / lz[..., None]
    c = 2 * case.D + 16 if spec else 24
    dd = c * U * S.masked_fill(~vmask, 0).amax(-1)
    delta = (m0 - d).masked_fill(~vmask, 0).amax(-1)
    rho = LN2 * (2 * dd + U * delta) + (n_chain + n_merge) * (U + EX2)
    pb = 2.0 ** -8 if spec else 0.0
    err = ((2 * rho + pb) / (1 - rho) + 4 * U)[..., None] * E
    tol = err + bf16_ulp(ref.abs() + err) / 2
    none = (l == 0)[..., None].expand_as(tol)
    return ref.masked_fill(none, 0), tol.masked_fill(none, 0)


def chain_lengths(case: Case, sms: int, spec: bool):
    """(n_chain, n_merge) of ``ref_and_bound``: the longest split bounds a lane's sequential steps (decode: one step per
    position it reads; spec: two per 16-slot mma k-step of each 64-slot tile plus the rescale); the merges are the warp
    shuffles and the 4-warp merge (decode: 8), the split merge (one per split) and v_scale."""
    splits = case.splits(sms, spec)
    per = max(max(s1 - s0 for s0, s1 in case.ranges(b, sms, spec)) for b in range(case.B))
    return (2 * (per // 16 + per // TILE) + 2 if spec else per), (splits + 4 if spec else splits + 8)


def check_random(case: Case, cache: str, run: Run, device, sms: int, spec: bool, seed: int = 3) -> float:
    """Probe C: every element within its bound, and the bound ≥ 10× tighter than the effect of losing one boosted
    split-edge slot somewhere.  Returns the worst error / bound."""
    q, kc, vc, kd, vd, (ks, vs), boosted = random_inputs(case, cache, device, sms, spec, seed)
    assert boosted, case.name
    vis = case.vis(device)
    n_chain, n_merge = chain_lengths(case, sms, spec)
    ref, tol = ref_and_bound(case, q, kd, vd, vis, spec, n_chain, n_merge)
    vis_drop = vis.clone()
    for b, j in boosted:
        vis_drop[b, :, j] = False
    ref_drop, _ = ref_and_bound(case, q, kd, vd, vis_drop, spec, n_chain, n_merge)
    margin = torch.where(tol > 0, (ref_drop - ref).abs() / tol, torch.zeros_like(tol)).max().item()
    assert margin >= 10, f"{case.name}: losing a split-edge slot moves the reference only {margin:.1f}× the bound"
    out = run(q, kc, vc, case.positions(device), ks, vs)
    assert out.shape == ref.shape and out.dtype == torch.bfloat16
    err = (out.to(F64) - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), (f"{case.name}: {int(bad.sum())} of {bad.numel()} outside the bound; worst err "
                           f"{err.max().item():.3e} at bound {tol.flatten()[err.flatten().argmax()].item():.3e}; first "
                           f"(b, w, h, d) {bad.nonzero()[0].tolist()}")
    return torch.where(tol > 0, err / tol, torch.zeros_like(tol)).max().item()


# ---- run functions --------------------------------------------------------------------------------------------------------
def spec_run(case: Case, torch_path: bool = False) -> Run:
    """``speculation_attention`` (or its torch path) for the case's tree, window and ring."""
    fn = attention.speculation_attention_torch if torch_path else attention.speculation_attention

    def run(q, kc, vc, pos, ks, vs):
        kw = {} if kc.dtype == torch.bfloat16 else {"k_scale": ks, "v_scale": vs}
        return fn(q, kc, vc, pos, case.mask, case.depth, sliding_window=case.window or None, scale=case.scale,
                  rolling=case.rolling, **kw)
    return run


def decode_run(case: Case) -> Run:
    def run(q, kc, vc, pos, ks, vs):
        kw = {} if kc.dtype == torch.bfloat16 else {"k_scale": ks, "v_scale": vs}
        return attention.decode_attention(q, kc, vc, pos, scale=case.scale, sliding_window=case.window or None,
                                          rolling=case.rolling, **kw)
    return run


def partial_run(case: Case) -> Run:
    from neuronx_distributed_b200.modules.attention.flash_decode import _local_partial

    def run(q, kc, vc, pos, ks, vs):
        return _local_partial(q, kc, vc, pos, case.scale, case.window or None, ks, vs)
    return run


def weighted_run(case: Case, weights: torch.Tensor, partial: bool = False) -> Run:
    """A simulated kernel that reads slot c of token w ``weights[b, w, c]`` times (0: skipped, 2: read twice), in float64,
    rounded as the kernels round their output (bf16, or fp32 for the partial)."""
    def run(q, kc, vc, pos, ks, vs):
        kd = kc.to(F64) * (ks if kc.dtype == E4M3 else 1.0)
        vd = vc.to(F64) * (vs if vc.dtype == E4M3 else 1.0)
        k64, v64 = _expand(kd, case.G), _expand(vd, case.G)
        d = torch.einsum("bwhd,blhd->bwhl", q.to(F64), k64) * case.scale
        wt = weights[:, :, None, :].to(F64)
        d = d.masked_fill(wt == 0, -math.inf)
        m = d.amax(-1, keepdim=True)
        m0 = torch.where(torch.isinf(m), torch.zeros_like(m), m)
        p = torch.exp(d - m0) * wt
        o = torch.einsum("bwhl,blhd->bwhd", p, v64)
        l = p.sum(-1)
        if partial:
            return o[:, 0].float(), m[:, 0, :, 0].float(), l[:, 0].float()
        return (o / l.clamp_min(1e-300)[..., None]).to(torch.bfloat16)
    return run


# ---- CPU checks -----------------------------------------------------------------------------------------------------------
SMS = 4                            # a small SM count, so that the small CPU shapes still get several splits

CPU_DECODE = [
    Case("decode", H=4, Hkv=2, D=64, L=300, pos=(0, 1, 77, 299)),
    Case("decode-window", H=4, Hkv=4, D=64, L=300, pos=(5, 150, 299), window=70),
    Case("decode-local-positions", H=2, Hkv=1, D=64, L=256, pos=(-40, -1, 0, 63, 255, 256, 400), window=100),
]
CPU_SPEC = [
    Case("chain", H=4, Hkv=2, D=64, L=256, pos=(0, 100, 251), W=5),
    Case("chain-window", H=4, Hkv=1, D=64, L=256, pos=(3, 200), W=5, window=40),
    Case("medusa-window", H=2, Hkv=2, D=64, L=256, pos=(30, 246), W=10, window=64, tree="medusa"),
    Case("random-tree", H=4, Hkv=2, D=64, L=256, pos=(64, 200), W=12, tree="random"),
    Case("rolling", H=2, Hkv=1, D=64, L=200, pos=(150, 470), W=5, window=196, rolling=True),
    Case("w-times-g-over-64", H=8, Hkv=1, D=64, L=256, pos=(20, 130), W=9),
]


def test_split_rules_at_the_bench_decode_shape():
    """Llama-2-13B at TP = 1, B = 1, a 2048-row cache, positions 1024 … 2047, 132 SMs: 20 splits of 52–103 rows."""
    assert decode_splits(1, 40, 2048, 0, 132) == 20
    lens = {max(s1 - s0 for s0, s1 in decode_ranges(p, 2048, 0, 20, False)) for p in range(1024, 2048)}
    assert min(lens) == 52 and max(lens) == 103
    assert decode_splits(1, 8, 32768, 0, 132) == 64 and decode_splits(128, 8, 1024, 0, 132) == 1
    # the non-empty ranges tile the visible slots with no gap and no overlap
    for p, win, roll in ((0, 0, False), (5, 0, False), (700, 300, False), (20384, 4096, True), (-3, 100, False),
                         (9000, 0, False)):
        case = Case("r", H=1, Hkv=1, D=64, L=8192, pos=(p,), window=win, rolling=roll)
        want = {case.row(c) for c in range(p - (win or p + 1) + 1, p + 1) if c >= 0 and (roll or c < 8192)}
        for s in (1, 7, 64):
            got = [case.row(c) for s0, s1 in decode_ranges(p, 8192, win, s, roll) for c in range(s0, s1)]
            assert len(got) == len(set(got)) and set(got) == want
            assert set(got) == set(case.vis("cpu")[0, 0].nonzero()[:, 0].tolist())


@pytest.mark.parametrize("case", CPU_DECODE, ids=lambda c: c.name)
@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
def test_probes_pass_on_the_local_partial_torch_path(case, cache):
    check_visibility_partial(case, cache, partial_run(case), "cpu")
    check_planted(case, cache, partial_run(case), "cpu", SMS, spec=False, partial=True)


@pytest.mark.parametrize("case", CPU_SPEC + CPU_DECODE[:2], ids=lambda c: c.name)
@pytest.mark.parametrize("cache", ("bf16", "e4m3"))
def test_probes_pass_on_the_speculation_torch_path(case, cache):
    run = spec_run(case, torch_path=True)
    check_visibility(case, cache, run, "cpu")
    check_planted(case, cache, run, "cpu", SMS, spec=case.W > 1)


@pytest.mark.parametrize("case", CPU_SPEC[:1] + CPU_SPEC[4:] + CPU_DECODE[:1], ids=lambda c: c.name)
def test_random_probe_bound_and_margin_on_a_float64_path(case):
    """Probe C against an exact path (float64 with the true visibility): within the bound, far from its 10× margin."""
    spec = case.W > 1
    vis = case.vis("cpu")
    worst = check_random(case, "bf16", weighted_run(case, vis.to(F64)), "cpu", SMS, spec)
    assert worst <= 1.0


MUTATIONS = ("drop", "double", "shift+1", "shift-1", "shift+64", "shift+D", "shift+split")


def mutate(case: Case, vis: torch.Tensor, b: int, j: int, kind: str, sms: int, spec: bool) -> torch.Tensor:
    """Read counts of a kernel that gets slot j of sequence b wrong for every token that sees it."""
    wt = vis.to(F64).clone()
    sees = vis[b, :, j]
    if kind == "drop":
        wt[b, sees, j] = 0
    elif kind == "double":
        wt[b, sees, j] = 2
    else:
        step = {"shift+1": 1, "shift-1": -1, "shift+64": 64, "shift+D": case.D,
                "shift+split": case.split_len(sms, spec)}[kind]
        t = j + step
        if not 0 <= t < case.L:
            t = (t % case.L) if case.rolling else j - step
        wt[b, sees, j] -= 1
        wt[b, sees, t] += 1
    return wt


@pytest.mark.parametrize("case", CPU_SPEC[:1] + CPU_SPEC[2:5] + CPU_DECODE[:2], ids=lambda c: c.name)
def test_probes_reject_wrong_visibility_at_every_planted_edge(case):
    """At every planted edge of sequence 0 (and the last sequence), each mutation is rejected by the visibility probe; a
    lost or shifted slot also by the planted probe (a doubled planted slot still wins its row: that is probe A's case)."""
    spec = case.W > 1
    vis = case.vis("cpu")
    edges = case.edges(SMS, spec, vis)
    checked = 0
    for b in (0, case.B - 1):
        slots = sorted({j for per_w in edges[b] for j in per_w})
        for j in slots:
            for kind in MUTATIONS:
                wt = mutate(case, vis, b, j, kind, SMS, spec)
                if torch.equal(wt, vis.to(F64)):
                    continue                                      # the shift landed on itself (only at tiny L)
                # a normalised output cannot tell a token's only slot read once from read twice (the partial's l can)
                alone = kind == "double" and bool((vis[b, vis[b, :, j]].sum(-1) == 1).all())
                if not alone:
                    with pytest.raises(AssertionError):
                        check_visibility(case, "bf16", weighted_run(case, wt), "cpu")
                if kind != "double":
                    with pytest.raises(AssertionError):
                        check_planted(case, "bf16", weighted_run(case, wt), "cpu", SMS, spec)
                if not spec and not case.rolling:
                    with pytest.raises(AssertionError):
                        check_visibility_partial(case, "e4m3", weighted_run(case, wt, partial=True), "cpu")
                checked += 1
    assert checked >= 20, checked


@pytest.mark.parametrize("case", CPU_SPEC[:1] + CPU_DECODE[:1], ids=lambda c: c.name)
def test_random_probe_rejects_a_lost_split_edge(case):
    """The boosted split-edge slot, lost: the kernel's output leaves the bound."""
    spec = case.W > 1
    _, _, _, _, _, _, boosted = random_inputs(case, "bf16", "cpu", SMS, spec)
    vis = case.vis("cpu")
    wt = vis.to(F64).clone()
    for b, j in boosted:
        wt[b, :, j] = 0
    with pytest.raises(AssertionError, match="outside the bound"):
        check_random(case, "bf16", weighted_run(case, wt), "cpu", SMS, spec)


def test_planted_probe_covers_every_edge():
    """Over its launches the planted probe plants every edge of every token at least once."""
    case = CPU_SPEC[2]
    vis = case.vis("cpu")
    edges = case.edges(SMS, True, vis)
    seen = set()
    for grp, rnd in planted_launches(case, edges):
        *_, pk, _ = planted_inputs(case, "bf16", edges, grp, rnd, "cpu")
        seen |= {(b, w, j) for b, w, _, j in pk.tolist()}
    want = {(b, w, j) for b in range(case.B) for w in range(case.W) for j in edges[b][w]}
    assert want <= seen
