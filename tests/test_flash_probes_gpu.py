"""The flash attention training kernels on the H100 (sm_90a), pair by pair: ``fa_fwd_kernel``, ``fa_bwd_prep_kernel``,
``fa_bwd_dkdv_kernel`` and ``fa_bwd_dq_kernel`` (``csrc/attention_sm90.cu``) at every head size, with and without the
key-padding mask, the sliding window (with context-parallel query offsets) and dropout, at real-model shapes and at the tile
edges.  The probes — exact visibility of every pair, planted keys and float64 with per-element bounds — and their
derivations are in ``test_flash_probes_cpu.py``.  Kernels are called through ``ops._ext.ext().flash_attn_fwd`` /
``flash_attn_bwd`` on ``attention._tma_view`` views, as the autograd front end calls them; the front end itself is checked
bit for bit against those calls with its launch count."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_flash_probes_cpu import (N_CODES, Case, Kernels, check_bwd_visibility, check_dlse,  # noqa: E402
                                   check_fwd_visibility, check_planted, check_random)

pytestmark = pytest.mark.gpu

DIMS = (64, 80, 96, 128)


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _layout(case: Case, q, k, v):
    """Logical [B, S, H, D] tensors → the case's memory layout (same values)."""
    if case.layout == "sbhd":
        return tuple(x.transpose(0, 1).contiguous().transpose(0, 1) for x in (q, k, v))
    if case.layout == "fused":
        assert case.S_q == case.S_kv
        H, Hkv = case.H, case.Hkv
        f = torch.empty(case.S_q, case.B, H + 2 * Hkv, case.D, dtype=q.dtype, device=q.device)
        f[:, :, :H] = q.transpose(0, 1)
        f[:, :, H:H + Hkv] = k.transpose(0, 1)
        f[:, :, H + Hkv:] = v.transpose(0, 1)
        return f[:, :, :H].transpose(0, 1), f[:, :, H:H + Hkv].transpose(0, 1), f[:, :, H + Hkv:].transpose(0, 1)
    return q, k, v


def _seed(case: Case, device):
    return torch.tensor([case.seed], dtype=torch.int64, device=device) if case.dropout else None


def cuda_kernels(record=None) -> Kernels:
    """The extension's forward and backward, called as ``ops.attention`` calls them; ``record`` collects the
    (kernel, HD, MASK, WINDOW, DROPOUT) instantiations launched."""
    from neuronx_distributed_b200.ops import _ext, attention

    e = _ext.ext()
    tv = attention._tma_view

    def fwd(case, q, k, v, mask, scale):
        q, k, v = _layout(case, q, k, v)
        o, lse = e.flash_attn_fwd(tv(q), tv(k), tv(v), case.causal, float(scale), case.sbhd_out, mask, case.window,
                                  case.q_offset, case.dropout, _seed(case, q.device), case.head_offset)
        assert o.is_cuda and o.shape == q.shape and lse.shape == (case.B, case.H, case.S_q)
        if record is not None:
            record.add(("fwd",) + case.instantiation())
        return o, lse

    def bwd(case, go, q, k, v, o, lse, dlse, mask, scale):
        q, k, v = _layout(case, q, k, v)
        dq, dk, dv = e.flash_attn_bwd(tv(go), tv(q), tv(k), tv(v), tv(o), lse.contiguous(), case.causal, float(scale),
                                      case.sbhd_out, dlse, mask, case.window, case.q_offset, case.dropout,
                                      _seed(case, q.device), case.head_offset)
        if record is not None:
            record.add(("dkdv",) + case.instantiation())
            record.add(("dq",) + case.instantiation())
        return dq, dk, dv
    return Kernels(fwd, bwd)


# ---- cases ----------------------------------------------------------------------------------------------------------------
MODELS = [
    # Llama-2-7B, the bench's training shape
    Case("llama2-7b", B=1, S_q=4096, S_kv=4096, H=32, Hkv=32, D=128, causal=True),
    # Llama-3-8B (GQA 4) at 8k; Llama-3-70B per TP = 8 rank (G = 8)
    Case("llama3-8b", B=1, S_q=8192, S_kv=8192, H=32, Hkv=8, D=128, causal=True),
    Case("llama3-70b-tp8", B=1, S_q=4096, S_kv=4096, H=8, Hkv=1, D=128, causal=True, layout="sbhd", sbhd_out=True),
    # Mistral-7B: W = 4096 at S = 8192
    Case("mistral-7b-w4096", B=1, S_q=8192, S_kv=8192, H=32, Hkv=8, D=128, causal=True, window=4096),
    # context-parallel off-diagonal blocks of a 32k Mistral sequence: zig-zag cp = 4 (chunks of 4096, offsets 4096 and
    # 12288 — the latter past the window: every row sees nothing), contiguous cp = 2 (chunks of 16384, offset 16384)
    Case("cp4-zigzag-off4096", B=1, S_q=4096, S_kv=4096, H=32, Hkv=8, D=128, causal=True, window=4096, q_offset=4096),
    Case("cp4-zigzag-off12288", B=1, S_q=4096, S_kv=4096, H=8, Hkv=8, D=128, causal=True, window=4096, q_offset=12288),
    Case("cp2-contig-off16384", B=1, S_q=16384, S_kv=16384, H=8, Hkv=2, D=128, causal=True, window=4096, q_offset=16384),
    # BERT-large: right padding at every tile edge, left padding, a random mask
    Case("bert-large-right", B=9, S_q=512, S_kv=512, H=16, Hkv=16, D=64, lens=(512, 511, 449, 257, 129, 65, 64, 63, 1)),
    Case("bert-large-left", B=8, S_q=512, S_kv=512, H=16, Hkv=16, D=64, left=(0, 1, 63, 64, 65, 128, 300, 511)),
    Case("bert-large-random", B=8, S_q=512, S_kv=512, H=16, Hkv=16, D=64, rand=0.6, layout="sbhd"),
    Case("vit-b16", B=2, S_q=197, S_kv=197, H=12, Hkv=12, D=64, layout="fused"),
    Case("neox-20b-tp8", B=1, S_q=2048, S_kv=2048, H=8, Hkv=8, D=96, causal=True, layout="fused", sbhd_out=True),
    Case("pythia-2.8b", B=1, S_q=2048, S_kv=2048, H=32, Hkv=32, D=80, causal=True, layout="sbhd"),
    Case("phi3-mini", B=1, S_q=4096, S_kv=4096, H=32, Hkv=32, D=96, causal=True),
]
LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257)
EDGES = [Case(f"causal-s{S}", B=2, S_q=S, S_kv=S, H=2, Hkv=1, D=64, causal=True) for S in LENGTHS]
EDGES += [Case(f"cross-{a}x{b}", B=2, S_q=a, S_kv=b, H=4, Hkv=2, D=128, rand=0.8 if a > b else 0.0)
          for a, b in ((1, 257), (257, 1), (63, 129), (129, 63), (65, 192), (192, 65), (127, 193), (193, 127), (2, 64),
                       (64, 2), (128, 191), (191, 128))]
# windows at the tile edges, with offsets ≡ 0, 1, 63 (mod 64) and past S
EDGES += [Case(f"window-w{W}-off{off}", B=1, S_q=257, S_kv=257, H=2, Hkv=1, D=64 if W % 2 else 96, causal=True, window=W,
               q_offset=off)
          for W in (1, 2, 63, 64, 65, 127, 128, 129, 257) for off in (0, 1, 63, 257 + 64)]
EDGES += [Case(f"window-full-off{off}", B=1, S_q=193, S_kv=193, H=2, Hkv=2, D=80, causal=True, window=193 + off,
               q_offset=off) for off in (1, 63, 65)]
# every (HD, MASK, WINDOW, DROPOUT) instantiation, GQA 2, ragged S
GRID = [Case(f"grid-d{D}" + ("-mask" if mk else "") + ("-w65-off63" if wd else "") + ("-p0.5" if dr else ""),
             B=2, S_q=300, S_kv=300, H=4, Hkv=2, D=D, causal=wd or D in (64, 96), window=65 if wd else 0,
             q_offset=63 if wd else 0, left=(0, 37) if mk and wd else None, rand=0.8 if mk and not wd else 0.0,
             dropout=0.5 if dr else 0.0, head_offset=3 if dr else 0, layout="sbhd" if D == 80 else "bshd",
             sbhd_out=D == 96)
        for D in DIMS for mk in (False, True) for wd in (False, True) for dr in (False, True)]
PROBED = MODELS + EDGES + GRID


def _id(c):
    return c.name


def _sync():
    torch.cuda.synchronize()


RECORD = set()


@pytest.mark.parametrize("case", PROBED, ids=_id)
def test_visibility_probe(case):
    """Probe A: every (query, key) pair, exactly, in the forward (and its LSE), the dK/dV kernel and the dQ kernel."""
    k = cuda_kernels(RECORD)
    check_fwd_visibility(case, k, "cuda")
    check_bwd_visibility(case, k, "cuda")
    _sync()


@pytest.mark.parametrize("case", [c for c in PROBED if c.masked or c.window or c.S_q <= 65 or c.name == "llama3-8b"],
                         ids=_id)
def test_dlse_probe(case):
    check_dlse(case, cuda_kernels(RECORD), "cuda")
    _sync()


@pytest.mark.parametrize("case", [c for c in PROBED if not c.dropout and c.S_kv <= N_CODES], ids=_id)
def test_planted_probe(case):
    check_planted(case, cuda_kernels(RECORD), "cuda")
    _sync()


def test_every_instantiation_is_probed_exactly():
    """All 96 (kernel, HD, MASK, WINDOW, DROPOUT) instantiations run the exact visibility probe: the table of what the
    cases of ``test_visibility_probe`` launch (each runs the forward and the backward, i.e. the dK/dV and dQ kernels),
    which ``cuda_kernels`` also records as the probes run."""
    want = {(kern, D, mk, wd, dr) for kern in ("fwd", "dkdv", "dq") for D in DIMS for mk in (False, True)
            for wd in (False, True) for dr in (False, True)}
    table = {(kern,) + c.instantiation() for c in PROBED for kern in ("fwd", "dkdv", "dq")}
    assert len(want) == 96 and want <= table, sorted(want - table)
    assert RECORD <= table


# ---- C. random inputs against float64 (a reduced head count at long S; the full H runs in the exact probes) ---------------
RANDOM = [
    Case("llama2-7b-h2", B=1, S_q=4096, S_kv=4096, H=2, Hkv=2, D=128, causal=True),
    Case("llama3-8b-g4", B=1, S_q=8192, S_kv=8192, H=4, Hkv=1, D=128, causal=True),
    Case("llama3-70b-tp8-g8", B=1, S_q=2048, S_kv=2048, H=8, Hkv=1, D=128, causal=True, layout="sbhd", sbhd_out=True),
    Case("mistral-7b-w4096-h2", B=1, S_q=8192, S_kv=8192, H=2, Hkv=1, D=128, causal=True, window=4096),
    Case("cp4-zigzag-off4096-h2", B=1, S_q=4096, S_kv=4096, H=2, Hkv=1, D=128, causal=True, window=4096, q_offset=4096),
    Case("bert-large-right-h2", B=9, S_q=512, S_kv=512, H=2, Hkv=2, D=64, lens=(512, 511, 449, 257, 129, 65, 64, 63, 1)),
    Case("vit-b16", B=2, S_q=197, S_kv=197, H=12, Hkv=12, D=64, layout="fused"),
    Case("neox-20b-tp8-h2", B=1, S_q=2048, S_kv=2048, H=2, Hkv=2, D=96, causal=True, layout="fused"),
    Case("pythia-2.8b-h2", B=1, S_q=2048, S_kv=2048, H=2, Hkv=2, D=80, causal=True, layout="sbhd"),
    Case("phi3-mini-h2", B=1, S_q=4096, S_kv=4096, H=2, Hkv=2, D=96, causal=True),
    Case("window-w63-off1", B=1, S_q=257, S_kv=257, H=2, Hkv=1, D=64, causal=True, window=63, q_offset=1),
] + [c for c in GRID if c.dropout or c.masked]


@pytest.mark.parametrize("case", RANDOM, ids=_id)
def test_random_vs_float64(case):
    worst = check_random(case, cuda_kernels(RECORD), "cuda")
    print(case.name, " ".join(f"{n}={w:.3f}" for n, w in worst.items()))
    _sync()


# ---- D. bytes the kernels must not read -----------------------------------------------------------------------------------
def _nan_view(x: torch.Tensor) -> torch.Tensor:
    """x [B, S, h, D] as a view into a NaN buffer [B, S + 64, h + 1, 128 (D < 128) or D]: rows ≥ S, columns D … 127 of
    a wider row and a neighbouring head hold NaN."""
    B, S, h, D = x.shape
    buf = torch.full((B, S + 64, h + 1, 128 if D < 128 else D), float("nan"), dtype=x.dtype, device=x.device)
    buf[:, :S, :h, :D] = x
    return buf[:, :S, :h, :D]


def _nan_fused(q, k, v):
    """q, k, v as slices of one NaN fused-QKV buffer [S + 64, B, H + 1 + Hkv + 1 + Hkv + 1, D]: a NaN head between and
    after them, and NaN rows past S."""
    B, S, H, D = q.shape
    Hkv = k.shape[2]
    f = torch.full((S + 64, B, H + 2 * Hkv + 3, D), float("nan"), dtype=q.dtype, device=q.device)
    f[:S, :, :H] = q.transpose(0, 1)
    f[:S, :, H + 1:H + 1 + Hkv] = k.transpose(0, 1)
    f[:S, :, H + 2 + Hkv:H + 2 + 2 * Hkv] = v.transpose(0, 1)
    return (f[:S, :, :H].transpose(0, 1), f[:S, :, H + 1:H + 1 + Hkv].transpose(0, 1),
            f[:S, :, H + 2 + Hkv:H + 2 + 2 * Hkv].transpose(0, 1))


NAN_CASES = [Case(f"nan-d{D}-{kind}", B=2, S_q=200, S_kv=200, H=4, Hkv=2, D=D, causal=kind != "mask",
                  window=65 if kind == "window" else 0, q_offset=1 if kind == "window" else 0,
                  lens=(200, 131) if kind != "causal" else None)
             for D in DIMS for kind in ("mask", "causal", "window")]


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("case", NAN_CASES, ids=_id)
def test_unused_bytes_are_not_read(case, fused):
    """Views whose unused bytes hold NaN (rows past S, columns D … 127 of a wider row, a neighbouring head, fused-QKV
    slices) and mask flags past S_kv set to 1: O, LSE, dQ, dK, dV bit-identical to a run on clean contiguous copies."""
    from neuronx_distributed_b200.ops import _ext

    e = _ext.ext()
    g = torch.Generator(device="cuda").manual_seed(case.D)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()         # noqa: E731
    q, k, v, go = (rn(case.B, case.S_q, case.H, case.D), rn(case.B, case.S_kv, case.Hkv, case.D),
                   rn(case.B, case.S_kv, case.Hkv, case.D), rn(case.B, case.S_q, case.H, case.D))
    mask = case.mask("cuda")
    args = (case.causal, case.scale, False)
    tail = dict(window=case.window, q_offset=case.q_offset)
    o, lse = e.flash_attn_fwd(q, k, v, *args, mask, **tail)
    dq, dk, dv = e.flash_attn_bwd(go, q, k, v, o, lse, *args, None, mask, **tail)
    if fused:
        qn, kn, vn = _nan_fused(q, k, v)
    else:
        qn, kn, vn = _nan_view(q), _nan_view(k), _nan_view(v)
    gon, on = _nan_view(go), _nan_view(o)
    mn = None
    if mask is not None:
        mb = torch.ones(case.B, case.S_kv + 64, dtype=torch.uint8, device="cuda")
        mb[:, :case.S_kv] = mask
        mn = mb[:, :case.S_kv]
    o2, lse2 = e.flash_attn_fwd(qn, kn, vn, *args, mn, **tail)
    dq2, dk2, dv2 = e.flash_attn_bwd(gon, qn, kn, vn, on, lse, *args, None, mn, **tail)
    for name, a, b in (("o", o, o2), ("lse", lse, lse2), ("dq", dq, dq2), ("dk", dk, dk2), ("dv", dv, dv2)):
        assert torch.equal(a, b), (case.name, name)


# ---- the autograd front end: same kernels, counted launches ---------------------------------------------------------------
@pytest.mark.parametrize("case", [MODELS[7], next(c for c in GRID if c.name == "grid-d128-mask-p0.5"), Case("llama-s1024", B=1, S_q=1024, S_kv=1024, H=8, Hkv=2, D=128,
                                                             causal=True, window=300)], ids=_id)
def test_front_end_runs_the_probed_kernels(_ext, case):
    """``ops.attention.flash_attention`` forward + backward launches the flash kernels (4 launches) and gives exactly what
    the direct calls the probes use give."""
    from neuronx_distributed_b200.ops import attention

    q, k, v, go = (torch.randn(case.B, S, h, case.D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(s))
                   .bfloat16() for s, (S, h) in enumerate(((case.S_q, case.H), (case.S_kv, case.Hkv), (case.S_kv, case.Hkv),
                                                           (case.S_q, case.H))))
    mask = case.mask("cuda")
    qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))
    n0 = _ext.launches()
    o = attention.flash_attention(qg, kg, vg, causal=case.causal, key_padding_mask=None if mask is None else mask.bool(),
                                  sliding_window=case.window or None, dropout_p=case.dropout,
                                  dropout_seed=_seed(case, "cuda"), head_offset=case.head_offset)
    o.backward(go)
    assert _ext.launches() == n0 + 4, "the flash kernels did not run"
    c = Case(**{**case.__dict__, "sbhd_out": True, "layout": "bshd"})
    kern = cuda_kernels()
    ro, rlse = kern.fwd(c, q, k, v, mask, c.scale)
    rdq, rdk, rdv = kern.bwd(c, go, q, k, v, ro, rlse, None, mask, c.scale)
    for a, b in ((o, ro), (qg.grad, rdq), (kg.grad, rdk), (vg.grad, rdv)):
        assert torch.equal(a, b)
