"""Row arg-max and top-k selection kernels (``csrc/select.cu`` through ``ops.select`` and the distributed ``operators``) against
a stable CPU oracle on torch's rule:
- descending order, NaN above +inf, -0 equal to +0;
- among equal values the smaller index first (a stable descending sort; ``torch.topk`` leaves that order open, so it is not
  the oracle);
- top-k returns k distinct indices and values ``x[idx]`` in fp32, ``-inf`` included; the arg-max of an all ``-inf`` row is
  index 0 (+ offset) with value ``-inf``.
Selection does no arithmetic, so every check is bit-exact on indices and on value bits (any NaN matches any NaN).

The rows are the ones that break a kernel using a finite number as "nothing yet" / "already taken": all ``-inf``, fewer
finite entries than k, the dtype's own extremes and infinities, a NaN, signed zeros, ties everywhere.  They are taken as
slices of a wider tensor (row stride not V, row starts unaligned) and at every vocab width the kernels serve, from one
element to the 51 200-element top-k limit and past it.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
# 128256/8 = 16032 (Llama-3 at TP 8), 151936/4 = 37984 (Qwen2 at TP 4), 51200 = the top-k kernel's limit (V * 4 B = 200 KiB)
V_TOPK = [1, 7, 8, 1001, 4000, 16032, 32000, 32016, 37984, 50257, 51200]
V_ARGMAX_ONLY = [51201, 128256, 152064]          # 51201: top-k falls back to torch, arg-max stays on the kernel
KS = (1, 2, 8, 50, 127, 128)
KINDS = ("randn", "grid", "equal", "all_neg_inf", "few_finite", "extremes", "nan", "signed_zeros")
OFFSET = 12345


@pytest.fixture(scope="module", autouse=True)
def _ext():
    from neuronx_distributed_b200 import ops

    assert ops.extension_available(), ops._ext.load_error()
    return ops._ext


def _row(kind: str, V: int, dtype, g: torch.Generator) -> torch.Tensor:
    """One fp32 row of ``kind`` whose values are exact in ``dtype``."""
    inf = float("inf")
    if kind == "randn":
        r = torch.randn(V, generator=g)
    elif kind == "grid":                                     # 13 distinct values: ties everywhere
        r = torch.randint(-6, 7, (V,), generator=g).float() * 0.25
    elif kind == "equal":
        r = torch.full((V,), 0.75)
    elif kind == "all_neg_inf":
        r = torch.full((V,), -inf)
    elif kind == "few_finite":                               # fewer finite entries than most k: then -inf in index order
        r = torch.full((V,), -inf)
        pos = torch.randperm(V, generator=g)[:min(V - 1, 5)]
        r[pos] = torch.randn(len(pos), generator=g)
    elif kind == "extremes":                                 # the dtype's own lowest / highest finite values and both infinities
        fi = torch.finfo(dtype)
        r = torch.randn(V, generator=g)
        pick = torch.randint(0, 6, (V,), generator=g)
        r = torch.where(pick == 0, torch.full_like(r, fi.min), r)
        r = torch.where(pick == 1, torch.full_like(r, -inf), r)
        if V > 2:
            r[torch.randint(0, V, (1,), generator=g)] = fi.max
            r[torch.randint(0, V, (1,), generator=g)] = inf
    elif kind == "nan":                                      # one NaN (sign bit set on half the rows): it ranks first
        r = torch.randn(V, generator=g)
        r[torch.randint(0, V, (1,), generator=g)] = float("nan") * (1 if torch.rand(1, generator=g).item() < 0.5 else -1)
    elif kind == "signed_zeros":                             # -0 and +0 tie: the smaller index wins whatever the sign
        r = torch.zeros(V)
        r[torch.rand(V, generator=g) < 0.5] = -0.0
        r[torch.rand(V, generator=g) < 0.1] = -1.0
    else:
        raise ValueError(kind)
    return r.to(dtype).float()


def _batch(kinds, V: int, dtype, g: torch.Generator, strided: bool) -> torch.Tensor:
    """[len(kinds), V] on the GPU; ``strided``: a column slice of a wider tensor (row stride V + 5, rows start at element 1)."""
    rows = torch.stack([_row(k, V, dtype, g) for k in kinds]).to(dtype)
    if not strided:
        return rows.cuda()
    wide = torch.zeros(len(kinds), V + 5, dtype=dtype, device="cuda")
    x = wide[:, 1:V + 1]
    x.copy_(rows.cuda())
    assert x.stride() == (V + 5, 1) and not x.is_contiguous()
    return x


def _oracle(x: torch.Tensor):
    """Stable descending sort of every row: (values fp32 [R, V], indices int64 [R, V])."""
    xf = x.float().cpu()
    _, idx = torch.sort(xf.double(), dim=-1, descending=True, stable=True)
    return xf.gather(1, idx), idx


def _same_bits(got: torch.Tensor, want: torch.Tensor, what: str):
    got = got.cpu()
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, got.shape, want.shape)
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), f"{what}: NaN at {gn.nonzero().tolist()[:4]}, expected at {wn.nonzero().tolist()[:4]}"
    bits = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}[got.dtype]
    diff = got.view(bits) != want.view(bits)
    diff &= ~gn
    assert not diff.any(), f"{what}: {int(diff.sum())} values differ, first {diff.nonzero().tolist()[:4]}"


def _same_idx(got: torch.Tensor, want: torch.Tensor, what: str):
    got = got.cpu()
    assert got.dtype == torch.int64 and torch.equal(got, want), \
        f"{what}: {int((got != want).sum())} indices differ, got {got.flatten()[:8].tolist()} want {want.flatten()[:8].tolist()}"


def _cases(V: int, dtype, g: torch.Generator):
    """(name, x, index_offset): every kind as 1 contiguous row and as 3 strided rows, plus 64 strided rows cycling the kinds."""
    for kind in KINDS:
        yield f"{kind} rows=1", _batch([kind], V, dtype, g, strided=False), 0
        yield f"{kind} rows=3 strided", _batch([kind] * 3, V, dtype, g, strided=True), OFFSET
    yield "mixed rows=64 strided", _batch([KINDS[i % len(KINDS)] for i in range(64)], V, dtype, g, strided=True), OFFSET


@pytest.mark.parametrize("V", V_TOPK + V_ARGMAX_ONLY)
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
def test_row_argmax_and_topk_follow_the_stable_rule(_ext, dtype, V):
    from neuronx_distributed_b200.ops import select

    g = torch.Generator().manual_seed(V * 7 + DTYPES.index(dtype))
    ks = sorted({k for k in KS if k <= V} | ({V} if V <= 128 else set()))
    topk_kernel = V <= 51200
    assert bool(_ext.ext().row_topk_supported(V, 1)) == topk_kernel
    for name, x, off in _cases(V, dtype, g):
        what = f"{dtype} V={V} {name} offset={off}"
        ov, oi = _oracle(x)
        n = _ext.launches()
        v, i = select.row_max(x, index_offset=off)
        assert _ext.launches() == n + 1, f"{what}: arg-max did not run on the kernel"
        torch.cuda.synchronize()
        _same_idx(i, oi[:, 0] + off, f"{what} arg-max index")
        _same_bits(v, ov[:, 0], f"{what} arg-max value")
        for k in ks:
            n = _ext.launches()
            tv, ti = select.row_topk(x, k, index_offset=off)
            torch.cuda.synchronize()
            if not topk_kernel:                              # torch.topk: same values, some order of equal ones
                assert _ext.launches() == n, f"{what}: top-k past the kernel's limit must take torch"
                if name.startswith(("randn", "grid")):
                    _same_bits(tv, ov[:, :k], f"{what} top-{k} values (torch fallback)")
                    assert all(len(set(r)) == k for r in ti.tolist())
                continue
            assert _ext.launches() == n + 1, f"{what}: top-{k} did not run on the kernel"
            _same_idx(ti, oi[:, :k] + off, f"{what} top-{k} indices")
            _same_bits(tv, ov[:, :k], f"{what} top-{k} values")


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
def test_adversarial_rows_spelled_out(_ext, dtype):
    """The defects a finite sentinel causes, written as literal rows: already-chosen indices returned again on a row with
    fewer finite entries than k, a finite stand-in for -inf, NaN never chosen."""
    from neuronx_distributed_b200.ops import select

    inf, nan = float("inf"), float("nan")
    x = torch.tensor([[5.0, -inf, -inf]], dtype=dtype, device="cuda")
    tv, ti = select.row_topk(x, 3)
    assert ti.tolist() == [[0, 1, 2]] and tv.tolist() == [[5.0, -inf, -inf]], (ti, tv)
    x = torch.full((2, 1001), -inf, dtype=dtype, device="cuda")
    v, i = select.row_max(x, index_offset=40)
    assert i.tolist() == [40, 40] and v.tolist() == [-inf, -inf], (i, v)
    x = torch.tensor([[1.0, nan, inf, nan, 2.0]], dtype=dtype, device="cuda")
    v, i = select.row_max(x)
    assert i.tolist() == [1] and torch.isnan(v).all(), (i, v)
    tv, ti = select.row_topk(x, 5)
    assert ti.tolist() == [[1, 3, 2, 4, 0]], ti


def _one_rank_model_parallel():
    import torch.distributed as dist

    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29544")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    if not ps.model_parallel_is_initialized():
        ps.initialize_model_parallel(1)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
def test_distributed_operators_at_world_size_one(_ext, dtype):
    """``operators.topk`` / ``operators.argmax`` on the last dim of a CUDA tensor run the kernels; at world size 1 they return
    the oracle's result (top-k values in the input dtype)."""
    from neuronx_distributed_b200 import operators

    _one_rank_model_parallel()
    g = torch.Generator().manual_seed(11)
    for V in (7, 32016):
        x = _batch([KINDS[i % len(KINDS)] for i in range(16)], V, dtype, g, strided=True)
        ov, oi = _oracle(x)
        n = _ext.launches()
        i = operators.argmax(x, dim=-1)
        _same_idx(i, oi[:, 0], f"{dtype} V={V} operators.argmax")
        i = operators.argmax(x, -1, keepdim=True)
        _same_idx(i, oi[:, :1], f"{dtype} V={V} operators.argmax keepdim")
        for k in (1, 5, 50):
            k = min(k, V)
            tv, ti = operators.topk(x, k, dim=-1)
            _same_idx(ti, oi[:, :k], f"{dtype} V={V} operators.topk k={k}")
            _same_bits(tv, ov[:, :k].to(dtype), f"{dtype} V={V} operators.topk k={k} values")
        assert _ext.launches() > n, "the operators did not reach the selection kernels"
