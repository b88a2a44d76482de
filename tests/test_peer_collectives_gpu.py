"""The peer-memory collectives on one GPU, element by element: the ZeRO-1 reduce-scatter and all-gather
(``csrc/zero1_comm.cu``), the one-shot all-reduce (``csrc/allreduce.cu``), the NVLS-layout collectives
(``csrc/nvls_coll.cu``) and the ZeRO-1 optimizer on top of them.

Two to four processes share ``cuda:0`` (``run_distributed(..., use_cuda="loopback")``): the control plane is gloo and the
kernels run their real flag / epoch protocols between the processes' contexts.  There is no multicast mapping between
contexts of one device, so the NVLS kernels take their unicast branch.  Every rank rebuilds every rank's inputs from seeds
and computes its references locally:

* an fp32 emulation in the kernel's own summation order, for bit-exact checks.  Every sum in these kernels is fp32 in a
  fixed order and rounded once: ``p = 0 .. world-1`` in the one-shot all-reduce and the unicast NVLS kernels,
  ``(rank + p) % world`` then ``* scale`` in the ZeRO-1 reduce-scatter.  The NVLS all-reduce with a residual rounds the sum
  to the storage type, then adds the residual in fp32 and rounds again.
* float64, for the bounds.

The kernels are built with ``--use_fast_math`` (flush-to-zero): the bit-exact inputs and all partial sums are normal
numbers, and one case pins that a subnormal gradient is flushed.  Order matters only when the fp32 sums round, so the
inputs spread over many binades, and ranks of one world make the same calls so that they compare results over gloo
only after all of them have run their kernels.
"""
import contextlib
import math

import pytest
import torch

from dist_utils import FLT_MIN, _bits, _Checks, _emulate, _randn, _same, run_distributed

pytestmark = pytest.mark.gpu

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
U = 2.0 ** -24                                  # fp32 unit roundoff


# =====================================================================================================================
# shared helpers: inputs from seeds, emulation in a given order, NaN guard fills, cross-rank comparison
# =====================================================================================================================
def _nan_filled(n, dtype=F32):
    return torch.full((n,), float("nan"), dtype=dtype, device="cuda")


def _gather_cpu(t):
    import torch.distributed as dist

    every = [None] * dist.get_world_size()
    dist.all_gather_object(every, t.detach().cpu())
    return every


def _rank_identical(chk, t, what):
    """``t`` is bit-identical on every rank (NaN as NaN)."""
    every = _gather_cpu(t)
    for r, o in enumerate(every):
        chk.true(_same(o, every[0]), f"{what}: rank {r} differs from rank 0")


def _f32(x):
    """The fp32 value a launcher receives for the Python float ``x``."""
    return float(torch.tensor(x, dtype=F32))


# =====================================================================================================================
# ZeRO-1 reduce-scatter and all-gather
# =====================================================================================================================
_RAGGED_BF16 = [1, 7, 129, 4099, 128 * 1000, 3001, 65541]          # bf16 parameters and bf16 gradients
_RAGGED_F32 = [33, 1000, 8191, 257, 50000]                         # fp32 parameters and fp32 gradients
# one decoder layer of Llama-2-7B at TP 8: input norm, q/k/v/o [4096/8 x 4096], gate/up/down [11008/8 x 4096], post norm
_LLAMA7B_TP8_LAYER = [4096, 512 * 4096, 512 * 4096, 512 * 4096, 4096 * 512, 1376 * 4096, 1376 * 4096, 4096 * 1376, 4096]
_SUBNORMAL = {BF16: 2.0 ** -130, F32: 1e-40}                      # both below FLT_MIN, exactly representable


def _arena_bytes(layouts, world):
    """An upper bound of what the _FlatGroups of ``layouts`` [(numels, param dtype, grad dtype)] take in one arena."""
    from neuronx_distributed_b200.optimizer.zero_redundancy_optimizer import _ALIGN

    total = 0
    for numels, pdt, gdt in layouts:
        n = sum((k + _ALIGN - 1) // _ALIGN * _ALIGN for k in numels) + world * _ALIGN
        total += n * (torch.empty((), dtype=pdt).element_size() + torch.empty((), dtype=gdt).element_size()) + 1024
    return total


def _flat_groups(arena, layouts, world, rank):
    from neuronx_distributed_b200.optimizer.zero_redundancy_optimizer import _FlatGroup

    fgs = []
    for gi, (numels, pdt, gdt) in enumerate(layouts):
        params = [torch.nn.Parameter(torch.zeros(k, dtype=pdt, device="cuda")) for k in numels]
        fgs.append(_FlatGroup(params, gi, world, rank, gdt, F32, pdt != F32, arena))
    return fgs


def _grads(fg, call, world, sub_pins):
    """Every rank's whole flat gradient buffer for ``call``; at ``sub_pins`` every rank holds a positive subnormal."""
    gdt = fg.grad_flat.dtype
    gs = [_randn(fg.total, 7919 * call + 31 * r + 1, gdt) for r in range(world)]
    for g in gs:
        g[sub_pins] = _SUBNORMAL[gdt]
    return gs


def _window(fg, rank, bucket):
    """``(sub_begin, sub_len)`` of this rank's shard inside the flat range ``bucket`` — what the overlapped optimizer passes."""
    if bucket is None:
        return 0, fg.shard_numel
    lo, hi = fg.shard_range
    a, b = max(bucket[0], lo), min(bucket[1], hi)
    return (a - lo, b - a) if a < b else (0, 0)


def _reduce_scatter_sequence(chk, arena, fgs, rank, world):
    """Back-to-back reduce-scatters on two flat groups that share the arena's epoch and completion counter.  After each call,
    on the same stream, this rank overwrites the gradient buffer the call read with the values of the next call on that
    group: a peer that still reads it (an exit barrier that lets a rank go early) sees the wrong values."""
    import torch.distributed as dist

    scales = {0: 1.0 / world, 1: 1.0 / 12.5}                  # 1/dp, and an explicit grad_scale_divisor of 12.5
    seq = []                                                   # (group, bucket or None, max_ctas)
    seq += [(0, None, 0), (1, None, 1), (0, None, 16), (1, None, 0)]
    cuts = {}
    for gi, fg in enumerate(fgs):
        c = sorted({0, fg.total} | {int(fg.total * f) // 8 * 8 for f in (0.13, 0.37, 0.52, 0.81)})
        cuts[gi] = list(zip(c[:-1], c[1:]))
    for k in range(max(len(b) for b in cuts.values())):       # bucket windows, the two groups interleaved
        for gi in (0, 1):
            if k < len(cuts[gi]):
                seq.append((gi, cuts[gi][k], (1, 16, 0)[k % 3]))
    pins = {gi: torch.tensor([r * fg.shard_numel + 8 for r in range(world)], device="cuda") for gi, fg in enumerate(fgs)}
    inputs = [_grads(fgs[gi], i, world, pins[gi]) for i, (gi, _, _) in enumerate(seq)]
    outs, snaps = [], []
    for gi in (0, 1):                                          # the first call on each group sees its values
        first = next(i for i, s in enumerate(seq) if s[0] == gi)
        fgs[gi].grad_flat.copy_(inputs[first][rank])
    torch.cuda.synchronize()
    dist.barrier()
    for i, (gi, bucket, ctas) in enumerate(seq):
        fg = fgs[gi]
        sb, sl = _window(fg, rank, bucket)
        out = _nan_filled(fg.shard_numel)
        arena.reduce_scatter(fg.grad_off, fg.grad_flat.dtype, fg.shard_numel, scales[gi], out, gi, sub_begin=sb, sub_len=sl,
                             max_ctas=ctas)
        snaps.append(fg.grad_flat.clone())
        nxt = next((j for j in range(i + 1, len(seq)) if seq[j][0] == gi), None)
        if nxt is not None:
            fg.grad_flat.copy_(inputs[nxt][rank])
        outs.append((out, sb, sl))
    torch.cuda.synchronize()
    for i, ((gi, bucket, ctas), (out, sb, sl)) in enumerate(zip(seq, outs)):
        fg = fgs[gi]
        what = f"reduce-scatter call {i} (group {gi}, {fg.grad_flat.dtype}, bucket {bucket}, max_ctas {ctas})"
        lo, hi = fg.shard_range
        parts = [g[lo:hi] for g in inputs[i]]
        s32 = _f32(scales[gi])
        want = _emulate(parts, [(rank + p) % world for p in range(world)]) * torch.tensor(s32, dtype=F32, device="cuda")
        chk.same(out[sb:sb + sl], want[sb:sb + sl], what + ": vs the fp32 (rank + p) % world emulation")
        outside = torch.ones(fg.shard_numel, dtype=torch.bool, device="cuda")
        outside[sb:sb + sl] = False
        chk.true(bool(torch.isnan(out[outside]).all()), what + ": wrote outside its window")
        g64 = torch.stack([p.to(F64) for p in parts])
        g64 = torch.where(g64.abs() < FLT_MIN, torch.zeros_like(g64), g64)
        ref = g64.sum(0) * s32
        bound = world * U * g64.abs().sum(0) * s32 * (1 + 2 ** -20)
        over = (out[sb:sb + sl].to(F64) - ref[sb:sb + sl]).abs() - bound[sb:sb + sl]
        chk.true(sl == 0 or float(over.max()) <= 0, what + f": outside the float64 bound by {float(over.max()) if sl else 0:.3g}")
        chk.same(snaps[i], inputs[i][rank], what + ": the gradient buffer changed")
        pin = 8
        if sb <= pin < sb + sl:
            chk.true(out[pin].item() == 0.0, what + f": a subnormal gradient on every rank gave {out[pin].item()!r}, not a flushed 0")
    chk.true(any(sl == 0 for (_, _, sl) in outs), "no bucket missed this rank's shard (sub_len = 0 untested)")


def _special_masters(n, seed):
    """fp32 master values for the all-gather: bf16 round-to-nearest-even ties (both directions, both signs), values that
    round past the largest bf16 to +-inf (and one just below that), +-inf, NaNs, +-0, and wide-range normals."""
    x = _randn(n, seed, F32, spread=40)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    ties = torch.randint(0x3E00, 0x4300, (n,), device="cuda", generator=g, dtype=torch.int32) << 16 | 0x8000
    ties = ties | (torch.randint(0, 2, (n,), device="cuda", generator=g, dtype=torch.int32) << 31)
    specials = [0x7F800000, 0xFF800000, 0x7FC00000, 0x7FA00001, 0xFFC00123, 0x00000000, 0x80000000, 0x7F7FFFFF, 0xFF7FFFFF,
                0x7F7F8000, 0xFF7F8000, 0x7F7F7FFF, 0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000]
    sp = torch.tensor([s - (1 << 32) if s >= 1 << 31 else s for s in specials], dtype=torch.int32, device="cuda")
    i = torch.arange(n, device="cuda")
    xb = x.view(torch.int32).clone()
    xb = torch.where(i % 5 == 1, ties, xb)
    xb = torch.where(i % 5 == 3, sp[(i // 5) % len(specials)], xb)
    return xb.view(F32)


def _all_gather_sequence(chk, arena, fgs, rank, world):
    """Every rank's whole flat parameter buffer must equal ``torch.cat(masters).to(dtype)`` — its own shard included, which the
    kernel rewrites through ``p = 0`` — and nothing else in the arena may change."""
    import torch.distributed as dist

    masters = {gi: [_special_masters(fg.shard_numel, 4409 * gi + 17 * r + 5) for r in range(world)] for gi, fg in enumerate(fgs)}
    for fg in fgs:
        fg.param_flat.fill_(-7.0)                              # stale values: the gather must overwrite every element
    whole = arena.ws.local_tensor(0, (arena.ws.nbytes,), torch.uint8)
    keep = torch.ones(arena.ws.nbytes, dtype=torch.bool, device="cuda")
    for fg in fgs:
        keep[fg.param_off:fg.param_off + fg.total * fg.param_flat.element_size()] = False
    before = whole.clone()
    torch.cuda.synchronize()
    dist.barrier()
    for gi, fg in enumerate(fgs):
        arena.all_gather(masters[gi][rank], fg.param_off, fg.model_dtype, fg.shard_numel, gi)
    torch.cuda.synchronize()
    dist.barrier()                                             # the peers' pushes into this rank have landed
    for gi, fg in enumerate(fgs):
        want = torch.cat(masters[gi]).to(fg.model_dtype)
        chk.same(fg.param_flat, want, f"all-gather group {gi} (fp32 -> {fg.model_dtype})")
    chk.true(torch.equal(whole[keep], before[keep]), "all-gather wrote outside the parameter buffers (gradients or padding)")


def _zero1_worker(rank, world):
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import zero1_comm

    chk = _Checks()
    layouts = [(_RAGGED_BF16, BF16, BF16), (_RAGGED_F32, F32, F32)]
    arena = zero1_comm.Zero1Symm(dist.group.WORLD, _arena_bytes(layouts, world))
    fgs = _flat_groups(arena, layouts, world, rank)
    _reduce_scatter_sequence(chk, arena, fgs, rank, world)
    chk.settle()
    _all_gather_sequence(chk, arena, fgs, rank, world)
    chk.settle()
    # a real-size shard: one Llama-2-7B layer at TP 8 in the fp32-gradient (use_grad_acc_hook) layout, its own arena
    layouts = [(_LLAMA7B_TP8_LAYER, BF16, F32)]
    big = zero1_comm.Zero1Symm(dist.group.WORLD, _arena_bytes(layouts, world))
    (fg,) = _flat_groups(big, layouts, world, rank)
    grads = [_randn(fg.total, 90001 + r, F32) for r in range(world)]
    fg.grad_flat.copy_(grads[rank])
    torch.cuda.synchronize()
    dist.barrier()
    out = _nan_filled(fg.shard_numel)
    big.reduce_scatter(fg.grad_off, F32, fg.shard_numel, 1.0 / world, out, 0)
    master = _randn(fg.shard_numel, 90101 + rank, F32, spread=20)
    big.all_gather(master, fg.param_off, BF16, fg.shard_numel, 0)
    torch.cuda.synchronize()
    dist.barrier()
    lo, hi = fg.shard_range
    want = _emulate([g[lo:hi] for g in grads], [(rank + p) % world for p in range(world)])
    chk.same(out, want * torch.tensor(_f32(1.0 / world), device="cuda"), "Llama-2-7B TP 8 layer reduce-scatter")
    chk.same(fg.param_flat, torch.cat([_randn(fg.shard_numel, 90101 + r, F32, spread=20) for r in range(world)]).to(BF16),
             "Llama-2-7B TP 8 layer all-gather")
    chk.settle()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_zero1_reduce_scatter_and_all_gather_bit_exact(world):
    run_distributed(_zero1_worker, world, use_cuda="loopback", timeout=300)


# =====================================================================================================================
# ZeRO-1 launcher checks: misuse raises before anything is launched
# =====================================================================================================================
def test_zero1_launchers_refuse_misuse_before_launch():
    """One process acting as a world of one: a launch would leave the epoch in the flag words.  Every misuse is
    combined with sizes at which a launch would touch no memory out of place, so a missing check shows as a
    flag that changed, not as a fault."""
    from neuronx_distributed_b200.ops import _ext

    e = _ext.ext()
    assert e is not None and hasattr(e, "zero1_all_gather"), _ext.load_error()
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(64, dtype=torch.int32, device="cuda")
    peers = torch.tensor([buf.data_ptr()] * 9, dtype=torch.int64, device="cuda")
    fpeers = torch.tensor([flags.data_ptr()] * 9, dtype=torch.int64, device="cuda")
    done = torch.zeros(8, dtype=torch.int32, device="cuda")
    master = torch.arange(16, dtype=F32, device="cuda")

    def ag(m=master, off=0, world=1, n=16):
        e.zero1_all_gather(m, peers, off, fpeers, 0, 1, 0, world, n, done, False)

    def rs(out=None, off=0, world=1, n=16, sub_len=0):
        out = torch.zeros(16, dtype=F32, device="cuda") if out is None else out
        e.zero1_reduce_scatter(peers, off, fpeers, 0, 1, 0, world, n, 1.0, out, done, True, 0, sub_len, 0)

    misuse = {
        "all-gather shard_numel % 8": lambda: ag(n=4),
        "all-gather master shorter than the shard": lambda: ag(m=master[:8]),
        "all-gather master not fp32": lambda: ag(m=master.to(BF16), n=0),
        "all-gather master not contiguous": lambda: ag(m=torch.zeros(32, dtype=F32, device="cuda")[::2], n=0),
        "all-gather param_off_bytes % 16": lambda: ag(off=8, n=0),
        "all-gather world > 8": lambda: ag(world=9, n=0),
        "reduce-scatter out not fp32": lambda: rs(out=torch.zeros(16, dtype=BF16, device="cuda"), n=0),
        "reduce-scatter out shorter than the shard": lambda: rs(out=torch.zeros(8, dtype=F32, device="cuda")),
        "reduce-scatter grad_off_bytes % 16": lambda: rs(off=8, n=0),
        "reduce-scatter world > 8": lambda: rs(world=9, n=0),
    }
    for what, call in misuse.items():
        with pytest.raises(RuntimeError):
            call()
        torch.cuda.synchronize()
        assert int(flags.count_nonzero()) == 0 and int(buf.count_nonzero()) == 0, f"{what}: launched"
    # the same arguments without the misuse do launch (the flag words show the epoch), so the checks above mean something
    ag()
    torch.cuda.synchronize()
    assert int(flags[16]) == 1 and torch.equal(buf[:64].view(F32), master)


# =====================================================================================================================
# one-shot all-reduce
# =====================================================================================================================
def _oneshot_worker(rank, world):
    """The launcher picks ``ctas = nbytes / 16384`` clamped to 1..64, so a sequence of sizes changes the CTA count from call
    to call and exercises the per-(source, CTA) flags and both parity halves.  (With that choice every CTA has work: the
    NVLS cases below cover empty CTAs.)"""
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import _ext, allreduce

    chk = _Checks()
    ws, state = allreduce._workspace(dist.group.WORLD)
    maxb = allreduce._MAX_BYTES
    e = _ext.ext()

    def call(x):
        return e.oneshot_allreduce(x, ws.ptrs, ws.flag_ptrs, maxb, state, ws.rank, ws.world)

    def n_of(dt, nbytes):
        return nbytes // torch.empty((), dtype=dt).element_size()

    sizes = [(BF16, 16), (BF16, maxb), (F32, 16), (F32, maxb), (BF16, 5120 * 2), (F32, 16384 * 64 + 16 * 7),
             (BF16, 16384 * 5 + 48), (F32, 16384 * 3 + 16), (BF16, 16), (F32, maxb), (BF16, 16384 * 2 + 16 * 5)]
    xs = [[_randn(n_of(dt, nb), 613 * i + r, dt) for r in range(world)] for i, (dt, nb) in enumerate(sizes)]
    torch.cuda.synchronize()
    dist.barrier()
    outs = [call(x[rank]) for x in xs]
    torch.cuda.synchronize()
    for i, ((dt, nb), x, out) in enumerate(zip(sizes, xs, outs)):
        what = f"one-shot all-reduce call {i} ({dt}, {nb} bytes)"
        chk.same(out, _emulate(x, range(world)).to(dt), what + ": vs the rank-ordered fp32 sum rounded once")
        _rank_identical(chk, out, what)
    chk.settle()

    # CUDA-graph replay with new inputs before each replay, eager calls of other sizes in between (one device epoch)
    n = 5120
    xin = torch.zeros(n, dtype=BF16, device="cuda")
    call(xin)
    torch.cuda.synchronize()
    dist.barrier()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = call(xin)
    dist.barrier()
    reps = [[_randn(n, 7001 + 11 * it + r, BF16) for r in range(world)] for it in range(3)]
    mids = [[_randn(n_of(F32, 16384 * 9), 7501 + 11 * it + r, F32) for r in range(world)] for it in range(3)]
    got, mid_out = [], []
    for it in range(3):
        xin.copy_(reps[it][rank])
        graph.replay()
        got.append(y.clone())
        mid_out.append(call(mids[it][rank]))
    torch.cuda.synchronize()
    for it in range(3):
        chk.same(got[it], _emulate(reps[it], range(world)).to(BF16), f"graph replay {it}")
        chk.same(mid_out[it], _emulate(mids[it], range(world)), f"eager call after graph replay {it}")
        _rank_identical(chk, got[it], f"graph replay {it}")
    chk.settle()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_oneshot_allreduce_bit_exact_and_rank_identical(world):
    run_distributed(_oneshot_worker, world, use_cuda="loopback", timeout=240)


# =====================================================================================================================
# NVLS-layout collectives, unicast branch
# =====================================================================================================================
def _gemv_bound(xs, ws_, res, world):
    """float64 reference of sum_r x_r @ w_r^T (+ res) and a per-element bound on the kernel's bf16 result.  Each lane runs
    K/32 fp32 FMAs, the warp adds 32 lanes in 5 steps, the ranks' partials are added in `world` steps (+1 for the residual);
    then one rounding to bf16 (at most 2^-8 relative, the half ulp of an 8-bit significand)."""
    K = xs[0].shape[1]
    ref = sum(x.to(F64) @ w.to(F64).t() for x, w in zip(xs, ws_))
    mag = sum(x.to(F64).abs() @ w.to(F64).abs().t() for x, w in zip(xs, ws_))
    if res is not None:
        ref = ref + res.to(F64)
        mag = mag + res.to(F64).abs()
    e32 = (math.ceil(K / 32) + 5 + world + 1) * U * 1.01 * mag
    return ref, e32 + 2.0 ** -8 * (ref.abs() + e32)


def _nvls_worker(rank, world):
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import nvls

    chk = _Checks()
    g = dist.group.WORLD
    # default halves of the regions (NXD_NVLS_AR_MAX_MB = 8; the GEMV's 1 MB rounded up to 2 MB): larger requests grow them
    ar_default_half, gemv_default_half = 8 << 20, 2 << 20
    steps = []                                                  # (kind, args, per-rank inputs, out)
    seed = [0]

    def ins(shape, dt, spread=12):
        seed[0] += 1
        n = math.prod(shape)
        return [_randn(n, 3301 * seed[0] + r, dt, spread).view(shape) for r in range(world)]

    def ar(n, dt, residual=False):
        x = ins((n,), dt)
        r = ins((n,), dt)[0] if residual else None
        steps.append(("ar", (dt, r), x, nvls.all_reduce_sum(x[rank], g, residual=r)))

    def ag(shape, dt):
        x = ins(shape, dt)
        steps.append(("ag", (), x, nvls.all_gather(x[rank], g)))

    def rs(n, dt):
        x = ins((world * n,), dt)
        steps.append(("rs", (dt, n), x, nvls.reduce_scatter_sum(x[rank], g)))

    def a2a(shape, dt):
        x = ins((world * shape[0],) + shape[1:], dt)
        steps.append(("a2a", (), x, nvls.all_to_all(x[rank], g)))

    def gemv(M, N, K, residual=False):
        x = ins((M, K), BF16, 2)
        w = [t * 0.05 for t in ins((N, K), BF16, 2)]
        r = ins((M, N), BF16, 2)[0] if residual else None
        steps.append(("gemv", (w, r), x, nvls.gemv_all_reduce(x[rank], w[rank], g, residual=r)))

    torch.cuda.synchronize()
    dist.barrier()
    # 16-byte minimum: one vector, the other 31 CTAs of the gather / scatter / all-to-all have nothing to do
    ar(8, BF16); ag((4,), F32); rs(8, BF16); a2a((4,), F32); gemv(1, 104, 360)
    # sizes that do not fill the CTA slicing evenly, interleaved kinds on one group
    ar(16384 * 3 // 4 + 20, F32); ar(5128, BF16, residual=True); ag((1001, 4), F32); rs(8008, BF16)
    a2a((1000, 4), F32); gemv(2, 296, 1000, residual=True); ar(4, F32, residual=True); ag((3, 40), BF16)
    rs(4 * 333, F32); a2a((24,), BF16)
    for M, (N, K) in zip(range(3, 9), [(104, 264), (8, 1000), (584, 520), (296, 8), (40, 2056), (1000, 776)]):
        gemv(M, N, K, residual=M % 2 == 0)
    # larger than the default half: the all-reduce and GEMV regions grow; the calls after the growth must be right too
    ar(ar_default_half // 4 + 4, F32); ar(5128, BF16, residual=True); ar(8, BF16)
    gemv(8, 65544, 264); gemv(3, 104, 360, residual=True)
    torch.cuda.synchronize()
    order = range(world)
    for i, (kind, args, x, out) in enumerate(steps):
        what = f"NVLS step {i} ({kind}, input {tuple(x[0].shape)} {x[0].dtype})"
        if kind == "ar":
            dt, r = args
            want = _emulate(x, order).to(dt)
            if r is not None:                                   # the sum is rounded, then the residual added and rounded again
                want = (want.float() + r.float()).to(dt)
            chk.same(out, want, what)
        elif kind == "ag":
            chk.same(out, torch.cat(x), what)
        elif kind == "rs":
            dt, n = args
            chk.same(out, _emulate([t[rank * n:(rank + 1) * n] for t in x], order).to(dt), what)
        elif kind == "a2a":
            n = x[0].shape[0] // world
            chk.same(out, torch.cat([t[rank * n:(rank + 1) * n] for t in x]), what)
        else:
            w, r = args
            ref, bound = _gemv_bound(x, w, r, world)
            err = (out.to(F64) - ref).abs()
            chk.true(bool((err <= bound).all()), what + f": outside the float64 bound by {(err - bound).max().item():.3g}")
            _rank_identical(chk, out, what)
    chk.true(nvls._STATE[(id(g), "ar")].half_bytes > ar_default_half, "the all-reduce region did not grow")
    chk.true(nvls._STATE[(id(g), "gemv_ar")].half_bytes > gemv_default_half, "the GEMV region did not grow")
    chk.settle()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_nvls_collectives_unicast_bit_exact(world):
    run_distributed(_nvls_worker, world, use_cuda="loopback", timeout=300)


# =====================================================================================================================
# ZeRO-1 optimizer end to end on the arena
# =====================================================================================================================
def _adamw_hf_ref(p, g, m, v, gs, lr, b1, b2, eps, wd, step):
    """One float64 step of the fused AdamW (HF form, bias-corrected step size, decoupled decay after the update) from its
    fp32 state, and a bound on the kernel's fp32 step: m's products and sum (4u on |m| + |gr|), v's (6u on v), the step size,
    sqrt, + eps and the division (16u together), half of v's relative error through the sqrt, the final products on p."""
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    b1, b2 = _f32(b1), _f32(b2)
    gr = g * gs
    m1 = b1 * m + (1 - b1) * gr
    v1 = b2 * v + (1 - b2) * gr * gr
    step_size, denom = lr * math.sqrt(bc2) / bc1, v1.sqrt() + eps
    upd = step_size * m1 / denom
    p1 = (p - upd) * (1 - lr * wd)
    m_err = 4 * U * (m.abs() + gr.abs())
    v_err = 6 * U * v1
    u_err = step_size / denom * (m_err + 16 * U * m1.abs()) + upd.abs() * (v_err / (2 * v1.clamp_min(1e-300)))
    p_err = 4 * U * (p.abs() + p1.abs()) + u_err
    return p1, m1, v1, p_err, m_err, v_err


_OPT_SHAPES = [[(1,), (7,), (129,), (4099,), (128, 1000)], [(1100, 1000)]]


def _optimizer_run(rank, world, overlap, chk):
    import torch.distributed as dist

    from neuronx_distributed_b200.optimizer.zero_redundancy_optimizer import Zero1Optimizer
    from neuronx_distributed_b200.utils.adamw_fp32_optim_params import AdamW_FP32OptimParams

    lr, betas, eps, wd = 1e-2, (0.9, 0.95), 1e-8, 0.1
    groups = []
    for gi, shapes in enumerate(_OPT_SHAPES):
        groups.append([torch.nn.Parameter(_randn(math.prod(s), 50 + 10 * gi + i, BF16, 2).view(s)) for i, s in enumerate(shapes)])
    opt = Zero1Optimizer([{"params": ps_} for ps_ in groups], AdamW_FP32OptimParams, lr=lr, betas=betas, eps=eps,
                         weight_decay=wd, use_grad_acc_hook=True, bucket_cap_mb_reduce_scatter=1, overlap_grad_reduce=overlap,
                         grad_clipping=True, max_norm=1.0)
    tag = f"overlap={overlap}"
    chk.true(opt.arena is not None and opt._overlap_active == overlap, f"{tag}: the optimizer is not on the peer-memory arena")
    if overlap:
        chk.true(len(opt._buckets) > 2, f"{tag}: only {len(opt._buckets)} buckets")
    params = [p for ps_ in groups for p in ps_]
    shards = []
    for step in (1, 2, 3):
        # loss = sum_i (p_i * c_i).sum(): the gradient of p_i is c_i exactly, summed over the micro-batches in fp32 by the hook
        cs = [[[_randn(p.numel(), 100000 * step + 1000 * mb + 10 * i + r, BF16, 6).view(p.shape) for i, p in enumerate(params)]
               for mb in (0, 1)] for r in range(world)]
        opt.zero_grad()
        for mb in (0, 1):
            with opt.no_sync() if mb == 0 else contextlib.nullcontext():
                loss = sum((p * c).float().sum() for p, c in zip(params, cs[rank][mb]))
                loss.backward()
        if overlap:
            chk.true(any(opt._bucket_launched), f"{tag} step {step}: no bucket was reduced during backward")
        prev = []
        for fg in opt.flat_groups:
            st = opt.base_optimizer.state.get(fg.base_param, {})
            z = torch.zeros_like(fg.master_shard)
            prev.append((fg.master_shard.clone(), st.get("exp_avg", z).clone(), st.get("exp_avg_sq", z).clone()))
        opt.step()
        torch.cuda.synchronize()
        gs = float(opt.base_optimizer.grad_scale)
        sq64, emu_shards = 0.0, []
        k = 0
        for gi, fg in enumerate(opt.flat_groups):
            flats = []
            for r in range(world):
                f = torch.zeros(fg.total, dtype=F32, device="cuda")
                for s, i in zip(fg.slots, range(k, k + len(fg.slots))):
                    f[s.offset:s.offset + s.numel] = cs[r][0][i].reshape(-1).float() + cs[r][1][i].reshape(-1).float()
                flats.append(f)
            k += len(fg.slots)
            s32 = torch.tensor(_f32(1.0 / world), device="cuda")
            every = [_emulate([f[q * fg.shard_numel:(q + 1) * fg.shard_numel] for f in flats],
                              [(q + p) % world for p in range(world)]) * s32 for q in range(world)]
            sq64 += sum(float(e.to(F64).pow(2).sum()) for e in every)
            emu = every[rank]
            emu_shards.append(emu)
            chk.same(fg.grad_shard, emu, f"{tag} step {step} group {gi}: reduced gradient shard")
            # the AdamW step from the previous state, in float64
            p0, m0, v0 = (t.to(F64) for t in prev[gi])
            p1, m1, v1, p_err, m_err, v_err = _adamw_hf_ref(p0, emu.to(F64), m0, v0, gs, lr, betas[0], betas[1], eps, wd, step)
            st = opt.base_optimizer.state[fg.base_param]
            for name, got, want, bound in (("master", fg.master_shard, p1, p_err), ("exp_avg", st["exp_avg"], m1, m_err),
                                           ("exp_avg_sq", st["exp_avg_sq"], v1, v_err)):
                err = (got.to(F64) - want).abs()
                chk.true(bool((err <= bound).all()), f"{tag} step {step} group {gi}: {name} outside the float64 AdamW bound "
                                                    f"by {(err - bound).max().item():.3g}")
            # every rank holds every rank's master shard, rounded to bf16 once
            masters = _gather_cpu(fg.master_shard)
            chk.same(fg.param_flat, torch.cat(masters).cuda().to(BF16), f"{tag} step {step} group {gi}: param_flat")
            _rank_identical(chk, fg.param_flat, f"{tag} step {step} group {gi}: param_flat")
        norm = float(opt.grad_norm)
        chk.true(abs(norm - math.sqrt(sq64)) <= 1e-5 * math.sqrt(sq64), f"{tag} step {step}: grad norm {norm} vs {math.sqrt(sq64)}")
        chk.true(gs < 1.0, f"{tag} step {step}: clipping did not engage (coefficient {gs})")
        shards.append([fg.grad_shard.clone() for fg in opt.flat_groups])
        chk.settle()
        dist.barrier()
    return shards


def _optimizer_worker(rank, world):
    from neuronx_distributed_b200 import ops

    # the arena's kernels need only peer memory; `available` also asks for an NCCL group, the loopback control plane is gloo
    ops.zero1_comm.available = lambda pg: True
    chk = _Checks()
    plain = _optimizer_run(rank, world, False, chk)
    overlapped = _optimizer_run(rank, world, True, chk)
    for step, (a, b) in enumerate(zip(plain, overlapped)):
        for gi, (x, y) in enumerate(zip(a, b)):
            chk.same(y, x, f"step {step + 1} group {gi}: overlapped rs_out vs the reduce-scatter at step()")
    chk.settle()


@pytest.mark.parametrize("world", [2, 3])
def test_zero1_optimizer_on_peer_arena_exact_gradients(world):
    run_distributed(_optimizer_worker, world, use_cuda="loopback", timeout=300)
