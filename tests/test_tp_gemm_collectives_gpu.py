"""The fused tensor-parallel GEMMs of ``csrc/gemm_sm90.cu`` bit for bit: all-gather→GEMM and GEMM→reduce-scatter on the
cudaIpc peer-memory kernels (MODE 1 / 2) and on the NVLS kernels (MODE 5 / 6), at the shard shapes of real models, and the
sequence-parallel Column / Row linears built on them.

Two to four processes share ``cuda:0`` (``run_distributed(..., use_cuda="loopback")``); the kernels run their real flag,
epoch and claim protocols between the processes' contexts.  There is no multicast mapping between contexts of one device, so
the NVLS kernels take their unicast branch.  Every rank rebuilds every rank's inputs from seeds.

With unicast peer memory every step after the MMA is fixed, so each result has an exact oracle:

* all-gather→GEMM: ``out = bf16(acc)``, where ``acc`` is the wgmma accumulation the plain GEMM (MODE 0) makes for the same A
  row and B column: same template, k-block order, wgmma and TMA zero fill.  The gathered buffer is ``torch.cat(shards)``.
* GEMM→reduce-scatter: every source's partial tile is the plain GEMM's accumulator, sent as bf16 (MODE 2 always; MODE 6
  unless ``NXD_TP_WIRE=fp32``, which keeps it fp32), summed at the owner in fp32 in the order ``p = 0 .. world-1`` from +0
  with flush-to-zero adds, and rounded to bf16 once.

The plain GEMM is called on the extension (``gemm_bf16`` with an fp32 output, i.e. the raw accumulator), so that no routing
sends a small M to the GEMV.  The A operands are Gaussian times 2^k with k per row in [-10, 10], so that the partials of
different ranks differ by up to 20 binades and their fp32 sum rounds; from three ranks on, every 8th row of the reduce-scatter
operands cancels between ranks 0 and 1 (``_Run.inputs``).  Each step asserts that its inputs tell the summation order and
the wire format apart.  Every result is also held to a per-element float64 bound (``_bound``), which is what still holds
where the order is unknown: ``multimem.ld_reduce`` on an NVSwitch (the ``multigpu`` variant).

Ranks collect failures and compare them over gloo only after all kernels have run (``_Checks``): a rank that left early
would leave its peers waiting on its flags.
"""
import os
import types

import pytest
import torch

from dist_utils import _Checks, _emulate, _same, run_distributed

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
U = 2.0 ** -24                      # fp32 unit roundoff
U_BF16 = 2.0 ** -8                  # bf16 unit roundoff: half an ulp of an 8-bit significand
ROW_SPREAD = 10

# (case, kind, N, K, trans_b).  N and K per rank of the TP shard; trans_b=False is the MN-major weight of a dgrad.
_CASES = [
    ("Llama-3-8B TP8 qkv", "ag", 768, 4096, True),
    ("Llama-3-8B TP8 o_proj", "rs", 4096, 512, True),
    ("Llama-3-8B TP8 gate_up", "ag", 3584, 4096, True),
    ("Llama-3-8B TP8 down", "rs", 4096, 1792, True),
    ("Llama-3-8B TP8 qkv dgrad", "rs", 4096, 768, False),
    ("Qwen2.5-7B TP4 qkv (N tail 128)", "ag", 1152, 3584, True),
    ("Qwen2.5-7B TP4 down", "rs", 3584, 4736, True),
    ("Qwen2.5-3B TP8 gate_up (N tail 192)", "ag", 2752, 2048, True),
    ("Qwen2.5-3B TP8 down (K tail 32)", "rs", 2048, 1376, True),
    ("Qwen2.5-3B TP8 down dgrad (N tail 96)", "ag", 1376, 2048, False),
    ("Qwen2.5-3B TP8 gate_up dgrad", "rs", 2048, 2752, False),
    ("Llama-2-13B TP8 gate_up (N tail 128)", "ag", 3456, 5120, True),
    ("GPT-NeoX-20B TP8 qkv", "ag", 2304, 6144, True),
    ("GPT-NeoX-20B TP8 dense_4h_to_h", "rs", 6144, 3072, True),
    ("BERT-large TP2 intermediate", "ag", 2048, 1024, True),
    ("BERT-large TP2 output", "rs", 1024, 2048, True),
    ("BERT-large TP2 output dgrad", "ag", 2048, 1024, False),
] + [(f"{what}", kind, n, k, tb) for what, n, k in (("minimal", 8, 8), ("one tile + 8", 264, 72))
     for kind in ("ag", "rs") for tb in (True, False)]


def _operand(shape, seed, row_spread=ROW_SPREAD):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, device="cuda", generator=g)
    if row_spread:
        x = x * torch.exp2(torch.randint(-row_spread, row_spread + 1, (shape[0], 1), device="cuda", generator=g).float())
    return x.to(BF16)


def _acc(a, b, trans_a, trans_b):
    """The plain GEMM's fp32 accumulator of op(a) @ op(b)."""
    from neuronx_distributed_b200.ops import _ext

    M = a.shape[1] if trans_a else a.shape[0]
    N = b.shape[0] if trans_b else b.shape[1]
    out = torch.empty(M, N, dtype=F32, device="cuda")
    _ext.ext().gemm_bf16(a, b, out, trans_a, trans_b, False)
    return out


def _op64(a, b, trans_a, trans_b):
    a64 = a.to(F64).t() if trans_a else a.to(F64)
    b64 = b.to(F64).t() if trans_b else b.to(F64)
    return a64 @ b64, a64.abs() @ b64.abs()


def _gemm_err(K, mag):
    """Error of the wgmma accumulator: K fp32 additions, each with at most 2^-23 of the magnitudes so far (a truncating
    adder loses up to one ulp, twice the round-to-nearest bound)."""
    return (K + 2) * 2 * U * mag


def _bound(parts64, mags, K, wire):
    """float64 value and per-element bound of the bf16 result of sum_p round_wire(P_p): the GEMM term of each partial,
    2^-8 |P_p| for a bf16 partial (none for an fp32 one), world * u * sum |P_p| for the fp32 sum and 2^-8 |result| for the
    final rounding."""
    ref = sum(parts64)
    e = torch.zeros_like(ref)
    absp = torch.zeros_like(ref)
    for p64, mag in zip(parts64, mags):
        eg = _gemm_err(K, mag)
        ew = U_BF16 * (p64.abs() + eg) if wire == "bf16" else 0.0
        e = e + eg + ew
        absp = absp + p64.abs() + eg + ew
    e = e + len(parts64) * U * 1.01 * absp
    return ref, e + U_BF16 * (ref.abs() + e)


# =====================================================================================================================
# kernel level: ws.ag_gemm / ws.gemm_rs on both paths
# =====================================================================================================================
class _Run:
    """One worker's calls.  ``steps`` keeps what every call needs to be checked after all ranks have run all calls."""

    def __init__(self, rank, world, chk):
        import torch.distributed as dist

        from neuronx_distributed_b200.ops import _ext, _fused_impl

        self.rank, self.world, self.chk = rank, world, chk
        self.fi, self.ext = _fused_impl, _ext
        self.ws = _fused_impl.workspace(dist.group.WORLD)
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.defaults = (_fused_impl._COMM_SMS, dict(_fused_impl.NVLS_CONFIG))
        self.steps = []
        self.seed = 0

    # ---------------------------------------------------------------- inputs
    def inputs(self, kind, rows, N, K, tb, seed):
        w = self.world
        b = _operand((N, K) if tb else (K, N), 7 * seed + 1, row_spread=0)
        if kind == "ag":
            return [_operand((rows, K), 7 * seed + 2 + r) for r in range(w)], b
        a = [_operand((w * rows, K), 7 * seed + 2 + r) for r in range(w)]
        if w >= 3:
            # every 8th row cancels: rank 1 sends exactly -(rank 0's partial) at 2^12 times the spread, the other ranks 2^-12
            # times it.  In the order 0, 1, 2, .. the sum is the small ranks' partials; an order that adds a small one to a
            # large one first loses it, 44 binades below.  The row-scaled rest shows the order only where bf16 rounding does.
            a[0][::8] *= 2.0 ** 12
            a[1][::8] = -a[0][::8]
            for p in range(2, w):
                a[p][::8] *= 2.0 ** -12
        return a, b

    # ---------------------------------------------------------------- one call
    def _path(self, path, split):
        fi = self.fi
        fi._NVLS_MODE = "force" if path == "nvls" else "0"
        fi._COMM_SMS, cfg = self.defaults[0], dict(self.defaults[1])
        if split == "min":
            fi._COMM_SMS, cfg = 1, {"comm_ctas_ag": 1, "comm_ctas_rs": 1}
        elif split == "max":
            cfg = {"comm_ctas_ag": self.sms - 1, "comm_ctas_rs": self.sms - 1}
        fi.NVLS_CONFIG.update(cfg)

    def prepare(self, kind, path, rows, N, K, wire):
        """Grow the region this call uses now (collective), so that the NaN fill lands where the call reads and writes."""
        M = self.world * rows
        if path == "nvls":
            self.ws._ensure_nvls(M * K * 2, 0) if kind == "ag" else self.ws._ensure_nvls(0, M * N * (4 if wire == "fp32" else 2))
        else:
            self.ws._ensure(M * K * 2, 0) if kind == "ag" else self.ws._ensure(0, M * N * 2)

    def poison(self):
        """NaN in both payload halves of both regions, flags untouched, with every rank at rest on both sides."""
        import torch.distributed as dist

        torch.cuda.synchronize()
        dist.barrier()
        ws = self.ws
        if ws.ws is not None:
            ws.ws.local_tensor(0, (ws.ws.nbytes // 2,), BF16).fill_(float("nan"))
        if ws.nv is not None:
            n = 2 * ws.nv_ag_bytes + 2 * ws.nv_rs_bytes
            ws.nv.local_tensor(self.fi._NVLS_FLAG_BYTES, (n // 2,), BF16).fill_(float("nan"))
        torch.cuda.synchronize()
        dist.barrier()

    def call(self, kind, path, rows, N, K, tb, wire="bf16", join=True, split="default", poisoned=False, what=""):
        self.seed += 1
        seed = 1000 * self.world + self.seed
        os.environ["NXD_TP_WIRE"] = wire
        self._path(path, split)
        if poisoned:
            self.prepare(kind, path, rows, N, K, wire)
            self.poison()
        xs, b = self.inputs(kind, rows, N, K, tb, seed)
        ws = self.ws
        ep0 = (ws.nv_ag_epoch, ws.nv_rs_epoch, ws.ag_epoch, ws.rs_calls)
        n0 = self.ext.launches()
        gathered = None
        if kind == "ag":
            out, g = ws.ag_gemm(xs[self.rank], b, tb)
            gathered = g.clone()            # stream-ordered before this rank's next call, which peers need to reuse the half
        else:
            out = ws.gemm_rs(xs[self.rank], b, tb, gemm_join=join)
        ep1 = (ws.nv_ag_epoch, ws.nv_rs_epoch, ws.ag_epoch, ws.rs_calls)
        want = {("nvls", "ag"): 0, ("nvls", "rs"): 1, ("ipc", "ag"): 2, ("ipc", "rs"): 3}[(path, kind)]
        other = (2, 3) if path == "nvls" else (0, 1)       # a cudaIpc re-layout restarts both of its own counters
        ran = ep1[want] != ep0[want] and all(ep1[i] == ep0[i] for i in other)
        step = dict(kind=kind, path=path, rows=rows, N=N, K=K, tb=tb, wire=wire, join=join, seed=seed, out=out,
                    gathered=gathered, what=f"{what} {path} {kind} rows={rows} N={N} K={K} trans_b={tb} wire={wire} "
                                            f"join={join} split={split}")
        self.chk.true(ran and self.ext.launches() == n0 + 1, f"{step['what']}: not one launch of the {path} kernel")
        if path == "nvls":
            step["counters"], step["claim_base"] = ws.nv_counters.clone(), ws.nv_claim_base
        self.steps.append(step)
        self.fi.NVLS_CONFIG.update(self.defaults[1])
        return step

    # ---------------------------------------------------------------- checks, after every rank made every call
    def check(self, stats):
        w, r, chk = self.world, self.rank, self.chk
        for st in self.steps:
            xs, b = self.inputs(st["kind"], st["rows"], st["N"], st["K"], st["tb"], st["seed"])
            rows, K, tb, what = st["rows"], st["K"], st["tb"], st["what"]
            multicast = st["path"] == "nvls" and self.ws.nv.has_multicast
            if st["kind"] == "ag":
                full = torch.cat(xs)
                chk.same(st["gathered"], full, what + ": gathered A")
                chk.same(st["out"], _acc(full, b, False, tb).to(BF16), what + ": out vs bf16(plain GEMM accumulator)")
                ref, mag = _op64(full, b, False, tb)
                eg = _gemm_err(K, mag)
                ref_b = eg + U_BF16 * (ref.abs() + eg)
                key = "MODE 5" if st["path"] == "nvls" else "MODE 1"
            else:
                wire = st["wire"] if st["path"] == "nvls" else "bf16"     # MODE 2 stages bf16 whatever NXD_TP_WIRE says
                sl = slice(r * rows, (r + 1) * rows)
                accs = [_acc(x, b, False, tb)[sl] for x in xs]
                parts = [a.to(BF16) if wire == "bf16" else a for a in accs]
                want = _emulate(parts, range(w)).to(BF16)
                other = [a if wire == "bf16" else a.to(BF16) for a in accs]
                if not multicast:
                    chk.same(st["out"], want, what + ": out vs the p = 0..world-1 emulation")
                    if w >= 3:          # two fp32 addends commute: the order shows from three ranks on
                        chk.true(not _same(_emulate(parts, reversed(range(w))).to(BF16), want),
                                 what + ": inputs do not tell the reversed rank order apart")
                    chk.true(not _same(_emulate(other, range(w)).to(BF16), want),
                             what + ": inputs do not tell the wire formats apart")
                p64 = [_op64(x[sl], b, False, tb) for x in xs]
                ref, ref_b = _bound([p for p, _ in p64], [m for _, m in p64], K, wire)
                key = f"MODE 6 {wire} wire" if st["path"] == "nvls" else "MODE 2"
            err = (st["out"].to(F64) - ref).abs()
            ratio = float((err / ref_b.clamp_min(1e-300)).max())
            chk.true(bool((err <= ref_b).all()) and not bool(torch.isnan(st["out"]).any()),
                     what + f": outside the float64 bound ({ratio:.3g} of it)")
            stats[key] = max(stats.get(key, 0.0), ratio)
            if st["path"] == "nvls":
                c = st["counters"]
                chk.true(int(c[0]) & 0xFFFFFFFF == st["claim_base"],
                         what + f": claim counter {int(c[0]) & 0xFFFFFFFF} at rest, claim base {st['claim_base']}")
                chk.true(not bool(c[64:].any()), what + ": tile_done counters not re-armed to zero")


def _kernel_worker(rank, world):
    os.environ["NXD_SYMM_MIN_MB"] = "1"            # regions sized by the calls: the growth below re-lays them out
    import torch.distributed as dist

    chk = _Checks()
    run = _Run(rank, world, chk)
    ws = run.ws
    torch.cuda.synchronize()
    dist.barrier()

    # (a) poisoned and barrier-separated: the real-model shard shapes, both paths, every wire and gemm_join on MODE 6
    modes6 = [("bf16", True), ("fp32", True), ("bf16", False), ("fp32", False)]
    for i, (case, kind, N, K, tb) in enumerate(_CASES):
        rows = (128, 384)[i % 2]
        run.call(kind, "ipc", rows, N, K, tb, wire=("bf16", "fp32")[i % 2], poisoned=True, what=case)
        small = N * K <= 264 * 72
        for wire, join in (modes6 if kind == "rs" and small else [modes6[i % 4]]):
            run.call(kind, "nvls", rows, N, K, tb, wire=wire, join=join, poisoned=True, what=case)
    # 64 row blocks per rank, the cudaIpc maximum, on both paths; 65 on NVLS only
    for path in ("ipc", "nvls"):
        for kind in ("ag", "rs"):
            run.call(kind, path, 8192, 264, 72, kind == "ag", wire="fp32", poisoned=True, what="64 blocks")
    for kind in ("ag", "rs"):
        run.call(kind, "nvls", 8320, 264, 72, kind == "rs", join=kind == "rs", poisoned=True, what="65 blocks")
    # ... which the cudaIpc path refuses before it launches anything
    run._path("ipc", "default")
    x, b = _operand((8320, 72), 5), _operand((264, 72), 6)
    for kind in ("ag", "rs"):
        n0 = run.ext.launches()
        try:
            ws.ag_gemm(x, b, True) if kind == "ag" else ws.gemm_rs(_operand((world * 8320, 72), 7), b, True)
            chk.true(False, f"cudaIpc {kind} at 65 row blocks per rank did not raise")
        except RuntimeError:
            pass
        chk.true(run.ext.launches() == n0, f"cudaIpc {kind} at 65 row blocks per rank launched")

    # (b) back to back, no host synchronisation: AG and RS, both weight layouts, small and large alternating, with the
    # comm-CTA splits (d) of both paths; one call grows both regions mid-stream
    ipc_rs0, nv_rs0 = ws.rs_bytes, ws.nv_rs_bytes
    torch.cuda.synchronize()
    dist.barrier()
    small = [(128, 264, 72), (256, 8, 8), (128, 520, 136)]
    large = [(384, 2752, 2048), (256, 4096, 1792), (384, 1376, 2048)]
    splits = {"ipc": ["min", "default"], "nvls": ["min", "default", "max"]}
    for path in ("ipc", "nvls", "ipc", "nvls"):
        for j in range(15):
            rows, N, K = (small if j % 2 == 0 else large)[(j // 2) % 3]
            kind, tb = ("ag", "rs")[j % 2 ^ (j // 4) % 2], (j // 2) % 2 == 0
            split = splits[path][j % len(splits[path])] if (rows, N, K) in small else "default"
            wire, join = modes6[j % 4]
            if j == 7 and path == "nvls":
                rows, N, K, kind, wire = 640, 6144, 512, "rs", "fp32"      # larger than any region so far
            elif j == 7:
                rows, N, K, kind = 640, 6144, 512, "rs"
            run.call(kind, path, rows, N, K, tb, wire=wire, join=join, split=split, what=f"back-to-back {j}")
    chk.true(ws.rs_bytes > ipc_rs0 and ws.nv_rs_bytes > nv_rs0, "no region grew during the back-to-back calls")

    stats = {}
    run.check(stats)
    every = [None] * world
    dist.all_gather_object(every, (len(run.steps), stats))
    if rank == 0:
        worst = {}
        for _, s in every:
            for k, v in s.items():
                worst[k] = max(worst.get(k, 0.0), v)
        print(f"\n[world {world}] {len(run.steps)} fused calls per rank; worst error / float64 bound: "
              + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())), flush=True)
    chk.settle()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
def test_fused_tp_gemms_bit_exact(world):
    run_distributed(_kernel_worker, world, use_cuda="loopback", timeout=400)


@pytest.mark.gpu
@pytest.mark.multigpu
def test_fused_tp_gemms_bit_exact_multigpu():
    """On separate GPUs MODE 5 / 6 run on the multicast mapping when the fabric has one: the all-gather stays exact, the
    in-switch sum is held to the float64 bound only (its order is the switch's)."""
    n = min(torch.cuda.device_count(), 4)
    run_distributed(_kernel_worker, n, use_cuda=True, timeout=400)


# =====================================================================================================================
# layer level: _TPLinear (Column + SP, Row + SP) on the fused path
# =====================================================================================================================
def _layer_worker(rank, world):
    import torch.distributed as dist

    from neuronx_distributed_b200.ops import _ext, _fused_impl
    from neuronx_distributed_b200.parallel_layers.layers import _TPLinear

    os.environ["NXD_TP_WIRE"] = "bf16"
    chk = _Checks()
    group = dist.group.WORLD
    ws = _fused_impl.workspace(group)
    seed = [0]
    results = []

    def ins(shape, scale_rows=True):
        seed[0] += 1
        return [_operand(shape, 100 * seed[0] + r, ROW_SPREAD if scale_rows else 0) for r in range(world)]

    cases = [(False, "bf16", None), (True, "fresh", None), (True, "accumulate", (96, 1.0 / 3)), (False, "accumulate", None)]
    for path in ("ipc", "nvls", "ipc", "nvls"):
        _fused_impl._NVLS_MODE = "force" if path == "nvls" else "0"
        for column in (True, False):
            for has_bias, grad, col_scale in cases:
                rows, N, K = (128, 264, 136) if column else (128, 136, 264)
                what = f"{path} {'Column' if column else 'Row'}+SP bias={has_bias} grad={grad} col_scale={col_scale is not None}"
                xs = ins((rows, K) if column else (world * rows, K))
                gys = ins((world * rows, N) if column else (rows, N))
                w = ins((N, K), False)[0]
                bias = torch.nn.Parameter(ins((N,), False)[0]) if has_bias else None
                old = ins((N, K), False)[0].float() if grad == "accumulate" else None
                weight = torch.nn.Parameter(w.clone())
                if grad != "bf16":
                    weight.main_grad = old.clone() if old is not None else torch.full((N, K), float("nan"), device="cuda")
                    weight.main_grad_fresh = grad == "fresh"
                x = xs[rank].clone().requires_grad_(True)
                eps = (ws.nv_ag_epoch + ws.nv_rs_epoch, ws.ag_epoch + ws.rs_calls)
                n0 = _ext.launches()
                y = _TPLinear.apply(x, weight, bias, "gather" if column else "none", "none" if column else "scatter", 0,
                                    group, None, True, col_scale if column else None)
                y.backward(gys[rank])
                after = None
                if not column:                  # the next all-gather right after a Row+SP backward (side-stream wgrad reader)
                    after = ins((rows, 264))
                    a_b = ins((136, 264), False)[0]
                    after = (after, a_b, ws.ag_gemm(after[rank], a_b, True)[0])
                k = 0 if path == "nvls" else 1
                now = (ws.nv_ag_epoch + ws.nv_rs_epoch, ws.ag_epoch + ws.rs_calls)
                chk.true(now[k] - eps[k] == 2 + (after is not None) and _ext.launches() - n0 >= 3,
                         what + ": the fused kernels did not run")
                results.append((what, column, rows, N, K, xs, gys, w, bias, old, col_scale, grad, y.detach(),
                                x.grad, weight.grad if grad == "bf16" else weight.main_grad.clone(), after))
                chk.true((weight.grad is None) == (grad != "bf16"), what + ": fused weight-gradient epilogue not used")
    torch.cuda.synchronize()
    for (what, column, rows, N, K, xs, gys, w, bias, old, col_scale, grad, y, dx, dw, after) in results:
        if column:
            full = torch.cat(xs)
            want_y = _acc(full, w, False, True).to(BF16)
            gd = [g.clone() for g in gys]
            if col_scale is not None:
                for g in gd:
                    g[..., col_scale[0]:] *= col_scale[1]
            parts = [_acc(g, w, False, False)[rank * rows:(rank + 1) * rows].to(BF16) for g in gd]
            want_dx = _emulate(parts, range(world)).to(BF16)
            acc_w = _acc(gys[rank], full, True, False)
            gy = gys[rank]
        else:
            parts = [_acc(x, w, False, True)[rank * rows:(rank + 1) * rows].to(BF16) for x in xs]
            want_y = _emulate(parts, range(world)).to(BF16)
            g_full = torch.cat(gys)
            want_dx = _acc(g_full, w, False, False).to(BF16)
            acc_w = _acc(g_full, xs[rank], True, False)
            gy = gys[rank]
        if bias is not None:
            want_y = want_y + bias.detach()
            chk.same(bias.grad, gy.float().sum(0).to(BF16), what + ": bias grad")
        chk.same(y, want_y, what + ": y")
        chk.same(dx, want_dx, what + ": dx")
        want_w = acc_w.to(BF16) if grad == "bf16" else acc_w if grad == "fresh" else old + acc_w
        chk.same(dw, want_w, what + ": dW / main_grad")
        if after is not None:
            a_in, a_b, a_out = after
            chk.same(a_out, _acc(torch.cat(a_in), a_b, False, True).to(BF16), what + ": the all-gather after the backward")
        # float64: y and dW within their bounds (dx and the reduce-scatter outputs are covered by the kernel-level test)
        w_ref, w_mag = _op64(gy if column else torch.cat(gys), torch.cat(xs) if column else xs[rank], True, False)
        e_w = _gemm_err(world * rows, w_mag)
        if grad == "bf16":
            e_w = e_w + U_BF16 * (w_ref.abs() + e_w)
        elif grad == "accumulate":
            w_ref = w_ref + old.to(F64)
            e_w = e_w + U * (w_ref.abs() + e_w)
        chk.true(bool(((dw.to(F64) - w_ref).abs() <= e_w).all()), what + ": dW outside its float64 bound")
    chk.settle()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_tp_linear_sequence_parallel_fused_bit_exact(world):
    run_distributed(_layer_worker, world, use_cuda="loopback", timeout=300)


# =====================================================================================================================
# selection: when the fused path is refused, without any launch
# =====================================================================================================================
class _FakeWorkspace:
    """Stands in for TPWorkspace in ``select``: reports whether the group has the NVLS kernels and can launch nothing."""

    def __init__(self, nvls):
        self.nvls, self.group, self.world = nvls, None, 2

    def nvls_enabled(self):
        return self.nvls


@pytest.fixture
def fake_group(monkeypatch):
    from neuronx_distributed_b200.ops import _ext, _fused_impl

    state = types.SimpleNamespace(world=2, nvls=False)
    monkeypatch.setattr(_fused_impl, "dist", types.SimpleNamespace(get_world_size=lambda g: state.world))
    monkeypatch.setattr(_fused_impl, "workspace", lambda g: _FakeWorkspace(state.nvls))
    monkeypatch.setattr(_fused_impl, "_LOGGED", set())
    _ext.ext()
    return state


def _bf(*shape):
    return torch.zeros(shape, dtype=BF16, device="cuda")


@pytest.mark.gpu
def test_fused_tp_selection_refusals_launch_nothing(fake_group):
    from neuronx_distributed_b200.ops import _ext, _fused_impl

    sel = _fused_impl.select
    n0 = _ext.launches()
    refusals = [
        ("rows per rank not a multiple of 128", lambda: sel(_bf(200, 64), _bf(256, 64), "gather", "none", 0, None)),
        ("Row+SP rows per rank not a multiple of 128", lambda: sel(_bf(2 * 192, 64), _bf(256, 64), "none", "scatter", 0, None)),
        ("N not a multiple of 8", lambda: sel(_bf(128, 64), _bf(260, 64), "gather", "none", 0, None)),
        ("K not a multiple of 8", lambda: sel(_bf(128, 68), _bf(256, 68), "gather", "none", 0, None)),
        ("fp32 input", lambda: sel(torch.zeros(128, 64, device="cuda"), _bf(256, 64), "gather", "none", 0, None)),
        ("fp16 weight", lambda: sel(_bf(128, 64), _bf(256, 64).half(), "none", "scatter", 0, None)),
        ("seq_dim 1", lambda: sel(_bf(1, 128, 64), _bf(256, 64), "gather", "none", 1, None)),
        ("65 blocks without NVLS", lambda: sel(_bf(8320, 64), _bf(256, 64), "gather", "none", 0, None)),
    ]
    for what, f in refusals:
        logged = len(_fused_impl._LOGGED)
        assert f() is None, what
        assert len(_fused_impl._LOGGED) == logged + 1, f"{what}: not logged"
        assert f() is None and len(_fused_impl._LOGGED) == logged + 1, f"{what}: logged twice"
    fake_group.world = 9
    assert sel(_bf(128, 64), _bf(256, 64), "gather", "none", 0, None) is None, "world 9"
    fake_group.world = 2
    assert _ext.launches() == n0
    # accepted: 64 blocks per rank on either path, 65 and more with NVLS
    assert isinstance(sel(_bf(8192, 64), _bf(256, 64), "gather", "none", 0, None), _fused_impl._ColumnSP)
    assert isinstance(sel(_bf(2 * 8192, 64), _bf(256, 64), "none", "scatter", 0, None), _fused_impl._RowSP)
    fake_group.nvls = True
    assert isinstance(sel(_bf(8320, 64), _bf(256, 64), "gather", "none", 0, None), _fused_impl._ColumnSP)
    assert _ext.launches() == n0


@pytest.mark.gpu
def test_fused_tp_not_selected_under_graph_capture(fake_group):
    """A captured call would bake its epochs, counter targets and claim base into the graph: replays would read stale
    partials without waiting.  ``dispatch`` refuses the fused path while the current stream captures."""
    from neuronx_distributed_b200.ops import _ext, _fused_impl, tp_fused

    x, w = _bf(256, 64), _bf(256, 64)
    assert isinstance(tp_fused.dispatch(x, w, "gather", "none", 0, None), _fused_impl._ColumnSP)
    n0 = _ext.launches()
    graph, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            got = [tp_fused.dispatch(x, w, kind[0], kind[1], 0, None) for kind in (("gather", "none"), ("none", "scatter"))]
            x.add_(1)
    torch.cuda.synchronize()
    assert got == [None, None]
    assert _ext.launches() == n0
    assert any("capture" in k for k in _fused_impl._LOGGED)


def test_all_gather_comm_cta_count_is_checked():
    from neuronx_distributed_b200.ops._fused_impl import checked_comm_sms

    for ok in (1, 16, 131):
        assert checked_comm_sms(ok, 132) == ok
    for bad in (0, -1, 132, 200):
        with pytest.raises(ValueError):
            checked_comm_sms(bad, 132)
